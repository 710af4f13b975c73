"""Non-grid interaction modules with the reference's constructors, parameters and plug signature
(trajnetbaselines/lstm/non_gridbased_pooling.py).

Built: HiddenStateMLPPooling (:150-239, `--type hiddenstatemlp`, the Social-GAN pooling): max over the
scene of per-neighbour embeddings of relative position, hidden state and relative velocity, then a linear
projection.  One kernel per step (csrc/mlp_pool.cu); same plug contract as GridBasedPooling (attribute
`out_dim`, `reset(...)`, `__call__(hidden [B, N, H], obs1, obs2) -> [B * N, out_dim]`).  Inside
`LSTM.forward` the module is not called -- the fused sequence entry point reads its parameters.

NearestNeighborMLP (:64-147, `--type nn`): relative position (and velocity) of the n nearest tracks, each through a
shared Linear + ReLU, concatenated.  One kernel per step (nn_mlp_pool_kernel in csrc/mlp_pool.cu).

AttentionMLPPooling (:242-351, `--type attentionmlp`): the embeddings of HiddenStateMLPPooling, wq / wk / wv and a
one-head torch.nn.MultiheadAttention over all slots of the scene, out_projection (attn_mlp_pool_kernel).

NearestNeighborLSTM (:354-451, `--type nn_lstm`): the NearestNeighborMLP features drive a per-track LSTMCell whose state
persists over the steps of a forward (nn_mlp_pool_kernel + pool_lstm_cell_kernel); the state lives in the model handle's
workspace, `reset()` zeroes it.

TrajectronPooling (:454-537, `--type traj_pool`): own (pos, vel) and the sum over the other visible tracks, embedded, then
the same per-track LSTMCell / hidden2pool (traj_scene_sum_kernel + traj_feat_kernel + pool_lstm_cell_kernel).

"""
import torch

from .. import _lib
from ..engine import PoolPlug


class HiddenStateMLPPooling(PoolPlug):
    _reads_hidden = True

    def __init__(self, hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=None):
        """Same arguments and sub-module names as the reference (non_gridbased_pooling.py:166-193)."""
        super().__init__()
        self.out_dim = out_dim or hidden_dim
        self.hidden_dim = hidden_dim
        self.mlp_dim = mlp_dim
        self.mlp_dim_spatial = mlp_dim_spatial
        self.mlp_dim_vel = mlp_dim_vel
        self.mlp_dim_hidden = mlp_dim - mlp_dim_spatial - mlp_dim_vel
        if self.mlp_dim_spatial < 1 or self.mlp_dim_vel < 0 or self.mlp_dim_hidden < 0:
            raise ValueError("mlp_dim must cover mlp_dim_spatial (>= 1) + mlp_dim_vel")
        self.spatial_embedding = torch.nn.Sequential(torch.nn.Linear(2, self.mlp_dim_spatial), torch.nn.ReLU())
        if self.mlp_dim_vel:
            self.vel_embedding = torch.nn.Sequential(torch.nn.Linear(2, self.mlp_dim_vel), torch.nn.ReLU())
        if self.mlp_dim_hidden:
            self.hidden_embedding = torch.nn.Sequential(torch.nn.Linear(self.hidden_dim, self.mlp_dim_hidden), torch.nn.ReLU())
        self.out_projection = torch.nn.Linear(self.mlp_dim, self.out_dim)

    # -- configuration shared with LSTM ---------------------------------------------------------
    def fill_config(self, cfg):
        cfg.pool_type = _lib.POOL_HIDDEN_MLP
        cfg.out_dim = int(self.out_dim)
        cfg.mlp_dim_spatial = int(self.mlp_dim_spatial)
        cfg.mlp_dim_vel = int(self.mlp_dim_vel)
        cfg.mlp_dim_hidden = int(self.mlp_dim_hidden)

    def weight_fields(self):
        fields = dict(pool_spatial_weight=self.spatial_embedding[0].weight, pool_spatial_bias=self.spatial_embedding[0].bias,
                      pool_out_weight=self.out_projection.weight, pool_out_bias=self.out_projection.bias)
        if self.mlp_dim_vel:
            fields.update(pool_vel_weight=self.vel_embedding[0].weight, pool_vel_bias=self.vel_embedding[0].bias)
        if self.mlp_dim_hidden:
            fields.update(pool_hidden_weight=self.hidden_embedding[0].weight, pool_hidden_bias=self.hidden_embedding[0].bias)
        return fields


class NearestNeighborMLP(PoolPlug):
    def __init__(self, n=4, out_dim=32, no_vel=False):
        """Same arguments and sub-module names as the reference (non_gridbased_pooling.py:78-91)."""
        super().__init__()
        if n < 1 or n > 32 or out_dim % n != 0:
            raise ValueError("NearestNeighborMLP needs 1 <= n <= 32 and n dividing out_dim (reference :87-88)")
        self.n = n
        self.out_dim = out_dim
        self.no_velocity = no_vel
        self.input_dim = 2 if self.no_velocity else 4
        self.embedding = torch.nn.Sequential(torch.nn.Linear(self.input_dim, int(out_dim / self.n)), torch.nn.ReLU())

    def fill_config(self, cfg):
        cfg.pool_type = _lib.POOL_NN_MLP
        cfg.n = int(self.n)
        cfg.out_dim = int(self.out_dim)
        cfg.mlp_dim_spatial = int(self.out_dim // self.n)
        cfg.mlp_dim_vel = 0 if self.no_velocity else 1
        cfg.mlp_dim_hidden = 0

    def weight_fields(self):
        return dict(pool_spatial_weight=self.embedding[0].weight, pool_spatial_bias=self.embedding[0].bias)


class AttentionMLPPooling(PoolPlug):
    _reads_hidden = True

    def __init__(self, hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=None, fill_value=-10):
        """Same arguments, sub-module names and parameters as the reference (non_gridbased_pooling.py:257-292)."""
        super().__init__()
        self.out_dim = out_dim or hidden_dim
        self.hidden_dim = hidden_dim
        self.fill_value = fill_value
        self.mlp_dim = mlp_dim
        self.mlp_dim_spatial = mlp_dim_spatial
        self.mlp_dim_vel = mlp_dim_vel
        self.mlp_dim_hidden = mlp_dim - mlp_dim_spatial - mlp_dim_vel
        if self.mlp_dim_spatial < 1 or self.mlp_dim_vel < 0 or self.mlp_dim_hidden < 0 or mlp_dim > 128:
            raise ValueError("mlp_dim (<= 128) must cover mlp_dim_spatial (>= 1) + mlp_dim_vel")
        self.spatial_embedding = torch.nn.Sequential(torch.nn.Linear(2, self.mlp_dim_spatial), torch.nn.ReLU())
        if self.mlp_dim_vel:
            self.vel_embedding = torch.nn.Sequential(torch.nn.Linear(2, self.mlp_dim_vel), torch.nn.ReLU())
        if self.mlp_dim_hidden:
            self.hidden_embedding = torch.nn.Sequential(torch.nn.Linear(self.hidden_dim, self.mlp_dim_hidden), torch.nn.ReLU())
        self.wq = torch.nn.Linear(self.mlp_dim, self.mlp_dim, bias=False)
        self.wk = torch.nn.Linear(self.mlp_dim, self.mlp_dim, bias=False)
        self.wv = torch.nn.Linear(self.mlp_dim, self.mlp_dim, bias=False)
        self.multihead_attn = torch.nn.MultiheadAttention(embed_dim=self.mlp_dim, num_heads=1)
        self.out_projection = torch.nn.Linear(self.mlp_dim, self.out_dim)

    def fill_config(self, cfg):
        cfg.pool_type = _lib.POOL_ATTN_MLP
        cfg.out_dim = int(self.out_dim)
        cfg.mlp_dim_spatial = int(self.mlp_dim_spatial)
        cfg.mlp_dim_vel = int(self.mlp_dim_vel)
        cfg.mlp_dim_hidden = int(self.mlp_dim_hidden)
        cfg.attn_fill = float(self.fill_value)

    def weight_fields(self):
        fields = dict(pool_spatial_weight=self.spatial_embedding[0].weight, pool_spatial_bias=self.spatial_embedding[0].bias,
                      pool_out_weight=self.out_projection.weight, pool_out_bias=self.out_projection.bias,
                      pool_attn_wq=self.wq.weight, pool_attn_wk=self.wk.weight, pool_attn_wv=self.wv.weight,
                      pool_attn_in_proj_weight=self.multihead_attn.in_proj_weight,
                      pool_attn_in_proj_bias=self.multihead_attn.in_proj_bias,
                      pool_attn_out_proj_weight=self.multihead_attn.out_proj.weight,
                      pool_attn_out_proj_bias=self.multihead_attn.out_proj.bias)
        if self.mlp_dim_vel:
            fields.update(pool_vel_weight=self.vel_embedding[0].weight, pool_vel_bias=self.vel_embedding[0].bias)
        if self.mlp_dim_hidden:
            fields.update(pool_hidden_weight=self.hidden_embedding[0].weight, pool_hidden_bias=self.hidden_embedding[0].bias)
        return fields


class NearestNeighborLSTM(PoolPlug):
    stateful = True

    def __init__(self, n=4, hidden_dim=256, out_dim=32):
        """Same arguments and sub-module names as the reference (non_gridbased_pooling.py:371-383)."""
        super().__init__()
        if n < 1 or n > 32 or out_dim % n != 0 or hidden_dim > 512 or out_dim > 1024:
            raise ValueError("NearestNeighborLSTM needs 1 <= n <= 32, n dividing out_dim, hidden_dim <= 512, out_dim <= 1024")
        self.n = n
        self.out_dim = out_dim
        self.input_dim = 4
        self.embedding = torch.nn.Sequential(torch.nn.Linear(self.input_dim, int(out_dim / self.n)), torch.nn.ReLU())
        self.hidden_dim = hidden_dim
        self.pool_lstm = torch.nn.LSTMCell(out_dim, hidden_dim)
        self.hidden2pool = torch.nn.Linear(hidden_dim, out_dim)
        self._reset_pending = True

    def fill_config(self, cfg):
        cfg.pool_type = _lib.POOL_NN_LSTM
        cfg.n = int(self.n)
        cfg.out_dim = int(self.out_dim)
        cfg.mlp_dim_spatial = int(self.out_dim // self.n)
        cfg.mlp_dim_vel = 1
        cfg.mlp_dim_hidden = int(self.hidden_dim)

    def weight_fields(self):
        return dict(pool_spatial_weight=self.embedding[0].weight, pool_spatial_bias=self.embedding[0].bias,
                    pool_lstm_weight_ih=self.pool_lstm.weight_ih, pool_lstm_weight_hh=self.pool_lstm.weight_hh,
                    pool_lstm_bias_ih=self.pool_lstm.bias_ih, pool_lstm_bias_hh=self.pool_lstm.bias_hh,
                    pool_out_weight=self.hidden2pool.weight, pool_out_bias=self.hidden2pool.bias)

    def reset(self, num_tracks, max_num_neigh, device):
        """Reference: fresh zero state per track (non_gridbased_pooling.py:385-389); here the state of the stand-alone plug
        lives in the handle's workspace and is zeroed before the next call (LSTM.forward zeroes its own)."""
        self._reset_pending = True

    def _plug_state(self, handle, layout):
        """A plug call advances the interaction-encoder state (non_gridbased_pooling.py:391-451)."""
        if self._reset_pending:
            handle.pool_state_reset(layout)
            self._reset_pending = False
            self._state_tracks = layout.num_tracks
        elif getattr(self, '_state_tracks', None) != layout.num_tracks:
            # the reference stacks `num_tracks` state rows from reset() against B * N feature rows and fails the same way
            raise RuntimeError("the interaction-encoder state holds %s tracks, this call has %d: call reset(num_tracks, ...)"
                               % (getattr(self, '_state_tracks', None), layout.num_tracks))


class TrajectronPooling(NearestNeighborLSTM):
    def __init__(self, n=4, hidden_dim=256, out_dim=32, track_mask=None):
        """Same arguments and sub-module names as the reference (non_gridbased_pooling.py:468-479; `n` is unused there)."""
        PoolPlug.__init__(self)
        if hidden_dim > 512 or out_dim > 1024:
            raise ValueError("TrajectronPooling needs hidden_dim <= 512 and out_dim <= 1024")
        self.n = n
        self.out_dim = out_dim
        self.embedding = torch.nn.Sequential(torch.nn.Linear(8, out_dim), torch.nn.ReLU())
        self.hidden_dim = hidden_dim
        self.pool_lstm = torch.nn.LSTMCell(out_dim, hidden_dim)
        self.hidden2pool = torch.nn.Linear(hidden_dim, out_dim)
        self.track_mask = track_mask
        self._reset_pending = True

    def fill_config(self, cfg):
        cfg.pool_type = _lib.POOL_TRAJECTRON
        cfg.n = int(self.n)
        cfg.out_dim = int(self.out_dim)
        cfg.mlp_dim_spatial = int(self.out_dim)
        cfg.mlp_dim_vel = 1
        cfg.mlp_dim_hidden = int(self.hidden_dim)
