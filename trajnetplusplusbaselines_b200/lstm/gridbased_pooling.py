"""GridBasedPooling with the reference's constructor, parameters and plug signature.

Mirrors trajnetbaselines/lstm/gridbased_pooling.py (GridBasedPooling :15-400).  The pool plug
contract the LSTM relies on (SURVEY.md 8b/B1): attribute `out_dim`, `reset(...)`, and
`__call__(hidden_state [B, N, H], obs1 [B, N, 2], obs2 [B, N, 2]) -> [B * N, out_dim]`.
The grid construction and its embedding MLP run in csrc/pool.cu; inside `LSTM.forward` the
pool is not even called -- the fused sequence entry point consumes its parameters directly.
"""
import torch

from .. import _lib
from ..engine import PoolPlug

_TYPES = {'occupancy': _lib.POOL_OCCUPANCY, 'directional': _lib.POOL_DIRECTIONAL,
          'social': _lib.POOL_SOCIAL}
_ARCH_LAYERS = {'None': 0, None: 0, 'one_layer': 1, 'two_layer': 2, 'three_layer': 3}


class GridBasedPooling(PoolPlug):
    def __init__(self, cell_side=2.0, n=4, hidden_dim=128, out_dim=None,
                 type_='occupancy', pool_size=1, blur_size=1, front=False,
                 embedding_arch='one_layer', pretrained_pool_encoder=None,
                 constant=0, norm=0, layer_dims=None, latent_dim=16):
        super().__init__()
        if type_ not in _TYPES:
            raise NotImplementedError("type_=%r is not built (reference CLI reaches only occupancy / "
                                      "directional / social, lstm/trainer.py:340-343)" % (type_,))
        if embedding_arch not in _ARCH_LAYERS:
            raise NotImplementedError("embedding_arch=%r is not built ('lstm_layer' is dead code at the "
                                      "reference HEAD, gridbased_pooling.py:94-110)" % (embedding_arch,))
        if pretrained_pool_encoder is not None:
            raise NotImplementedError("pretrained_pool_encoder is not built")
        if pool_size != 1 or blur_size != 1:
            raise NotImplementedError("pool_size / blur_size != 1 are not built (never set by the "
                                      "reference CLI, lstm/trainer.py:483-487)")
        self.cell_side = cell_side
        self.n = n
        self.type_ = type_
        self.pool_size = pool_size
        self.blur_size = blur_size
        self.norm_pool = False
        self.front = front
        if self.front:
            self.norm_pool = True
        self.constant = constant
        self.norm = norm
        self.pool_scale = 1.0
        self.hidden_dim = hidden_dim
        self.latent_dim = latent_dim

        self.pooling_dim = 1
        if self.type_ == 'directional':
            self.pooling_dim = 2
        if self.type_ == 'social':
            self.hidden_dim_encoding = torch.nn.Linear(hidden_dim, latent_dim)
            self.pooling_dim = latent_dim

        if out_dim is None:
            out_dim = hidden_dim
        self.out_dim = out_dim
        self.pretrained_model = None

        self.embedding = None
        self.embedding_arch = embedding_arch
        self.layer_dims = list(layer_dims) if layer_dims is not None else None
        input_dim = self.n * self.n * self.pooling_dim
        n_layers = _ARCH_LAYERS[embedding_arch]
        if n_layers:
            if n_layers > 1 and (layer_dims is None or len(layer_dims) < n_layers - 1):
                raise ValueError("layer_dims must hold %d widths for %s" % (n_layers - 1, embedding_arch))
            dims = [input_dim] + [int(d) for d in (layer_dims or [])[:n_layers - 1]] + [self.out_dim]
            mods = []
            for i in range(n_layers):
                mods += [torch.nn.Linear(dims[i], dims[i + 1]), torch.nn.ReLU()]
            self.embedding = torch.nn.Sequential(*mods)

    # -- configuration shared with LSTM ---------------------------------------------------------
    def fill_config(self, cfg):
        """Write the pooling fields of a tb2_lstm_config."""
        cfg.pool_type = _TYPES[self.type_]
        cfg.n = int(self.n)
        cfg.cell_side = float(self.cell_side / self.pool_size)
        cfg.pool_size = int(self.pool_size)
        cfg.blur_size = int(self.blur_size)
        cfg.front = int(bool(self.front))
        cfg.constant = float(self.constant)
        cfg.latent_dim = int(self.latent_dim)
        n_layers = _ARCH_LAYERS[self.embedding_arch]
        cfg.num_layers = n_layers
        for i in range(2):
            cfg.layer_dims[i] = int(self.layer_dims[i]) if (self.layer_dims and i < min(len(self.layer_dims), n_layers - 1)) else 0
        cfg.out_dim = int(self.out_dim)

    def weight_fields(self):
        fields = {}
        if self.type_ == 'social':
            fields['pool_encoding_weight'] = self.hidden_dim_encoding.weight
            fields['pool_encoding_bias'] = self.hidden_dim_encoding.bias
        if self.embedding is not None:
            linears = [m for m in self.embedding if isinstance(m, torch.nn.Linear)]
            fields['pool_embedding_weight'] = [l.weight for l in linears]
            fields['pool_embedding_bias'] = [l.bias for l in linears]
        return fields

    # -- the plug (gridbased_pooling.py:94-110; reset: the reference resets its dead pool-LSTM state, :345-351) -------
    @property
    def _reads_hidden(self):
        return self.type_ == 'social'

    def _plug_out_dim(self):
        return int(self.out_dim if self.embedding is not None else self.n * self.n * self.pooling_dim)

    def _plug_device(self, obs1):
        params = list(self.parameters())
        device = params[0].device if params else obs1.device
        if device.type != 'cuda':
            if obs1.device.type == 'cuda':
                device = obs1.device
            elif not params:      # nothing to .cuda(): parameter-free grid on host inputs
                device = torch.device('cuda', torch.cuda.current_device())
            else:
                raise RuntimeError("GridBasedPooling runs on CUDA only: move the module (or inputs) to the GPU")
        return device
