"""numpy (fp32) restatement of the reference LSTM hot path -- TEST INFRASTRUCTURE.

Restates, function by function, what the reference computes (all paths relative to
/root/reference/trajnetbaselines/):

  grid_cells          lstm/gridbased_pooling.py:248-249,257-263,273-287  (binning)
  occupancy_grid      lstm/gridbased_pooling.py:227-305                  (scatter-overwrite)
  pool_forward        lstm/gridbased_pooling.py:94-110,112-170,308-335
  input_embedding     lstm/modules.py:24-30
  hidden2normal       lstm/modules.py:56-64
  lstm_cell           torch.nn.LSTMCell as used at lstm/lstm.py:84-85,154
  step                lstm/lstm.py:91-168 (+ generate_pooling_inputs :25-42)
  forward             lstm/lstm.py:170-264 (decoder input rule :240-250)
  prediction_loss     lstm/loss.py:24-91
  ade_fde             evaluator/eval_utils.py:3-19

The arithmetic is float32 throughout, like the reference run on CPU.  Weights are a
dict keyed by the reference's state_dict names (SURVEY.md section 8b, B2).
Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs use this.
"""
import math

import numpy as np

F32 = np.float32
NAN = float("nan")


class PoolConfig:
    """Constructor arguments of GridBasedPooling (gridbased_pooling.py:16-19)."""

    def __init__(self, type_="occupancy", cell_side=2.0, n=4, hidden_dim=128, out_dim=None,
                 pool_size=1, blur_size=1, front=False, embedding_arch="one_layer",
                 constant=0, norm=0, layer_dims=None, latent_dim=16):
        self.type_ = type_
        self.cell_side = cell_side
        self.n = n
        self.hidden_dim = hidden_dim
        self.out_dim = hidden_dim if out_dim is None else out_dim
        self.pool_size = pool_size
        self.blur_size = blur_size
        self.front = front
        self.embedding_arch = embedding_arch
        self.constant = constant
        self.norm = norm
        self.layer_dims = layer_dims
        self.latent_dim = latent_dim
        # gridbased_pooling.py:57-67
        self.pooling_dim = {"occupancy": 1, "directional": 2, "social": latent_dim,
                            "dir_social": latent_dim + 2}[type_]


class MlpPoolConfig:
    """Constructor arguments of HiddenStateMLPPooling (non_gridbased_pooling.py:166-193)."""

    def __init__(self, hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=None):
        self.type_ = "hiddenstatemlp"
        self.hidden_dim = hidden_dim
        self.mlp_dim = mlp_dim
        self.mlp_dim_spatial = mlp_dim_spatial
        self.mlp_dim_vel = mlp_dim_vel
        self.mlp_dim_hidden = mlp_dim - mlp_dim_spatial - mlp_dim_vel
        self.out_dim = hidden_dim if out_dim is None else out_dim


class AttnPoolConfig:
    """Constructor arguments of AttentionMLPPooling (non_gridbased_pooling.py:257-292)."""

    def __init__(self, hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=None, fill_value=-10):
        self.type_ = "attentionmlp"
        self.hidden_dim = hidden_dim
        self.mlp_dim = mlp_dim
        self.mlp_dim_spatial = mlp_dim_spatial
        self.mlp_dim_vel = mlp_dim_vel
        self.mlp_dim_hidden = mlp_dim - mlp_dim_spatial - mlp_dim_vel
        self.out_dim = hidden_dim if out_dim is None else out_dim
        self.fill_value = fill_value


class NnLstmPoolConfig:
    """Constructor arguments of NearestNeighborLSTM (non_gridbased_pooling.py:371-383)."""

    def __init__(self, n=4, hidden_dim=256, out_dim=32):
        self.type_ = "nn_lstm"
        self.n = n
        self.hidden_dim = hidden_dim
        self.out_dim = out_dim
        self.no_vel = False
        self.input_dim = 4


class TrajectronPoolConfig:
    """Constructor arguments of TrajectronPooling (non_gridbased_pooling.py:468-479; `n` is unused there)."""

    def __init__(self, n=4, hidden_dim=256, out_dim=32):
        self.type_ = "traj_pool"
        self.n = n
        self.hidden_dim = hidden_dim
        self.out_dim = out_dim


class NnPoolConfig:
    """Constructor arguments of NearestNeighborMLP (non_gridbased_pooling.py:78-91)."""

    def __init__(self, n=4, out_dim=32, no_vel=False):
        self.type_ = "nn"
        self.n = n
        self.out_dim = out_dim
        self.no_vel = no_vel
        self.input_dim = 2 if no_vel else 4


def _sigmoid(x):
    x = np.asarray(x, dtype=F32)
    return (F32(1.0) / (F32(1.0) + np.exp(-x, dtype=F32))).astype(F32)


def _linear(x, w, b):
    """torch.nn.Linear: x @ w.T + b in fp32."""
    return (x.astype(F32) @ w.astype(F32).T + b.astype(F32)).astype(F32)


# ----------------------------------------------------------------------------------------
# grid binning + scatter (gridbased_pooling.py:227-305)
# ----------------------------------------------------------------------------------------
def grid_cells(obs, cfg):
    """Cell index of every ordered pair (i, j != i) of a padded batch.

    obs [B, N, 2] fp32, NaN = absent / padded.  Returns (oi int64 [B, N, N-1],
    in_range bool [B, N, N-1]); neighbour slot jj of row i is j = jj + (jj >= i)
    (diagonal removed, gridbased_pooling.py:261-263).  Out-of-range pairs get index 0
    (gridbased_pooling.py:281).
    """
    obs = np.array(obs, dtype=F32, copy=True)
    B, N, _ = obs.shape
    absent = np.isnan(obs).any(axis=-1)                      # :248
    obs[absent] = F32(-500.0)                                # :249
    rel = obs[:, None, :, :] - obs[:, :, None, :]            # :257-258  rel[b,i,j] = x_j - x_i
    keep = ~np.eye(N, dtype=bool)
    rel = rel[:, keep].reshape(B, N, N - 1, 2)               # :261-263
    side = F32(cfg.cell_side / cfg.pool_size)                # python double -> fp32 scalar
    width = cfg.n * cfg.pool_size
    if cfg.front:                                            # :273-274
        off = np.array([width / 2, 0], dtype=F32)
    else:                                                    # :276
        off = np.array([width / 2, width / 2], dtype=F32)
    oij = (rel / side).astype(F32) + off                     # fp32 true division, fp32 add
    in_range = ~(((oij < 0) | (oij >= F32(width))).any(axis=-1))   # :278-279
    oij = np.where(in_range[..., None], oij, F32(0.0))       # :281
    oij_l = oij.astype(np.int64)                             # :284 truncation
    oi = oij_l[..., 0] * cfg.n * cfg.pool_size + oij_l[..., 1]     # :287
    return oi, in_range


def occupancy_grid(obs, other_values, cfg):
    """gridbased_pooling.py:227-305 -> [B*N, C, n, n] fp32.

    other_values [B, N, N-1, C] or None (occupancy: ones).  Scatter is an OVERWRITE in
    ascending neighbour order (index_put_ at :293); out-of-range neighbours write
    `constant` into cell 0 in that same order (:281-282).
    """
    obs = np.asarray(obs, dtype=F32)
    B, N, _ = obs.shape
    C = cfg.pooling_dim
    width = cfg.n * cfg.pool_size
    const = F32(cfg.constant)
    if N == 1:                                               # :252-253 (per row; ref: B == 1 only)
        return np.full((B, C, cfg.n, cfg.n), const, dtype=F32)
    oi, in_range = grid_cells(obs, cfg)
    if other_values is None:                                 # :266-267
        other_values = np.ones((B, N, N - 1, C), dtype=F32)
    vals = np.where(in_range[..., None], other_values.astype(F32), const)   # :282
    vals = vals.reshape(B * N, N - 1, C)
    oi = oi.reshape(B * N, N - 1)
    occ = np.full((B * N, width * width, C), const, dtype=F32)              # :290
    rows = np.arange(B * N)
    for jj in range(N - 1):                                  # :293, explicit ascending-j overwrite
        occ[rows, oi[:, jj]] = vals[:, jj]
    occ2d = occ.transpose(0, 2, 1).reshape(B * N, C, width, width)          # :294-295
    if cfg.blur_size != 1:                                   # :300-301 avg_pool2d(k, 1, k//2, include pad)
        k = cfg.blur_size
        p = k // 2
        padded = np.zeros((B * N, C, width + 2 * p, width + 2 * p), dtype=F32)
        padded[:, :, p:p + width, p:p + width] = occ2d
        out_w = width + 2 * p - k + 1
        acc = np.zeros((B * N, C, out_w, out_w), dtype=F32)
        for dx in range(k):
            for dy in range(k):
                acc += padded[:, :, dx:dx + out_w, dy:dy + out_w]
        occ2d = (acc / F32(k * k)).astype(F32)
        width_b = out_w
    else:
        width_b = width
    ps = cfg.pool_size                                       # :303 lp_pool2d(p=1) = window sum
    if ps != 1:
        nw = width_b // ps
        occ2d = occ2d[:, :, :nw * ps, :nw * ps].reshape(B * N, C, nw, ps, nw, ps).sum(axis=(3, 5))
        occ2d = occ2d.astype(F32)
    return occ2d


def pair_values(cfg, weights, hidden, obs1, obs2, prefix="pool."):
    """Per-pair payload (gridbased_pooling.py:112-170).  None for plain occupancy."""
    B, N, _ = obs2.shape
    keep = ~np.eye(N, dtype=bool)
    vals = []
    if cfg.type_ in ("directional", "dir_social"):           # :131-140
        vel = (obs2 - obs1).astype(F32)
        rel = vel[:, None, :, :] - vel[:, :, None, :]
        rel = rel[:, keep].reshape(B, N, N - 1, 2)
        vals.append(np.nan_to_num(rel, nan=0.0).astype(F32))
    if cfg.type_ in ("social", "dir_social"):                # :160-167
        h = np.broadcast_to(hidden[:, None, :, :], (B, N, N, hidden.shape[-1]))
        h = h[:, keep].reshape(B, N, N - 1, -1)
        h = np.nan_to_num(h, nan=0.0).astype(F32)
        lat = _linear(h.reshape(-1, h.shape[-1]), weights[prefix + "hidden_dim_encoding.weight"],
                      weights[prefix + "hidden_dim_encoding.bias"])
        vals.append(lat.reshape(B, N, N - 1, -1))
    if not vals:
        return None
    return np.concatenate(vals, axis=-1) if len(vals) > 1 else vals[0]


def embed_grid(cfg, weights, grid, prefix="pool."):
    """gridbased_pooling.py:308-335 (one/two/three_layer), 'None' = raw grid."""
    x = grid.astype(F32)
    if cfg.embedding_arch in (None, "None"):
        return x
    n_layers = {"one_layer": 1, "two_layer": 2, "three_layer": 3}[cfg.embedding_arch]
    for l in range(n_layers):
        x = _linear(x, weights[prefix + "embedding.%d.weight" % (2 * l)],
                    weights[prefix + "embedding.%d.bias" % (2 * l)])
        x = np.maximum(x, F32(0.0))
    return x


def _embed_with_masking(x, w, b, fill=-100.0):
    """embed_with_masking (non_gridbased_pooling.py:49-58): relu(Linear) where no input is NaN, else `fill`."""
    bad = np.isnan(x).any(axis=-1)
    out = np.full(x.shape[:-1] + (w.shape[0],), F32(fill), dtype=F32)
    out[~bad] = np.maximum(_linear(x[~bad].astype(F32), w, b), F32(0.0))
    return out


def hidden_mlp_pool_forward(cfg, weights, hidden, obs1, obs2, prefix="pool."):
    """HiddenStateMLPPooling.forward (non_gridbased_pooling.py:197-239) -> [B*N, out_dim]: max over ALL tracks j of
    the scene (the track itself included) of [spatial(pos_j - pos_i) | hidden(h_j) | vel(4 (v_j - v_i))]."""
    obs1 = np.asarray(obs1, dtype=F32)
    obs2 = np.asarray(obs2, dtype=F32)
    hidden = np.asarray(hidden, dtype=F32)
    B, N, _ = obs2.shape
    rel = obs2[:, None, :, :] - obs2[:, :, None, :]                         # rel_obs :13-23: [b, i, j] = pos_j - pos_i
    parts = [_embed_with_masking(rel, weights[prefix + "spatial_embedding.0.weight"], weights[prefix + "spatial_embedding.0.bias"])]
    if cfg.mlp_dim_hidden:
        hid = _embed_with_masking(hidden, weights[prefix + "hidden_embedding.0.weight"], weights[prefix + "hidden_embedding.0.bias"])
        parts.append(np.broadcast_to(hid[:, None, :, :], (B, N, N, hid.shape[-1])))
    if cfg.mlp_dim_vel:
        vel = obs2 - obs1
        relv = (vel[:, None, :, :] - vel[:, :, None, :]) * F32(4.0)        # rel_directional :26-39, x 4 :233
        parts.append(_embed_with_masking(relv, weights[prefix + "vel_embedding.0.weight"], weights[prefix + "vel_embedding.0.bias"]))
    emb = np.concatenate(parts, axis=-1)
    pooled = emb.max(axis=2)                                                # :237
    return _linear(pooled.reshape(B * N, -1).astype(F32), weights[prefix + "out_projection.weight"],
                   weights[prefix + "out_projection.bias"])


def attn_mlp_pool_forward(cfg, weights, hidden, obs1, obs2, prefix="pool."):
    """AttentionMLPPooling.forward (non_gridbased_pooling.py:297-351) -> [B*N, out_dim].  For track i the sequence is
    the embedding e_ij = [spatial(pos_j - pos_i) | hidden(h_j) | vel(4 (v_j - v_i))] of EVERY slot j of the (padded)
    scene -- NaN inputs become the fill value (-10; 0 for the hidden part), nothing is masked in the attention --,
    query / key / value = wq / wk / wv (no bias) followed by torch.nn.MultiheadAttention (1 head: in-projection with
    bias, softmax(q k^T / sqrt(E)) v, out-projection); the output at sequence position i is kept (:349-350)."""
    obs1 = np.asarray(obs1, dtype=F32)
    obs2 = np.asarray(obs2, dtype=F32)
    hidden = np.asarray(hidden, dtype=F32)
    B, N, _ = obs2.shape
    E = cfg.mlp_dim
    rel = obs2[:, None, :, :] - obs2[:, :, None, :]
    parts = [_embed_with_masking(rel, weights[prefix + "spatial_embedding.0.weight"], weights[prefix + "spatial_embedding.0.bias"],
                                 fill=cfg.fill_value)]
    if cfg.mlp_dim_hidden:
        hid = _embed_with_masking(hidden, weights[prefix + "hidden_embedding.0.weight"], weights[prefix + "hidden_embedding.0.bias"],
                                  fill=0.0)
        parts.append(np.broadcast_to(hid[:, None, :, :], (B, N, N, hid.shape[-1])))
    if cfg.mlp_dim_vel:
        vel = obs2 - obs1
        relv = (vel[:, None, :, :] - vel[:, :, None, :]) * F32(4.0)
        parts.append(_embed_with_masking(relv, weights[prefix + "vel_embedding.0.weight"], weights[prefix + "vel_embedding.0.bias"],
                                         fill=cfg.fill_value))
    emb = np.concatenate(parts, axis=-1).astype(F32)                        # [B, i, j, E]
    zero = np.zeros(E, dtype=F32)
    q = _linear(emb, weights[prefix + "wq.weight"], zero)
    k = _linear(emb, weights[prefix + "wk.weight"], zero)
    v = _linear(emb, weights[prefix + "wv.weight"], zero)
    w_in, b_in = weights[prefix + "multihead_attn.in_proj_weight"], weights[prefix + "multihead_attn.in_proj_bias"]
    q = _linear(q, w_in[:E], b_in[:E]) * F32(math.sqrt(1.0 / E))
    k = _linear(k, w_in[E:2 * E], b_in[E:2 * E])
    v = _linear(v, w_in[2 * E:], b_in[2 * E:])
    idx = np.arange(N)
    qi = q[:, idx, idx, :]                                                   # the query at sequence position i
    scores = np.einsum("bie,bije->bij", qi, k).astype(F32)
    scores = scores - scores.max(axis=-1, keepdims=True)
    w = np.exp(scores, dtype=F32)
    w = (w / w.sum(axis=-1, keepdims=True)).astype(F32)
    att = np.einsum("bij,bije->bie", w, v).astype(F32)
    att = _linear(att, weights[prefix + "multihead_attn.out_proj.weight"], weights[prefix + "multihead_attn.out_proj.bias"])
    return _linear(att.reshape(B * N, E), weights[prefix + "out_projection.weight"], weights[prefix + "out_projection.bias"])


def nn_mlp_pool_forward(cfg, weights, obs1, obs2, prefix="pool."):
    """NearestNeighborMLP.forward (non_gridbased_pooling.py:96-147) -> [B*N, out_dim]: features of the n nearest other
    tracks in ascending distance (NaN distances count as 1000, :131-132; NaN features become 0, :141; fewer than n other
    tracks: zero rows, :134-136), shared Linear + ReLU per neighbour, concatenated."""
    obs1 = np.asarray(obs1, dtype=F32)
    obs2 = np.asarray(obs2, dtype=F32)
    B, N, _ = obs2.shape
    w, b = weights[prefix + "embedding.0.weight"], weights[prefix + "embedding.0.bias"]
    vel = obs2 - obs1
    out = np.zeros((B, N, cfg.n, w.shape[0]), dtype=F32)
    for bi in range(B):
        for i in range(N):
            others = [j for j in range(N) if j != i]
            rel = np.stack([obs2[bi, j] - obs2[bi, i] for j in others]) if others else np.zeros((0, 2), F32)
            relv = np.stack([vel[bi, j] - vel[bi, i] for j in others]) if others else np.zeros((0, 2), F32)
            with np.errstate(invalid="ignore"):
                dist = np.sqrt((rel[:, 0] * rel[:, 0] + rel[:, 1] * rel[:, 1]).astype(F32)).astype(F32)
            dist = np.where(np.isnan(dist), F32(1000.0), dist)
            order = np.argsort(dist, kind="stable")[:cfg.n]                  # torch.topk(-dist): ascending distance
            feats = np.zeros((cfg.n, cfg.input_dim), dtype=F32)
            for k, o in enumerate(order):
                f = rel[o] if cfg.no_vel else np.concatenate([rel[o], relv[o]])
                feats[k] = np.nan_to_num(f.astype(F32))
            out[bi, i] = np.maximum(_linear(feats, w, b), F32(0.0))
    return out.reshape(B * N, -1)


def nn_lstm_pool_forward(cfg, weights, obs1, obs2, state, prefix="pool."):
    """NearestNeighborLSTM.forward (non_gridbased_pooling.py:391-451): the NearestNeighborMLP features of every slot
    (absent ones included: zero features) drive a per-slot LSTMCell whose state persists over the steps of a forward
    (reset at its start, lstm.py:213-216); the interaction vector is hidden2pool(h').  `state` = {"h", "c"} [B*N, Hp],
    updated in place."""
    feats = nn_mlp_pool_forward(cfg, weights, obs1, obs2, prefix)
    h2, c2 = lstm_cell(weights, prefix + "pool_lstm.", feats, state["h"], state["c"])
    state["h"], state["c"] = h2, c2
    return _linear(h2, weights[prefix + "hidden2pool.weight"], weights[prefix + "hidden2pool.bias"])


def trajectron_pool_forward(cfg, weights, obs1, obs2, state, prefix="pool."):
    """TrajectronPooling.forward (non_gridbased_pooling.py:487-537): every VISIBLE slot of the flattened batch embeds
    [own (pos, vel) | sum of the (pos, vel) of all OTHER visible slots of the batch] (Linear(8, out_dim) + ReLU; the sum
    runs over the whole [B * N] batch, :516-527), invisible slots get zeros; then the per-slot LSTMCell and hidden2pool
    like NearestNeighborLSTM."""
    obs1 = np.asarray(obs1, dtype=F32)
    obs2 = np.asarray(obs2, dtype=F32)
    B, N, _ = obs2.shape
    states = np.concatenate([obs2, obs2 - obs1], axis=-1).reshape(B * N, 4).astype(F32)
    vis = ~np.isnan(states).any(axis=-1)
    feats = np.zeros((B * N, cfg.out_dim), dtype=F32)
    sv = states[vis]
    if len(sv):
        rows = []
        for i in range(len(sv)):
            others = np.delete(sv, i, axis=0)
            rows.append(np.concatenate([sv[i], others.sum(axis=0, dtype=F32) if len(others) else np.zeros(4, F32)]))
        x = np.stack(rows).astype(F32)
        feats[vis] = np.maximum(_linear(x, weights[prefix + "embedding.0.weight"], weights[prefix + "embedding.0.bias"]), F32(0.0))
    h2, c2 = lstm_cell(weights, prefix + "pool_lstm.", feats, state["h"], state["c"])
    state["h"], state["c"] = h2, c2
    return _linear(h2, weights[prefix + "hidden2pool.weight"], weights[prefix + "hidden2pool.bias"])


def pool_forward(cfg, weights, hidden, obs1, obs2, prefix="pool.", state=None):
    """GridBasedPooling.forward (gridbased_pooling.py:94-110) -> [B*N, out_dim]."""
    if getattr(cfg, "type_", None) == "traj_pool":
        return trajectron_pool_forward(cfg, weights, obs1, obs2, state, prefix)
    if getattr(cfg, "type_", None) == "nn_lstm":
        return nn_lstm_pool_forward(cfg, weights, obs1, obs2, state, prefix)
    if getattr(cfg, "type_", None) == "hiddenstatemlp":
        return hidden_mlp_pool_forward(cfg, weights, hidden, obs1, obs2, prefix)
    if getattr(cfg, "type_", None) == "nn":
        return nn_mlp_pool_forward(cfg, weights, obs1, obs2, prefix)
    if getattr(cfg, "type_", None) == "attentionmlp":
        return attn_mlp_pool_forward(cfg, weights, hidden, obs1, obs2, prefix)
    obs1 = np.asarray(obs1, dtype=F32)
    obs2 = np.asarray(obs2, dtype=F32)
    B, N, _ = obs2.shape
    vals = None if N == 1 else pair_values(cfg, weights, hidden, obs1, obs2, prefix)
    grid = occupancy_grid(obs2, vals, cfg)
    return embed_grid(cfg, weights, grid.reshape(B * N, -1), prefix)


# ----------------------------------------------------------------------------------------
# leaf modules
# ----------------------------------------------------------------------------------------
def input_embedding(weights, vel, scale=4.0, prefix="input_embedding."):
    """modules.py:24-30."""
    e = _linear(vel.astype(F32) * F32(scale), weights[prefix + "input_embeddings.0.weight"],
                weights[prefix + "input_embeddings.0.bias"])
    e = np.maximum(e, F32(0.0))
    return np.concatenate([e, np.zeros((vel.shape[0], 2), dtype=F32)], axis=1)


def hidden2normal(weights, h, prefix="hidden2normal."):
    """modules.py:56-64."""
    nrm = _linear(h, weights[prefix + "linear.weight"], weights[prefix + "linear.bias"])
    nrm[:, 2] = F32(0.01) + F32(0.2) * _sigmoid(nrm[:, 2])
    nrm[:, 3] = F32(0.01) + F32(0.2) * _sigmoid(nrm[:, 3])
    nrm[:, 4] = F32(0.7) * _sigmoid(nrm[:, 4])
    return nrm


def lstm_cell(weights, prefix, x, h, c):
    """torch.nn.LSTMCell (gate order i, f, g, o)."""
    gates = (_linear(x, weights[prefix + "weight_ih"], weights[prefix + "bias_ih"]) +
             _linear(h, weights[prefix + "weight_hh"], weights[prefix + "bias_hh"])).astype(F32)
    H = h.shape[1]
    i = _sigmoid(gates[:, 0:H])
    f = _sigmoid(gates[:, H:2 * H])
    g = np.tanh(gates[:, 2 * H:3 * H]).astype(F32)
    o = _sigmoid(gates[:, 3 * H:4 * H])
    c2 = (f * c + i * g).astype(F32)
    h2 = (o * np.tanh(c2).astype(F32)).astype(F32)
    return h2, c2


# ----------------------------------------------------------------------------------------
# step / forward (lstm/lstm.py)
# ----------------------------------------------------------------------------------------
def _pad_scenes(x, batch_split, n_max, fill):
    """generate_pooling_inputs (lstm.py:25-42): ragged [M, ...] -> padded [B, Nmax, ...]."""
    B = len(batch_split) - 1
    out = np.full((B, n_max) + x.shape[1:], fill, dtype=x.dtype)
    for b in range(B):
        s, e = int(batch_split[b]), int(batch_split[b + 1])
        out[b, :e - s] = x[s:e]
    return out


def step(weights, pool_cfg, phase, h, c, obs1, obs2, batch_split, pool_to_input=True,
         return_pooled=False, pool_state=None):
    """LSTM.step (lstm.py:91-168).  h, c [M, H] are updated functionally.

    phase = 'encoder' | 'decoder'.  Returns (h', c', normal [M, 5]); rows whose track is
    absent at obs1 or obs2 keep h, c and get normal = NaN (lstm.py:118,158).
    """
    obs1 = np.asarray(obs1, dtype=F32)
    obs2 = np.asarray(obs2, dtype=F32)
    M = obs2.shape[0]
    mask = ~np.isnan(obs1[:, 0]) & ~np.isnan(obs2[:, 0])                   # :118
    vel = (obs2 - obs1)[mask]                                               # :127-128
    x = input_embedding(weights, vel)                                       # :129
    hm, cm = h[mask].astype(F32), c[mask].astype(F32)
    pooled_all = None
    if pool_cfg is not None:
        bs = np.asarray(batch_split, dtype=np.int64)
        n_max = int((bs[1:] - bs[:-1]).max())                               # :29
        cur = _pad_scenes(obs2, bs, n_max, F32(NAN))
        prev = _pad_scenes(obs1, bs, n_max, F32(NAN))
        hid = _pad_scenes(h.astype(F32), bs, n_max, F32(NAN))               # :26,39 (ALL tracks)
        mpos = _pad_scenes(mask, bs, n_max, False)
        if getattr(pool_cfg, "type_", None) in ("nn_lstm", "traj_pool") and pool_state is not None and "h" not in pool_state:
            Hp = pool_cfg.hidden_dim                                        # pool.reset(B * Nmax, ...) lstm.py:213-216
            pool_state["h"] = np.zeros((cur.shape[0] * cur.shape[1], Hp), dtype=F32)
            pool_state["c"] = np.zeros((cur.shape[0] * cur.shape[1], Hp), dtype=F32)
        pooled_all = pool_forward(pool_cfg, weights, hid, prev, cur, state=pool_state)        # :145
        pooled = pooled_all[mpos.reshape(-1)]                               # :146
        if pool_to_input:
            x = np.concatenate([x, pooled], axis=1)                         # :149
        else:
            hm = (hm + pooled).astype(F32)                                  # :151
    h2, c2 = lstm_cell(weights, phase + ".", x, hm, cm)                     # :154
    nrm = hidden2normal(weights, h2)                                        # :155
    h_out = h.astype(F32).copy()
    c_out = c.astype(F32).copy()
    normal = np.full((M, 5), NAN, dtype=F32)                                # :158
    h_out[mask] = h2
    c_out[mask] = c2
    normal[mask] = nrm
    if return_pooled:
        return h_out, c_out, normal, pooled_all
    return h_out, c_out, normal


def forward(weights, pool_cfg, observed, batch_split, prediction_truth=None, n_predict=None,
            hidden_dim=128, pool_to_input=True, return_states=False, between=None):
    """LSTM.forward (lstm.py:170-264), goals off (goal_flag=False in all BASELINE configs).

    Returns rel_pred_scene [S, M, 5], pred_scene [S(+1), M, 2].
    """
    assert (prediction_truth is None) + (n_predict is None) == 1           # :197
    observed = np.asarray(observed, dtype=F32)
    if n_predict is not None:
        truth = [None] * (n_predict - 1)                                    # :200
    else:
        truth = [np.array(t, dtype=F32, copy=True) for t in prediction_truth]   # deepcopy :235
    M = observed.shape[1]
    h = np.zeros((M, hidden_dim), dtype=F32)                                # :207-210
    c = np.zeros((M, hidden_dim), dtype=F32)
    bs = np.asarray(batch_split, dtype=np.int64)
    primaries = bs[:-1]
    normals, positions, states = [], [], []
    pool_state = {}                                                         # interaction-encoder LSTM state (nn_lstm)
    if len(observed) == 2:                                                  # :222-223
        positions = [observed[-1]]
    for obs1, obs2 in zip(observed[:-1], observed[1:]):                     # :226-232
        h, c, normal = step(weights, pool_cfg, "encoder", h, c, obs1, obs2, bs, pool_to_input, pool_state=pool_state)
        normals.append(normal)
        positions.append((obs2 + normal[:, :2]).astype(F32))
        states.append((h, c))
    if between is not None:      # hook between encoder and decoder (S-GAN noise injection, sgan.py:373)
        h, c = between(h, c)
    seq = [observed[-1].copy()] + truth                                     # :235-237
    for k in range(len(seq) - 1):                                           # :240-255
        obs1, obs2 = seq[k], seq[k + 1]
        if obs1 is None:
            obs1 = positions[-2]
        else:
            obs1[primaries] = positions[-2][primaries]
        if obs2 is None:
            obs2 = positions[-1]
        else:
            obs2[primaries] = positions[-1][primaries]
        h, c, normal = step(weights, pool_cfg, "decoder", h, c, obs1, obs2, bs, pool_to_input, pool_state=pool_state)
        normals.append(normal)
        positions.append((obs2 + normal[:, :2]).astype(F32))
        states.append((h, c))
    rel = np.stack(normals, axis=0)
    pred = np.stack(positions, axis=0)
    if return_states:
        return rel, pred, states
    return rel, pred


# ----------------------------------------------------------------------------------------
# loss + metrics
# ----------------------------------------------------------------------------------------
def gaussian_2d(p, x):
    """loss.py:24-50."""
    x1, x2 = x[:, 0], x[:, 1]
    mu1, mu2, s1, s2, rho = p[:, 0], p[:, 1], p[:, 2], p[:, 3], p[:, 4]
    n1 = x1 - mu1
    n2 = x2 - mu2
    s12 = s1 * s2
    z = (n1 / s1) ** 2 + (n2 / s2) ** 2 - 2 * rho * n1 * n2 / s12
    num = np.exp(-z / (2 * (1 - rho ** 2)))
    den = 2 * math.pi * s12 * np.sqrt(1 - rho ** 2)
    return (num / den).astype(F32)


def prediction_loss(inputs, targets, batch_split, background_rate=0.2):
    """PredictionLoss.forward (loss.py:52-91), col_wt = 0, keep_batch_dim False."""
    prim = np.asarray(batch_split, dtype=np.int64)[:-1]
    t = np.asarray(targets, dtype=F32)[:, prim].reshape(-1, 2)
    p = np.asarray(inputs, dtype=F32)[:, prim].reshape(-1, 5)
    bg = p.copy()
    bg[:, 2] = 3.0
    bg[:, 3] = 3.0
    bg[:, 4] = 0.0
    vals = -np.log(F32(0.01) + F32(background_rate) * gaussian_2d(bg, t) +
                   F32(0.99 - background_rate) * gaussian_2d(p, t))
    return F32(vals.astype(F32).mean())


def ade_fde(pred, ref):
    """evaluator/eval_utils.py:3-19 for one track: pred, ref [T, 2] -> (ADE, FDE)."""
    d = np.linalg.norm(np.asarray(pred, dtype=np.float64) - np.asarray(ref, dtype=np.float64), axis=-1)
    return float(d.mean()), float(d[-1])


# ----------------------------------------------------------------------------------------
# synthetic scenes (SURVEY.md section 8d) -- shared by tests and bench
# ----------------------------------------------------------------------------------------
def synthetic_scenes(num_scenes, peds_per_scene, n_frames=21, seed=0, ragged=False,
                     nan_tracks=False, start_std=2.0, vel_std=0.3):
    """Seeded random-walk scenes: xy [T, M, 2] fp32 and batch_split int64 [B+1].

    start ~ N(0, start_std^2 I), per-frame velocity ~ N(0, vel_std^2 I).  ragged: scene
    sizes uniform in [2, peds_per_scene].  nan_tracks: ~10 % of neighbours enter at frame 3
    and ~5 % leave after frame 5 (the primary, first row of a scene, is always present).
    """
    rng = np.random.RandomState(seed)
    if ragged:
        sizes = rng.randint(2, peds_per_scene + 1, size=num_scenes)
    else:
        sizes = np.full(num_scenes, peds_per_scene, dtype=np.int64)
    bs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    M = int(bs[-1])
    p0 = rng.randn(M, 2) * start_std
    v = rng.randn(n_frames, M, 2) * vel_std
    xy = (p0[None] + np.cumsum(v, axis=0)).astype(F32)
    if nan_tracks:
        u = rng.rand(M)
        prim = np.zeros(M, dtype=bool)
        prim[bs[:-1]] = True
        late = (u < 0.10) & ~prim
        early = (u > 0.95) & ~prim
        xy[:3, late] = NAN
        xy[6:, early] = NAN
    return xy, bs


def scenes_of_sizes(sizes, n_frames=21, seed=0):
    """Seeded random-walk scenes with the given numbers of tracks (e.g. one crowded scene next to small
    ones): start ~ N(0, 9 I), per-frame velocity ~ N(0, 0.09 I); xy [T, M, 2] fp32, batch_split int64."""
    rng = np.random.RandomState(seed)
    xs = [rng.randn(n, 2)[None] * 3.0 + np.cumsum(rng.randn(n_frames, n, 2) * 0.3, axis=0) for n in sizes]
    xy = np.concatenate(xs, axis=1).astype(F32)
    bs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return xy, bs


# ----------------------------------------------------------------------------------------
# model specs + seeded weights (shapes = the reference's state_dict, SURVEY.md 8b/B2)
# ----------------------------------------------------------------------------------------
MODEL_SPECS = {
    # BASELINE.json configs
    "vanilla": None,
    "occupancy": dict(type_="occupancy", hidden_dim=128, cell_side=0.6, n=12, out_dim=256,
                      embedding_arch="one_layer"),
    "directional": dict(type_="directional", hidden_dim=128, cell_side=0.6, n=12, out_dim=256,
                        embedding_arch="one_layer"),
    "social": dict(type_="social", hidden_dim=128, cell_side=0.6, n=16, out_dim=256,
                   embedding_arch="two_layer", layer_dims=[1024], latent_dim=16),
    # small / odd variants for edge-case coverage
    "social_small": dict(type_="social", hidden_dim=128, cell_side=0.8, n=6, out_dim=48,
                         embedding_arch="two_layer", layer_dims=[96], latent_dim=8, constant=0),
    "directional_const": dict(type_="directional", hidden_dim=128, cell_side=0.5, n=7, out_dim=40,
                              embedding_arch="one_layer", constant=1),
    "occupancy_front": dict(type_="occupancy", hidden_dim=128, cell_side=0.7, n=8, out_dim=32,
                            embedding_arch="three_layer", layer_dims=[80, 56], front=True),
    # social pooling in each configuration the CUDA library dispatches differently (tests/test_social_backward.py)
    "social_default": dict(type_="social", hidden_dim=128, cell_side=0.6, n=12, out_dim=256,    # reference trainer's
                           embedding_arch="one_layer", latent_dim=16),                          # --type social defaults
    "social_c4": dict(type_="social", hidden_dim=128, cell_side=0.6, n=12, out_dim=128,
                      embedding_arch="one_layer", latent_dim=4),
    "social_c32": dict(type_="social", hidden_dim=128, cell_side=0.7, n=8, out_dim=64,
                       embedding_arch="two_layer", layer_dims=[128], latent_dim=32),
    "social_d96": dict(type_="social", hidden_dim=128, cell_side=0.6, n=10, out_dim=128,
                       embedding_arch="two_layer", layer_dims=[96], latent_dim=16),
    "social_d200": dict(type_="social", hidden_dim=128, cell_side=0.6, n=10, out_dim=128,
                        embedding_arch="two_layer", layer_dims=[200], latent_dim=16),
    # occupancy / directional training in each configuration the grid backward indexes differently
    # (tests/test_grid_backward.py): the front offset, grid sizes, pool widths up to the 1024 limit
    "directional_front": dict(type_="directional", hidden_dim=128, cell_side=0.6, n=12, out_dim=256,
                              embedding_arch="one_layer", front=True),
    "occupancy_front_n4": dict(type_="occupancy", hidden_dim=128, cell_side=0.6, n=4, out_dim=256,
                               embedding_arch="one_layer", front=True),
    "directional_n24": dict(type_="directional", hidden_dim=128, cell_side=0.6, n=24, out_dim=256,
                            embedding_arch="one_layer"),
    "occupancy_p1024": dict(type_="occupancy", hidden_dim=128, cell_side=0.6, n=12, out_dim=1024,
                            embedding_arch="one_layer"),
    "directional_p29": dict(type_="directional", hidden_dim=128, cell_side=0.6, n=12, out_dim=29,
                            embedding_arch="one_layer"),
    # grids whose first Linear each first-layer kernel of the forward takes (tests/test_step_forward.py): the row
    # kernel's 64-column chunk (n = 16), weights too large for it (cells x C > 1280), no embedding (the grid itself)
    "directional_n16": dict(type_="directional", hidden_dim=128, cell_side=0.6, n=16, out_dim=256,
                            embedding_arch="one_layer"),
    "occupancy_n36": dict(type_="occupancy", hidden_dim=128, cell_side=0.3, n=36, out_dim=64,
                          embedding_arch="one_layer"),
    "directional_n26": dict(type_="directional", hidden_dim=128, cell_side=0.4, n=26, out_dim=64,
                            embedding_arch="one_layer"),
    "occupancy_raw": dict(type_="occupancy", hidden_dim=128, cell_side=0.6, n=8, out_dim=64, embedding_arch="None"),
}


# non-grid interaction modules (reference lstm/non_gridbased_pooling.py); trainer.py builds
# HiddenStateMLPPooling(hidden_dim, out_dim=args.pool_dim (256), mlp_dim_vel=args.vel_dim (32))
NONGRID_SPECS = {
    "hiddenstatemlp": dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256),
    "hiddenstatemlp_small": dict(hidden_dim=128, mlp_dim=48, mlp_dim_spatial=16, mlp_dim_vel=8, out_dim=40),
}


# NearestNeighborMLP(n=args.neigh (4), out_dim=args.pool_dim, no_vel=args.no_vel) (lstm/trainer.py:476-477)
NN_SPECS = {
    "nn": dict(n=4, out_dim=256, no_vel=False),
    "nn_small": dict(n=3, out_dim=24, no_vel=True),
}


# AttentionMLPPooling(hidden_dim, out_dim=args.pool_dim, mlp_dim_spatial=args.spatial_dim (32), mlp_dim_vel=args.vel_dim (32))
ATTN_SPECS = {
    "attentionmlp": dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256),
    "attentionmlp_small": dict(hidden_dim=128, mlp_dim=48, mlp_dim_spatial=16, mlp_dim_vel=8, out_dim=40),
}


# NearestNeighborLSTM(n=args.neigh (4), hidden_dim=args.hidden_dim (128), out_dim=args.pool_dim) (lstm/trainer.py:478-479)
NN_LSTM_SPECS = {
    "nn_lstm": dict(n=4, hidden_dim=128, out_dim=256),
    "nn_lstm_small": dict(n=3, hidden_dim=40, out_dim=24),
}


# TrajectronPooling(hidden_dim=args.hidden_dim (128), out_dim=args.pool_dim) (lstm/trainer.py:480-481)
TRAJ_SPECS = {
    "traj_pool": dict(hidden_dim=128, out_dim=256),
    "traj_pool_small": dict(hidden_dim=40, out_dim=24),
}


def pool_config(kind):
    if kind in TRAJ_SPECS:
        return TrajectronPoolConfig(**TRAJ_SPECS[kind])
    if kind in NN_LSTM_SPECS:
        return NnLstmPoolConfig(**NN_LSTM_SPECS[kind])
    if kind in ATTN_SPECS:
        return AttnPoolConfig(**ATTN_SPECS[kind])
    if kind in NONGRID_SPECS:
        return MlpPoolConfig(**NONGRID_SPECS[kind])
    if kind in NN_SPECS:
        return NnPoolConfig(**NN_SPECS[kind])
    spec = MODEL_SPECS[kind]
    return None if spec is None else PoolConfig(**spec)


def random_weights(kind, seed=0, scale=1.0, embedding_dim=64, hidden_dim=128, relu_bias=None, out_dim=None,
                   pool_to_input=True):
    """Seeded weights in the reference's state_dict layout (uniform(-1/sqrt(fan_in), ..) like
    torch's default init, times `scale`).  numpy RandomState => identical on every machine.

    relu_bias = beta: the biases of the grid embedding's Linears (pool.embedding.*.bias) become +beta
    (even units) and -beta (odd units).  The pre-activations of those ReLUs then stay far from 0, so
    rounding differences between implementations cannot flip a ReLU mask, and half of the units are
    still dead, so a backward that ignores the mask is still caught.  The other weights are unchanged.

    out_dim: the interaction module's out_dim instead of the kind's.  pool_to_input=False: the LSTM input is
    the embedding alone (the pooled vector is added to h, lstm.py:151), so weight_ih has embedding_dim columns."""
    rng = np.random.RandomState(seed)
    cfg = pool_config(kind)
    if cfg is not None and out_dim is not None:
        cfg.out_dim = out_dim
    W = {}

    def lin(name_w, name_b, out_f, in_f):
        k = scale / math.sqrt(in_f)
        W[name_w] = rng.uniform(-k, k, size=(out_f, in_f)).astype(F32)
        W[name_b] = rng.uniform(-k, k, size=(out_f,)).astype(F32)

    E, H = embedding_dim, hidden_dim
    pool_dim = 0
    if cfg is not None and cfg.type_ in ("nn_lstm", "traj_pool"):
        if cfg.type_ == "traj_pool":
            lin("pool.embedding.0.weight", "pool.embedding.0.bias", cfg.out_dim, 8)
        else:
            lin("pool.embedding.0.weight", "pool.embedding.0.bias", cfg.out_dim // cfg.n, cfg.input_dim)
        kp = scale / math.sqrt(cfg.hidden_dim)
        W["pool.pool_lstm.weight_ih"] = rng.uniform(-kp, kp, size=(4 * cfg.hidden_dim, cfg.out_dim)).astype(F32)
        W["pool.pool_lstm.weight_hh"] = rng.uniform(-kp, kp, size=(4 * cfg.hidden_dim, cfg.hidden_dim)).astype(F32)
        W["pool.pool_lstm.bias_ih"] = rng.uniform(-kp, kp, size=(4 * cfg.hidden_dim,)).astype(F32)
        W["pool.pool_lstm.bias_hh"] = rng.uniform(-kp, kp, size=(4 * cfg.hidden_dim,)).astype(F32)
        lin("pool.hidden2pool.weight", "pool.hidden2pool.bias", cfg.out_dim, cfg.hidden_dim)
        pool_dim = cfg.out_dim
    elif cfg is not None and cfg.type_ == "nn":
        lin("pool.embedding.0.weight", "pool.embedding.0.bias", cfg.out_dim // cfg.n, cfg.input_dim)
        pool_dim = cfg.out_dim
    elif cfg is not None and cfg.type_ == "attentionmlp":
        lin("pool.spatial_embedding.0.weight", "pool.spatial_embedding.0.bias", cfg.mlp_dim_spatial, 2)
        if cfg.mlp_dim_vel:
            lin("pool.vel_embedding.0.weight", "pool.vel_embedding.0.bias", cfg.mlp_dim_vel, 2)
        if cfg.mlp_dim_hidden:
            lin("pool.hidden_embedding.0.weight", "pool.hidden_embedding.0.bias", cfg.mlp_dim_hidden, H)
        Ea = cfg.mlp_dim
        ka = scale / math.sqrt(Ea)
        for nm in ("wq", "wk", "wv"):
            W["pool.%s.weight" % nm] = rng.uniform(-ka, ka, size=(Ea, Ea)).astype(F32)
        W["pool.multihead_attn.in_proj_weight"] = rng.uniform(-ka, ka, size=(3 * Ea, Ea)).astype(F32)
        W["pool.multihead_attn.in_proj_bias"] = rng.uniform(-ka, ka, size=(3 * Ea,)).astype(F32)
        lin("pool.multihead_attn.out_proj.weight", "pool.multihead_attn.out_proj.bias", Ea, Ea)
        lin("pool.out_projection.weight", "pool.out_projection.bias", cfg.out_dim, Ea)
        pool_dim = cfg.out_dim
    elif cfg is not None and cfg.type_ == "hiddenstatemlp":
        lin("pool.spatial_embedding.0.weight", "pool.spatial_embedding.0.bias", cfg.mlp_dim_spatial, 2)
        if cfg.mlp_dim_vel:
            lin("pool.vel_embedding.0.weight", "pool.vel_embedding.0.bias", cfg.mlp_dim_vel, 2)
        if cfg.mlp_dim_hidden:
            lin("pool.hidden_embedding.0.weight", "pool.hidden_embedding.0.bias", cfg.mlp_dim_hidden, H)
        lin("pool.out_projection.weight", "pool.out_projection.bias", cfg.out_dim, cfg.mlp_dim)
        pool_dim = cfg.out_dim
    elif cfg is not None:
        if cfg.type_ in ("social", "dir_social"):
            lin("pool.hidden_dim_encoding.weight", "pool.hidden_dim_encoding.bias", cfg.latent_dim, H)
        n_layers = {"None": 0, None: 0, "one_layer": 1, "two_layer": 2, "three_layer": 3}[cfg.embedding_arch]
        dims = [cfg.n * cfg.n * cfg.pooling_dim] + list((cfg.layer_dims or [])[:max(n_layers - 1, 0)]) + [cfg.out_dim]
        for l in range(n_layers):
            lin("pool.embedding.%d.weight" % (2 * l), "pool.embedding.%d.bias" % (2 * l), dims[l + 1], dims[l])
        pool_dim = cfg.out_dim if n_layers else dims[0]
    lin("input_embedding.input_embeddings.0.weight", "input_embedding.input_embeddings.0.bias", E - 2, 2)
    lin("goal_embedding.input_embeddings.0.weight", "goal_embedding.input_embeddings.0.bias", E - 2, 2)
    k = scale / math.sqrt(H)
    if not pool_to_input:
        pool_dim = 0
    for ph in ("encoder", "decoder"):
        W[ph + ".weight_ih"] = rng.uniform(-k, k, size=(4 * H, E + pool_dim)).astype(F32)
        W[ph + ".weight_hh"] = rng.uniform(-k, k, size=(4 * H, H)).astype(F32)
        W[ph + ".bias_ih"] = rng.uniform(-k, k, size=(4 * H,)).astype(F32)
        W[ph + ".bias_hh"] = rng.uniform(-k, k, size=(4 * H,)).astype(F32)
    lin("hidden2normal.linear.weight", "hidden2normal.linear.bias", 5, H)
    if relu_bias is not None:
        for name in W:
            if name.startswith("pool.embedding.") and name.endswith(".bias"):
                b = np.full(W[name].shape, relu_bias, dtype=F32)
                b[1::2] = -relu_bias
                W[name] = b
    return W
