"""Differentiable torch restatement of LSTM.forward + PredictionLoss (fp32 or fp64) -- TEST INFRASTRUCTURE.

Used to check the hand-written CUDA backward (csrc/train.cu).  Follows oracle/lstm_oracle.py (which is
pinned to the reference) line by line, with torch ops so autograd provides the gradients;
test_training.py, test_social_backward.py and test_grid_backward.py pin THIS file's gradients to gradients
of the unmodified reference (tests/golden/train_golden.npz, social_train_golden.npz, grid_train_golden.npz).

The non-grid interaction modules (nongrid_pool, and `forward` with such a pool) are restated from the reference's
lstm/non_gridbased_pooling.py directly, not from the oracle, and checked against csrc/mlp_pool.cu in
test_nongrid_kernels.py; that file pins them to tests/golden/nongrid_golden.npz.
"""
import math

import torch
import torch.nn.functional as F

NAN = float("nan")


def _mm(x, w, kernel=None):
    """x @ w.T, or kernel.mm(x, w) when a kernel emulation (see bf16_product) is given."""
    mm = getattr(kernel, "mm", None)
    return x @ w.T if mm is None else mm(x, w)


def bf16_product(passes=3):
    """x @ w.T as the tensor-core kernels compute it from fp32 operands: hi = bf16(v), lo = bf16(v - hi) of both,
    then hi.hi + hi.lo + lo.hi summed in float64 (passes=3); passes=2 drops lo.hi."""
    def split(v):
        hi = v.to(torch.bfloat16).to(v.dtype)
        return hi, (v - hi).to(torch.bfloat16).to(v.dtype)

    def mm(x, w):
        (xh, xl), (wh, wl) = split(x), split(w)
        out = xh @ wh.T + xh @ wl.T
        return out + xl @ wh.T if passes == 3 else out
    return mm


def _grid(pool_cfg, W, obs1, obs2, hidden, dtype, stats, primary_edges, kernel=None):
    """[B, N, ...] padded -> pooled [B*N, out] (gridbased_pooling.py:112-170,227-305,308-335), cf.
    oracle.lstm_oracle.occupancy_grid / pool_forward.  embedding_arch None / 'None': the grid itself.

    kernel: an emulation of a kernel's arithmetic: kernel.mm(x, w) replaces the embedding's products and
    kernel.grid(grid [B*N, C, n, n]) edits the grid before the embedding (either may be absent).

    The cells are binned in fp32 on the fp32 positions, like the reference, whatever `dtype` the
    arithmetic runs in.  The reference writes the grid with ONE index_put (gridbased_pooling.py:293): in
    the forward a later writer of a cell overwrites an earlier one, and in the backward every writer,
    overwritten ones included, receives the cell's gradient.  For social pooling that gradient reaches
    pool.hidden_dim_encoding, so a loop of sequential writes (which would credit the last writer only)
    would be wrong.

    stats["relu_pool<l>"] collects the smallest |pre-activation| of each embedding Linear.  With
    primary_edges, stats["edge_primary"] collects the smallest distance (in cells) of a primary-involving
    pair's offset to a cell edge: in the decoder the primaries' positions are fed back predictions,
    so another implementation may bin exactly those pairs differently."""
    B, N, _ = obs2.shape
    n = pool_cfg.n
    C = pool_cfg.pooling_dim
    if N > 1:
        obs = obs2.detach().clone()
        absent = torch.isnan(obs).any(dim=-1)
        obs[absent] = -500.0
        rel = obs[:, None, :, :] - obs[:, :, None, :]
        keep = ~torch.eye(N, dtype=torch.bool)
        rel = rel[:, keep].reshape(B, N, N - 1, 2)
        off = torch.tensor([n / 2, 0.0 if pool_cfg.front else n / 2])
        oij = rel / float(pool_cfg.cell_side) + off
        if primary_edges:
            prim_pair = torch.zeros(B, N, N - 1, dtype=torch.bool)
            prim_pair[:, 0, :] = True                   # row 0 of a padded scene is its primary
            prim_pair[:, 1:, 0] = True                  # neighbour slot 0 of the other rows is the primary
            present = (~absent)[:, :, None] & (~absent)[:, None, :]
            prim_pair &= present[:, keep].reshape(B, N, N - 1)
            edge = oij.round().clamp(0, n)              # the edges that decide cell / in-range
            d = (oij - edge).abs()[prim_pair]
            if d.numel():
                _note(stats, "edge_primary", float(d.min()))
        ok = ~(((oij < 0) | (oij >= n)).any(dim=-1))
        oij = torch.where(ok[..., None], oij, torch.zeros_like(oij)).long()
        oi = (oij[..., 0] * n + oij[..., 1]).reshape(B * N, N - 1)
        if pool_cfg.type_ == "social":
            hg = hidden[:, None, :, :].expand(B, N, N, hidden.shape[-1])[:, keep].reshape(B, N, N - 1, -1)
            hg = torch.nan_to_num(hg)
            vals = hg @ W["pool.hidden_dim_encoding.weight"].T + W["pool.hidden_dim_encoding.bias"]
        elif pool_cfg.type_ == "directional":
            vel = (obs2 - obs1).detach()
            rv = vel[:, None, :, :] - vel[:, :, None, :]
            vals = torch.nan_to_num(rv[:, keep].reshape(B, N, N - 1, 2)).to(dtype)
        else:
            vals = torch.ones(B, N, N - 1, 1, dtype=dtype)
        vals = torch.where(ok[..., None], vals, torch.full_like(vals, float(pool_cfg.constant))).reshape(B * N, N - 1, C)
        # index_put's write order among duplicate indices is unspecified (on the CPU it runs in parallel above a
        # few ten thousand elements); the reference's semantics are those of its sequential run: the last writer
        # (ascending neighbour slot) wins.  Winners are written first, the overwritten writers then add
        # v - v.detach() (exactly 0) so that they receive their cell's gradient like index_put's backward gives.
        rows = torch.arange(B * N)[:, None].expand(B * N, N - 1)
        later = torch.ones(N - 1, N - 1, dtype=torch.bool).triu(1)
        win = ~((oi[:, :, None] == oi[:, None, :]) & later).any(dim=-1)
        grid = torch.full((B * N, n * n, C), float(pool_cfg.constant), dtype=dtype)
        grid = grid.index_put((rows[win], oi[win]), vals[win])
        grid = grid.index_put((rows[~win], oi[~win]), vals[~win] - vals[~win].detach(), accumulate=True)
    else:
        grid = torch.full((B * N, n * n, C), float(pool_cfg.constant), dtype=dtype)
    # lp_pool2d(p=1, window 1) (gridbased_pooling.py:303) is the identity in the forward, but its gradient is 0
    # where a cell holds exactly 0: the writers of a cell that an out-of-range pair (value `constant` = 0)
    # overwrote last receive no gradient
    grid = F.lp_pool2d(grid.transpose(1, 2).reshape(B * N, C, n, n), 1, 1)
    if getattr(kernel, "grid", None) is not None:
        grid = kernel.grid(grid)
    x = grid.reshape(B * N, -1)
    n_layers = {None: 0, "None": 0, "one_layer": 1, "two_layer": 2, "three_layer": 3}[pool_cfg.embedding_arch]
    for l in range(n_layers):
        z = _mm(x, W["pool.embedding.%d.weight" % (2 * l)], kernel) + W["pool.embedding.%d.bias" % (2 * l)]
        _note(stats, "relu_pool%d" % l, float(z.detach().abs().min()))
        x = torch.relu(z)
    return x


def _note(stats, key, value):
    if stats is not None:
        stats[key] = min(value, stats.get(key, math.inf))


NONGRID = ("hiddenstatemlp", "attentionmlp", "nn", "nn_lstm", "traj_pool")


def _embed_masked(x, w, b, fill):
    """embed_with_masking (non_gridbased_pooling.py:52-60): relu(Linear(x)) where x has no NaN, else `fill`."""
    bad = torch.isnan(x).any(dim=-1, keepdim=True)
    y = torch.relu(torch.nan_to_num(x) @ w.T + b)
    return torch.where(bad, torch.full_like(y, float(fill)), y)


def _pad_slots(x, slots):
    """[n, ...] -> [slots, ...]: the slots past the scene's tracks are absent tracks (NaN)."""
    return torch.cat([x, torch.full((slots - x.shape[0],) + tuple(x.shape[1:]), NAN, dtype=x.dtype)])


def _hidden_mlp(cfg, W, hid, p1, p2):
    """HiddenStateMLPPooling (:197-239) on one scene [N, ...]: max over every slot j (i included) of
    [spatial(p_j - p_i) | hidden(h_j) | vel(4 (v_j - v_i))], NaN inputs -> -100, then out_projection."""
    N = p2.shape[0]
    parts = [_embed_masked(p2[None, :, :] - p2[:, None, :], W["pool.spatial_embedding.0.weight"],
                           W["pool.spatial_embedding.0.bias"], -100.0)]
    if cfg.mlp_dim_hidden:
        e = _embed_masked(hid, W["pool.hidden_embedding.0.weight"], W["pool.hidden_embedding.0.bias"], -100.0)
        parts.append(e[None].expand(N, N, e.shape[-1]))
    if cfg.mlp_dim_vel:
        v = p2 - p1
        parts.append(_embed_masked((v[None, :, :] - v[:, None, :]) * 4.0, W["pool.vel_embedding.0.weight"],
                                   W["pool.vel_embedding.0.bias"], -100.0))
    pooled = torch.cat(parts, dim=-1).max(dim=1).values
    return pooled @ W["pool.out_projection.weight"].T + W["pool.out_projection.bias"]


def _attention(cfg, W, hid, p1, p2, n, stats=None, rows=None):
    """AttentionMLPPooling (:297-351) on one scene of N slots whose first n are tracks: for track i the sequence is
    e_ij over every slot j, NaN inputs -> fill_value (spatial, velocity) / 0 (hidden); wq / wk / wv, then one-head
    MultiheadAttention computed the plain way (in-projection, softmax(q k / sqrt(E)), value sum, out_proj); the
    output at position i, then out_projection.  The slots past n all embed to one vector: its key and value are
    computed once and repeated.  rows: only the first `rows` tracks query (default n).
    stats["attn_span"]: the smallest (over the tracks) max - min of a track's logits."""
    N, E, fill = p2.shape[0], cfg.mlp_dim, float(cfg.fill_value)

    def emb(rel, h, relv):
        parts = [_embed_masked(rel, W["pool.spatial_embedding.0.weight"], W["pool.spatial_embedding.0.bias"], fill)]
        if cfg.mlp_dim_hidden:
            parts.append(_embed_masked(h, W["pool.hidden_embedding.0.weight"], W["pool.hidden_embedding.0.bias"], 0.0))
        if cfg.mlp_dim_vel:
            parts.append(_embed_masked(relv, W["pool.vel_embedding.0.weight"], W["pool.vel_embedding.0.bias"], fill))
        return torch.cat(parts, dim=-1)

    v = p2 - p1
    r = n if rows is None else rows
    e = emb((p2[None, :n] - p2[:r, None]), hid[None, :n].expand(r, n, hid.shape[-1]),
            (v[None, :n] - v[:r, None]) * 4.0)                                   # [i < r, j < n, E]
    nan2 = torch.full((2,), NAN, dtype=p2.dtype)
    e_pad = emb(nan2, torch.full((hid.shape[-1],), NAN, dtype=p2.dtype), nan2)  # [E]: a slot past n
    Win, bin_ = W["pool.multihead_attn.in_proj_weight"], W["pool.multihead_attn.in_proj_bias"]
    diag = torch.arange(r)
    q = (e[diag, diag] @ W["pool.wq.weight"].T) @ Win[:E].T + bin_[:E]         # [i, E]: the query at position i

    def kv(x, r):
        return (x @ W["pool.w%s.weight" % "kv"[r]].T) @ Win[(r + 1) * E:(r + 2) * E].T + bin_[(r + 1) * E:(r + 2) * E]
    k = torch.cat([kv(e, 0), kv(e_pad, 0)[None, None].expand(r, N - n, E)], dim=1)
    val = torch.cat([kv(e, 1), kv(e_pad, 1)[None, None].expand(r, N - n, E)], dim=1)
    s = torch.einsum("ie,ije->ij", q, k) / math.sqrt(E)
    _note(stats, "attn_span", float((s.max(dim=1).values - s.min(dim=1).values).min()))
    a = torch.exp(s - s.max(dim=1, keepdim=True).values)
    a = a / a.sum(dim=1, keepdim=True)
    att = torch.einsum("ij,ije->ie", a, val)
    att = att @ W["pool.multihead_attn.out_proj.weight"].T + W["pool.multihead_attn.out_proj.bias"]
    return att @ W["pool.out_projection.weight"].T + W["pool.out_projection.bias"]


def _nearest(cfg, W, p1, p2, stats):
    """NearestNeighborMLP (:96-147) on one scene [N, 2]: the n nearest other slots in ascending distance (NaN -> 1000),
    features [p_j - p_i | v_j - v_i] (NaN -> 0; zero rows when there are fewer than n), shared Linear + ReLU.

    stats["nn_gap"]: the smallest gap between consecutive ranks up to rank n + 1 of a track whose two neighbours have
    different features (a tie between equal feature rows cannot change the output)."""
    N, nn = p2.shape[0], cfg.n
    keep = ~torch.eye(N, dtype=torch.bool)
    rel = (p2[None, :, :] - p2[:, None, :])[keep].reshape(N, N - 1, 2)
    feat = rel
    if not cfg.no_vel:
        v = p2 - p1
        feat = torch.cat([rel, (v[None, :, :] - v[:, None, :])[keep].reshape(N, N - 1, 2)], dim=-1)
    feat = torch.nan_to_num(feat)
    dist = torch.nan_to_num(torch.sqrt(rel[..., 0] ** 2 + rel[..., 1] ** 2), nan=1000.0)
    d_sorted, order = torch.sort(dist, dim=1, stable=True)
    g = torch.gather(feat, 1, order[..., None].expand(N, N - 1, feat.shape[-1]))
    r = min(nn + 1, N - 1)
    if stats is not None and r >= 2:
        gap = d_sorted[:, 1:r] - d_sorted[:, :r - 1]
        same = (g[:, 1:r] == g[:, :r - 1]).all(dim=-1)
        gap = gap[~same]
        if gap.numel():
            _note(stats, "nn_gap", float(gap.min()))
    g = g[:, :nn]
    if g.shape[1] < nn:
        g = torch.cat([g, torch.zeros(N, nn - g.shape[1], g.shape[-1], dtype=g.dtype)], dim=1)
    return torch.relu(g @ W["pool.embedding.0.weight"].T + W["pool.embedding.0.bias"]).reshape(N, -1)


def _pool_lstm(W, x, state):
    """The interaction-encoder LSTMCell (:445-451): advances state = {"h", "c"} row by row, returns hidden2pool(h')."""
    g = x @ W["pool.pool_lstm.weight_ih"].T + W["pool.pool_lstm.bias_ih"] + \
        state["h"] @ W["pool.pool_lstm.weight_hh"].T + W["pool.pool_lstm.bias_hh"]
    H = state["h"].shape[1]
    c2 = torch.sigmoid(g[:, H:2 * H]) * state["c"] + torch.sigmoid(g[:, :H]) * torch.tanh(g[:, 2 * H:3 * H])
    h2 = torch.sigmoid(g[:, 3 * H:]) * torch.tanh(c2)
    state["h"], state["c"] = h2, c2
    return h2 @ W["pool.hidden2pool.weight"].T + W["pool.hidden2pool.bias"]


def _trajectron_feat(W, p1, p2):
    """TrajectronPooling's features (:509-529) over the rows it is given (the whole flattened batch): a visible row
    embeds [own (pos, vel) | sum of (pos, vel) over the OTHER visible rows], an invisible row is 0."""
    st = torch.cat([p2, p2 - p1], dim=-1)
    vis = ~torch.isnan(st).any(dim=-1)
    others = st[vis].sum(dim=0)[None] - st
    y = torch.relu(torch.cat([st, others], dim=-1) @ W["pool.embedding.0.weight"].T + W["pool.embedding.0.bias"])
    return torch.where(vis[:, None], y, torch.zeros_like(y))


def nongrid_pool(cfg, W, hidden, obs1, obs2, dtype=torch.float64, state=None, stats=None):
    """The stand-alone plug of a non-grid module: hidden [B, N, H] (or None), obs1 / obs2 [B, N, 2] fp32 (NaN = absent)
    -> [B * N, out_dim] in `dtype`.  state: {"h", "c"} [B * N, Hp] of nn_lstm / traj_pool, advanced in place.
    stats: see _nearest."""
    W = {k: torch.as_tensor(v).to(dtype) for k, v in W.items() if k.startswith("pool.")}
    p1, p2 = torch.as_tensor(obs1).to(dtype), torch.as_tensor(obs2).to(dtype)
    B, N, _ = p2.shape
    hid = torch.as_tensor(hidden).to(dtype) if hidden is not None else None
    if cfg.type_ == "traj_pool":
        return _pool_lstm(W, _trajectron_feat(W, p1.reshape(B * N, 2), p2.reshape(B * N, 2)), state)
    out = []
    for b in range(B):
        if cfg.type_ == "hiddenstatemlp":
            out.append(_hidden_mlp(cfg, W, hid[b], p1[b], p2[b]))
        elif cfg.type_ == "attentionmlp":
            out.append(_attention(cfg, W, hid[b], p1[b], p2[b], N, stats))
        else:
            out.append(_nearest(cfg, W, p1[b], p2[b], stats))
    out = torch.cat(out)
    return _pool_lstm(W, out, state) if cfg.type_ == "nn_lstm" else out


def nongrid_pool_ragged(pool_cfg, W, h, obs1, obs2, bs, pad_to_batch_max=True, dtype=torch.float64, pool_state=None,
                        stats=None):
    """The non-grid pool as LSTM.step calls it, on ragged rows: h [M, H] (or None), obs1 / obs2 [M, 2] -> [M, out_dim].
    Scenes padded to the batch maximum (the reference's batched call) or each scene on its own slots
    (pad_to_batch_max=False); the interaction-encoder state is one row per track."""
    bs = [int(v) for v in bs]
    B = len(bs) - 1
    n_max = max(bs[b + 1] - bs[b] for b in range(B))
    p1, p2 = torch.as_tensor(obs1).to(dtype), torch.as_tensor(obs2).to(dtype)
    h = torch.as_tensor(h).to(dtype) if h is not None else torch.full((bs[-1], 1), NAN, dtype=dtype)
    Wp = {k: torch.as_tensor(v).to(dtype) for k, v in W.items() if k.startswith("pool.")}
    if pool_cfg.type_ == "traj_pool":
        if pad_to_batch_max:
            feat = _trajectron_feat(Wp, p1, p2)
        else:
            feat = torch.cat([_trajectron_feat(Wp, p1[bs[b]:bs[b + 1]], p2[bs[b]:bs[b + 1]]) for b in range(B)])
        return _pool_lstm(Wp, feat, pool_state)
    out = []
    for b in range(B):
        s, e = bs[b], bs[b + 1]
        n = e - s
        slots = n_max if pad_to_batch_max else n
        q1, q2 = _pad_slots(p1[s:e], slots), _pad_slots(p2[s:e], slots)
        if pool_cfg.type_ == "hiddenstatemlp":
            y = _hidden_mlp(pool_cfg, Wp, _pad_slots(h[s:e], slots), q1, q2)
        elif pool_cfg.type_ == "attentionmlp":
            y = _attention(pool_cfg, Wp, _pad_slots(h[s:e], slots), q1, q2, n, stats)
        else:
            y = _nearest(pool_cfg, Wp, q1, q2, stats)
        out.append(y[:n])
    out = torch.cat(out)
    return _pool_lstm(Wp, out, pool_state) if pool_cfg.type_ == "nn_lstm" else out


def _pad(x, bs, fill):
    """ragged [M, ...] -> padded [B, Nmax, ...] (generate_pooling_inputs, lstm.py:25-42)."""
    B = len(bs) - 1
    n_max = max(bs[b + 1] - bs[b] for b in range(B))
    out = torch.full((B, n_max) + tuple(x.shape[1:]), fill, dtype=x.dtype)
    for b in range(B):
        out[b, :bs[b + 1] - bs[b]] = x[bs[b]:bs[b + 1]]
    return out


def pool_state_zeros(pool_cfg, M, dtype):
    """The interaction-encoder state of nn_lstm / traj_pool after pool.reset (lstm.py:213-216), else None."""
    if getattr(pool_cfg, "type_", None) in ("nn_lstm", "traj_pool"):
        return {"h": torch.zeros(M, pool_cfg.hidden_dim, dtype=dtype), "c": torch.zeros(M, pool_cfg.hidden_dim, dtype=dtype)}
    return None


def step(W, pool_cfg, phase, h, c, obs1, obs2, batch_split, hidden_dim, dtype, pool_to_input=True, stats=None,
         pad_to_batch_max=True, pool_state=None, kernel=None):
    """LSTM.step (lstm.py:91-168): h, c [M, H] `dtype`, obs1 / obs2 [M, 2] fp32 (NaN = absent) -> (h', c', normal
    [M, 5]); rows absent at obs1 or obs2 keep h, c and get normal = NaN.

    pool_to_input=False: the pooled vector of the present rows is added to their h before the W_hh product
    (lstm.py:151), and the LSTM input is the embedding alone.  pool_state: see pool_state_zeros (advanced in place).
    kernel: see _grid; kernel.mm also replaces the gate product."""
    bs = [int(v) for v in batch_split]
    M = obs2.shape[0]
    mask = ~torch.isnan(obs1[:, 0]) & ~torch.isnan(obs2[:, 0])
    vel = (obs2 - obs1)[mask].to(dtype)
    e = torch.relu((vel * 4.0) @ W["input_embedding.input_embeddings.0.weight"].T +
                   W["input_embedding.input_embeddings.0.bias"])
    x = torch.cat([e, torch.zeros(e.shape[0], 2, dtype=dtype)], dim=1)
    hm = h[mask]
    if getattr(pool_cfg, "type_", None) in NONGRID:
        pooled = nongrid_pool_ragged(pool_cfg, W, h.detach(), obs1, obs2, bs, pad_to_batch_max, dtype, pool_state,
                                     stats)[mask]
    elif pool_cfg is not None:
        pooled = _grid(pool_cfg, W, _pad(obs1, bs, NAN), _pad(obs2, bs, NAN), _pad(h, bs, NAN), dtype, stats,
                       primary_edges=phase == "decoder", kernel=kernel)[_pad(mask, bs, False).reshape(-1)]
    if pool_cfg is not None:
        if pool_to_input:
            x = torch.cat([x, pooled], dim=1)
        else:
            hm = hm + pooled
    gates = (_mm(x, W[phase + ".weight_ih"], kernel) + W[phase + ".bias_ih"] + _mm(hm, W[phase + ".weight_hh"], kernel)
             + W[phase + ".bias_hh"])
    H = hidden_dim
    i, f = torch.sigmoid(gates[:, :H]), torch.sigmoid(gates[:, H:2 * H])
    g, o = torch.tanh(gates[:, 2 * H:3 * H]), torch.sigmoid(gates[:, 3 * H:])
    c2 = f * c[mask] + i * g
    h2 = o * torch.tanh(c2)
    raw = h2 @ W["hidden2normal.linear.weight"].T + W["hidden2normal.linear.bias"]
    nrm = torch.cat([raw[:, :2], 0.01 + 0.2 * torch.sigmoid(raw[:, 2:4]), 0.7 * torch.sigmoid(raw[:, 4:5])], dim=1)
    idx = mask.nonzero().flatten()
    h_out = h.index_copy(0, idx, h2)
    c_out = c.index_copy(0, idx, c2)
    normal = torch.full((M, 5), NAN, dtype=dtype).index_copy(0, idx, nrm)
    return h_out, c_out, normal


def forward(W, pool_cfg, observed, batch_split, prediction_truth=None, n_predict=None, hidden_dim=128,
            dtype=torch.float32, stats=None, feed_back=None, pad_to_batch_max=True, pool_to_input=True, kernel=None):
    """W: dict of `dtype` tensors (requires_grad as wanted).  Returns rel [S, M, 5] (`dtype`), pred [S, M, 2]
    (fp32: the positions the model feeds back are fp32 data, as in the reference).  stats: see _grid.

    feed_back: fp32 positions [S(+1), M, 2] of another implementation's forward (aligned with pred).  The
    decoder is then fed those (detached) positions instead of this forward's own, so the gradients are
    exact for that implementation's trajectory and no fed-back position can be binned differently.

    pad_to_batch_max: with a non-grid pool, False gives each scene its own slots (the per-scene layout): the
    attention keys stop at the scene's tracks and Trajectron's sums at its scene.  pool_to_input, kernel: see step."""
    bs = [int(v) for v in batch_split]
    M = observed.shape[1]
    prim = torch.tensor(bs[:-1])
    h = torch.zeros(M, hidden_dim, dtype=dtype)
    c = torch.zeros(M, hidden_dim, dtype=dtype)
    truth = [None] * (n_predict - 1) if n_predict is not None else [t.clone() for t in prediction_truth]
    pool_state = pool_state_zeros(pool_cfg, M, dtype)

    def step_(phase, h, c, obs1, obs2):
        return step(W, pool_cfg, phase, h, c, obs1, obs2, bs, hidden_dim, dtype, pool_to_input, stats,
                    pad_to_batch_max, pool_state, kernel)

    normals, positions = [], []
    if observed.shape[0] == 2:
        positions = [observed[-1]]

    def fed(i):     # the position fed back as step i's input (i < 0 counts from the end)
        i = i % len(positions)
        return feed_back[i] if feed_back is not None else positions[i].detach()

    for t in range(observed.shape[0] - 1):
        h, c, normal = step_("encoder", h, c, observed[t], observed[t + 1])
        normals.append(normal)
        positions.append(observed[t + 1] + normal[:, :2].to(observed.dtype))
    seq = [observed[-1].clone()] + truth
    for k in range(len(seq) - 1):
        obs1, obs2 = seq[k], seq[k + 1]
        if obs1 is None:
            obs1 = fed(-2)
        else:
            obs1 = obs1.clone()
            obs1[prim] = fed(-2)[prim]
        if obs2 is None:
            obs2 = fed(-1)
        else:
            obs2 = obs2.clone()
            obs2[prim] = fed(-1)[prim]
            seq[k + 1] = obs2
        h, c, normal = step_("decoder", h, c, obs1, obs2)
        normals.append(normal)
        positions.append(obs2 + normal[:, :2].to(obs2.dtype))
    return torch.stack(normals), torch.stack(positions)


def gaussian_2d(p, x):
    n1, n2 = x[:, 0] - p[:, 0], x[:, 1] - p[:, 1]
    s1, s2, rho = p[:, 2], p[:, 3], p[:, 4]
    z = (n1 / s1) ** 2 + (n2 / s2) ** 2 - 2 * rho * n1 * n2 / (s1 * s2)
    return torch.exp(-z / (2 * (1 - rho ** 2))) / (2 * math.pi * s1 * s2 * torch.sqrt(1 - rho ** 2))


def prediction_loss_values(inputs, targets, batch_split, background_rate=0.2):
    """[pred_length, batch_size] values of the primaries (reference lstm/loss.py:52-91 before the mean)."""
    prim = torch.tensor([int(v) for v in batch_split[:-1]])
    t = targets[:, prim].reshape(-1, 2)
    p = inputs[:, prim].reshape(-1, 5)
    bg = torch.cat([p[:, :2], torch.full_like(p[:, 2:4], 3.0), torch.zeros_like(p[:, 4:5])], dim=1)
    v = -torch.log(0.01 + background_rate * gaussian_2d(bg, t) + (0.99 - background_rate) * gaussian_2d(p, t))
    return v.reshape(targets.shape[0], len(prim))


def prediction_loss(inputs, targets, batch_split, background_rate=0.2):
    return prediction_loss_values(inputs, targets, batch_split, background_rate).mean()


def l2_loss(inputs, targets, batch_split):
    """Reference lstm/loss.py:93-135 without the collision term: 100 x MSE of the primaries' means."""
    prim = torch.tensor([int(v) for v in batch_split[:-1]])
    return ((inputs[:, prim][:, :, :2] - targets[:, prim]) ** 2).mean() * 100


def collision_loss(positions, batch_split, col_wt=10.0, col_distance=0.2, stats=None):
    """Reference lstm/loss.py:138-162: the primary is penalised for neighbours within col_distance.
    stats["col_margin"]: the smallest |distance - col_distance| over the primary-neighbour pairs (a pair that
    crosses col_distance changes the loss continuously but its gradient by ~col_wt / col_distance)."""
    batch_split = [int(v) for v in batch_split]
    pos = torch.where(torch.isnan(positions[..., :2]), torch.full_like(positions[..., :2], -1000.0), positions[..., :2])
    sizes = torch.as_tensor([b - a for a, b in zip(batch_split[:-1], batch_split[1:])])
    prim_of_row = torch.repeat_interleave(torch.as_tensor(batch_split[:-1]), sizes)
    is_neigh = torch.ones(batch_split[-1], dtype=torch.bool)
    is_neigh[torch.as_tensor(batch_split[:-1])] = False
    dist = torch.norm(pos[:, prim_of_row] - pos.detach(), dim=-1)[:, is_neigh]
    hit = (dist <= col_distance).detach()
    if dist.numel():
        _note(stats, "col_margin", float((dist.detach() - col_distance).abs().min()))
    return col_wt * (1 - dist[hit] / col_distance).sum()


def train_loss_and_grads(W_np, pool_cfg, xy, batch_split, obs_length=9, pred_length=12, dtype=torch.float32,
                         stats=None, loss="pred", col_wt=0.0, col_distance=0.2, feed_back=None, outputs=None):
    """What Trainer.train_batch computes (trainer.py:252-263): teacher-forced forward, the criterion on the
    last pred_length outputs x batch_size; returns (loss, {name: grad ndarray}).  The weights and the
    arithmetic are `dtype`; xy stays fp32 (it is data).  The embedding width is that of W.

    loss: "pred" (PredictionLoss) or "l2" (L2Loss), with the collision term when col_wt > 0 on the
    trainer's primary_prediction (the data with the primaries replaced by the predicted positions); like
    the reference, each loss's multiplier (1 / 100) also scales the collision term.  Or a callable
    loss(rel, positions) -> scalar (not scaled by the batch size).
    stats: see _grid and collision_loss.  feed_back: see forward.  outputs: dict that receives "positions"."""
    W = {k: torch.tensor(v, dtype=dtype, requires_grad=True) for k, v in W_np.items()}
    xy = torch.tensor(xy)
    observed = xy[:obs_length]
    truth = xy[obs_length:-1]
    targets = (xy[obs_length:obs_length + pred_length] - xy[obs_length - 1:obs_length + pred_length - 1]).to(dtype)
    fb = torch.as_tensor(feed_back) if feed_back is not None else None
    rel, positions = forward(W, pool_cfg, observed, batch_split, prediction_truth=truth, dtype=dtype, stats=stats,
                             feed_back=fb)
    if callable(loss):
        total = loss(rel, positions)
    else:
        batch_size = len(batch_split) - 1
        if loss == "pred":
            total, mult = prediction_loss(rel[-pred_length:], targets, batch_split), 1.0
        elif loss == "l2":
            total, mult = l2_loss(rel[-pred_length:], targets, batch_split), 100.0
        else:
            raise ValueError(loss)
        if col_wt:
            prim = torch.tensor([int(v) for v in batch_split[:-1]])
            primary_prediction = xy[-pred_length:].clone()
            primary_prediction[:, prim] = positions[-pred_length:, prim]
            total = total + collision_loss(primary_prediction, batch_split, col_wt, col_distance, stats) * mult
        total = total * batch_size
    total.backward()
    if outputs is not None:
        outputs["positions"] = positions.detach().numpy()
    grads = {k: (v.grad.numpy() if v.grad is not None else None) for k, v in W.items()}
    return float(total.detach()), grads
