"""Differentiable torch restatement of LSTM.forward + PredictionLoss (fp32 or fp64) -- TEST INFRASTRUCTURE.

Used only to check the hand-written CUDA backward (csrc/train.cu).  Follows oracle/lstm_oracle.py (which is
pinned to the reference) line by line, with torch ops so autograd provides the gradients;
test_training.py and test_social_backward.py pin THIS file's gradients to gradients of the unmodified
reference (tests/golden/train_golden.npz, social_train_golden.npz).
"""
import math

import torch
import torch.nn.functional as F

NAN = float("nan")


def _grid(pool_cfg, W, obs1, obs2, hidden, dtype, stats, primary_edges):
    """[B, N, ...] padded -> pooled [B*N, out] (gridbased_pooling.py:112-170,227-305,308-335), cf.
    oracle.lstm_oracle.occupancy_grid / pool_forward.

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
    x = grid.reshape(B * N, -1)
    n_layers = {"one_layer": 1, "two_layer": 2, "three_layer": 3}[pool_cfg.embedding_arch]
    for l in range(n_layers):
        z = x @ W["pool.embedding.%d.weight" % (2 * l)].T + W["pool.embedding.%d.bias" % (2 * l)]
        _note(stats, "relu_pool%d" % l, float(z.detach().abs().min()))
        x = torch.relu(z)
    return x


def _note(stats, key, value):
    if stats is not None:
        stats[key] = min(value, stats.get(key, math.inf))


def forward(W, pool_cfg, observed, batch_split, prediction_truth=None, n_predict=None, hidden_dim=128,
            dtype=torch.float32, stats=None):
    """W: dict of `dtype` tensors (requires_grad as wanted).  Returns rel [S, M, 5] (`dtype`), pred [S, M, 2]
    (fp32: the positions the model feeds back are fp32 data, as in the reference).  stats: see _grid."""
    bs = [int(v) for v in batch_split]
    B = len(bs) - 1
    M = observed.shape[1]
    n_max = max(bs[i + 1] - bs[i] for i in range(B))
    prim = torch.tensor(bs[:-1])
    h = torch.zeros(M, hidden_dim, dtype=dtype)
    c = torch.zeros(M, hidden_dim, dtype=dtype)
    truth = [None] * (n_predict - 1) if n_predict is not None else [t.clone() for t in prediction_truth]

    def pad(x, fill):
        out = torch.full((B, n_max) + tuple(x.shape[1:]), fill, dtype=x.dtype)
        for b in range(B):
            out[b, :bs[b + 1] - bs[b]] = x[bs[b]:bs[b + 1]]
        return out

    def step(phase, h, c, obs1, obs2):
        mask = ~torch.isnan(obs1[:, 0]) & ~torch.isnan(obs2[:, 0])
        vel = (obs2 - obs1)[mask].to(dtype)
        e = torch.relu((vel * 4.0) @ W["input_embedding.input_embeddings.0.weight"].T +
                       W["input_embedding.input_embeddings.0.bias"])
        x = torch.cat([e, torch.zeros(e.shape[0], 2, dtype=dtype)], dim=1)
        if pool_cfg is not None:
            pooled = _grid(pool_cfg, W, pad(obs1, NAN), pad(obs2, NAN), pad(h, NAN), dtype, stats,
                           primary_edges=phase == "decoder")
            x = torch.cat([x, pooled[pad(mask, False).reshape(-1)]], dim=1)
        gates = x @ W[phase + ".weight_ih"].T + W[phase + ".bias_ih"] + h[mask] @ W[phase + ".weight_hh"].T + W[phase + ".bias_hh"]
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

    normals, positions = [], []
    if observed.shape[0] == 2:
        positions = [observed[-1]]
    for t in range(observed.shape[0] - 1):
        h, c, normal = step("encoder", h, c, observed[t], observed[t + 1])
        normals.append(normal)
        positions.append(observed[t + 1] + normal[:, :2].to(observed.dtype))
    seq = [observed[-1].clone()] + truth
    for k in range(len(seq) - 1):
        obs1, obs2 = seq[k], seq[k + 1]
        if obs1 is None:
            obs1 = positions[-2].detach()
        else:
            obs1 = obs1.clone()
            obs1[prim] = positions[-2][prim].detach()
        if obs2 is None:
            obs2 = positions[-1].detach()
        else:
            obs2 = obs2.clone()
            obs2[prim] = positions[-1][prim].detach()
            seq[k + 1] = obs2
        h, c, normal = step("decoder", h, c, obs1, obs2)
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


def collision_loss(positions, batch_split, col_wt=10.0, col_distance=0.2):
    """Reference lstm/loss.py:138-162: the primary is penalised for neighbours within col_distance."""
    batch_split = [int(v) for v in batch_split]
    pos = torch.where(torch.isnan(positions[..., :2]), torch.full_like(positions[..., :2], -1000.0), positions[..., :2])
    sizes = torch.as_tensor([b - a for a, b in zip(batch_split[:-1], batch_split[1:])])
    prim_of_row = torch.repeat_interleave(torch.as_tensor(batch_split[:-1]), sizes)
    is_neigh = torch.ones(batch_split[-1], dtype=torch.bool)
    is_neigh[torch.as_tensor(batch_split[:-1])] = False
    dist = torch.norm(pos[:, prim_of_row] - pos.detach(), dim=-1)[:, is_neigh]
    hit = (dist <= col_distance).detach()
    return col_wt * (1 - dist[hit] / col_distance).sum()


def train_loss_and_grads(W_np, pool_cfg, xy, batch_split, obs_length=9, pred_length=12, dtype=torch.float32,
                         stats=None):
    """What Trainer.train_batch computes (trainer.py:252-263): teacher-forced forward, PredictionLoss
    on the last pred_length outputs x batch_size; returns (loss, {name: grad ndarray}).  The weights and
    the arithmetic are `dtype`; xy stays fp32 (it is data).  stats: see _grid."""
    W = {k: torch.tensor(v, dtype=dtype, requires_grad=True) for k, v in W_np.items()}
    xy = torch.tensor(xy)
    observed = xy[:obs_length]
    truth = xy[obs_length:-1]
    targets = (xy[obs_length:obs_length + pred_length] - xy[obs_length - 1:obs_length + pred_length - 1]).to(dtype)
    rel, _ = forward(W, pool_cfg, observed, batch_split, prediction_truth=truth, dtype=dtype, stats=stats)
    batch_size = len(batch_split) - 1
    loss = prediction_loss(rel[-pred_length:], targets, batch_split) * batch_size
    loss.backward()
    grads = {k: (v.grad.numpy() if v.grad is not None else None) for k, v in W.items()}
    return float(loss.detach()), grads
