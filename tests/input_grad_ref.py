"""Differentiable float64 restatement of LSTM.forward with gradients wrt `observed` -- TEST INFRASTRUCTURE.

tests/torch_ref.py restates the forward for parameter gradients: it treats positions as data (the directional grid's
velocities are detached there, and the decoder's first input frame is a plain clone of observed[-1]).  This module
restates the same forward for the gradient wrt the observed positions, as autograd gives it on the reference's graph
(lstm/lstm.py:170-264) with its deep copy of observed[-1] (:235) read as a detached copy:

  * the velocity input of every step, vel = obs2 - obs1 (:123-125);
  * the directional grid's relative velocities (gridbased_pooling.py:118-140), written with one index_put: every
    writer of a cell, overwritten ones included, receives the cell's gradient; out-of-range pairs write the constant;
  * the hidden states social pooling reads (:145-170), not detached (lstm.py:26);
  * pred = obs2 + mu.

Decoder inputs (teacher-forced truth, the copy of observed[-1], fed-back positions) carry no gradient.  Grid models
only (vanilla, occupancy, directional, social): the non-grid modules have no backward.  Pinned to the unmodified
reference by tests/golden/input_grad_golden.npz (oracle/make_input_grad_golden.py).
"""
import torch
import torch.nn.functional as F

import torch_ref as TR

NAN = float("nan")


def grid(pool_cfg, W, obs1, obs2, hidden, dtype, stats):
    """[B, N, ...] padded -> pooled [B*N, out] (gridbased_pooling.py:94-110,112-170,227-305), cells binned in fp32 on
    the fp32 positions; the grid values keep their graph back to obs1 / obs2 / hidden."""
    B, N, _ = obs2.shape
    n, C = pool_cfg.n, pool_cfg.pooling_dim
    g = torch.full((B * N, n * n, C), float(pool_cfg.constant), dtype=dtype)
    if N > 1:
        obs = obs2.detach().clone()
        obs[torch.isnan(obs).any(dim=-1)] = -500.0
        keep = ~torch.eye(N, dtype=torch.bool)
        rel = (obs[:, None, :, :] - obs[:, :, None, :])[:, keep].reshape(B, N, N - 1, 2)
        oij = rel / float(pool_cfg.cell_side) + torch.tensor([n / 2, 0.0 if pool_cfg.front else n / 2])
        ok = ~(((oij < 0) | (oij >= n)).any(dim=-1))
        oij = torch.where(ok[..., None], oij, torch.zeros_like(oij)).long()
        oi = (oij[..., 0] * n + oij[..., 1]).reshape(B * N, N - 1)
        if pool_cfg.type_ == "social":
            hg = hidden[:, None, :, :].expand(B, N, N, hidden.shape[-1])[:, keep].reshape(B, N, N - 1, -1)
            vals = torch.nan_to_num(hg) @ W["pool.hidden_dim_encoding.weight"].T + W["pool.hidden_dim_encoding.bias"]
        elif pool_cfg.type_ == "directional":
            vel = (obs2 - obs1).to(dtype)
            vals = torch.nan_to_num((vel[:, None, :, :] - vel[:, :, None, :])[:, keep].reshape(B, N, N - 1, 2))
        else:
            vals = torch.ones(B, N, N - 1, 1, dtype=dtype)
        vals = torch.where(ok[..., None], vals, torch.full_like(vals, float(pool_cfg.constant))).reshape(B * N, N - 1, C)
        # the reference's sequential index_put: the last writer of a cell wins the forward, every writer gets the cell's
        # gradient (overwritten ones add v - v.detach(), exactly 0)
        rows = torch.arange(B * N)[:, None].expand(B * N, N - 1)
        win = ~((oi[:, :, None] == oi[:, None, :]) & torch.ones(N - 1, N - 1, dtype=torch.bool).triu(1)).any(dim=-1)
        g = g.index_put((rows[win], oi[win]), vals[win])
        g = g.index_put((rows[~win], oi[~win]), vals[~win] - vals[~win].detach(), accumulate=True)
    # lp_pool2d(p=1, window 1) (:303): identity forward, zero gradient where a cell holds exactly 0
    x = F.lp_pool2d(g.transpose(1, 2).reshape(B * N, C, n, n), 1, 1).reshape(B * N, -1)
    n_layers = {None: 0, "None": 0, "one_layer": 1, "two_layer": 2, "three_layer": 3}[pool_cfg.embedding_arch]
    for layer in range(n_layers):
        z = x @ W["pool.embedding.%d.weight" % (2 * layer)].T + W["pool.embedding.%d.bias" % (2 * layer)]
        TR._note(stats, "relu_pool%d" % layer, float(z.detach().abs().min()))
        x = torch.relu(z)
    return x


def step(W, pool_cfg, phase, h, c, obs1, obs2, bs, hidden_dim, dtype, stats):
    """LSTM.step (lstm.py:91-168) with pool_to_input: rows absent at obs1 or obs2 keep h, c and get normal = NaN."""
    M = obs2.shape[0]
    mask = ~torch.isnan(obs1[:, 0]) & ~torch.isnan(obs2[:, 0])
    e = torch.relu(((obs2 - obs1)[mask].to(dtype) * 4.0) @ W["input_embedding.input_embeddings.0.weight"].T +
                   W["input_embedding.input_embeddings.0.bias"])
    x = torch.cat([e, torch.zeros(e.shape[0], 2, dtype=dtype)], dim=1)
    if pool_cfg is not None:
        pooled = grid(pool_cfg, W, TR._pad(obs1, bs, NAN), TR._pad(obs2, bs, NAN), TR._pad(h, bs, NAN), dtype,
                      stats)[TR._pad(mask, bs, False).reshape(-1)]
        x = torch.cat([x, pooled], dim=1)
    H = hidden_dim
    gates = (x @ W[phase + ".weight_ih"].T + W[phase + ".bias_ih"] + h[mask] @ W[phase + ".weight_hh"].T
             + W[phase + ".bias_hh"])
    i, f = torch.sigmoid(gates[:, :H]), torch.sigmoid(gates[:, H:2 * H])
    g, o = torch.tanh(gates[:, 2 * H:3 * H]), torch.sigmoid(gates[:, 3 * H:])
    c2 = f * c[mask] + i * g
    h2 = o * torch.tanh(c2)
    raw = h2 @ W["hidden2normal.linear.weight"].T + W["hidden2normal.linear.bias"]
    nrm = torch.cat([raw[:, :2], 0.01 + 0.2 * torch.sigmoid(raw[:, 2:4]), 0.7 * torch.sigmoid(raw[:, 4:5])], dim=1)
    idx = mask.nonzero().flatten()
    return (h.index_copy(0, idx, h2), c.index_copy(0, idx, c2),
            torch.full((M, 5), NAN, dtype=dtype).index_copy(0, idx, nrm))


def forward(W, pool_cfg, observed, batch_split, prediction_truth=None, n_predict=None, hidden_dim=128,
            dtype=torch.float64, stats=None, feed_back=None):
    """observed [obs_length, M, 2] fp32 (it may carry a graph: an fp64 leaf cast to fp32).  Returns rel [S, M, 5]
    (`dtype`) and pred [S(+1), M, 2] (fp32).  feed_back: fp32 positions of another implementation's forward, fed to the
    decoder instead of this forward's own (see torch_ref.forward)."""
    bs = [int(v) for v in batch_split]
    M = observed.shape[1]
    prim = torch.tensor(bs[:-1])
    h = torch.zeros(M, hidden_dim, dtype=dtype)
    c = torch.zeros(M, hidden_dim, dtype=dtype)
    truth = [None] * (n_predict - 1) if n_predict is not None else [t.clone() for t in prediction_truth]
    normals, positions = [], ([observed[-1]] if observed.shape[0] == 2 else [])

    def fed(i):
        i = i % len(positions)
        return feed_back[i] if feed_back is not None else positions[i].detach()

    for t in range(observed.shape[0] - 1):
        h, c, normal = step(W, pool_cfg, "encoder", h, c, observed[t], observed[t + 1], bs, hidden_dim, dtype, stats)
        normals.append(normal)
        positions.append(observed[t + 1] + normal[:, :2].to(observed.dtype))
    seq = [observed[-1].detach().clone()] + truth         # the reference's deep copy (lstm.py:235)
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
        h, c, normal = step(W, pool_cfg, "decoder", h, c, obs1, obs2, bs, hidden_dim, dtype, stats)
        normals.append(normal)
        positions.append(obs2 + normal[:, :2].to(obs2.dtype))
    return torch.stack(normals), torch.stack(positions)
