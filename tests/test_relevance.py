"""lstm.explain.relevance / tb2_lstm_relevance: layer-wise relevance of a free-running forecast, against a float64
restatement of the rules (lstm/explain.py's docstring) written here from the forward's own quantities.

The restatement runs the forward in float64 with the decoder fed the GPU's positions (so every grid cell is binned
alike), keeps each primary's per-step records (gate operand, gate pre-activations, grid, embedding layers, winners) and
applies the rules explicitly, with the eps-rule's denominators taken from the pre-activations.  Device comparisons run
at eps = 2e-2, which keeps every |z'| the rules divide by at least 2e-2 away from 0; the restatement also checks that no
gate or cell pre-activation of an explained chain is so close to 0 that fp32 could see the other sign of it.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import lstm_oracle as O  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 2e-2
TOL = 2e-3             # max |gpu - float64| / max |float64| per tensor
f32 = np.float32


def _is_bias(name):
    return name.split(".")[-1].startswith("bias")


def _stab(z, eps):
    return z + eps * np.where(z >= 0, 1.0, -1.0)


def _cfg(kind):
    return O.pool_config(kind) if O.MODEL_SPECS[kind] is not None else None


def _layers(W):
    out = []
    for l in range(3):
        if "pool.embedding.%d.weight" % (2 * l) in W:
            out.append((W["pool.embedding.%d.weight" % (2 * l)], W["pool.embedding.%d.bias" % (2 * l)]))
    return out


def _winners(p32, i, n_s, n_slots, cfg):
    """{cell: scene-local j} of observer i's grid: last writer in ascending neighbour slot wins; an out-of-range writer
    (a padded slot too) leaves cell 0 at the constant"""
    n = cfg.n
    offx, offy = f32(n / 2), f32(0.0 if cfg.front else n / 2)
    side = f32(cfg.cell_side)
    win = {}
    for jj in range(n_slots - 1):
        j = jj + (jj >= i)
        pj = p32[j] if j < n_s else np.array([-500, -500], dtype=f32)
        ox = f32(f32(f32(pj[0] - p32[i][0]) / side) + offx)
        oy = f32(f32(f32(pj[1] - p32[i][1]) / side) + offy)
        if ox < 0 or ox >= n or oy < 0 or oy >= n:
            win.pop(0, None)
        else:
            win[int(ox) * n + int(oy)] = j
    return win


def _step_inputs(observed, pos_steps, bs, s):
    """(obs1, obs2) of step s as the forward resolves them (the decoder reads its own fed-back positions)"""
    obs_length = observed.shape[0]
    if s < obs_length - 1:
        return observed[s], observed[s + 1]
    pm2 = pos_steps[s - 2] if s >= 2 else observed[-1]
    if s == obs_length - 1:
        o1 = observed[-1].copy()
        o1[bs[:-1]] = pm2[bs[:-1]]
    else:
        o1 = pm2
    return o1, pos_steps[s - 1]


def restate(W, cfg, observed, bs, n_predict, H, pos_steps, eps, pad=False, mistake=None, biases=True):
    """float64 relevance [n_predict, S, M], explained [n_predict, B] and the smallest |z| of the explained chains' g-gate
    and cell pre-activations.  pos_steps: the GPU's positions of the S steps.  mistake: None, 'f_gate' (relevance also
    sent through the f gate), 'lost_winner' (the largest cell of each grid loses its winner), 'no_relu' (the grid rule
    takes the embedding's pre-activations as its values: no ReLU mask)."""
    W = {k: np.asarray(v, dtype=np.float64) * (1.0 if biases or not _is_bias(k) else 0.0) for k, v in W.items()}
    observed = np.asarray(observed, dtype=f32)
    bs = np.asarray(bs)
    obs_length, M = observed.shape[0], observed.shape[1]
    B = len(bs) - 1
    S_enc = obs_length - 1
    S = S_enc + n_predict - 1
    n_max = int(np.max(np.diff(bs)))
    We, be = W["input_embedding.input_embeddings.0.weight"], W["input_embedding.input_embeddings.0.bias"]
    E = We.shape[0] + 2
    layers = _layers(W) if cfg is not None else []
    h, c = np.zeros((M, H)), np.zeros((M, H))
    recs = []
    hs = []
    for s in range(S):
        o1, o2 = _step_inputs(observed, pos_steps, bs, s)
        phase = "encoder" if s < S_enc else "decoder"
        mask = ~np.isnan(o1[:, 0]) & ~np.isnan(o2[:, 0])
        v32 = (o2 - o1).astype(f32)
        vel4 = np.nan_to_num((v32 * f32(4.0)).astype(np.float64))
        zemb = vel4 @ We.T + be
        emb = np.concatenate([np.maximum(zemb, 0), np.zeros((M, 2))], axis=1)
        pooled = np.zeros((M, 0))
        grids = {}
        if cfg is not None:
            p32 = np.where(np.isnan(o2), f32(-500), o2).astype(f32)
            if cfg.type_ == "social":
                vals = np.nan_to_num(h) @ W["pool.hidden_dim_encoding.weight"].T + W["pool.hidden_dim_encoding.bias"]
            C, cells = cfg.pooling_dim, cfg.n * cfg.n
            pooled = np.zeros((M, layers[-1][0].shape[0]))
            for b in range(B):
                r0, n_s = bs[b], bs[b + 1] - bs[b]
                for i in range(n_s):
                    win = _winners(p32[r0:r0 + n_s], i, n_s, n_max if pad else n_s, cfg)
                    G = np.zeros((C, cells))
                    for cell, j in win.items():
                        if j >= n_s:          # a padded slot wins only in the row of an absent observer
                            continue
                        if cfg.type_ == "occupancy":
                            G[0, cell] = 1.0
                        elif cfg.type_ == "directional":
                            G[:, cell] = np.nan_to_num((v32[r0 + j] - v32[r0 + i]).astype(np.float64))
                        else:
                            G[:, cell] = vals[r0 + j]
                    acts, pre = [G.reshape(-1)], []
                    for w, bb in layers:
                        pre.append(w @ acts[-1] + bb)
                        acts.append(np.maximum(pre[-1], 0))
                    pooled[r0 + i] = acts[-1]
                    if i == 0:
                        grids[b] = (win, acts, pre)
        X = np.concatenate([emb, pooled, h], axis=1)
        Wih, Whh = W[phase + ".weight_ih"], W[phase + ".weight_hh"]
        gp = X[:, :E + pooled.shape[1]] @ Wih.T + W[phase + ".bias_ih"] + h @ Whh.T + W[phase + ".bias_hh"]
        sg = lambda x: 1 / (1 + np.exp(-x))
        ig, fg, gg, og = sg(gp[:, :H]), sg(gp[:, H:2 * H]), np.tanh(gp[:, 2 * H:3 * H]), sg(gp[:, 3 * H:])
        c2 = fg * c + ig * gg
        h2 = og * np.tanh(c2)
        recs.append(dict(mask=mask, X=X, gp=gp, c_prev=c.copy(), vel4=vel4, zemb=zemb, grids=grids, phase=phase))
        h = np.where(mask[:, None], h2, h)
        c = np.where(mask[:, None], c2, c)
        hs.append(h.copy())
    Wn, bn = W["hidden2normal.linear.weight"], W["hidden2normal.linear.bias"]
    rel = np.zeros((n_predict, S, M))
    explained = np.zeros((n_predict, B))
    zmin = np.inf
    P = X.shape[1] - E - H
    for t in range(n_predict):
        st = obs_length - 2 + t
        for b in range(B):
            m = bs[b]
            if not recs[st]["mask"][m]:
                continue
            hh = hs[st][m]
            mu = Wn[:2] @ hh + bn[:2]
            y = float(np.hypot(*mu))
            if not (y > 0 and np.isfinite(y)):
                continue
            explained[t, b] = y
            d = mu / y
            Rh = hh * (d @ Wn[:2]) / (y + eps) * y
            Rc = np.zeros(H)
            for s in range(st, -1, -1):
                r = recs[s]
                if not r["mask"][m]:
                    continue
                gp = r["gp"][m]
                i_, f_, g_ = 1 / (1 + np.exp(-gp[:H])), 1 / (1 + np.exp(-gp[H:2 * H])), np.tanh(gp[2 * H:3 * H])
                cp = r["c_prev"][m]
                cz = f_ * cp + i_ * g_
                zmin = min(zmin, float(np.abs(cz).min()), float(np.abs(gp[2 * H:3 * H]).min()))
                Rtot = Rh + Rc
                Rc = f_ * cp / _stab(cz, eps) * Rtot
                Rg = i_ * g_ / _stab(cz, eps) * Rtot
                Wih, Whh = W[r["phase"] + ".weight_ih"], W[r["phase"] + ".weight_hh"]
                V = Rg / _stab(gp[2 * H:3 * H], eps)
                Qin, Qh = V @ Wih[2 * H:3 * H], V @ Whh[2 * H:3 * H]
                if mistake == "f_gate":
                    Vf = Rg / _stab(gp[H:2 * H], eps)
                    Qin, Qh = Qin + Vf @ Wih[H:2 * H], Qh + Vf @ Whh[H:2 * H]
                X = r["X"][m]
                Rh = X[E + P:] * Qh
                Remb = X[:E - 2] * Qin[:E - 2]
                Vemb = np.where(X[:E - 2] > 0, Remb / _stab(r["zemb"][m], eps), 0.0)
                rel[t, s, m] = float((r["vel4"][m] * (Vemb @ We)).sum())
                if cfg is None:
                    continue
                win, acts, pre = r["grids"][b]
                top = pre[-1] if mistake == "no_relu" else acts[-1]
                R = top * Qin[E:E + P]
                for l in range(len(layers) - 1, -1, -1):
                    live = pre[l] > 0 if mistake != "no_relu" else pre[l] != 0
                    Vl = np.where(live, R, 0.0) / np.where(live, _stab(pre[l], eps), 1.0)
                    R = acts[l] * (Vl @ layers[l][0])
                Rcell = R.reshape(cfg.pooling_dim, -1).sum(axis=0)
                lost = int(np.argmax(np.abs(Rcell))) if mistake == "lost_winner" else -1
                for cell, j in win.items():
                    if cell != lost:
                        rel[t, s, m + j] += Rcell[cell]
    return rel, explained, zmin


def _inputs(kind, B, N, obs_length, n_predict, seed, H=128, biases=True):
    xy, bs = O.synthetic_scenes(B, N, n_frames=obs_length + n_predict, seed=seed, ragged=True, nan_tracks=True)
    W = O.random_weights(kind, seed=seed, hidden_dim=H, relu_bias=3.0)
    if not biases:
        W = {k: (v * 0 if _is_bias(k) else v) for k, v in W.items()}
    return xy[:obs_length].astype(f32), bs, W


def _model(kind, W, H):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    spec = O.MODEL_SPECS[kind]
    pool = GridBasedPooling(**dict(spec, hidden_dim=H)) if spec is not None else None
    model = LSTM(hidden_dim=H, pool=pool)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v, dtype=f32).copy()) for k, v in W.items()})
    return model


def _rel_err(got, ref):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert np.isfinite(got).all() and np.isfinite(ref).all()
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def _gate(got, ref, bs):
    """the larger error of the two tensors a relevance array holds: the primaries' own columns and the neighbours'"""
    own = np.zeros(ref.shape[-1], dtype=bool)
    own[np.asarray(bs[:-1])] = True
    errs = [_rel_err(got[..., own], ref[..., own])]
    if (~own).any() and np.abs(ref[..., ~own]).max() > 0:
        errs.append(_rel_err(got[..., ~own], ref[..., ~own]))
    return max(errs)


def _self_positions(W, cfg, observed, bs, n_predict, H):
    """the restatement's own fed-back positions (float64 forward through torch_ref), for the CPU cases"""
    import torch_ref as TR
    W64 = {k: torch.tensor(v, dtype=torch.float64) for k, v in W.items()}
    _, pos = TR.forward(W64, cfg, torch.from_numpy(observed), bs, n_predict=n_predict, hidden_dim=H,
                        dtype=torch.float64, pad_to_batch_max=False)
    S = observed.shape[0] - 1 + n_predict - 1
    return pos.numpy().astype(f32)[-S:]


# ---------------------------------------------------------------------------------------------------------- CPU cases
@pytest.mark.parametrize("kind", ["vanilla", "occupancy", "directional", "social_default", "social_d96"])
def test_conservation_without_biases_and_eps(kind):
    observed, bs, W = _inputs(kind, 3, 5, 9, 4, seed=3, H=64, biases=False)
    cfg = _cfg(kind)
    pos = _self_positions(W, cfg, observed, bs, 4, 64)
    rel, expl, _ = restate(W, cfg, observed, bs, 4, 64, pos, 0.0, biases=False)
    summed = np.stack([rel[:, :, bs[b]:bs[b + 1]].sum(axis=(1, 2)) for b in range(len(bs) - 1)], axis=1)
    assert (expl > 0).any()
    assert np.abs(summed - expl).max() <= 1e-10 * max(1.0, np.abs(expl).max()), kind


def _two_track_scene(offsets, obs_length=9):
    """primary walking along x from the origin, neighbours at fixed offsets from it"""
    T = obs_length
    prim = np.stack([np.arange(T) * 0.3, np.zeros(T)], axis=1)
    tracks = [prim] + [prim + np.asarray(o) for o in offsets]
    return np.stack(tracks, axis=1).astype(f32), np.array([0, 1 + len(offsets)])


def test_known_cell_and_overwritten_writer():
    kind, H, n_predict = "directional", 64, 3
    cfg = _cfg(kind)
    W = O.random_weights(kind, seed=4, hidden_dim=H, relu_bias=3.0)
    # one neighbour 0.9 m to the side: every step it sits in one cell of the primary's grid, and takes all the
    # neighbour relevance
    observed, bs = _two_track_scene([(0.0, 0.9)])
    observed[:, 1, 0] += np.arange(observed.shape[0]) * 0.05          # a relative velocity: non-zero grid values
    pos = _self_positions(W, cfg, observed, bs, n_predict, H)
    rel, expl, _ = restate(W, cfg, observed, bs, n_predict, H, pos, 1e-3)
    win = _winners(observed[0], 0, 2, 2, cfg)
    assert list(win.values()) == [1]
    assert np.abs(rel[:, :, 1]).max() > 0
    # two neighbours in the same cell: the later slot wins, the overwritten one gets exactly 0
    observed, bs = _two_track_scene([(0.0, 0.9), (0.05, 0.95)])
    observed[:, 1:, 0] += np.arange(observed.shape[0])[:, None] * 0.05
    pos = _self_positions(W, cfg, observed, bs, n_predict, H)
    rel, _, _ = restate(W, cfg, observed, bs, n_predict, H, pos, 1e-3)
    win = _winners(observed[0], 0, 3, 3, cfg)
    assert list(win.values()) == [2]
    assert np.all(rel[:, :, 1] == 0.0)
    assert np.abs(rel[:, :, 2]).max() > 0


@pytest.mark.parametrize("mistake,kind", [("f_gate", "directional"), ("lost_winner", "occupancy"),
                                          ("no_relu", "social_d96")])
def test_gate_fails_for_emulated_mistakes(mistake, kind):
    observed, bs, W = _inputs(kind, 3, 6, 9, 4, seed=5, H=64)
    cfg = _cfg(kind)
    pos = _self_positions(W, cfg, observed, bs, 4, 64)
    ref, expl, _ = restate(W, cfg, observed, bs, 4, 64, pos, EPS)
    bad, _, _ = restate(W, cfg, observed, bs, 4, 64, pos, EPS, mistake=mistake)
    assert _gate(bad, ref, bs) > 10 * TOL, mistake


def test_refusals_before_any_launch():
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM, HiddenStateMLPPooling
    from trajnetplusplusbaselines_b200.lstm.explain import relevance
    bad = [LSTM(goal_flag=True), LSTM(pool=HiddenStateMLPPooling()),
           LSTM(pool=GridBasedPooling(type_="occupancy", embedding_arch="three_layer", layer_dims=[64, 32])),
           LSTM(pool=GridBasedPooling(type_="directional", constant=1)),
           LSTM(pool=GridBasedPooling(type_="occupancy"), pool_to_input=False)]
    for model in bad:
        with pytest.raises(NotImplementedError):
            relevance(model, torch.zeros(9, 2, 2), torch.tensor([0, 2]))


def _write_ndjson(path, n_scenes=3, n_peds=4, frames=21, seed=0):
    rs = np.random.RandomState(seed)
    lines = []
    for s in range(n_scenes):
        peds = list(range(10 * s, 10 * s + n_peds))
        for f in range(frames):
            for k, p in enumerate(peds):
                if k == n_peds - 1 and f < 3:
                    continue
                lines.append(json.dumps({"track": {"f": f * 10, "p": p, "x": round(0.4 * f + k + rs.randn() * 0.01, 3),
                                                   "y": round(0.5 * k, 3)}}))
        lines.append(json.dumps({"scene": {"id": s, "p": peds[0], "s": 0, "e": (frames - 1) * 10, "fps": 2.5,
                                           "tag": [1, []]}}))
    with open(path, "w") as fh:
        fh.write("\n".join(lines) + "\n")


def _cli(args):
    return subprocess.run([sys.executable, "-m", "trajnetplusplusbaselines_b200.lstm.explain"] + args, cwd=ROOT,
                          capture_output=True, text=True)


def _save(model, path):
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    LSTMPredictor(model).save(None, path)


def test_cli_refuses_before_reading_input(tmp_path):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    missing = str(tmp_path / "absent.ndjson")
    model_path = str(tmp_path / "m.pkl")
    _save(LSTM(pool=GridBasedPooling(type_="directional", constant=1)), model_path)
    out = _cli(["--model", model_path, "--input", missing, "--output", str(tmp_path / "r.npz")])
    assert out.returncode != 0 and "constant" in out.stderr, out.stderr
    _save(LSTM(), model_path)
    out = _cli(["--model", model_path, "--input", missing, "--output", str(tmp_path / "r.npz"), "--eps", "-1"])
    assert out.returncode != 0 and "--eps" in out.stderr, out.stderr
    out = _cli(["--model", model_path, "--input", missing, "--output", str(tmp_path / "r.npz"), "--n_predict", "0"])
    assert out.returncode != 0 and "--n_predict" in out.stderr, out.stderr


# ---------------------------------------------------------------------------------------------------------- GPU cases
def _tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")


def _run(model, observed, bs, n_predict, eps, pad=True):
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm.explain import relevance
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 16)
    lib.tb2_profile_begin()
    try:
        res = relevance(model, torch.from_numpy(observed).cuda(), torch.from_numpy(bs), n_predict, eps,
                        pad_to_batch_max=pad)
        torch.cuda.synchronize()
    finally:
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
    return res, set(json.loads(buf.value.decode()))


def _case(name, kind, H=128, obs_length=9, n_predict=12, data=(6, 8), seed=1, pad=True):
    return (name, kind, H, obs_length, n_predict, data, seed, pad)


GPU_CASES = [
    _case("vanilla", "vanilla", seed=3),
    _case("occupancy", "occupancy", seed=2),
    _case("directional", "directional", seed=3),
    _case("social_one_l16", "social_default", data=(4, 8), seed=4),
    _case("social_two_1024_n16", "social", data=(3, 6), seed=5),
    _case("dir_h64", "directional", H=64, seed=6),
    _case("social_h96", "social_d96", H=96, data=(4, 6), seed=7),
    _case("occ_h256", "occupancy", H=256, seed=10),
    _case("dir_ragged_60", "directional", data=(3, 60), seed=9, pad=False),
    _case("occ_obs2_pred1", "occupancy", obs_length=2, n_predict=1, seed=10),
    _case("social_obs2_pred1", "social_d96", obs_length=2, n_predict=1, data=(4, 6), seed=11),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_relevance_matches_float64_restatement(monkeypatch, case, tc):
    name, kind, H, obs_length, n_predict, (B, N), seed, pad = case
    _tc(monkeypatch, tc)
    observed, bs, W = _inputs(kind, B, N, obs_length, n_predict, seed, H=H)
    if name == "dir_ragged_60":       # scenes of 1 to 60 tracks
        observed, bs = observed[:, :61], np.array([0, 1, 31, 61])
    cfg = _cfg(kind)
    model = _model(kind, W, H).cuda().eval()
    res, kernels = _run(model, observed, bs, n_predict, EPS, pad)
    want = {"bwd_gather", "rel_head", "rel_cell", "rel_operand", "rel_gemm", "bwd_gemm"}
    if cfg is not None:
        want |= {"pool_prepare", "rel_owner", "rel_relu_scale", "rel_neighbours"}
    if cfg is not None and cfg.type_ == "social":
        want.add("rel_social_grid")
    assert want <= kernels, (name, want - kernels)
    S = obs_length - 1 + n_predict - 1
    pos = res.positions.cpu().numpy()[-S:]
    ref, expl, zmin = restate(W, cfg, observed, bs, n_predict, H, pos, EPS, pad=pad)
    assert zmin > 3e-6, (name, zmin)
    e_rel = _gate(res.relevance.cpu().numpy(), ref, bs)
    e_expl = _rel_err(res.explained.cpu().numpy(), expl)
    print("%s [%s]: relevance %.2e explained %.2e" % (name, "tc" if tc else "no_tc", e_rel, e_expl))
    assert e_rel <= TOL and e_expl <= TOL, (name, e_rel, e_expl)
    if cfg is not None and name != "occ_obs2_pred1":
        nb = np.ones(observed.shape[1], dtype=bool)
        nb[bs[:-1]] = False
        assert np.abs(res.relevance.cpu().numpy()[:, :, nb]).max() > 0, name


@pytest.mark.gpu
def test_properties():
    from trajnetplusplusbaselines_b200.lstm.explain import relevance
    kind, H, n_predict = "directional", 128, 12
    observed, bs, W = _inputs(kind, 6, 8, 9, n_predict, seed=12, H=H)
    model = _model(kind, W, H).cuda().eval()
    obs = torch.from_numpy(observed).cuda()
    split = torch.from_numpy(bs)
    a = relevance(model, obs, split, n_predict)
    b = relevance(model, obs, split, n_predict)
    assert torch.equal(a.relevance, b.relevance) and torch.equal(a.explained, b.explained)
    # the forecast is model(...)'s, bit for bit
    with torch.no_grad():
        nrm, pos = model(obs, None, split, n_predict=n_predict)
    assert torch.equal(torch.nan_to_num(a.normals, 7.0), torch.nan_to_num(nrm, 7.0))
    assert torch.equal(torch.nan_to_num(a.positions, 7.0), torch.nan_to_num(pos, 7.0))
    # the residual is y minus the scene's summed relevance (what the biases and eps absorbed; without biases it vanishes
    # as eps -> 0, test_conservation_without_biases_and_eps)
    assert (a.explained > 0).all()
    summed = torch.stack([a.relevance[:, :, bs[i]:bs[i + 1]].double().sum(dim=(1, 2)) for i in range(len(bs) - 1)], 1)
    assert float((a.residual.double() - (a.explained.double() - summed)).abs().max()) <= 1e-6 * float(a.explained.max())
    # per-scene layout: the batched call equals per-scene calls bit for bit
    full = relevance(model, obs, split, n_predict, pad_to_batch_max=False)
    for i in range(len(bs) - 1):
        one = relevance(model, obs[:, bs[i]:bs[i + 1]].contiguous(), torch.tensor([0, bs[i + 1] - bs[i]]), n_predict,
                        pad_to_batch_max=False)
        assert torch.equal(one.relevance, full.relevance[:, :, bs[i]:bs[i + 1]]), i
        assert torch.equal(one.explained[:, 0], full.explained[:, i]), i
    # a one-track scene: only its own column is non-zero
    one = relevance(model, obs[:, :1].contiguous(), torch.tensor([0, 1]), n_predict)
    assert one.relevance.abs().max() > 0
    # vanilla: every neighbour column exactly 0
    Wv = O.random_weights("vanilla", seed=12, hidden_dim=H)
    van = relevance(_model("vanilla", Wv, H).cuda().eval(), obs, split, n_predict)
    nb = torch.ones(observed.shape[1], dtype=torch.bool)
    nb[split[:-1]] = False
    assert torch.all(van.relevance[:, :, nb.cuda()] == 0)
    # a neighbour far away never wins a cell and gets exactly 0
    far = observed[:, :3].copy()
    far[:, 2] = far[:, 0] + 50.0
    r = relevance(model, torch.from_numpy(far).cuda(), torch.tensor([0, 3]), n_predict)
    assert torch.all(r.relevance[:, :, 2] == 0)


@pytest.mark.gpu
def test_cli_end_to_end(tmp_path):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    from trajnetplusplusbaselines_b200.lstm.explain import explain_scenes
    from trajnetplusplusbaselines_b200.data import load_test_scenes_xy
    src = str(tmp_path / "test.ndjson")
    _write_ndjson(src)
    model_path = str(tmp_path / "m.pkl")
    torch.manual_seed(0)
    model = LSTM(pool=GridBasedPooling(type_="directional"))
    _save(model, model_path)
    out_path = str(tmp_path / "rel.npz")
    out = _cli(["--model", model_path, "--input", src, "--output", out_path, "--n_predict", "12", "--normalize_scene"])
    assert out.returncode == 0, out.stderr
    z = np.load(out_path)
    scenes = load_test_scenes_xy(src, 9)
    assert int(z["num_scenes"]) == len(scenes) == 3
    api = explain_scenes(model.cuda(), [xy for xy, _ in scenes], 12, 9, 1e-3, normalize_scene=True)
    for i, ((xy, meta), (rel, expl, resid)) in enumerate(zip(scenes, api)):
        assert int(z["scene_id_%d" % i]) == meta.scene_id
        assert list(z["ped_ids_%d" % i]) == [meta.pedestrian] + list(meta.neigh_ids)
        assert z["relevance_%d" % i].shape == rel.shape == (12, 19, xy.shape[1])
        assert z["explained_%d" % i].shape == expl.shape == (12,)
        assert z["residual_%d" % i].shape == resid.shape == (12,)
        np.testing.assert_array_equal(z["relevance_%d" % i], rel)
