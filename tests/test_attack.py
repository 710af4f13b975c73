"""The collision attack (attack.py, csrc/attack.cu): the objective and step kernels against float64 restatements, the
batched attack end to end, and its CLI."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

LIMIT = 0.2


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatements
# ---------------------------------------------------------------------------------------------------------------------
def objective_ref(pos, split, first):
    """D [B] and its subgradient [F, M, 2] as tb2_attack_objective defines them (metrics.cu `collides` geometry)."""
    pos = np.asarray(pos, dtype=np.float64)
    F, M = pos.shape[:2]
    D = np.full(len(split) - 1, np.inf)
    grad = np.zeros((F, M, 2))
    for b in range(len(split) - 1):
        r0, best, arg = split[b], np.inf, None
        for j in range(r0 + 1, split[b + 1]):
            prev = -1
            for t in range(first, F):
                if not (np.isfinite(pos[t, r0]).all() and np.isfinite(pos[t, j]).all()):
                    continue
                if prev >= 0:
                    p1, p2, p3, p4 = pos[prev, r0], pos[t, r0], pos[prev, j], pos[t, j]
                    a = [p1, p1 + (p2 - p1) / 2.0, p2]
                    c = [p3, p3 + (p4 - p3) / 2.0, p4]
                    for k in range(3):
                        d = np.sqrt((a[k][0] - c[k][0]) ** 2 + (a[k][1] - c[k][1]) ** 2)
                        if d < best:
                            best, arg = d, (j, prev, t, k, (a[k] - c[k]))
                prev = t
        D[b] = best
        if arg is not None and best > 0:
            j, prev, t, k, diff = arg
            u, w = diff / best, 0.5 * k
            grad[prev, r0], grad[t, r0] = (1 - w) * u, w * u
            grad[prev, j], grad[t, j] = -(1 - w) * u, -w * u
    return D, grad


def step_ref(d_obs, obs, delta, D, best_D, split, eps, alpha, move):
    delta, best_D = delta.astype(np.float64).copy(), best_D.copy()
    improved = D < best_D
    best_D[improved] = D[improved]
    if move:
        for b, r0 in enumerate(split[:-1]):
            if best_D[b] <= LIMIT:
                continue
            for t in range(obs.shape[0]):
                g = d_obs[t, r0].astype(np.float64)
                gn = np.sqrt(g[0] * g[0] + g[1] * g[1])
                if not (np.isfinite(obs[t, r0]).all() and np.isfinite(gn) and gn > 0):
                    continue
                v = delta[t, b] - alpha * (g / gn)
                vn = np.sqrt(v[0] * v[0] + v[1] * v[1])
                if vn > eps:
                    v = v * (eps / vn)
                delta[t, b] = v
    return delta, best_D, improved


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ---------------------------------------------------------------------------------------------------------------------
_LAYOUTS = []


def _layout(split):
    from trajnetplusplusbaselines_b200.engine import LayoutCache
    if not _LAYOUTS:
        _LAYOUTS.append(LayoutCache())
    return _LAYOUTS[0].get(torch.from_numpy(np.asarray(split, dtype=np.int64)), pad_to_batch_max=False,
                             device=torch.device("cuda"))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _random_predictions(seed, sizes, F=13):
    rs = np.random.RandomState(seed)
    split = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    M = int(split[-1])
    pos = (rs.randn(M, 2)[None] * 1.5 + np.cumsum(rs.randn(F, M, 2) * 0.1, axis=0)).astype(np.float32)
    for b in range(len(sizes)):            # NaN frames of neighbours, one whole NaN neighbour, an exact tie
        if sizes[b] > 2:
            pos[rs.randint(0, F, 3), split[b] + 1] = np.nan
            pos[:, split[b] + 2] = np.nan
        if sizes[b] > 4:
            pos[:, split[b] + 4] = pos[:, split[b] + 3]
    return pos, split


@pytest.mark.gpu
def test_objective_matches_float64_and_the_scorer():
    from trajnetplusplusbaselines_b200 import _lib, scoring
    lib = _lib.load()
    sizes = [1, 2, 3, 5, 7, 6, 2, 4] * 8
    pos, split = _random_predictions(3, sizes)
    first = 1
    layout = _layout(split)
    P = torch.from_numpy(pos).cuda()
    D = torch.empty(len(sizes), dtype=torch.float64, device="cuda")
    G = torch.full_like(P, 5.0)
    _lib.check(lib.tb2_attack_objective(layout.handle, _p(P), pos.shape[0], first, _p(D), _p(G), None))
    D_ref, G_ref = objective_ref(pos, split, first)
    Dg = D.cpu().numpy()
    assert np.array_equal(np.isinf(Dg), np.isinf(D_ref))
    fin = np.isfinite(D_ref)
    assert np.abs(Dg[fin] - D_ref[fin]).max() <= 1e-12          # measured: one ulp
    assert np.abs(G.cpu().numpy() - G_ref).max() <= 1e-6
    assert np.isinf(D_ref[0]) and np.all(G.cpu().numpy()[:, 0] == 0)         # a single-track scene
    # D <= 0.2 m <=> the scorer's Col-I, away from the threshold
    T = pos.shape[0] - first
    pr = pos[first:].astype(np.float64)
    nb_off = np.concatenate([[0], np.cumsum(np.asarray(sizes) - 1)]).astype(np.int32)
    nb = np.concatenate([pr[:, split[b] + 1:split[b + 1]].transpose(1, 0, 2) for b in range(len(sizes))])
    mask = np.isfinite(nb).all(axis=-1).astype(np.uint8)
    a = dict(gt_primary=pr[:, split[:-1]].transpose(1, 0, 2).copy(), pred_primary=pr[:, split[:-1]].transpose(1, 0, 2)[:, None].copy(),
             num_modes=np.ones(len(sizes), dtype=np.int32), gt_neigh_off=np.zeros(len(sizes) + 1, dtype=np.int32),
             gt_neigh=np.empty((0, T, 2)), gt_neigh_mask=np.empty((0, T), np.uint8), pred_neigh_off=nb_off,
             pred_neigh=np.nan_to_num(nb), pred_neigh_mask=mask)
    flags = scoring.score_arrays(a, False)['flags']
    hit = (flags & _lib.SCORE_COL_PRED) != 0
    far = np.abs(D_ref - LIMIT) > 1e-6
    assert np.array_equal(hit[far], (D_ref <= LIMIT)[far])
    assert hit.any() and (~hit).any()


@pytest.mark.gpu
def test_step_matches_float64_and_keeps_the_rules():
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(5)
    sizes = [3, 1, 4, 2, 5, 3, 2, 6]
    split = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    B, M, L, F = len(sizes), int(split[-1]), 9, 13
    obs = rs.randn(L, M, 2).astype(np.float32)
    obs[4, split[2]] = np.nan                                    # a NaN frame of a primary
    d_obs = rs.randn(L, M, 2).astype(np.float32)
    d_obs[2, split[3]] = 0.0                                     # g = 0
    eps, alpha = 0.1, 0.03
    delta = rs.randn(L, B, 2) * 0.05
    delta = (delta * np.minimum(1.0, 0.1 / np.sqrt((delta ** 2).sum(-1, keepdims=True)))).astype(np.float32)
    D = np.array([0.5, np.inf, 0.3, 0.15, 0.7, 0.7, 0.4, 0.9])
    best_D = np.array([0.6, np.inf, 0.3, 0.5, 0.1, 0.8, 0.4, 1.0])   # ties keep the earlier; scene 4 is frozen
    pos = rs.randn(F, M, 2).astype(np.float32)
    t = {k: torch.from_numpy(v.copy()).cuda() for k, v in dict(d_obs=d_obs, obs=obs, delta=delta, D=D, best_D=best_D,
                                                               pos=pos).items()}
    best_delta = torch.full((L, B, 2), 7.0, device="cuda")
    best_pos = torch.full((F, M, 2), 7.0, device="cuda")
    adv = t["obs"].clone() * 0 + 9.0
    layout = _layout(split)
    _lib.check(lib.tb2_attack_step(layout.handle, _p(t["d_obs"]), _p(t["obs"]), L, _p(t["delta"]), _p(t["D"]), F,
                                   _p(t["pos"]), _p(t["best_D"]), _p(best_delta), _p(best_pos), _p(adv), eps, alpha, 1,
                                   None))
    want, want_best, improved = step_ref(d_obs, obs, delta, D, best_D, split, np.float32(eps), np.float32(alpha), True)
    got = t["delta"].cpu().numpy()
    assert np.abs(got - want).max() <= 1e-6
    assert np.array_equal(t["best_D"].cpu().numpy(), want_best)
    assert np.all(np.sqrt((got.astype(np.float64) ** 2).sum(-1)) <= eps * (1 + 1e-6))
    assert not np.array_equal(got, delta)
    assert np.array_equal(got[4, 2], delta[4, 2]) and np.array_equal(got[2, 3], delta[2, 3])   # NaN frame, g = 0
    assert np.array_equal(got[:, 4], delta[:, 4]) and np.array_equal(got[:, 3], delta[:, 3])   # frozen scenes
    bd, bp = best_delta.cpu().numpy(), best_pos.cpu().numpy()
    for b in range(B):
        rows = slice(split[b], split[b + 1])
        if improved[b]:
            assert np.array_equal(bd[:, b], delta[:, b]) and np.array_equal(bp[:, rows], pos[:, rows])
        else:
            assert np.all(bd[:, b] == 7.0) and np.all(bp[:, rows] == 7.0)
    a = adv.cpu().numpy()
    prim = split[:-1]
    assert np.array_equal(np.nan_to_num(a[:, prim], nan=3.0), np.nan_to_num(obs[:, prim] + got, nan=3.0))
    others = np.ones(M, dtype=bool)
    others[prim] = False
    assert np.all(a[:, others] == 9.0)                           # non-primary rows untouched


# ---------------------------------------------------------------------------------------------------------------------
# GPU: end to end
# ---------------------------------------------------------------------------------------------------------------------
def _model(kind, seed=1):
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    spec = O.MODEL_SPECS[kind]
    model = LSTM(pool=GridBasedPooling(**spec) if spec is not None else None)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=seed, relu_bias=3.0).items()})
    return model.cuda()


def _scenes(seed, n=12):
    from oracle import lstm_oracle as O
    xy, bs = O.synthetic_scenes(n, 5, n_frames=21, seed=seed, ragged=True, nan_tracks=False)
    return [xy[:, bs[i]:bs[i + 1]].astype(np.float64) for i in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["directional", "social_default"])
def test_attack_end_to_end(kind):
    from trajnetplusplusbaselines_b200.attack import collision_attack
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    from types import SimpleNamespace
    model = _model(kind)
    xys = _scenes(4)
    for norm in (False, True):
        clean = LSTMPredictor(model).predict_batch_xy(xys, n_predict=12, args=SimpleNamespace(normalize_scene=norm))
        r0 = collision_attack(model, xys, eps=0.0, steps=3, normalize_scene=norm, chunk=5)
        assert np.all(r0.delta == 0)
        for a, b in zip(r0.predictions, clean):
            assert np.array_equal(a[0][0], b[0][0]) and np.array_equal(a[0][1], b[0][1])
        assert np.array_equal(r0.d_clean, r0.d_attacked)
        r = collision_attack(model, xys, eps=0.3, steps=6, normalize_scene=norm, chunk=5)
        assert np.all(r.d_attacked <= r.d_clean)
        assert np.all(np.sqrt((r.delta ** 2).sum(-1)) <= 0.3 * (1 + 1e-6))
        assert np.any(r.d_attacked < r.d_clean)
        r2 = collision_attack(model, xys, eps=0.3, steps=6, normalize_scene=norm, chunk=5)
        assert np.array_equal(r.delta, r2.delta) and np.array_equal(r.d_attacked, r2.d_attacked)
        for a, b in zip(r.predictions, r2.predictions):
            assert np.array_equal(a[0][0], b[0][0])
    with pytest.raises(ValueError):
        collision_attack(model, xys, eps=-1.0)
    with pytest.raises(ValueError):
        collision_attack(model, xys, steps=0)


def sample_gap(pos, split, first):
    """Per scene the gap between the smallest and the second-smallest distance over the distinct sample points of the
    objective (each kept frame's endpoints once, each segment's midpoint), +inf with fewer than two samples.  A gap far
    above the positions' last bits keeps the objective's minimiser, and so its subgradient, from switching."""
    pos = np.asarray(pos, dtype=np.float64)
    gaps = np.full(len(split) - 1, np.inf)
    for b in range(len(split) - 1):
        r0, d = split[b], []
        for j in range(r0 + 1, split[b + 1]):
            kept = [t for t in range(first, pos.shape[0])
                    if np.isfinite(pos[t, r0]).all() and np.isfinite(pos[t, j]).all()]
            d += [np.hypot(*(pos[t, r0] - pos[t, j])) for t in kept] if len(kept) > 1 else []
            d += [np.hypot(*((pos[p, r0] + pos[t, r0]) / 2 - (pos[p, j] + pos[t, j]) / 2)) for p, t in zip(kept, kept[1:])]
        if len(d) > 1:
            d = np.sort(d)
            gaps[b] = d[1] - d[0]
    return gaps


@pytest.mark.gpu
@pytest.mark.parametrize("kind, seed", [("vanilla", 9), ("directional", 10)])
def test_attack_matches_a_torch_pgd_loop(kind, seed):
    """PGD written out in torch over differentiable_rollout, with the float64 restatements of the objective and the step,
    gives the attack's perturbations.  Scenes are independent, and the comparison is made on the scenes whose objective
    has a unique minimiser by a clear margin (>= 1e-5 m, far above the positions' last bits) at every iterate of the
    loop: at least half of them."""
    from trajnetplusplusbaselines_b200.attack import collision_attack
    from trajnetplusplusbaselines_b200.lstm import differentiable_rollout
    model = _model(kind, seed=3)
    xys = _scenes(seed, n=8)
    eps, steps = 0.2, 4
    res = collision_attack(model, xys, eps=eps, steps=steps)
    split = np.concatenate([[0], np.cumsum([xy.shape[1] for xy in xys])])
    observed = torch.Tensor(np.concatenate([xy[:9] for xy in xys], axis=1)).cuda()
    delta = np.zeros((9, len(xys), 2), dtype=np.float32)
    best_D, best_delta = np.full(len(xys), np.inf), delta.copy()
    gap = np.full(len(xys), np.inf)
    for it in range(steps + 1):
        adv = observed.clone()
        adv[:, split[:-1]] += torch.from_numpy(delta).cuda()
        adv.requires_grad_()
        _, pos = differentiable_rollout(model, adv, torch.from_numpy(split), 12, pad_to_batch_max=False)
        P = pos.detach().cpu().numpy()
        D, G = objective_ref(P, split, pos.shape[0] - 12)
        gap = np.minimum(gap, sample_gap(P, split, pos.shape[0] - 12))
        improved = D < best_D
        best_delta[:, improved] = delta[:, improved]
        if it < steps:
            (d_obs,) = torch.autograd.grad(pos, adv, grad_outputs=torch.from_numpy(G).float().cuda())
            delta, best_D, _ = step_ref(d_obs.cpu().numpy(), observed.cpu().numpy(), delta, D, best_D, split, eps,
                                        np.float32(2.5 * eps / steps), True)
            delta = delta.astype(np.float32)
        else:
            best_D[improved] = D[improved]
    clear = gap >= 1e-5
    assert clear.sum() >= len(xys) // 2, gap
    assert np.any(best_D[clear] < np.inf) and np.any(np.abs(best_delta[:, clear]) > 0)
    assert np.abs(res.delta[clear] - best_delta.transpose(1, 0, 2)[clear]).max() <= 1e-6
    assert np.abs(res.d_attacked[clear] - best_D[clear]).max() <= 1e-5      # positions differ in delta's last bits


@pytest.mark.gpu
@pytest.mark.parametrize("norm", [False, True])
def test_scenes_without_a_pair_keep_the_clean_forecast(norm):
    """A one-track scene, and a scene whose neighbours all leave before the last observed frame (forecast as NaN), have
    D = +inf on every iterate: the attack returns their clean forecast bit for bit, with delta = 0."""
    from types import SimpleNamespace
    from trajnetplusplusbaselines_b200.attack import collision_attack
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    model = _model("directional")
    xys = _scenes(4, n=6)
    gone = xys[2].copy()
    gone[6:, 1:] = np.nan
    xys = [xys[0][:, :1], xys[1], gone] + xys[3:]
    clean = LSTMPredictor(model).predict_batch_xy(xys, n_predict=12, args=SimpleNamespace(normalize_scene=norm))
    for eps in (0.0, 0.3):
        r = collision_attack(model, xys, eps=eps, steps=3, normalize_scene=norm)
        assert np.isinf(r.d_clean[[0, 2]]).all() and np.isinf(r.d_attacked[[0, 2]]).all()
        assert np.all(r.delta[[0, 2]] == 0)
        scenes = range(len(xys)) if eps == 0 else (0, 2)
        for i in scenes:
            for a, b in zip(r.predictions[i][0], clean[i][0]):
                assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True), i
            for a, b in zip(r.clean_predictions[i][0], clean[i][0]):
                assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True), i


# ---------------------------------------------------------------------------------------------------------------------
# CLI
# ---------------------------------------------------------------------------------------------------------------------
def _block(root, name="synth", sizes=(3, 1, 5, 2, 4)):
    from test_multimodal_batch import _write_scenes
    for part in ("test", "test_private"):
        os.makedirs(os.path.join(root, "DATA_BLOCK", name, part))
        _write_scenes(os.path.join(root, "DATA_BLOCK", name, part, name + ".ndjson"), list(sizes), 4)


@pytest.mark.parametrize("argv, word", [(["--eps", "0"], "--eps"), (["--eps", "-0.1"], "--eps"),
                                        (["--steps", "0"], "--steps")])
def test_cli_refuses_bad_arguments_before_reading(tmp_path, monkeypatch, argv, word):
    from trajnetplusplusbaselines_b200 import attack
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit) as e:
        attack.main(["--path", "synth", "--output", "missing.pkl"] + argv)
    assert word in str(e.value.code)
    assert os.listdir(tmp_path) == []


def test_cli_refuses_unsupported_models(tmp_path, monkeypatch):
    from trajnetplusplusbaselines_b200 import attack
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor, NearestNeighborMLP
    monkeypatch.chdir(tmp_path)
    _block(str(tmp_path))
    LSTMPredictor(LSTM(pool=NearestNeighborMLP())).save({}, "nn.pkl")
    before = sorted(os.listdir(os.path.join(tmp_path, "DATA_BLOCK", "synth")))
    with pytest.raises(SystemExit) as e:
        attack.main(["--path", "synth", "--output", "nn.pkl"])
    assert "NearestNeighborMLP" in str(e.value.code)
    assert sorted(os.listdir(os.path.join(tmp_path, "DATA_BLOCK", "synth"))) == before


@pytest.mark.gpu
def test_cli_writes_and_scores(tmp_path, monkeypatch, capsys):
    from trajnetplusplusbaselines_b200 import attack, scoring
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    monkeypatch.chdir(tmp_path)
    _block(str(tmp_path))
    LSTMPredictor(_model("directional").cpu()).save({}, "dlstm.pkl")
    attack.main(["--path", "synth", "--output", "dlstm.pkl", "--eps", "0.2", "--steps", "3"])
    out = capsys.readouterr().out
    name = "dlstm_attack_eps0.2_steps3"
    pred = os.path.join("DATA_BLOCK", "synth", "test_pred", name, "synth.ndjson")
    assert os.path.exists(pred)
    rec = np.load(os.path.join("DATA_BLOCK", "synth", "test_pred", name + ".npz"))
    assert rec["delta"].shape == (5, 9, 2) and len(rec["scene_id"]) == 5
    assert np.all(rec["d_attacked"] <= rec["d_clean"])
    res = scoring.score_file(os.path.join("DATA_BLOCK", "synth", "test_private", "synth.ndjson"), pred)
    assert scoring.format_table("dlstm attacked", {"synth": res}, "NA") in out
    assert "attacked 5 scenes, %d reached" % int(np.sum(rec["d_attacked"] <= LIMIT)) in out
