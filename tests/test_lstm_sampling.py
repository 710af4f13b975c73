"""Sampled multi-modal predictions of LSTM models (trajnetplusplusbaselines_b200/lstm/sampling.py, sample_positions_kernel
in csrc/sgan.cu, tb2_lstm_forward_steps with eps_dev / tb2_lstm_sample_positions).

Mode q >= 1 draws every predicted position from its step's bivariate normal,
pos = obs2 + mu + (sx e1, sy (rho e1 + sqrt(1 - rho^2) e2)), and feeds that draw back; mode 0 (e = 0) is the mean.

CPU: the offset against the reference's own PredictionLoss.gaussian_2d (its exponent at the sampled point is e1^2 + e2^2,
its mean -log density the entropy), and the evaluator's refusal of --sample for a predictor that is not an LSTM.
GPU, with the tensor cores on and with TB2_DISABLE_TC=1: e = 0 gives LSTMPredictor's bits in every mode; random e against
a float64 restatement fed the GPU's positions; the batched decode equals the per-scene call bit for bit, whatever the
mode grouping; stateful pools run per scene only; reruns are bit-identical; the first step's draws have the covariance
of the device's normals; the evaluator end to end.
"""
import io
import json
import math
import os
import sys
import types
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from test_multimodal_batch import _paths, _scenes, _write_scenes  # noqa: E402

PLAIN = types.SimpleNamespace(normalize_scene=False)
NORMALIZED = types.SimpleNamespace(normalize_scene=True)
SIZES = (1, 5, 60, 2, 13, 7, 30, 3)        # tracks per scene: a lone primary up to a crowd
KINDS = ["vanilla", "directional", "social", "hiddenstatemlp", "attentionmlp", "nn"]
STATEFUL = ["nn_lstm", "traj_pool"]
GATE_TC, GATE_FFMA = 1e-4, 2e-5             # metres: the forward gates of test_hidden_dim.py / test_nongrid_kernels.py
EDGE_MARGIN = 1e-5                          # cells between a fed-back pair's offset and a grid-cell edge
NN_GAP = 2e-5                               # metres between consecutive neighbour ranks (test_nongrid_kernels.py)


def offset(normals, eps):
    """The sampled offset in float64: normals [..., 5], eps [..., 2] -> [..., 2]."""
    normals, eps = np.asarray(normals, np.float64), np.asarray(eps, np.float64)
    sx, sy, rho = normals[..., 2], normals[..., 3], normals[..., 4]
    e1, e2 = eps[..., 0], eps[..., 1]
    return np.stack([sx * e1, sy * (rho * e1 + np.sqrt(1.0 - rho * rho) * e2)], axis=-1)


def _random_normals(rng, n):
    """n normals in the ranges Hidden2Normal produces (sigma in (0.01, 0.21), rho in (0, 0.7)), with rho near 0.7 and
    the smallest sigmas included."""
    mu = rng.randn(n, 2) * 0.3
    s = 0.01 + 0.2 * rng.rand(n, 2)
    rho = 0.7 * rng.rand(n)
    s[: n // 8] = 0.01 + 1e-4 * rng.rand(n // 8, 2)
    rho[n // 8: n // 4] = 0.7 - 1e-6 * rng.rand(n // 4 - n // 8)
    return np.concatenate([mu, s, rho[:, None]], axis=1)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the offset is a draw of the density the reference's loss trains
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref_gaussian_2d():
    from oracle.ref_shim import import_reference
    import_reference()
    from trajnetbaselines.lstm.loss import PredictionLoss
    return PredictionLoss.gaussian_2d


@pytest.mark.needs_reference
def test_sampled_offset_exponent_is_e_squared(ref_gaussian_2d):
    """The reference's exponent z / (1 - rho^2) at mu + offset(e) is |e|^2: the offset is L e with L L^T = Sigma."""
    rng = np.random.RandomState(0)
    n = 4096
    normals = _random_normals(rng, n)
    eps = rng.randn(n, 2) * 1.5
    x = normals[:, :2] + offset(normals, eps)
    p = ref_gaussian_2d(torch.from_numpy(normals), torch.from_numpy(x)).numpy()
    s1, s2, rho = normals[:, 2], normals[:, 3], normals[:, 4]
    denom = 2 * math.pi * s1 * s2 * np.sqrt(1 - rho ** 2)
    exponent = -2.0 * np.log(p * denom)          # the reference's z / (1 - rho^2)
    err = np.abs(exponent - (eps ** 2).sum(axis=1))
    assert err.max() <= 1e-12, err.max()


@pytest.mark.needs_reference
def test_sampled_offset_mean_nll_is_the_entropy(ref_gaussian_2d):
    """Over 10^5 draws the mean -log density of the reference's gaussian_2d is log(2 pi sx sy sqrt(1 - rho^2)) + 1."""
    rng = np.random.RandomState(1)
    normals = np.array([[0.1, -0.2, 0.01, 0.01, 0.0], [0.0, 0.0, 0.05, 0.02, 0.6999], [0.3, 0.1, 0.1, 0.08, 0.35],
                        [-0.1, 0.0, 0.011, 0.09, 0.7 - 1e-7]])
    for nrm in normals:
        eps = rng.randn(100000, 2)
        rows = np.repeat(nrm[None], len(eps), axis=0)
        x = rows[:, :2] + offset(rows, eps)
        nll = -np.log(ref_gaussian_2d(torch.from_numpy(rows), torch.from_numpy(x)).numpy()).mean()
        want = math.log(2 * math.pi * nrm[2] * nrm[3] * math.sqrt(1 - nrm[4] ** 2)) + 1.0
        assert abs(nll - want) <= 0.01 * abs(want), (nrm, nll, want)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the evaluator's --sample
# ------------------------------------------------------------------------------------------------------------------
class _NotAnLSTM:
    def __call__(self, paths, scene_goal, n_predict=12, modes=1, predict_all=True, obs_length=9, start_length=0,
                 args=None):
        raise AssertionError("never called")


def _block(root, name="synth", sizes=(3, 1, 8, 2, 25, 4), seed=2):
    for part in ("test", "test_private"):
        os.makedirs(os.path.join(root, "DATA_BLOCK", name, part))
        _write_scenes(os.path.join(root, "DATA_BLOCK", name, part, name + ".ndjson"), list(sizes), seed)
    return types.SimpleNamespace(path=os.path.join(root, "DATA_BLOCK", name, "test_pred") + os.sep, output=["m/lstm.pkl"],
                                 modes=3, obs_length=9, pred_length=12, chunk=4, normalize_scene=False, labels=None,
                                 disable_collision=False, sample=True)


def test_cli_refuses_sample_for_other_predictors(tmp_path):
    from trajnetplusplusbaselines_b200.evaluator import get_predictions, prediction_folder
    from trajnetplusplusbaselines_b200.lstm import LSTM, SampledLSTMPredictor
    args = _block(str(tmp_path))
    assert prediction_folder("m/lstm.pkl", args) == "lstm_sample_modes3"
    assert prediction_folder("m/lstm.pkl", types.SimpleNamespace(modes=3)) == "lstm_modes3"
    with pytest.raises(SystemExit) as e:
        get_predictions(args, load_predictor=lambda fn: _NotAnLSTM())
    assert "--sample" in str(e.value.code) and "_NotAnLSTM" in str(e.value.code)
    assert not os.path.exists(args.path)                          # nothing written
    with pytest.raises(NotImplementedError):
        SampledLSTMPredictor(LSTM(goal_flag=True))


# ------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ------------------------------------------------------------------------------------------------------------------
def _spec(kind):
    for table in (O.ATTN_SPECS, O.NONGRID_SPECS, O.NN_SPECS, O.NN_LSTM_SPECS, O.TRAJ_SPECS):
        if kind in table:
            return dict(table[kind])
    spec = O.MODEL_SPECS[kind]
    return None if spec is None else dict(spec)


def _model(kind, seed=5, device="cuda"):
    from trajnetplusplusbaselines_b200.lstm import (LSTM, AttentionMLPPooling, GridBasedPooling, HiddenStateMLPPooling,
                                                    NearestNeighborLSTM, NearestNeighborMLP, TrajectronPooling)
    spec = _spec(kind)
    cls = {"attentionmlp": AttentionMLPPooling, "hiddenstatemlp": HiddenStateMLPPooling, "nn": NearestNeighborMLP,
           "nn_lstm": NearestNeighborLSTM, "traj_pool": TrajectronPooling}.get(kind, GridBasedPooling)
    model = LSTM(pool=cls(**spec) if spec is not None else None)
    W = O.random_weights(kind, seed=seed)
    sd = model.state_dict()
    sd.update({k: torch.from_numpy(v.copy()) for k, v in W.items() if k in sd})
    model.load_state_dict(sd)
    return model.to(device).eval(), W


def _set_tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")     # read when the model's handle is created


def _assert_same(a, b, modes):
    assert len(a) == len(b)
    for i, (s, t) in enumerate(zip(a, b)):
        assert sorted(s) == sorted(t) == list(range(modes))
        for q in range(modes):
            assert s[q][0].shape == t[q][0].shape and np.array_equal(s[q][0], t[q][0], equal_nan=True), (i, q)
        assert np.array_equal(np.asarray(s[0][1]), np.asarray(t[0][1]), equal_nan=True), i
        for q in range(1, modes):
            assert len(s[q][1]) == 0 and len(t[q][1]) == 0


def _singles(predictor, xys, eps, modes, args):
    """The per-scene __call__ of every scene with the columns of `eps` [n_predict, modes * M, 2] of its tracks."""
    M = sum(xy.shape[1] for xy in xys)
    eps = np.asarray(eps).reshape(eps.shape[0], modes, M, 2)
    outs, lo = [], 0
    try:
        for xy in xys:
            hi = lo + xy.shape[1]
            predictor.fixed_eps = torch.from_numpy(eps[:, :, lo:hi].reshape(eps.shape[0], -1, 2).copy())
            outs.append(predictor(_paths(xy), np.zeros((xy.shape[1], 2)), n_predict=12, modes=modes, obs_length=9,
                                  args=args))
            lo = hi
    finally:
        predictor.fixed_eps = None
    return outs


def _eps(modes, M, seed, n_predict=12, zero_mode0=True):
    e = np.random.RandomState(seed).standard_normal((n_predict, modes * M, 2)).astype(np.float32)
    if zero_mode0:
        e[:, :M] = 0.0
    return e


# ------------------------------------------------------------------------------------------------------------------
# GPU: e = 0 is the mean, bit for bit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalized"])
@pytest.mark.parametrize("kind", KINDS)
def test_zero_eps_every_mode_is_lstm_predictor(monkeypatch, kind, normalize, tc):
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor, SampledLSTMPredictor
    _set_tc(monkeypatch, tc)
    model, _ = _model(kind)
    args = NORMALIZED if normalize else PLAIN
    xys = _scenes(SIZES, seed=len(kind))
    M = sum(xy.shape[1] for xy in xys)
    mean = LSTMPredictor(model).predict_batch_xy(xys, n_predict=12, obs_length=9, args=args)
    sampled = SampledLSTMPredictor(model)
    for modes in (1, 3, 20):
        got = sampled.predict_batch_xy(xys, n_predict=12, obs_length=9, args=args, modes=modes,
                                       fixed_eps=np.zeros((12, modes * M, 2), np.float32))
        for i, (g, w) in enumerate(zip(got, mean)):
            for q in range(modes):
                assert np.array_equal(g[q][0], w[0][0], equal_nan=True), (i, q)
            assert np.array_equal(g[0][1], w[0][1], equal_nan=True), i


# ------------------------------------------------------------------------------------------------------------------
# GPU: random e against the float64 restatement
# ------------------------------------------------------------------------------------------------------------------
def _edge_margin(cfg, pos, bs):
    """Smallest distance (cells) of a present pair's grid offset to a cell edge, over the positions pos [T, M, 2]."""
    n = cfg.n
    off = np.array([n / 2, 0.0 if cfg.front else n / 2])
    worst = math.inf
    for b in range(len(bs) - 1):
        p = np.asarray(pos[:, bs[b]:bs[b + 1]], np.float64)
        if p.shape[1] < 2:
            continue
        oij = (p[:, None, :, :] - p[:, :, None, :]) / float(cfg.cell_side) + off
        d = np.abs(oij - np.clip(np.round(oij), 0, n)).min(axis=-1)
        keep = ~np.eye(p.shape[1], dtype=bool)[None] & ~np.isnan(d)
        if keep.any():
            worst = min(worst, float(d[keep].min()))
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", KINDS)
def test_random_eps_matches_float64_restatement(monkeypatch, kind, tc):
    """The sampled forward (tb2_lstm_forward_steps with eps_dev over a ragged per-scene layout) against torch_ref.forward
    fed the GPU's positions, with the offset of its own float64 normals at the same eps added to every predicted
    position."""
    _set_tc(monkeypatch, tc)
    model, W = _model(kind, seed=11)
    cfg = O.pool_config(kind)
    obs_length, n_predict = 9, 12
    first = obs_length - 2
    grid = cfg is not None and hasattr(cfg, "cell_side")
    # The scenes: the first data seed whose fed-back pairs all keep EDGE_MARGIN from a grid-cell edge (grid pools; about
    # one pair-step in 10^5 falls closer, where fp32 and float64 may bin a pair apart).  The forward is deterministic.
    for seed in range(3, 11):
        xy, bs = O.synthetic_scenes(10, 16, seed=seed, ragged=True, nan_tracks=True)
        M = xy.shape[1]
        eps = torch.from_numpy(_eps(1, M, seed=seed + 1, zero_mode0=False)).cuda()
        with torch.no_grad():
            seq = model._sequence(torch.from_numpy(xy[:obs_length]).cuda(), torch.from_numpy(bs), None, n_predict,
                                  pad_to_batch_max=False)
            seq.handle.forward_steps_sampled(seq.layout, seq.obs, None, seq.n_decode, 0, seq.S, eps, seq.normals,
                                             seq.positions, seq.h, seq.c)
        pos, normals = seq.positions.cpu().numpy(), seq.normals.cpu().numpy()
        if not grid or _edge_margin(cfg, pos[first:-1], bs) >= EDGE_MARGIN:     # every fed-back decoder position
            break
    else:
        raise AssertionError("no data seed keeps the fed-back pairs off the grid-cell edges")
    eps = eps.cpu().numpy()
    Wt = {k: torch.tensor(v, dtype=torch.float64) for k, v in W.items()}
    worst = 0.0
    stats = {}
    for b in range(len(bs) - 1):
        lo, hi = int(bs[b]), int(bs[b + 1])
        with torch.no_grad():
            rel, pred = TR.forward(Wt, cfg, torch.from_numpy(xy[:obs_length, lo:hi]), [0, hi - lo], n_predict=n_predict,
                                   dtype=torch.float64, stats=stats, feed_back=torch.from_numpy(pos[:, lo:hi]),
                                   pad_to_batch_max=False)
        ref = pred.numpy().astype(np.float64)
        ref[first:] += offset(rel.numpy()[first:], eps[:, lo:hi])
        got = pos[:, lo:hi]
        assert (np.isnan(got) == np.isnan(ref)).all(), b
        assert (np.isnan(normals[:, lo:hi]).any(-1) == np.isnan(got).any(-1)).all(), b
        if np.isfinite(ref).any():
            worst = max(worst, float(np.nanmax(np.abs(got - ref))))
    if kind == "nn":
        assert stats.get("nn_gap", math.inf) >= NN_GAP, stats
    print("sampled %s [%s]: max |cuda - float64| = %.2e m" % (kind, "tc" if tc else "no_tc", worst))
    assert worst <= (GATE_TC if tc else GATE_FFMA), (kind, tc, worst)
    assert np.nanmax(np.abs(offset(normals[first:], eps))) > 1e-2           # the draws moved the positions


@pytest.mark.gpu
def test_sample_positions_kernel_and_refusals():
    """tb2_lstm_sample_positions: the offset in place; a (0, 0) pair keeps the bits (signed zeros too); NaN normals stay
    NaN.  A sampled forward of a goal-conditioned model is refused; NULL eps is the mean forward, bit for bit that of
    all-zero eps."""
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import _ptr, _stream
    from trajnetplusplusbaselines_b200.lstm import LSTM
    lib = _lib.load()
    rng = np.random.RandomState(7)
    rows = 1000
    normals = _random_normals(rng, rows).astype(np.float32)
    normals[5] = np.nan
    pos = rng.randn(rows, 2).astype(np.float32)
    pos[10] = [-0.0, -0.0]
    eps = rng.randn(rows, 2).astype(np.float32)
    eps[10:20] = 0.0
    eps[20] = [-0.0, 0.0]
    n_d, p_d, e_d = (torch.from_numpy(a).cuda() for a in (normals, pos, eps))
    stream = _stream(torch.device("cuda"))
    assert lib.tb2_lstm_sample_positions(_ptr(n_d), _ptr(p_d), _ptr(e_d), rows, stream) == 0
    got = p_d.cpu().numpy()
    want = pos.astype(np.float64) + offset(normals, eps)
    keep = np.zeros(rows, bool)
    keep[10:21] = True
    assert np.array_equal(got[keep].view(np.uint32), pos[keep].view(np.uint32))
    assert np.isnan(got[5]).all()
    fin = ~keep & np.isfinite(want).all(-1)
    assert np.abs(got[fin] - want[fin]).max() <= 1e-6
    assert lib.tb2_lstm_sample_positions(_ptr(n_d), _ptr(p_d), _ptr(None), rows, stream) != 0
    model = LSTM(goal_flag=True).cuda().eval()
    xy = torch.zeros(9, 3, 2, device="cuda")
    seq = model._sequence(xy, torch.tensor([0, 3]), None, 12, goals=torch.zeros(3, 2))
    eps = torch.zeros(12, 3, 2, device="cuda")
    ws, need = seq.handle.workspace(seq.layout)

    def call(e):
        return lib.tb2_lstm_forward_steps(seq.handle.handle, seq.layout.handle, _ptr(seq.obs), 9, _ptr(None), 11,
                                          _ptr(None), _ptr(e), 0, seq.S, _ptr(seq.normals), _ptr(seq.positions),
                                          _ptr(seq.h), _ptr(seq.c), _ptr(None), _ptr(None), 0, _ptr(None), _ptr(None),
                                          _ptr(None), _ptr(ws), need, stream)
    assert call(eps) == -3 and b"goal" in lib.tb2_last_error()          # TB2_ERR_UNSUPPORTED
    plain, _ = _model("vanilla")
    seq = plain._sequence(xy, torch.tensor([0, 3]), None, 12)
    ws, need = seq.handle.workspace(seq.layout)
    assert call(None) == 0                                              # the mean forward
    mean = seq.positions.clone(), seq.normals.clone()
    assert call(eps) == 0
    for a, b in zip(mean, (seq.positions, seq.normals)):
        assert np.array_equal(a.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------
# GPU: batched == per scene, groups, stateful pools, reruns
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", KINDS)
def test_batched_equals_per_scene(monkeypatch, kind, tc):
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor, SampledLSTMPredictor
    _set_tc(monkeypatch, tc)
    model, _ = _model(kind)
    predictor = SampledLSTMPredictor(model)
    xys = _scenes(SIZES, seed=20 + len(kind))
    M = sum(xy.shape[1] for xy in xys)
    for args, modes in ((PLAIN, 3), (NORMALIZED, 4)):
        eps = _eps(modes, M, seed=modes)
        singles = _singles(predictor, xys, eps, modes, args)
        mean = LSTMPredictor(model).predict_batch_xy(xys, n_predict=12, obs_length=9, args=args)
        for max_rows in (None, 1, 2 * M, 3 * M - 1):         # one group; a mode per group; two; two then two
            got = predictor.predict_batch_xy(xys, n_predict=12, obs_length=9, args=args, modes=modes, fixed_eps=eps,
                                             max_rows=max_rows)
            _assert_same(singles, got, modes)
        for g, w in zip(got, mean):                             # mode 0 is the mean
            assert np.array_equal(g[0][0], w[0][0], equal_nan=True)
            assert np.array_equal(g[0][1], w[0][1], equal_nan=True)
        assert max(np.abs(g[1][0] - g[0][0]).max() for g in got) > 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("kind", STATEFUL)
def test_stateful_pools_run_per_scene(kind):
    from trajnetplusplusbaselines_b200.evaluator import _column_pipeline
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor, SampledLSTMPredictor
    model, _ = _model(kind)
    predictor = SampledLSTMPredictor(model)
    assert not predictor.batch_decode_supported()
    assert not _column_pipeline(predictor, 3) and not _column_pipeline(predictor, 1)
    xys = _scenes((4, 1, 9), seed=3)
    with pytest.raises(NotImplementedError):
        predictor.predict_batch_xy(xys, args=PLAIN, modes=3)
    M = sum(xy.shape[1] for xy in xys)
    zero = _singles(predictor, xys, np.zeros((12, 3 * M, 2), np.float32), 3, PLAIN)
    sampled = _singles(predictor, xys, _eps(3, M, seed=1), 3, PLAIN)
    for xy, z, s in zip(xys, zero, sampled):
        want = LSTMPredictor(model)(_paths(xy), np.zeros((xy.shape[1], 2)), n_predict=12, args=PLAIN)
        for q in range(3):
            assert np.array_equal(z[q][0], want[0][0], equal_nan=True), q
        assert np.array_equal(s[0][0], want[0][0]) and np.array_equal(s[0][1], want[0][1], equal_nan=True)
        assert np.abs(s[1][0] - s[0][0]).max() > 1e-3 and np.abs(s[2][0] - s[1][0]).max() > 1e-3


@pytest.mark.gpu
def test_reruns_with_one_seed_are_bit_identical():
    from trajnetplusplusbaselines_b200.lstm import SampledLSTMPredictor
    predictor = SampledLSTMPredictor(_model("social")[0])
    xys = _scenes((4, 11, 1, 6), seed=8)
    outs = []
    for max_rows in (None, None, 7):
        torch.manual_seed(123)
        outs.append(predictor.predict_batch_xy(xys, args=NORMALIZED, modes=5, max_rows=max_rows))
    for other in outs[1:]:
        _assert_same(outs[0], other, 5)
    assert np.abs(outs[0][1][3][0] - outs[0][1][4][0]).max() > 1e-3        # two modes of one scene differ
    assert np.abs(outs[0][0][2][0] - outs[0][1][2][0]).max() > 1e-3        # two scenes of one mode differ
    singles = []
    for _ in range(2):
        torch.manual_seed(9)
        singles.append([predictor(_paths(xy), np.zeros((xy.shape[1], 2)), modes=3, args=PLAIN) for xy in xys])
    _assert_same(singles[0], singles[1], 3)


@pytest.mark.gpu
def test_first_step_covariance_is_the_normals():
    """4096 modes of one scene: the offsets of the first predicted position (the sampled output of the last encoder
    step) from the mean have the covariance built from that step's normal on the device, within 5 %."""
    from trajnetplusplusbaselines_b200.lstm import SampledLSTMPredictor
    model, _ = _model("directional")
    xy = _scenes((5,), seed=6)[0]
    torch.manual_seed(0)
    out = SampledLSTMPredictor(model).predict_batch_xy([xy], args=PLAIN, modes=4096)[0]
    first = np.array([out[q][0][0] for q in range(1, 4096)], np.float64)
    d = first - np.asarray(out[0][0][0], np.float64)
    with torch.no_grad():
        rel, _ = model(torch.from_numpy(xy[:9]), torch.zeros(5, 2), torch.tensor([0, 5]), n_predict=12)
    sx, sy, rho = (float(v) for v in rel[7, 0, 2:5])
    sigma = np.array([[sx * sx, rho * sx * sy], [rho * sx * sy, sy * sy]])
    cov = d.T @ d / len(d)                 # the mean of the draws is 0
    scale = np.sqrt(np.outer(np.diag(sigma), np.diag(sigma)))
    assert (np.abs(cov - sigma) <= 0.05 * scale).all(), (cov, sigma)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the evaluator end to end
# ------------------------------------------------------------------------------------------------------------------
def _mode0_lines(path):
    lines = []
    for line in open(path):
        track = json.loads(line).get("track")
        if track is None or track.get("prediction_number", 0) == 0:
            lines.append(line)
    return lines


@pytest.mark.gpu
def test_evaluator_sample_end_to_end(tmp_path, monkeypatch):
    from trajnetplusplusbaselines_b200 import evaluator, scoring
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    model, _ = _model("directional", device="cpu")
    LSTMPredictor(model).save({"epoch": 0}, str(tmp_path / "lstm.pkl"))
    args = _block(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    evaluator.main(["--path", "synth", "--output", "lstm.pkl"])
    torch.manual_seed(0)
    buf = io.StringIO()
    with redirect_stdout(buf):
        evaluator.main(["--path", "synth", "--output", "lstm.pkl", "--sample", "--modes", "3", "--evaluate"])
    assert "lstm_sample_modes3" in buf.getvalue() and "Top3 ADE" in buf.getvalue()
    pred = os.path.join("DATA_BLOCK", "synth", "test_pred")
    one = os.path.join(pred, "lstm_modes1", "synth.ndjson")
    three = os.path.join(pred, "lstm_sample_modes3", "synth.ndjson")
    assert '"prediction_number": 2' in open(three).read()
    assert _mode0_lines(three) == _mode0_lines(one) == open(one).readlines()
    args.path = pred + os.sep
    args.output = ["lstm.pkl"]
    m3 = scoring.trajnet_evaluate(args, out=lambda s: None)["lstm_sample_modes3"]["synth"][0]
    m1 = scoring.trajnet_evaluate(types.SimpleNamespace(**dict(vars(args), sample=False, modes=1)),
                                  out=lambda s: None)["lstm_modes1"]["synth"][0]
    assert m3.average_l2 == m1.average_l2 and m3.final_l2 == m1.final_l2
    assert m3.pred_col == m1.pred_col and m3.gt_col == m1.gt_col
    assert m3.topk_ade != m3.average_l2 and m3.topk_ade <= m3.average_l2
    torch.manual_seed(1)
    evaluator.main(["--path", "synth", "--output", "lstm.pkl", "--sample", "--modes", "50"])
    args.modes = 50
    m50 = scoring.trajnet_evaluate(args, out=lambda s: None)["lstm_sample_modes50"]["synth"][0]
    assert np.isfinite(m50.nll) and m50.nll != 0
