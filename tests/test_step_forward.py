"""One forward step and one stand-alone grid pool against the float64 restatement (tests/torch_ref.py).

CPU:
  * torch_ref.step / _grid and the oracle pinned to the unmodified reference (tests/golden/step_golden.npz,
    oracle/make_step_golden.py): LSTM.step from non-zero (h, c) at H = 32, 160, 224, pool_to_input=False, and the
    grids whose first Linear no other fixture reaches (occupancy n = 36, directional n = 26, embedding_arch 'None');
  * the gates bite: an emulation of the tensor cores' 3-pass bf16 product stays inside the step gate, a 2-pass
    product and a grid that lost one winning pair do not; the same errors measured against the end-to-end 1e-4 m
    position gate of a Social-LSTM forward.

GPU, each case with the tensor cores on and with TB2_DISABLE_TC=1, fed the same fp32 inputs as the restatement:
  * test_step_matches_float64: one LSTM.step of the encoder and the decoder from random non-zero (h, c) on ragged
    scenes with absent tracks, at every width 32..256, for no pool, each grid first-layer kernel of the step (the row
    kernel, the social tensor-core kernel writing the bf16 split, the BASELINE social grid's wgmma second layer, an
    FFMA second layer, three layers, no embedding) and the hidden-state MLP;
  * test_gate_row_tiles: the gate kernels across their row tiles (M = 1 .. ~1000, absent tracks on tile edges) at
    H = 64, 128, 192, 256 (lstm_gates_tc, clusters of 1 .. 4 CTAs) and 96, 224 (lstm_gates, 32-row blocks);
  * test_pool_added_to_h_step / _forward: LSTM(pool_to_input=False) for every interaction module;
  * test_grid_pool_matches_float64: GridBasedPooling called on its own, one case per first-layer kernel.
Every case asserts the kernels it covers (tb2_profile_begin / end) and that no pool ReLU pre-activation lies within
1e-2 of 0, so both sides apply the same ReLU masks.  A single step bins the same fp32 positions on both sides.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_step_golden import (ADD_TO_H_CASES, PHASES, POOL_KINDS, STEP_CASES, pool_config,  # noqa: E402
                                     pool_inputs, step_inputs, weights)
from test_hidden_dim import RELU_MARGIN, _nan_rel, _profiled, _set_tc  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
WIDTHS = list(range(32, 257, 32))
BF16_KERNELS = {"lstm_gates_tc", "sparse_layer1_mma", "dense_layer_tc"}
STEP_GATE = {False: 1e-5, True: 5e-5}      # relative to the tensor's largest |entry|: fp32 kernels / 3-pass bf16 ones
POOL_GATE = {False: 2e-6, True: 2e-5}
NONGRID = ("hiddenstatemlp", "attentionmlp", "nn", "nn_lstm", "traj_pool")


def _table(kind):
    for table in (O.ATTN_SPECS, O.NONGRID_SPECS, O.NN_SPECS, O.NN_LSTM_SPECS, O.TRAJ_SPECS, O.MODEL_SPECS):
        if kind in table:
            return table
    raise KeyError(kind)


def _spec(kind, H, out_dim=None):
    """Constructor arguments of the kind's module next to an LSTM of width H (None: no pool).  NearestNeighborLSTM /
    Trajectron keep their own interaction-encoder width."""
    table = _table(kind)
    spec = table[kind]
    if spec is None:
        return None
    spec = dict(spec)
    if table not in (O.NN_SPECS, O.NN_LSTM_SPECS, O.TRAJ_SPECS):
        spec["hidden_dim"] = H
    if out_dim is not None:
        spec["out_dim"] = out_dim
    return spec


def _cfg(kind, H, out_dim=None):
    spec = _spec(kind, H, out_dim)
    if spec is None:
        return None
    cls = {id(O.ATTN_SPECS): O.AttnPoolConfig, id(O.NONGRID_SPECS): O.MlpPoolConfig, id(O.NN_SPECS): O.NnPoolConfig,
           id(O.NN_LSTM_SPECS): O.NnLstmPoolConfig, id(O.TRAJ_SPECS): O.TrajectronPoolConfig}.get(id(_table(kind)),
                                                                                                O.PoolConfig)
    return cls(**spec)


def _pool_module(kind, H, out_dim=None):
    from trajnetplusplusbaselines_b200.lstm import (AttentionMLPPooling, GridBasedPooling, HiddenStateMLPPooling,
                                                    NearestNeighborLSTM, NearestNeighborMLP, TrajectronPooling)
    spec = _spec(kind, H, out_dim)
    if spec is None:
        return None
    cls = {id(O.ATTN_SPECS): AttentionMLPPooling, id(O.NONGRID_SPECS): HiddenStateMLPPooling,
           id(O.NN_SPECS): NearestNeighborMLP, id(O.NN_LSTM_SPECS): NearestNeighborLSTM,
           id(O.TRAJ_SPECS): TrajectronPooling}.get(id(_table(kind)), GridBasedPooling)
    return cls(**spec)


def _model(kind, H, W, pool_to_input=True):
    from trajnetplusplusbaselines_b200.lstm import LSTM
    model = LSTM(hidden_dim=H, pool=_pool_module(kind, H, None if pool_to_input else H), pool_to_input=pool_to_input)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    return model.cuda().eval()


def _has_relus(cfg):
    return isinstance(cfg, O.PoolConfig) and cfg.embedding_arch not in (None, "None")


def _restated_step(W, cfg, phase, obs1, obs2, bs, h, c, H, pool_to_input=True, stats=None, kernel=None):
    """torch_ref.step in float64 on the fp32 inputs; (h', c', normal) as float64 arrays."""
    Wt = {k: torch.tensor(v, dtype=F64) for k, v in W.items()}
    with torch.no_grad():
        out = TR.step(Wt, cfg, phase, torch.from_numpy(h).to(F64), torch.from_numpy(c).to(F64), torch.from_numpy(obs1),
                      torch.from_numpy(obs2), bs, H, F64, pool_to_input, stats,
                      pool_state=TR.pool_state_zeros(cfg, obs2.shape[0], F64), kernel=kernel)
    return [t.numpy() for t in out]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement and the oracle against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "step_golden.npz"))


GOLDEN_STEPS = [(k, H, True) for k, H in STEP_CASES] + [(k, H, False) for k, H in ADD_TO_H_CASES]


@pytest.mark.parametrize("kind,H,pool_to_input", GOLDEN_STEPS,
                         ids=["%s-%d-%s" % (k, H, "input" if p else "add_to_h") for k, H, p in GOLDEN_STEPS])
def test_step_restatement_and_oracle_match_reference(golden, kind, H, pool_to_input):
    W = weights(kind, H, seed=H + 3, pool_to_input=pool_to_input)
    cfg = pool_config(kind, H, pool_to_input)
    obs1, obs2, bs, h, c = step_inputs(H, seed=H)
    for phase in PHASES:
        key = "step/%s/%d/%s/%s/" % (kind, H, "input" if pool_to_input else "add_to_h", phase)
        stats = {}
        restated = _restated_step(W, cfg, phase, obs1, obs2, bs, h, c, H, pool_to_input, stats)
        oracle = O.step(W, cfg, phase, h, c, obs1, obs2, bs, pool_to_input)
        if _has_relus(cfg):
            assert stats["relu_pool0"] >= RELU_MARGIN, stats
        for name, got_t, got_o in zip(("h", "c", "normal"), restated, oracle):
            assert _nan_rel(got_t, golden[key + name]) <= 2e-6, (kind, H, phase, name)
            assert _nan_rel(got_o, golden[key + name]) <= 2e-6, (kind, H, phase, name)


def _restated_pool(kind, W, hid, obs1, obs2, stats=None, kernel=None):
    Wt = {k: torch.tensor(v, dtype=F64) for k, v in W.items()}
    with torch.no_grad():
        return TR._grid(O.pool_config(kind), Wt, torch.from_numpy(obs1), torch.from_numpy(obs2),
                        torch.from_numpy(hid).to(F64), F64, stats, primary_edges=False, kernel=kernel).numpy()


@pytest.mark.parametrize("kind", POOL_KINDS)
def test_pool_restatement_and_oracle_match_reference(golden, kind):
    W = O.random_weights(kind, seed=17, relu_bias=3.0)
    hid, obs1, obs2 = pool_inputs(kind, seed=19)
    assert _nan_rel(_restated_pool(kind, W, hid, obs1, obs2), golden["pool/" + kind]) <= 2e-6
    assert _nan_rel(O.pool_forward(O.pool_config(kind), W, hid, obs1, obs2), golden["pool/" + kind]) <= 2e-6


@pytest.mark.needs_reference
@pytest.mark.parametrize("kind,H,pool_to_input", [("occupancy_front", 96, True), ("directional", 64, False),
                                                  ("social_small", 128, False), ("hiddenstatemlp", 256, False)])
def test_step_restatement_matches_live_reference(kind, H, pool_to_input):
    from oracle.make_step_golden import build_reference_model, reference_step
    from oracle.ref_shim import import_reference
    import_reference()
    W = weights(kind, H, seed=H + 5, pool_to_input=pool_to_input)
    model = build_reference_model(kind, W, H, pool_to_input)
    obs1, obs2, bs, h, c = step_inputs(H, seed=H + 7)
    for phase in PHASES:
        ref = reference_step(model, phase, obs1, obs2, bs, h, c)
        got = _restated_step(W, pool_config(kind, H, pool_to_input), phase, obs1, obs2, bs, h, c, H, pool_to_input)
        for name, g, r in zip(("h", "c", "normal"), got, ref):
            assert _nan_rel(g, r) <= 2e-6, (kind, H, phase, name)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the gates bite
# ---------------------------------------------------------------------------------------------------------------------
def _drop_one_winner(grid):
    """The grid [rows, C, n, n] with its first occupied cell back at `constant` (0): one (pair, cell) contribution
    lost."""
    grid = grid.clone()
    row, cell = [int(v) for v in (grid != 0).any(dim=1).flatten(1).nonzero()[0]]
    grid[row, :, cell // grid.shape[3], cell % grid.shape[3]] = 0.0
    return grid


KERNEL_ERRORS = {"3-pass bf16": SimpleNamespace(mm=TR.bf16_product(3)),
                 "2-pass bf16": SimpleNamespace(mm=TR.bf16_product(2)),
                 "one winning pair lost": SimpleNamespace(grid=_drop_one_winner)}


def _baseline_social(H=128):
    W = O.random_weights("social", seed=41, hidden_dim=H, relu_bias=3.0)
    xy, bs = O.scenes_of_sizes([20, 20], seed=43)
    return W, O.pool_config("social"), xy, bs


def test_step_gate_catches_subtle_kernel_errors():
    """One BASELINE Social-LSTM step (n = 16, two layers of 1024 / 256, H = 128) from random (h, c): the worst
    relative error of h, c, normal against float64 is inside the bf16 step gate for the 3-pass product, outside it for
    a 2-pass product and for one lost winning pair."""
    W, cfg, xy, bs = _baseline_social()
    obs1, obs2 = xy[7], xy[8]
    rng = np.random.RandomState(3)
    h = rng.uniform(-1, 1, size=(xy.shape[1], 128)).astype(np.float32)
    c = rng.uniform(-3, 3, size=(xy.shape[1], 128)).astype(np.float32)
    exact = _restated_step(W, cfg, "decoder", obs1, obs2, bs, h, c, 128)
    errs = {}
    for name, kernel in KERNEL_ERRORS.items():
        got = _restated_step(W, cfg, "decoder", obs1, obs2, bs, h, c, 128, kernel=kernel)
        errs[name] = max(_nan_rel(g, e) for g, e in zip(got, exact))
    print("step: " + ", ".join("%s %.1e" % kv for kv in errs.items()))
    assert errs["3-pass bf16"] <= STEP_GATE[True], errs
    assert errs["2-pass bf16"] > STEP_GATE[True], errs
    assert errs["one winning pair lost"] > STEP_GATE[True], errs


def test_end_to_end_position_gate_on_kernel_errors():
    """The same emulated errors through a teacher-forced BASELINE Social-LSTM forward (2 scenes of 20, 9 + 12 frames):
    the largest position error against float64, next to the 1e-4 m gate the forward tests use: the 3-pass product
    stays inside it, the two errors do not."""
    W, cfg, xy, bs = _baseline_social()
    Wt = {k: torch.tensor(v, dtype=F64) for k, v in W.items()}
    obs, truth = torch.from_numpy(xy[:9]), torch.from_numpy(xy[9:20])

    def positions(kernel=None):
        with torch.no_grad():
            return TR.forward(Wt, cfg, obs, bs, prediction_truth=truth, dtype=F64, kernel=kernel)[1].numpy()
    exact = positions()
    errs = {name: float(np.nanmax(np.abs(positions(k) - exact))) for name, k in KERNEL_ERRORS.items()}
    print("forward (m): " + ", ".join("%s %.1e" % kv for kv in errs.items()))
    assert errs["3-pass bf16"] <= 1e-4, errs
    assert errs["2-pass bf16"] > 1e-4, errs
    assert errs["one winning pair lost"] > 1e-4, errs


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _gpu_step(model, phase, obs1, obs2, bs, h, c, reset_pool_state=False):
    """LSTM.step on the device; (h', c', normal) as arrays and the kernels it ran."""
    def run():
        if reset_pool_state:          # the interaction-encoder state right after LSTM.forward's reset
            handle = model._engine()
            handle.pool_state_reset(model._layouts.get(bs, device=handle.device))
        with torch.no_grad():
            (h2, c2), normal = model.step(getattr(model, phase), (torch.from_numpy(h).cuda(), torch.from_numpy(c).cuda()),
                                          torch.from_numpy(obs1), torch.from_numpy(obs2), None, torch.from_numpy(bs))
        return [t.cpu().numpy() for t in (h2, c2, normal)]
    return _profiled(run)


def _compare_step(got, ref, gate, label):
    worst = 0.0
    for name, g, r in zip(("h", "c", "normal"), got, ref):
        err = _nan_rel(g, r)
        worst = max(worst, err)
        assert err <= gate, (label, name, err, gate)
    return worst


def _state(M, H, seed):
    rng = np.random.RandomState(seed)
    return (rng.uniform(-1, 1, size=(M, H)).astype(np.float32), rng.uniform(-3, 3, size=(M, H)).astype(np.float32))


def _gate_for(kernels, tc):
    return STEP_GATE[bool(tc and kernels & BF16_KERNELS)]


# kind -> (first-layer kernels with the tensor cores on, the same without)
STEP_KINDS = {
    "vanilla": (set(), set()),
    "directional": ({"pool_rows"}, {"pool_rows"}),
    "social_default": ({"sparse_layer1_mma"}, {"sparse_layer1"}),               # one_layer, 16 latent channels
    "social": ({"sparse_layer1_mma", "dense_layer_tc"}, {"sparse_layer1", "dense_layer"}),   # BASELINE two_layer
    "social_d96": ({"sparse_layer1_mma", "dense_layer"}, {"sparse_layer1", "dense_layer"}),  # FFMA second layer
    "occupancy_front": ({"pool_rows", "dense_layer"}, {"pool_rows", "dense_layer"}),          # three layers
    "occupancy_raw": ({"dense_grid"}, {"dense_grid"}),                                      # no embedding, P = 64
    "hiddenstatemlp": ({"hidden_mlp_pool"}, {"hidden_mlp_pool"}),
}
# (kind, H) -> weight seed where the default H + 13 puts a ReLU pre-activation of the second or third grid layer
# within 1e-2 of 0 (the +-3 biases keep the first layer's far from it, not always the later layers')
STEP_SEEDS = {("social", 160): 1173, ("social_d96", 32): 1045, ("social_d96", 224): 1237, ("occupancy_front", 96): 3109,
              ("occupancy_front", 160): 1173, ("occupancy_front", 256): 1269}


def _step_scenes(seed):
    """Ragged scenes (2..12 tracks) between frames 2 and 3, where ~10 % of the neighbours enter (absent at obs1);
    two more tracks absent at obs2."""
    xy, bs = O.synthetic_scenes(8, 12, seed=seed, ragged=True, nan_tracks=True)
    obs1, obs2 = xy[2].copy(), xy[3].copy()
    obs2[[3, xy.shape[1] - 1]] = np.nan
    return obs1, obs2, bs


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("kind", list(STEP_KINDS))
def test_step_matches_float64(monkeypatch, kind, H, tc):
    _set_tc(monkeypatch, tc)
    W = O.random_weights(kind, seed=STEP_SEEDS.get((kind, H), H + 13), hidden_dim=H, relu_bias=3.0)
    cfg = _cfg(kind, H)
    model = _model(kind, H, W)
    obs1, obs2, bs = _step_scenes(seed=H)
    h, c = _state(obs2.shape[0], H, seed=H + 1)
    P = 0 if cfg is None else (cfg.n * cfg.n * cfg.pooling_dim if getattr(cfg, "embedding_arch", 1) in (None, "None")
                               else cfg.out_dim)
    gate_kernel = "lstm_gates_tc" if tc and H % 64 == 0 and P % 64 == 0 else "lstm_gates"
    worst = 0.0
    for phase in PHASES:
        got, kernels = _gpu_step(model, phase, obs1, obs2, bs, h, c)
        assert gate_kernel in kernels and ({"lstm_gates", "lstm_gates_tc"} - {gate_kernel}).isdisjoint(kernels), \
            sorted(kernels)
        assert STEP_KINDS[kind][0 if tc else 1] <= kernels, sorted(kernels)
        stats = {}
        ref = _restated_step(W, cfg, phase, obs1, obs2, bs, h, c, H, stats=stats)
        if _has_relus(cfg):
            assert min(v for k, v in stats.items() if k.startswith("relu_pool")) >= RELU_MARGIN, stats
        worst = max(worst, _compare_step(got, ref, _gate_for(kernels, tc), (kind, H, tc, phase)))
    print("%s H=%d [%s]: worst relative error %.1e" % (kind, H, "tc" if tc else "no_tc", worst))


TILE_ROWS = [1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1003]


def _tile_scenes(M, seed):
    """M tracks in scenes of up to 20 (the last one smaller); tracks absent at obs2 on the rows of the 32- and 128-row
    tile edges and the last row (M > 1: one present row at least)."""
    sizes = [20] * (M // 20) + ([M % 20] if M % 20 else [])
    xy, bs = O.scenes_of_sizes(sizes, seed=seed)
    obs1, obs2 = xy[7].copy(), xy[8].copy()
    absent = [r for r in (31, 32, 127, 128, M - 1) if 0 < r < M]
    obs2[absent] = np.nan
    return obs1, obs2, bs


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("M", TILE_ROWS)
@pytest.mark.parametrize("H", [64, 128, 192, 256, 96, 224])
@pytest.mark.parametrize("kind", ["vanilla", "directional"])
def test_gate_row_tiles(monkeypatch, kind, H, M, tc):
    _set_tc(monkeypatch, tc)
    W = O.random_weights(kind, seed=H + 17, hidden_dim=H, relu_bias=3.0)
    cfg = _cfg(kind, H)
    model = _model(kind, H, W)
    obs1, obs2, bs = _tile_scenes(M, seed=M)
    h, c = _state(M, H, seed=M + H)
    got, kernels = _gpu_step(model, "encoder", obs1, obs2, bs, h, c)
    assert ("lstm_gates_tc" if tc and H % 64 == 0 else "lstm_gates") in kernels, sorted(kernels)
    stats = {}
    ref = _restated_step(W, cfg, "encoder", obs1, obs2, bs, h, c, H, stats=stats)
    if cfg is not None and M > 1:
        assert stats["relu_pool0"] >= RELU_MARGIN, stats
    worst = _compare_step(got, ref, _gate_for(kernels, tc), (kind, H, M, tc))
    print("%s H=%d M=%d [%s]: worst relative error %.1e" % (kind, H, M, "tc" if tc else "no_tc", worst))


ADD_TO_H_KINDS = ["occupancy", "directional", "social_default", "hiddenstatemlp", "attentionmlp", "nn", "nn_lstm",
                  "traj_pool"]


def _add_to_h_model(kind, H, seed):
    W = O.random_weights(kind, seed=seed, hidden_dim=H, relu_bias=3.0, out_dim=H, pool_to_input=False)
    return W, _cfg(kind, H, out_dim=H), _model(kind, H, W, pool_to_input=False)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("H", [32, 128, 224])
@pytest.mark.parametrize("kind", ADD_TO_H_KINDS)
def test_pool_added_to_h_step(monkeypatch, kind, H, tc):
    _set_tc(monkeypatch, tc)
    W, cfg, model = _add_to_h_model(kind, H, seed=H + 19)
    obs1, obs2, bs = _step_scenes(seed=H + 2)
    h, c = _state(obs2.shape[0], H, seed=H + 3)
    worst = 0.0
    for phase in PHASES:
        got, kernels = _gpu_step(model, phase, obs1, obs2, bs, h, c, reset_pool_state=kind in ("nn_lstm", "traj_pool"))
        assert "lstm_gates" in kernels and "lstm_gates_tc" not in kernels, sorted(kernels)
        stats = {}
        ref = _restated_step(W, cfg, phase, obs1, obs2, bs, h, c, H, pool_to_input=False, stats=stats)
        if _has_relus(cfg):
            assert stats["relu_pool0"] >= RELU_MARGIN, stats
        worst = max(worst, _compare_step(got, ref, _gate_for(kernels, tc), (kind, H, tc, phase)))
    print("%s H=%d pool added to h [%s]: worst relative error %.1e" % (kind, H, "tc" if tc else "no_tc", worst))


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("H", [32, 128, 224])
@pytest.mark.parametrize("kind", ADD_TO_H_KINDS)
def test_pool_added_to_h_forward(monkeypatch, kind, H, tc):
    """Teacher-forced and free LSTM.forward against the oracle, with test_hidden_dim's position gates."""
    _set_tc(monkeypatch, tc)
    W, cfg, model = _add_to_h_model(kind, H, seed=H + 23)
    xy, bs = O.synthetic_scenes(6, 9, seed=71, ragged=True, nan_tracks=True)
    M = xy.shape[1]
    with torch.no_grad():
        _, pred_f = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs), n_predict=12)
        _, pred_t = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs),
                          prediction_truth=torch.from_numpy(xy[9:20]).clone())
    _, ref_f = O.forward(W, cfg, xy[:9], bs, n_predict=12, hidden_dim=H, pool_to_input=False)
    _, ref_t = O.forward(W, cfg, xy[:9], bs, prediction_truth=xy[9:20], hidden_dim=H, pool_to_input=False)
    tol = (3e-4 if kind in NONGRID else 1e-4) if tc else 2e-5
    for got, ref in ((pred_f, ref_f), (pred_t, ref_t)):
        got = got.numpy()
        assert (np.isnan(got) == np.isnan(ref)).all()
        assert float(np.nanmax(np.abs(got - ref))) <= tol, (kind, H, tc, float(np.nanmax(np.abs(got - ref))))


def _grid_inputs(sizes, seed, spread=2.0):
    """[B, N, 2] positions / [B, N, 128] hidden states of scenes of the given sizes padded to the largest (NaN),
    with one track absent at obs1 and one at obs2."""
    rng = np.random.RandomState(seed)
    B, N = len(sizes), max(sizes)
    obs2 = (rng.randn(B, N, 2) * spread).astype(np.float32)
    obs1 = obs2 - (rng.randn(B, N, 2) * 0.3).astype(np.float32)
    hid = (rng.randn(B, N, 128) * 0.5).astype(np.float32)
    for b, n in enumerate(sizes):
        obs1[b, n:] = obs2[b, n:] = hid[b, n:] = np.nan
    obs1[0, 1] = np.nan
    obs2[B - 1, min(sizes[-1], N) - 1] = np.nan
    return hid, obs1, obs2


# (id, kind, scene sizes, spread, first-layer kernels with the tensor cores on, the same without)
# weight seed: len(sizes) + 29, or 1037 for social_baseline (37 puts a second-layer ReLU pre-activation 1e-4 from 0)
POOL_CASES = [
    ("rows_ch256", "occupancy_front_n4", [9] * 6, 2.0, {"pool_rows"}, {"pool_rows"}),
    ("rows_ch128", "directional", [9] * 6, 2.0, {"pool_rows"}, {"pool_rows"}),
    ("rows_ch64", "directional_n16", [9] * 6, 2.0, {"pool_rows"}, {"pool_rows"}),
    ("rows_ch32", "directional_n24", [9] * 6, 2.0, {"pool_rows"}, {"pool_rows"}),
    ("l1_occupancy", "occupancy_n36", [9] * 6, 2.0, {"sparse_layer1"}, {"sparse_layer1"}),
    ("l1_directional", "directional_n26", [9] * 6, 2.0, {"sparse_layer1"}, {"sparse_layer1"}),
    ("l1_social_c4", "social_c4", [9] * 6, 2.0, {"sparse_layer1"}, {"sparse_layer1"}),
    ("l1_social_c8", "social_small", [9] * 6, 2.0, {"sparse_layer1", "dense_layer"}, {"sparse_layer1", "dense_layer"}),
    ("l1_social_c32", "social_c32", [9] * 6, 2.0, {"sparse_layer1", "dense_layer_tc"}, {"sparse_layer1", "dense_layer"}),
    ("l1_social_c16", "social_default", [20] * 8, 2.5, {"sparse_layer1_mma"}, {"sparse_layer1"}),
    ("l1_social_c16_crowd", "social_default", [96], 6.0, {"sparse_layer1_mma"}, {"sparse_layer1"}),
    ("social_baseline", "social", [20] * 8, 2.5, {"sparse_layer1_mma", "dense_layer_tc"}, {"sparse_layer1", "dense_layer"}),
    ("dense_grid", "occupancy_raw", [9] * 6, 2.0, {"dense_grid"}, {"dense_grid"}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("case", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_grid_pool_matches_float64(monkeypatch, case, tc):
    _set_tc(monkeypatch, tc)
    name, kind, sizes, spread, k_tc, k_plain = case
    W = O.random_weights(kind, seed=1037 if name == "social_baseline" else len(sizes) + 29, relu_bias=3.0)
    pool = _pool_module(kind, 128)
    pool.load_state_dict({k[len("pool."):]: torch.from_numpy(v.copy()) for k, v in W.items() if k.startswith("pool.")},
                         strict=True)
    pool = pool.cuda()
    hid, obs1, obs2 = _grid_inputs(sizes, seed=31, spread=spread)

    def run():
        return pool(torch.from_numpy(hid).cuda(), torch.from_numpy(obs1).cuda(), torch.from_numpy(obs2).cuda()).cpu()
    out, kernels = _profiled(run)
    assert (k_tc if tc else k_plain) <= kernels, sorted(kernels)
    stats = {}
    ref = _restated_pool(kind, W, hid, obs1, obs2, stats)
    if _has_relus(O.pool_config(kind)):
        assert min(v for k, v in stats.items() if k.startswith("relu_pool")) >= RELU_MARGIN, stats
    err = _nan_rel(out.numpy(), ref)
    print("%s [%s]: relative error %.1e" % (name, "tc" if tc else "no_tc", err))
    assert err <= POOL_GATE[bool(tc and kernels & BF16_KERNELS)], (name, tc, err)
