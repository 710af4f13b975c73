"""The non-grid interaction modules (csrc/mlp_pool.cu: hidden_mlp_pool, attn_mlp_pool, nn_mlp_pool, traj_scene_sum +
traj_feat, pool_lstm_cell) against the float64 restatement of tests/torch_ref.py, at the widths, scene sizes and
inputs where the kernels branch.

The restatement is pinned on the CPU to vectors of the unmodified reference (tests/golden/nongrid_golden.npz,
oracle/make_nongrid_golden.py).  On the GPU the stand-alone plug (the kernel itself) is compared on the same fp32
inputs within GATE x the largest entry of each output, and LSTM.forward within FWD_GATE metres, with the tensor cores
on and off.

Gates.  Every output here is a sum of at most ~1200 fp32 products of terms of size <= the output's largest entry (the
128-, 256- or 1024-term Linears, the 8-term Trajectron input, an LSTMCell of D + Hp <= 1536 inputs); fp32 rounding
leaves ~1e-6 relative for such sums, so 2e-5 of the largest entry is 10-20x above the kernels' error and 5-50x below
the 1e-4 gates of test_nongrid.py.  Attention computes exp with __expf (2 ulp + a relative error growing with |x|,
~1e-6 for |x| <= 30) and 1 / sqrt(E) with rsqrtf: its gate is 5e-5.

Nearest-neighbour selection is a discontinuity: every nn / nn_lstm case asserts that, in float64, consecutive ranks up
to rank n + 1 are >= 1e-4 m apart (2e-5 m in LSTM.forward, see NN_GAP_FWD) unless the two neighbours have identical
features (then their order cannot change the output).
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_nongrid_golden import KINDS, ATTN_KINDS, NN_KINDS, NN_LSTM_KINDS, TRAJ_KINDS, plug_inputs, scene_inputs  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALL_KINDS = KINDS + NN_KINDS + ATTN_KINDS + NN_LSTM_KINDS + TRAJ_KINDS
STATEFUL_KINDS = NN_LSTM_KINDS + TRAJ_KINDS
GATE = 2e-5             # of max |float64 output|
ATTN_GATE = 5e-5        # __expf / rsqrtf
FWD_GATE = 2e-5         # metres, LSTM.forward positions, fp32 FFMA gate kernel (TB2_DISABLE_TC=1)
# With the tensor cores the gate GEMM reads the pooled vector as a bf16 (hi, lo) pair: ~2^-16 of each entry is lost.
# The hidden-state MLP pool max-pools ReLU embeddings of relative positions, so on the 93-track scene (offsets of tens
# of metres) its pooled entries are the largest of the five modules and the positions move by up to 1.7e-4 m
# (measured on an H100; the fp32 path stays at 5.7e-6 m, so the pooled vector itself is right).
FWD_GATE_TC = 3e-4
NN_GAP = 1e-4           # metres between consecutive neighbour ranks (plug)
# LSTM.forward: ~620 tracks x 19 steps of random walks always hold a few closer pairs of ranks.  The float64 forward is
# fed the GPU's positions, so both sides rank the same inputs and differ only by the fp32 rounding of a distance
# (a few ulp: <= 1.2e-5 m at 50 m)
NN_GAP_FWD = 2e-5


def _rel_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert (np.isnan(got) == np.isnan(ref)).all()
    scale = max(float(np.nanmax(np.abs(ref))) if np.isfinite(ref).any() else 0.0, 1e-30)
    return float(np.nanmax(np.abs(got - ref)) / scale) if np.isfinite(ref).any() else 0.0


# ---------------------------------------------------------------------------------------------
# CPU: the restatement against the reference
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nongrid_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "nongrid_golden.npz"))


@pytest.mark.parametrize("kind", ALL_KINDS)
def test_restatement_matches_reference_vectors(nongrid_golden, kind):
    cfg = O.pool_config(kind)
    W = O.random_weights(kind, seed=13)
    hid, obs1, obs2 = plug_inputs()
    stats = {}
    st = None
    if kind in STATEFUL_KINDS:
        n = obs2.shape[0] * obs2.shape[1]
        st = {"h": torch.zeros(n, cfg.hidden_dim, dtype=torch.float64), "c": torch.zeros(n, cfg.hidden_dim, dtype=torch.float64)}
    got = TR.nongrid_pool(cfg, W, hid, obs1, obs2, state=st, stats=stats)
    assert _rel_err(got.numpy(), nongrid_golden[kind + "/plug"]) <= 2e-6, kind
    if kind in STATEFUL_KINDS:
        got2 = TR.nongrid_pool(cfg, W, hid, obs2, obs2 + (obs2 - obs1), state=st, stats=stats)
        assert _rel_err(got2.numpy(), nongrid_golden[kind + "/plug2"]) <= 2e-6, kind
    xy, bs = scene_inputs()
    Wt = {k: torch.tensor(v, dtype=torch.float64) for k, v in W.items()}
    obs = torch.from_numpy(xy[:9])
    with torch.no_grad():
        rel, pred = TR.forward(Wt, cfg, obs, bs, n_predict=12, dtype=torch.float64, stats=stats)
        _, pred_t = TR.forward(Wt, cfg, obs, bs, prediction_truth=torch.from_numpy(xy[9:20]), dtype=torch.float64,
                               stats=stats)
    for got, key in ((rel, "/rel_free"), (pred, "/pred_free"), (pred_t, "/pred_teacher")):
        assert _rel_err(got.numpy(), nongrid_golden[kind + key]) <= 2e-6, (kind, key)


# ---------------------------------------------------------------------------------------------
# GPU: the stand-alone plug (the kernel itself) against the float64 restatement
# ---------------------------------------------------------------------------------------------
CLASSES = {"hiddenstatemlp": "HiddenStateMLPPooling", "attentionmlp": "AttentionMLPPooling", "nn": "NearestNeighborMLP",
           "nn_lstm": "NearestNeighborLSTM", "traj_pool": "TrajectronPooling"}
CONFIGS = {"hiddenstatemlp": O.MlpPoolConfig, "attentionmlp": O.AttnPoolConfig, "nn": O.NnPoolConfig,
           "nn_lstm": O.NnLstmPoolConfig, "traj_pool": O.TrajectronPoolConfig}


def _module(kind, seed=0, scale=1.0, **kw):
    """The module with torch's default initialisation from `seed` (weights times `scale`), on the GPU, and its
    restatement config and weights."""
    from trajnetplusplusbaselines_b200 import lstm as L
    torch.manual_seed(seed)
    m = getattr(L, CLASSES[kind])(**kw)
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)
    W = {"pool." + k: v.detach().numpy().copy() for k, v in m.state_dict().items()}
    return m.cuda(), CONFIGS[kind](**kw), W


def _scenes(B, N, seed=0, density=0.16):
    """obs1, obs2 [B, N, 2] fp32 and hidden [B, N, 128]: tracks uniform on a square of N / density m^2 (so that the
    nearest distances stay ~1 m at every N), velocities ~ N(0, 0.3^2)."""
    rng = np.random.RandomState(seed)
    side = math.sqrt(N / density)
    obs2 = (rng.rand(B, N, 2) * side).astype(np.float32)
    obs1 = (obs2 - rng.randn(B, N, 2) * 0.3).astype(np.float32)
    hid = (rng.randn(B, N, 128) * 0.5).astype(np.float32)
    return hid, obs1, obs2


def _nn_margin(stats, gap=NN_GAP):
    assert stats.get("nn_gap", math.inf) >= gap, stats


def _plug(m, hid, obs1, obs2):
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    with torch.no_grad():
        return m(cuda(hid), cuda(obs1), cuda(obs2)).cpu().numpy()


def _check_plug(name, kind, m, cfg, W, hid, obs1, obs2, gate=None, state=None):
    stats = {}
    ref = TR.nongrid_pool(cfg, W, hid, obs1, obs2, state=state, stats=stats).numpy()
    if kind in ("nn", "nn_lstm"):
        _nn_margin(stats)
    got = _plug(m, hid, obs1, obs2)
    err = _rel_err(got, ref)
    gate = gate or (ATTN_GATE if kind == "attentionmlp" else GATE)
    print("%s: max|cuda - float64| / max|float64| = %.2e" % (name, err))
    assert err <= gate, (name, err)
    return stats


def _fresh_state(cfg, rows):
    if cfg.type_ not in ("nn_lstm", "traj_pool"):
        return None
    return {"h": torch.zeros(rows, cfg.hidden_dim, dtype=torch.float64), "c": torch.zeros(rows, cfg.hidden_dim, dtype=torch.float64)}


def _absent(hid, obs1, obs2, seed):
    """~10 % of the tracks absent now, ~10 % absent at the previous step (velocity NaN) -- not track 0 of a scene."""
    rng = np.random.RandomState(seed)
    u = rng.rand(*obs2.shape[:2])
    u[:, 0] = 0.5
    obs2[u < 0.1] = np.nan
    obs1[u > 0.9] = np.nan


def _m_hidden_nan_row(hid, obs1, obs2):            # NaN only in hidden rows: the position / velocity parts stay
    hid[:, 1, 5] = np.nan
    hid[:, 3] = np.nan


def _m_fewer(hid, obs1, obs2):                     # NaN tracks past the first three: fewer than n others present
    obs2[:, 3:] = np.nan
    obs1[:, 3:] = np.nan


def _m_all_absent(hid, obs1, obs2):                # every other track absent: all at 1000 m
    obs2[:, 1:] = np.nan


def _m_vel_nan(hid, obs1, obs2):                   # the nearest neighbour is present now, absent before (velocity NaN -> 0)
    obs2[:, 1] = obs2[:, 0] + np.float32(0.25)
    obs1[:, 1] = np.nan


def _m_tie(hid, obs1, obs2):                       # tracks 1 and 2: same position and velocity, nearest to track 0
    obs2[:, 1] = obs2[:, 2] = obs2[:, 0] + np.float32(0.3)
    obs1[:, 1] = obs1[:, 2] = obs2[:, 1] - np.float32(0.2)


def _m_traj_invisible(hid, obs1, obs2):            # an invisible primary, and a scene with a single visible track
    obs2[0, 0] = np.nan
    obs1[1, 1:] = np.nan


# (id, kind, constructor arguments, B, N, input mutation, weight scale)
PLUG_CASES = [
    ("hid_default", "hiddenstatemlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 8, 20, None, 1.0),
    ("hid_no_hidden", "hiddenstatemlp", dict(hidden_dim=128, mlp_dim=64, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 8, 20, None, 1.0),
    ("hid_no_vel", "hiddenstatemlp", dict(hidden_dim=128, mlp_dim=96, mlp_dim_spatial=32, mlp_dim_vel=0, out_dim=256), 8, 20, None, 1.0),
    # D = 37 and out_dim = 41: the odd tail of the two-accumulator output loop
    ("hid_odd", "hiddenstatemlp", dict(hidden_dim=128, mlp_dim=37, mlp_dim_spatial=5, mlp_dim_vel=3, out_dim=41), 8, 20, None, 1.0),
    ("hid_nan_hidden_row", "hiddenstatemlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 8, 20,
     _m_hidden_nan_row, 1.0),
    ("attn_default", "attentionmlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 8, 20, None, 1.0),
    ("attn_e37", "attentionmlp", dict(hidden_dim=128, mlp_dim=37, mlp_dim_spatial=5, mlp_dim_vel=3, out_dim=41), 8, 20, None, 1.0),
    # dsv = 128: all four per-lane feature registers hold spatial / velocity features
    ("attn_96_32_0", "attentionmlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=96, mlp_dim_vel=32, out_dim=256), 8, 20, None, 1.0),
    ("attn_no_vel", "attentionmlp", dict(hidden_dim=128, mlp_dim=96, mlp_dim_spatial=32, mlp_dim_vel=0, out_dim=256), 8, 20, None, 1.0),
    ("attn_fill10", "attentionmlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256, fill_value=-10),
     8, 20, None, 1.0),
    ("attn_fill100", "attentionmlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256, fill_value=-100),
     8, 20, None, 1.0),
    # weights x 3.5: each track's logits span > 30, the softmax is peaked and the online rescaling matters
    ("attn_peaked", "attentionmlp", dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 8, 20, None, 3.5),
    ("nn_n1", "nn", dict(n=1, out_dim=32), 8, 20, None, 1.0),
    ("nn_n4", "nn", dict(n=4, out_dim=256), 8, 20, None, 1.0),
    ("nn_n32", "nn", dict(n=32, out_dim=256), 4, 40, None, 1.0),
    # out_dim / n = 65 > 32: the output loop strides
    ("nn_n2_d130", "nn", dict(n=2, out_dim=130), 8, 20, None, 1.0),
    ("nn_no_vel", "nn", dict(n=4, out_dim=256, no_vel=True), 8, 20, None, 1.0),
    ("nn_fewer_than_n", "nn", dict(n=4, out_dim=256), 8, 20, _m_fewer, 1.0),
    ("nn_all_absent", "nn", dict(n=4, out_dim=256), 8, 20, _m_all_absent, 1.0),
    ("nn_vel_nan", "nn", dict(n=4, out_dim=256), 8, 20, _m_vel_nan, 1.0),
    ("nn_exact_tie", "nn", dict(n=4, out_dim=256), 8, 20, _m_tie, 1.0),
    ("nn_lstm_default", "nn_lstm", dict(n=4, hidden_dim=128, out_dim=256), 8, 20, None, 1.0),
    ("traj_default", "traj_pool", dict(hidden_dim=128, out_dim=256), 8, 20, None, 1.0),
    ("traj_invisible", "traj_pool", dict(hidden_dim=128, out_dim=256), 8, 20, _m_traj_invisible, 1.0),
]


# data seeds chosen once so that the neighbour margin holds
DATA_SEEDS = {"nn_n32": 5}
SIZE_SEEDS = {("nn", 3071): 3, ("nn_lstm", 3071): 3}


@pytest.mark.gpu
@pytest.mark.parametrize("case", PLUG_CASES, ids=[c[0] for c in PLUG_CASES])
def test_cuda_plug_matches_float64(case):
    name, kind, kw, B, N, mutate, scale = case
    m, cfg, W = _module(kind, seed=len(name), scale=scale, **kw)
    hid, obs1, obs2 = _scenes(B, N, seed=DATA_SEEDS.get(name, len(name) + 1))
    if mutate is None:
        _absent(hid, obs1, obs2, seed=2)
    else:
        mutate(hid, obs1, obs2)
    stats = _check_plug(name, kind, m, cfg, W, hid, obs1, obs2, state=_fresh_state(cfg, B * N))
    if name == "attn_peaked":
        assert stats["attn_span"] > 30, stats


# Largest scene each launcher takes at the default widths (the shared-memory formulas in csrc/mlp_pool.cu):
#   hidden_mlp_pool  (n (4 + dh + D) + dh) 4 B + 16 <= 200 KB       dh = 64, D = 128:  260
#   attn_mlp_pool    (32 x 2 E + n (4 + dh)) 4 B <= 200 KB           E = 128, dh = 64:  632
#   nn_mlp_pool      16 n B + 16 <= 48 KB                                              3071
#   traj_feat        48 n B + 16 <= 48 KB                                              1023
DEFAULTS = {
    "hiddenstatemlp": (dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 260,
                       "hidden-state MLP pooling"),
    "attentionmlp": (dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256), 632, "attention pooling"),
    "nn": (dict(n=4, out_dim=256), 3071, "nearest-neighbour pooling"),
    "nn_lstm": (dict(n=4, hidden_dim=128, out_dim=256), 3071, "nearest-neighbour pooling"),
    "traj_pool": (dict(hidden_dim=128, out_dim=256), 1023, "Trajectron pooling"),
}
SIZE_CASES = [(k, n) for k in DEFAULTS for n in (1, 2, 33, 93, 256, "max")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,N", SIZE_CASES, ids=["%s-%s" % c for c in SIZE_CASES])
def test_cuda_plug_scene_sizes(kind, N):
    """One scene of 1, 2, 33 (beyond one warp), 93 (the largest scene of crowds_students001) and 256 tracks, and of the
    largest size the launcher takes; one track more raises before any launch."""
    kw, n_max, label = DEFAULTS[kind]
    n = n_max if N == "max" else N
    m, cfg, W = _module(kind, seed=n, **kw)
    hid, obs1, obs2 = _scenes(1, n, seed=SIZE_SEEDS.get((kind, n), n))
    if n > 2:
        _absent(hid, obs1, obs2, seed=n)
    if kind == "attentionmlp" and n > 256:
        # the float64 attention of every track of a 632-track scene is ~70 GFLOP on the host: check 64 tracks, each
        # attending over every slot
        rows = np.random.RandomState(0).choice(n, 64, replace=False)
        got = _plug(m, hid, obs1, obs2)[rows]
        Wt = {k: torch.as_tensor(v).double() for k, v in W.items()}
        perm = np.concatenate([rows, np.setdiff1d(np.arange(n), rows)])
        ref = TR._attention(cfg, Wt, torch.as_tensor(hid[0, perm]).double(), torch.as_tensor(obs1[0, perm]).double(),
                            torch.as_tensor(obs2[0, perm]).double(), n, rows=64)
        err = _rel_err(got, ref.numpy())
        print("%s-%d (64 tracks): %.2e" % (kind, n, err))
        assert err <= ATTN_GATE
    else:
        _check_plug("%s-%d" % (kind, n), kind, m, cfg, W, hid, obs1, obs2, state=_fresh_state(cfg, n))
    if N == "max":
        m2, _, _ = _module(kind, seed=n, **kw)
        hid, obs1, obs2 = _scenes(1, n + 1, seed=1)
        with pytest.raises(RuntimeError, match="scene too large for the %s kernel" % label):
            _plug(m2, hid, obs1, obs2)


# ---------------------------------------------------------------------------------------------
# GPU: the interaction-encoder LSTMCell (pool_lstm_cell_kernel) at every width class and over a sequence of calls
# ---------------------------------------------------------------------------------------------
LSTM_WIDTHS = [(hp, d) for hp in (40, 128, 512) for d in (24, 256, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("hp,d", LSTM_WIDTHS, ids=["hp%d-d%d" % c for c in LSTM_WIDTHS])
def test_cuda_pool_lstm_cell_widths(hp, d):
    """Trajectron pooling (D = out_dim is free of n) with Hp x D from the narrowest to the constructor limits; 3 x 15
    tracks: M = 45 is not a multiple of the 16- or 8-row tile.  Hp = 512 with D >= 128 needs the 8-row tile."""
    m, cfg, W = _module("traj_pool", seed=hp + d, hidden_dim=hp, out_dim=d)
    hid, obs1, obs2 = _scenes(3, 15, seed=hp)
    _absent(hid, obs1, obs2, seed=hp)
    st = _fresh_state(cfg, 45)
    for k in range(3):          # the state advances: the recurrent half of the gate sums is non-zero from call 2 on
        _check_plug("traj hp%d d%d call %d" % (hp, d, k), "traj_pool", m, cfg, W, hid, obs1, obs2, state=st)
        obs1, obs2 = obs2, obs2 + (obs2 - obs1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["nn_lstm", "traj_pool"])
def test_cuda_pool_state_over_calls(kind):
    """20 consecutive plug calls with the state carried, reset() after the tenth; a call with another track count
    raises."""
    kw = dict(n=4, hidden_dim=128, out_dim=256) if kind == "nn_lstm" else dict(hidden_dim=128, out_dim=256)
    m, cfg, W = _module(kind, seed=7, **kw)
    B, N = 6, 21
    hid, obs1, obs2 = _scenes(B, N, seed=8)
    vel = (obs2 - obs1).copy()
    st = _fresh_state(cfg, B * N)
    for k in range(20):
        if k == 10:
            m.reset(B * N, N - 1, device=torch.device("cuda"))
            st = _fresh_state(cfg, B * N)
        o1 = obs2 + vel * np.float32(k - 1)
        o2 = obs2 + vel * np.float32(k)
        _check_plug("%s call %d" % (kind, k), kind, m, cfg, W, hid, o1.astype(np.float32), o2.astype(np.float32), state=st)
    hid, obs1, obs2 = _scenes(B, N + 1, seed=9)
    with pytest.raises(RuntimeError, match="interaction-encoder state holds"):
        _plug(m, hid, obs1, obs2)


def test_pool_lstm_constructors_accept_the_widest_pairs():
    """The constructors' limits (hidden_dim <= 512, out_dim <= 1024) are what the kernel takes (CPU: construction)."""
    from trajnetplusplusbaselines_b200.lstm import NearestNeighborLSTM, TrajectronPooling
    NearestNeighborLSTM(n=4, hidden_dim=512, out_dim=1024)
    TrajectronPooling(hidden_dim=512, out_dim=1024)
    with pytest.raises(ValueError):
        TrajectronPooling(hidden_dim=513, out_dim=256)


# ---------------------------------------------------------------------------------------------
# GPU: ragged batches in both layouts (attention: padded slots are keys; Trajectron: whole-batch sums)
# ---------------------------------------------------------------------------------------------
LAYOUT_CASES = [("attentionmlp", True), ("attentionmlp", False), ("traj_pool", True), ("traj_pool", False),
                ("hiddenstatemlp", True), ("nn_lstm", True)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,pad", LAYOUT_CASES, ids=["%s-%s" % (k, "padded" if p else "per_scene") for k, p in LAYOUT_CASES])
def test_cuda_ragged_layouts_match_float64(kind, pad):
    """64 ragged scenes of 1..20 tracks and one of 93 through the handle's ragged layout, padded to the batch maximum
    (the trainer) or each scene on its own slots (the evaluator)."""
    kw = DEFAULTS[kind][0]
    m, cfg, W = _module(kind, seed=11, **kw)
    rng = np.random.RandomState(12)
    sizes = list(rng.randint(1, 21, size=64)) + [93]
    bs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    parts = [_scenes(1, int(n), seed=100 + b) for b, n in enumerate(sizes)]
    hid = np.concatenate([p[0][0] for p in parts])
    obs1 = np.concatenate([p[1][0] for p in parts])
    obs2 = np.concatenate([p[2][0] for p in parts])
    u = rng.rand(len(obs2))
    obs2[u < 0.08] = np.nan
    obs1[u > 0.92] = np.nan
    dev = torch.device("cuda")
    handle = m._plug_handle(dev)
    layout = m._layouts.get(bs, pad_to_batch_max=pad, device=dev)
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    st = _fresh_state(cfg, len(obs2))
    if st is not None:
        handle.pool_state_reset(layout)
    stats = {}
    ref = TR.nongrid_pool_ragged(cfg, W, hid, obs1, obs2, bs, pad_to_batch_max=pad, pool_state=st, stats=stats).numpy()
    if kind == "nn_lstm":
        _nn_margin(stats)
    with torch.no_grad():
        got = handle.pool_forward(layout, cuda(hid) if kind in ("attentionmlp", "hiddenstatemlp") else None,
                                  cuda(obs1), cuda(obs2), m.out_dim).cpu().numpy()
    err = _rel_err(got, ref)
    print("%s %s: %.2e" % (kind, "padded" if pad else "per-scene", err))
    assert err <= (ATTN_GATE if kind == "attentionmlp" else GATE)
    if kind == "traj_pool" and pad:
        # the padded layout differs from the per-scene one exactly by the other scenes' sums
        st2 = _fresh_state(cfg, len(obs2))
        per_scene = TR.nongrid_pool_ragged(cfg, W, hid, obs1, obs2, bs, pad_to_batch_max=False, pool_state=st2).numpy()
        assert np.abs(per_scene - ref).max() > 1e-3 * np.abs(ref).max()


# ---------------------------------------------------------------------------------------------
# GPU: LSTM.forward with each module against the float64 forward
# ---------------------------------------------------------------------------------------------
FWD_KINDS = ["hiddenstatemlp", "attentionmlp", "nn", "nn_lstm", "traj_pool"]


def _fwd_inputs(seed=None):
    """48 ragged scenes of 2..20 tracks (entering / leaving neighbours) and one scene of 93 tracks."""
    seed = FWD_SEED if seed is None else seed
    xy, bs = O.synthetic_scenes(48, 20, seed=seed, ragged=True, nan_tracks=True, start_std=FWD_SPREAD)
    big, bs_big = O.scenes_of_sizes([93], seed=seed + 1)
    big = big * np.float32(FWD_SPREAD / 3.0)
    xy = np.concatenate([xy, big], axis=1)
    bs = np.concatenate([bs, bs[-1] + bs_big[1:]]).astype(np.int64)
    return xy, bs


FWD_SPREAD = 12.0       # start_std (m) of the ragged scenes; the 93-track scene is spread alike
FWD_SEED = 116


@pytest.fixture(scope="module")
def fwd_model_weights():
    from trajnetplusplusbaselines_b200 import lstm as L
    cache = {}

    def get(kind):
        if kind not in cache:
            _, _, Wp = _module(kind, seed=21, **DEFAULTS[kind][0])
            torch.manual_seed(22)
            model = L.LSTM(pool=getattr(L, CLASSES[kind])(**DEFAULTS[kind][0]))
            W = {k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
            W.update(Wp)
            cache[kind] = W
        return cache[kind]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("teacher", [True, False], ids=["teacher", "free"])
@pytest.mark.parametrize("kind", FWD_KINDS)
def test_cuda_forward_matches_float64(fwd_model_weights, monkeypatch, kind, teacher, tc):
    from trajnetplusplusbaselines_b200 import lstm as L
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")
    W = fwd_model_weights(kind)
    xy, bs = _fwd_inputs()
    M = xy.shape[1]
    model = L.LSTM(pool=getattr(L, CLASSES[kind])(**DEFAULTS[kind][0]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().eval()
    obs = torch.from_numpy(xy[:9])
    truth = torch.from_numpy(xy[9:20]).clone()
    with torch.no_grad():
        if teacher:
            _, pred = model(obs, torch.zeros(M, 2), torch.from_numpy(bs), prediction_truth=truth.clone())
        else:
            _, pred = model(obs, torch.zeros(M, 2), torch.from_numpy(bs), n_predict=12)
    pred = pred.cpu().numpy()
    Wt = {k: torch.tensor(v, dtype=torch.float64) for k, v in W.items()}
    stats = {}
    # nearest-neighbour selection is discontinuous: the float64 forward is fed the GPU's positions, so both select
    # from the same inputs (and the margin is asserted on those)
    feed = torch.from_numpy(pred) if kind in ("nn", "nn_lstm") else None
    with torch.no_grad():
        _, ref = TR.forward(Wt, CONFIGS[kind](**DEFAULTS[kind][0]), obs, bs, dtype=torch.float64, stats=stats,
                            feed_back=feed, **(dict(prediction_truth=truth) if teacher else dict(n_predict=12)))
    ref = ref.numpy()
    if kind in ("nn", "nn_lstm"):
        _nn_margin(stats, NN_GAP_FWD)
    assert (np.isnan(pred) == np.isnan(ref)).all()
    err = float(np.nanmax(np.abs(pred - ref)))
    print("forward %s %s [%s]: max |cuda - float64| = %.2e m" % (kind, "teacher" if teacher else "free", "tc" if tc else "no_tc", err))
    assert err <= (FWD_GATE_TC if tc else FWD_GATE), (kind, err)
