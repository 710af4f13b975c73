"""Social force and ORCA rollouts against their CPU restatements, in both launch forms of csrc/classical.cu.

simulate_batch picks the form from the batch's largest scene: the warp form (four scenes per 128-thread CTA, one warp
each) when n_max <= 32, the CTA form (one CTA per scene, one thread per pedestrian, up to 1024) otherwise.  The sweeps
split the same way per scene (packed lane segments for n <= 32, a CTA per scene above).  Each case below runs a batch
through the device and compares every sampled position of every scene with oracle.classical_oracle.sf_simulate
(float64) and oracle.orca_oracle.c (C float, -ffp-contract=off):

  * ORCA: bit-identical everywhere;
  * social force: within SF_GATE = 1e-9 m over a rollout; after one step from random states within SF_STEP_GATE,
    near float64 rounding -- what a rollout shows above that is amplification of last-bit differences between the
    device's and the host's exp / cos, not a different operation (the force sum runs b = 0 .. n-1 on both sides).

Each case states the restatement branches it is there for (its counters must be > 0) and the launch form it runs in
(n_max of its batch).  The restatements run once per session (_sf_ref / _orca_ref cache them), so the CPU tests that
check counters and the device tests share them.
"""
import functools
import glob
import itertools
import os
from collections import namedtuple

import numpy as np
import pytest

from oracle import classical_oracle as C
from oracle.build_c import orca_simulate
from oracle.ref_shim import reference_root
from trajnetplusplusbaselines_b200.classical import sweep
from trajnetplusplusbaselines_b200.classical.common import sampling_rate

SF_GATE = 1e-9                # m, a rollout
SF_STEP_GATE = 1e-14          # m, one step: a few float64 ulp of positions of up to ~20 m (1 ulp = 3.6e-15 m)
SF_GRID = list(itertools.product((0.3, 0.5, 1.0), (1.0, 2.1, 5.0), (0.2, 0.3, 0.6)))
WARP_MAX = 32                 # largest n_max of the warp / packed form
N_LIMIT = 1024                # largest scene the host accepts


# ---- scenes -------------------------------------------------------------------------------------------------------
def _scene(n, seed, dense=0, stand=None, goal_steps=4.8):
    """One scene of n pedestrians: positions spread by 1 + 0.15 sqrt(n) m (the sweep tests' density), the first
    `dense` packed into a cluster of about 0.15 sqrt(dense) m; speeds 0.3 .. 1.5 m/s in random directions; the goal
    `goal_steps` seconds ahead.  `stand`: that pedestrian's goal is its position (social force: NaN direction).
    -> state [n, 6] float64 (x, y, vx, vy, dx, dy), speeds [n]."""
    rng = np.random.RandomState(seed)
    pos = rng.randn(n, 2) * (1.0 + 0.15 * np.sqrt(n))
    if dense:
        pos[:dense] = rng.randn(dense, 2) * 0.15 * np.sqrt(dense)
    ang = rng.rand(n) * 2 * np.pi
    spd = 0.3 + rng.rand(n) * 1.2
    vel = np.stack([spd * np.cos(ang), spd * np.sin(ang)], axis=1)
    goal = pos + vel * goal_steps + rng.randn(n, 2) * 0.3
    if stand is not None:
        goal[stand] = pos[stand]
    return np.concatenate([pos, vel, goal], axis=1), spd


def _batch(sizes, seed, dense=(), stand=None, goal_steps=4.8):
    """Scenes of `sizes` (scene b from seed + b; dense[b] pedestrians clustered) -> state [A, 6], speeds [A],
    offsets [B + 1]."""
    dense = list(dense) + [0] * (len(sizes) - len(dense))
    parts = [_scene(n, seed + b, dense[b], stand, goal_steps) for b, n in enumerate(sizes)]
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]), offs


# ---- the case table -----------------------------------------------------------------------------------------------
# sf / orca: keyword settings of the rollout (None: that simulator does not run the case); sf_hits / orca_hits: the
# restatement counters that must be > 0.
Case = namedtuple("Case", "sizes seed dense stand goal_steps sf orca sf_hits orca_hits")


def _case(sizes, seed=0, dense=(), stand=None, goal_steps=4.8, sf=None, orca=None, sf_hits=("out_of_view",),
          orca_hits=()):
    return Case(tuple(sizes), seed, tuple(dense), stand, goal_steps, sf, orca, tuple(sf_hits), tuple(orca_hits))


SF_DEF = {}
ORCA_DEF = {}
SHORT = dict(n_steps=9, sample_every=4)             # the largest scenes: the float64 restatement is O(n^2) per step
ORCA_FULL = dict(neighbor_dist=4.0, time_horizon=4.0, radius=0.6)      # the sweep's default: fills the cap, lp3
DENSE_HITS = ("out_of_view", "speed_clip")
ORCA_DENSE_HITS = ("at_cap", "collision_lines", "lp3")

CASES = {
    # the form boundary: the same four scenes once in the warp form, once beside a 33-pedestrian scene
    "boundary-warp": _case([1, 2, 31, 32], seed=10, dense=(0, 2, 12, 12), sf=SF_DEF, orca=ORCA_FULL,
                           sf_hits=DENSE_HITS, orca_hits=ORCA_DENSE_HITS),
    "boundary-cta": _case([1, 2, 31, 32, 33], seed=10, dense=(0, 2, 12, 12, 12), sf=SF_DEF, orca=ORCA_FULL,
                          sf_hits=DENSE_HITS, orca_hits=ORCA_DENSE_HITS),
    # warp form: B = 1, 5 and 4k + 3 (the last CTA holds three scenes)
    "warp-B1": _case([17], seed=20, dense=(8,), sf=SF_DEF, orca=ORCA_DEF, sf_hits=DENSE_HITS,
                     orca_hits=("collision_lines",)),
    "warp-B5": _case([3, 9, 16, 24, 32], seed=21, dense=(3, 6, 8, 8, 16), sf=SF_DEF, orca=ORCA_FULL,
                     sf_hits=DENSE_HITS, orca_hits=ORCA_DENSE_HITS),
    "warp-B11": _case([1, 5, 32, 7, 12, 30, 2, 19, 25, 8, 31], seed=22, dense=(0, 4, 16, 4, 8, 12, 2, 8, 8, 4, 12),
                      sf=SF_DEF, orca=dict(max_neighbors=16, **ORCA_FULL), sf_hits=DENSE_HITS,
                      orca_hits=ORCA_DENSE_HITS),
    # CTA form: single scenes and mixed batches up to the host's limit, and either side of the register limits the
    # forms had without launch bounds (social force 800, its sweep 672, the ORCA sweep 896 threads)
    "cta-33": _case([33], seed=30, dense=(12,), sf=SF_DEF, orca=ORCA_FULL, sf_hits=DENSE_HITS,
                    orca_hits=ORCA_DENSE_HITS),
    "cta-64": _case([64], seed=31, dense=(24,), sf=SF_DEF, orca=ORCA_FULL, sf_hits=DENSE_HITS,
                    orca_hits=ORCA_DENSE_HITS),
    "cta-mixed": _case([5, 100, 2, 40, 33], seed=32, dense=(4, 24, 2, 12, 8), sf=SF_DEF, orca=ORCA_DEF,
                       sf_hits=DENSE_HITS, orca_hits=("at_cap", "collision_lines", "lp3")),
    "cta-257": _case([257, 100], seed=33, dense=(32, 16), sf=SF_DEF, orca=ORCA_FULL, sf_hits=DENSE_HITS,
                     orca_hits=ORCA_DENSE_HITS),
    "cta-512": _case([512], seed=34, dense=(48,), sf=dict(n_steps=24), orca=ORCA_FULL, sf_hits=DENSE_HITS,
                     orca_hits=ORCA_DENSE_HITS),
    "cta-672": _case([672, 673], seed=35, dense=(48, 48), sf=SHORT, orca=ORCA_FULL, sf_hits=DENSE_HITS,
                     orca_hits=ORCA_DENSE_HITS),
    "cta-800": _case([800, 801], seed=36, dense=(48, 48), sf=SHORT, orca=ORCA_FULL, sf_hits=DENSE_HITS,
                     orca_hits=ORCA_DENSE_HITS),
    "cta-896": _case([896, 897], seed=37, dense=(48, 48), sf=SHORT, orca=ORCA_FULL, sf_hits=DENSE_HITS,
                     orca_hits=ORCA_DENSE_HITS),
    "cta-1024": _case([1024], seed=38, dense=(64,), sf=SHORT, orca=dict(max_neighbors=16, **ORCA_FULL),
                      sf_hits=DENSE_HITS, orca_hits=ORCA_DENSE_HITS),
    # social-force settings on a batch of both forms' sizes (CTA form) and on a warp batch
    "sf-grid-low": _case([5, 12, 40], seed=40, dense=(4, 8, 12), sf=dict(tau=0.3, v0=1.0, sigma=0.2),
                         sf_hits=DENSE_HITS),
    "sf-grid-high": _case([5, 12, 40], seed=40, dense=(4, 8, 12), sf=dict(tau=1.0, v0=5.0, sigma=0.6),
                          sf_hits=DENSE_HITS),
    "sf-grid-opt": _case([6, 20, 31], seed=41, dense=(4, 8, 12), sf=dict(tau=0.5, v0=5.0, sigma=0.3),
                         sf_hits=DENSE_HITS),
    "sf-fps10": _case([5, 12, 40], seed=42, dense=(4, 8, 12), sf=dict(fps=10, n_steps=48), sf_hits=DENSE_HITS),
    "sf-fps15": _case([6, 20, 31], seed=43, dense=(4, 8, 12), sf=dict(fps=15, n_steps=72), sf_hits=DENSE_HITS),
    "sf-fps25": _case([5, 12, 40], seed=44, dense=(4, 8, 12), sf=dict(fps=25, n_steps=120), sf_hits=DENSE_HITS),
    "sf-ragged-steps": _case([5, 12, 40], seed=45, dense=(4, 8, 12), sf=dict(n_steps=45), sf_hits=DENSE_HITS),
    "sf-one-step": _case([5, 12, 40], seed=46, dense=(4, 8, 12), sf=dict(n_steps=1), sf_hits=("out_of_view",)),
    # ORCA settings: neighbour distance / horizon / radius across the tool's values, the neighbour cap at 1 and 16,
    # other frame rates, and an end_range the agents reach
    "orca-small": _case([6, 20, 31], seed=50, dense=(4, 8, 12), orca=dict(neighbor_dist=0.5, time_horizon=0.5,
                                                                          radius=0.2),
                        orca_hits=("collision_lines",)),
    "orca-mixed-a": _case([5, 12, 40], seed=51, dense=(4, 8, 12), orca=dict(neighbor_dist=4.0, time_horizon=0.5,
                                                                            radius=0.2),
                          orca_hits=("at_cap", "collision_lines")),
    "orca-mixed-b": _case([5, 12, 40], seed=52, dense=(4, 8, 12), orca=dict(neighbor_dist=0.5, time_horizon=4.0,
                                                                            radius=0.6),
                          orca_hits=("collision_lines", "lp3")),
    "orca-cap1": _case([6, 20, 31], seed=53, dense=(4, 8, 12), orca=dict(max_neighbors=1, **ORCA_FULL),
                       orca_hits=("at_cap", "collision_lines")),
    "orca-cap16": _case([5, 12, 40], seed=54, dense=(4, 8, 12), orca=dict(max_neighbors=16, **ORCA_FULL),
                        orca_hits=ORCA_DENSE_HITS),
    "orca-end-range": _case([5, 12, 40], seed=55, goal_steps=1.5, orca=dict(end_range=0.5),
                            orca_hits=("end_range_stops",)),
    "orca-end-range-warp": _case([6, 20, 31], seed=56, goal_steps=1.0, orca=dict(end_range=1.0, **ORCA_FULL),
                                 orca_hits=("end_range_stops", "at_cap")),
    "orca-fps10": _case([5, 12, 40], seed=57, dense=(4, 8, 12), orca=dict(fps=10, n_steps=49, sample_every=4),
                        orca_hits=("collision_lines",)),
    "orca-fps25": _case([5, 12, 40], seed=58, dense=(4, 8, 12), orca=dict(fps=25, n_steps=121, sample_every=10,
                                                                          **ORCA_FULL),
                        orca_hits=ORCA_DENSE_HITS),
    # a pedestrian standing on its destination: NaN desired direction (social force), pref-velocity 0 (ORCA)
    "nan-destination": _case([6, 40], seed=60, dense=(4, 8), stand=2, sf=SF_DEF, orca=ORCA_DEF,
                             sf_hits=("out_of_view",), orca_hits=("end_range_stops",)),
}


def _n_max(case):
    return max(case.sizes)


def _sf_kwargs(s):
    fps = s.get("fps", 20)
    return dict(tau=s.get("tau", 0.5), v0=s.get("v0", 2.1), sigma=s.get("sigma", 0.3), fps=fps,
                n_steps=s.get("n_steps", 96), sample_every=s.get("sample_every", sampling_rate(fps)))


def _orca_kwargs(s):
    fps = s.get("fps", 20)
    return dict(neighbor_dist=s.get("neighbor_dist", 1.5), time_horizon=s.get("time_horizon", 1.5),
                radius=s.get("radius", 0.4), max_neighbors=s.get("max_neighbors", 10),
                end_range=s.get("end_range", 0.05), fps=fps, n_steps=s.get("n_steps", 97),
                sample_every=s.get("sample_every", sampling_rate(fps)))


def _inputs(case):
    return _batch(case.sizes, case.seed, case.dense, case.stand, case.goal_steps)


def _sf_restated(state, k, counters=None):
    return C.sf_simulate(state, delta_t=1.0 / k["fps"], tau=k["tau"], v0=k["v0"], sigma=k["sigma"],
                         n_steps=k["n_steps"], sample_every=k["sample_every"], counters=counters)


def _orca_restated(state, spd, k, counters=None):
    return orca_simulate(state[:, 0:2], state[:, 2:4], state[:, 4:6], spd, time_step=1.0 / k["fps"],
                         neighbor_dist=k["neighbor_dist"], max_neighbors=k["max_neighbors"],
                         time_horizon=k["time_horizon"], radius=k["radius"], end_range=k["end_range"],
                         n_steps=k["n_steps"], sample_every=k["sample_every"], counters=counters)


@functools.lru_cache(maxsize=None)
def _sf_ref(name):
    """Per scene of CASES[name]: the restatement's samples; and its counters summed over the scenes."""
    case = CASES[name]
    state, _, offs = _inputs(case)
    k = _sf_kwargs(case.sf)
    counters = {}
    with np.errstate(invalid="ignore", divide="ignore"):
        out = [_sf_restated(state[offs[b]:offs[b + 1]], k, counters) for b in range(len(case.sizes))]
    return out, counters


@functools.lru_cache(maxsize=None)
def _orca_ref(name):
    case = CASES[name]
    state, spd, offs = _inputs(case)
    k = _orca_kwargs(case.orca)
    counters = {}
    out = [_orca_restated(state[offs[b]:offs[b + 1]], spd[offs[b]:offs[b + 1]], k, counters)
           for b in range(len(case.sizes))]
    return out, counters


SF_CASES = [n for n, c in CASES.items() if c.sf is not None]
ORCA_CASES = [n for n, c in CASES.items() if c.orca is not None]


# ---- CPU: what each case reaches -----------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SF_CASES)
def test_sf_case_reaches_its_branches(name):
    case = CASES[name]
    _, counters = _sf_ref(name)
    for key in case.sf_hits:
        assert counters[key] > 0, (name, key, counters)


@pytest.mark.parametrize("name", ORCA_CASES)
def test_orca_case_reaches_its_branches(name):
    case = CASES[name]
    _, counters = _orca_ref(name)
    for key in case.orca_hits:
        assert counters[key] > 0, (name, key, counters)


def test_case_forms():
    """The launch form is a function of the batch's n_max: the names say which form a case is for."""
    for name, case in CASES.items():
        if name.startswith(("warp", "boundary-warp")):
            assert _n_max(case) <= WARP_MAX, name
        if name.startswith(("cta", "boundary-cta")):
            assert _n_max(case) > WARP_MAX, name
    sizes = sorted({n for c in CASES.values() for n in c.sizes})
    for n in (1, 2, 31, 32, 33, 64, 100, 257, 512, 672, 673, 800, 801, 896, 897, 1024):
        assert n in sizes, n


# ---- CPU: the social-force gate bites -------------------------------------------------------------------------------
def _sf_variant(state0, variant, tau=0.5, v0=2.1, sigma=0.3, fps=20, n_steps=96, sample_every=8):
    """sf_simulate with one of the mistakes a kernel could make, from sf_step:
      skip_last -- the neighbour loop stops at b = n - 2 (an off-by-one thread bound);
      stale     -- pedestrian 0 reads pedestrian 1's previous-step state (a missing barrier);
      late      -- every sample taken one step late."""
    dt = 1.0 / fps
    state = np.concatenate([state0, np.full((len(state0), 1), tau)], axis=1)
    s0 = np.linalg.norm(state[:, 2:4], axis=-1)
    smax = 1.3 * s0
    prev = state.copy()
    late = int(variant == "late")
    out = []
    with np.errstate(invalid="ignore", divide="ignore"):
        for k in range(n_steps):
            cur = state.copy()
            state = C.sf_step(cur.copy(), s0, smax, dt, v0, sigma)
            if variant == "skip_last" and len(cur) > 1:
                state[:-1] = C.sf_step(cur[:-1].copy(), s0[:-1], smax[:-1], dt, v0, sigma)
            if variant == "stale" and len(cur) > 1:
                mixed = cur.copy()
                mixed[1] = prev[1]
                state[0] = C.sf_step(mixed, s0, smax, dt, v0, sigma)[0]
            prev = cur
            if k >= late and (k - late) % sample_every == 0:
                out.append(state[:, 0:2].copy())
    return np.stack(out)


@pytest.mark.parametrize("variant", ["skip_last", "stale", "late"])
def test_sf_gate_catches_kernel_mistakes(variant):
    """Each mistake moves some sampled position past SF_GATE by a factor of 1000 on one of the table's scenes."""
    worst = 0.0
    for name in ("cta-33", "cta-64", "warp-B5"):
        case = CASES[name]
        state, _, offs = _inputs(case)
        k = _sf_kwargs(case.sf)
        ref, _ = _sf_ref(name)
        for b in range(len(case.sizes)):
            if case.sizes[b] < 2:
                continue
            got = _sf_variant(state[offs[b]:offs[b + 1]], variant, k["tau"], k["v0"], k["sigma"], k["fps"],
                              k["n_steps"], k["sample_every"])
            m = min(len(got), len(ref[b]))
            worst = max(worst, float(np.nanmax(np.abs(got[:m] - ref[b][:m]))))
    assert worst > 1e3 * SF_GATE, (variant, worst)


def test_sf_force_sum_runs_in_index_order():
    """The restatement sums the pairwise forces b = 0 .. n-1 before adding the driving force, like the kernel: the
    same step with the sum reordered (b = n-1 .. 0) is a different float64 result somewhere on a dense scene."""
    state, _, _ = _batch([64], seed=31, dense=(24,))
    st = np.concatenate([state, np.full((64, 1), 0.5)], axis=1)
    s0 = np.linalg.norm(st[:, 2:4], axis=-1)
    a = C.sf_step(st.copy(), s0, 1.3 * s0, 0.05, 2.1, 0.3)
    rev = st[::-1].copy()
    b = C.sf_step(rev, s0[::-1].copy(), 1.3 * s0[::-1], 0.05, 2.1, 0.3)[::-1]
    assert np.abs(a - b).max() < 1e-12 and not np.array_equal(a, b)


# ---- GPU: rollouts ------------------------------------------------------------------------------------------------
def _layout_n_max(offs):
    from trajnetplusplusbaselines_b200.engine import SceneLayout
    return SceneLayout(offs).max_scene


def _sf_device(name):
    from trajnetplusplusbaselines_b200.classical import socialforce
    case = CASES[name]
    state, _, offs = _inputs(case)
    assert _layout_n_max(offs) == _n_max(case)
    k = _sf_kwargs(case.sf)
    out = socialforce.simulate_batch(state, offs.tolist(), (k["tau"], k["v0"], k["sigma"]), n_steps=k["n_steps"],
                                     sample_every=k["sample_every"], fps=k["fps"]).cpu().numpy()
    return [out[:, offs[b]:offs[b + 1]] for b in range(len(case.sizes))]


def _orca_device(name):
    from trajnetplusplusbaselines_b200.classical import orca
    case = CASES[name]
    state, spd, offs = _inputs(case)
    assert _layout_n_max(offs) == _n_max(case)
    k = _orca_kwargs(case.orca)
    out = orca.simulate_batch(state[:, 0:2], state[:, 2:4], state[:, 4:6], spd, offs.tolist(),
                              (k["neighbor_dist"], k["time_horizon"], k["radius"]), n_steps=k["n_steps"],
                              sample_every=k["sample_every"], fps=k["fps"], max_neighbors=k["max_neighbors"],
                              end_range=k["end_range"]).cpu().numpy()
    return [out[:, offs[b]:offs[b + 1]] for b in range(len(case.sizes))]


def _sf_error(got, ref):
    """max |device - restatement| over the finite samples; the NaN patterns must be equal."""
    assert got.shape == ref.shape
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    return float(np.abs(got[fin] - ref[fin]).max()) if fin.any() else 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("name", SF_CASES)
def test_sf_rollout_matches_restatement(name):
    ref, _ = _sf_ref(name)
    got = _sf_device(name)
    worst = max(_sf_error(g, r) for g, r in zip(got, ref))
    print("sf   %-20s n_max %4d  worst %.3g m" % (name, _n_max(CASES[name]), worst))
    assert worst < SF_GATE, (name, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ORCA_CASES)
def test_orca_rollout_matches_restatement_bit_exact(name):
    ref, _ = _orca_ref(name)
    got = _orca_device(name)
    for b, (g, r) in enumerate(zip(got, ref)):
        assert g.shape == r.shape
        assert np.array_equal(g, r), (name, b, int((g != r).sum()), float(np.abs(g - r).max()))


@pytest.mark.gpu
def test_form_boundary_is_bit_identical():
    """Scenes of 1, 2, 31 and 32 pedestrians give the same bits in the warp form and in the CTA form."""
    for dev in (_sf_device, _orca_device):
        warp, cta = dev("boundary-warp"), dev("boundary-cta")
        for b in range(4):
            assert warp[b].tobytes() == cta[b].tobytes(), (dev.__name__, b)


@pytest.mark.gpu
def test_nan_destination_pattern():
    got = _sf_device("nan-destination")
    ref, _ = _sf_ref("nan-destination")
    for g, r in zip(got, ref):
        assert np.isnan(r).any() and np.array_equal(np.isnan(g), np.isnan(r))


ONE_STEP_SIZES = (1, 2, 31, 32, 33, 64, 100, 257, 512, 672, 673, 800, 801, 896, 897, 1024)


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["warp", "cta"])
def test_sf_one_step_near_float64_rounding(form):
    """One step (n_steps = sample_every = 1) from random states at every size of the table: the kernel's arithmetic
    against the restatement's, before any amplification."""
    from trajnetplusplusbaselines_b200.classical import socialforce
    sizes = [n for n in ONE_STEP_SIZES if (n <= WARP_MAX) == (form == "warp")]
    state, _, offs = _batch(sizes, seed=70, dense=[min(n, 32) for n in sizes])
    assert (_layout_n_max(offs) <= WARP_MAX) == (form == "warp")
    out = socialforce.simulate_batch(state, offs.tolist(), n_steps=1, sample_every=1).cpu().numpy()
    for b, n in enumerate(sizes):
        ref = C.sf_simulate(state[offs[b]:offs[b + 1]], n_steps=1, sample_every=1)
        err = _sf_error(out[:, offs[b]:offs[b + 1]], ref)
        print("sf one step n %4d  %.3g m" % (n, err))
        assert err < SF_STEP_GATE, (n, err)


@pytest.mark.gpu
def test_host_refuses_scenes_above_1024():
    from trajnetplusplusbaselines_b200.classical import common, orca, socialforce
    state, spd, offs = _batch([3, N_LIMIT + 1], seed=80)
    with pytest.raises(RuntimeError, match="1024"):
        socialforce.simulate_batch(state, offs.tolist())
    with pytest.raises(RuntimeError, match="1024"):
        orca.simulate_batch(state[:, :2], state[:, 2:4], state[:, 4:], spd, offs.tolist())
    prepared = common.to_device(state, spd, offs, np.zeros((2, 12, 2)))
    with pytest.raises(RuntimeError, match="1024"):
        socialforce.sweep(prepared, [sweep.SF_DEFAULT])
    with pytest.raises(RuntimeError, match="1024"):
        orca.sweep(prepared, [sweep.ORCA_DEFAULT])


# ---- GPU: sweeps against the restatement ---------------------------------------------------------------------------
def _truth(state, offs, T, seed):
    rng = np.random.RandomState(seed)
    p0, v0 = state[offs[:-1], 0:2], state[offs[:-1], 2:4]
    return p0[:, None] + v0[:, None] * 0.4 * np.arange(1, T + 1)[None, :, None] + rng.randn(len(offs) - 1, T, 2) * 0.2


def _check_sweep(sizes, seed, dense, T, fps, sf_grid, orca_grid, max_neighbors=10, end_range=0.05):
    """socialforce.sweep / orca.sweep on the scenes against sweep.score of the restatement's primary."""
    from trajnetplusplusbaselines_b200.classical import common, orca, socialforce
    state, spd, offs = _batch(sizes, seed, dense)
    truth = _truth(state, offs, T, seed)
    prepared = common.to_device(state, spd, offs, truth)
    assert prepared.layout.max_scene == max(sizes)
    rate = sampling_rate(fps)
    worst = 0.0
    if sf_grid:
        ade, fde = (t.cpu().numpy() for t in socialforce.sweep(prepared, sf_grid, fps=fps))
        for s, (tau, v0, sigma) in enumerate(sf_grid):
            k = dict(tau=tau, v0=v0, sigma=sigma, fps=fps, n_steps=T * rate, sample_every=rate)
            for b in range(len(sizes)):
                with np.errstate(invalid="ignore", divide="ignore"):
                    pos = _sf_restated(state[offs[b]:offs[b + 1]], k)
                ea, ef = sweep.score(truth[b], pos[:, 0])
                worst = max(worst, abs(ade[s, b] - ea), abs(fde[s, b] - ef))
        assert worst < SF_GATE, worst
    if orca_grid:
        ade, fde = (t.cpu().numpy() for t in orca.sweep(prepared, orca_grid, fps=fps, max_neighbors=max_neighbors,
                                                        end_range=end_range))
        for s, (nd, th, r) in enumerate(orca_grid):
            k = dict(neighbor_dist=nd, time_horizon=th, radius=r, max_neighbors=max_neighbors, end_range=end_range,
                     fps=fps, n_steps=T * rate + 1, sample_every=rate)
            for b in range(len(sizes)):
                pos = _orca_restated(state[offs[b]:offs[b + 1]], spd[offs[b]:offs[b + 1]], k)
                ea, ef = sweep.score(truth[b], pos[:, 0].astype(np.float64))
                assert ade[s, b] == ea and fde[s, b] == ef, ("orca", s, b, sizes[b], ade[s, b], ea)
    print("sweep sizes %s: sf worst %.3g" % (sizes[:4], worst))


PACKED_SIZES = [1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 100]
PACKED_DENSE = [0, 2, 3, 4, 4, 4, 6, 6, 8, 8, 8, 12, 12, 12, 24]
ORCA_SWEEP = [sweep.ORCA_DEFAULT, (1.5, 1.5, 0.4), (0.5, 0.5, 0.2), (8.0, 0.5, 0.2), (1.5, 4.0, 0.6)]


@pytest.mark.gpu
def test_sweep_packed_and_cta_match_restatement():
    """Packing widths 1 .. 32 and the CTA form in one batch; P = 3 / 5 settings, a multiple of no packing."""
    _check_sweep(PACKED_SIZES, 90, PACKED_DENSE, 12, 20, [sweep.SF_DEFAULT, SF_GRID[0], SF_GRID[-1]], ORCA_SWEEP)


@pytest.mark.gpu
def test_sweep_fields_match_restatement():
    """fps 10 and 25 (sample_every 4 and 10), max_neighbors 1 and 16, an end_range the agents reach."""
    _check_sweep(PACKED_SIZES, 91, PACKED_DENSE, 6, 10, [(0.5, 5.0, 0.3), SF_GRID[4]], ORCA_SWEEP[:3],
                 max_neighbors=1, end_range=1.0)
    _check_sweep(PACKED_SIZES, 92, PACKED_DENSE, 4, 25, [sweep.SF_DEFAULT], ORCA_SWEEP, max_neighbors=16)


@pytest.mark.gpu
def test_sweep_largest_scenes_match_restatement():
    """The CTA form at the former register limits and at 1024; truth shortened to keep the restatement short."""
    _check_sweep([672, 673, 1024], 93, [48, 48, 64], 2, 10, [sweep.SF_DEFAULT, (1.0, 5.0, 0.6)], None)
    _check_sweep([896, 897, 1024, 40], 94, [48, 48, 64, 12], 12, 20, None, ORCA_SWEEP[:3], max_neighbors=16)


# ---- GPU: a training file in the CTA form ---------------------------------------------------------------------------
def _train_file_or_skip(name):
    root = reference_root()
    files = glob.glob(os.path.join(root, "DATA_BLOCK", "trajdata", "train", name)) if root else []
    if not files:
        pytest.skip("DATA_BLOCK not present (build() copies it under oracle/_ref)")
    return files[0]


@pytest.mark.gpu
def test_crowds_students001_in_the_cta_form():
    """Every scene of crowds_students001 runs in the CTA form; a subset, its largest scene included, matches the
    restatements, as positions (simulate_batch) and as ADE / FDE (sweep)."""
    from trajnetplusplusbaselines_b200.classical import orca, socialforce
    prepared = sweep.prepare_file(_train_file_or_skip("crowds_students001.ndjson"))
    offs = prepared.agent_offsets
    sizes = np.diff(offs)
    assert prepared.layout.max_scene == sizes.max() > WARP_MAX
    state, spd, truth = (t.cpu().numpy() for t in (prepared.state, prepared.speeds, prepared.truth))
    sf_pos = socialforce.simulate_batch(state, offs.tolist(), sweep.SF_DEFAULT).cpu().numpy()
    orca_pos = orca.simulate_batch(state[:, :2], state[:, 2:4], state[:, 4:], spd, offs.tolist()).cpu().numpy()
    sf_ade, sf_fde = (t.cpu().numpy()[0] for t in socialforce.sweep(prepared, [sweep.SF_DEFAULT]))
    o_ade, o_fde = (t.cpu().numpy()[0] for t in orca.sweep(prepared, [sweep.ORCA_DEFAULT]))
    pick = sorted({int(np.argmax(sizes)), int(np.argmin(sizes)), 0, len(sizes) // 2, len(sizes) - 1})
    worst = 0.0
    for b in pick:
        lo, hi = offs[b], offs[b + 1]
        with np.errstate(invalid="ignore", divide="ignore"):
            ref = C.sf_simulate(state[lo:hi], tau=sweep.SF_DEFAULT[0], v0=sweep.SF_DEFAULT[1],
                                sigma=sweep.SF_DEFAULT[2])
        worst = max(worst, _sf_error(sf_pos[:, lo:hi], ref))
        k = _orca_kwargs({})
        assert np.array_equal(orca_pos[:, lo:hi], _orca_restated(state[lo:hi], spd[lo:hi], k)), b
        ea, ef = sweep.score(truth[b], ref[:, 0])
        assert (np.isnan(ea) and np.isnan(sf_ade[b])) or abs(sf_ade[b] - ea) < SF_GATE, b
        assert (np.isnan(ef) and np.isnan(sf_fde[b])) or abs(sf_fde[b] - ef) < SF_GATE, b
        k = _orca_kwargs(dict(zip(("neighbor_dist", "time_horizon", "radius"), sweep.ORCA_DEFAULT)))
        ea, ef = sweep.score(truth[b], _orca_restated(state[lo:hi], spd[lo:hi], k)[:, 0].astype(np.float64))
        assert o_ade[b] == ea and o_fde[b] == ef, b
    print("crowds_students001 scenes %s (sizes %s): sf worst %.3g m" % (pick, sizes[pick].tolist(), worst))
    assert worst < SF_GATE, worst
