"""Social-force / ORCA parameter sweeps (classical.sweep, tb2_sf_sweep / tb2_orca_sweep) and their host preparation.

The sweep is defined against this package's own simulate_batch (parity with upstream socialforce / rvo2 stays unpinned,
DESIGN.md section 2): per setting, its ADE / FDE equal bit for bit the primary's distances to the truth computed from
simulate_batch's positions, summed in sample order in float64.
"""
import glob
import itertools
import os
import sys
import types

import numpy as np
import pytest

from oracle.ref_shim import reference_root
from trajnetplusplusbaselines_b200 import data
from trajnetplusplusbaselines_b200.classical import common, sweep
from trajnetplusplusbaselines_b200.classical.common import initial_states, initial_states_xy

SF_GRID = list(itertools.product((0.3, 0.5, 1.0), (1.0, 2.1, 5.0), (0.2, 0.3, 0.6)))          # 27, defaults included
ORCA_GRID = list(itertools.product((1.5, 4.0, 8.0), (1.5, 4.0, 0.5), (0.4, 0.6, 0.2)))       # 27: predict's and the tool's


def _train_files():
    root = reference_root()
    return sorted(glob.glob(os.path.join(root, "DATA_BLOCK", "trajdata", "train", "*.ndjson"))) if root else []


def _assert_same_prep(scenes_xy, scenes_rows, dest_type, obs_length=9, pred_length=12):
    """initial_states_xy over the xy list == initial_states per scene on the rows, bit for bit."""
    try:
        got = initial_states_xy(scenes_xy, obs_length, pred_length, dest_type)
    except IndexError:
        got = None
    ref_st, ref_sp, ref_tr, counts, ref_err = [], [], [], [], False
    for _, paths in scenes_rows:
        try:
            st, sp = initial_states(paths, paths[0][obs_length - 1].frame, pred_length, None, dest_type)
        except IndexError:
            ref_err = True
            break
        ref_st.append(st)
        ref_sp.append(sp)
        counts.append(len(st))
        ref_tr.append([[r.x, r.y] for r in paths[0][-pred_length:]])
    assert (got is None) == ref_err
    if got is None:
        return
    state, speeds, offsets, truth = got
    assert np.array_equal(state, np.concatenate(ref_st), equal_nan=True)
    assert np.array_equal(speeds, np.concatenate(ref_sp), equal_nan=True)
    assert np.array_equal(offsets, np.concatenate([[0], np.cumsum(counts)]))
    assert np.array_equal(truth, np.array(ref_tr, dtype=np.float64))


# ---- host preparation (CPU) ---------------------------------------------------------------------------------------
def test_initial_states_xy_matches_paths_on_training_files():
    files = _train_files()
    if not files:
        pytest.skip("DATA_BLOCK not present (neither the reference tree nor oracle/_ref)")
    assert len(files) == 7
    for fn in files:
        scenes_xy = sweep.load_scenes(fn)
        rows = list(data.read_ndjson_scenes(fn))
        assert len(scenes_xy) == len(rows)
        for dest_type in ("interp", "vel"):
            _assert_same_prep(scenes_xy, rows, dest_type)
        for (sx, xy), (sr, paths) in zip(scenes_xy, rows):       # pred_end: every scene on its own (some raise)
            assert sx == sr
            _assert_same_prep([(sx, xy)], [(sr, paths)], "pred_end")


def _synthetic_rows(seed):
    """Scenes with late entries, 1-3 past rows, gaps, stationary tracks and tracks that leave early."""
    rng = np.random.RandomState(seed)
    scenes = []
    for s in range(30):
        n = rng.randint(1, 9)
        paths = []
        for p in range(n):
            x0, v = rng.randn(2) * 3, rng.randn(2) * 0.4
            if p == 0:
                frames = list(range(21))
            else:
                kind = rng.randint(6)
                frames = {0: range(21), 1: range(8 - rng.randint(0, 3), 21),          # 1-3 past rows
                          2: [f for f in range(21) if f % 3 != 1],                    # gaps
                          3: range(rng.randint(0, 8), 21),                            # late entry
                          4: range(0, rng.randint(3, 15)),                            # leaves (maybe before start)
                          5: range(21)}[kind]
                if kind == 5:
                    v = np.zeros(2)                                                   # stationary
            if p == 0 and s % 7 == 3:
                v = np.zeros(2)                                                       # stationary primary
            paths.append([data.TrackRow(10 * f, 100 * s + p, float(x0[0] + v[0] * f + 0.01 * rng.randn()),
                                        float(x0[1] + v[1] * f)) for f in frames])
        paths = [paths[0]] + [pp for pp in paths[1:] if len(pp)]
        scenes.append((s, paths))
    return scenes


@pytest.mark.parametrize("dest_type", ["interp", "vel", "pred_end"])
def test_initial_states_xy_matches_paths_on_synthetic_scenes(dest_type):
    rows = _synthetic_rows(seed=11)
    scenes_xy = [(sid, data.paths_to_xy(paths)) for sid, paths in rows]
    if dest_type == "pred_end":
        for x, r in zip(scenes_xy, rows):
            _assert_same_prep([x], [r], dest_type)
    else:
        _assert_same_prep(scenes_xy, rows, dest_type)
    _assert_same_prep([(sid, paths) for sid, paths in rows[:5]], rows[:5], "interp")          # rows pass through


def test_unrepresentable_scenes_go_through_the_rows(tmp_path):
    """A neighbour with a row between the primary's frames counts as a past row in the reference; the xy array drops
    it, so load_scenes hands that scene over as rows."""
    lines = ['{"scene": {"id": 0, "p": 1, "s": 0, "e": 200, "fps": 2.5, "tag": 1}}',
             '{"scene": {"id": 1, "p": 3, "s": 80, "e": 280, "fps": 2.5, "tag": 1}}']            # after the odd row
    for f in range(0, 290, 10):
        lines.append('{"track": {"f": %d, "p": 1, "x": %.2f, "y": 0.5}}' % (f, 0.04 * f))
        lines.append('{"track": {"f": %d, "p": 2, "x": 1.0, "y": %.2f}}' % (f, 0.03 * f))
        lines.append('{"track": {"f": %d, "p": 3, "x": %.2f, "y": 2.0}}' % (f, -0.02 * f))
        if f == 70:
            lines.append('{"track": {"f": 75, "p": 2, "x": 1.0, "y": 9.0}}')
    fn = tmp_path / "odd.ndjson"
    fn.write_text("\n".join(lines) + "\n")
    scenes = sweep.load_scenes(str(fn))
    assert not isinstance(scenes[0][1], np.ndarray) and isinstance(scenes[1][1], np.ndarray)
    rows = list(data.read_ndjson_scenes(str(fn)))
    _assert_same_prep(scenes, rows, "interp")
    xy_only = [(sid, data.paths_to_xy(p)) for sid, p in rows]
    assert not np.array_equal(initial_states_xy(xy_only)[0], initial_states_xy(scenes)[0])


def test_argument_validation():
    fake = types.SimpleNamespace(truth=np.zeros((3, 12, 2)))
    from trajnetplusplusbaselines_b200.classical import orca, socialforce
    for bad in ([], [[0.5, 2.1]], [[0.0, 2.1, 0.3]], [[0.5, 2.1, -1.0]], [[np.nan, 2.1, 0.3]], [[0.5, np.inf, 0.3]]):
        with pytest.raises(ValueError):
            socialforce.sweep(fake, bad)
    for bad in ([], [[1.5, 0.0, 0.4]], [[1.5, 1.5, 0.0]], [[np.nan, 1.5, 0.4]], [[1.5, 1e39, 0.4]]):   # 1e39: inf in float
        with pytest.raises(ValueError):
            orca.sweep(fake, bad)
    with pytest.raises(ValueError):
        socialforce.sweep(types.SimpleNamespace(truth=np.zeros((2 ** 21, 12, 2))), np.ones((1024, 3)))
    with pytest.raises(ValueError):
        initial_states_xy([(0, np.full((21, 2, 2), np.nan))])                   # primary missing at some frame
    with pytest.raises(ValueError):
        initial_states_xy([(0, np.zeros((21, 2, 2)))], dest_type="true")
    with pytest.raises(NotImplementedError):
        initial_states_xy([(0, np.zeros((21, 2, 2)))], dest_type="nope")
    with pytest.raises(ValueError):
        initial_states_xy([(0, np.zeros((10, 2, 2)))])                           # truth shorter than pred_length


def test_fit_picks_lowest_finite_mean():
    ade = np.array([[1.0, 2.0, np.nan], [0.5, 2.5, 3.0], [1.0, 0.5, 1.5], [np.nan, np.nan, np.nan]])
    r = sweep.fit([ade[:, :2], ade[:, 2:]])
    assert r["files"][0]["best"] == 2 and list(r["files"][0]["ade"][:3]) == [1.5, 1.5, 0.75]
    assert r["files"][1]["best"] == 2 and list(r["files"][1]["skipped"]) == [1, 0, 0, 1]
    assert r["pooled"]["best"] == 2 and r["pooled"]["finite"][0] == 2
    assert sweep.fit([np.array([[1.0, 2.0], [2.0, 1.0]])])["pooled"]["best"] == 0          # tie -> lowest index
    assert sweep.fit([np.full((2, 3), np.nan)])["pooled"]["best"] is None


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _ragged(sizes, seed, nan_primary=False):
    """Synthetic prepared arrays: scene b has sizes[b] pedestrians heading roughly at each other."""
    rng = np.random.RandomState(seed)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    A = int(offs[-1])
    pos = rng.randn(A, 2) * (1.0 + 0.15 * np.sqrt(np.repeat(sizes, sizes)))[:, None]
    ang = rng.rand(A) * 2 * np.pi
    spd = 0.3 + rng.rand(A) * 1.2
    vel = np.stack([spd * np.cos(ang), spd * np.sin(ang)], axis=1)
    goal = pos + vel * 4.8 + rng.randn(A, 2) * 0.3
    if nan_primary:
        goal[offs[1]] = pos[offs[1]]                            # scene 1's primary stands on its destination
    state = np.concatenate([pos, vel, goal], axis=1)
    truth = pos[offs[:-1]][:, None] + vel[offs[:-1]][:, None] * 0.4 * np.arange(1, 13)[None, :, None] \
        + rng.randn(len(sizes), 12, 2) * 0.2
    return state, spd, offs, truth


def _expected(positions, offs, truth):
    """(ade [B], fde [B]) from simulate_batch's positions [12, A, 2], in the kernels' documented order."""
    pos = positions.astype(np.float64)
    out = np.array([sweep.score(truth[b], pos[:, offs[b]]) for b in range(len(offs) - 1)])
    return out[:, 0], out[:, 1]


def _check_equal(prepared, state, spd, offs, truth, sf_grid, orca_grid):
    from trajnetplusplusbaselines_b200.classical import orca, socialforce
    ade, fde = (t.cpu().numpy() for t in socialforce.sweep(prepared, sf_grid))
    assert ade.shape == (len(sf_grid), len(offs) - 1)
    for s, prm in enumerate(sf_grid):
        ref = socialforce.simulate_batch(state, offs, prm, n_steps=96, sample_every=8).cpu().numpy()
        ea, ef = _expected(ref, offs, truth)
        assert np.array_equal(ade[s], ea, equal_nan=True) and np.array_equal(fde[s], ef, equal_nan=True), ("sf", prm)
    ade, fde = (t.cpu().numpy() for t in orca.sweep(prepared, orca_grid))
    for s, prm in enumerate(orca_grid):
        ref = orca.simulate_batch(state[:, 0:2], state[:, 2:4], state[:, 4:6], spd, offs, prm, n_steps=97,
                                  sample_every=8).cpu().numpy()
        ea, ef = _expected(ref, offs, truth)
        assert np.array_equal(ade[s], ea, equal_nan=True) and np.array_equal(fde[s], ef, equal_nan=True), ("orca", prm)


@pytest.mark.gpu
def test_sweep_equals_simulate_batch_on_ragged_scenes():
    """Packing widths 1, 2, 4, 8, 16, 32 and one 40-pedestrian scene (a CTA per item); 27 settings (not a multiple of
    any packing), P = 1 and B = 1."""
    sizes = [1, 2, 3, 5, 8, 9, 16, 17, 31, 32, 40, 4, 6, 12]
    state, spd, offs, truth = _ragged(sizes, seed=4)
    prepared = common.to_device(state, spd, offs, truth)
    _check_equal(prepared, state, spd, offs, truth, SF_GRID, ORCA_GRID)
    _check_equal(prepared, state, spd, offs, truth, [sweep.SF_DEFAULT], [sweep.ORCA_DEFAULT])       # P = 1
    for b in (0, 4, 10):                                                                          # B = 1
        s, e = offs[b], offs[b + 1]
        one = common.to_device(state[s:e], spd[s:e], [0, e - s], truth[b:b + 1])
        _check_equal(one, state[s:e], spd[s:e], np.array([0, e - s]), truth[b:b + 1], SF_GRID[:5], ORCA_GRID[:3])


def _train_file_or_skip(name="biwi_hotel.ndjson"):
    files = [f for f in _train_files() if f.endswith(name)]
    if not files:
        pytest.skip("DATA_BLOCK not present (build() copies it under oracle/_ref)")
    return files[0]


@pytest.mark.gpu
def test_sweep_equals_simulate_batch_on_a_training_file():
    prepared = sweep.prepare_file(_train_file_or_skip())
    state, spd = prepared.state.cpu().numpy(), prepared.speeds.cpu().numpy()
    _check_equal(prepared, state, spd, prepared.agent_offsets, prepared.truth.cpu().numpy(), SF_GRID, ORCA_GRID)


@pytest.mark.gpu
def test_sweep_against_reference_metrics():
    """The same ADE / FDE through metrics_oracle.average_l2 / final_l2 on TrackRows (NumPy's pairwise mean)."""
    from oracle import metrics_oracle as M
    from trajnetplusplusbaselines_b200.classical import orca, socialforce
    state, spd, offs, truth = _ragged([3, 7, 12, 33, 1], seed=9)
    prepared = common.to_device(state, spd, offs, truth)
    rows = lambda xy: [data.TrackRow(9 + i, 0, float(x), float(y)) for i, (x, y) in enumerate(xy)]
    for sim, grid in ((socialforce, SF_GRID[::5]), (orca, ORCA_GRID[::5])):
        ade, fde = (t.cpu().numpy() for t in sim.sweep(prepared, grid))
        for s, prm in enumerate(grid):
            if sim is socialforce:
                pos = socialforce.simulate_batch(state, offs, prm).cpu().numpy()
            else:
                pos = orca.simulate_batch(state[:, :2], state[:, 2:4], state[:, 4:], spd, offs, prm).cpu().numpy()
            for b in range(len(offs) - 1):
                gt, pred = rows(truth[b]), rows(pos[:, offs[b]].astype(np.float64))
                assert ade[s, b] == pytest.approx(M.average_l2(gt, pred), rel=1e-12, abs=0)
                assert fde[s, b] == pytest.approx(M.final_l2(gt, pred), rel=1e-12, abs=0)


@pytest.mark.gpu
def test_dropin_reference_socialforce_eval():
    """The reference's own socialforce_eval.Evaluator.aggregate, with this package's predictors and metrics_oracle
    standing in for trajnetplusplustools.metrics, equals sweep.evaluate on one training file.

    Deviation from the shipped tool: aggregate passes `args=` to the social-force and ORCA predictors (:46, :48), which
    neither accepts, and never passes n_predict / obs_length; so it is handed thin adapters that drop `args` and forward
    args.pred_length / args.obs_length.  The trajnetplusplustools.metrics / .interactions stubs it imports are registered
    here for the duration of the test."""
    from oracle import metrics_oracle as M
    from oracle.ref_shim import import_reference
    from trajnetplusplusbaselines_b200.classical import kalman, orca, socialforce
    fn = _train_file_or_skip()
    import_reference()
    mp = pytest.MonkeyPatch()
    try:
        tools = sys.modules["trajnetplusplustools"]
        mp.setattr(tools, "metrics", M, raising=False)
        inter = types.ModuleType("trajnetplusplustools.interactions")
        inter.collision_avoidance = None
        mp.setitem(sys.modules, "trajnetplusplustools.interactions", inter)
        mp.setattr(tools, "interactions", inter, raising=False)
        from trajnetbaselines.classical import socialforce_eval as ref
        args = types.SimpleNamespace(obs_length=9, pred_length=12)
        sf = lambda paths, dest, dest_type, params, args: socialforce.predict(
            paths, dest, dest_type, params, n_predict=args.pred_length, obs_length=args.obs_length)
        oc = lambda paths, dest, dest_type, params, args: orca.predict(
            paths, dest, dest_type, params, n_predict=args.pred_length, obs_length=args.obs_length)
        scenes = [paths for _, paths in data.read_ndjson_scenes(fn)]
        prepared = sweep.prepare_file(fn)
        for sfp, op in ((sweep.SF_DEFAULT, sweep.ORCA_DEFAULT), ((0.3, 5.0, 0.6), (1.5, 1.5, 0.4))):
            ev = ref.Evaluator(scenes, None, {"sf": list(sfp), "orca": list(op)}, args)
            ev.aggregate("orcainterp", oc, "interp")
            ev.aggregate("sfinterp", sf, "interp")
            np.random.seed(3)
            ev.aggregate("kf", kalman.predict)
            r_avg, r_fin = ev.result()
            np.random.seed(3)
            avg, fin, bad = sweep.evaluate(prepared, "all", sf_params=sfp, orca_params=op)
            assert r_avg["N"] == avg["N"] == len(scenes)
            for k in ("orcainterp", "sfinterp", "kf"):
                for r, g in ((r_avg[k], avg[k]), (r_fin[k], fin[k])):
                    assert (np.isnan(r) and np.isnan(g)) or g == pytest.approx(r, rel=1e-12, abs=0), (k, sfp, op, r, g)
                assert (bad[k] > 0) == bool(np.isnan(r_avg[k]))
    finally:
        mp.undo()


@pytest.mark.gpu
def test_nan_scene_in_table_and_fit():
    from trajnetplusplusbaselines_b200.classical import orca, socialforce
    state, spd, offs, truth = _ragged([4, 3, 6], seed=2, nan_primary=True)
    prepared = common.to_device(state, spd, offs, truth)
    ade, fde = socialforce.sweep(prepared, SF_GRID[:3])
    ade, fde = ade.cpu().numpy(), fde.cpu().numpy()
    assert np.isnan(ade[:, 1]).all() and np.isnan(fde[:, 1]).all() and np.isfinite(ade[:, [0, 2]]).all()
    avg, fin, bad = sweep.evaluate(prepared, "sf", sf_params=SF_GRID[0])
    assert np.isnan(avg["sfinterp"]) and np.isnan(fin["sfinterp"]) and bad["sfinterp"] == 1
    r = sweep.fit([ade], [fde])["files"][0]
    assert list(r["skipped"]) == [1, 1, 1] and list(r["finite"]) == [2, 2, 2]
    assert r["best"] == int(np.argmin((ade[:, 0] + ade[:, 2]) / 2))
    oa, _ = orca.sweep(prepared, ORCA_GRID[:2])
    assert np.isfinite(oa.cpu().numpy()).all()                    # ORCA stops at the goal instead


@pytest.mark.gpu
def test_sweep_is_deterministic():
    from trajnetplusplusbaselines_b200.classical import orca, socialforce
    state, spd, offs, truth = _ragged([5, 9, 33, 2, 16] * 20, seed=6)
    prepared = common.to_device(state, spd, offs, truth)
    for sim, grid in ((socialforce, SF_GRID), (orca, ORCA_GRID)):
        a1, f1 = sim.sweep(prepared, grid)
        a2, f2 = sim.sweep(prepared, grid)
        assert a1.cpu().numpy().tobytes() == a2.cpu().numpy().tobytes()
        assert f1.cpu().numpy().tobytes() == f2.cpu().numpy().tobytes()


@pytest.mark.gpu
def test_c_abi_refuses_invalid_sweeps():
    """The C entry points refuse what the Python checks would have caught."""
    import ctypes
    import torch
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import _ptr, _stream
    lib = _lib.load()
    state, spd, offs, truth = _ragged([3, 4], seed=1)
    pr = common.to_device(state, spd, offs, truth)
    dev = pr.state.device
    ade = torch.empty((4, 2), dtype=torch.float64, device=dev)
    fde = torch.empty_like(ade)
    p = _lib.SfParams(0.05, 0.5, 2.1, 0.3, 96, 8)
    q = _lib.OrcaParams(0.05, 1.5, 10, 1.5, 0.4, 0.05, 97, 8)
    pos = pr.state[:, :2].float().contiguous()
    vel = pr.state[:, 2:4].float().contiguous()
    goal = pr.state[:, 4:].contiguous()

    def sf(prm, P=None, T=12):
        t = torch.tensor(prm, dtype=torch.float64, device=dev)
        return lib.tb2_sf_sweep(pr.layout.handle, ctypes.byref(p), _ptr(t), len(prm) if P is None else P,
                                _ptr(pr.state), _ptr(pr.truth), T, _ptr(ade), _ptr(fde), _stream(dev))

    def oc(prm, P=None, T=12):
        t = torch.tensor(prm, dtype=torch.float32, device=dev)
        return lib.tb2_orca_sweep(pr.layout.handle, ctypes.byref(q), _ptr(t), len(prm) if P is None else P, _ptr(pos),
                                  _ptr(vel), _ptr(goal), _ptr(pr.speeds), _ptr(pr.truth), T, _ptr(ade), _ptr(fde),
                                  _stream(dev))

    assert sf([[0.5, 2.1, 0.3]]) == 0 and oc([[1.5, 1.5, 0.4]]) == 0
    torch.cuda.synchronize()
    for rc in (sf([[0.5, 2.1, 0.3]], P=0), sf([[0.5, float("nan"), 0.3]]), sf([[0.0, 2.1, 0.3]]), sf([[0.5, 2.1, -0.3]]),
               sf([[0.5, 2.1, 0.3]], T=11), sf([[0.5, 2.1, 0.3]], P=2 ** 30),
               oc([[1.5, 1.5, 0.4]], P=0), oc([[float("inf"), 1.5, 0.4]]), oc([[1.5, 0.0, 0.4]]), oc([[1.5, 1.5, 0.0]]),
               oc([[1.5, 1.5, 0.4]], T=11)):
        assert rc == -1
        assert lib.tb2_last_error()
