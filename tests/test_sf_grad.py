"""Social-force parameter derivatives (tb2_sf_sweep_grad, socialforce.sweep_grad) and the gradient fit (classical.fit).

The derivatives are checked against the complex-step restatement tests/sf_cs_oracle.py, which is itself pinned to
central differences of oracle/classical_oracle.sf_simulate; the values against socialforce.sweep, bit for bit.
"""
import itertools
import json
import os
import types

import numpy as np
import pytest

import sf_cs_oracle as CS
from oracle import classical_oracle as O
from trajnetplusplusbaselines_b200.classical import common, fit, sweep

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sf_grad_golden.npz")
MAX_SCENE = 256                                   # tb2_sf_sweep_grad's largest scene (socialforce.MAX_GRAD_SCENE)
GRID = list(itertools.product((0.3, 0.5, 1.0), (1.0, 2.1, 5.0), (0.2, 0.3, 0.6)))
# Derivative tolerance: |cuda - complex step| <= RTOL * |d| + ATOL.  Both are float64 derivatives of the same rollout
# and differ by rounding only, amplified over 96 steps by the rollout's sensitivity: on an H100 the worst relative error
# over the fixture's scenes (up to 74 pedestrians, three settings) was 4.8e-11, so RTOL keeps a margin of 20.
RTOL, ATOL = 1e-9, 1e-11


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


def _counters(state, theta):
    c = {}
    O.sf_simulate(state, tau=theta[0], v0=theta[1], sigma=theta[2], counters=c)
    return c


def _no_switch(state, theta, h):
    """SF_COUNTERS equal at theta and theta +- h e_i for every parameter: no branch changes in between (as far as the
    counts show)."""
    c0 = _counters(state, theta)
    for i in range(3):
        for sgn in (-1, 1):
            t = list(theta)
            t[i] += sgn * h[i]
            if _counters(state, t) != c0:
                return False
    return True


def _close(got, want, rtol=RTOL, atol=ATOL):
    return np.abs(got - want) <= rtol * np.abs(want) + atol


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_complex_step_oracle_matches_central_differences():
    """The complex-step rollout's derivatives equal central differences of the real oracle (h = 1e-6 relative) on
    scenes whose branch counters do not change over the interval; its real part equals sf_simulate."""
    checked = 0
    for seed in range(6):
        state, _, offs, truth = _ragged([4], seed)
        theta = (0.5, 2.1, 0.3) if seed % 2 == 0 else (0.35, 3.0, 0.45)
        h = [1e-6 * v for v in theta]
        if not _no_switch(state, theta, h):
            continue
        ref = O.sf_simulate(state, tau=theta[0], v0=theta[1], sigma=theta[2])
        for i in range(3):
            cs = CS.sf_simulate_cs(state, *theta, which=i)
            assert np.allclose(cs.real, ref, rtol=1e-12, atol=1e-12)
            tp, tm = list(theta), list(theta)
            tp[i] += h[i]
            tm[i] -= h[i]
            fd = (O.sf_simulate(state, tau=tp[0], v0=tp[1], sigma=tp[2])
                  - O.sf_simulate(state, tau=tm[0], v0=tm[1], sigma=tm[2])) / (2 * h[i])
            d = cs.imag / CS.H
            assert np.allclose(d, fd, rtol=1e-5, atol=1e-7), (seed, i, np.abs(d - fd).max())
        checked += 1
    assert checked >= 3


def test_complex_step_exact_cases():
    """One pedestrian: v0 and sigma never enter; a destination equal to the position: NaN value and derivative."""
    state, _, _, truth = _ragged([1], 3)
    a, f, da, df = CS.score_grad(state, truth[0], 0.5, 2.1, 0.3)
    assert np.isfinite(a) and da[1] == 0.0 and da[2] == 0.0 and df[1] == 0.0 and df[2] == 0.0 and da[0] != 0.0
    state, _, _, truth = _ragged([3, 2], 3, nan_primary=True)
    a, f, da, df = CS.score_grad(state[3:], truth[1], 0.5, 2.1, 0.3)
    assert np.isnan(a) and np.isnan(da).all()


class _Quadratic:
    """Stand-in for the device: scene b of a file has ADE c_b + |theta - opt|^2_W, FDE twice that; scene `bad` of
    file 0 is NaN everywhere; `wall` makes every ADE NaN where tau > wall (a region the fit must back off from)."""
    opt = np.array([0.7, 1.6, 0.45])
    W = np.array([3.0, 0.5, 8.0])

    def __init__(self, consts, bad=None, wall=np.inf):
        self.consts, self.bad, self.wall, self.calls = consts, bad, wall, 0

    def _one(self, p, theta):
        theta = np.asarray(theta, dtype=np.float64)
        c = np.asarray(self.consts[p], dtype=np.float64)
        q = float((self.W * (theta - self.opt) ** 2).sum())
        g = 2 * self.W * (theta - self.opt)
        ade, dade = c + q, np.tile(g, (len(c), 1))
        if theta[0] > self.wall:
            ade = ade * np.nan
        if self.bad is not None and p == 0:
            ade[self.bad] = np.nan
            dade[self.bad] = np.nan
        return ade, 2 * ade, dade, 2 * dade

    def grads(self, p, theta):
        self.calls += 1
        return self._one(p, theta)

    def values(self, p, settings):
        out = [self._one(p, s) for s in settings]
        return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def test_fit_reaches_the_minimum_with_a_stub_provider():
    q = _Quadratic({0: [0.1, 0.2, 0.3], 1: [0.5]}, bad=1)
    grid = list(itertools.product((0.3, 1.2), (1.0, 3.0), (0.2, 0.9)))
    r = fit.fit([0, 1], grid, grads=q.grads, values=q.values, starts=2)
    for g in r["files"] + [r["pooled"]]:
        assert np.allclose(g["theta"], q.opt, atol=1e-5)
        assert g["ade"] <= g["start_ade"]
    assert r["files"][0]["used"] == 2 and r["files"][0]["skipped"] == 1               # the NaN scene stays out
    assert r["pooled"]["used"] == 3 and r["pooled"]["skipped"] == 1
    assert r["files"][1]["ade"] == pytest.approx(0.5, abs=1e-9)
    assert r["pooled"]["ade"] == pytest.approx((0.1 + 0.3 + 0.5) / 3, abs=1e-9)
    assert r["pooled"]["fde"] == pytest.approx(2 * (0.1 + 0.3 + 0.5) / 3, abs=1e-9)
    assert r["pooled"]["nfev"] >= 2 and r["pooled"]["nit"] >= 1
    fd = fit.fit([0, 1], grid, objective="fde", grads=q.grads, values=q.values)
    assert np.allclose(fd["pooled"]["theta"], q.opt, atol=1e-5)


def test_fit_respects_bounds_and_backs_off_non_finite_iterates():
    q = _Quadratic({0: [0.1, 0.2]})
    q.opt = np.array([-0.5, -1.0, -0.2])                                                 # minimum outside the bounds
    th, value, _ = fit.minimize(fit.Objective([0], (0.5, 2.0, 0.3), grads=q.grads), (0.5, 2.0, 0.3))
    assert np.allclose(th, fit.LOWER, atol=1e-8) and (th >= np.array(fit.LOWER)).all()
    wall = _Quadratic({0: [0.1, 0.2]}, wall=0.6)                                          # opt tau 0.7 lies past the wall
    obj = fit.Objective([0], (0.3, 2.0, 0.3), grads=wall.grads)
    assert obj((0.65, 1.6, 0.45)) == (np.inf, pytest.approx(np.zeros(3)))
    th, value, _ = fit.minimize(obj, (0.3, 2.0, 0.3))
    assert np.isfinite(value) and th[0] <= 0.6 and value < obj.best[0] + 1e-15
    assert value < wall._one(0, (0.3, 2.0, 0.3))[0].mean()


def test_fit_holds_the_scene_set_fixed():
    """A scene that is non-finite at the start stays out even where it turns finite; one counted at the start that
    turns non-finite makes the objective +inf."""
    class Flip(_Quadratic):
        def _one(self, p, theta):
            ade, fde, dade, dfde = super()._one(p, theta)
            if theta[1] < 1.5:
                ade[0] = np.nan                                                          # scene 0 lost below v0 1.5
            else:
                ade[1] = np.nan                                                          # scene 1 only finite below
            return ade, fde, dade, dfde
    q = Flip({0: [0.1, 0.2, 0.3]})
    obj = fit.Objective([0], (0.5, 1.0, 0.3), grads=q.grads)
    assert obj.used == 2 and list(obj.masks[0]) == [False, True, True]
    assert obj((0.5, 1.2, 0.3))[0] == pytest.approx(0.25 + float((q.W * (np.array([0.5, 1.2, 0.3]) - q.opt) ** 2).sum()))
    assert obj((0.5, 2.0, 0.3))[0] == np.inf


def test_cli_arguments():
    a = fit.parse_args(["x.ndjson", "y.ndjson", "--tau", "0.3", "0.5", "--vo", "2", "--sigma", "0.2", "0.3", "0.4",
                        "--starts", "3", "--objective", "fde", "--max_iter", "7"])
    assert a.files == ["x.ndjson", "y.ndjson"] and a.tau == [0.3, 0.5] and a.vo == [2.0] and a.sigma == [0.2, 0.3, 0.4]
    assert a.starts == 3 and a.objective == "fde" and a.max_iter == 7
    d = fit.parse_args(["x.ndjson"])
    assert (d.tau, d.vo, d.sigma) == ([0.5], [2.1], [0.3]) and d.starts == 1 and d.objective == "ade"
    for bad in (["x.ndjson", "--objective", "mse"], ["x.ndjson", "--starts", "0"], []):
        with pytest.raises(SystemExit):
            fit.parse_args(bad)
    with pytest.raises(ValueError):
        fit.Objective([0], (0.5, 2.1, 0.3), objective="mse", grads=_Quadratic({0: [0.1]}).grads)


def test_sweep_grad_argument_validation():
    from trajnetplusplusbaselines_b200.classical import socialforce
    fake = types.SimpleNamespace(truth=np.zeros((3, 12, 2)))
    for bad in ([], [[0.5, 2.1]], [[0.0, 2.1, 0.3]], [[0.5, 2.1, -1.0]], [[np.nan, 2.1, 0.3]], [[0.5, np.inf, 0.3]]):
        with pytest.raises(ValueError):
            socialforce.sweep_grad(fake, bad)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _golden():
    g = np.load(GOLDEN)
    return {k: g[k] for k in g.files}


def _grad(prepared, grid):
    from trajnetplusplusbaselines_b200.classical import socialforce
    return tuple(t.cpu().numpy() for t in socialforce.sweep_grad(prepared, grid))


def _value(prepared, grid):
    from trajnetplusplusbaselines_b200.classical import socialforce
    return tuple(t.cpu().numpy() for t in socialforce.sweep(prepared, grid))


def _same(a, b):
    return np.array_equal(a, b, equal_nan=True)


@pytest.mark.gpu
def test_values_equal_sweep_bit_for_bit():
    """Packed widths 1 .. 32 and CTA scenes up to the cap, 27 settings, P = 1; the fixture's real scenes."""
    sizes = [1, 2, 3, 5, 8, 9, 16, 17, 31, 32, 33, 40, 64, 100, 200, MAX_SCENE, 4, 12]
    state, spd, offs, truth = _ragged(sizes, seed=4)
    pr = common.to_device(state, spd, offs, truth)
    for grid in (GRID, [sweep.SF_DEFAULT]):
        ade, fde, dade, dfde = _grad(pr, grid)
        va, vf = _value(pr, grid)
        assert _same(ade, va) and _same(fde, vf)
        assert dade.shape == dfde.shape == (len(grid), len(sizes), 3)
        assert np.isfinite(dade).all() and np.isfinite(dfde).all()
    g = _golden()
    pr = common.to_device(g["state"], np.zeros(len(g["state"])), g["offsets"], g["truth"])
    ade, fde, _, _ = _grad(pr, GRID)
    va, vf = _value(pr, GRID)
    assert _same(ade, va) and _same(fde, vf)


@pytest.mark.gpu
def test_derivatives_match_complex_step():
    g = _golden()
    pr = common.to_device(g["state"], np.zeros(len(g["state"])), g["offsets"], g["truth"])
    ade, fde, dade, dfde = _grad(pr, g["settings"])
    fin = np.isfinite(g["ade"])
    assert (np.isfinite(ade) == fin).all()
    assert np.allclose(ade[fin], g["ade"][fin], rtol=1e-12, atol=0)
    worst = 0.0
    for got, want in ((dade, g["dade"]), (dfde, g["dfde"])):
        ok = _close(got[fin], want[fin])
        worst = max(worst, float((np.abs(got[fin] - want[fin]) / (np.abs(want[fin]) + ATOL / RTOL)).max()))
        assert ok.all(), (np.argwhere(~ok), worst)
        assert not np.isfinite(got[~fin]).any()
    print("golden: worst relative derivative error %.2e" % worst)
    # fresh complex-step runs on synthetic scenes of both forms
    sizes = [2, 3, 6, 11, 33]
    state, spd, offs, truth = _ragged(sizes, seed=12)
    pr = common.to_device(state, spd, offs, truth)
    settings = [(0.5, 2.1, 0.3), (0.8, 1.2, 0.5)]
    _, _, dade, dfde = _grad(pr, settings)
    worst = 0.0
    for s, th in enumerate(settings):
        for b in range(len(sizes)):
            _, _, da, df = CS.score_grad(state[offs[b]:offs[b + 1]], truth[b], *th)
            assert _close(dade[s, b], da).all() and _close(dfde[s, b], df).all(), (s, b, dade[s, b], da)
            for got, want in ((dade[s, b], da), (dfde[s, b], df)):
                worst = max(worst, float((np.abs(got - want) / (np.abs(want) + ATOL / RTOL)).max()))
    print("synthetic: worst relative derivative error %.2e" % worst)


@pytest.mark.gpu
def test_exact_cases():
    state, spd, offs, truth = _ragged([1, 1, 4, 3], seed=7, nan_primary=True)
    pr = common.to_device(state, spd, offs, truth)
    ade, fde, dade, dfde = _grad(pr, GRID)
    assert (dade[:, 0, 1:] == 0).all() and (dfde[:, 0, 1:] == 0).all() and (dade[:, 0, 0] != 0).any()
    va, _ = _value(pr, GRID)
    bad = ~np.isfinite(va)
    assert bad[:, 1].all() and not bad[:, [0, 2, 3]].any()
    assert (~np.isfinite(ade) == bad).all() and (~np.isfinite(fde) == bad).all()
    assert (~np.isfinite(dade).all(axis=2) == bad).all() and (~np.isfinite(dfde).all(axis=2) == bad).all()


@pytest.mark.gpu
def test_tangents_match_central_differences_of_the_value_kernel():
    """theta and theta +- h e_i (h = 1e-6 relative) in one tb2_sf_sweep launch of P = 7, on scenes whose oracle
    counters show no branch switch in the interval."""
    sizes = [2, 3, 4, 5, 6, 8, 34]
    state, spd, offs, truth = _ragged(sizes, seed=21)
    pr = common.to_device(state, spd, offs, truth)
    used = 0
    for theta in ((0.5, 2.1, 0.3), (0.4, 1.5, 0.5)):
        h = [1e-6 * v for v in theta]
        grid = [theta]
        for i in range(3):
            for sgn in (1, -1):
                t = list(theta)
                t[i] += sgn * h[i]
                grid.append(tuple(t))
        va, vf = _value(pr, grid)
        _, _, dade, dfde = _grad(pr, [theta])
        for b in range(len(sizes)):
            if not _no_switch(state[offs[b]:offs[b + 1]], theta, h):
                continue
            used += 1
            for i in range(3):
                fa = (va[1 + 2 * i, b] - va[2 + 2 * i, b]) / (2 * h[i])
                ff = (vf[1 + 2 * i, b] - vf[2 + 2 * i, b]) / (2 * h[i])
                assert abs(fa - dade[0, b, i]) <= 1e-5 * abs(dade[0, b, i]) + 1e-7, (b, i, fa, dade[0, b, i])
                assert abs(ff - dfde[0, b, i]) <= 1e-5 * abs(dfde[0, b, i]) + 1e-7, (b, i, ff, dfde[0, b, i])
    assert used >= 4


@pytest.mark.gpu
def test_reruns_are_bit_identical_and_large_scenes_are_refused():
    state, spd, offs, truth = _ragged([5, 9, 33, 2, 16, 70] * 10, seed=6)
    pr = common.to_device(state, spd, offs, truth)
    a = _grad(pr, GRID)
    b = _grad(pr, GRID)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    state, spd, offs, truth = _ragged([3, MAX_SCENE + 1], seed=1)
    pr = common.to_device(state, spd, offs, truth)
    from trajnetplusplusbaselines_b200 import _lib
    launches = int(_lib.load().tb2_launch_count())
    with pytest.raises(RuntimeError, match="larger than %d pedestrians" % MAX_SCENE):
        _grad(pr, GRID)
    assert int(_lib.load().tb2_launch_count()) == launches
    assert np.isfinite(_value(pr, GRID)[0]).all()                    # the value sweep keeps its 1024


def _simulated_truth(state, offs, theta, noise, seed):
    from trajnetplusplusbaselines_b200.classical import socialforce
    pos = socialforce.simulate_batch(state, offs, theta, n_steps=96, sample_every=8).cpu().numpy()
    rng = np.random.RandomState(seed)
    return np.stack([pos[:, offs[b]] for b in range(len(offs) - 1)]) + rng.randn(len(offs) - 1, 12, 2) * noise


@pytest.mark.gpu
def test_fit_recovers_a_known_setting():
    """Truth = a tb2_sf_simulate rollout at theta* plus 1 cm noise; the grid leaves theta* out.  On an H100 the fit
    landed within 0.6 % of theta* in every parameter (0.6235, 1.6953, 0.4087); 2 % is asserted."""
    theta_star = (0.62, 1.7, 0.41)
    sizes = [3, 4, 5, 6, 8, 10, 12, 7, 5, 9] * 4
    state, spd, offs, _ = _ragged(sizes, seed=31)
    truth = _simulated_truth(state, offs, theta_star, 0.01, seed=32)
    pr = common.to_device(state, spd, offs, truth)
    grid = list(itertools.product((0.3, 1.0), (1.0, 3.0), (0.2, 0.7)))
    r = fit.fit([pr], grid, starts=2, max_iter=200)["pooled"]
    star = fit.masked_mean(_value(pr, [theta_star])[0][0], np.ones(len(sizes), dtype=bool))
    best_cell = np.nanmin(sweep.fit([_value(pr, grid)[0]])["pooled"]["ade"])
    print("fit %s (theta* %s): ADE %.6f, at theta* %.6f, grid best %.6f, %d iterations, %d evaluations"
          % (np.round(r["theta"], 4), theta_star, r["ade"], star, best_cell, r["nit"], r["nfev"]))
    assert r["ade"] <= star and r["ade"] <= best_cell
    assert np.allclose(r["theta"], theta_star, rtol=0.02, atol=0), r["theta"]


def _write_ndjson(path, xy, xy_offsets):
    lines, ped = [], 0
    for s in range(len(xy_offsets) - 1):
        x = xy[:, xy_offsets[s]:xy_offsets[s + 1]]
        f0 = 10000 * s
        lines.append(json.dumps({"scene": {"id": s, "p": ped, "s": f0, "e": f0 + 10 * (len(x) - 1), "fps": 2.5,
                                           "tag": 1}}))
        for t in range(len(x)):
            for j in range(x.shape[1]):
                if not np.isnan(x[t, j, 0]):
                    lines.append(json.dumps({"track": {"f": f0 + 10 * t, "p": ped + j, "x": float(x[t, j, 0]),
                                                       "y": float(x[t, j, 1])}}))
        ped += x.shape[1]
    path.write_text("\n".join(lines) + "\n")


@pytest.mark.gpu
def test_cli_on_fixture_scenes(tmp_path, capsys):
    g = _golden()
    xo = g["xy_offsets"]
    half = (len(xo) - 1) // 2
    files = [tmp_path / "a.ndjson", tmp_path / "b.ndjson"]
    _write_ndjson(files[0], g["xy"][:, :xo[half]], xo[:half + 1])
    _write_ndjson(files[1], g["xy"][:, xo[half]:], xo[half:] - xo[half])
    prepared = [sweep.prepare_file(str(f)) for f in files]
    assert np.allclose(np.concatenate([p.state.cpu().numpy() for p in prepared]), g["state"], rtol=0, atol=1e-9)
    r = fit.main([str(f) for f in files] + ["--tau", "0.3", "1.0", "--vo", "1.0", "3.0", "--sigma", "0.2", "0.6",
                                            "--max_iter", "15"])
    out = capsys.readouterr().out
    assert "pooled" in out and "Average L2" in out and "Final L2" in out
    grid_r = r["grid"]
    for fr, gr in list(zip(r["files"], grid_r["files"])) + [(r["pooled"], grid_r["pooled"])]:
        assert fr["start_ade"] == gr["ade"][gr["best"]]
        assert fr["ade"] <= gr["ade"][gr["best"]]
