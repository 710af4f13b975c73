"""Scoring of prediction files (trajnetplusplusbaselines_b200/scoring.py, csrc/metrics.cu tb2_score_scenes,
csrc/ndjson.cu tb2_ndjson_parse_meta) against tests/golden/scoring_golden.npz (oracle/make_scoring_golden.py): the
reference's eval_utils / TrajnetEvaluator.aggregate and scipy.stats.gaussian_kde."""
import glob
import io
import os
import types
from contextlib import redirect_stdout

import numpy as np
import pytest

from oracle import metrics_oracle as MO
from trajnetplusplusbaselines_b200 import scoring
from trajnetplusplusbaselines_b200.data import TrackRow

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "scoring_golden.npz"))
SYN = ("modes1", "modes3", "modes50")
AGG = sorted({k.split("/")[1] for k in GOLD.files if k.startswith("agg/")})
T = 12


def _syn(case):
    keys = ("gt_primary", "pred_primary", "num_modes", "gt_neigh_off", "gt_neigh", "gt_neigh_mask", "pred_neigh_off",
            "pred_neigh", "pred_neigh_mask")
    return {k: GOLD["syn/%s/%s" % (case, k)] for k in keys}


def _text(key):
    return GOLD[key].tobytes().decode()


def _write(path, text):
    with open(path, "w") as f:
        f.write(text)
    return str(path)


def _rows(xy, frames, mode=None):
    return [TrackRow(int(f), 1, float(x), float(y), mode, 0) for f, (x, y) in zip(frames, xy)]


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the oracle (CPU side of scripts/score_bench.py) against the golden values; the metadata parser
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", SYN)
def test_oracle_matches_golden(case):
    d = _syn(case)
    S, K = d["pred_primary"].shape[:2]
    frames = np.arange(T) * 10
    for s in range(S):
        gt = _rows(d["gt_primary"][s], frames)
        modes = [_rows(d["pred_primary"][s, m], frames, m) for m in range(K)]
        ade = [MO.average_l2(gt, m) for m in modes]
        fde = [MO.final_l2(gt, m) for m in modes]
        np.testing.assert_allclose(ade, GOLD["syn/%s/expect_ade" % case][s], rtol=0, atol=1e-12)
        np.testing.assert_allclose(fde, GOLD["syn/%s/expect_fde" % case][s], rtol=0, atol=1e-12)
        for kind, want in (("gt", "expect_col_gt"), ("pred", "expect_col_pred")):
            off = d[kind + "_neigh_off"]
            hit = any(MO.collision(modes[0], [r for r, keep in zip(_rows(d[kind + "_neigh"][j], frames), d[kind + "_neigh_mask"][j])
                                              if keep])
                      for j in range(off[s], off[s + 1]))
            assert int(hit) == GOLD["syn/%s/%s" % (case, want)][s], (case, s, kind)
        ta, tf = MO.topk([r for m in modes for r in m], gt)
        assert ta == GOLD["syn/%s/expect_topk_ade" % case][s] or np.isclose(ta, GOLD["syn/%s/expect_topk_ade" % case][s], atol=1e-12)
        assert np.isclose(tf, GOLD["syn/%s/expect_topk_fde" % case][s], atol=1e-12)
        want = GOLD["syn/%s/expect_nll" % case][s]
        if np.isnan(want):
            with pytest.raises(Exception, match="All Predictions are Identical"):
                MO.nll([r for m in modes for r in m], gt)
        else:
            assert np.isclose(MO.nll([r for m in modes for r in m], gt), want, rtol=0, atol=1e-9)


def test_oracle_kde_matches_scipy_golden():
    for i, (n, pts, q) in enumerate(zip(GOLD["kde/count"], GOLD["kde/samples"], GOLD["kde/point"])):
        got = MO.kde_logpdf(pts[:n], q)
        want = GOLD["kde/logpdf"][i]
        assert (got is None) == bool(np.isnan(want)), i
        if got is not None:
            assert np.isclose(got, want, rtol=1e-12, atol=1e-12), (i, got, want)


def _assert_meta_agrees(path):
    native = scoring.parse_ndjson_meta(path)
    python = scoring.parse_ndjson_meta(path, native=False)
    assert sorted(native) == sorted(python)
    for k in native:
        assert native[k].dtype == python[k].dtype and native[k].shape == python[k].shape, k
        assert np.array_equal(native[k], python[k], equal_nan=True), k
    return native


def test_meta_parser_matches_json_loads_on_golden_files(tmp_path):
    for key in [k for k in GOLD.files if k.startswith("agg/") and k.endswith(("/gt", "/pred"))] + \
            ["collision_test/test", "collision_test/test_private"]:
        cols = _assert_meta_agrees(_write(tmp_path / "f.ndjson", _text(key)))
        if key.endswith("/gt"):
            assert (cols["scene_tag"] >= 1).all() and (cols["track_scene_id"] == -1).all()
        if key.endswith("/pred"):
            assert (cols["prediction_number"] >= 0).all() and (cols["scene_tag"] == 0).all()


@pytest.mark.needs_reference
def test_meta_parser_matches_json_loads_on_the_data_block():
    from oracle.ref_shim import reference_root
    files = sorted(glob.glob(os.path.join(reference_root(), "DATA_BLOCK", "**", "*.ndjson"), recursive=True))
    assert files
    scenes = 0
    for fn in files:
        cols = _assert_meta_agrees(fn)
        scenes += len(cols["scene_id"]) if "/train/" in fn else 0
    assert scenes == 13718


def test_meta_parser_on_written_predictions(tmp_path):
    """Files write_predictions_xy produces (the native writer), incl. NaN neighbours and several modes."""
    from trajnetplusplusbaselines_b200.data import SceneMeta, write_predictions_xy
    rng = np.random.RandomState(0)
    metas = [SceneMeta(i, 10 + i, 100 * i, 10, 100 * i + 80, [50 + i, 60 + i]) for i in range(6)]
    preds = []
    for _ in metas:
        neigh = rng.randn(T, 2, 2)
        neigh[7:, 1] = np.nan
        preds.append({m: [rng.randn(T, 2), neigh if m == 0 else []] for m in range(3)})
    fn = str(tmp_path / "p.ndjson")
    write_predictions_xy(preds, metas, fn)
    cols = _assert_meta_agrees(fn)
    assert sorted(set(cols["prediction_number"].tolist())) == [0, 1, 2]
    assert sorted(set(cols["track_scene_id"].tolist())) == list(range(6))


def test_meta_parser_refuses_unusual_metadata(tmp_path):
    """Metadata outside the plain format sends the file to json.loads; the plain parser keeps skipping the tag."""
    from trajnetplusplusbaselines_b200 import data
    base = ['{"scene": {"id": 0, "p": 1, "s": 0, "e": 20, "fps": 2.5, "tag": [3, [1, 2]]}}',
            '{"track": {"f": 0, "p": 1, "x": 0.5, "y": 1.0, "prediction_number": 2, "scene_id": 0}}']
    for odd in ('{"scene": {"id": 1, "p": 1, "s": 0, "e": 20, "tag": [3, [2], {"k": "v"}]}}',
                '{"scene": {"id": 1, "p": 1, "s": 0, "e": 20, "tag": [3, [2.5]]}}',
                '{"scene": {"id": 1, "p": 1, "s": 0, "e": 20, "tag": [3, [63]]}}',
                '{"scene": {"id": 1, "p": 1, "s": 0, "e": 20, "tag": null}}',
                '{"track": {"f": 0, "p": 1, "x": 0.5, "y": 1.0, "prediction_number": null}}',
                '{"track": {"f": 0, "p": 1, "x": 0.5, "y": 1.0, "scene_id": 1.0}}',
                '{"track": {"f": 0, "p": 1, "x": 0.5, "y": 1.0, "scene_id": -3}}'):
        text = "\n".join(base + [odd]) + "\n"
        assert scoring._parse_meta_native(text.encode()) is None, odd
        assert data.parse_ndjson_columns(_write(tmp_path / "odd.ndjson", text)) is not None, odd
    cols = scoring.parse_ndjson_meta(_write(tmp_path / "ok.ndjson", "\n".join(base) + "\n"))
    assert cols["scene_tag"].tolist() == [3] and cols["scene_subs"].tolist() == [0b110]
    assert cols["prediction_number"].tolist() == [2] and cols["track_scene_id"].tolist() == [0]
    _assert_meta_agrees(tmp_path / "ok.ndjson")
    cols = scoring.parse_ndjson_meta(_write(tmp_path / "plain.ndjson", '{"scene": {"id": 4, "p": 1, "s": 0, "e": 20, "tag": 2}}\n'
                                                                     '{"track": {"f": 0, "p": 1, "x": 0.5, "y": 1.0}}\n'))
    assert cols["scene_tag"].tolist() == [2] and cols["scene_subs"].tolist() == [0]
    assert cols["prediction_number"].tolist() == [-1] and cols["track_scene_id"].tolist() == [-1]
    _assert_meta_agrees(tmp_path / "plain.ndjson")


def test_assembly_checks_frames_and_counts_predictions(tmp_path):
    case = "zara_modes3"
    gt = _write(tmp_path / "gt.ndjson", _text("agg/%s/gt" % case))
    a = scoring.assemble(gt, _write(tmp_path / "pred.ndjson", _text("agg/%s/pred" % case)))
    assert a["num_predictions"] == 2 and a["pred_primary"].shape == (60, 3, T, 2) and (a["num_modes"] == 3).all()
    assert not np.isnan(a["pred_primary"]).any() and (a["tag"] >= 1).all()
    assert (np.diff(a["gt_neigh_off"]) == np.diff(a["pred_neigh_off"])).all()
    lines = _text("agg/%s/pred" % case).splitlines()
    k = next(i for i, line in enumerate(lines) if '"prediction_number": 0' in line)
    lines[k] = lines[k].replace('"f": ', '"f": 1')                      # mode 0 of the first scene off its frames
    with pytest.raises(Exception, match="frame numbers are not consistent"):
        scoring.assemble(gt, _write(tmp_path / "bad.ndjson", "\n".join(lines) + "\n"))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: tb2_score_scenes records, score_file, the evaluator CLI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", SYN)
def test_device_records_match_golden(case):
    from trajnetplusplusbaselines_b200 import _lib
    d = _syn(case)
    rec = scoring.score_arrays(d, with_nll=True)
    g = lambda k: GOLD["syn/%s/expect_%s" % (case, k)]
    for k in ("ade", "fde"):
        assert np.array_equal(np.isnan(rec[k]), np.isnan(g(k))), k
        np.testing.assert_allclose(rec[k], g(k), rtol=0, atol=1e-6, equal_nan=True)
    assert np.array_equal((rec["flags"] & _lib.SCORE_COL_GT) != 0, g("col_gt") == 1)
    assert np.array_equal((rec["flags"] & _lib.SCORE_COL_PRED) != 0, g("col_pred") == 1)
    counts = lambda off: np.diff(d[off])
    assert np.array_equal((rec["flags"] & _lib.SCORE_NEIGH_COUNT_DIFFERS) != 0, counts("gt_neigh_off") != counts("pred_neigh_off"))
    skipped = (rec["flags"] & _lib.SCORE_NLL_ALL_SKIPPED) != 0
    assert np.array_equal(skipped, np.isnan(g("nll")))
    np.testing.assert_allclose(rec["nll"][~skipped], g("nll")[~skipped], rtol=0, atol=1e-6)
    np.testing.assert_allclose([scoring._topk(r) for r in rec["ade"]], g("topk_ade"), rtol=0, atol=1e-6)
    np.testing.assert_allclose([scoring._topk(r) for r in rec["fde"]], g("topk_fde"), rtol=0, atol=1e-6)
    again = scoring.score_arrays(d, with_nll=True)
    for k in rec:
        assert np.array_equal(rec[k].view(np.uint8), again[k].view(np.uint8)), k          # bit-identical


@pytest.mark.gpu
@pytest.mark.parametrize("horizon", [16, 20, 40])
def test_device_records_long_horizons_match_oracle(horizon):
    """pred_length above 15 with NLL: more timesteps than warps per CTA.  Also a NaN ground-truth point, whose timestep
    the NLL skips (scipy's density is NaN there)."""
    from trajnetplusplusbaselines_b200 import _lib
    rng = np.random.RandomState(horizon)
    S, K = 6, 50
    gt = np.round(np.cumsum(rng.randn(S, horizon, 2) * 0.3, axis=1), 2)
    modes = np.round(gt[:, None] + rng.randn(S, K, horizon, 2) * rng.uniform(0.05, 0.5, (S, 1, 1, 1)), 2)
    gt[1, 3] = np.nan
    nb = np.round(modes[:, 0, None] + rng.randn(S, 3, 1, 2) * 0.3, 2).reshape(-1, horizon, 2)
    mask = (rng.rand(S * 3, horizon) < 0.8).astype(np.uint8)
    nb[mask == 0] = np.nan
    off = np.arange(S + 1, dtype=np.int32) * 3
    d = dict(gt_primary=gt, pred_primary=modes, num_modes=np.full(S, K, np.int32), gt_neigh_off=off, gt_neigh=nb,
             gt_neigh_mask=mask, pred_neigh_off=off, pred_neigh=nb[::-1].copy(), pred_neigh_mask=mask[::-1].copy())
    rec = scoring.score_arrays(d, with_nll=True)
    frames = np.arange(horizon) * 10
    for s in range(S):
        g = _rows(gt[s], frames)
        rows = [_rows(modes[s, m], frames, m) for m in range(K)]
        np.testing.assert_allclose(rec["ade"][s], [MO.average_l2(g, r, n_predictions=horizon) for r in rows], rtol=0,
                                   atol=1e-6, equal_nan=True)
        np.testing.assert_allclose(rec["fde"][s], [MO.final_l2(g, r) for r in rows], rtol=0, atol=1e-6)
        for kind, bit in (("gt", _lib.SCORE_COL_GT), ("pred", _lib.SCORE_COL_PRED)):
            want = any(MO.collision(rows[0], [r for r, keep in zip(_rows(d[kind + "_neigh"][j], frames), d[kind + "_neigh_mask"][j])
                                              if keep], n_predictions=horizon) for j in range(off[s], off[s + 1]))
            assert bool(rec["flags"][s] & bit) == want, (s, kind)
        assert not rec["flags"][s] & _lib.SCORE_NLL_ALL_SKIPPED
        assert np.isclose(rec["nll"][s], MO.nll([r for m in rows for r in m], g, n_predictions=horizon), rtol=0, atol=1e-6)


@pytest.mark.gpu
def test_device_kde_matches_scipy():
    from trajnetplusplusbaselines_b200 import _lib
    n, pts, q, want = GOLD["kde/count"], GOLD["kde/samples"], GOLD["kde/point"], GOLD["kde/logpdf"]
    S, K = pts.shape[:2]
    d = dict(gt_primary=q[:, None], pred_primary=np.nan_to_num(pts)[:, :, None], num_modes=n,
             gt_neigh_off=np.zeros(S + 1, np.int32), gt_neigh=np.empty((0, 1, 2)), gt_neigh_mask=np.empty((0, 1), np.uint8),
             pred_neigh_off=np.zeros(S + 1, np.int32), pred_neigh=np.empty((0, 1, 2)), pred_neigh_mask=np.empty((0, 1), np.uint8))
    rec = scoring.score_arrays(d, with_nll=True)
    skipped = (rec["flags"] & _lib.SCORE_NLL_ALL_SKIPPED) != 0
    assert np.array_equal(skipped, np.isnan(want))
    np.testing.assert_allclose(rec["nll"][~skipped], -np.maximum(want[~skipped], -20.0), rtol=0, atol=1e-6)


def _table(result):
    metrics, categories, sub_categories = result
    rows = [metrics] + [getattr(categories, n) for n in scoring.CATEGORY_FIELDS]
    rows += [getattr(sub_categories, n) for n in scoring.SUB_CATEGORY_FIELDS]
    return np.array([[float(getattr(m, f)) for f in ("N", "average_l2", "final_l2", "gt_col", "pred_col", "topk_ade", "topk_fde",
                                                      "nll")] for m in rows])


@pytest.mark.gpu
@pytest.mark.parametrize("case", AGG)
def test_score_file_matches_reference_aggregate(case, tmp_path):
    gt = _write(tmp_path / "gt.ndjson", _text("agg/%s/gt" % case))
    pred = _write(tmp_path / "pred.ndjson", _text("agg/%s/pred" % case))
    got = _table(scoring.score_file(gt, pred, disable_collision=bool(GOLD["agg/%s/disable_collision" % case])))
    want = GOLD["agg/%s/result" % case]
    np.testing.assert_array_equal(got[:, [0, 3, 4]], want[:, [0, 3, 4]])          # N, Col-II, Col-I: counts
    np.testing.assert_allclose(got, want, rtol=1e-9, atol=1e-6)
    again = _table(scoring.score_file(gt, pred, disable_collision=bool(GOLD["agg/%s/disable_collision" % case])))
    assert np.array_equal(got, again)
    if "mismatch" in case:
        assert got[0, 4] == -1


class _ConstantVelocity:
    """Constant-velocity predictor with the reference's call signature."""

    def __call__(self, paths, scene_goal, n_predict=12, modes=1, predict_all=True, obs_length=9, start_length=0, args=None):
        from trajnetplusplusbaselines_b200.data import paths_to_xy
        xy = paths_to_xy(paths)
        v = xy[obs_length - 1] - xy[obs_length - 2]
        pred = xy[obs_length - 1][None] + np.arange(1, n_predict + 1)[:, None, None] * v[None]
        return {0: [pred[:, 0], pred[:, 1:]]}


def _dataset(root, name="demo", collision=True):
    """DATA_BLOCK/<name>/{test,test_private}: two DATA_BLOCK-derived files (the ground truth serves as the test input: the
    writer keeps only the observation) and the head-on collision test."""
    for part in ("test", "test_private"):
        os.makedirs(os.path.join(root, "DATA_BLOCK", name, part))
        for case in ("zara_modes3", "hotel_modes1"):
            _write(os.path.join(root, "DATA_BLOCK", name, part, case.split("_")[0] + ".ndjson"), _text("agg/%s/gt" % case))
        if collision:
            _write(os.path.join(root, "DATA_BLOCK", name, part, "collision_test.ndjson"), _text("collision_test/" + part))
    return os.path.join(root, "DATA_BLOCK", name)


def _args(root, modes=1, name="demo"):
    return types.SimpleNamespace(path=os.path.join(root, "DATA_BLOCK", name, "test_pred") + os.sep, output=["m/cv.pkl"],
                                 modes=modes, obs_length=9, pred_length=12, chunk=64, normalize_scene=False, labels=None,
                                 disable_collision=False)


@pytest.mark.gpu
def test_cli_evaluate_end_to_end(tmp_path, monkeypatch):
    """--evaluate writes the same prediction files as the plain tool, then prints the table; the collision test fails
    for a predictor that walks the head-on pair into each other."""
    import torch
    from trajnetplusplusbaselines_b200 import evaluator
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor
    torch.manual_seed(0)
    LSTMPredictor(LSTM()).save({"epoch": 0}, str(tmp_path / "vanilla.pkl"))
    for name in ("plain", "scored"):
        _dataset(str(tmp_path), name)
    monkeypatch.chdir(tmp_path)
    evaluator.main(["--path", "plain", "--output", "vanilla.pkl"])
    buf = io.StringIO()
    with redirect_stdout(buf):
        evaluator.main(["--path", "scored", "--output", "vanilla.pkl", "--evaluate"])
    text = buf.getvalue()
    out = {n: os.path.join("DATA_BLOCK", n, "test_pred", "vanilla_modes1") for n in ("plain", "scored")}
    assert sorted(os.listdir(out["plain"])) == sorted(os.listdir(out["scored"])) == ["collision_test.ndjson", "hotel.ndjson",
                                                                                     "zara.ndjson"]
    for f in os.listdir(out["plain"]):
        assert open(os.path.join(out["plain"], f), "rb").read() == open(os.path.join(out["scored"], f), "rb").read()
    for word in ("ADE", "FDE", "Col I", "Col II", "hotel", "zara", "Overall", "Type IV", "Col_test"):
        assert word in text, word

    args = _args(str(tmp_path), name="scored")
    evaluator.get_predictions(args, load_predictor=lambda fn: _ConstantVelocity())
    lines = []
    results = scoring.trajnet_evaluate(args, out=lines.append)
    assert "Col_test: Fail" in lines[0]
    overall = scoring.summarize(results["cv_modes1"])["overall"]
    assert overall.N == 100 and 0 < overall.average_l2 / overall.N < 5


@pytest.mark.gpu
def test_sgan_fifty_modes_get_predictions_then_evaluate(tmp_path):
    """S-GAN with 50 modes: get_predictions writes 50 primary modes per scene, trajnet_evaluate scores Top-3 and NLL."""
    import torch
    from trajnetplusplusbaselines_b200.evaluator import get_predictions
    from trajnetplusplusbaselines_b200.sgan import SGAN, LSTMGenerator, SGANPredictor
    torch.manual_seed(0)
    model = SGAN(generator=LSTMGenerator(), k=50, d_steps=0).to("cuda").eval()
    _dataset(str(tmp_path), collision=False)
    args = _args(str(tmp_path), modes=50)
    get_predictions(args, load_predictor=lambda fn: SGANPredictor(model))
    lines = []
    results = scoring.trajnet_evaluate(args, out=lines.append)["cv_modes50"]
    for metrics, _, _ in results.values():
        assert metrics.topk_ade > 0 and metrics.topk_ade <= metrics.average_l2
        assert np.isfinite(metrics.nll) and metrics.nll != 0
    assert "NLL" in lines[0]
