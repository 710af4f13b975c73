"""The handcrafted baselines file to file: the device Kalman filter (tb2_kalman_predict_device) against the host one, the
batched predictors of classical/batch.py on the evaluator's column pipeline against the per-scene `predict` functions on
the row pipeline, and the classical trajnet_evaluator tool."""
import ctypes
import glob
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, load_test_scenes_xy, trajnet_line

MODELS = ('kf', 'sf', 'sf_opt', 'orca', 'orca_opt', 'cv')


def _write_scenes(filename, sizes, seed, n_frames=21):
    """Scenes of `sizes` pedestrians; neighbours enter during the observation (2 rows or 1 row before its end), leave
    before its end, or appear after it."""
    rng = np.random.RandomState(seed)
    kinds = [(0, n_frames), (3, n_frames), (0, 6), (12, n_frames), (7, n_frames), (8, n_frames)]
    with open(filename, "w") as f:
        for sid, n in enumerate(sizes):
            frames = [1000 * sid + 10 * t for t in range(n_frames)]
            start, vel = rng.randn(n, 2) * 3.0, rng.randn(n, 2) * 0.3
            f.write(trajnet_line(SceneRow(sid, 100 * sid, frames[0], frames[-1], 2.5, 1 + sid % 4)) + "\n")
            for p in range(n):
                t0, t1 = (0, n_frames) if p == 0 else kinds[p % len(kinds)]
                for t in range(t0, t1):
                    x, y = start[p] + vel[p] * t + rng.randn(2) * 0.05
                    f.write(trajnet_line(TrackRow(frames[t], 100 * sid + p, x, y)) + "\n")


class _Rows:
    """The reference's predict_scene (classical/trajnet_evaluator.py:14-28) around this package's per-scene `predict`
    functions, with the evaluator's call signature: evaluate_file takes the row pipeline for it."""

    def __init__(self, model):
        self.model = model

    def __call__(self, paths, scene_goal, n_predict=12, obs_length=9, modes=1, args=None):
        from trajnetplusplusbaselines_b200.classical import constant_velocity, kalman, orca, socialforce
        kw = dict(n_predict=n_predict, obs_length=obs_length)
        if self.model == 'kf':
            return kalman.predict(paths, n_samples=0, **kw)
        if self.model == 'sf_opt':
            return socialforce.predict(paths, sf_params=[0.5, 5.0, 0.3], **kw)
        if self.model == 'orca_opt':
            return orca.predict(paths, orca_params=[0.4, 1.0, 0.3], **kw)
        if self.model == 'sf':
            return socialforce.predict(paths, **kw)
        if self.model == 'orca':
            return orca.predict(paths, **kw)
        return constant_velocity.predict(paths, **kw)


def _batched(model):
    from trajnetplusplusbaselines_b200.classical.batch import load_predictor
    return load_predictor(model, kf_samples=0)


def _both_pipelines(model, infile, tmp_path, chunk=1024, modes=1):
    from trajnetplusplusbaselines_b200.evaluator import _column_pipeline, evaluate_file
    cols, rows = str(tmp_path / ("%s_cols.ndjson" % model)), str(tmp_path / ("%s_rows.ndjson" % model))
    predictor = _batched(model)
    assert _column_pipeline(predictor, modes) and not _column_pipeline(_Rows(model), modes)
    n = evaluate_file(predictor, infile, cols, modes=modes, chunk=chunk)
    assert evaluate_file(_Rows(model), infile, rows) == n
    return open(cols, "rb").read(), open(rows, "rb").read()


# ------------------------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("modes", [1, 3])
def test_cv_batched_writes_the_per_scene_bytes(tmp_path, modes):
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 8, 2, 25, 6, 4], seed=1)
    cols, rows = _both_pipelines('cv', infile, tmp_path, chunk=3, modes=modes)
    assert cols == rows and b'"prediction_number": 1' not in cols


def test_kalman_tracks_of_a_scene_are_the_per_scene_ones(tmp_path):
    """kalman_tracks_xy picks from the xy array what kalman.predict picks from the paths (kalman.py:25-29)."""
    from trajnetplusplusbaselines_b200.classical.batch import kalman_tracks_xy
    from trajnetplusplusbaselines_b200.evaluator import load_test_scenes
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 8, 2, 25, 6, 4], seed=2)
    xys = load_test_scenes_xy(infile)
    for (xy, _), (_, _, paths) in zip(xys, load_test_scenes(infile)):
        start = paths[0][8].frame
        want = [np.array([(r.x, r.y) for r in p if r.frame <= start]) for p in paths
                if start in [r.frame for r in p] and len([r for r in p if r.frame <= start]) >= 2]
        cols, rows, lengths = kalman_tracks_xy(xy, 9)
        assert cols[0] == 0 and len(lengths) == len(want)
        assert np.array_equal(rows, np.concatenate(want)) and list(lengths) == [len(w) for w in want]


def test_kalman_device_refuses_a_one_row_track_before_any_launch():
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    offs = np.array([0, 3, 4, 9], dtype=np.int64)
    fake = ctypes.c_void_p(256)                     # never dereferenced: the call is refused on the host offsets
    before = lib.tb2_launch_count()
    rc = lib.tb2_kalman_predict_device(fake, offs.ctypes.data, fake, 3, 12, 10, 5, fake, fake, None, None, None, fake,
                                       1 << 30, None)
    assert rc == -1 and b"at least 2 observations" in lib.tb2_last_error()
    assert lib.tb2_launch_count() == before
    # the same track set is refused by the host entry point
    obs = np.zeros((9, 2))
    pred = np.zeros((3, 12, 2))
    assert lib.tb2_kalman_predict(obs.ctypes.data, offs.ctypes.data, 3, 12, 10, pred.ctypes.data, None, None, None) == -1
    # workspace: T_max x 76 doubles per track; nothing for no track
    assert lib.tb2_kalman_workspace_bytes(offs.ctypes.data, 3) == 5 * 76 * 3 * 8
    assert lib.tb2_kalman_workspace_bytes(offs.ctypes.data, 0) == 0
    assert lib.tb2_kalman_predict_device(None, offs.ctypes.data, None, 0, 12, 10, 5, None, None, None, None, None, None,
                                         0, None) == 0
    assert lib.tb2_launch_count() == before


def _tree(root, name, sizes, seed):
    for sub in ("test", "test_private"):
        os.makedirs(os.path.join(root, "DATA_BLOCK", name, sub))
    for i, s in enumerate(sizes):
        path = os.path.join(root, "DATA_BLOCK", name, "test", "file%d.ndjson" % i)
        _write_scenes(path, s, seed + i)
        with open(path) as f, open(path.replace(os.sep + "test" + os.sep, os.sep + "test_private" + os.sep), "w") as g:
            g.write(f.read())


def test_cli_model_list_folders_and_skipping(tmp_path, monkeypatch, capsys):
    from trajnetplusplusbaselines_b200.classical import trajnet_evaluator as T
    from trajnetplusplusbaselines_b200.classical.batch import ConstantVelocityBatch, load_predictor
    args = T.parser().parse_args(['--kf', '--sf', '--orca', '--cv', '--normalize_scene'])
    assert T.model_list(args) == ['/kf.pkl', '/sf.pkl', '/sf_opt.pkl', '/orca.pkl', '/orca_opt.pkl', '/cv.pkl']
    assert T.model_list(T.parser().parse_args(['--orca'])) == ['/orca.pkl', '/orca_opt.pkl']
    assert [type(load_predictor(m)).__name__ for m in MODELS] == [
        'KalmanBatch', 'SocialForceBatch', 'SocialForceBatch', 'OrcaBatch', 'OrcaBatch', 'ConstantVelocityBatch']
    assert load_predictor('sf_opt_modes1').sf_params == [0.5, 5.0, 0.3]
    assert load_predictor('orca_opt_modes1').orca_params == [0.4, 1.0, 0.3]
    assert load_predictor('orca_modes3').orca_params == [1.5, 1.5, 0.4]
    with pytest.raises(SystemExit):
        T.main(['--path', 'synth'])
    # every model served by constant velocity (CPU): the folders, their order, the skipped one
    _tree(str(tmp_path), "synth", [[3, 5, 2], [4]], seed=3)
    monkeypatch.chdir(str(tmp_path))
    pred_dir = os.path.join("DATA_BLOCK", "synth", "test_pred")
    os.makedirs(os.path.join(pred_dir, "sf_modes2"))
    seen = []
    assert T.main(['--path', 'synth', '--kf', '--sf', '--orca', '--cv', '--write_only', '--modes', '2', '--chunk', '2'],
                  load_predictor=lambda m: seen.append(m) or ConstantVelocityBatch()) is None
    assert seen == ['/kf.pkl', '/sf_opt.pkl', '/orca.pkl', '/orca_opt.pkl', '/cv.pkl']
    out = capsys.readouterr().out
    assert 'Predictions corresponding to sf_modes2 already exist.' in out
    assert 'kf_modes2: 4 scenes written' in out
    assert sorted(os.listdir(pred_dir)) == sorted(m + '_modes2' for m in MODELS)
    assert os.listdir(os.path.join(pred_dir, "sf_modes2")) == []
    for m in ('kf', 'cv'):
        assert sorted(os.listdir(os.path.join(pred_dir, m + '_modes2'))) == ['file0.ndjson', 'file1.ndjson']
    text = open(os.path.join(pred_dir, "cv_modes2", "file0.ndjson")).read()
    assert '"prediction_number": 0' in text and '"prediction_number": 1' not in text


# ------------------------------------------------------------------------------------------------------------------
# GPU: the device Kalman filter against the host one
# ------------------------------------------------------------------------------------------------------------------
def _concat(tracks):
    offs = np.zeros(len(tracks) + 1, dtype=np.int64)
    offs[1:] = np.cumsum([len(t) for t in tracks])
    return (np.concatenate(tracks) if tracks else np.zeros((0, 2))), offs


def _host(obs, offs, n_predict, em_iterations):
    from trajnetplusplusbaselines_b200 import _lib
    n = len(offs) - 1
    obs = np.ascontiguousarray(obs, dtype=np.float64)
    pred, q, r, last = np.zeros((n, n_predict, 2)), np.zeros((n, 4, 4)), np.zeros((n, 2, 2)), np.zeros((n, 4))
    _lib.check(_lib.load().tb2_kalman_predict(obs.ctypes.data, offs.ctypes.data, n, n_predict, em_iterations,
                                              pred.ctypes.data, q.ctypes.data, r.ctypes.data, last.ctypes.data))
    return pred, q, r, last


def _assert_device_equals_host(obs, offs, n_predict, em_iterations):
    from trajnetplusplusbaselines_b200.classical.kalman import predict_concat_device
    dev = [t.cpu().numpy() for t in predict_concat_device(obs, offs, n_predict=n_predict, n_samples=0,
                                                          em_iterations=em_iterations)]
    host = _host(obs, offs, n_predict, em_iterations)
    for name, d, h in zip(("pred", "q", "r", "last"), dev, host):
        assert d.shape == h.shape, name
        differ = d.view(np.int64) != h.view(np.int64)
        assert not differ.any(), "%s: %d of %d values differ (max %.3g)" % (name, differ.sum(), d.size,
                                                                             np.abs(d - h).max())


def _random_tracks(n, seed, t_lo=2, t_hi=20):
    rng = np.random.RandomState(seed)
    return [np.cumsum(rng.randn(rng.randint(t_lo, t_hi + 1), 2) * 0.3, axis=0) + rng.randn(2) * 5 for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("em_iterations", [0, 1, 10])
@pytest.mark.parametrize("n_predict", [1, 12])
def test_kalman_device_bit_identical_to_host_random_tracks(em_iterations, n_predict):
    obs, offs = _concat(_random_tracks(777, seed=em_iterations * 13 + n_predict))
    _assert_device_equals_host(obs, offs, n_predict, em_iterations)


@pytest.mark.gpu
def test_kalman_device_zero_tracks():
    from trajnetplusplusbaselines_b200.classical.kalman import predict_tracks_device
    pred = predict_tracks_device([], n_predict=12)
    assert pred.is_cuda and tuple(pred.shape) == (0, 12, 2)
    with pytest.raises(RuntimeError, match="at least 2 observations"):
        predict_tracks_device([np.zeros((3, 2)), np.zeros((1, 2))], n_samples=0)


@pytest.mark.gpu
@pytest.mark.needs_reference
@pytest.mark.parametrize("em_iterations,n_predict", [(10, 12), (1, 1)])
def test_kalman_device_bit_identical_to_host_trajdata(em_iterations, n_predict):
    """The tracks of every scene of the reference's seven training files cut at the observation."""
    from oracle.ref_shim import reference_root
    from trajnetplusplusbaselines_b200.classical.batch import kalman_tracks_xy
    files = sorted(glob.glob(os.path.join(reference_root(), "DATA_BLOCK", "trajdata", "train", "*.ndjson")))
    assert len(files) == 7
    rows, lengths = [], []
    for f in files:
        for xy, _ in load_test_scenes_xy(f, 9):
            _, r, n = kalman_tracks_xy(xy, 9)
            rows.append(r)
            lengths.extend(n)
    offs = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    assert len(lengths) > 10000
    _assert_device_equals_host(np.concatenate(rows), offs, n_predict, em_iterations)


def _chol_psd(S):
    """NumPy restatement of chol_psd (csrc/kalman.cu): lower Cholesky of the symmetric part with a zero-pivot guard."""
    n = S.shape[0]
    S = 0.5 * (S + S.T)
    L = np.zeros_like(S)
    tol = 1e-12 * max(0.0, S.diagonal().max())
    for j in range(n):
        d = S[j, j] - np.dot(L[j, :j], L[j, :j])
        if not d > tol:
            continue
        L[j, j] = np.sqrt(d)
        for i in range(j + 1, n):
            L[i, j] = (S[i, j] - np.dot(L[i, :j], L[j, :j])) / L[j, j]
    return L


_A = np.array([[1, 1, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 0, 1]], dtype=np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("n_samples", [1, 5])
def test_kalman_device_injected_noise_matches_numpy(n_samples):
    from trajnetplusplusbaselines_b200.classical.kalman import predict_concat_device
    tracks = _random_tracks(300, seed=21) + [np.array([[1.0, 2.0], [1.0, 2.0]]), np.array([[0.0, 0.0]] * 5)]
    obs, offs = _concat(tracks)
    n, T = len(tracks), 12
    eps = np.random.RandomState(22).standard_normal((n, T, 6))
    pred = predict_concat_device(obs, offs, n_predict=T, n_samples=n_samples, eps=eps)[0].cpu().numpy()
    mean, q, r, last = _host(obs, offs, T, 10)
    s = 1.0 / np.sqrt(n_samples)
    worst = 0.0
    for i in range(n):
        LQ, LR = _chol_psd(q[i]), _chol_psd(r[i])
        # the factor reproduces the fitted covariance (zero pivots of a singular one included); the EM's sums leave
        # it symmetric only up to rounding, so the factor is that of its symmetric part
        for S, L in ((q[i], LQ), (r[i], LR)):
            assert np.abs(L @ L.T - 0.5 * (S + S.T)).max() <= 1e-9 * max(S.diagonal().max(), 1e-300), i
        dx = np.zeros(4)
        want = np.empty((T, 2))
        for k in range(T):
            dx = _A @ dx + s * (LQ @ eps[i, k, :4])
            want[k] = mean[i, k] + dx[[0, 2]] + s * (LR @ eps[i, k, 4:])
        worst = max(worst, np.abs(pred[i] - want).max())
    assert worst <= 1e-12, worst


@pytest.mark.gpu
def test_kalman_device_sampled_statistics():
    """20 k copies of one track: pred - expectation has mean 0 and covariance (C P_k C^T + R) / n, P_k = A P_{k-1} A^T
    + Q from P_0 = 0 -- the covariance of the mean of n sampled rollouts."""
    from trajnetplusplusbaselines_b200.classical.kalman import predict_concat_device
    track = _random_tracks(1, seed=5, t_lo=9, t_hi=9)[0]
    N, T, n = 20000, 12, 5
    obs, offs = _concat([track] * N)
    gen = torch.Generator(device="cuda").manual_seed(1234)
    pred = predict_concat_device(obs, offs, n_predict=T, n_samples=n, generator=gen)[0].cpu().numpy()
    mean, q, r, _ = _host(obs[:len(track)], offs[:2], T, 10)
    dev = pred - mean[0]
    P = np.zeros((4, 4))
    for k in range(T):
        P = _A @ P @ _A.T + q[0]
        S = (P[np.ix_([0, 2], [0, 2])] + r[0]) / n
        sd = np.sqrt(S.diagonal())
        m = dev[:, k].mean(axis=0)
        C = np.cov(dev[:, k].T)
        assert (np.abs(m) <= 5 * sd / np.sqrt(N)).all(), (k, m, sd)
        assert (np.abs(C - S) <= 0.06 * np.outer(sd, sd)).all(), (k, C, S)


# ------------------------------------------------------------------------------------------------------------------
# GPU: evaluate_file through the batched predictors writes the per-scene row pipeline's bytes
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_batched_model_writes_the_per_scene_bytes_synthetic(tmp_path, model):
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 8, 2, 25, 6, 4, 40, 12, 5], seed=7)
    cols, rows = _both_pipelines(model, infile, tmp_path, chunk=4)
    assert cols == rows
    assert cols.count(b'"scene"') == 10


def _first_scenes(src, dst, n):
    """`src` with its first n scene records only (every track record kept)."""
    kept = 0
    with open(src) as f, open(dst, "w") as g:
        for line in f:
            if line.startswith('{"scene"'):
                kept += 1
                if kept > n:
                    continue
            g.write(line)


@pytest.mark.gpu
@pytest.mark.needs_reference
@pytest.mark.parametrize("model", MODELS)
def test_batched_model_writes_the_per_scene_bytes_reference_files(tmp_path, model):
    """The reference's collision test scene and its seven training files read as test files: every scene for kf and cv;
    for the simulators, whose per-scene path costs a scene layout and a launch per scene, the first 150 scenes of each
    training file."""
    from oracle.ref_shim import reference_root
    root = os.path.join(reference_root(), "DATA_BLOCK")
    files = [os.path.join(root, "collision_test", "test", "collision_test.ndjson")]
    train = sorted(glob.glob(os.path.join(root, "trajdata", "train", "*.ndjson")))
    assert len(train) == 7
    for f in train:
        if model in ('kf', 'cv'):
            files.append(f)
        else:
            files.append(str(tmp_path / os.path.basename(f)))
            _first_scenes(f, files[-1], 150)
    for f in files:
        cols, rows = _both_pipelines(model, f, tmp_path)
        assert cols == rows, (model, f)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _eval_worker(rank, world, port, infile, outfile, model):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file
    assert evaluate_file(_batched(model), infile, outfile, chunk=3) == 9
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("model", ['kf', 'sf', 'orca_opt'])
def test_batched_model_sharded_world2_gloo(tmp_path, model):
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 6, 2, 2, 9, 4, 30, 5], seed=8)
    single = str(tmp_path / "single.ndjson")
    assert evaluate_file(_Rows(model), infile, single) == 9
    sharded = str(tmp_path / "sharded.ndjson")
    mp.spawn(_eval_worker, args=(2, _free_port(), infile, sharded, model), nprocs=2, join=True)
    assert open(sharded, "rb").read() == open(single, "rb").read()


@pytest.mark.gpu
def test_cli_end_to_end_scores_like_the_row_pipeline(tmp_path, monkeypatch, capsys):
    import types
    from trajnetplusplusbaselines_b200.classical import trajnet_evaluator as T
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file
    from trajnetplusplusbaselines_b200.scoring import trajnet_evaluate
    _tree(str(tmp_path), "synth", [[3, 5, 2, 8, 1], [4, 12, 6]], seed=9)
    monkeypatch.chdir(str(tmp_path))
    results = T.main(['--path', 'synth', '--kf', '--sf', '--orca', '--cv'])
    out = capsys.readouterr().out
    pred_dir = os.path.join("DATA_BLOCK", "synth", "test_pred")
    assert sorted(os.listdir(pred_dir)) == sorted(m + '_modes1' for m in MODELS)
    assert sorted(results) == sorted(m + '_modes1' for m in MODELS)
    # the row pipeline's files of the deterministic models, scored in a tree of their own
    row_dir = os.path.join("DATA_BLOCK", "rows", "test_pred")
    for sub in ("test", "test_private"):
        os.makedirs(os.path.join("DATA_BLOCK", "rows", sub))
        for f in ("file0.ndjson", "file1.ndjson"):
            with open(os.path.join("DATA_BLOCK", "synth", sub, f)) as src, \
                    open(os.path.join("DATA_BLOCK", "rows", sub, f), "w") as dst:
                dst.write(src.read())
    for m in ('sf', 'sf_opt', 'orca', 'orca_opt', 'cv'):
        os.makedirs(os.path.join(row_dir, m + '_modes1'))
        for f in ("file0.ndjson", "file1.ndjson"):
            evaluate_file(_Rows(m), os.path.join("DATA_BLOCK", "rows", "test", f), os.path.join(row_dir, m + '_modes1', f))
            assert open(os.path.join(row_dir, m + '_modes1', f), "rb").read() == \
                open(os.path.join(pred_dir, m + '_modes1', f), "rb").read()
    tables = []
    args = types.SimpleNamespace(path=row_dir + os.sep, output=['/sf.pkl', '/sf_opt.pkl', '/orca.pkl', '/orca_opt.pkl',
                                                                 '/cv.pkl'],
                                 modes=1, obs_length=9, pred_length=12, labels=None, disable_collision=False)
    trajnet_evaluate(args, out=tables.append)
    assert len(tables) == 5
    for table in tables:
        assert table in out
