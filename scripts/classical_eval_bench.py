"""The handcrafted baselines file to file, and the Kalman filter on the device.

Kalman, at 10 k / 100 k / 500 k tracks of 2-9 observations (em 10, 12 predicted steps):
  * tb2_kalman_predict_device, expectation: the kernel alone (CUDA events over repeated launches on resident buffers) and
    predict_concat_device end to end (host arrays in, device tensors out, synchronised);
  * the same with the noise of 5 sampled rollouts (torch.randn on the device included);
  * tb2_kalman_predict on the host's threads (expectation), and the host n_samples=5 path (NumPy sampling loop) on a
    subset;
  * float64 operations and workspace bytes per track, computed from the shapes (flops_per_track below).
evaluate_file per model (kf, sf, sf_opt, orca, orca_opt, cv) against the per-scene loop of this package's `predict`
followed by write_predictions, on a synthetic 1024-scene test file of 2-20 pedestrians and, when the DATA_BLOCK copy of
the reference is present, on its seven trajdata/train files read as test files.  The per-scene loop is timed on at most
`PER_SCENE_CAP` scenes per file (its rate does not depend on the count).  kf in the per-scene loop is the expectation
(n_samples=0), like the batched kf it is compared with; the batched kf with 5 samples is reported beside it.

Prints one JSON line per measurement, then one with the GPU's name and power limit (read in the same call).
"""
import glob
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from trajnetplusplusbaselines_b200 import _lib
from trajnetplusplusbaselines_b200.classical import constant_velocity, kalman, orca, socialforce
from trajnetplusplusbaselines_b200.classical.batch import MODELS, load_predictor
from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, trajnet_line, write_predictions
from trajnetplusplusbaselines_b200.engine import _ptr, _stream
from trajnetplusplusbaselines_b200.evaluator import evaluate_file, load_test_scenes

PER_SCENE_CAP = int(os.environ.get("TB2_BENCH_PER_SCENE_CAP", "150"))
KF_SIZES = [int(v) for v in os.environ.get("TB2_BENCH_KF_TRACKS", "10000,100000,500000").split(",")]


def emit(**kw):
    print(json.dumps(kw), flush=True)


def flops_per_track(T, em_iterations=10, n_predict=12):
    """float64 additions, multiplications and divisions of the EM / smoother code of csrc/kalman.cu for one track of T
    observations (a 4x4 product = 64 mul + 64 add, a matrix-vector product 32; inv4 counted in full, 256)."""
    filt = 117 * T + 304 * (T - 1)             # per step: gain, update, covariance; predict from step 1 on
    smooth = 840 * (T - 1)                     # inv4, gain, mean and covariance per step back
    mstep = 14 * T + 644 * (T - 1) + 20        # R, Q sums and their divisions
    return (em_iterations + 1) * (filt + smooth) + em_iterations * mstep + 32 * n_predict


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return torch.cuda.get_device_name(0), q


def synced(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def bench_kalman(n_tracks, rng):
    lengths = rng.randint(2, 10, size=n_tracks)
    offs = np.zeros(n_tracks + 1, dtype=np.int64)
    offs[1:] = np.cumsum(lengths)
    steps = rng.randn(int(offs[-1]), 2) * 0.3
    obs = np.cumsum(steps, axis=0)                               # random walks, one per track after re-centring
    obs -= np.repeat(obs[offs[:-1]], lengths, axis=0)
    obs += np.repeat(rng.randn(n_tracks, 2) * 5, lengths, axis=0)
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    # kernel alone on resident buffers
    obs_t, offs_t = torch.from_numpy(obs).to(dev), torch.from_numpy(offs).to(dev)
    pred = torch.empty((n_tracks, 12, 2), dtype=torch.float64, device=dev)
    ws_bytes = int(lib.tb2_kalman_workspace_bytes(offs.ctypes.data, n_tracks))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)

    def launch():
        _lib.check(lib.tb2_kalman_predict_device(_ptr(obs_t), offs.ctypes.data, _ptr(offs_t), n_tracks, 12, 10, 0, None,
                                                 _ptr(pred), None, None, None, _ptr(ws), ws_bytes, _stream(dev)))
    launch()
    reps = max(3, min(20, 2000000 // n_tracks))
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        launch()
    end.record()
    torch.cuda.synchronize()
    t_kernel = start.elapsed_time(end) / 1e3 / reps
    # end to end, expectation and 5 samples
    kalman.predict_concat_device(obs, offs, n_samples=0)
    (dev_pred, _, _, _), t_e2e = synced(lambda: kalman.predict_concat_device(obs, offs, n_samples=0))
    gen = torch.Generator(device=dev).manual_seed(0)
    _, t_e2e5 = synced(lambda: kalman.predict_concat_device(obs, offs, n_samples=5, generator=gen))
    # host threads, expectation
    host_pred = np.zeros((n_tracks, 12, 2))
    t0 = time.perf_counter()
    _lib.check(lib.tb2_kalman_predict(obs.ctypes.data, offs.ctypes.data, n_tracks, 12, 10, host_pred.ctypes.data,
                                      None, None, None))
    t_host = time.perf_counter() - t0
    identical = bool(np.array_equal(dev_pred.cpu().numpy().view(np.int64), host_pred.view(np.int64)))
    # host n_samples=5 (the reference's sampled mean, NumPy loop) on a subset
    sub = min(n_tracks, 200)
    tracks = [obs[offs[i]:offs[i + 1]] for i in range(sub)]
    t0 = time.perf_counter()
    kalman.predict_tracks(tracks, n_predict=12, n_samples=5)
    t_host5 = (time.perf_counter() - t0) / sub
    flops = float(np.mean([flops_per_track(int(T)) for T in lengths]))
    emit(bench="kalman", tracks=n_tracks, obs_per_track="2-9", em_iterations=10, n_predict=12,
         device_kernel_s=t_kernel, device_kernel_tracks_per_s=n_tracks / t_kernel,
         device_e2e_expectation_tracks_per_s=n_tracks / t_e2e, device_e2e_5_samples_tracks_per_s=n_tracks / t_e2e5,
         host_threads=os.cpu_count(), host_expectation_tracks_per_s=n_tracks / t_host,
         host_5_samples_tracks_per_s=1.0 / t_host5, host_5_samples_subset=sub,
         kernel_vs_host_expectation=t_host / t_kernel, e2e_vs_host_expectation=t_host / t_e2e,
         flops_per_track=flops, kernel_gflops=flops * n_tracks / t_kernel / 1e9,
         workspace_bytes_per_track=ws_bytes / n_tracks, device_equals_host_bitwise=identical)
    del ws, obs_t, offs_t, pred
    torch.cuda.empty_cache()


def write_synthetic(filename, n_scenes, rng):
    with open(filename, "w") as f:
        for sid in range(n_scenes):
            n = rng.randint(2, 21)
            frames = [1000 * sid + 10 * t for t in range(21)]
            start, vel = rng.randn(n, 2) * 3.0, rng.randn(n, 2) * 0.3
            f.write(trajnet_line(SceneRow(sid, 100 * sid, frames[0], frames[-1], 2.5, 1)) + "\n")
            for p in range(n):
                t0, t1 = (0, 21) if p == 0 else [(0, 21), (3, 21), (0, 6), (12, 21)][p % 4]
                for t in range(t0, t1):
                    x, y = start[p] + vel[p] * t + rng.randn(2) * 0.05
                    f.write(trajnet_line(TrackRow(frames[t], 100 * sid + p, x, y)) + "\n")


def per_scene(model, paths):
    kw = dict(n_predict=12, obs_length=9)
    if model == 'kf':
        return kalman.predict(paths, n_samples=0, **kw)
    if model == 'sf_opt':
        return socialforce.predict(paths, sf_params=[0.5, 5.0, 0.3], **kw)
    if model == 'orca_opt':
        return orca.predict(paths, orca_params=[0.4, 1.0, 0.3], **kw)
    if model == 'sf':
        return socialforce.predict(paths, **kw)
    if model == 'orca':
        return orca.predict(paths, **kw)
    return constant_velocity.predict(paths, **kw)


def bench_files(label, files, d):
    scenes = {f: load_test_scenes(f) for f in files}
    n_total = sum(len(s) for s in scenes.values())
    for model in MODELS + ('kf_5_samples',):
        predictor = load_predictor(model, kf_samples=5 if model == 'kf_5_samples' else 0)
        out = os.path.join(d, "out.ndjson")
        evaluate_file(predictor, files[0], out)                    # warm-up
        _, t_batch = synced(lambda: [evaluate_file(predictor, f, out) for f in files])
        row = dict(bench="evaluate_file", files=label, model=model, scenes=n_total,
                   batched_scenes_per_s=n_total / t_batch)
        if model != 'kf_5_samples':
            n_loop, t_loop = 0, 0.0
            for f in files:
                part = scenes[f][:PER_SCENE_CAP]
                def loop():
                    preds = [per_scene(model, paths) for _, _, paths in part]
                    write_predictions(preds, part, out)
                _, t = synced(loop)
                n_loop += len(part)
                t_loop += t
            row.update(per_scene_scenes_per_s=n_loop / t_loop, per_scene_timed_scenes=n_loop,
                       speedup=(t_loop / n_loop) / (t_batch / n_total))
        emit(**row)


def main():
    _lib.require_cuda()
    torch.cuda.set_device(0)
    rng = np.random.RandomState(0)
    for n in KF_SIZES:
        bench_kalman(n, rng)
    with tempfile.TemporaryDirectory() as d:
        synth = os.path.join(d, "synthetic.ndjson")
        write_synthetic(synth, 1024, rng)
        bench_files("synthetic 1024 scenes of 2-20 pedestrians", [synth], d)
        from oracle.ref_shim import reference_root
        root = reference_root()
        train = sorted(glob.glob(os.path.join(root, "DATA_BLOCK", "trajdata", "train", "*.ndjson"))) if root else []
        if train:
            bench_files("trajdata/train, 7 files read as test files", train, d)
        else:
            emit(bench="evaluate_file", files="trajdata/train", skipped="DATA_BLOCK copy of the reference not present")
    name, power = device_info()
    emit(gpu=name, name_power_limit=power, host_cpus=os.cpu_count())


if __name__ == "__main__":
    main()
