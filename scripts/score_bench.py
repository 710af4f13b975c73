"""Device scorer against the CPU path on the DATA_BLOCK training scenes.

    python scripts/score_bench.py [--modes 1 3 50] [--cpu-scenes 200] [--out DIR]

Ground truth: every scene of the reference's DATA_BLOCK/trajdata/train files (13 718 scenes, real tags; read from
oracle/_ref, which build() makes, or the reference tree).  Predictions: per scene the primary's last 12 frames plus seeded
noise for every mode and mode 0 of every neighbour seen during the observation, written with the project's writer.

  device  scoring.score_file per file: parse, assembly, one tb2_score_scenes launch, aggregation (wall clock, the
          launch ends in a device synchronise), and score_arrays alone (CUDA events around the copies to the device,
          the launch and the copies back);
  cpu     the reference's TrajnetEvaluator.aggregate over oracle/metrics_oracle.py (scipy gaussian_kde for the NLL) on
          the first --cpu-scenes scenes of each file, paths already in memory (the reader is not timed).
Prints one JSON line per mode count with scenes/s of both sides, the GPU name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_label():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def write_predictions(gt_file, out_file, modes, rng, obs_length=9, pred_length=12):
    from trajnetplusplusbaselines_b200 import scoring
    from trajnetplusplusbaselines_b200.data import SceneMeta, write_predictions_xy
    r = scoring.SceneReader(scoring.parse_ndjson_meta(gt_file))
    metas, preds = [], []
    for i in range(len(r)):
        w = r.window(i)
        f, p, xy = r.f[w], r.p[w], r.xy[w]
        prim = p == r.ped[i]
        pf = f[prim]
        if len(pf) < obs_length + pred_length:
            continue
        frames = pf[-pred_length:]
        peds, first = scoring.first_appearance(f, p, r.ped[i])
        peds = peds[first <= pf[obs_length - 1]]
        nb = scoring.tracks_on_frames(f, p, xy, peds, frames)[0].transpose(1, 0, 2)
        gt = xy[prim][-pred_length:]
        scale = 0.05 + 0.1 * np.arange(pred_length)[:, None] / pred_length
        preds.append({m: [gt + rng.randn(pred_length, 2) * scale * (1 + m % 4),
                          nb + rng.randn(*nb.shape) * 0.1 if m == 0 and len(peds) else []] for m in range(modes)})
        metas.append(SceneMeta(int(r.scene_id[i]), int(r.ped[i]), int(pf[0]), int(pf[1] - pf[0]), int(pf[obs_length - 1]),
                               peds.tolist()))
    write_predictions_xy(preds, metas, out_file, obs_length=obs_length, pred_length=pred_length)
    return len(metas)


def time_cpu(gt_file, pred_file, n_scenes):
    from oracle import make_scoring_golden as G
    _, trajnet_evaluator = G.reference()
    gt_text, pred_text = open(gt_file).read(), open(pred_file).read()
    cut = -1                                   # the writer puts each scene's rows after its scene line: keep n_scenes
    for _ in range(n_scenes + 1):
        cut = pred_text.find('{"scene"', cut + 1)
        if cut < 0:
            break
    if cut >= 0:
        pred_text = pred_text[:cut]
    gt, scenes_by_id = G.read_paths(gt_text, n_scenes)
    pred, _ = G.read_paths(pred_text, n_scenes)
    from collections import defaultdict
    indexes, sub_indexes = defaultdict(list), defaultdict(list)
    for sid, s in scenes_by_id.items():
        indexes[s.tag[0]].append(sid)
        for sub in s.tag[1]:
            sub_indexes[sub].append(sid)
    args = types.SimpleNamespace(pred_length=12, obs_length=9, disable_collision=False)
    ev = trajnet_evaluator.TrajnetEvaluator([p for _, p in gt], [sid for sid, _ in gt], [p for _, p in pred], indexes,
                                            sub_indexes, args)
    import contextlib
    import io
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        ev.aggregate()
    return time.perf_counter() - t0, len(gt)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", type=int, nargs="+", default=[1, 3, 50])
    ap.add_argument("--cpu-scenes", type=int, default=200, help="scenes per file timed on the CPU path (0: skip it)")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None, help="also append the JSON lines to DIR/score_bench.jsonl")
    a = ap.parse_args()
    import torch
    from oracle.ref_shim import reference_root
    from trajnetplusplusbaselines_b200 import _lib, scoring
    _lib.require_cuda()
    root = reference_root()
    if root is None:
        raise SystemExit("DATA_BLOCK not found: run build() (oracle/_ref) first")
    train = os.path.join(root, "DATA_BLOCK", "trajdata", "train")
    files = sorted(os.path.join(train, f) for f in os.listdir(train) if f.endswith(".ndjson"))
    gpu = gpu_label()
    with tempfile.TemporaryDirectory() as tmp:
        for modes in a.modes:
            rng = np.random.RandomState(modes)
            preds, scenes = [], 0
            for fn in files:
                out = os.path.join(tmp, "m%d_%s" % (modes, os.path.basename(fn)))
                scenes += write_predictions(fn, out, modes, rng)
                preds.append(out)
            print("modes %d: %d scenes written" % (modes, scenes), flush=True)
            for fn, pr in zip(files, preds):                            # warm-up: module load, allocator
                scoring.score_file(fn, pr)
            walls, kernels = [], []
            for _ in range(a.repeats):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for fn, pr in zip(files, preds):
                    scoring.score_file(fn, pr)
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t0)
                k = 0.0
                for fn, pr in zip(files, preds):
                    arr = scoring.assemble(fn, pr)
                    with_nll = arr["num_predictions"] > scoring.NLL_MIN_PREDICTIONS
                    scoring.score_arrays(arr, with_nll)                 # the allocator holds the sizes before timing
                    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    start.record()
                    scoring.score_arrays(arr, with_nll)
                    stop.record()
                    stop.synchronize()
                    k += start.elapsed_time(stop) / 1e3
                kernels.append(k)
                print("modes %d: device pass %.2f s" % (modes, walls[-1]), flush=True)
            rec = dict(bench="score_files", gpu=gpu, modes=modes, scenes=scenes, files=len(files),
                       device_wall_s=min(walls), device_scenes_per_s=scenes / min(walls),
                       device_launch_incl_copies_s=min(kernels))
            if a.cpu_scenes:
                cpu_t, cpu_n = 0.0, 0
                for fn, pr in zip(files, preds):
                    t, n = time_cpu(fn, pr, a.cpu_scenes)
                    cpu_t += t
                    cpu_n += n
                rec.update(cpu_scenes=cpu_n, cpu_s=cpu_t, cpu_scenes_per_s=cpu_n / cpu_t,
                           speedup_scenes_per_s=(scenes / min(walls)) / (cpu_n / cpu_t))
            line = json.dumps(rec)
            print(line, flush=True)
            if a.out:
                os.makedirs(a.out, exist_ok=True)
                with open(os.path.join(a.out, "score_bench.jsonl"), "a") as f:
                    f.write(line + "\n")


if __name__ == "__main__":
    main()
