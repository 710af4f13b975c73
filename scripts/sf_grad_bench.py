"""Cost of the social-force derivatives: tb2_sf_sweep against tb2_sf_sweep_grad on the same scenes, and the fit's
wall-clock.

    python scripts/sf_grad_bench.py [--scenes 2000] [--P 1 64] [--rounds 7] [--reps 5]

Synthetic scenes with a trajdata-like size mix (mostly 2-20 pedestrians, a few up to 70; all under the tangent
kernel's 256), truth a social-force rollout at a known setting plus 1 cm noise.  Per P the two sweeps run in
alternating rounds of `reps` launches each, timed with CUDA events; the median seconds per launch of each are
reported with their ratio.  Then classical.fit.fit runs once from a 27-cell grid (pooled over the scenes as one file),
wall-clock with its evaluation count.  Prints one JSON line with the GPU's name and power limit."""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from trajnetplusplusbaselines_b200.classical import common, fit, socialforce

THETA_STAR = (0.62, 1.7, 0.41)


def scenes(B, seed=0):
    rng = np.random.RandomState(seed)
    sizes = np.where(rng.rand(B) < 0.95, rng.randint(2, 21, B), rng.randint(21, 71, B))
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    A = int(offs[-1])
    pos = rng.randn(A, 2) * (1.0 + 0.15 * np.sqrt(np.repeat(sizes, sizes)))[:, None]
    ang = rng.rand(A) * 2 * np.pi
    spd = 0.3 + rng.rand(A) * 1.2
    vel = np.stack([spd * np.cos(ang), spd * np.sin(ang)], axis=1)
    state = np.concatenate([pos, vel, pos + vel * 4.8 + rng.randn(A, 2) * 0.3], axis=1)
    sim = socialforce.simulate_batch(state, offs, THETA_STAR).cpu().numpy()
    truth = np.stack([sim[:, offs[b]] for b in range(B)]) + rng.randn(B, 12, 2) * 0.01
    return common.to_device(state, spd, offs, truth), sizes


def timed(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1000.0 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=2000)
    ap.add_argument("--P", type=int, nargs="+", default=[1, 64])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    prepared, sizes = scenes(args.scenes)
    out = {"gpu": gpu, "scenes": int(len(sizes)), "pedestrians": int(sizes.sum()), "max_scene": int(sizes.max())}
    rng = np.random.RandomState(1)
    for P in args.P:
        grid = [tuple(float(v) for v in THETA_STAR * (0.7 + 0.6 * rng.rand(3))) for _ in range(P)]
        value = lambda: socialforce.sweep(prepared, grid)
        grad = lambda: socialforce.sweep_grad(prepared, grid)
        value()
        grad()
        torch.cuda.synchronize()
        tv, tg = [], []
        for _ in range(args.rounds):
            tv.append(timed(value, args.reps))
            tg.append(timed(grad, args.reps))
        mv, mg = float(np.median(tv)), float(np.median(tg))
        out["P%d" % P] = {"sweep_s": mv, "sweep_grad_s": mg, "ratio": mg / mv,
                          "sweep_spread": [min(tv), max(tv)], "sweep_grad_spread": [min(tg), max(tg)],
                          "scene_simulations_per_s": {"sweep": len(sizes) * P / mv, "sweep_grad": len(sizes) * P / mg}}
    grid = list(itertools.product((0.3, 0.5, 1.0), (1.0, 2.1, 5.0), (0.2, 0.3, 0.6)))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fit.fit([prepared], grid)["pooled"]
    torch.cuda.synchronize()
    out["fit"] = {"seconds": time.perf_counter() - t0, "grid": len(grid), "nit": r["nit"], "nfev": r["nfev"],
                  "theta": r["theta"], "theta_star": THETA_STAR, "start": r["start"], "start_ade": r["start_ade"],
                  "ade": r["ade"]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
