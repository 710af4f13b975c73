"""Social-force / ORCA parameter sweeps over the TrajNet++ training files: one launch per grid (socialforce.sweep /
orca.sweep) against the per-setting loop a user has without it (simulate_batch + NumPy scoring per setting) and the
CPU restatement (oracle/classical_oracle.py, oracle/orca_oracle.c) on a bounded sample.

    python scripts/classical_sweep_bench.py DATA_BLOCK/trajdata/train/*.ndjson [--P 1 64 1000] [--loop 16] [--cpu 40]

All scenes of the given files are prepared once (sweep.prepare_file) and swept together.  Prints one JSON object:
per simulator and P, device-timed seconds, scene-simulations/s (scenes x settings / s) and settings/s; the loop's rates
over `--loop` settings (a loop's cost is linear in P); the CPU restatement's scene-simulations/s over `--cpu` scenes; the
lane occupancy of the packed sweep on these scenes (simulated pedestrians / lanes held), and the GPU's name and power
limit.  The grids are Cartesian products around the reference tool's defaults."""
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

from trajnetplusplusbaselines_b200.classical import common, orca, socialforce, sweep


def grid(P, center, spread):
    """P settings: a Cartesian product of k values per parameter around `center`, cut to P (the center first)."""
    k = max(1, int(np.ceil(P ** (1.0 / 3.0))))
    axes = [sorted(set([c] + list(c * np.linspace(1.0 - spread, 1.0 + spread, k))), key=lambda v: abs(v - c))
            for c in center]
    return [tuple(float(v) for v in s) for s in itertools.product(*axes)][:P]


def device_time(fn, reps, warm):
    warm()                                               # modules loaded, layouts built: one setting is enough
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / 1000.0 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("files", nargs="+")
    ap.add_argument("--P", type=int, nargs="+", default=[1, 64, 1000])
    ap.add_argument("--loop", type=int, default=16, help="settings timed in the per-setting loop")
    ap.add_argument("--cpu", type=int, default=40, help="scenes of the CPU restatement")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()

    parts = [sweep.prepare_file(f) for f in args.files]
    state = np.concatenate([p.state.cpu().numpy() for p in parts])
    speeds = np.concatenate([p.speeds.cpu().numpy() for p in parts])
    truth = np.concatenate([p.truth.cpu().numpy() for p in parts])
    counts = np.concatenate([np.diff(p.agent_offsets) for p in parts])
    offs = np.concatenate([[0], np.cumsum(counts)])
    prepared = common.to_device(state, speeds, offs, truth)
    B = len(counts)
    packed = counts[counts <= 32]
    width = np.array([1 << int(np.ceil(np.log2(n))) for n in packed])
    out = {"gpu": gpu, "files": [os.path.basename(f) for f in args.files], "scenes": int(B),
           "pedestrians": int(offs[-1]), "scene_size_hist": np.bincount(counts).tolist(),
           "packed_scenes": int(len(packed)), "packed_lane_occupancy": float(packed.sum() / width.sum()),
           "cta_scenes": int(B - len(packed))}

    sims = {"sf": (socialforce, sweep.SF_DEFAULT, 0.5), "orca": (orca, sweep.ORCA_DEFAULT, 0.5)}
    for name, (mod, center, spread) in sims.items():
        res = {}
        for P in args.P:
            g = grid(P, center, spread)
            t = device_time(lambda: mod.sweep(prepared, g), reps=3 if P < 100 else 1, warm=lambda: mod.sweep(prepared, g[:1]))
            res["sweep_P%d" % P] = {"seconds": t, "scene_simulations_per_s": B * P / t, "settings_per_s": P / t}

        g = grid(args.loop, center, spread)
        truth_np = truth

        def loop():
            for prm in g:
                if mod is socialforce:
                    pos = socialforce.simulate_batch(state, offs, prm).cpu().numpy()
                else:
                    pos = orca.simulate_batch(state[:, :2], state[:, 2:4], state[:, 4:], speeds, offs, prm)
                    pos = pos.cpu().numpy().astype(np.float64)
                prim = pos[:, offs[:-1]].transpose(1, 0, 2)                # [B, 12, 2]
                d = np.sqrt(((truth_np - prim) ** 2).sum(-1))
                d.mean(axis=1), d[:, -1]
        loop()
        t0 = time.perf_counter()
        loop()
        t = time.perf_counter() - t0
        res["loop_simulate_batch_numpy"] = {"settings": len(g), "seconds": t, "scene_simulations_per_s": B * len(g) / t,
                                            "settings_per_s": len(g) / t}

        from oracle import classical_oracle as C
        from oracle.build_c import orca_simulate
        pick = np.random.RandomState(0).choice(B, size=min(args.cpu, B), replace=False)
        t0 = time.perf_counter()
        for b in pick:
            s, e = offs[b], offs[b + 1]
            if mod is socialforce:
                C.sf_simulate(state[s:e], tau=center[0], v0=center[1], sigma=center[2])
            else:
                orca_simulate(state[s:e, :2], state[s:e, 2:4], state[s:e, 4:], speeds[s:e], neighbor_dist=center[0],
                              time_horizon=center[1], radius=center[2])
        t = time.perf_counter() - t0
        res["cpu_restatement"] = {"scenes": len(pick), "seconds": t, "scene_simulations_per_s": len(pick) / t}
        out[name] = res
        print(json.dumps({name: res}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
