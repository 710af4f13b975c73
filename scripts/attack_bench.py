"""Time the rollout backward and the collision attack on bench.py's batch (256 scenes x 20 tracks, H = 128).

For D-LSTM (directional grid) and S-LSTM (social grid), median, min and max of `--reps` calls of
  * a free-running forward + the backward of a fixed linear loss on the positions through LSTM.forward's graph
    (tb2_lstm_sequence_backward, decoder inputs detached, d observed on);
  * forward + the rollout backward of lstm.differentiable_rollout (tb2_lstm_rollout_backward);
  * one PGD iteration of attack.collision_attack: (median of `--steps` + 1 steps - median of 1 step) / `--steps`.
Each call ends in a device synchronise.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O  # noqa: E402
from trajnetplusplusbaselines_b200.attack import collision_attack  # noqa: E402
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM, differentiable_rollout  # noqa: E402


def _times(fn, reps):
    """Milliseconds of `reps` calls after one warm-up call, each ending in a device synchronise."""
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return np.array(out)


def _stat(ms):
    return {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(float(ms.min()), 3),
            "max_ms": round(float(ms.max()), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"gpu": q[0] if q else torch.cuda.get_device_name()}
    xy, bs = O.synthetic_scenes(256, 20, n_frames=21, seed=0)
    xys = [xy[:, bs[i]:bs[i + 1]].astype(np.float64) for i in range(256)]
    for name, kind in (("D-LSTM", "directional"), ("S-LSTM", "social_default")):
        model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
        model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=1).items()})
        model.cuda().requires_grad_(False)
        split = torch.from_numpy(bs)
        w = torch.randn(21, xy.shape[1], 2, device="cuda")

        def run(fn):
            obs = torch.from_numpy(xy[:9].copy()).cuda().requires_grad_()
            _, pos = fn(obs)
            (torch.nan_to_num(pos) * w[-pos.shape[0]:]).sum().backward()
        detached = _times(lambda: run(lambda o: model(o, None, split, n_predict=12)), args.reps)
        rollout = _times(lambda: run(lambda o: differentiable_rollout(model, o, split, 12)), args.reps)
        n = max(3, args.reps // 3)
        one = _times(lambda: collision_attack(model, xys, eps=0.1, steps=1, chunk=256), n)
        many = _times(lambda: collision_attack(model, xys, eps=0.1, steps=args.steps + 1, chunk=256), n)
        res[name] = {"fwd_bwd_detached": _stat(detached), "fwd_bwd_rollout": _stat(rollout),
                     "pgd_iteration_ms": round(float(np.median(many) - np.median(one)) / args.steps, 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
