"""Time the relevance pass (lstm.explain.relevance) on bench.py's batch (256 scenes x 20 tracks, 9 + 12, H = 128).

For D-LSTM (directional grid, one_layer) and S-LSTM (social grid, two_layer 1024, n = 16, latent 16), median, min and
max of `--reps` calls of
  * the forward the pass rests on (the free-running forward with the per-step states kept);
  * one relevance call (that forward and tb2_lstm_relevance).
Each call ends in a device synchronise.  Prints one JSON line per model with the card's name and power limit.
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
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.explain import relevance  # noqa: E402


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
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    gpu = q[0] if q else torch.cuda.get_device_name()
    xy, bs = O.synthetic_scenes(256, 20, n_frames=21, seed=0)
    split = torch.from_numpy(bs)
    obs = torch.from_numpy(xy[:9].copy()).cuda()
    for name, kind in (("D-LSTM", "directional"), ("S-LSTM", "social")):
        model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
        model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=1).items()})
        model.cuda().eval()

        def forward():
            with torch.no_grad():
                model._forward_nograd(obs, split, None, 12, want_states=True)
        fwd = _times(forward, args.reps)
        rel = _times(lambda: relevance(model, obs, split, 12), args.reps)
        print(json.dumps({"gpu": gpu, "model": name, "scenes": 256, "tracks": int(bs[-1]), "forward": _stat(fwd),
                          "relevance": _stat(rel)}))


if __name__ == "__main__":
    main()
