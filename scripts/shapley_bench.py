"""Time the Shapley attribution (lstm.shapley.shapley) on bench.py's batch (256 scenes x 20 tracks, 9 + 12, H = 128).

For D-LSTM (directional grid, one_layer), S-LSTM (social grid, two_layer 1024, n = 16, latent 16) and nn_lstm (the
reference trainer's defaults: n = 4, pool width 256) at K = 4 and 8 players, median, min and max of `--reps` shapley
calls after one warm-up call, each ending in a device synchronise; instances per second; and the coalition forwards'
pedestrian-steps per second (rows of the instance batch x 19 steps, bench.py's count, over the call's median time).
Prints one JSON line per model and K with the card's name and power limit.
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
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM, NearestNeighborLSTM  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.shapley import instance_split, num_players, shapley  # noqa: E402

STEPS_PER_FORWARD = 19          # obs_length - 1 + n_predict - 1


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    gpu = q[0] if q else torch.cuda.get_device_name()
    xy, bs = O.synthetic_scenes(256, 20, n_frames=21, seed=0)
    split = torch.from_numpy(bs)
    obs = torch.from_numpy(xy[:9].copy()).cuda()
    truth = torch.from_numpy(xy[9:21, bs[:-1]].transpose(1, 0, 2).astype(np.float64)).cuda()
    sizes = np.diff(bs)
    for name, kind in (("D-LSTM", "directional"), ("S-LSTM", "social"), ("nn_lstm", "nn_lstm")):
        pool = NearestNeighborLSTM(**O.NN_LSTM_SPECS[kind]) if kind == "nn_lstm" else GridBasedPooling(**O.MODEL_SPECS[kind])
        model = LSTM(pool=pool)
        model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=1).items()})
        model.cuda().eval()
        for players in (4, 8):
            K = num_players(sizes, players)
            instances = int((1 << K).sum())
            rows = int(instance_split(sizes, K)[-1])
            ms = _times(lambda: shapley(model, obs, truth, split, players=players), args.reps)
            med = float(np.median(ms))
            print(json.dumps({"gpu": gpu, "model": name, "scenes": 256, "tracks": int(bs[-1]), "players": players,
                              "instances": instances, "instance_rows": rows,
                              "shapley": {"median_ms": round(med, 3), "min_ms": round(float(ms.min()), 3),
                                          "max_ms": round(float(ms.max()), 3)},
                              "instances_per_s": round(instances / (med * 1e-3)),
                              "ped_steps_per_s": round(rows * STEPS_PER_FORWARD / (med * 1e-3))}))


if __name__ == "__main__":
    main()
