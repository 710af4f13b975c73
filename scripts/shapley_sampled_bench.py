"""Time the sampled Shapley attribution (lstm.shapley.sampled_shapley) on bench.py's batch (256 scenes x 20 tracks,
9 + 12, H = 128) and measure its accuracy against the exact values.

For D-LSTM (directional grid, one_layer), S-LSTM (social grid, two_layer 1024, n = 16, latent 16) and nn_lstm (the
reference trainer's defaults: n = 4, pool width 256), as in scripts/shapley_bench.py:

  cost      players=None (K = 19) at P = 64, 256 and 1024: median, min and max of `--reps` calls after one warm-up call,
            each ending in a device synchronise; instances per second; the instance forwards' pedestrian-steps per
            second (rows of the instance batch x 19 steps, bench.py's count, over the median call); and, from one more
            call under tb2_profile_*, the CUDA-event time of the expansion kernels (shapley_sample_players /
            shapley_sample_expand), the value kernels (shapley_sample_score / shapley_sample_reduce) and every other
            library kernel (the forward).
  accuracy  players=8 at P = 64, 256 and 1024 against one shapley(players=8) call: the mean |phi - phi_exact| and the
            mean se over every (scene, player) of the ADE and FDE attributions, with the time of each call (one call
            each, after a warm-up call of shapley()).

Prints one JSON line per case with the card's name and power limit.
"""
import argparse
import ctypes
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
from trajnetplusplusbaselines_b200 import _lib  # noqa: E402
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM, NearestNeighborLSTM  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.shapley import (num_players, sampled_instance_counts,  # noqa: E402
                                                        sampled_instance_split, sampled_shapley, shapley)

STEPS_PER_FORWARD = 19          # obs_length - 1 + n_predict - 1
EXPAND = ("shapley_sample_players", "shapley_sample_expand")
VALUES = ("shapley_sample_score", "shapley_sample_reduce")


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def _profile(fn):
    """{"expand_ms", "forward_ms", "values_ms"}: CUDA-event kernel time of one call by kernel group."""
    lib = _lib.load()
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 16)
    lib.tb2_profile_begin()
    fn()
    _lib.check(lib.tb2_profile_end(buf, len(buf)))
    prof = json.loads(buf.value.decode())
    group = lambda names: sum(v["total_ms"] for k, v in prof.items() if k in names)
    rest = sum(v["total_ms"] for k, v in prof.items() if k not in EXPAND + VALUES)
    return {"expand_ms": round(group(EXPAND), 3), "forward_ms": round(rest, 3), "values_ms": round(group(VALUES), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    gpu = q[0] if q else torch.cuda.get_device_name()
    xy, bs = O.synthetic_scenes(256, 20, n_frames=21, seed=0)
    split = torch.from_numpy(bs)
    obs = torch.from_numpy(xy[:9].copy()).cuda()
    truth = torch.from_numpy(xy[9:21, bs[:-1]].transpose(1, 0, 2).astype(np.float64)).cuda()
    sizes = np.diff(bs)
    base = {"gpu": gpu, "scenes": 256, "tracks": int(bs[-1])}
    for name, kind in (("D-LSTM", "directional"), ("S-LSTM", "social"), ("nn_lstm", "nn_lstm")):
        pool = NearestNeighborLSTM(**O.NN_LSTM_SPECS[kind]) if kind == "nn_lstm" else GridBasedPooling(**O.MODEL_SPECS[kind])
        model = LSTM(pool=pool)
        model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=1).items()})
        model.cuda().eval()
        sampled_shapley(model, obs, truth, split, players=None, permutations=64)
        for P in (64, 256, 1024):
            K = num_players(sizes, 6143)
            instances = int(sampled_instance_counts(K, P).sum())
            rows = int(sampled_instance_split(sizes, K, P)[-1])
            call = lambda: sampled_shapley(model, obs, truth, split, players=None, permutations=P)
            ms = np.array([_timed(call)[1] for _ in range(args.reps)])
            med = float(np.median(ms))
            print(json.dumps(dict(base, model=name, case="cost", players="all", K=int(K.max()), permutations=P,
                                  instances=instances, instance_rows=rows,
                                  sampled_shapley={"median_ms": round(med, 3), "min_ms": round(float(ms.min()), 3),
                                                   "max_ms": round(float(ms.max()), 3)},
                                  instances_per_s=round(instances / (med * 1e-3)),
                                  ped_steps_per_s=round(rows * STEPS_PER_FORWARD / (med * 1e-3)),
                                  kernels=_profile(call))), flush=True)
        shapley(model, obs, truth, split, players=8)
        ex, ex_ms = _timed(lambda: shapley(model, obs, truth, split, players=8))
        for P in (64, 256, 1024):
            sa, sa_ms = _timed(lambda: sampled_shapley(model, obs, truth, split, players=8, permutations=P))
            err = {m: float(torch.mean(torch.abs(getattr(sa, "phi_" + m) - getattr(ex, "phi_" + m)[:, :8])))
                   for m in ("ade", "fde")}
            se = {m: float(torch.mean(getattr(sa, "se_" + m))) for m in ("ade", "fde")}
            print(json.dumps(dict(base, model=name, case="accuracy", players=8, permutations=P,
                                  mean_abs_err_ade=float("%.4g" % err["ade"]), mean_se_ade=float("%.4g" % se["ade"]),
                                  mean_abs_err_fde=float("%.4g" % err["fde"]), mean_se_fde=float("%.4g" % se["fde"]),
                                  exact_ms=round(ex_ms, 3), sampled_ms=round(sa_ms, 3))), flush=True)


if __name__ == "__main__":
    main()
