"""An external interaction module (lstm/external.py) against the fused path: the reference's HiddenStateMLPPooling run by
torch between the step's kernels, against this package's HiddenStateMLPPooling fused into them, same weights.

Workload: 256 scenes x 20 tracks, obs_length 9, pred_length 12, teacher-forced (the trainer's forward).  Timed, each
between CUDA events with a device synchronise on both sides, alternating the two models every round:
  * forward: LSTM.forward under torch.no_grad();
  * train step: forward, PredictionLoss, backward and an SGD step (the fused model trains through its own backward only
    for the grid pools, so the fused column is the no-grad forward only).
One JSON line per (path, measurement) with the median, min and max over --runs rounds, and the GPU's name and power limit.

    python scripts/custom_pool_bench.py [--scenes 256] [--tracks 20] [--runs 10] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle import lstm_oracle as O
from oracle.ref_shim import import_reference


def device_info():
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        limit = "unknown"
    return torch.cuda.get_device_name(0), limit


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end)


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--scenes", type=int, default=256)
    parser.add_argument("--tracks", type=int, default=20)
    parser.add_argument("--runs", type=int, default=10)
    parser.add_argument("--warmup", type=int, default=3)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("custom_pool_bench needs a CUDA device")
    import_reference()
    from trajnetbaselines.lstm.non_gridbased_pooling import HiddenStateMLPPooling as RefPool
    from trajnetplusplusbaselines_b200.lstm import LSTM, HiddenStateMLPPooling, PredictionLoss
    kw = dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256)
    torch.manual_seed(0)
    ext = LSTM(pool=RefPool(**kw))
    fused = LSTM(pool=HiddenStateMLPPooling(**kw))
    fused.load_state_dict(ext.state_dict())
    ext, fused = ext.cuda(), fused.cuda()
    xy, bs = O.synthetic_scenes(args.scenes, args.tracks, seed=1, nan_tracks=True, start_std=6.0)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    goals = torch.zeros(xy.shape[1], 2, device="cuda")
    obs, truth = scene[:9], scene[9:20]
    targets = scene[9:21] - scene[8:20]
    opt = torch.optim.SGD(ext.parameters(), lr=1e-4)
    loss_fn = PredictionLoss()

    def forward(model):
        def run():
            with torch.no_grad():
                model(obs, goals, split, truth.clone())
        return run

    def train_step():
        ext.train()
        rel, _ = ext(obs, goals, split, truth.clone())
        loss = loss_fn(rel[-12:], targets, split.cuda()) * args.scenes
        opt.zero_grad()
        loss.backward()
        opt.step()

    cases = [("external", "forward", forward(ext)), ("fused", "forward", forward(fused)),
             ("external", "train_step", train_step)]
    for _ in range(args.warmup):
        for _, _, fn in cases:
            fn()
    times = {(p, w): [] for p, w, _ in cases}
    for _ in range(args.runs):
        for p, w, fn in cases:
            times[(p, w)].append(timed(fn))
    gpu, limit = device_info()
    for (p, w), t in times.items():
        print(json.dumps({"path": p, "measure": w, "scenes": args.scenes, "tracks": args.tracks, "runs": args.runs,
                          "median_ms": round(statistics.median(t), 3), "min_ms": round(min(t), 3),
                          "max_ms": round(max(t), 3), "gpu": gpu, "power_limit": limit}))


if __name__ == "__main__":
    main()
