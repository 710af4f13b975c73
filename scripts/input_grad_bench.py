"""Cost of gradients wrt the observed trajectories (d observed) on bench.py's batch: 256 scenes x 20 tracks,
obs_length 9, pred_length 12, hidden_dim 128, for D-LSTM (directional) and S-LSTM (social).

Timed between CUDA events with a device synchronise on both sides; the median, min and max over --runs calls:
  * params:        teacher-forced forward, PredictionLoss on the primaries, backward into the parameters;
  * params_obs:    the same with observed.requires_grad_() (parameter gradients and d observed);
  * obs_frozen:    frozen parameters, d observed only;
  * pgd20:         20 iterations of an L-inf bounded PGD (eps 0.1 m, step 0.02 m) on the primaries' observed tracks
                   that maximises the collision loss of the free-running prediction (frozen parameters).
One JSON line per (model, measurement), with the GPU's name and power limit.

    python scripts/input_grad_bench.py [--runs 10] [--warmup 3]
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

SCENES, PEDS, OBS, PRED = 256, 20, 9, 12
MODELS = {"D-LSTM": "directional", "S-LSTM": "social"}


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
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM, PredictionLoss
    from trajnetplusplusbaselines_b200.lstm.loss import collision_loss
    gpu, limit = device_info()
    xy, bs = O.synthetic_scenes(SCENES, PEDS, n_frames=OBS + PRED, seed=100)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    prim = split[:-1].cuda()
    targets = scene[OBS:] - scene[OBS - 1:-1]
    criterion = PredictionLoss()
    for label, kind in MODELS.items():
        model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
        model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=1).items()})
        model = model.cuda()

        def train_step(obs_grad):
            observed = scene[:OBS].clone().requires_grad_(obs_grad)
            rel, _ = model(observed, None, split, scene[OBS:-1].clone())
            model.zero_grad()
            (criterion(rel[-PRED:], targets, split) * SCENES).backward()

        def pgd():
            base = scene[:OBS].clone()
            delta = torch.zeros_like(base)
            mask = torch.zeros_like(base)
            mask[:, prim] = 1.0
            for _ in range(20):
                d = delta.clone().requires_grad_()
                _, pos = model(base + d * mask, None, split, n_predict=PRED)
                loss = collision_loss(pos[-PRED:], bs.tolist())
                (g,) = torch.autograd.grad(loss, d)
                delta = (delta + 0.02 * g.sign() * mask).clamp(-0.1, 0.1)
            return delta

        cases = [("params", lambda: train_step(False)), ("params_obs", lambda: train_step(True))]
        for name, fn in cases + [("obs_frozen", None), ("pgd20", pgd)]:
            if name == "obs_frozen":
                model.requires_grad_(False)
                fn = lambda: train_step(True)     # noqa: E731
            for _ in range(args.warmup):
                fn()
            ms = [timed(fn) for _ in range(args.runs)]
            print(json.dumps({"model": label, "measure": name, "median_ms": round(statistics.median(ms), 3),
                              "min_ms": round(min(ms), 3), "max_ms": round(max(ms), 3), "runs": args.runs,
                              "scenes": SCENES, "tracks": SCENES * PEDS, "gpu": gpu, "power_limit": limit}))
            sys.stdout.flush()


if __name__ == "__main__":
    main()
