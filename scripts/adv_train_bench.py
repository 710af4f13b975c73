"""Time adversarial training against the collision attack, and what the inputs-only rollout backward saves.

For D-LSTM (directional grid) and S-LSTM (social grid) at H = 128, on two batches of seeded synthetic scenes (20 tracks
each, 9 + 12 frames): the CLI's --batch_size 8 (8 scenes) and bench.py's 256 scenes. Median, min and max of `--reps`
calls of
  * a clean training step (Trainer.train_batch, adv_eps = 0: forward, PredictionLoss, backward, Adam);
  * an adversarial training step at K = 1, 5, 10 PGD iterations (adv_eps = 0.1, adv_wt = 0.5);
  * a free-running forward + the rollout backward of a fixed linear loss on the positions, with the parameters as
    inputs of the graph (every parameter gradient) and with parameters=False (d observed alone).
Each call ends in a device synchronise. Prints one JSON line with the card's name and power limit.
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
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM, differentiable_rollout  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.trainer import Trainer  # noqa: E402


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


def _model(kind):
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=1).items()})
    return model.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"gpu": q[0] if q else torch.cuda.get_device_name()}
    for scenes in (8, 256):
        xy, bs = O.synthetic_scenes(scenes, 20, n_frames=21, seed=0)
        batch = torch.from_numpy(xy).cuda()
        split = torch.from_numpy(bs)
        w = torch.randn(21, xy.shape[1], 2, device="cuda")
        for name, kind in (("D-LSTM", "directional"), ("S-LSTM", "social_default")):
            out = res.setdefault("%s_%dx20" % (name, scenes), {})
            model = _model(kind)
            goals = torch.zeros(xy.shape[1], 2, device="cuda")
            for label, kw in (("train_step_clean", {}),) + tuple(
                    ("train_step_adv_k%d" % k, dict(adv_eps=0.1, adv_steps=k, adv_wt=0.5)) for k in (1, 5, 10)):
                trainer = Trainer(model, batch_size=scenes, augment=False, **kw)
                model.train()
                out[label] = _stat(_times(lambda: trainer.train_batch(batch, goals, split), args.reps))
            for label, parameters in (("rollout_fwd_bwd_params", True), ("rollout_fwd_bwd_inputs_only", False)):
                def run():
                    obs = batch[:9].clone().requires_grad_()
                    _, pos = differentiable_rollout(model, obs, split, 12, parameters=parameters)
                    (torch.nan_to_num(pos) * w[-pos.shape[0]:]).sum().backward()
                out[label] = _stat(_times(run, args.reps))
                model.zero_grad(set_to_none=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
