"""Time the Social-NCE term (lstm/contrast.py) inside Trainer.train_batch.

For D-LSTM (directional grid, one_layer) and S-LSTM (social grid, two_layer 1024, n = 16, latent 16), H = 128, at 8 and
256 scenes x 20 tracks (9 + 12 frames, seeded synthetic scenes), the median, min and max of `--reps` train_batch calls
after `--warmup` calls, each ending in a device synchronise: the clean step (contrast_weight = 0) and the step with the
term (contrast_weight = 1, horizon 4).  The hidden-state plumbing alone: forward + backward of the task loss through
`model(...)` against the same through `sequence_with_hidden` with a zero-weighted term on the query step's hidden
states (the dense d hidden, its scan for active rows and the copy of the states).  Then, in a separate profiled run
of the same steps, the device time of the term's two launches (snce_forward_kernel, snce_backward_kernel) per step and their share of the step's median time.
Last, the same term written in torch fp32 on the device (padded to the batch's largest scene, masked, autograd for the
gradients): the median time of its forward + backward against the same of the module's, and the two losses.
Prints one JSON line per model and batch size with the card's name and power limit.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O  # noqa: E402
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.contrast import SocialNCE  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.trainer import Trainer  # noqa: E402
from trajnetplusplusbaselines_b200.lstm.training import sequence_with_hidden  # noqa: E402

OBS, PRED, PEDS = 9, 12, 20


def _times(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return np.array(out)


def _stats(ms):
    return {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(float(ms.min()), 3),
            "max_ms": round(float(ms.max()), 3)}


def torch_term(nce, scene, hidden, idx, live, prim, eps):
    """The term of SocialNCE in torch fp32: samples padded to [B, horizon, 1 + 8 (n_max - 1)], masked."""
    f0, hz = OBS - 1, nce.horizon
    ang = torch.arange(8, device=scene.device, dtype=torch.float32) * (math.pi / 4)
    ring = nce.rho * torch.stack([torch.cos(ang), torch.sin(ang)], dim=1)
    P = scene[f0 + 1:f0 + 1 + hz][:, idx]                                   # [hz, B, n_max, 2]
    ok = live[None] & torch.isfinite(P).all(-1)                             # [hz, B, n_max]
    rel = P - scene[f0, prim][None, :, None]
    B, n_max = idx.shape
    neg = (rel[:, :, 1:, None, :] + ring).reshape(hz, B, 8 * (n_max - 1), 2)
    samples = torch.cat([rel[:, :, :1], neg], 2).transpose(0, 1) + nce.sigma * eps      # [B, hz, NS, 2]
    mask = torch.cat([ok[:, :, :1], ok[:, :, 1:, None].expand(-1, -1, -1, 8).reshape(hz, B, -1)], 2).transpose(0, 1)
    samples = torch.where(mask[..., None], samples, torch.zeros_like(samples))
    d = torch.arange(1, hz + 1, device=scene.device, dtype=torch.float32)[None, :, None, None].expand(B, hz,
                                                                                                   samples.shape[2], 1)
    keys = F.normalize(nce.event_encoder(torch.cat([samples, d], -1)), dim=-1)
    q = F.normalize(nce.head(hidden[prim]), dim=-1)
    logits = torch.einsum('bhne,be->bhn', keys, q) / nce.temperature
    logits = logits.masked_fill(~mask, float('-inf'))
    pair = mask[..., 0]
    term = torch.where(pair, torch.logsumexp(logits, -1) - logits[..., 0], torch.zeros_like(logits[..., 0]))
    return term.sum() / pair.sum().clamp(min=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    gpu = q[0] if q else torch.cuda.get_device_name()
    for name, kind in (("D-LSTM", "directional"), ("S-LSTM", "social")):
        W = O.random_weights(kind, seed=1)
        for B in (8, 256):
            xy, bs = O.synthetic_scenes(B, PEDS, n_frames=OBS + PRED, seed=100)
            scene = torch.from_numpy(xy).cuda()
            split = torch.from_numpy(bs)
            goals = torch.zeros(xy.shape[1], 2, device="cuda")
            steps = {}
            for weight in (0.0, 1.0):
                model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
                model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
                torch.manual_seed(0)
                trainer = Trainer(model.cuda(), device=torch.device("cuda"), batch_size=B, augment=False,
                                  contrast_weight=weight)
                steps[weight] = (trainer, _times(lambda: trainer.train_batch(scene, goals, split), args.reps,
                                                 args.warmup))
            trainer = steps[1.0][0]
            model = trainer.model

            def task(rel):
                targets = scene[OBS:OBS + PRED] - scene[OBS - 1:OBS + PRED - 1]
                return trainer.criterion(rel[-PRED:], targets, split) * B

            def plain():
                rel, _ = model(scene[:OBS], goals, split, scene[OBS:-1].clone())
                model.zero_grad()
                task(rel).backward()

            def with_hidden():
                rel, _, hid = sequence_with_hidden(model, scene[:OBS], split, scene[OBS:-1].clone(), None)
                model.zero_grad()
                (task(rel) + 0.0 * hid[OBS - 2].sum()).backward()
            fb_plain = _times(plain, args.reps, args.warmup)
            fb_hidden = _times(with_hidden, args.reps, args.warmup)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    trainer.train_batch(scene, goals, split)
                torch.cuda.synchronize()
            kern_us = sum(e.device_time_total for e in prof.key_averages() if "snce_" in e.key) / 10
            # the term alone: the module against torch fp32
            nce = trainer.contrast
            hidden = torch.randn(xy.shape[1], 128, device="cuda", requires_grad=True)
            n_max = int(np.diff(bs).max())
            j = torch.arange(n_max)
            rows = torch.from_numpy(bs[:-1])[:, None] + j
            idx = torch.minimum(rows, torch.from_numpy(bs[1:])[:, None] - 1).cuda()
            live = (j[None] < torch.from_numpy(np.diff(bs))[:, None]).cuda()
            prim = torch.from_numpy(bs[:-1]).cuda()
            eps = torch.randn(nce.eps_shape(bs), device="cuda")
            nce.fixed_eps = eps
            fused = _times(lambda: nce(scene, hidden, split, OBS).backward(), args.reps, args.warmup)
            unfused = _times(lambda: torch_term(nce, scene, hidden, idx, live, prim, eps).backward(), args.reps,
                             args.warmup)
            with torch.no_grad():
                l_fused = float(nce(scene, hidden, split, OBS))
                l_torch = float(torch_term(nce, scene, hidden, idx, live, prim, eps))
            nce.fixed_eps = None
            clean_ms, nce_ms = float(np.median(steps[0.0][1])), float(np.median(steps[1.0][1]))
            print(json.dumps({"gpu": gpu, "model": name, "scenes": B, "tracks": int(bs[-1]), "horizon": nce.horizon,
                              "train_batch_clean": _stats(steps[0.0][1]), "train_batch_nce": _stats(steps[1.0][1]),
                              "nce_added_ms": round(nce_ms - clean_ms, 3),
                              "fwd_bwd_model": _stats(fb_plain), "fwd_bwd_sequence_with_hidden": _stats(fb_hidden),
                              "nce_kernels_ms_per_step": round(kern_us * 1e-3, 4),
                              "nce_kernels_share_of_step": round(kern_us * 1e-3 / nce_ms, 4),
                              "term_fwd_bwd_module": _stats(fused), "term_fwd_bwd_torch_fp32": _stats(unfused),
                              "loss_module": l_fused, "loss_torch_fp32": l_torch}))


if __name__ == "__main__":
    main()
