"""Generate tests/golden/train_golden.npz from the UNMODIFIED reference (build container).

    python -m oracle.make_train_golden

What Trainer.train_batch computes (trajnetbaselines/lstm/trainer.py:252-263): teacher-forced
LSTM.forward, PredictionLoss on the last 12 outputs x batch_size, backward.  Stored: the loss and
the parameter gradients (small tensors in full; large ones as sum / |sum| / 2000 seeded samples).
TEST INFRASTRUCTURE.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O          # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from oracle.make_golden import build_reference_model  # noqa: E402

# (name, kind, scenes, peds, ragged, nan_tracks, data seed, weight seed)
TRAIN_CASES = [
    ("train_vanilla", "vanilla", 5, 6, True, True, 31, 11),
    ("train_directional", "directional", 6, 8, True, True, 32, 12),
    ("train_occupancy", "occupancy", 4, 7, False, False, 33, 13),
    # social pooling: the hidden-state scatter couples the tracks of a scene (SURVEY 8a/A12)
    ("train_social_small", "social_small", 5, 6, True, True, 34, 14),
    ("train_social", "social", 4, 7, False, True, 35, 15),
]
FULL_LIMIT = 20000
N_SAMPLES = 2000


def summarize(name, grad, out):
    g = np.asarray(grad, dtype=np.float32)
    if g.size <= FULL_LIMIT:
        out[name + "/full"] = g
    else:
        idx = np.random.RandomState(12345).randint(0, g.size, size=N_SAMPLES)
        out[name + "/samples"] = g.reshape(-1)[idx]
        out[name + "/sum"] = np.array([g.sum(dtype=np.float64), np.abs(g).sum(dtype=np.float64)])


def check_summary(name, grad, golden, rtol, atol):
    """Compare a gradient tensor with its stored summary; returns max abs deviation."""
    g = np.asarray(grad, dtype=np.float32)
    if name + "/full" in golden:
        ref = golden[name + "/full"]
        assert ref.shape == g.shape, name
        dev = float(np.abs(g - ref).max())
        assert np.allclose(g, ref, rtol=rtol, atol=atol), (name, dev)
        return dev
    idx = np.random.RandomState(12345).randint(0, g.size, size=N_SAMPLES)
    ref = golden[name + "/samples"]
    dev = float(np.abs(g.reshape(-1)[idx] - ref).max())
    assert np.allclose(g.reshape(-1)[idx], ref, rtol=rtol, atol=atol), (name, dev)
    s = golden[name + "/sum"]
    assert abs(g.sum(dtype=np.float64) - s[0]) <= rtol * s[1] + atol * 10, name
    assert abs(np.abs(g).sum(dtype=np.float64) - s[1]) <= rtol * s[1] + atol * 10, name
    return dev


def rel_to_max(name, grad, golden):
    """max |grad - reference| / max |reference| over the stored entries of a gradient tensor."""
    g = np.asarray(grad, dtype=np.float32)
    if name + "/full" in golden:
        ref = golden[name + "/full"]
        assert ref.shape == g.shape, name
        got = g
    else:
        idx = np.random.RandomState(12345).randint(0, g.size, size=N_SAMPLES)
        ref = golden[name + "/samples"]
        got = g.reshape(-1)[idx]
    return float(np.abs(got - ref).max()) / max(float(np.abs(ref).max()), 1e-12)


def main():
    import_reference()
    from trajnetbaselines.lstm import PredictionLoss
    out = {}
    for name, kind, B, N, ragged, nan_tracks, dseed, wseed in TRAIN_CASES:
        xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
        W = O.random_weights(kind, seed=wseed)
        model = build_reference_model(kind, W)
        model.train()
        scene = torch.from_numpy(xy)
        batch_split = torch.from_numpy(bs)
        observed = scene[0:9].clone()
        prediction_truth = scene[9:-1].clone()
        targets = scene[9:21] - scene[8:20]
        rel_outputs, outputs = model(observed, torch.zeros(xy.shape[1], 2), batch_split, prediction_truth)
        loss = PredictionLoss()(rel_outputs[-12:], targets, batch_split) * B
        model.zero_grad()
        loss.backward()
        out[name + "/loss"] = np.array([loss.item()], dtype=np.float64)
        for pname, p in model.named_parameters():
            if p.grad is not None:
                summarize(name + "/" + pname, p.grad.numpy(), out)
        print(name, "loss %.6f" % loss.item(), "params with grad:", sum(p.grad is not None for p in model.parameters()))
    path = os.path.join(ROOT, "tests", "golden", "train_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
