"""Generate tests/golden/social_train_golden.npz from the UNMODIFIED reference (build container).

    python -m oracle.make_social_train_golden

Training-step gradients of Social-LSTM in each pooling configuration the CUDA library dispatches to
different kernels (one_layer / two_layer embedding, latent_dim 4 / 16 / 32, first-layer widths that
are and are not multiples of 32, a 2-frame observation), at tiny shapes.  Same step and storage as
oracle/make_train_golden.py.  The grid embedding's biases are +-3 (random_weights(relu_bias=3)), so no
ReLU pre-activation sits near 0 and the fixture does not depend on how a ReLU kink rounds.
TEST INFRASTRUCTURE: tests/test_social_backward.py pins tests/torch_ref.py to this file on the CPU.
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
from oracle.make_train_golden import summarize  # noqa: E402

RELU_BIAS = 3.0
# (name, kind, scenes, peds, ragged, nan_tracks, obs_length, pred_length, data seed, weight seed)
SOCIAL_TRAIN_CASES = [
    ("social_default", "social_default", 5, 7, True, True, 9, 12, 141, 21),
    ("social_c4", "social_c4", 5, 7, True, True, 9, 12, 42, 22),
    ("social_c32", "social_c32", 5, 7, True, True, 9, 12, 43, 23),
    ("social_d96", "social_d96", 5, 7, True, True, 9, 12, 44, 24),
    ("social_d200", "social_d200", 5, 7, True, True, 9, 12, 45, 25),
    ("social_baseline", "social", 4, 7, False, True, 9, 12, 46, 35),
    ("social_default_short", "social_default", 5, 7, True, True, 2, 3, 49, 27),
]


def case_inputs(case):
    """(xy, batch_split, weights) of a SOCIAL_TRAIN_CASES entry."""
    name, kind, B, N, ragged, nan_tracks, obs_length, pred_length, dseed, wseed = case
    xy, bs = O.synthetic_scenes(B, N, n_frames=obs_length + pred_length, seed=dseed, ragged=ragged,
                                nan_tracks=nan_tracks)
    return xy, bs, O.random_weights(kind, seed=wseed, relu_bias=RELU_BIAS)


def main():
    # the reference writes the grid with one index_put_ whose duplicate indices (several neighbours in one cell)
    # are written in ascending neighbour order only when the CPU kernel runs on one thread; on several threads the
    # surviving writer of a cell can differ from run to run
    torch.set_num_threads(1)
    import_reference()
    from trajnetbaselines.lstm import PredictionLoss
    out = {}
    for case in SOCIAL_TRAIN_CASES:
        name, kind, B, _, _, _, obs_length, pred_length = case[:8]
        xy, bs, W = case_inputs(case)
        model = build_reference_model(kind, W)
        model.train()
        scene = torch.from_numpy(xy)
        batch_split = torch.from_numpy(bs)
        observed = scene[:obs_length].clone()
        prediction_truth = scene[obs_length:-1].clone()
        targets = scene[obs_length:obs_length + pred_length] - scene[obs_length - 1:obs_length + pred_length - 1]
        rel_outputs, _ = model(observed, torch.zeros(xy.shape[1], 2), batch_split, prediction_truth)
        loss = PredictionLoss()(rel_outputs[-pred_length:], targets, batch_split) * B
        model.zero_grad()
        loss.backward()
        out[name + "/loss"] = np.array([loss.item()], dtype=np.float64)
        for pname, p in model.named_parameters():
            if p.grad is not None:
                summarize(name + "/" + pname, p.grad.numpy(), out)
        print(name, "loss %.6f" % loss.item())
    path = os.path.join(ROOT, "tests", "golden", "social_train_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
