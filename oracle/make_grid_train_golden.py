"""Generate tests/golden/grid_train_golden.npz from the UNMODIFIED reference (build container).

    python -m oracle.make_grid_train_golden

Training-step gradients of vanilla / occupancy / directional LSTMs in the configurations the reference
trainer reaches through its options and the CUDA backward indexes differently: `--front`, `--n`,
`--pool_dim` up to the 1024 limit and not a multiple of 4, `--coordinate-embedding-dim`, `--loss L2`,
`--col_wt`, a 2-frame observation (`--obs_dropout`), `--pred_length 1` (no decoder step), and a loss that
reaches every track.  Same step and storage as oracle/make_train_golden.py: Trainer.train_batch
(trainer.py:252-263), the criterion on the last pred_length outputs x batch size.  The grid embedding's
biases are +-3 (random_weights(relu_bias=3)), so no ReLU pre-activation sits near 0.  The collision cases
use col_distance = 1 m, so the random-walk scenes collide.
TEST INFRASTRUCTURE: tests/test_grid_backward.py pins tests/torch_ref.py to this file on the CPU.
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
# (name, kind, embedding dim, (scenes, max peds), obs_length, pred_length, loss, col_wt, col_distance,
#  data seed, weight seed); every scene set is ragged with entering / leaving neighbours (NaN frames)
GRID_TRAIN_CASES = [
    ("occ_col", "occupancy", 64, (5, 7), 9, 12, "pred", 2.0, 1.0, 61, 31),
    ("dir_front", "directional_front", 64, (5, 7), 9, 12, "pred", 0.0, 0.2, 62, 32),
    ("occ_front_n4", "occupancy_front_n4", 64, (5, 7), 9, 12, "l2", 0.0, 0.2, 63, 33),
    ("dir_n24", "directional_n24", 64, (5, 7), 9, 12, "pred", 0.0, 0.2, 64, 34),
    ("occ_p1024", "occupancy_p1024", 64, (5, 7), 9, 12, "l2", 2.0, 1.0, 65, 35),
    ("dir_p29", "directional_p29", 64, (5, 7), 9, 12, "pred", 0.0, 0.2, 66, 36),
    ("dir_e30", "directional", 30, (5, 7), 9, 12, "pred", 0.0, 0.2, 67, 37),
    ("vanilla_l2_col", "vanilla", 64, (5, 7), 9, 12, "l2", 2.0, 1.0, 68, 38),
    ("dir_obs2", "directional", 64, (5, 7), 2, 12, "pred", 0.0, 0.2, 69, 39),
    ("occ_obs5_pred1", "occupancy", 64, (5, 7), 5, 1, "pred", 0.0, 0.2, 70, 40),
    ("dir_all_tracks", "directional", 64, (5, 7), 9, 12, "all_tracks", 0.0, 0.2, 71, 41),
]


def all_tracks_loss(rel, positions):
    """sum over every track and step of fixed random weights x nan_to_num(rel): every present track receives
    gradient in all five outputs, absent steps none."""
    w = np.random.RandomState(7).uniform(-1.0, 1.0, size=tuple(rel.shape))
    return (torch.nan_to_num(rel) * torch.from_numpy(w).to(rel)).sum()


def case_inputs(case, data=None, data_seed=None):
    """(xy, batch_split, weights) of a GRID_TRAIN_CASES-shaped entry; `data` / `data_seed` override its
    scene set: (scenes, max peds, ragged)."""
    name, kind, E, shape, obs_length, pred_length = case[:6]
    dseed, wseed = case[9:11]
    B, N, ragged = data if data is not None else shape + (True,)
    xy, bs = O.synthetic_scenes(B, N, n_frames=obs_length + pred_length,
                                seed=dseed if data_seed is None else data_seed, ragged=ragged, nan_tracks=ragged)
    return xy, bs, O.random_weights(kind, seed=wseed, embedding_dim=E, relu_bias=RELU_BIAS)


def loss_args(case):
    """keyword arguments of tests/torch_ref.train_loss_and_grads for the case's criterion."""
    loss, col_wt, col_distance = case[6:9]
    return dict(loss=all_tracks_loss if loss == "all_tracks" else loss, col_wt=col_wt, col_distance=col_distance)


def main():
    torch.set_num_threads(1)
    import_reference()
    from trajnetbaselines.lstm import L2Loss, PredictionLoss
    out = {}
    for case in GRID_TRAIN_CASES:
        name, kind, E, _, obs_length, pred_length, loss_kind, col_wt, col_distance = case[:9]
        xy, bs, W = case_inputs(case)
        model = build_reference_model(kind, W, embedding_dim=E)
        model.train()
        scene = torch.from_numpy(xy)
        batch_split = torch.from_numpy(bs)
        B = len(bs) - 1
        observed = scene[:obs_length].clone()
        prediction_truth = scene[obs_length:-1].clone()
        targets = scene[obs_length:obs_length + pred_length] - scene[obs_length - 1:obs_length + pred_length - 1]
        rel_outputs, outputs = model(observed, torch.zeros(xy.shape[1], 2), batch_split, prediction_truth)
        outputs.retain_grad()
        if loss_kind == "all_tracks":
            loss = all_tracks_loss(rel_outputs, outputs)
        else:
            criterion = (PredictionLoss if loss_kind == "pred" else L2Loss)(col_wt=col_wt, col_distance=col_distance)
            primary_prediction = scene[-pred_length:].clone()
            primary_prediction[:, batch_split[:-1]] = outputs[-pred_length:, batch_split[:-1]]
            loss = criterion(rel_outputs[-pred_length:], targets, batch_split, primary_prediction) * B
        model.zero_grad()
        loss.backward()
        out[name + "/loss"] = np.array([loss.item()], dtype=np.float64)
        # d loss / d positions: non-zero only through the collision term (the scenes must collide)
        d_pos = outputs.grad if outputs.grad is not None else torch.zeros_like(outputs)
        out[name + "/positions_grad"] = d_pos.numpy().astype(np.float32)
        for pname, p in model.named_parameters():
            if p.grad is not None:
                summarize(name + "/" + pname, p.grad.numpy(), out)
        print(name, "loss %.6f" % loss.item())
    path = os.path.join(ROOT, "tests", "golden", "grid_train_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
