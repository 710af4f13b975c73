"""Generate tests/golden/input_grad_golden.npz from the UNMODIFIED reference (build container).

    python -m oracle.make_input_grad_golden

d loss / d observed of the reference's LSTM.forward (lstm/lstm.py:170-264) in float64 on the CPU, for a loss on
rel_pred_scene plus one on pred_scene (fixed random weights on every track and step, NaN entries weighted 0).

The reference cannot run this as it stands: `copy.deepcopy(list(chain(observed[-1:], prediction_truth)))`
(lstm.py:235) raises "Only Tensors created explicitly by the user (graph leaves) support the deepcopy protocol" as soon
as `observed` requires grad.  Its `lstm` module's `copy.deepcopy` is therefore shimmed, for this script only, to
`detach().clone()` of each tensor of the list: what deepcopy does to a leaf, a new tensor with no path back to
`observed`.  Nothing else of the reference is touched.

Cases: vanilla, occupancy, directional, social one_layer and two_layer; teacher-forced and free-running; obs_length 9
and 2; ragged scenes with entering / leaving tracks (NaN frames).  The pool embeddings' biases are +-3
(random_weights(relu_bias=3)), so no pool ReLU pre-activation sits near 0.
TEST INFRASTRUCTURE: tests/test_input_grad.py pins tests/input_grad_ref.py to this file on the CPU.
"""
import copy
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O          # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

PRED_LENGTH = 12
# (name, kind, teacher forcing, obs_length, data seed, weight seed); 4 ragged scenes of up to 6 tracks
INPUT_GRAD_CASES = [
    ("vanilla_tf", "vanilla", True, 9, 81, 51),
    ("vanilla_free_obs2", "vanilla", False, 2, 82, 52),
    ("occ_tf", "occupancy", True, 9, 83, 53),
    ("occ_free", "occupancy", False, 9, 84, 54),
    ("dir_tf", "directional", True, 9, 85, 55),
    ("dir_free", "directional", False, 9, 86, 56),
    ("dir_tf_obs2", "directional", True, 2, 87, 57),
    ("social_one_tf", "social_default", True, 9, 88, 58),
    ("social_one_free_obs2", "social_default", False, 2, 89, 59),
    ("social_two_tf", "social_small", True, 9, 90, 60),
    ("social_two_free", "social_small", False, 9, 91, 61),
]


def case_inputs(case):
    """(xy fp32 [obs_length + PRED_LENGTH, M, 2], batch_split, weights) of an INPUT_GRAD_CASES entry."""
    _, kind, _, obs_length, dseed, wseed = case
    xy, bs = O.synthetic_scenes(4, 6, n_frames=obs_length + PRED_LENGTH, seed=dseed, ragged=True, nan_tracks=True)
    return xy, bs, O.random_weights(kind, seed=wseed, relu_bias=3.0)


def loss_weights(S_pos, S, M):
    """Fixed weights of the loss sum(w_rel . nan_to_num(rel)) + sum(w_pos . nan_to_num(pred))."""
    rs = np.random.RandomState(23)
    return rs.uniform(-1, 1, size=(S, M, 5)), rs.uniform(-1, 1, size=(S_pos, M, 2))


def _leaf_deepcopy(x):
    return [t.detach().clone() if torch.is_tensor(t) else copy.deepcopy(t) for t in x]


def main():
    torch.set_num_threads(1)
    import_reference()
    from trajnetbaselines.lstm import LSTM, GridBasedPooling
    from trajnetbaselines.lstm import lstm as ref_lstm
    saved = ref_lstm.copy
    ref_lstm.copy = types.SimpleNamespace(deepcopy=_leaf_deepcopy)
    old_dtype = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    out = {}
    try:
        for case in INPUT_GRAD_CASES:
            name, kind, teacher, obs_length = case[:4]
            xy, bs, W = case_inputs(case)
            spec = O.MODEL_SPECS[kind]
            model = LSTM(pool=GridBasedPooling(**spec) if spec is not None else None)
            model.load_state_dict({k: torch.from_numpy(v.copy()).double() for k, v in W.items()}, strict=True)
            model = model.double().train()
            scene = torch.from_numpy(xy).double()
            observed = scene[:obs_length].clone().requires_grad_()
            kw = dict(prediction_truth=scene[obs_length:-1].clone()) if teacher else dict(n_predict=PRED_LENGTH)
            rel, pred = model(observed, torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), **kw)
            wr, wp = loss_weights(pred.shape[0], rel.shape[0], xy.shape[1])
            loss = (torch.nan_to_num(rel) * torch.from_numpy(wr)).sum() + \
                (torch.nan_to_num(pred) * torch.from_numpy(wp)).sum()
            loss.backward()
            out[name + "/d_observed"] = observed.grad.numpy()
            out[name + "/loss"] = np.array([loss.item()])
            print(name, "loss %.6f" % loss.item(), "max |d observed| %.4f" % float(observed.grad.abs().max()))
    finally:
        ref_lstm.copy = saved
        torch.set_default_dtype(old_dtype)
    path = os.path.join(ROOT, "tests", "golden", "input_grad_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
