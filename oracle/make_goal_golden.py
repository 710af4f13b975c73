"""Golden vectors of goal-conditioned LSTM models (LSTM(goal_flag=True), trajnetbaselines/lstm/lstm.py:72-85,131-139),
produced by the UNMODIFIED reference.

TEST INFRASTRUCTURE.  Run where the reference is importable: python -m oracle.make_goal_golden
-> tests/golden/goal_golden.npz.  The fixture holds the inputs (ragged scenes with absent tracks, goals with one goal
equal to a track's position at the last observed frame: a zero-norm direction) and per case LSTM.forward's outputs,
free-running and teacher-forced.  The weights of a case are regenerated from its seed (goal_weights), as for the other
golden files, which keeps the fixture small."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O          # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

# (case, model kind, goal_dim, weight seed)
CASES = [
    ("vanilla", "vanilla", 64, 1),
    ("vanilla_g32", "vanilla", 32, 2),
    ("occupancy", "occupancy", 64, 3),
    ("directional", "directional", 64, 4),
    ("social_small", "social_small", 64, 5),
    ("hiddenstatemlp_small", "hiddenstatemlp_small", 64, 6),
    ("nn_small", "nn_small", 64, 7),
]


def goal_weights(kind, goal_dim, seed, hidden_dim=128, embedding_dim=64, **kw):
    """random_weights(kind, **kw) with the goal columns spliced into weight_ih after the input embedding's and a goal
    embedding of goal_dim - 2 outputs (uniform in +-1 / sqrt(fan_in), like torch's default init)."""
    W = dict(O.random_weights(kind, seed=seed, hidden_dim=hidden_dim, embedding_dim=embedding_dim, **kw))
    rng = np.random.RandomState(seed + 1000)
    for phase in ("encoder", "decoder"):
        w = W[phase + ".weight_ih"]
        bound = 1.0 / np.sqrt(w.shape[1] + goal_dim)
        cols = rng.uniform(-bound, bound, size=(w.shape[0], goal_dim)).astype(np.float32)
        W[phase + ".weight_ih"] = np.ascontiguousarray(np.concatenate([w[:, :embedding_dim], cols, w[:, embedding_dim:]],
                                                                      axis=1))
    bound = 1.0 / np.sqrt(2.0)
    W["goal_embedding.input_embeddings.0.weight"] = rng.uniform(-bound, bound, size=(goal_dim - 2, 2)).astype(np.float32)
    W["goal_embedding.input_embeddings.0.bias"] = rng.uniform(-bound, bound, size=(goal_dim - 2,)).astype(np.float32)
    return W


def goal_inputs(seed=41):
    """Ragged scenes with absent tracks, 9 + 12 frames; goals ~ 4 m ahead of each track's last observation, with one
    goal exactly at a track's last observed position."""
    xy, bs = O.synthetic_scenes(5, 8, seed=seed, ragged=True, nan_tracks=True)
    rng = np.random.RandomState(seed + 1)
    last = np.nan_to_num(xy[8])                             # tracks absent there: goals around the origin
    goals = (last + rng.randn(*last.shape) * 4.0).astype(np.float32)
    present = np.nonzero(~np.isnan(xy[8, :, 0]) & ~np.isnan(xy[7, :, 0]))[0]
    goals[present[1]] = xy[8, present[1]]                  # zero norm at the last encoder step
    return xy, bs, goals


def model_kwargs(kind):
    for table in (O.NONGRID_SPECS, O.NN_SPECS, O.ATTN_SPECS, O.NN_LSTM_SPECS, O.TRAJ_SPECS):
        if kind in table:
            return table, table[kind]
    return O.MODEL_SPECS, O.MODEL_SPECS[kind]


def build_reference_model(kind, goal_dim, W):
    from trajnetbaselines.lstm import LSTM, GridBasedPooling
    from trajnetbaselines.lstm.non_gridbased_pooling import HiddenStateMLPPooling, NearestNeighborMLP
    table, spec = model_kwargs(kind)
    pool = None
    if table is O.NONGRID_SPECS:
        pool = HiddenStateMLPPooling(**spec)
    elif table is O.NN_SPECS:
        pool = NearestNeighborMLP(**spec)
    elif spec is not None:
        pool = GridBasedPooling(**spec)
    model = LSTM(pool=pool, goal_flag=True, goal_dim=goal_dim)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    return model.eval()


def main():
    import_reference()
    xy, bs, goals = goal_inputs()
    out = {"xy": xy, "batch_split": bs, "goals": goals}
    for case, kind, goal_dim, seed in CASES:
        W = goal_weights(kind, goal_dim, seed)
        model = build_reference_model(kind, goal_dim, W)
        with torch.no_grad():
            rel, pred = model(torch.from_numpy(xy[:9]), torch.from_numpy(goals), torch.from_numpy(bs), n_predict=12)
            rel_t, pred_t = model(torch.from_numpy(xy[:9]), torch.from_numpy(goals), torch.from_numpy(bs),
                                  prediction_truth=torch.from_numpy(xy[9:20]).clone())
        out[case + "/rel_free"] = rel.numpy()
        out[case + "/pred_free"] = pred.numpy()
        out[case + "/rel_teacher"] = rel_t.numpy()
        out[case + "/pred_teacher"] = pred_t.numpy()
    path = os.path.join(ROOT, "tests", "golden", "goal_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
