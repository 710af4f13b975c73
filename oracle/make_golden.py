"""Generate tests/golden/lstm_golden.npz by running the UNMODIFIED reference (build container).

    python -m oracle.make_golden

Inputs and weights are regenerated from seeds (oracle.lstm_oracle.synthetic_scenes /
random_weights, numpy RandomState), so the fixture only stores the reference's OUTPUTS:
rel_pred_scene / pred_scene of LSTM.forward (free-running and teacher-forced), grid cell
indices of GridBasedPooling.occupancy, and raw grids for the adapted golden vectors of the
reference's own (stale) tests (SURVEY.md section 4).  TEST INFRASTRUCTURE.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O          # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

# (name, model kind, scenes, peds/scene, ragged, nan_tracks, data seed, weight seed, weight scale)
CASES = [
    ("vanilla_a", "vanilla", 6, 7, False, False, 11, 1, 1.0),
    ("vanilla_nan", "vanilla", 5, 9, True, True, 12, 2, 1.0),
    ("occupancy_a", "occupancy", 5, 8, True, True, 13, 3, 1.0),
    ("directional_a", "directional", 6, 10, False, False, 14, 4, 1.0),
    ("directional_nan", "directional", 5, 12, True, True, 15, 5, 2.0),
    ("directional_const", "directional_const", 4, 6, True, True, 16, 6, 1.0),
    ("occupancy_front", "occupancy_front", 4, 7, True, False, 17, 7, 1.0),
    ("social_small", "social_small", 5, 9, True, True, 18, 8, 1.0),
    ("social_single", "social_small", 1, 6, False, False, 19, 9, 1.0),
]


def build_reference_model(kind, weights, embedding_dim=64):
    from trajnetbaselines.lstm import LSTM, GridBasedPooling
    spec = O.MODEL_SPECS[kind]
    pool = GridBasedPooling(**spec) if spec is not None else None
    model = LSTM(embedding_dim=embedding_dim, pool=pool)
    sd = {k: torch.from_numpy(v.copy()) for k, v in weights.items()}
    model.load_state_dict(sd, strict=True)
    model.eval()
    return model


def reference_cells(kind, obs_padded):
    """Cell index / in-range flag of every ordered pair, read back from the reference itself.

    The reference never exposes `oi` (gridbased_pooling.py:287), so each pair (i, j) is probed
    with a two-pedestrian scene [i, j] through GridBasedPooling.occupancy: row 0 of the returned
    occupancy grid has exactly one non-zero cell iff j is in range of i, and no later writer
    can clobber it."""
    from trajnetbaselines.lstm import GridBasedPooling
    spec = dict(O.MODEL_SPECS[kind])
    spec.update(type_="occupancy", embedding_arch="None", constant=0)
    pool = GridBasedPooling(**spec)
    B, N, _ = obs_padded.shape
    cells = np.zeros((B, N, N - 1), dtype=np.int64)
    inr = np.zeros((B, N, N - 1), dtype=bool)
    for i in range(N):
        for jj in range(N - 1):
            j = jj + (jj >= i)
            obs = torch.from_numpy(np.stack([obs_padded[:, i], obs_padded[:, j]], axis=1).copy())
            grid = pool.occupancy(obs, None).reshape(B, 2, -1)[:, 0].numpy()   # [B, n*n]
            for b in range(B):
                idx = np.nonzero(grid[b] > 0.5)[0]
                if len(idx) == 1:
                    cells[b, i, jj] = idx[0]
                    inr[b, i, jj] = True
    return cells, inr


def main():
    import_reference()
    out = {}
    for name, kind, B, N, ragged, nan_tracks, dseed, wseed, wscale in CASES:
        xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
        W = O.random_weights(kind, seed=wseed, scale=wscale)
        model = build_reference_model(kind, W)
        M = xy.shape[1]
        goals = torch.zeros(M, 2)
        with torch.no_grad():
            rel_f, pred_f = model(torch.from_numpy(xy[:9]), goals, torch.from_numpy(bs), n_predict=12)
            rel_t, pred_t = model(torch.from_numpy(xy[:9]), goals, torch.from_numpy(bs),
                                  prediction_truth=torch.from_numpy(xy[9:20]).clone())
        out[name + "/rel_free"] = rel_f.numpy()
        out[name + "/pred_free"] = pred_f.numpy()
        out[name + "/rel_teacher"] = rel_t.numpy()
        out[name + "/pred_teacher"] = pred_t.numpy()
        print(name, "ok", rel_f.shape)

    # grid cell indices on positions that stress the bin boundaries (multiples of cell_side +- ulp)
    for kind in ("social", "directional", "occupancy_front"):
        cfg = O.pool_config(kind)
        rng = np.random.RandomState(77)
        B, N = 3, 6
        obs = (rng.randn(B, N, 2) * 2.0).astype(np.float32)
        side = np.float32(cfg.cell_side)
        for b in range(B):           # snap some neighbours exactly onto / next to cell edges
            for j in range(1, N, 2):
                k = rng.randint(-cfg.n // 2, cfg.n // 2 + 1, size=2)
                edge = obs[b, 0] + (k.astype(np.float32) * side)
                obs[b, j] = np.nextafter(edge, edge + rng.choice([-1, 1], size=2).astype(np.float32), dtype=np.float32) \
                    if j % 4 == 1 else edge
        obs[1, N - 1] = np.nan
        cells, inr = reference_cells(kind, obs)
        out["cells_%s/obs" % kind] = obs
        out["cells_%s/cells" % kind] = cells.astype(np.int32)
        out["cells_%s/in_range" % kind] = inr
        print("cells", kind, int(inr.sum()), "in range of", inr.size)

    # adapted golden vectors of the reference's stale tests (SURVEY.md section 4), re-run at HEAD
    from trajnetbaselines.lstm import GridBasedPooling
    def grid_of(obs1, obs2, **kw):
        pool = GridBasedPooling(embedding_arch="None", **kw)
        o1 = torch.tensor([obs1], dtype=torch.float32)
        o2 = torch.tensor([obs2], dtype=torch.float32)
        h = torch.zeros(1, len(obs1), 128)
        return pool(h, o1, o2).detach().numpy()
    nanv = float("nan")
    out["sec4/simple_grid"] = grid_of([[0, 0], [-1, -1]], [[0, 0], [-1, -1]], n=2, pool_size=4, blur_size=3, cell_side=2.0)
    out["sec4/simple_grid_midpoint"] = grid_of([[0, 0], [-1, 0]], [[0, 0], [-1, 0]], n=2, pool_size=100, blur_size=99, cell_side=2.0)
    out["sec4/nan"] = grid_of([[0, 0], [nanv, nanv]], [[0, 0], [nanv, nanv]], n=2, cell_side=2.0)
    out["sec4/directional"] = grid_of([[0, 0], [-1, -1]], [[0.1, 0.1], [-1.1, -1.1]], n=2, pool_size=4, cell_side=2.0, type_="directional")
    out["sec4/simple_grid_ps1"] = grid_of([[0, 0], [-1, -1]], [[0, 0], [-1, -1]], n=2, cell_side=2.0)
    out["sec4/directional_ps1"] = grid_of([[0, 0], [-1, -1]], [[0.1, 0.1], [-1.1, -1.1]], n=2, cell_side=2.0, type_="directional")

    # loss known answer (tests/test_lstm_loss.py:12-25 of the reference)
    from trajnetbaselines.lstm import PredictionLoss
    crit = PredictionLoss(background_rate=0.0) if False else PredictionLoss()
    gauss = torch.tensor([[[0.0, 0.0, 1.0, 1.0, 0.0]]])
    tgt = torch.tensor([[[0.0, 0.0]]])
    out["sec4/loss_simple"] = np.array([crit(gauss, tgt, torch.tensor([0, 1])).item()], dtype=np.float64)

    path = os.path.join(ROOT, "tests", "golden", "lstm_golden.npz")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
