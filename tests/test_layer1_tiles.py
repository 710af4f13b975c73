"""The tile list of the social grid's first Linear (sparse_layer1_mma).

Each CTA lays the (track, cell) pairs of its scene group out as one list of 16-row tiles in ascending cell order, every
cell padded to whole tiles.  These tests run a cell that needs three tiles, groups whose cells all fit in half a tile,
absent tracks, a 90-pedestrian scene (which takes the second, smaller scene grouping) and a first layer narrower than
one 256-column chunk, against the oracle; every case runs twice and must give bit-identical outputs.
"""
import numpy as np
import pytest
import torch

from oracle import lstm_oracle as O

pytestmark = pytest.mark.gpu

TOL_POS = 1e-4      # metres, the parity gate of every forward test
OBS, PRED = 9, 12


def pairs_per_cell(xy, bs, cfg):
    """[scenes, cells] winning (track, neighbour) pairs per cell at one frame xy [M, 2], counted over every track
    (absent ones too, so the counts are upper bounds)."""
    cells = cfg.n * cfg.n
    out = np.zeros((len(bs) - 1, cells), dtype=np.int64)
    for b in range(len(bs) - 1):
        n = int(bs[b + 1] - bs[b])
        if n < 2:
            continue
        oi, in_range = O.grid_cells(xy[None, bs[b]:bs[b + 1]], cfg)
        oi, in_range = oi.reshape(n, n - 1), in_range.reshape(n, n - 1)
        last = np.full((n, cells), -1, dtype=np.int64)        # last writer per cell (out of range writes cell 0)
        for jj in range(n - 1):
            last[np.arange(n), oi[:, jj]] = jj
        win = (last >= 0) & in_range[np.arange(n)[:, None], np.maximum(last, 0)]
        out[b] = win.sum(axis=0)
    return out


def crowded_scenes(seed=0):
    """A scene of 40 pedestrians within a few centimetres of each other (every track has a neighbour in each of the
    four cells around its own position: 40 pairs, three tiles, in each of those cells) next to three random
    20-pedestrian scenes."""
    rng = np.random.RandomState(seed)
    n, T = 40, OBS + PRED
    crowd = rng.randn(n, 2)[None] * 0.05 + np.cumsum(rng.randn(T, n, 2) * 0.005, axis=0)
    rest, bs_rest = O.synthetic_scenes(3, 20, n_frames=T, seed=seed + 1)
    xy = np.concatenate([crowd.astype(np.float32), rest], axis=1)
    return xy, np.concatenate([[0, n], bs_rest[1:] + n]).astype(np.int64)


def _model(kind, seed):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    W = O.random_weights(kind, seed=seed)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    return W, model.cuda().eval()


def _forward(model, xy, bs):
    with torch.no_grad():
        rel, pred = model(torch.from_numpy(xy[:OBS]), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs),
                          n_predict=PRED)
    return rel.numpy(), pred.numpy()


def _check(kind, xy, bs, seed=7):
    """Oracle parity, and a second run with bit-identical outputs."""
    W, model = _model(kind, seed)
    rel, pred = _forward(model, xy, bs)
    rel2, pred2 = _forward(model, xy, bs)
    assert np.array_equal(rel, rel2, equal_nan=True)
    assert np.array_equal(pred, pred2, equal_nan=True)
    rel_o, pred_o = O.forward(W, O.pool_config(kind), xy[:OBS], bs, n_predict=PRED)
    assert (np.isnan(pred) == np.isnan(pred_o)).all()
    assert np.nanmax(np.abs(pred - pred_o)) < TOL_POS
    assert np.nanmax(np.abs(rel - rel_o)) < TOL_POS


@pytest.mark.parametrize("kind", ["social", "social_d96"])
def test_cell_of_three_tiles(kind):
    """One cell of the group holds at least 33 pairs at every observed frame.  social_d96 (d1 = 96) leaves most
    warps of its only column chunk without columns."""
    xy, bs = crowded_scenes()
    cfg = O.pool_config(kind)
    for f in range(OBS):
        assert pairs_per_cell(xy[f], bs, cfg)[0].max() >= 33
    _check(kind, xy, bs)


def test_half_padded_tiles_only():
    """Two small scenes in one group: no cell ever holds more than 8 pairs, so every tile is at least half
    padding."""
    xy, bs = O.synthetic_scenes(2, 5, n_frames=OBS + PRED, seed=31)
    cfg = O.pool_config("social")
    for f in range(OBS):
        assert pairs_per_cell(xy[f], bs, cfg).sum(axis=0).max() <= 8
    _check("social", xy, bs)


def test_absent_tracks():
    """Ragged scenes with tracks that enter late or leave early (NaN positions)."""
    xy, bs = O.synthetic_scenes(11, 20, n_frames=OBS + PRED, seed=32, ragged=True, nan_tracks=True)
    _check("social", xy, bs)


def test_ninety_pedestrians():
    """A 90-pedestrian scene (89 neighbour slots per track) next to a crowded one and a small one: the large
    scene grouping no longer fits in shared memory and the second grouping (groups of at most 90 rows) runs."""
    big, bs_big = O.scenes_of_sizes([90, 3], n_frames=OBS + PRED, seed=33)
    crowd, bs_crowd = crowded_scenes(seed=34)
    xy = np.concatenate([big, crowd], axis=1)
    bs = np.concatenate([bs_big, bs_crowd[1:] + bs_big[-1]]).astype(np.int64)
    xy[:4, 5] = np.nan                      # a late entry and an early exit inside the big scene
    xy[12:, 7] = np.nan
    _check("social", xy, bs)
