"""The shared-memory layout of the social grid's first Linear (sparse_layer1_mma).

An accumulator row keeps each warp's 16 columns as four 128-bit words (one per lane of a quad: columns 2t, 2t + 1 of
both 8-column halves), the kernel's first and last passes apply and undo that order four columns at a time, and a tile
slot is 16 bits (8-bit latent row, 8-bit accumulator row).  These tests run first-layer widths that end inside a
128-bit word and inside a four-column store (203), on a four-column but not an eight-column boundary (204, 100), and
the largest single scene the first layer's launch takes at 256 cells (114 pedestrians; 107 with 32-bit slots and
264-float accumulator rows), against the oracle.
"""
import numpy as np
import pytest
import torch

from oracle import lstm_oracle as O

pytestmark = pytest.mark.gpu

TOL_POS = 1e-4      # metres, the parity gate of every forward test
OBS, PRED = 9, 12


def _check(kind, xy, bs, seed):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    W = O.random_weights(kind, seed=seed)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().eval()
    with torch.no_grad():
        rel, pred = model(torch.from_numpy(xy[:OBS]), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs),
                          n_predict=PRED)
    rel, pred = rel.numpy(), pred.numpy()
    rel_o, pred_o = O.forward(W, O.pool_config(kind), xy[:OBS], bs, n_predict=PRED)
    assert (np.isnan(pred) == np.isnan(pred_o)).all()
    assert np.nanmax(np.abs(pred - pred_o)) < TOL_POS
    assert np.nanmax(np.abs(rel - rel_o)) < TOL_POS


@pytest.mark.parametrize("d1", [100, 203, 204])
def test_first_layer_width_inside_a_column_word(monkeypatch, d1):
    """Widths that are not a multiple of 16: the last warp with columns owns 4, 11 and 12 of its 16, so some of its
    128-bit accumulator words are half or wholly past the layer's width; 203 also takes the element-wise stores."""
    kind = "social_d%d" % d1
    monkeypatch.setitem(O.MODEL_SPECS, kind, dict(O.MODEL_SPECS["social_d96"], layer_dims=[d1]))
    xy, bs = O.synthetic_scenes(19, 20, n_frames=OBS + PRED, seed=41, nan_tracks=True)
    _check(kind, xy, bs, seed=11)


@pytest.mark.parametrize("peds", [108, 114])
def test_largest_single_scene(peds):
    """One scene of 108 and of 114 pedestrians at 256 cells next to two small ones: more rows than 32-bit slots
    left room for, and the most the launch takes now.  Latent and accumulator rows reach 113 of the 8-bit fields'
    254."""
    xy, bs = O.scenes_of_sizes([peds, 7, 20], n_frames=OBS + PRED, seed=42)
    xy[:3, 11] = np.nan
    _check("social", xy, bs.astype(np.int64), seed=12)
