"""The social grid's first Linear on the tensor cores (sparse_layer1_mma).

A CTA holds one scene group (up to 160 rows at 20 pedestrians per scene, i.e. 8 scenes) and 256 output columns, and
each of its 16 warps owns 16 of those columns.  These tests move the same scenes across scene groups, run batches
from one scene to 33 groups, and first-layer widths that leave a partial column chunk, so some warps own columns past
the layer's width.
"""
import ctypes
import json

import numpy as np
import pytest
import torch

from oracle import lstm_oracle as O

pytestmark = pytest.mark.gpu

TOL_POS = 1e-4      # metres, the parity gate of every forward test
PEDS = 20
SCENES_PER_GROUP = 160 // PEDS


def _model(kind, seed):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    W = O.random_weights(kind, seed=seed)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    return W, model.cuda().eval()


def _forward(model, xy, bs):
    with torch.no_grad():
        rel, pred = model(torch.from_numpy(xy[:9]), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), n_predict=12)
    return rel.numpy(), pred.numpy()


def _check_oracle(kind, W, model, xy, bs):
    rel, pred = _forward(model, xy, bs)
    rel_o, pred_o = O.forward(W, O.pool_config(kind), xy[:9], bs, n_predict=12)
    assert (np.isnan(pred) == np.isnan(pred_o)).all()
    assert np.nanmax(np.abs(pred - pred_o)) < TOL_POS
    assert np.nanmax(np.abs(rel - rel_o)) < TOL_POS


@pytest.mark.parametrize("extra", [1, 2, 3, 4])
def test_predictions_do_not_depend_on_the_scene_group(extra):
    """The same 12 scenes behind 0 and `extra` other scenes: they land in other scene groups and at other rows of
    them, and every output must be bit-identical."""
    _, model = _model("social", seed=1)
    xy, bs = O.synthetic_scenes(12, PEDS, seed=21)
    xy_x, bs_x = O.synthetic_scenes(extra, PEDS, seed=22)
    rel0, pred0 = _forward(model, xy, bs)
    both = np.concatenate([xy_x, xy], axis=1)
    rel1, pred1 = _forward(model, both, np.concatenate([bs_x, bs[1:] + bs_x[-1]]))
    m0 = int(bs_x[-1])
    assert np.array_equal(rel1[:, m0:], rel0, equal_nan=True)
    assert np.array_equal(pred1[:, m0:], pred0, equal_nan=True)


@pytest.mark.parametrize("scenes", [1, SCENES_PER_GROUP, 2 * SCENES_PER_GROUP, 3 * SCENES_PER_GROUP,
                                    5 * SCENES_PER_GROUP, 33 * SCENES_PER_GROUP])
def test_group_counts_match_the_oracle(scenes):
    """1 scene, and 1, 2, 3, 5 and 33 full scene groups."""
    W, model = _model("social", seed=3)
    xy, bs = O.synthetic_scenes(scenes, PEDS, seed=23, nan_tracks=True)
    _check_oracle("social", W, model, xy, bs)


@pytest.mark.parametrize("kind", ["social_d96", "social_d200", "social"])
def test_first_layer_widths_match_the_oracle(kind):
    """d1 = 96 and 200 leave a partial 256-column chunk (warps whose columns lie past d1 load zero weights and
    store nothing); 1024 is the benchmark's width."""
    W, model = _model(kind, seed=5)
    xy, bs = O.synthetic_scenes(2 * SCENES_PER_GROUP + 3, PEDS, seed=24, nan_tracks=True)
    _check_oracle(kind, W, model, xy, bs)


def test_benchmark_shape_runs_the_tensor_core_layer():
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    _, model = _model("social", seed=1)
    xy, bs = O.synthetic_scenes(256, PEDS, seed=0)
    buf = ctypes.create_string_buffer(1 << 16)
    lib.tb2_profile_begin()
    try:
        _forward(model, xy, bs)
    finally:
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
    prof = json.loads(buf.value.decode())
    assert "sparse_layer1_mma" in prof and "sparse_layer1" not in prof
    assert prof["sparse_layer1_mma"]["launches"] == 19
