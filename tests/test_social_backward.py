"""Social-LSTM training (csrc/train.cu social_backward) in every configuration the library dispatches
to different kernels, against a float64 autograd restatement (tests/torch_ref.py).

The restatement is pinned on the CPU to gradients of the unmodified reference at tiny shapes
(tests/golden/social_train_golden.npz, oracle/make_social_train_golden.py).  On the GPU each case runs a
teacher-forced training step with the tensor cores on and with TB2_DISABLE_TC=1, checks that the step
took the kernels the case is meant to cover (kernel names from tb2_profile_begin / end) with the
forward's training cache, and compares the loss and every parameter gradient with the float64
restatement at realistic shapes.

Preconditions, asserted before comparing: the grid embedding's biases are +-3 (random_weights
(relu_bias=3)), so every pool ReLU pre-activation is >= 1e-2 away from 0 and no ReLU mask can flip
between the GPU forward and the CPU one; and the fed-back primaries' offsets are >= 1e-5 cells from a
cell edge, so both bin every pair alike.  The data seeds were chosen once so that these hold.
"""
import ctypes
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_social_train_golden import SOCIAL_TRAIN_CASES, case_inputs  # noqa: E402
from oracle.make_train_golden import rel_to_max  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RELU_MARGIN = 1e-2      # smallest |pre-activation| of a pool Linear
EDGE_MARGIN = 1e-5      # smallest distance (cells) of a fed-back primary's pair offset to a cell edge


def _check_margins(name, stats):
    relu = [v for k, v in stats.items() if k.startswith("relu_pool")]
    assert relu and min(relu) >= RELU_MARGIN, (name, stats)
    assert stats.get("edge_primary", math.inf) >= EDGE_MARGIN, (name, stats)


# ---------------------------------------------------------------------------------------------
# CPU: the restatement against the reference
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def social_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "social_train_golden.npz"))


@pytest.mark.parametrize("case", SOCIAL_TRAIN_CASES, ids=[c[0] for c in SOCIAL_TRAIN_CASES])
def test_torch_restatement_matches_social_reference(social_golden, case):
    name, kind = case[:2]
    obs_length, pred_length = case[6:8]
    xy, bs, W = case_inputs(case)
    stats = {}
    loss, grads = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs, obs_length, pred_length,
                                          dtype=torch.float64, stats=stats)
    _check_margins(name, stats)
    ref_loss = float(social_golden[name + "/loss"][0])
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)    # the reference's loss is fp32
    for pname, g in grads.items():
        if g is None:
            assert pname.startswith("goal_embedding")
            continue
        rel = rel_to_max(name + "/" + pname, g, social_golden)
        assert rel <= 2e-6, (name, pname, rel)


# ---------------------------------------------------------------------------------------------
# GPU: the CUDA training step against the float64 restatement
# ---------------------------------------------------------------------------------------------
TC_KERNELS = {"sparse_layer1_mma", "social_dgrid_mma", "social_dw1_mma", "dense_layer_tc"}
FFMA_KERNELS = {"sparse_layer1", "social_dgrid", "social_dw1"}

# (id, kind, data, obs_length, pred_length, data seed, weight seed, kernels the step runs with the tensor cores on).
# data: (scenes, max peds, ragged) or a list of scene sizes.
# With TB2_DISABLE_TC=1 every case runs on FFMA_KERNELS and none of TC_KERNELS.
GPU_CASES = [
    # the reference trainer's --type social: one_layer, the first Linear writes the gates' operand directly
    ("reference_default", "social_default", (16, 20, True), 9, 12, 2, 102,
     {"sparse_layer1_mma", "social_dgrid_mma", "social_dw1_mma", "dense_layer_tc"}),
    ("latent4", "social_c4", (16, 20, True), 9, 12, 1, 101,
     {"sparse_layer1", "social_dgrid", "social_dw1", "dense_layer_tc"}),
    ("latent32", "social_c32", (16, 20, True), 9, 12, 1, 101,
     {"sparse_layer1", "social_dgrid", "social_dw1", "dense_layer_tc"}),
    # d1 % 32 == 0 but < 256: a partial 256-column chunk; no wgmma second layer, so fp32 records + fp32 row GEMMs
    ("latent16_d96", "social_d96", (16, 20, True), 9, 12, 1, 101,
     {"sparse_layer1_mma", "social_dgrid_mma", "social_dw1_mma"}),
    # d1 % 32 != 0: FFMA dgrid / dW1 after a tensor-core forward
    ("latent16_d200", "social_d200", (16, 20, True), 9, 12, 1, 101,
     {"sparse_layer1_mma", "social_dgrid", "social_dw1"}),
    ("baseline", "social", (16, 20, False), 9, 12, 3, 103,
     {"sparse_layer1_mma", "social_dgrid_mma", "social_dw1_mma", "dense_layer_tc"}),
    ("large_scene", "social", [70, 2, 25], 9, 12, 3, 103,
     {"sparse_layer1_mma", "social_dgrid_mma", "social_dw1_mma", "dense_layer_tc"}),
    ("short_sequence", "social_default", (16, 20, True), 2, 3, 1, 101,
     {"sparse_layer1_mma", "social_dgrid_mma", "social_dw1_mma", "dense_layer_tc"}),
]


def _case_inputs(case):
    _, kind, data, obs_length, pred_length, dseed, wseed = case[:7]
    if isinstance(data, list):
        xy, bs = O.scenes_of_sizes(data, n_frames=obs_length + pred_length, seed=dseed)
    else:
        B, N, ragged = data
        xy, bs = O.synthetic_scenes(B, N, n_frames=obs_length + pred_length, seed=dseed, ragged=ragged,
                                    nan_tracks=True)
    return xy, bs, O.random_weights(kind, seed=wseed, relu_bias=3.0)


@pytest.fixture(scope="module")
def restated():
    """float64 restatement per case id, computed once for both tensor-core settings."""
    cache = {}

    def get(case):
        if case[0] not in cache:
            name, kind, _, obs_length, pred_length = case[:5]
            xy, bs, W = _case_inputs(case)
            stats = {}
            loss, grads = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs, obs_length, pred_length,
                                                  dtype=torch.float64, stats=stats)
            _check_margins(name, stats)
            cache[name] = (loss, grads)
        return cache[case[0]]
    return get


def _train_step(kind, W, xy, bs, obs_length, pred_length):
    """Trainer.train_batch on the CUDA model: teacher-forced forward, PredictionLoss x batch size, backward.
    Returns (model, loss, kernel names launched, training-cache bytes of the layout)."""
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    scene = torch.from_numpy(xy).cuda()
    batch_split = torch.from_numpy(bs)
    targets = scene[obs_length:obs_length + pred_length] - scene[obs_length - 1:obs_length + pred_length - 1]
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 16)
    lib.tb2_profile_begin()
    try:
        rel, _ = model(scene[:obs_length], torch.zeros(xy.shape[1], 2), batch_split, scene[obs_length:-1].clone())
        loss = PredictionLoss()(rel[-pred_length:], targets, batch_split) * (len(bs) - 1)
        model.zero_grad()
        loss.backward()
    finally:
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
    kernels = set(json.loads(buf.value.decode()))
    layout = model._layouts.get(bs.tolist(), device=scene.device)
    cache_bytes = model._engine().train_cache_bytes(layout, obs_length + pred_length - 2)
    return model, float(loss.item()), kernels, cache_bytes


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_cuda_social_backward_matches_float64_restatement(restated, monkeypatch, case, tc):
    name, kind, _, obs_length, pred_length, _, _, tc_kernels = case
    if not tc:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")     # read when the model's handle is created
    else:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    loss_ref, grads_ref = restated(case)
    xy, bs, W = _case_inputs(case)
    model, loss, kernels, cache_bytes = _train_step(kind, W, xy, bs, obs_length, pred_length)

    # the branch this case exists for, trained from the forward's cache
    assert cache_bytes > 0, (name, cache_bytes)
    want = tc_kernels if tc else FFMA_KERNELS
    unwanted = (TC_KERNELS | FFMA_KERNELS) - want
    assert want <= kernels and not (unwanted & kernels), (name, sorted(kernels & (TC_KERNELS | FFMA_KERNELS)))

    assert abs(loss - loss_ref) <= 1e-5 * abs(loss_ref), (name, loss, loss_ref)
    worst, worst_name = 0.0, ""
    for pname, p in model.named_parameters():
        g_ref = grads_ref[pname]
        if g_ref is None:
            assert p.grad is None, pname
            continue
        assert p.grad is not None, pname
        g = p.grad.cpu().numpy()
        rel = float(np.abs(g - g_ref).max() / max(np.abs(g_ref).max(), 1e-30))
        if rel > worst:
            worst, worst_name = rel, pname
        assert rel <= 1e-4, (name, pname, rel)
    print("%s [%s]: loss rel err %.1e, worst max|grad - float64| / max|float64| = %.2e (%s)"
          % (name, "tc" if tc else "no_tc", abs(loss - loss_ref) / abs(loss_ref), worst, worst_name))

    # the backward has no floating-point atomics: a second step gives bit-identical gradients
    model2, loss2, _, _ = _train_step(kind, W, xy, bs, obs_length, pred_length)
    assert loss2 == loss
    for (n1, p1), (_, p2) in zip(model.named_parameters(), model2.named_parameters()):
        assert (p1.grad is None) == (p2.grad is None), n1
        if p1.grad is not None:
            assert torch.equal(p1.grad, p2.grad), n1


@pytest.mark.gpu
def test_social_backward_without_cache_is_refused(monkeypatch):
    """The social backward reads its grid-embedding records from the training forward's cache only: a backward
    handed no cache is refused, naming the call that fills it."""
    case = GPU_CASES[0]
    _, kind, _, obs_length, pred_length = case[:5]
    xy, bs, W = _case_inputs(case)
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    forward = model._forward_nograd

    def forward_dropping_cache(*args, **kwargs):
        normals, positions, states, (obs, truth, layout, cache) = forward(*args, **kwargs)
        assert cache is not None
        return normals, positions, states, (obs, truth, layout, None)
    monkeypatch.setattr(model, "_forward_nograd", forward_dropping_cache)
    scene = torch.from_numpy(xy).cuda()
    batch_split = torch.from_numpy(bs)
    rel, _ = model(scene[:obs_length], torch.zeros(xy.shape[1], 2), batch_split, scene[obs_length:-1].clone())
    targets = scene[obs_length:obs_length + pred_length] - scene[obs_length - 1:obs_length + pred_length - 1]
    loss = PredictionLoss()(rel[-pred_length:], targets, batch_split)
    with pytest.raises(RuntimeError, match=r"error -1: .*tb2_lstm_forward_steps call \(cache_dev\)"):
        loss.backward()


# ---------------------------------------------------------------------------------------------
# GPU: inference with the same pooling configurations against the oracle
# ---------------------------------------------------------------------------------------------
TOL_POS = 1e-4      # metres


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["social_default", "social_c4", "social_c32", "social_d96", "social_d200"])
def test_social_forward_matches_oracle(kind):
    """Free-running and teacher-forced forwards (one_layer direct-split first Linear, FFMA latent 4 / 32
    first Linears, narrow two_layer widths) against oracle.lstm_oracle.forward."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    xy, bs = O.synthetic_scenes(6, 9, seed=61, ragged=True, nan_tracks=True)
    W = O.random_weights(kind, seed=62, relu_bias=3.0)
    cfg = O.pool_config(kind)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    model = model.cuda().eval()
    M = xy.shape[1]
    with torch.no_grad():
        rel_f, pred_f = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs), n_predict=12)
        rel_t, pred_t = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs),
                              prediction_truth=torch.from_numpy(xy[9:20]).clone())
    rel_fo, pred_fo = O.forward(W, cfg, xy[:9], bs, n_predict=12)
    rel_to, pred_to = O.forward(W, cfg, xy[:9], bs, prediction_truth=xy[9:20])
    for got, ref in ((rel_f, rel_fo), (pred_f, pred_fo), (rel_t, rel_to), (pred_t, pred_to)):
        got = got.numpy()
        assert got.shape == ref.shape
        assert (np.isnan(got) == np.isnan(ref)).all()
        assert float(np.nanmax(np.abs(got - ref))) < TOL_POS, (kind, float(np.nanmax(np.abs(got - ref))))


@pytest.mark.gpu
def test_unsupported_latent_dim_is_refused():
    """Social pooling is built for latent_dim 4, 8, 16 and 32; anything else is refused on the first forward."""
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling
    pool = GridBasedPooling(type_="social", n=4, cell_side=0.6, latent_dim=12).cuda()
    obs = torch.zeros(1, 3, 2, device="cuda")
    obs[0, 1] = 0.5
    obs[0, 2] = -0.5
    with pytest.raises(RuntimeError, match="latent_dim must be 4, 8, 16 or 32"):
        pool(torch.zeros(1, 3, 128, device="cuda"), obs, obs)
