"""Vanilla / occupancy / directional training (csrc/train.cu, the active-row backward of
tb2_lstm_sequence_backward) across the reference trainer's options, against a float64 autograd
restatement (tests/torch_ref.py).

The restatement is pinned on the CPU to gradients of the unmodified reference at tiny shapes
(tests/golden/grid_train_golden.npz, oracle/make_grid_train_golden.py).  On the GPU each case runs one
Trainer.train_batch step with the tensor cores on and with TB2_DISABLE_TC=1, checks that the backward ran
the GEMM branches the case is meant to cover (timer names from tb2_profile_begin / end), and compares the
loss and every parameter gradient with the float64 restatement at realistic shapes.

The GEMM branches (gemm_nn / gemm_tn in train.cu): a product of m * n * k >= 3.2e7 runs on cuBLAS
(bwd_gemm_cublas, bwd_gemm_tn_cublas), a smaller one on the FFMA kernels (bwd_gemm, bwd_gemm_tn), which
load float4 only when the leading dimensions are multiples of 4 and the base pointers 16-byte aligned, and
split the rows of a weight gradient over CTAs when its output has few tiles.

Preconditions, asserted before comparing: the grid embedding's biases are +-3 (random_weights
(relu_bias=3)), so every pool ReLU pre-activation is >= 1e-2 away from 0; the fed-back primaries'
offsets are >= 1e-5 cells from a cell edge, so both forwards bin every pair alike (or the restatement is
fed the GPU's own positions: `feed_back`); and with a collision term, every primary-neighbour distance is
>= 1e-5 m away from col_distance, so both count the same hits.  The data seeds were chosen once so that
these hold.
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
from oracle.make_grid_train_golden import GRID_TRAIN_CASES, all_tracks_loss, case_inputs, loss_args  # noqa: E402
from oracle.make_train_golden import rel_to_max  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RELU_MARGIN = 1e-2      # smallest |pre-activation| of the pool Linear
EDGE_MARGIN = 1e-5      # smallest distance (cells) of a fed-back primary's pair offset to a cell edge
COL_MARGIN = 1e-5       # smallest |primary-neighbour distance - col_distance| (metres)


def _check_margins(name, kind, stats, col_wt, feed_back=False):
    if O.MODEL_SPECS[kind] is not None:
        assert stats.get("relu_pool0", 0.0) >= RELU_MARGIN, (name, stats)
        if not feed_back:
            assert stats.get("edge_primary", math.inf) >= EDGE_MARGIN, (name, stats)
    if col_wt:
        assert stats.get("col_margin", 0.0) >= COL_MARGIN, (name, stats)


# ---------------------------------------------------------------------------------------------
# CPU: the restatement against the reference
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def grid_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "grid_train_golden.npz"))


@pytest.mark.parametrize("case", GRID_TRAIN_CASES, ids=[c[0] for c in GRID_TRAIN_CASES])
def test_torch_restatement_matches_grid_reference(grid_golden, case):
    name, kind, _, _, obs_length, pred_length = case[:6]
    col_wt = case[7]
    xy, bs, W = case_inputs(case)
    stats = {}
    loss, grads = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs, obs_length, pred_length,
                                          dtype=torch.float64, stats=stats, **loss_args(case))
    _check_margins(name, kind, stats, col_wt)
    # the collision cases collide: the reference's loss reaches the predicted positions
    assert (np.abs(grid_golden[name + "/positions_grad"]).max() > 0) == bool(col_wt), name
    ref_loss = float(grid_golden[name + "/loss"][0])
    assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (loss, ref_loss)    # the reference's loss is fp32
    for pname, g in grads.items():
        if g is None:       # goal_embedding; the decoder without a decoder step: the reference leaves .grad None
            assert not any(k.startswith(name + "/" + pname + "/") for k in grid_golden.files), (name, pname)
            assert pname.startswith("goal_embedding") or (pname.startswith("decoder.") and pred_length == 1)
            continue
        rel = rel_to_max(name + "/" + pname, g, grid_golden)
        assert rel <= 2e-6, (name, pname, rel)


# ---------------------------------------------------------------------------------------------
# GPU: the CUDA training step against the float64 restatement
# ---------------------------------------------------------------------------------------------
GEMMS = {"bwd_gemm", "bwd_gemm_cublas", "bwd_gemm_tn", "bwd_gemm_tn_cublas"}
FFMA_NN, BLAS_NN, FFMA_TN, BLAS_TN = "bwd_gemm", "bwd_gemm_cublas", "bwd_gemm_tn", "bwd_gemm_tn_cublas"


def _case(name, kind, E, data, obs_length, pred_length, loss, col_wt, col_distance, dseed, wseed, gemms,
          feed_back=False):
    """data: (scenes, max peds, ragged); ragged scene sets also have entering / leaving neighbours."""
    return (name, kind, E, data, obs_length, pred_length, loss, col_wt, col_distance, dseed, wseed, gemms, feed_back)


# R = active rows (the primaries: one per scene; every present track for all_tracks), S_enc = obs_length - 1 and
# S_dec = pred_length - 1 steps, K = E + P + 128.  The gates GEMM of a phase is (S_phase R) x 512 x K.
GPU_CASES = [
    # P = 256, K = 448: the gates GEMM runs FFMA in the encoder (8 x 16 = 128 rows) and cuBLAS in the decoder
    # (176 rows); the W_ih gradient (320 x 512 output) splits its rows over 2 CTAs; the collision term sends
    # gradient into the positions output
    _case("occ_default_col", "occupancy", 64, (16, 20, True), 9, 12, "pred", 2.0, 1.0, 2, 101,
          {FFMA_NN, BLAS_NN, FFMA_TN}),
    _case("dir_front", "directional_front", 64, (16, 20, True), 9, 12, "pred", 0.0, 0.2, 1, 102,
          {FFMA_NN, BLAS_NN, FFMA_TN}),
    # a 4 x 4 grid in front of the pedestrian: most pairs are out of range and write cell 0's slot
    _case("occ_front_n4", "occupancy_front_n4", 64, (16, 20, True), 9, 12, "l2", 0.0, 0.2, 1, 103,
          {FFMA_NN, BLAS_NN, FFMA_TN}),
    # grid rows of C n n = 1152: the pool-weight gradient (256 x 1152 x 304 rows) runs on cuBLAS
    _case("dir_n24", "directional_n24", 64, (16, 20, True), 9, 12, "pred", 0.0, 0.2, 1, 104,
          {FFMA_NN, BLAS_NN, FFMA_TN, BLAS_TN}),
    # P at the 1024 limit: every thread of bwd_gather holds 4 accumulators; K = 1216, so the row GEMMs run on
    # cuBLAS from 96 rows, and so does the pool-weight gradient (1024 x 144 x 228)
    _case("occ_p1024", "occupancy_p1024", 64, (12, 20, True), 9, 12, "l2", 2.0, 1.0, 1, 105,
          {BLAS_NN, FFMA_TN, BLAS_TN}),
    # E + P = 93 and K = 221 are odd: the FFMA GEMMs load scalars, cuBLAS gets odd leading dimensions and
    # operands at X + 93.  64 scenes so that the decoder's d X_in / W_ih gradient (704 x 93 x 512) reach cuBLAS
    # while the encoder's (512 rows) stay FFMA
    _case("dir_p29", "directional_p29", 64, (64, 20, True), 9, 12, "pred", 0.0, 0.2, 5, 106,
          {FFMA_NN, BLAS_NN, FFMA_TN, BLAS_TN}),
    # E = 30: the pooled block and h_prev start at misaligned offsets 30 and 286; bwd_embed has 28 units
    _case("dir_e30", "directional", 30, (16, 20, True), 9, 12, "pred", 0.0, 0.2, 1, 107,
          {FFMA_NN, BLAS_NN, FFMA_TN}),
    # no pool: K = 192, every GEMM FFMA
    _case("vanilla_l2_col", "vanilla", 64, (16, 20, True), 9, 12, "l2", 2.0, 1.0, 1, 108, {FFMA_NN, FFMA_TN}),
    # one encoder step (positions has S + 1 entries, the first one the last observation)
    _case("dir_obs2", "directional", 64, (16, 20, True), 2, 12, "pred", 0.0, 0.2, 3, 109,
          {FFMA_NN, BLAS_NN, FFMA_TN}),
    # no decoder step: the decoder phase of every GEMM is skipped
    _case("occ_obs5_pred1", "occupancy", 64, (16, 20, True), 5, 1, "pred", 0.0, 0.2, 1, 110, {FFMA_NN, FFMA_TN}),
    # every present track is an active row (R = M ~ 180), with the NaN gaps of entering / leaving tracks
    _case("dir_all_tracks", "directional", 64, (16, 20, True), 9, 12, "all_tracks", 0.0, 0.2, 1, 111,
          {BLAS_NN, FFMA_TN, BLAS_TN}),
    # bench.py's training step: its model and scenes (256 x 20, seed 100); cuBLAS everywhere but the
    # hidden2normal gradient.  The edge margin cannot hold at this size, so the restatement is fed the GPU's
    # positions
    _case("bench_shape", "directional", 64, (256, 20, False), 9, 12, "pred", 0.0, 0.2, 100, 1,
          {BLAS_NN, FFMA_TN, BLAS_TN}, feed_back=True),
]


def _gpu_inputs(case):
    return case_inputs(case, data=case[3])


def _restate(case, feed_back=None, outputs=None):
    name, kind, _, _, obs_length, pred_length, _, col_wt = case[:8]
    xy, bs, W = _gpu_inputs(case)
    stats = {}
    loss, grads = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs, obs_length, pred_length,
                                          dtype=torch.float64, stats=stats, feed_back=feed_back, outputs=outputs,
                                          **loss_args(case))
    _check_margins(name, kind, stats, col_wt, feed_back=feed_back is not None)
    return loss, grads


@pytest.fixture(scope="module")
def restated():
    """float64 restatement per case id, computed once for both tensor-core settings."""
    cache = {}

    def get(case):
        if case[0] not in cache:
            cache[case[0]] = _restate(case)
        return cache[case[0]]
    return get


def _train_step(case, W, xy, bs):
    """Trainer.train_batch on the CUDA model.  Returns (model, loss, timer names, positions)."""
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, L2Loss, PredictionLoss
    _, kind, E, _, obs_length, pred_length, loss_kind, col_wt, col_distance = case[:9]
    spec = O.MODEL_SPECS[kind]
    model = LSTM(embedding_dim=E, pool=GridBasedPooling(**spec) if spec is not None else None)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    scene = torch.from_numpy(xy).cuda()
    batch_split = torch.from_numpy(bs)
    prim = batch_split[:-1].cuda()
    targets = scene[obs_length:obs_length + pred_length] - scene[obs_length - 1:obs_length + pred_length - 1]
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 16)
    lib.tb2_profile_begin()
    try:
        rel, positions = model(scene[:obs_length], torch.zeros(xy.shape[1], 2), batch_split,
                               scene[obs_length:-1].clone())
        if loss_kind == "all_tracks":
            loss = all_tracks_loss(rel, positions)
        else:
            criterion = (PredictionLoss if loss_kind == "pred" else L2Loss)(col_wt=col_wt, col_distance=col_distance)
            primary_prediction = scene[-pred_length:].clone()
            primary_prediction[:, prim] = positions[-pred_length:, prim]
            loss = criterion(rel[-pred_length:], targets, batch_split, primary_prediction) * (len(bs) - 1)
        model.zero_grad()
        loss.backward()
    finally:
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
    kernels = set(json.loads(buf.value.decode()))
    return model, float(loss.item()), kernels, positions.detach().cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_cuda_grid_backward_matches_float64_restatement(restated, monkeypatch, case, tc):
    name, kind, _, _, obs_length, pred_length = case[:6]
    gemms, feed_back = case[11:13]
    if not tc:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")     # read when the model's handle is created
    else:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    xy, bs, W = _gpu_inputs(case)
    model, loss, kernels, positions = _train_step(case, W, xy, bs)

    # the GEMM branches this case exists for
    assert kernels & GEMMS == gemms, (name, sorted(kernels & GEMMS))

    if feed_back:
        # exact gradients of the GPU's trajectory.  Every position the GPU fed back is what the float64 model
        # predicts from the same inputs, to 1e-4 m.  (The restatement's free trajectory is not a yardstick here:
        # at 256 x 20 a primary pair lies 4.8e-7 cells from a cell edge, and a flipped bin moves that primary by
        # millimetres from then on.)
        outputs = {}
        loss_ref, grads_ref = _restate(case, feed_back=positions, outputs=outputs)
        prim = bs[:-1]
        drift = float(np.abs(positions[:, prim] - outputs["positions"][:, prim]).max())
        assert drift <= 1e-4, (name, drift)
        print("%s [%s]: fed-back primaries within %.1e m of the float64 step" % (name, "tc" if tc else "no_tc", drift))
    else:
        loss_ref, grads_ref = restated(case)

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
    model2, loss2, _, _ = _train_step(case, W, xy, bs)
    assert loss2 == loss
    for (n1, p1), (_, p2) in zip(model.named_parameters(), model2.named_parameters()):
        assert (p1.grad is None) == (p2.grad is None), n1
        if p1.grad is not None:
            assert torch.equal(p1.grad, p2.grad), n1


# ---------------------------------------------------------------------------------------------
# GPU: inference with the same configurations against the oracle
# ---------------------------------------------------------------------------------------------
TOL_POS = 1e-4      # metres


@pytest.mark.gpu
@pytest.mark.parametrize("kind,E", [("directional_front", 64), ("occupancy_front_n4", 64), ("directional_n24", 64),
                                    ("occupancy_p1024", 64), ("directional_p29", 64), ("directional", 30)])
def test_grid_forward_matches_oracle(kind, E):
    """Free-running and teacher-forced forwards against oracle.lstm_oracle.forward: a forward bug shows here
    rather than as a gradient mismatch."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    xy, bs = O.synthetic_scenes(6, 9, seed=71, ragged=True, nan_tracks=True)
    W = O.random_weights(kind, seed=72, embedding_dim=E, relu_bias=3.0)
    cfg = O.pool_config(kind)
    model = LSTM(embedding_dim=E, pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
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
        assert float(np.nanmax(np.abs(got - ref))) < TOL_POS, (kind, E, float(np.nanmax(np.abs(got - ref))))


# ---------------------------------------------------------------------------------------------
# GPU: grid configurations the backward does not support are refused, not trained wrongly
# ---------------------------------------------------------------------------------------------
UNSUPPORTED = [
    ("occupancy_two_layer", dict(type_="occupancy", n=4, cell_side=0.6, out_dim=32, embedding_arch="two_layer",
                                 layer_dims=[48])),
    ("occupancy_three_layer", dict(type_="occupancy", n=4, cell_side=0.6, out_dim=32, embedding_arch="three_layer",
                                   layer_dims=[48, 40])),
    ("occupancy_no_embedding", dict(type_="occupancy", n=4, cell_side=0.6, out_dim=16, embedding_arch="None")),
    ("directional_constant1", dict(type_="directional", n=4, cell_side=0.6, out_dim=32, constant=1)),
    ("occupancy_p1025", dict(type_="occupancy", n=4, cell_side=0.6, out_dim=1025)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("spec", [s for _, s in UNSUPPORTED], ids=[n for n, _ in UNSUPPORTED])
def test_unsupported_grid_training_is_refused(spec):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    torch.manual_seed(0)
    model = LSTM(pool=GridBasedPooling(**spec)).cuda().train()
    xy, bs = O.synthetic_scenes(4, 5, seed=3)
    scene = torch.from_numpy(xy).cuda()
    batch_split = torch.from_numpy(bs)
    rel, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), batch_split, scene[9:-1].clone())
    loss = PredictionLoss()(rel[-12:], scene[9:21] - scene[8:20], batch_split) * 4
    model.zero_grad()
    with pytest.raises(RuntimeError, match="training backward supports one_layer grid embeddings with constant = 0"):
        loss.backward()
    assert all(p.grad is None for p in model.parameters())
