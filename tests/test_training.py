"""Training path (SURVEY.md 8a/A12): hand-written CUDA BPTT vs (i) gradients of the unmodified
reference stored in tests/golden/train_golden.npz and (ii) a differentiable torch restatement
(tests/torch_ref.py) which is itself pinned to the same golden file on CPU."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_train_golden import TRAIN_CASES, check_summary, rel_to_max  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def train_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "train_golden.npz"))


@pytest.mark.parametrize("case", TRAIN_CASES, ids=[c[0] for c in TRAIN_CASES])
def test_torch_restatement_matches_reference_gradients(train_golden, case):
    """CPU: pins tests/torch_ref.py (the checker of the CUDA backward) to the reference."""
    name, kind, B, N, ragged, nan_tracks, dseed, wseed = case
    xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
    W = O.random_weights(kind, seed=wseed)
    loss, grads = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs)
    assert abs(loss - float(train_golden[name + "/loss"][0])) < 1e-4
    for pname, g in grads.items():
        if g is None:
            assert pname.startswith("goal_embedding")
            continue
        check_summary(name + "/" + pname, g, train_golden, rtol=2e-3, atol=2e-5)


def _cuda_train_step(kind, W, xy, bs):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    spec = O.MODEL_SPECS[kind]
    model = LSTM(pool=GridBasedPooling(**spec) if spec is not None else None)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    scene = torch.from_numpy(xy).cuda()
    batch_split = torch.from_numpy(bs)
    observed = scene[0:9]
    prediction_truth = scene[9:-1].clone()
    targets = scene[9:21] - scene[8:20]
    rel_outputs, outputs = model(observed, torch.zeros(xy.shape[1], 2), batch_split, prediction_truth)
    loss = PredictionLoss()(rel_outputs[-12:], targets, batch_split) * (len(bs) - 1)
    model.zero_grad()
    loss.backward()
    return model, float(loss.item())


@pytest.mark.gpu
@pytest.mark.parametrize("case", TRAIN_CASES, ids=[c[0] for c in TRAIN_CASES])
def test_cuda_backward_matches_reference_gradients(train_golden, case):
    name, kind, B, N, ragged, nan_tracks, dseed, wseed = case
    xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
    W = O.random_weights(kind, seed=wseed)
    model, loss = _cuda_train_step(kind, W, xy, bs)
    # forward runs the 3-pass bf16 tensor-core path: loss agrees to ~1e-5 relative
    ref_loss = float(train_golden[name + "/loss"][0])
    assert abs(loss - ref_loss) < 1e-4 * max(1.0, abs(ref_loss))
    worst, worst_name = 0.0, ""
    for pname, p in model.named_parameters():
        if pname.startswith("goal_embedding"):
            assert p.grad is None
            continue
        assert p.grad is not None, pname
        g = p.grad.cpu().numpy()
        rel = rel_to_max(name + "/" + pname, g, train_golden)
        if rel > worst:
            worst, worst_name = rel, pname
        # every parameter tensor within 1e-4 of its largest reference entry (measured: a few 1e-6, the fp32
        # summation order of the backward), plus the sum / |sum| checks of the stored summaries
        assert rel < 1e-4, (name, pname, rel)
        check_summary(name + "/" + pname, g, train_golden, rtol=1e-3, atol=1e-5)
    print("%s: worst max|grad - reference| / max|reference| = %.2e (%s)" % (name, worst, worst_name))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["vanilla", "directional", "occupancy"])
def test_cuda_backward_baseline_shape_vs_torch(kind):
    """N = 20, T = 9 + 12 (BASELINE D-LSTM training shape) at a batch the CPU autograd finishes
    in seconds; every gradient tensor compared in full."""
    xy, bs = O.synthetic_scenes(24, 20, seed=5, nan_tracks=True)
    W = O.random_weights(kind, seed=17)
    loss_ref, grads_ref = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs)
    model, loss = _cuda_train_step(kind, W, xy, bs)
    assert abs(loss - loss_ref) < 1e-3 * max(1.0, abs(loss_ref))
    for pname, p in model.named_parameters():
        g_ref = grads_ref[pname]
        if g_ref is None:
            assert p.grad is None
            continue
        g = p.grad.cpu().numpy()
        scale = max(np.abs(g_ref).max(), 1e-6)
        assert np.abs(g - g_ref).max() < 1e-4 * scale + 1e-7, (pname, float(np.abs(g - g_ref).max() / scale))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["directional", "occupancy"])
def test_cuda_backward_large_scene_vs_torch(kind):
    """A 90-pedestrian scene next to scenes of 3 and 40: the grid kernels at a large n_max.  The pool
    biases are +-3 (random_weights(relu_bias=3)), so no ReLU mask can flip between the two forwards; the
    precondition is asserted, with the distance of the fed-back primaries' offsets to a cell edge."""
    xy, bs = O.scenes_of_sizes([90, 3, 40], seed=1)
    W = O.random_weights(kind, seed=51, relu_bias=3.0)
    stats = {}
    loss_ref, grads_ref = TR.train_loss_and_grads(W, O.pool_config(kind), xy, bs, dtype=torch.float64,
                                                  stats=stats)
    assert stats["relu_pool0"] >= 1e-2 and stats["edge_primary"] >= 1e-5, stats
    model, loss = _cuda_train_step(kind, W, xy, bs)
    assert abs(loss - loss_ref) < 1e-5 * abs(loss_ref)
    for pname, p in model.named_parameters():
        g_ref = grads_ref[pname]
        if g_ref is None:
            assert p.grad is None
            continue
        g = p.grad.cpu().numpy()
        scale = max(np.abs(g_ref).max(), 1e-6)
        assert np.abs(g - g_ref).max() < 1e-4 * scale, (pname, float(np.abs(g - g_ref).max() / scale))


@pytest.mark.gpu
def test_optimizer_step_moves_loss_down():
    """A few Adam steps (trainer.py:497: lr 1e-3, weight_decay 1e-4) on one batch reduce the loss."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    kind = "directional"
    xy, bs = O.synthetic_scenes(32, 12, seed=8)
    W = O.random_weights(kind, seed=3)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
    crit = PredictionLoss()
    scene = torch.from_numpy(xy).cuda()
    targets = scene[9:21] - scene[8:20]
    losses = []
    for _ in range(6):
        rel, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), scene[9:-1].clone())
        loss = crit(rel[-12:], targets, torch.from_numpy(bs)) * 32
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0]


@pytest.mark.gpu
def test_social_training_is_deterministic_and_learns():
    """Social pooling: every track of a scene receives gradient (hidden-state scatter).  The backward
    has no floating-point atomics: two runs give bit-identical gradients; a few Adam steps reduce
    the loss."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    xy, bs = O.synthetic_scenes(12, 9, seed=21, ragged=True, nan_tracks=True)
    W = O.random_weights("social", seed=9)
    g1 = {n: p.grad.clone() for n, p in _cuda_train_step("social", W, xy, bs)[0].named_parameters() if p.grad is not None}
    g2 = {n: p.grad.clone() for n, p in _cuda_train_step("social", W, xy, bs)[0].named_parameters() if p.grad is not None}
    assert set(g1) == set(g2) and "pool.hidden_dim_encoding.weight" in g1 and "pool.embedding.2.weight" in g1
    for n in g1:
        assert torch.equal(g1[n], g2[n]), n
        assert torch.isfinite(g1[n]).all(), n
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS["social"]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
    scene = torch.from_numpy(xy).cuda()
    targets = scene[9:21] - scene[8:20]
    crit = PredictionLoss()
    losses = []
    for _ in range(6):
        rel, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), scene[9:-1].clone())
        loss = crit(rel[-12:], targets, torch.from_numpy(bs)) * 12
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < losses[0]


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [False, True])
def test_optimizer_updates_reach_the_device_weights(fused):
    """Fused optimizers update parameters without bumping `_version`; the device-side repack must
    still follow (engine.weights_key): identical loss trajectories for both Adam implementations."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    xy, bs = O.synthetic_scenes(16, 8, seed=3)
    W = O.random_weights("directional", seed=2)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS["directional"]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4, fused=fused)
    scene = torch.from_numpy(xy).cuda()
    targets = scene[9:21] - scene[8:20]
    crit = PredictionLoss()
    losses = []
    for _ in range(4):
        rel, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), scene[9:-1].clone())
        loss = crit(rel[-12:], targets, torch.from_numpy(bs)) * 16
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[1] < losses[0] and losses[3] < losses[1], losses
    model.eval()
    with torch.no_grad():      # the step taken after the last training forward is seen in eval mode too
        rel, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), scene[9:-1].clone())
        after = crit(rel[-12:], targets, torch.from_numpy(bs)).item() * 16
    assert after < losses[3], (after, losses)


@pytest.mark.gpu
def test_social_training_large_scene():
    """BPTT through social pooling with a 70-pedestrian scene next to small ones: finite, repeatable,
    and the primaries' loss matches the value the oracle computes for the same forward (default weights;
    the gradients of this layout are compared with the float64 restatement in test_social_backward.py)."""
    xy, bs = O.scenes_of_sizes([70, 2, 25], seed=3)
    W = O.random_weights("social", seed=6)
    m1, loss1 = _cuda_train_step("social", W, xy, bs)
    m2, loss2 = _cuda_train_step("social", W, xy, bs)
    rel_o, _ = O.forward(W, O.pool_config("social"), xy[:9], bs, prediction_truth=xy[9:-1])
    loss_o = float(O.prediction_loss(rel_o[-12:], xy[9:21] - xy[8:20], bs)) * (len(bs) - 1)
    assert abs(loss1 - loss_o) < 1e-3 * max(1.0, abs(loss_o))
    assert loss1 == loss2
    for (n1, p1), (n2, p2) in zip(m1.named_parameters(), m2.named_parameters()):
        if p1.grad is None:
            continue
        assert torch.isfinite(p1.grad).all(), n1
        assert torch.equal(p1.grad, p2.grad), n1
