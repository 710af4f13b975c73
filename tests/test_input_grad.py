"""Gradients wrt the observed trajectories (d observed): tb2_lstm_grads.d_observed / d_obs1 / d_obs2 (csrc/train.cu,
input_grad_kernel) behind LSTM.forward, against the float64 autograd restatement tests/input_grad_ref.py.

The gradient is autograd's on the reference's graph with its deep copy of observed[-1] read as a detached copy: it
reaches observed through the encoder steps' velocity inputs, the directional grid's relative velocities, the hidden
states social pooling reads and pred = obs2 + mu of the encoder steps.  The decoder's inputs are detached.

On the CPU the restatement is pinned to the unmodified reference (tests/golden/input_grad_golden.npz,
oracle/make_input_grad_golden.py).  On the GPU it is fed the GPU's positions (`feed_back`), so no fed-back position
can be binned differently, and its observed positions stay fp32 (an fp64 leaf cast to fp32, so the gradient flows
through the cast): both forwards bin every pair alike.
"""
import ctypes
import json
import os
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import input_grad_ref as IR  # noqa: E402
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_input_grad_golden import INPUT_GRAD_CASES, case_inputs, loss_weights  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RELU_MARGIN = 1e-2
TOL = 1e-4              # max |d observed - float64| / max |float64|
PRED_LENGTH = 12


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_lstm_grads_fields_match_header():
    from trajnetplusplusbaselines_b200 import _lib
    with open(os.path.join(ROOT, "include", "trajnet_b200.h")) as f:
        header = f.read()
    body = re.search(r"typedef struct tb2_lstm_grads \{(.*?)\} tb2_lstm_grads;", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    names = re.findall(r"float\s*\*\s*(\w+)\s*;", body)
    assert names == [n for n, _ in _lib.LstmGrads._fields_]
    assert names[-3:] == ["d_observed", "d_obs1", "d_obs2"]


@pytest.mark.parametrize("case", INPUT_GRAD_CASES, ids=[c[0] for c in INPUT_GRAD_CASES])
def test_restatement_matches_reference_input_grad(case):
    """tests/input_grad_ref.py's d observed against the unmodified reference's, both in float64."""
    golden = np.load(os.path.join(ROOT, "tests", "golden", "input_grad_golden.npz"))
    name, kind, teacher, obs_length = case[:4]
    xy, bs, W = case_inputs(case)
    W64 = {k: torch.tensor(v, dtype=torch.float64) for k, v in W.items()}
    leaf = torch.tensor(xy[:obs_length], dtype=torch.float64, requires_grad=True)
    truth = torch.from_numpy(xy[obs_length:-1]).double() if teacher else None
    spec = O.MODEL_SPECS[kind]
    stats = {}
    rel, pos = IR.forward(W64, O.pool_config(kind) if spec is not None else None, leaf, bs, prediction_truth=truth,
                          n_predict=None if teacher else PRED_LENGTH, stats=stats)
    wr, wp = loss_weights(pos.shape[0], rel.shape[0], xy.shape[1])
    loss = (torch.nan_to_num(rel) * torch.from_numpy(wr)).sum() + (torch.nan_to_num(pos) * torch.from_numpy(wp)).sum()
    loss.backward()
    if spec is not None and spec.get("embedding_arch") is not None:
        assert stats.get("relu_pool0", 0.0) >= RELU_MARGIN, (name, stats)
    ref_loss = float(golden[name + "/loss"][0])
    assert abs(loss.item() - ref_loss) <= 1e-9 * max(abs(ref_loss), 1.0), (loss.item(), ref_loss)
    ref = golden[name + "/d_observed"]
    g = leaf.grad.numpy()
    assert np.isfinite(ref).all() and np.abs(ref).max() > 0
    assert np.abs(g - ref).max() <= 2e-6 * np.abs(ref).max(), (name, float(np.abs(g - ref).max()))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: d observed against the float64 restatement
# ---------------------------------------------------------------------------------------------------------------------
def _case(name, kind, teacher, obs_length, loss, data=(12, 12), dseed=1, wseed=1):
    return (name, kind, teacher, obs_length, loss, data, dseed, wseed)


# loss: "all" weighs every track's rel_pred_scene and pred_scene; "prim" the primaries' only (the active rows are the
# primaries, and a directional grid still carries gradient to their neighbours).  Scenes are ragged with NaN gaps.
CASES = [
    _case("vanilla_tf", "vanilla", True, 9, "all"),
    _case("vanilla_free_obs2", "vanilla", False, 2, "all", dseed=2),
    _case("occ_tf", "occupancy", True, 9, "prim", dseed=3),
    _case("dir_tf", "directional", True, 9, "all", dseed=4),
    _case("dir_free_prim", "directional", False, 9, "prim", dseed=5),
    _case("dir_obs2", "directional", True, 2, "prim", dseed=6),
    _case("dir_bench_shape", "directional", True, 9, "prim", data=(256, 20), dseed=7),
    _case("social_one_tf", "social_default", True, 9, "all", data=(8, 10), dseed=8),
    _case("social_one_free_obs2", "social_default", False, 2, "prim", data=(8, 10), dseed=9),
    _case("social_two_tf", "social_d96", True, 9, "prim", data=(8, 10), dseed=10),
    _case("social_two_free", "social_d96", False, 9, "all", data=(8, 10), dseed=11),
]


def _spec(kind):
    return O.MODEL_SPECS[kind]


def _pool_cfg(kind):
    return O.pool_config(kind)


def _inputs(case):
    _, kind, _, obs_length, _, (B, N), dseed, wseed = case
    ragged = B < 100          # the bench shape is bench.py's scene set: full scenes
    xy, bs = O.synthetic_scenes(B, N, n_frames=obs_length + PRED_LENGTH, seed=dseed, ragged=ragged, nan_tracks=ragged)
    return xy, bs, O.random_weights(kind, seed=wseed, relu_bias=3.0)


def _loss_weights(case, S_pos, S, M, bs):
    rs = np.random.RandomState(17)
    wr = rs.uniform(-1, 1, size=(S, M, 5))
    wp = rs.uniform(-1, 1, size=(S_pos, M, 2)).astype(np.float32)
    if case[4] == "prim":
        keep = np.zeros(M, dtype=bool)
        keep[bs[:-1]] = True
        wr[:, ~keep] = 0.0
        wp[:, ~keep] = 0.0
    return torch.from_numpy(wr), torch.from_numpy(wp)


def _loss(rel, pos, wr, wp):
    return (torch.nan_to_num(rel) * wr.to(rel)).sum() + (torch.nan_to_num(pos) * wp.to(pos)).sum()


def _model(case, W):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    spec = _spec(case[1])
    model = LSTM(pool=GridBasedPooling(**spec) if spec is not None else None)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    return model.cuda()


def _gpu_run(case, model, xy, bs, obs_grad=True, prof=False, observed_device="cuda"):
    """forward + backward of the case's loss.  Returns (observed leaf, positions, kernel names, truth leaf)."""
    from trajnetplusplusbaselines_b200 import _lib
    _, _, teacher, obs_length = case[:4]
    observed = torch.from_numpy(xy[:obs_length].copy()).to(observed_device).requires_grad_(obs_grad)
    truth = torch.from_numpy(xy[obs_length:-1].copy()).cuda().requires_grad_(True) if teacher else None
    kw = dict(prediction_truth=truth) if teacher else dict(n_predict=PRED_LENGTH)
    lib = _lib.load()
    buf = ctypes.create_string_buffer(1 << 16)
    if prof:
        lib.tb2_profile_begin()
    try:
        rel, pos = model(observed, torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), **kw)
        wr, wp = _loss_weights(case, pos.shape[0], rel.shape[0], xy.shape[1], bs)
        model.zero_grad()
        _loss(rel, pos, wr, wp).backward()
    finally:
        if prof:
            _lib.check(lib.tb2_profile_end(buf, len(buf)))
    kernels = set(json.loads(buf.value.decode())) if prof else set()
    return observed, pos.detach().cpu(), kernels, truth


def _restate(case, xy, bs, W, feed_back):
    _, kind, teacher, obs_length = case[:4]
    W64 = {k: torch.tensor(v, dtype=torch.float64) for k, v in W.items()}
    leaf = torch.tensor(xy[:obs_length], dtype=torch.float64, requires_grad=True)
    truth = torch.from_numpy(xy[obs_length:-1]) if teacher else None
    stats = {}
    spec = _spec(kind)
    rel, pos = IR.forward(W64, _pool_cfg(kind) if spec is not None else None, leaf.float(), bs,
                          prediction_truth=truth, n_predict=None if teacher else PRED_LENGTH, stats=stats,
                          feed_back=feed_back)
    wr, wp = _loss_weights(case, pos.shape[0], rel.shape[0], xy.shape[1], bs)
    _loss(rel, pos, wr, wp).backward()
    if spec is not None and spec.get("embedding_arch") is not None:
        assert stats.get("relu_pool0", 0.0) >= RELU_MARGIN, (case[0], stats)
    return leaf.grad.numpy()


def _tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")


def _rel_err(got, ref):
    assert np.isfinite(got).all() and np.isfinite(ref).all()
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_observed_grad_matches_float64_restatement(monkeypatch, case, tc):
    _tc(monkeypatch, tc)
    xy, bs, W = _inputs(case)
    model = _model(case, W)
    observed, pos, kernels, truth = _gpu_run(case, model, xy, bs, prof=True)
    g = observed.grad.cpu().numpy()
    ref = _restate(case, xy, bs, W, feed_back=pos)
    err = _rel_err(g, ref)
    print("%s [%s]: max |d observed - float64| / max |float64| = %.2e" % (case[0], "tc" if tc else "no_tc", err))
    assert err <= TOL, (case[0], err)
    if case[1].startswith("directional") or case[4] == "all":
        # neighbours receive gradient (through the grid's pairs, or their own loss terms)
        nb = np.ones(xy.shape[1], dtype=bool)
        nb[bs[:-1]] = False
        assert np.abs(g[:, nb]).max() > 0
    # the directional pair kernel runs for directional grids only
    assert ("bwd_input_dir_pairs" in kernels) == case[1].startswith("directional"), sorted(kernels)
    assert ("bwd_input_vel" in kernels) != case[1].startswith("directional"), sorted(kernels)
    if truth is not None:
        assert truth.grad is None          # teacher-forced truth is a deep copy in the reference

    # parameter gradients are bit-identical whether or not observed requires grad, and d observed is run-to-run
    # identical
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    observed2, _, _, _ = _gpu_run(case, model, xy, bs)
    assert torch.equal(observed2.grad, observed.grad)
    _gpu_run(case, model, xy, bs, obs_grad=False)
    for k, p in model.named_parameters():
        assert (p.grad is None) == (k not in grads), k
        if p.grad is not None:
            assert torch.equal(p.grad, grads[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("case", [CASES[3], CASES[7]], ids=[CASES[3][0], CASES[7][0]])
def test_frozen_parameters_and_host_observed(case):
    xy, bs, W = _inputs(case)
    model = _model(case, W)
    observed, _, _, _ = _gpu_run(case, model, xy, bs)
    want = observed.grad.cpu()
    model.requires_grad_(False)
    for device in ("cuda", "cpu"):
        obs, _, _, _ = _gpu_run(case, model, xy, bs, observed_device=device)
        assert all(p.grad is None for p in model.parameters())
        assert obs.grad.device.type == device and obs.grad.dtype == torch.float32
        assert torch.equal(obs.grad.cpu(), want)
    # outputs of a frozen model carry a grad_fn only when observed asks for a gradient
    obs = torch.from_numpy(xy[:9].copy()).cuda().requires_grad_()
    rel, pos = model(obs, None, torch.from_numpy(bs), n_predict=PRED_LENGTH)
    assert rel.grad_fn is not None and pos.grad_fn is not None
    rel, pos = model(obs.detach(), None, torch.from_numpy(bs), n_predict=PRED_LENGTH)
    assert rel.grad_fn is None


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the external-module path (tb2_lstm_step_backward's d_obs1 / d_obs2, the padded inputs' backward)
# ---------------------------------------------------------------------------------------------------------------------
class HiddenMLP(torch.nn.Module):
    """HiddenStateMLPPooling (reference non_gridbased_pooling.py:197-239) as a user module, from the restatement
    tests/torch_ref._hidden_mlp: positions, velocities and hidden states all reach its output."""

    def __init__(self, hidden_dim=128, out_dim=64):
        super().__init__()
        self.out_dim = out_dim
        self.spatial_embedding = torch.nn.Linear(2, 16)
        self.vel_embedding = torch.nn.Linear(2, 16)
        self.hidden_embedding = torch.nn.Linear(hidden_dim, 32)
        self.out_projection = torch.nn.Linear(64, out_dim)

    def reset(self, *args, **kwargs):
        pass

    def forward(self, hidden, obs1, obs2):
        B = hidden.shape[0]
        W = {"pool.%s.0.%s" % (m, a): getattr(getattr(self, m), a)
             for m in ("spatial_embedding", "vel_embedding", "hidden_embedding") for a in ("weight", "bias")}
        W.update({"pool.out_projection.weight": self.out_projection.weight,
                  "pool.out_projection.bias": self.out_projection.bias})
        cfg = SimpleNamespace(mlp_dim_hidden=True, mlp_dim_vel=True)
        return torch.cat([TR._hidden_mlp(cfg, W, hidden[b], obs1[b], obs2[b]) for b in range(B)], dim=0)


def _ext_forward64(W, pool, observed, bs, feed_back, obs_length, n_predict, H=128):
    """LSTM.forward (lstm.py:170-264) around `pool` in float64 on the CPU: generate_pooling_inputs, the module, the
    LSTMCell; decoder inputs detached (feed_back = the GPU's positions)."""
    M = observed.shape[1]
    h = torch.zeros(M, H, dtype=torch.float64)
    c = torch.zeros(M, H, dtype=torch.float64)
    bsl = [int(v) for v in bs]

    def step(phase, h, c, o1, o2):
        mask = ~torch.isnan(o1[:, 0]) & ~torch.isnan(o2[:, 0])
        e = torch.relu(((o2 - o1)[mask].double() * 4.0) @ W["input_embedding.input_embeddings.0.weight"].T +
                       W["input_embedding.input_embeddings.0.bias"])
        pooled = pool(TR._pad(h, bsl, float("nan")), TR._pad(o1.double(), bsl, float("nan")),
                      TR._pad(o2.double(), bsl, float("nan")))[TR._pad(mask, bsl, False).reshape(-1)]
        x = torch.cat([e, torch.zeros(e.shape[0], 2, dtype=torch.float64), pooled], dim=1)
        gates = x @ W[phase + ".weight_ih"].T + W[phase + ".bias_ih"] + h[mask] @ W[phase + ".weight_hh"].T + \
            W[phase + ".bias_hh"]
        i, f = torch.sigmoid(gates[:, :H]), torch.sigmoid(gates[:, H:2 * H])
        g, o = torch.tanh(gates[:, 2 * H:3 * H]), torch.sigmoid(gates[:, 3 * H:])
        c2 = f * c[mask] + i * g
        h2 = o * torch.tanh(c2)
        raw = h2 @ W["hidden2normal.linear.weight"].T + W["hidden2normal.linear.bias"]
        nrm = torch.cat([raw[:, :2], 0.01 + 0.2 * torch.sigmoid(raw[:, 2:4]), 0.7 * torch.sigmoid(raw[:, 4:5])], dim=1)
        idx = mask.nonzero().flatten()
        return (h.index_copy(0, idx, h2), c.index_copy(0, idx, c2),
                torch.full((M, 5), float("nan"), dtype=torch.float64).index_copy(0, idx, nrm))

    normals, positions = [], ([observed[-1]] if obs_length == 2 else [])
    for t in range(obs_length - 1):
        h, c, n = step("encoder", h, c, observed[t], observed[t + 1])
        normals.append(n)
        positions.append(observed[t + 1] + n[:, :2].float())
    off = 1 if obs_length == 2 else 0
    for k in range(n_predict - 1):
        s = obs_length - 1 + k
        o1 = feed_back[off + s - 2]
        if k == 0:        # seq[0] is the deep copy of observed[-1]: a tensor, whose primary rows take the fed-back position
            o1 = observed[-1].detach().clone()
            o1[bsl[:-1]] = feed_back[off + s - 2][bsl[:-1]]
        o2 = feed_back[off + s - 1]
        h, c, n = step("decoder", h, c, o1, o2)
        normals.append(n)
        positions.append(o2 + n[:, :2].float())
    return torch.stack(normals), torch.stack(positions)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("obs_length", [9, 2])
def test_external_module_observed_grad(monkeypatch, obs_length, tc):
    import copy
    from trajnetplusplusbaselines_b200.lstm import LSTM
    _tc(monkeypatch, tc)
    xy, bs = O.synthetic_scenes(6, 8, n_frames=obs_length + PRED_LENGTH, seed=31, ragged=True, nan_tracks=True,
                                start_std=3.0)
    torch.manual_seed(41)
    pool = HiddenMLP()
    torch.manual_seed(42)
    model = LSTM(pool=copy.deepcopy(pool))
    W = {k: v.detach().double().clone() for k, v in model.state_dict().items() if not k.startswith("pool.")}
    model = model.cuda()
    observed = torch.from_numpy(xy[:obs_length].copy()).cuda().requires_grad_()
    rel, pos = model(observed, None, torch.from_numpy(bs), n_predict=PRED_LENGTH)
    wr, wp = _loss_weights(("ext", None, False, obs_length, "all"), pos.shape[0], rel.shape[0], xy.shape[1], bs)
    _loss(rel, pos, wr, wp).backward()
    g = observed.grad.cpu().numpy()

    leaf = torch.tensor(xy[:obs_length], dtype=torch.float64, requires_grad=True)
    rel64, pos64 = _ext_forward64(W, pool.double(), leaf.float(), bs, pos.detach().cpu(), obs_length, PRED_LENGTH)
    _loss(rel64, pos64, wr, wp).backward()
    err = _rel_err(g, leaf.grad.numpy())
    print("external obs %d [%s]: max |d observed - float64| / max |float64| = %.2e"
          % (obs_length, "tc" if tc else "no_tc", err))
    assert err <= TOL, err


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the losses' d targets, refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pred", "l2"])
def test_loss_target_gradient_matches_float64(kind):
    from trajnetplusplusbaselines_b200.lstm import L2Loss, PredictionLoss
    rs = np.random.RandomState(3)
    T, M = 12, 30
    bs = np.array([0, 7, 15, 30])
    inputs = np.concatenate([rs.normal(0, 0.3, (T, M, 2)), rs.uniform(0.05, 0.2, (T, M, 2)),
                             rs.uniform(-0.5, 0.5, (T, M, 1))], axis=2).astype(np.float32)
    targets = rs.normal(0, 0.3, (T, M, 2)).astype(np.float32)
    t_gpu = torch.from_numpy(targets).cuda().requires_grad_()
    i_gpu = torch.from_numpy(inputs).cuda().requires_grad_()
    crit = PredictionLoss() if kind == "pred" else L2Loss()
    crit(i_gpu, t_gpu, torch.from_numpy(bs)).backward()
    t64 = torch.tensor(targets, dtype=torch.float64, requires_grad=True)
    i64 = torch.tensor(inputs, dtype=torch.float64)
    (TR.prediction_loss(i64, t64, bs) if kind == "pred" else TR.l2_loss(i64, t64, bs)).backward()
    assert _rel_err(t_gpu.grad.cpu().numpy(), t64.grad.numpy()) <= 1e-5
    assert torch.equal(t_gpu.grad[..., :2], -i_gpu.grad[..., :2])


@pytest.mark.gpu
def test_refusals():
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, HiddenStateMLPPooling
    from trajnetplusplusbaselines_b200.lstm.trainer import GOALS_MESSAGE
    from trajnetplusplusbaselines_b200.sgan import LSTMDiscriminator, LSTMGenerator
    from trajnetplusplusbaselines_b200.vae import VAE
    xy, bs = O.synthetic_scenes(2, 4, n_frames=9 + PRED_LENGTH, seed=2)
    split = torch.from_numpy(bs)
    obs = torch.from_numpy(xy[:9].copy()).cuda().requires_grad_()
    M = xy.shape[1]

    goal = LSTM(goal_flag=True).cuda().requires_grad_(False)
    with pytest.raises(NotImplementedError, match=re.escape(GOALS_MESSAGE[:40])):
        goal(obs, torch.zeros(M, 2), split, n_predict=PRED_LENGTH)
    nongrid = LSTM(pool=HiddenStateMLPPooling(hidden_dim=128)).cuda().requires_grad_(False)
    with pytest.raises(NotImplementedError, match="inference only"):
        nongrid(obs, None, split, n_predict=PRED_LENGTH)
    gen = LSTMGenerator(pool=GridBasedPooling(type_="directional", hidden_dim=128)).cuda().requires_grad_(False)
    with pytest.raises(NotImplementedError, match="inputs"):
        gen(obs, None, split, n_predict=PRED_LENGTH)
    disc = LSTMDiscriminator().cuda().requires_grad_(False)
    with pytest.raises(NotImplementedError, match="inputs"):
        disc(obs, torch.zeros(PRED_LENGTH, M, 2).cuda(), None, split)
    vae = VAE().cuda().eval().requires_grad_(False)
    with pytest.raises(NotImplementedError, match="inputs"):
        vae(obs, None, split, n_predict=PRED_LENGTH)
    # without grad mode, the same calls run
    with torch.no_grad():
        gen(obs, None, split, n_predict=PRED_LENGTH)
