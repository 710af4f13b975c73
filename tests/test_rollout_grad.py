"""lstm.differentiable_rollout / tb2_lstm_rollout_backward: the gradient of a free-running forecast with nothing detached,
against a float64 autograd restatement built from tests/input_grad_ref.step with the decoder fed its own positions.

The restatement feeds each fed-back position in the straight-through form own + (gpu - own).detach(): its value is the
GPU's, so every grid cell is binned alike, and its gradient is the restatement's own.
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import input_grad_ref as IR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402

PRED_LENGTH = 12
TOL = 1e-4              # max |gpu - float64| / max |float64| per tensor


def _case(name, kind, obs_length, loss, H=128, data=(10, 8), dseed=1):
    return (name, kind, obs_length, loss, H, data, dseed)


CASES = [
    _case("vanilla_all", "vanilla", 9, "all"),
    _case("vanilla_prim_obs2_h64", "vanilla", 2, "prim", H=64, dseed=2),
    _case("occ_prim", "occupancy", 9, "prim", dseed=3),
    _case("occ_all_obs2_h192", "occupancy", 2, "all", H=192, dseed=4),
    _case("dir_prim", "directional", 9, "prim", dseed=5),
    _case("dir_all_obs2", "directional", 2, "all", dseed=6),
    _case("dir_all_h64", "directional", 9, "all", H=64, dseed=7),
    _case("social_one_all", "social_default", 9, "all", data=(6, 8), dseed=8),
    _case("social_one_prim_obs2_h192", "social_default", 2, "prim", H=192, data=(6, 8), dseed=9),
    _case("social_two_prim", "social_d96", 9, "prim", data=(6, 8), dseed=10),
    _case("social_two_all_obs2", "social_d96", 2, "all", data=(6, 8), dseed=11),
]


def _inputs(case):
    _, kind, obs_length, _, H, (B, N), dseed = case
    xy, bs = O.synthetic_scenes(B, N, n_frames=obs_length + PRED_LENGTH, seed=dseed, ragged=True, nan_tracks=True)
    return xy, bs, O.random_weights(kind, seed=dseed, hidden_dim=H, relu_bias=3.0)


def _model(case, W):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    spec = O.MODEL_SPECS[case[1]]
    H = case[4]
    pool = GridBasedPooling(**dict(spec, hidden_dim=H)) if spec is not None else None
    model = LSTM(hidden_dim=H, pool=pool)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    return model.cuda()


def _weights(case, S_pos, S, M, bs):
    rs = np.random.RandomState(23)
    wr = torch.from_numpy(rs.uniform(-1, 1, size=(S, M, 5)))
    wp = torch.from_numpy(rs.uniform(-1, 1, size=(S_pos, M, 2)))
    if case[3] == "prim":
        keep = torch.zeros(M, dtype=torch.bool)
        keep[torch.from_numpy(bs[:-1])] = True
        wr[:, ~keep] = 0.0
        wp[:, ~keep] = 0.0
    return wr, wp


def _loss(rel, pos, wr, wp):
    return (torch.nan_to_num(rel) * wr.to(rel)).sum() + (torch.nan_to_num(pos) * wp.to(pos)).sum()


def restate(W, pool_cfg, observed, bs, n_predict, H, gpu_pos, stats=None):
    """Float64 restatement of the free-running forward with the fed-back positions NOT detached.  observed: fp32 (an
    fp64 leaf cast); gpu_pos: the GPU's positions [S(+1), M, 2] fed in the straight-through form."""
    bs = [int(v) for v in bs]
    prim = torch.tensor(bs[:-1])
    M = observed.shape[1]
    h = torch.zeros(M, H, dtype=torch.float64)
    c = torch.zeros(M, H, dtype=torch.float64)
    normals, positions = [], ([observed[-1]] if observed.shape[0] == 2 else [])

    def fed(i):
        own = positions[i]
        return own + (gpu_pos[i] - own).detach()

    for t in range(observed.shape[0] - 1):
        h, c, normal = IR.step(W, pool_cfg, "encoder", h, c, observed[t], observed[t + 1], bs, H, torch.float64, stats)
        normals.append(normal)
        positions.append(observed[t + 1] + normal[:, :2].float())
    for k in range(n_predict - 1):
        L = len(positions)
        if k == 0:                  # lstm.py:240-241: the copy of observed[-1], primaries from positions[-2]
            obs1 = observed[-1].clone()
            obs1[prim] = fed(L - 2)[prim]
        else:
            obs1 = fed(L - 2)
        obs2 = fed(L - 1)
        h, c, normal = IR.step(W, pool_cfg, "decoder", h, c, obs1, obs2, bs, H, torch.float64, stats)
        normals.append(normal)
        positions.append(obs2 + normal[:, :2].float())
    return torch.stack(normals), torch.stack(positions)


def _tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")


def _rel_err(got, ref):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert np.isfinite(got).all() and np.isfinite(ref).all()
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


def _gpu(case, model, xy, bs):
    from trajnetplusplusbaselines_b200.lstm import differentiable_rollout
    observed = torch.from_numpy(xy[:case[2]].copy()).cuda().requires_grad_()
    rel, pos = differentiable_rollout(model, observed, torch.from_numpy(bs), PRED_LENGTH)
    wr, wp = _weights(case, pos.shape[0], rel.shape[0], xy.shape[1], bs)
    model.zero_grad()
    _loss(rel, pos, wr, wp).backward()
    return observed, rel.detach(), pos.detach()


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_rollout_grad_matches_float64_restatement(monkeypatch, case, tc):
    _tc(monkeypatch, tc)
    xy, bs, W = _inputs(case)
    model = _model(case, W)
    observed, rel, pos = _gpu(case, model, xy, bs)
    # the forward is LSTM.forward's, bit for bit
    with torch.no_grad():
        rel0, pos0 = model(observed.detach(), None, torch.from_numpy(bs), n_predict=PRED_LENGTH)
    assert torch.equal(torch.nan_to_num(rel, 7.0), torch.nan_to_num(rel0, 7.0))
    assert torch.equal(torch.nan_to_num(pos, 7.0), torch.nan_to_num(pos0, 7.0))
    # restatement
    spec = O.MODEL_SPECS[case[1]]
    W64 = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in W.items()}
    leaf = torch.tensor(xy[:case[2]], dtype=torch.float64, requires_grad=True)
    stats = {}
    rel_r, pos_r = restate(W64, O.pool_config(case[1]) if spec is not None else None, leaf.float(), bs, PRED_LENGTH,
                           case[4], pos.cpu(), stats)
    wr, wp = _weights(case, pos_r.shape[0], rel_r.shape[0], xy.shape[1], bs)
    _loss(rel_r, pos_r, wr, wp).backward()
    g = observed.grad.cpu().numpy()
    err = _rel_err(g, leaf.grad.numpy())
    print("%s [%s]: d observed %.2e" % (case[0], "tc" if tc else "no_tc", err))
    assert err <= TOL, (case[0], err)
    # the gradient differs from LSTM.forward's detached one: the fed-back positions carry gradient
    assert np.abs(g[-1]).max() > 0
    for name, p in model.named_parameters():
        ref = W64[name].grad
        if ref is None or not torch.any(ref != 0):
            assert p.grad is None or not torch.any(p.grad != 0), name
            continue
        e = _rel_err(p.grad.cpu().numpy(), ref.numpy())
        assert e <= TOL, (case[0], name, e)
    if case[1] == "directional":
        nb = np.ones(xy.shape[1], dtype=bool)
        nb[bs[:-1]] = False
        assert np.abs(g[:, nb]).max() > 0
    # run to run identical
    d1 = observed.grad.clone()
    grads = {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}
    observed2, _, _ = _gpu(case, model, xy, bs)
    assert torch.equal(observed2.grad, d1)
    for k, p in model.named_parameters():
        if k in grads:
            assert torch.equal(p.grad, grads[k]), k


@pytest.mark.gpu
def test_frozen_parameters_and_host_observed():
    from trajnetplusplusbaselines_b200.lstm import differentiable_rollout
    case = CASES[4]
    xy, bs, W = _inputs(case)
    model = _model(case, W)
    observed, _, _ = _gpu(case, model, xy, bs)
    want = observed.grad.cpu()
    model.requires_grad_(False)
    model.zero_grad(set_to_none=True)
    for device in ("cuda", "cpu"):
        obs = torch.from_numpy(xy[:9].copy()).to(device).requires_grad_()
        rel, pos = differentiable_rollout(model, obs, torch.from_numpy(bs), PRED_LENGTH)
        wr, wp = _weights(case, pos.shape[0], rel.shape[0], xy.shape[1], bs)
        _loss(rel, pos, wr, wp).backward()
        assert all(p.grad is None for p in model.parameters())
        assert obs.grad.device.type == device and torch.equal(obs.grad.cpu(), want)


def test_refusals():
    """Goal models, the non-grid modules, user-defined modules and S-GAN's generator are refused before anything runs."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, differentiable_rollout, NearestNeighborMLP
    from trajnetplusplusbaselines_b200.sgan.sgan import LSTMGenerator
    from test_input_grad import HiddenMLP
    obs = torch.zeros(9, 2, 2)
    bs = torch.tensor([0, 2])
    for model, word in ((LSTM(goal_flag=True), "goal"), (LSTM(pool=NearestNeighborMLP()), "NearestNeighborMLP"),
                        (LSTMGenerator(), "LSTMGenerator"), (LSTM(pool=HiddenMLP()), "HiddenMLP")):
        with pytest.raises(NotImplementedError, match=word):
            differentiable_rollout(model, obs, bs, PRED_LENGTH)


def test_rollout_backward_refuses_goal_models_and_missing_buffers():
    """On the C boundary: no d_positions / d_observed is an invalid call, checked before anything else."""
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    g = _lib.LstmGrads()
    rc = lib.tb2_lstm_rollout_backward(None, None, None, None, 9, 11, None, None, None, None, None, 0, g, None, 0, None,
                                       0, None, 0, None)
    assert rc == -1 and b"d_positions" in lib.tb2_last_error()
