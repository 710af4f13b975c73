"""The training backward's NULL-field rule (tb2_lstm_grads): tb2_lstm_sequence_backward and tb2_lstm_rollout_backward
compute only the gradients they are given, and d observed is the same bits whichever parameter fields are set.

Each backward call autograd makes is repeated through ctypes, with the call's own arguments, once per field set: all
parameter fields, none, the encoder's only and the pool's only, each with fresh zeroed buffers.
"""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import lstm_oracle as O  # noqa: E402

PRED_LENGTH = 12
KINDS = ["vanilla", "occupancy", "directional", "social_default", "social_d96"]     # social_d96: two_layer, latent 16


def _model(kind, H, seed):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, LSTM
    spec = O.MODEL_SPECS[kind]
    pool = GridBasedPooling(**dict(spec, hidden_dim=H)) if spec is not None else None
    model = LSTM(hidden_dim=H, pool=pool)
    W = O.random_weights(kind, seed=seed, hidden_dim=H, relu_bias=3.0)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    return model.cuda()


def _scenes(kind, seed):
    B, N = (6, 8) if kind.startswith("social") else (10, 8)
    return O.synthetic_scenes(B, N, n_frames=9 + PRED_LENGTH, seed=seed, ragged=True, nan_tracks=True)


def _loss(rel, pos, seed):
    rs = np.random.RandomState(seed)
    wr = torch.from_numpy(rs.uniform(-1, 1, size=tuple(rel.shape))).to(rel)
    wp = torch.from_numpy(rs.uniform(-1, 1, size=tuple(pos.shape))).to(pos)
    return (torch.nan_to_num(rel) * wr).sum() + (torch.nan_to_num(pos) * wp).sum()


def _subsets(names):
    enc = [k for k in names if k.startswith("encoder_")]
    pool = [k for k in names if k.startswith("pool_")]
    out = {"all": list(names), "none": [], "encoder": enc}
    if pool:
        out["pool"] = pool
    return out


def _replay(monkeypatch, results):
    """Wrap training._run_backward: after each real call, repeat it once per field subset into `results`."""
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import training as T
    run = T._run_backward

    def wrapped(ctx, active, d_obs, launch):
        targets = T._grad_targets(ctx.model)

        def spy(lib, handle, w, g, *rest):
            rc = launch(lib, handle, w, g, *rest)
            out = {}
            for name, fields in _subsets(targets).items():
                g2 = _lib.LstmGrads()
                bufs = {k: torch.zeros_like(targets[k], dtype=torch.float32) for k in fields}
                for k, t in bufs.items():
                    setattr(g2, k, t.data_ptr())
                d2 = torch.zeros_like(d_obs)
                g2.d_observed = d2.data_ptr()
                _lib.check(launch(lib, handle, w, g2, *rest))
                out[name] = (d2, bufs)
            torch.cuda.synchronize()
            results.append(out)
            return rc
        return run(ctx, active, d_obs, spy)
    monkeypatch.setattr(T, "_run_backward", wrapped)


def _check_subsets(out):
    d_all, g_all = out["all"]
    assert float(d_all.abs().max()) > 0
    assert any(float(t.abs().max()) > 0 for t in g_all.values())
    for name, (d, bufs) in out.items():
        assert torch.equal(d, d_all), name
        for k, t in bufs.items():
            assert torch.equal(t, g_all[k]), (name, k)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [64, 128])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("call", ["sequence", "rollout"])
def test_d_observed_does_not_depend_on_parameter_fields(monkeypatch, call, kind, H):
    from trajnetplusplusbaselines_b200.lstm import differentiable_rollout
    seed = 5 + KINDS.index(kind)
    model = _model(kind, H, seed)
    xy, bs = _scenes(kind, seed)
    results = []
    _replay(monkeypatch, results)
    observed = torch.from_numpy(xy[:9].copy()).cuda().requires_grad_()
    split = torch.from_numpy(bs)
    if call == "sequence":
        truth = torch.from_numpy(xy[9:-1].copy()).cuda()
        rel, pos = model(observed, None, split, truth)
    else:
        rel, pos = differentiable_rollout(model, observed, split, PRED_LENGTH)
    _loss(rel, pos, seed).backward()
    assert len(results) == 1
    _check_subsets(results[0])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_rollout_without_parameters(kind):
    """parameters=False: observed.grad is parameters=True's, bit for bit, and no parameter's .grad is touched."""
    from trajnetplusplusbaselines_b200.lstm import differentiable_rollout
    seed = 31 + KINDS.index(kind)
    model = _model(kind, 128, seed)
    xy, bs = _scenes(kind, seed)
    grads = []
    for parameters in (True, False):
        model.zero_grad(set_to_none=True)
        if not parameters:
            for p in model.parameters():
                p.grad = torch.full_like(p, 0.5)
        observed = torch.from_numpy(xy[:9].copy()).cuda().requires_grad_()
        rel, pos = differentiable_rollout(model, observed, torch.from_numpy(bs), PRED_LENGTH, parameters=parameters)
        if not parameters:
            assert all(p.requires_grad for p in model.parameters())
        _loss(rel, pos, seed).backward()
        grads.append(observed.grad.clone())
        if parameters:
            assert any(p.grad is not None and float(p.grad.abs().max()) > 0 for p in model.parameters())
        else:
            assert all(torch.equal(p.grad, torch.full_like(p, 0.5)) for p in model.parameters())
    assert torch.equal(grads[0], grads[1])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["directional", "social_default"])
def test_frozen_model_gets_the_same_d_observed(kind):
    """A frozen model's sequence backward is the inputs-only call; its d observed equals the trainable model's."""
    seed = 41 + KINDS.index(kind)
    model = _model(kind, 128, seed)
    xy, bs = _scenes(kind, seed)
    truth = torch.from_numpy(xy[9:-1].copy()).cuda()
    out = []
    for frozen in (False, True):
        model.requires_grad_(not frozen)
        model.zero_grad(set_to_none=True)
        observed = torch.from_numpy(xy[:9].copy()).cuda().requires_grad_()
        rel, pos = model(observed, None, torch.from_numpy(bs), truth)
        _loss(rel, pos, seed).backward()
        out.append(observed.grad.clone())
        if frozen:
            assert all(p.grad is None for p in model.parameters())
    assert torch.equal(out[0], out[1])

