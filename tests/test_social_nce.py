"""Social-NCE training (lstm/contrast.py, csrc/contrast.cu, DESIGN.md §1 A24) and the hidden-state gradients of the
training backward it rests on (tb2_lstm_sequence_backward_dh, lstm.training.sequence_with_hidden).

On the CPU: a float64 restatement of the term, pinned to a closed-form case; the CLI and API refusals; a zero weight
builds no heads and draws no numbers.  On the GPU (tensor cores on and off):
  * d_hidden = 0 gives the gradients of tb2_lstm_sequence_backward, bit for bit;
  * a loss task + sum C . h against float64 autograd through tests/torch_ref.step, every gradient tensor;
  * the term against the restatement: loss, d h and every head gradient; per-scene results bit-identical alone and in a
    batch, and from run to run; no host synchronisation;
  * whole Trainer.train_batch steps with the term against the float64 restatement of task + NCE;
  * contrast_weight = 0 is today's loop bit for bit, and the CLI trains, resumes and evaluates.
"""
import ctypes
import json
import math
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_hidden_dim_golden import pool_config, pool_spec, weights  # noqa: E402
from trajnetplusplusbaselines_b200.lstm import trainer as TRN  # noqa: E402

RELU_MARGIN = 1e-2      # smallest |pre-activation| of a pool Linear (relu_bias = 3 weights)
OBS, PRED = 9, 12


# ---------------------------------------------------------------------------------------------------------------------
# the float64 restatement of the term
# ---------------------------------------------------------------------------------------------------------------------
def _normalize(v):
    return v / v.norm(dim=-1, keepdim=True).clamp(min=1e-12)


def snce_restated(scene, hidden, bs, obs_length, horizon, params, temperature=0.1, rho=0.2, sigma=0.05, eps=None,
                  logits_out=None):
    """L_nce, terms [B, horizon] and valid [B, horizon] in float64.  scene [T, M, 2] (data), hidden [M, H] and params
    (W1, b1, W2, b2, V1, c1, V2, c2) float64 tensors (autograd follows them), eps [B, horizon, 1 + 8 (n_max - 1), 2]."""
    W1, b1, W2, b2, V1, c1, V2, c2 = params
    X = torch.as_tensor(scene).to(torch.float64)
    eps = torch.as_tensor(eps).to(torch.float64)
    bs = [int(v) for v in bs]
    f0 = obs_length - 1
    ang = torch.arange(8, dtype=torch.float64) * math.pi / 4
    ring = rho * torch.stack([torch.cos(ang), torch.sin(ang)], dim=1)
    terms, valid = [], []
    for b in range(len(bs) - 1):
        p, n = bs[b], bs[b + 1] - bs[b]
        q = _normalize(torch.relu(hidden[p] @ V1.T + c1) @ V2.T + c2)
        x0 = X[f0, p]
        for d in range(1, horizon + 1):
            f = f0 + d
            if not (torch.isfinite(X[f, p]).all() and torch.isfinite(x0).all()):
                terms.append(torch.zeros((), dtype=torch.float64))
                valid.append(0.0)
                continue
            samples = [(X[f, p] - x0 + sigma * eps[b, d - 1, 0])[None]]
            for jj in range(n - 1):
                xj = X[f, p + 1 + jj]
                if torch.isfinite(xj).all():
                    samples.append(xj - x0 + ring + sigma * eps[b, d - 1, 1 + 8 * jj:9 + 8 * jj])
            s = torch.cat(samples)
            inp = torch.cat([s, torch.full((s.shape[0], 1), float(d), dtype=torch.float64)], dim=1)
            keys = _normalize(torch.relu(inp @ W1.T + b1) @ W2.T + b2)
            logits = keys @ q / temperature
            if logits_out is not None:
                logits_out.append(logits.detach())
            terms.append(torch.logsumexp(logits, 0) - logits[0])
            valid.append(1.0)
    terms = torch.stack(terms).reshape(len(bs) - 1, horizon)
    valid = torch.tensor(valid, dtype=torch.float64).reshape(len(bs) - 1, horizon)
    return terms.sum() / max(float(valid.sum()), 1.0), terms, valid


def _params64(module):
    return [p.detach().cpu().to(torch.float64).requires_grad_(True) for p in module.parameters()]


def test_restatement_closed_form():
    """One neighbour, sigma = 0, and weights for which keys and query are known unit vectors: the key of (x, y) is
    (x, y, 0, 0) / |(x, y)| and the query (1, 0, 0, 0).  The positive (1, 0) has logit 1 / tau, the eight negatives at
    (0, 1) (rho = 0) logit 0; at horizon 2 the positive is NaN, so the mean is over one pair."""
    tau = 0.5
    D, H = 16, 3
    W1 = torch.zeros(D, 3, dtype=torch.float64)
    W1[0, 0] = W1[1, 1] = 1.0
    b1 = torch.zeros(D, dtype=torch.float64)
    b1[:2] = 10.0                          # relu(x + 10) = x + 10 for |x| < 10
    W2 = torch.zeros(4, D, dtype=torch.float64)
    W2[0, 0] = W2[1, 1] = 1.0
    b2 = torch.tensor([-10.0, -10.0, 0.0, 0.0], dtype=torch.float64)
    V1 = torch.zeros(D, H, dtype=torch.float64)
    c1 = torch.zeros(D, dtype=torch.float64)
    c1[0] = 2.0
    V2 = torch.zeros(4, D, dtype=torch.float64)
    V2[0, 0] = 1.0
    c2 = torch.zeros(4, dtype=torch.float64)
    params = [W1, b1, W2, b2, V1, c1, V2, c2]
    scene = np.zeros((OBS + 2, 2, 2), dtype=np.float32)
    scene[OBS, 0] = (1.0, 0.0)            # the primary at horizon 1, relative to its last observation (0, 0)
    scene[OBS, 1] = (0.0, 1.0)            # the neighbour
    scene[OBS + 1, 0] = np.nan
    eps = np.zeros((1, 2, 9, 2))
    hidden = torch.zeros(2, H, dtype=torch.float64)
    loss, terms, valid = snce_restated(scene, hidden, [0, 2], OBS, 2, params, temperature=tau, rho=0.0, sigma=0.0,
                                       eps=eps)
    expect = math.log(math.exp(1 / tau) + 8.0) - 1 / tau
    assert abs(float(terms[0, 0]) - expect) < 1e-12 and float(terms[0, 1]) == 0.0
    assert valid.tolist() == [[1.0, 0.0]]
    assert abs(float(loss) - expect) < 1e-12
    # no negatives: exactly 0
    scene[OBS, 1] = np.nan
    loss, terms, _ = snce_restated(scene, hidden, [0, 2], OBS, 2, params, temperature=tau, rho=0.0, sigma=0.0, eps=eps)
    assert float(terms[0, 0]) == 0.0 and float(loss) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# refusals and the zero weight (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("argv, flag", [
    (["--contrast_weight", "-1"], "--contrast_weight"),
    (["--contrast_weight", "1", "--contrast_horizon", "0"], "--contrast_horizon"),
    (["--contrast_weight", "1", "--contrast_horizon", "13"], "--contrast_horizon"),
    (["--contrast_weight", "1", "--contrast_temperature", "0"], "--contrast_temperature"),
    (["--contrast_weight", "1", "--adv_eps", "0.1"], "--adv_eps"),
])
def test_cli_refuses_bad_contrast_flags(argv, flag, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit) as e:
        TRN.main(["--path", "nowhere", "--type", "directional"] + argv)
    assert flag in str(e.value.code)
    assert os.listdir(tmp_path) == []


class _Reached(Exception):
    pass


@pytest.mark.parametrize("argv", [["--pred_length", "1"], ["--pred_length", "3"],
                                  ["--contrast_horizon", "0", "--contrast_temperature", "-1", "--adv_eps", "0.1"]])
def test_cli_ignores_contrast_flags_when_the_term_is_off(argv, tmp_path, monkeypatch):
    """Without --contrast_weight the term's flags are not checked: a pred_length below the default horizon of 4 trains
    as before (the CLI goes on to build the model)."""
    monkeypatch.chdir(tmp_path)

    def reached(args):
        raise _Reached
    monkeypatch.setattr(TRN, "build_model", reached)
    with pytest.raises(_Reached):
        TRN.main(["--path", "nowhere", "--type", "directional"] + argv)


def test_cli_keeps_the_training_refusals_first(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit) as e:
        TRN.main(["--path", "nowhere", "--type", "hiddenstatemlp", "--contrast_weight", "1"])
    assert "training of HiddenStateMLPPooling is not built" in str(e.value.code)
    assert os.listdir(tmp_path) == []


def test_trainer_refusals():
    from test_input_grad import HiddenMLP
    from trajnetplusplusbaselines_b200.lstm import LSTM, HiddenStateMLPPooling
    from trajnetplusplusbaselines_b200.lstm.contrast import SocialNCE
    cpu = torch.device("cpu")
    with pytest.raises(NotImplementedError, match="training of HiddenStateMLPPooling is not built"):
        TRN.Trainer(LSTM(pool=HiddenStateMLPPooling()), device=cpu, contrast_weight=1.0)
    with pytest.raises(NotImplementedError, match="user-defined"):
        TRN.Trainer(LSTM(pool=HiddenMLP()), device=cpu, contrast_weight=1.0)
    with pytest.raises(ValueError, match="adv_eps"):
        TRN.Trainer(LSTM(), device=cpu, contrast_weight=1.0, adv_eps=0.1)
    with pytest.raises(ValueError, match="contrast_weight"):
        TRN.Trainer(LSTM(), device=cpu, contrast_weight=-1.0)
    with pytest.raises(ValueError, match="horizon"):
        TRN.Trainer(LSTM(), device=cpu, contrast_weight=1.0, pred_length=3)          # the default horizon is 4
    with pytest.raises(ValueError, match="hidden_dim"):
        TRN.Trainer(LSTM(hidden_dim=64), device=cpu, contrast_weight=1.0, contrast=SocialNCE(128))
    for kw in (dict(temperature=0.0), dict(horizon=0), dict(mlp_dim=48), dict(head_dim=3)):
        with pytest.raises(ValueError):
            SocialNCE(128, **kw)


def test_zero_weight_builds_no_heads_and_draws_nothing():
    from trajnetplusplusbaselines_b200.lstm import LSTM
    torch.manual_seed(0)
    model = LSTM()
    state = torch.get_rng_state()
    trainer = TRN.Trainer(model, device=torch.device("cpu"), contrast_weight=0.0)
    assert trainer.contrast is None and len(trainer.optimizer.param_groups) == 1
    assert torch.equal(torch.get_rng_state(), state)
    assert set(trainer._state(0)) == {"epoch", "state_dict", "optimizer", "scheduler"}
    # with the term on, the heads are built after the model and join the optimizer
    trainer = TRN.Trainer(LSTM(), device=torch.device("cpu"), contrast_weight=1.0)
    assert trainer.contrast is not None and len(trainer.optimizer.param_groups) == 2
    assert "contrast" in trainer._state(0)


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def _tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")     # read when the model's handle is created


def _model(kind, H, W):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    spec = pool_spec(kind, H)
    model = LSTM(hidden_dim=H, pool=GridBasedPooling(**spec) if spec is not None else None)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    return model.cuda().train()


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def restated_sequence(W_np, cfg, xy, bs, H, feed_back, obs_length=OBS, stats=None):
    """The teacher-forced forward of tests/torch_ref in float64, through torch_ref.step, with every step's h:
    (W, rel [S, M, 5], hidden [S, M, H]).  The decoder is fed the (detached) positions feed_back [S, M, 2] of the GPU's
    forward, so the gradients are exact for its trajectory."""
    W = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in W_np.items()}
    X = torch.tensor(xy)
    fb = torch.as_tensor(feed_back)
    prim = torch.tensor([int(v) for v in bs[:-1]])
    M = xy.shape[1]
    h = torch.zeros(M, H, dtype=torch.float64)
    c = torch.zeros(M, H, dtype=torch.float64)
    normals, hs = [], []

    def step(phase, h, c, o1, o2):
        return TR.step(W, cfg, phase, h, c, o1, o2, bs, H, torch.float64, stats=stats)
    for t in range(obs_length - 1):
        h, c, nrm = step("encoder", h, c, X[t], X[t + 1])
        normals.append(nrm)
        hs.append(h)
    S_enc = obs_length - 1
    seq = [X[obs_length - 1].clone()] + [X[t].clone() for t in range(obs_length, X.shape[0] - 1)]
    for k in range(len(seq) - 1):
        o1 = seq[k].clone()
        o1[prim] = fb[S_enc + k - 2][prim]
        o2 = seq[k + 1].clone()
        o2[prim] = fb[S_enc + k - 1][prim]
        seq[k + 1] = o2
        h, c, nrm = step("decoder", h, c, o1, o2)
        normals.append(nrm)
        hs.append(h)
    return W, torch.stack(normals), torch.stack(hs)


def _task_restated(rel, xy, bs, obs_length=OBS, pred_length=PRED):
    X = torch.tensor(xy)
    targets = (X[obs_length:obs_length + pred_length] - X[obs_length - 1:obs_length + pred_length - 1]).double()
    return TR.prediction_loss(rel[-pred_length:], targets, bs) * (len(bs) - 1)


def _task(rel, scene, batch_split, obs_length=OBS, pred_length=PRED):
    from trajnetplusplusbaselines_b200.lstm import PredictionLoss
    targets = scene[obs_length:obs_length + pred_length] - scene[obs_length - 1:obs_length + pred_length - 1]
    return PredictionLoss()(rel[-pred_length:], targets, batch_split) * (len(batch_split) - 1)


def _check_relu(stats, kind):
    if pool_spec(kind, 128) is not None:
        relu = [v for k, v in stats.items() if k.startswith("relu_pool")]
        assert relu and min(relu) >= RELU_MARGIN, (kind, stats)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the hidden-state gradients of the training backward
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", ["vanilla", "directional", "social_default"])
def test_zero_d_hidden_equals_the_plain_backward(monkeypatch, kind, tc):
    from trajnetplusplusbaselines_b200.lstm.training import sequence_with_hidden
    _tc(monkeypatch, tc)
    xy, bs = O.synthetic_scenes(6, 8, seed=61, ragged=True, nan_tracks=True)
    W = weights(kind, 128, seed=62)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    grads = []
    for with_hidden in (False, True):
        model = _model(kind, 128, W)
        if with_hidden:
            rel, pos, hid = sequence_with_hidden(model, scene[:OBS], split, scene[OBS:-1].clone(), None)
            loss = _task(rel, scene, split) + 0.0 * hid.sum()
        else:
            rel, pos = model(scene[:OBS], torch.zeros(xy.shape[1], 2), split, scene[OBS:-1].clone())
            loss = _task(rel, scene, split)
        outputs = (rel.detach(), pos.detach())
        loss.backward()
        grads.append((outputs, {n: p.grad for n, p in model.named_parameters()}))
    (o0, g0), (o1, g1) = grads
    assert torch.equal(o0[0].nan_to_num(), o1[0].nan_to_num()) and torch.equal(o0[1].nan_to_num(), o1[1].nan_to_num())
    assert g0.keys() == g1.keys()
    for n in g0:
        assert (g0[n] is None) == (g1[n] is None), (kind, n)
        assert g0[n] is None or torch.equal(g0[n], g1[n]), (kind, n)


def _hidden_data(seed):
    """Ragged scenes whose tracks enter late (absent at frames 0-2) and, for two more, leave after frame 5."""
    xy, bs = O.synthetic_scenes(6, 9, seed=seed, ragged=True, nan_tracks=True)
    xy = xy.copy()
    prim = set(int(v) for v in bs[:-1])
    full = [m for m in range(xy.shape[1]) if m not in prim and not np.isnan(xy[:, m]).any()]
    xy[6:, full[0]] = xy[6:, full[-1]] = np.nan
    return xy, bs


def _hidden_weights(xy, bs, S, H, seed):
    """C [S, M, H]: random rows at chosen (step, track) pairs: late-entering tracks at absent and present steps,
    leaving tracks after they left (a carried state), the last step, primaries and random rows."""
    rng = np.random.RandomState(seed)
    M = xy.shape[1]
    prim = set(int(v) for v in bs[:-1])
    late = [m for m in range(M) if np.isnan(xy[0, m, 0]) and not np.isnan(xy[OBS - 1, m, 0])]
    gone = [m for m in range(M) if m not in prim and np.isnan(xy[OBS - 1, m, 0]) and not np.isnan(xy[0, m, 0])]
    assert late and len(gone) == 2, "the data must have entering and leaving tracks"
    pairs = {(0, late[0]), (1, late[0]), (4, late[0]), (S - 1, late[-1]), (S - 1, gone[0]), (OBS - 2, gone[-1]),
             (S - 1, int(bs[0])), (OBS - 2, int(bs[1])), (OBS + 1, int(bs[-2]))}
    for _ in range(6):
        pairs.add((int(rng.randint(S)), int(rng.randint(M))))
    C = np.zeros((S, M, H))
    for s, m in sorted(pairs):
        C[s, m] = rng.randn(H) * 0.3
    return C


HIDDEN_KINDS = ["vanilla", "occupancy", "directional", "social_default", "social_small"]


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("H", [32, 128, 256])
@pytest.mark.parametrize("kind", HIDDEN_KINDS)
def test_d_hidden_matches_float64(monkeypatch, kind, H, tc):
    from trajnetplusplusbaselines_b200.lstm.training import sequence_with_hidden
    _tc(monkeypatch, tc)
    xy, bs = _hidden_data(70 + H // 32)
    S = xy.shape[0] - 2
    W = weights(kind, H, seed=H + 11)
    C = _hidden_weights(xy, bs, S, H, seed=H)
    model = _model(kind, H, W)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    rel, pos, hid = sequence_with_hidden(model, scene[:OBS], split, scene[OBS:-1].clone(), None)
    with torch.no_grad():
        rel0, pos0 = model(scene[:OBS], torch.zeros(xy.shape[1], 2), split, scene[OBS:-1].clone())
    assert torch.equal(rel.detach().nan_to_num(), rel0.nan_to_num()) and torch.equal(pos.detach().nan_to_num(),
                                                                                    pos0.nan_to_num())
    loss = _task(rel, scene, split) + (torch.from_numpy(C).float().cuda() * hid).sum()
    loss.backward()

    stats = {}
    W64, rel64, hid64 = restated_sequence(W, pool_config(kind, H), xy, bs, H, pos.detach().cpu().numpy(), stats=stats)
    _check_relu(stats, kind)
    assert float((hid.detach().cpu().double() - hid64.detach()).abs().max()) < 1e-4
    loss64 = _task_restated(rel64, xy, bs) + (torch.from_numpy(C) * hid64).sum()
    loss64.backward()
    assert abs(float(loss) - float(loss64)) <= 1e-4 * abs(float(loss64)), (float(loss), float(loss64))
    worst = 0.0
    for name, p in model.named_parameters():
        g_ref = W64[name].grad if name in W64 else None
        if g_ref is None:             # the goal embedding, which a model without goals does not use
            assert p.grad is None or not p.grad.any(), name
            continue
        assert p.grad is not None, name
        rel_err = _rel(p.grad.cpu().numpy(), g_ref.numpy())
        worst = max(worst, rel_err)
        assert rel_err <= 1e-4, (kind, H, name, rel_err)
    print("%s H=%d [%s]: worst max|grad - float64| / max|float64| = %.2e" % (kind, H, "tc" if tc else "no_tc", worst))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the contrastive term against the restatement
# ---------------------------------------------------------------------------------------------------------------------
def _directional_heads(nce, seed):
    """Weights for which the key mostly follows the direction of (x, y) and the query one fixed direction, so logits
    cover nearly [-1 / tau, 1 / tau]: small random weights around the closed-form case."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in nce.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.01)
        W1, b1 = nce.event_encoder[0].weight, nce.event_encoder[0].bias
        W2, b2 = nce.event_encoder[2].weight, nce.event_encoder[2].bias
        W1[0, 0] += 1.0
        W1[1, 1] += 1.0
        b1[:2] += 10.0
        W2[0, 0] += 1.0
        W2[1, 1] += 1.0
        b2[:2] -= 10.0
        nce.head[0].bias[0] += 1.0
        nce.head[2].weight[0, 0] += 1.0


def _case_data(name):
    """(scene [T, M, 2] float32, batch_split) of a case."""
    if name == "one_track":
        xy, _ = O.synthetic_scenes(8, 1, seed=81)
        return xy, np.arange(9, dtype=np.int64)
    if name == "track93":
        xy_a, bs_a = O.synthetic_scenes(1, 93, seed=82, nan_tracks=True)
        xy_b, bs_b = O.synthetic_scenes(3, 6, seed=83, ragged=True, nan_tracks=True)
        return np.concatenate([xy_b[:, :bs_b[1]], xy_a, xy_b[:, bs_b[1]:]], axis=1), \
            np.concatenate([bs_b[:2], bs_b[1] + bs_a[1:], 93 + bs_b[2:]])
    if name == "bench":
        return O.synthetic_scenes(256, 20, seed=100)
    xy, bs = O.synthetic_scenes(10, 9, seed=84, ragged=True, nan_tracks=True)
    xy = xy.copy()
    xy[OBS + 1, bs[2] + 1] = np.nan        # neighbours missing at some horizons
    xy[OBS + 3, bs[3] + 1:bs[4]] = np.nan
    if name == "primary_nan":
        xy[OBS + 1, bs[1]] = np.nan        # a primary without a future at horizon 2
    return xy, bs


# (name, data, H, mlp_dim, head_dim, horizon, temperature, directional heads)
NCE_CASES = [
    ("one_track", "one_track", 128, 32, 8, 4, 0.1, False),
    ("missing_neighbours", "missing", 128, 32, 8, 4, 0.1, False),
    ("primary_nan", "primary_nan", 128, 32, 8, 4, 0.1, False),
    ("horizon1_h32", "missing", 32, 32, 8, 1, 0.1, False),
    ("horizon12_h256", "missing", 256, 32, 8, 12, 0.1, False),
    ("tau007", "missing", 128, 32, 8, 4, 0.07, True),
    ("tau002_span80", "missing", 128, 16, 4, 4, 0.02, True),
    ("mlp64_head16", "missing", 64, 64, 16, 4, 0.1, False),
    ("track93_horizon12", "track93", 128, 32, 8, 12, 0.1, False),
    ("bench_256x20", "bench", 128, 32, 8, 4, 0.1, False),
]


def _nce_inputs(case):
    from trajnetplusplusbaselines_b200.lstm.contrast import SocialNCE
    name, data, H, D, E, horizon, tau, directional = case
    xy, bs = _case_data(data)
    torch.manual_seed(5)
    nce = SocialNCE(H, mlp_dim=D, head_dim=E, horizon=horizon, temperature=tau)
    if directional:
        _directional_heads(nce, 6)
    g = torch.Generator().manual_seed(7)
    hidden = torch.randn((xy.shape[1], H), generator=g)
    eps = torch.randn(nce.eps_shape(bs), generator=g)
    return xy, bs, nce, hidden, eps


@pytest.mark.gpu
@pytest.mark.parametrize("case", NCE_CASES, ids=[c[0] for c in NCE_CASES])
def test_term_matches_restatement(case):
    """The term's two launches use no tensor-core path (TB2_DISABLE_TC does not reach them): one run per case."""
    xy, bs, nce, hidden, eps = _nce_inputs(case)
    name, horizon, tau = case[0], case[5], case[6]
    nce = nce.cuda()
    nce.fixed_eps = eps.cuda()
    h = hidden.cuda().requires_grad_(True)
    loss, terms, valid = nce(torch.from_numpy(xy).cuda(), h, torch.from_numpy(bs), OBS, return_terms=True)
    loss.backward()

    h64 = hidden.double().requires_grad_(True)
    params = _params64(nce)
    logits = []
    loss64, terms64, valid64 = snce_restated(xy, h64, bs, OBS, horizon, params, temperature=tau, eps=eps,
                                             logits_out=logits)
    loss64.backward()
    assert valid.cpu().double().equal(valid64)
    assert float((terms.cpu().double() - terms64.detach()).abs().max()) <= 2e-5 * max(float(terms64.abs().max()), 1.0)
    assert abs(float(loss) - float(loss64)) <= 2e-5 * max(abs(float(loss64)), 1.0), (float(loss), float(loss64))
    if name == "one_track":
        assert float(loss) == 0.0 and not terms.any() and not h.grad.any()
        assert all(not p.grad.any() for p in nce.parameters())
        return
    if name == "primary_nan":
        assert float(valid[1, 1]) == 0.0 and float(terms[1, 1]) == 0.0
    if name.startswith("tau002"):
        assert max(float(l.max() - l.min()) for l in logits) > 80.0
    got = [h.grad] + [p.grad for p in nce.parameters()]
    ref = [h64.grad] + [p.grad for p in params]
    worst = 0.0
    for i, (g, r) in enumerate(zip(got, ref)):
        e = _rel(g.cpu().numpy(), r.numpy())
        worst = max(worst, e)
        assert e <= 2e-5, (name, i, e)
    print("%s: loss %.6f, worst max|grad - float64| / max|float64| = %.2e" % (name, float(loss), worst))


def _forward_raw(nce, xy, bs, hidden, eps):
    """tb2_snce_forward's four outputs for the scenes of bs."""
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import SceneLayout, _ptr, _stream
    lib = _lib.load()
    layout = SceneLayout([int(v) for v in bs])
    B = len(bs) - 1
    theta = torch.cat([p.detach().reshape(-1) for p in nce.parameters()]).cuda()
    out = [torch.empty((B, nce.horizon), device="cuda"), torch.empty((B, nce.horizon), device="cuda"),
           torch.empty((B, nce.hidden_dim), device="cuda"), torch.empty((B, theta.numel()), device="cuda")]
    X, h, e = torch.from_numpy(xy).cuda(), hidden.cuda().contiguous(), eps.cuda().contiguous()
    _lib.check(lib.tb2_snce_forward(layout.handle, _ptr(X), xy.shape[0], OBS - 1, nce.horizon, _ptr(h), nce.hidden_dim,
                                    _ptr(theta), nce.mlp_dim, nce.head_dim, nce.temperature, nce.rho, nce.sigma,
                                    _ptr(e), *[_ptr(t) for t in out], _stream(torch.device("cuda"))))
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
def test_scene_results_do_not_depend_on_the_batch():
    case = ("track93_horizon12", "track93", 128, 32, 8, 12, 0.1, False)
    xy, bs, nce, hidden, eps = _nce_inputs(case)
    full = _forward_raw(nce, xy, bs, hidden, eps)
    again = _forward_raw(nce, xy, bs, hidden, eps)
    for a, b in zip(full, again):
        assert torch.equal(a, b)
    for b in range(len(bs) - 1):
        lo, hi = int(bs[b]), int(bs[b + 1])
        ns = 1 + 8 * (hi - lo - 1)
        alone = _forward_raw(nce, np.ascontiguousarray(xy[:, lo:hi]), np.array([0, hi - lo]), hidden[lo:hi],
                             eps[b:b + 1, :, :ns])
        for t_full, t_alone in zip(full, alone):
            assert torch.equal(t_full[b:b + 1], t_alone), b


@pytest.mark.gpu
def test_term_makes_no_host_synchronisation():
    case = NCE_CASES[1]
    xy, bs, nce, hidden, eps = _nce_inputs(case)
    nce = nce.cuda()
    scene = torch.from_numpy(xy).cuda()
    h = hidden.cuda().requires_grad_(True)
    split = torch.from_numpy(bs)
    nce(scene, h, split, OBS).backward()          # warm-up: layout, module load
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = nce(scene, h, split, OBS)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and h.grad.abs().sum() > 0


@pytest.mark.gpu
def test_social_nce_step_makes_no_host_synchronisation():
    """A social model's training forward with hidden states, the term on its query step, and the backward into every
    parameter.  The task term is a device-only stand-in: PredictionLoss copies the primaries to the device, a
    synchronisation of its own that this change does not touch."""
    from trajnetplusplusbaselines_b200.lstm.contrast import SocialNCE
    from trajnetplusplusbaselines_b200.lstm.training import sequence_with_hidden
    xy, bs = O.synthetic_scenes(8, 9, seed=95, ragged=True, nan_tracks=True)
    model = _model("social_default", 128, weights("social_default", 128, seed=96))
    torch.manual_seed(0)
    nce = SocialNCE(128).cuda()
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)

    def step():
        rel, _, hid = sequence_with_hidden(model, scene[:OBS], split, scene[OBS:-1].clone(), None)
        loss = torch.nan_to_num(rel).square().mean() + nce(scene, hid[OBS - 2], split, OBS, layouts=model._layouts)
        model.zero_grad()
        nce.zero_grad()
        loss.backward()
        return loss
    step()                                        # warm-up: layout, handles, workspaces
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    assert all(p.grad is not None and p.grad.abs().sum() > 0 for p in nce.parameters())
    assert model.encoder.weight_hh.grad.abs().sum() > 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: whole training steps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", ["directional", "social_default"])
def test_train_batch_matches_float64(monkeypatch, kind, tc):
    from trajnetplusplusbaselines_b200.lstm.contrast import SocialNCE
    _tc(monkeypatch, tc)
    H = 128
    xy, bs = O.synthetic_scenes(8, 9, seed=91, ragged=True, nan_tracks=True)
    W = weights(kind, H, seed=92)
    model = _model(kind, H, W)
    torch.manual_seed(9)
    nce = SocialNCE(H)
    eps = torch.randn(nce.eps_shape(bs), generator=torch.Generator().manual_seed(10))
    nce.fixed_eps = eps.cuda()
    trainer = TRN.Trainer(model, optimizer=torch.optim.SGD(model.parameters(), lr=0.0), device=torch.device("cuda"),
                          batch_size=len(bs) - 1, augment=False, contrast_weight=1.0, contrast=nce)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    loss = trainer.train_batch(scene, trainer._goals(xy.shape[1]), split)
    with torch.no_grad():
        _, pos = model(scene[:OBS], torch.zeros(xy.shape[1], 2), split, scene[OBS:-1].clone())

    stats = {}
    W64, rel64, hid64 = restated_sequence(W, pool_config(kind, H), xy, bs, H, pos.cpu().numpy(), stats=stats)
    _check_relu(stats, kind)
    params = _params64(nce)
    l_nce, _, _ = snce_restated(xy, hid64[OBS - 2], bs, OBS, nce.horizon, params, eps=eps)
    loss64 = _task_restated(rel64, xy, bs) + l_nce
    loss64.backward()
    assert abs(float(loss) - float(loss64)) <= 1e-4 * abs(float(loss64)), (float(loss), float(loss64))
    got = [(n, p.grad) for n, p in model.named_parameters()] + [("nce%d" % i, p.grad) for i, p in
                                                                  enumerate(nce.parameters())]
    ref = [W64[n].grad if n in W64 else None for n, _ in model.named_parameters()] + [p.grad for p in params]
    worst = 0.0
    for (n, g), r in zip(got, ref):
        if r is None:                 # the goal embedding, which a model without goals does not use
            assert g is None or not g.any(), n
            continue
        assert g is not None, n
        e = _rel(g.cpu().numpy(), r.numpy())
        worst = max(worst, e)
        assert e <= 1e-4, (kind, n, e)
    print("%s [%s]: train_batch with Social-NCE, worst rel err %.2e" % (kind, "tc" if tc else "no_tc", worst))


def _store(seed, n=24):
    xy, bs = O.synthetic_scenes(n, 6, n_frames=OBS + PRED, seed=seed, ragged=True, nan_tracks=True)
    return TRN.SceneStore([("synth", i, xy[:, bs[i]:bs[i + 1]].astype(np.float64)) for i in range(n)])


def _restated_epoch(model, optimizer, store, batch_size):
    """One epoch of the trainer without the term, written here from public pieces: the epoch plan, the gathered
    batches, the teacher-forced forward, PredictionLoss x batch_size and the optimizer step.  Returns the batch losses."""
    from trajnetplusplusbaselines_b200.lstm import PredictionLoss
    plan = TRN.draw_epoch_plan(store.order, store.kept, batch_size, store.T, OBS, True, True, False)
    model.train()
    optimizer.zero_grad()
    losses = []
    for batch_scene, split in store.gather(plan.order, batch_size, thetas=plan.thetas, noise=plan.noise,
                                           noise_off=plan.noise_off):
        split = torch.from_numpy(split)
        targets = batch_scene[OBS:OBS + PRED] - batch_scene[OBS - 1:OBS + PRED - 1]
        rel, _ = model(batch_scene[:OBS].clone(), torch.zeros(batch_scene.shape[1], 2), split,
                       batch_scene[OBS:OBS + PRED - 1].clone())
        loss = PredictionLoss()(rel[-PRED:], targets, split) * batch_size
        optimizer.zero_grad()
        loss.backward()
        optimizer.step()
        losses.append(float(loss))
    return losses


@pytest.mark.gpu
def test_zero_weight_is_the_plain_loop_bit_for_bit(caplog):
    """Trainer(contrast_weight=0) against the plain loop: the same losses, parameters and Adam state, bit for bit, and
    train-epoch records with the keys of a run without the term."""
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    store = _store(31)
    runs = []
    for restated in (False, True):
        store.order = list(range(len(store)))         # an epoch shuffles the scene list in place
        torch.manual_seed(3)
        model = LSTM(pool=GridBasedPooling(type_="directional", hidden_dim=128, n=12, cell_side=0.6,
                                           out_dim=256)).cuda()
        optimizer = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
        random.seed(4)
        np.random.seed(5)
        if restated:
            losses = [_restated_epoch(model, optimizer, store, 8) for _ in range(2)]
            records = [{"type": "train-epoch", "epoch": e + 1, "loss": round(sum(v) / len(store), 5)}
                       for e, v in enumerate(losses)]
        else:
            trainer = TRN.Trainer(model, optimizer=optimizer, device=torch.device("cuda"), augment=True,
                                  augment_noise=True, contrast_weight=0.0)
            caplog.clear()
            with caplog.at_level("INFO"):
                for epoch in range(2):
                    trainer.train(store, None, epoch)
            records = [{k: v for k, v in r.msg.items() if k != "time"} for r in caplog.records
                       if isinstance(r.msg, dict)]
            assert trainer.contrast is None
        runs.append((records, {n: p.detach().clone() for n, p in model.named_parameters()}, optimizer.state_dict()))
    (r0, p0, o0), (r1, p1, o1) = runs
    assert r0 == r1, (r0, r1)
    for n in p0:
        assert torch.equal(p0[n], p1[n]), n
    assert o0["state"].keys() == o1["state"].keys()
    for k in o0["state"]:
        for f in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(o0["state"][k][f], o1["state"][k][f]), (k, f)


@pytest.mark.gpu
def test_cli_trains_resumes_and_evaluates(tmp_path, monkeypatch):
    from test_multimodal_batch import _write_scenes
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    monkeypatch.chdir(tmp_path)
    for part, sizes, seed in (("train", [3, 5, 2, 4, 6, 3] * 4, 1), ("val", [3, 4, 2], 2), ("test", [3, 5, 2, 4], 3)):
        os.makedirs(os.path.join("DATA_BLOCK", "synth", part))
        _write_scenes(os.path.join("DATA_BLOCK", "synth", part, "synth.ndjson"), sizes, seed)
    common = ["--path", "synth", "--type", "social", "--n", "8", "--contrast_weight", "1", "--contrast_horizon", "6",
              "--contrast_temperature", "0.2", "--save_every", "1", "--output", "nce"]
    TRN.main(common + ["--epochs", "1"])
    out = os.path.join("OUTPUT_BLOCK", "synth")
    base = os.path.join(out, "lstm_social_nce.pkl")
    state = torch.load(base + ".state", map_location="cuda", weights_only=False)
    assert set(state) == {"epoch", "state_dict", "optimizer", "scheduler", "contrast"} and state["epoch"] == 1
    assert len(state["optimizer"]["param_groups"]) == 2
    # a full state with heads needs the term, and one without heads cannot resume with it
    plain = ["--path", "synth", "--type", "social", "--n", "8", "--save_every", "1", "--output", "nce", "--epochs", "2"]
    with pytest.raises(SystemExit) as e:
        TRN.main(plain + ["--load-full-state", base + ".state"])
    assert "holds Social-NCE heads" in str(e.value.code)
    TRN.main(common + ["--epochs", "2", "--load-full-state", base + ".state"])
    resumed = torch.load(base + ".state", map_location="cuda", weights_only=False)
    assert resumed["epoch"] == 2 and any(not torch.equal(resumed["contrast"][k], state["contrast"][k])
                                         for k in state["contrast"])
    with open(base + ".log") as f:
        records = [json.loads(line) for line in f if line.strip()]
    epochs = [r for r in records if r["type"] == "train-epoch"]
    assert [r["epoch"] for r in epochs] == [1, 2]
    for r in epochs:
        assert set(r) == {"type", "message", "levelname", "name", "asctime", "epoch", "loss", "time", "loss_nce"}
        assert math.isfinite(r["loss_nce"]) and r["loss_nce"] > 0
    predictor = LSTMPredictor.load(base)
    assert type(predictor.model).__name__ == "LSTM"
    predictor.model.cuda()
    n = evaluate_file(predictor, os.path.join("DATA_BLOCK", "synth", "test", "synth.ndjson"),
                      os.path.join(str(tmp_path), "pred.ndjson"))
    assert n == 4
