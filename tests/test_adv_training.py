"""Adversarial training against the collision attack (Trainer(adv_eps > 0), --adv_eps): the Trainer against a loop written
here from public pieces, the constraints on the attacked batch, the CLI end to end and its refusals."""
import json
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import lstm_oracle as O  # noqa: E402
from trajnetplusplusbaselines_b200.lstm import trainer as TR  # noqa: E402

OBS, PRED, BS = 9, 12, 8
LIMIT = 0.2


def _model(kind):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    torch.manual_seed(3)
    pool = GridBasedPooling(type_=kind, hidden_dim=128, cell_side=0.6, n=12, out_dim=256, embedding_arch="one_layer",
                            constant=0, layer_dims=[512], latent_dim=16)
    return LSTM(pool=pool, embedding_dim=64, hidden_dim=128).cuda()


def _store(seed, n=24, lone=False):
    """n seeded scenes of 21 frames packed close together (collisions within reach), NaN tracks included; lone: scene 1 is
    its primary alone (no pair: D = +inf)."""
    xy, bs = O.synthetic_scenes(n, 6, n_frames=OBS + PRED, seed=seed, ragged=True, nan_tracks=True, start_std=0.8,
                                vel_std=0.15)
    entries = []
    for i in range(n):
        s = xy[:, bs[i]:bs[i + 1]].astype(np.float64)
        entries.append(("synth", i, s[:, :1] if lone and i == 1 else s))
    return TR.SceneStore(entries)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement: the epoch plan, a PGD loop over differentiable_rollout and the attack kernels, two teacher-forced
# forwards, the criterion and Adam
# ---------------------------------------------------------------------------------------------------------------------
def _p(t):
    import ctypes
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _pgd(model, observed, split, eps, steps, layouts):
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import differentiable_rollout
    lib = _lib.load()
    split_t = torch.from_numpy(split)
    layout = layouts.get(split_t, pad_to_batch_max=True, device=observed.device)
    T, B = observed.shape[0], len(split) - 1
    delta = torch.zeros((T, B, 2), dtype=torch.float32, device="cuda")
    best_delta = torch.zeros_like(delta)
    best_D = torch.full((B,), float("inf"), dtype=torch.float64, device="cuda")
    D = torch.empty_like(best_D)
    adv = observed.clone()
    d_clean = best_pos = None
    for it in range(steps + 1):
        move = it < steps
        obs_in = adv.clone().requires_grad_(move)
        with torch.enable_grad():
            _, pos = differentiable_rollout(model, obs_in, split_t, PRED, pad_to_batch_max=True, parameters=False)
        pos = pos.contiguous()
        F = pos.shape[0]
        dpos = torch.empty_like(pos)
        _lib.check(lib.tb2_attack_objective(layout.handle, _p(pos), F, F - PRED, _p(D), _p(dpos), None))
        d_obs = torch.autograd.grad(pos, obs_in, grad_outputs=dpos)[0].contiguous() if move else None
        if it == 0:
            d_clean, best_pos = D.clone(), pos.detach().clone()
        _lib.check(lib.tb2_attack_step(layout.handle, _p(d_obs), _p(observed), T, _p(delta), _p(D), F, _p(pos),
                                       _p(best_D), _p(best_delta), _p(best_pos), _p(adv), float(eps),
                                       float(2.5 * eps / steps), int(move), None))
    out = observed.clone()
    out[:, split[:-1]] = observed[:, split[:-1]] + best_delta
    return out, d_clean, best_D


def _restated_epochs(model, opt, sched, criterion, store, cfg, epochs):
    from trajnetplusplusbaselines_b200.engine import LayoutCache
    layouts = LayoutCache()
    losses, after, cols = [], [], []
    for _ in range(epochs):
        plan = TR.draw_epoch_plan(store.order, store.kept, BS, store.T, OBS, cfg["augment"], False, cfg["obs_dropout"])
        model.train()
        opt.zero_grad()
        frame = store.frames(OBS) if cfg["normalize_scene"] else None
        batches = store.gather(plan.order, BS, frame=frame, thetas=plan.thetas, noise=plan.noise,
                               noise_off=plan.noise_off)
        starts = iter(plan.start_lengths) if plan.start_lengths is not None else None
        counts = np.zeros(2)
        for batch_scene, split in batches:
            start = next(starts) if starts is not None else 0
            split_t = torch.from_numpy(split)
            observed = batch_scene[start:OBS].clone()
            truth = batch_scene[OBS:OBS + PRED - 1].clone()
            targets = batch_scene[OBS:OBS + PRED] - batch_scene[OBS - 1:OBS + PRED - 1]
            adv, d_clean, d_best = _pgd(model, observed, split, cfg["eps"], cfg["steps"], layouts)
            counts += [int((d_clean <= LIMIT).sum()), int((d_best <= LIMIT).sum())]

            def batch_loss(obs):
                rel, out = model(obs, None, split_t, truth)
                primary = batch_scene[-PRED:].clone()
                primary[:, split_t[:-1]] = out[-PRED:, split_t[:-1]]
                return criterion(rel[-PRED:], targets, split_t, primary) * BS
            w = cfg["wt"]
            loss = (1 - w) * batch_loss(observed) + w * batch_loss(adv) if w < 1 else w * batch_loss(adv)
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(float(loss))
        sched.step()
        after.append(_snapshot(model, opt))
        cols.append(tuple(counts / len(store)))
    return losses, after, cols


def _snapshot(model, opt):
    return ({k: v.detach().cpu().clone() for k, v in model.state_dict().items()},
            {i: {k: v.cpu().clone() if torch.is_tensor(v) else v for k, v in st.items()}
             for i, st in opt.state_dict()["state"].items()})


def _trainer_epochs(trainer, store, epochs):
    losses, after, records = [], [], []
    tb = trainer.train_batch

    def train_batch(*a):
        loss = tb(*a)
        losses.append(float(loss))
        return loss
    trainer.train_batch = train_batch

    class Log(object):
        def info(self, record):
            records.append(record)
    trainer.log = Log()
    for epoch in range(epochs):
        trainer.train(store, None, epoch)
        after.append(_snapshot(trainer.model, trainer.optimizer))
    cols = [(r["col_clean"], r["col_attacked"]) for r in records if r["type"] == "train-epoch"]
    return losses, after, cols


def _seed():
    random.seed(21)
    np.random.seed(22)
    torch.manual_seed(23)


CONFIGS = {
    "directional_w05_augment": dict(kind="directional", wt=0.5, augment=True, normalize_scene=False, obs_dropout=False,
                                    col_wt=0.0),
    "directional_w1_obs_dropout": dict(kind="directional", wt=1.0, augment=False, normalize_scene=False,
                                       obs_dropout=True, col_wt=0.0),
    "social_w05_normalize": dict(kind="social", wt=0.5, augment=False, normalize_scene=True, obs_dropout=False,
                                 col_wt=0.1),
    "social_w1_augment_obs_dropout": dict(kind="social", wt=1.0, augment=True, normalize_scene=False, obs_dropout=True,
                                          col_wt=0.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CONFIGS))
def test_trainer_matches_restated_loop_bitwise(name):
    from trajnetplusplusbaselines_b200.lstm import PredictionLoss
    cfg = dict(CONFIGS[name], eps=0.15, steps=3)
    runs = []
    for mode in ("trainer", "trainer", "restated"):
        _seed()
        model = _model(cfg["kind"])
        opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
        sched = torch.optim.lr_scheduler.StepLR(opt, 1)
        criterion = PredictionLoss(col_wt=cfg["col_wt"]).cuda()
        store = _store(7)
        if mode == "trainer":
            trainer = TR.Trainer(model, criterion=criterion, optimizer=opt, lr_scheduler=sched,
                                 device=torch.device("cuda"), batch_size=BS, augment=cfg["augment"],
                                 normalize_scene=cfg["normalize_scene"], obs_dropout=cfg["obs_dropout"],
                                 val_flag=False, adv_eps=cfg["eps"], adv_steps=cfg["steps"], adv_wt=cfg["wt"])
            runs.append(_trainer_epochs(trainer, store, 2))
        else:
            runs.append(_restated_epochs(model, opt, sched, criterion, store, cfg, 2))
    for other in runs[1:]:
        assert runs[0][0] == other[0]                      # per-batch losses
        assert runs[0][2] == other[2]                      # col_clean / col_attacked per epoch
        for (sd_a, st_a), (sd_b, st_b) in zip(runs[0][1], other[1]):
            for k in sd_a:
                assert torch.equal(sd_a[k], sd_b[k]), k
            assert list(st_a) == list(st_b)
            for i in st_a:
                for k, v in st_a[i].items():
                    assert torch.equal(v, st_b[i][k]) if torch.is_tensor(v) else v == st_b[i][k], (i, k)
    losses, _, cols = runs[0]
    assert len(losses) == 6 and all(np.isfinite(losses))
    assert all(0 <= c <= a <= 1 for c, a in cols), cols


@pytest.mark.gpu
def test_attacked_batch_constraints(monkeypatch):
    """Only the primary rows of the observed frames change, inside the ball; the attack never raises D; a scene without a
    pair keeps delta = 0; the attacked forward gets the clean prediction truth."""
    from trajnetplusplusbaselines_b200 import attack
    from trajnetplusplusbaselines_b200.lstm import LSTM
    eps = 0.15
    calls, forwards = [], []
    pgd = attack.pgd_collision

    def recording_pgd(model, observed, batch_split, *a, **k):
        res = pgd(model, observed, batch_split, *a, **k)
        calls.append((observed.clone(), np.asarray(batch_split).copy(), res))
        return res
    monkeypatch.setattr(attack, "pgd_collision", recording_pgd)
    fwd = LSTM.forward

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None):
        forwards.append((observed.detach().clone(), prediction_truth.clone()))
        return fwd(self, observed, goals, batch_split, prediction_truth, n_predict)
    monkeypatch.setattr(LSTM, "forward", forward)
    _seed()
    model = _model("directional")
    store = _store(11, lone=True)
    trainer = TR.Trainer(model, device=torch.device("cuda"), batch_size=BS, augment=True, obs_dropout=True,
                         val_flag=False, adv_eps=eps, adv_steps=3, adv_wt=0.5)
    trainer.train(store, None, 0)
    assert len(calls) == 3 and len(forwards) == 6
    lone_seen = moved = False
    for k, (observed, split, res) in enumerate(calls):
        prim = split[:-1]
        other = np.setdiff1d(np.arange(observed.shape[1]), prim)
        clean_fwd, adv_fwd = forwards[2 * k], forwards[2 * k + 1]
        for got, want in ((clean_fwd[0], observed), (adv_fwd[0], res.observed), (clean_fwd[1], adv_fwd[1])):
            assert torch.equal(torch.nan_to_num(got, 7.0), torch.nan_to_num(want, 7.0))
        assert 2 <= observed.shape[0] <= OBS
        a, o = res.observed.cpu().numpy(), observed.cpu().numpy()
        assert np.array_equal(a[:, other], o[:, other], equal_nan=True)
        assert np.array_equal(np.isnan(a), np.isnan(o))
        assert np.array_equal(a[:, prim], o[:, prim] + res.delta.cpu().numpy(), equal_nan=True)
        norms = np.linalg.norm(res.delta.double().cpu().numpy(), axis=2)
        assert norms.max() <= eps * (1 + 1e-6)
        d_clean, d_best = res.d_clean.cpu().numpy(), res.d_best.cpu().numpy()
        assert np.all(d_best <= d_clean)
        no_pair = np.isinf(d_clean)
        assert np.all(res.delta.cpu().numpy()[:, no_pair] == 0)
        moved |= bool(np.any(norms > 0))
        lone_seen |= bool(np.any(np.diff(split) == 1) and no_pair[np.diff(split) == 1].all())
    assert lone_seen and moved


# ---------------------------------------------------------------------------------------------------------------------
# the CLI
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cli_end_to_end(tmp_path, monkeypatch, capsys):
    from test_multimodal_batch import _write_scenes
    from trajnetplusplusbaselines_b200 import attack
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    monkeypatch.chdir(tmp_path)
    for part, sizes, seed in (("train", [3, 5, 2, 4, 6, 3] * 4, 1), ("val", [3, 4, 2], 2), ("test", [3, 5, 2, 4], 3),
                              ("test_private", [3, 5, 2, 4], 3)):
        os.makedirs(os.path.join("DATA_BLOCK", "synth", part))
        _write_scenes(os.path.join("DATA_BLOCK", "synth", part, "synth.ndjson"), sizes, seed)
    TR.main(["--path", "synth", "--type", "directional", "--adv_eps", "0.1", "--adv_steps", "2", "--epochs", "2",
             "--save_every", "1", "--output", "adv"])
    out = os.path.join("OUTPUT_BLOCK", "synth")
    base = "lstm_directional_adv.pkl"
    expect = {base, base + ".state", base + ".log"}
    for k in range(3):
        expect |= {base + ".epoch%d" % k, base + ".epoch%d.state" % k}
    assert set(os.listdir(out)) == expect
    with open(os.path.join(out, base + ".log")) as f:
        records = [json.loads(line) for line in f if line.strip()]
    epochs = [r for r in records if r["type"] == "train-epoch"]
    assert [r["epoch"] for r in epochs] == [1, 2]
    for r in epochs:
        assert set(r) == {"type", "message", "levelname", "name", "asctime", "epoch", "loss", "time", "col_clean",
                          "col_attacked"}
        assert 0 <= r["col_clean"] <= 1 and 0 <= r["col_attacked"] <= 1 and np.isfinite(r["loss"])
    assert records[0]["args"]["adv_eps"] == 0.1
    predictor = LSTMPredictor.load(os.path.join(out, base))
    assert type(predictor.model.pool).__name__ == "GridBasedPooling"
    capsys.readouterr()
    attack.main(["--path", "synth", "--output", os.path.join(out, base), "--eps", "0.1", "--steps", "2"])
    assert "attacked 4 scenes" in capsys.readouterr().out
    assert os.path.exists(os.path.join("DATA_BLOCK", "synth", "test_pred", "lstm_directional_adv_attack_eps0.1_steps2.npz"))


@pytest.mark.parametrize("argv, flag", [(["--adv_eps", "-0.1"], "--adv_eps"), (["--adv_steps", "0"], "--adv_steps"),
                                        (["--adv_wt", "0"], "--adv_wt"), (["--adv_wt", "1.5"], "--adv_wt")])
def test_cli_refuses_bad_adversarial_flags(argv, flag, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit) as e:
        TR.main(["--path", "nowhere", "--type", "directional", "--adv_eps", "0.1"] + argv)
    assert flag in str(e.value.code)
    assert os.listdir(tmp_path) == []


def test_cli_keeps_the_training_refusals_first(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(SystemExit) as e:
        TR.main(["--path", "nowhere", "--type", "hiddenstatemlp", "--adv_eps", "0.1"])
    assert "training of HiddenStateMLPPooling is not built" in str(e.value.code)
    assert os.listdir(tmp_path) == []


def test_trainer_refuses_what_the_attack_cannot_differentiate():
    from test_input_grad import HiddenMLP
    from trajnetplusplusbaselines_b200.lstm import LSTM
    TR.Trainer(LSTM(pool=HiddenMLP()), device=torch.device("cpu"))            # clean training of a user module stays
    with pytest.raises(NotImplementedError, match="user-defined"):
        TR.Trainer(LSTM(pool=HiddenMLP()), device=torch.device("cpu"), adv_eps=0.1)
    for kw in (dict(adv_eps=-1.0), dict(adv_eps=0.1, adv_steps=0), dict(adv_eps=0.1, adv_wt=0.0)):
        with pytest.raises(ValueError):
            TR.Trainer(LSTM(), device=torch.device("cpu"), **kw)


class _Stop(Exception):
    pass


def test_epoch_plan_does_not_depend_on_the_adversarial_flags(monkeypatch):
    """Trainer.train draws its epoch plan with the same arguments, and leaves the generators in the same state, with and
    without the attack (the attack draws no random numbers)."""
    from types import SimpleNamespace
    from trajnetplusplusbaselines_b200.lstm import LSTM
    draw = TR.draw_epoch_plan
    seen = []

    def recording_draw(order, *a):
        plan = draw(order, *a)
        seen.append((list(plan.order), None if plan.thetas is None else plan.thetas.tolist(), plan.start_lengths,
                     plan.noise.tolist(), [x.tolist() if isinstance(x, np.ndarray) else x for x in a], random.getstate(), np.random.get_state()[1].tolist()))
        raise _Stop
    monkeypatch.setattr(TR, "draw_epoch_plan", recording_draw)
    for kw in ({}, dict(adv_eps=0.2, adv_steps=7, adv_wt=1.0)):
        trainer = TR.Trainer(LSTM(), device=torch.device("cpu"), augment=True, augment_noise=True, obs_dropout=True,
                             **kw)
        scenes = SimpleNamespace(order=list(range(20)), kept=np.arange(20) % 4 + 1, T=21)
        random.seed(5)
        np.random.seed(6)
        with pytest.raises(_Stop):
            trainer.train(scenes, None, 0)
    assert len(seen) == 2 and seen[0] == seen[1]
