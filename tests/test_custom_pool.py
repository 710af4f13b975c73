"""LSTM models with an external interaction module: a torch.nn.Module without `fill_config` that follows the
reference's pool plug (reset / forward(hidden [B, N, H], obs1, obs2) -> [B * N, out_dim] / out_dim).  The library runs
the LSTM step and torch runs the module between the step's kernels (lstm/external.py, csrc/external_pool.cu).

The reference's own module classes (oracle.ref_shim.import_reference()) stand in for user modules: they have no
fill_config.  On the GPU, with the tensor cores on and with TB2_DISABLE_TC=1:
  * the forward against this package's fused module of the same weights, teacher-forced and free-running, on ragged
    scenes with entering / leaving tracks and a 93-track scene, in the padded and the per-scene layout;
  * training against the reference's LSTM, module and PredictionLoss run in float64 on the CPU;
  * the reference's unmodified Trainer.train_batch driving this package's model;
  * a sync-free module under torch.cuda.set_sync_debug_mode("error");
  * two epochs of the native Trainer, the saved model through evaluator.evaluate_file;
  * the refusals (S-GAN / VAE, sampled predictions, goals).
"""
import copy
import json
import os

import numpy as np
import pytest
import torch

from oracle import lstm_oracle as O

pytestmark = pytest.mark.needs_reference

CLASSES = {"hiddenstatemlp": "HiddenStateMLPPooling", "attentionmlp": "AttentionMLPPooling", "nn": "NearestNeighborMLP",
           "nn_lstm": "NearestNeighborLSTM", "traj_pool": "TrajectronPooling"}
KW = {"hiddenstatemlp": dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256),
      "attentionmlp": dict(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256),
      "nn": dict(n=4, out_dim=256),
      "nn_lstm": dict(n=4, hidden_dim=128, out_dim=256),
      "traj_pool": dict(hidden_dim=128, out_dim=256)}
BUILTIN_KERNELS = ("hidden_mlp_pool", "attn_mlp_pool", "nn_mlp_pool", "pool_lstm_cell", "traj_feat", "traj_scene_sum",
                   "pool_prepare", "sparse_layer1", "sparse_layer1_mma", "dense_grid")
FWD_GATE = 2e-5         # metres, fp32 FFMA gate kernel (the gates of test_nongrid_kernels.py)
FWD_GATE_TC = 3e-4      # metres, the bf16 (hi, lo) pooled operand of the tensor-core gate kernel


def _ref():
    from oracle.ref_shim import import_reference
    return import_reference()


def _tc(monkeypatch, tc):
    if tc:
        monkeypatch.delenv("TB2_DISABLE_TC", raising=False)
    else:
        monkeypatch.setenv("TB2_DISABLE_TC", "1")


class MixPool(torch.nn.Module):
    """A user module that mixes the hidden states and positions of a scene's present tracks: every track gets
    tanh(W_h h + W_p [pos, vel] + b) plus the mean of that over the present tracks of its scene.  No host
    synchronisation (no boolean indexing): padding and absent tracks are masked with torch.where.  Records every call."""

    def __init__(self, hidden_dim=128, out_dim=32):
        super().__init__()
        self.out_dim = out_dim
        self.hidden = torch.nn.Linear(hidden_dim, out_dim)
        self.spatial = torch.nn.Linear(4, out_dim)
        self.calls = []

    def reset(self, num_tracks, max_num_neigh, device):
        self.calls.append(("reset", num_tracks, max_num_neigh, device))

    def forward(self, hidden, obs1, obs2):
        self.calls.append(("forward", tuple(hidden.shape), tuple(obs1.shape), tuple(obs2.shape)))
        B, N, _ = hidden.shape
        valid = ~(torch.isnan(obs1[..., 0]) | torch.isnan(obs2[..., 0]))
        v = valid.unsqueeze(-1)
        pos = torch.where(v, torch.cat([obs2, obs2 - obs1], dim=-1), torch.zeros((), dtype=obs2.dtype, device=obs2.device))
        hid = torch.where(v, hidden, torch.zeros((), dtype=hidden.dtype, device=hidden.device))
        feat = torch.tanh(self.hidden(hid) + self.spatial(pos))
        w = v.to(feat.dtype)
        scene = (feat * w).sum(dim=1, keepdim=True) / w.sum(dim=1, keepdim=True).clamp(min=1.0)
        return (feat + scene).reshape(B * N, self.out_dim)


def _ref_module(kind, seed):
    from trajnetbaselines.lstm import non_gridbased_pooling as NG
    torch.manual_seed(seed)
    return getattr(NG, CLASSES[kind])(**KW[kind])


def _models(kind, seed=21, pool_to_input=True):
    """(external model, fused model) on the GPU with the same weights: this package's LSTM around the reference's
    module, and around this package's built-in module of that name."""
    from trajnetplusplusbaselines_b200 import lstm as L
    _ref()
    ext_pool = _ref_module(kind, seed)
    torch.manual_seed(seed + 1)
    ext = L.LSTM(pool=ext_pool, pool_to_input=pool_to_input)
    fused = L.LSTM(pool=getattr(L, CLASSES[kind])(**KW[kind]), pool_to_input=pool_to_input)
    fused.load_state_dict(ext.state_dict())
    return ext.cuda(), fused.cuda()


def _scenes(seed=116, big=True, n=24, spread=12.0):
    """Ragged scenes of 2..20 tracks with entering / leaving neighbours, and one 93-track scene."""
    xy, bs = O.synthetic_scenes(n, 20, seed=seed, ragged=True, nan_tracks=True, start_std=spread)
    if big:
        xb, bsb = O.scenes_of_sizes([93], seed=seed + 1)
        xy = np.concatenate([xy, xb * np.float32(spread / 3.0)], axis=1)
        bs = np.concatenate([bs, bs[-1] + bsb[1:]]).astype(np.int64)
    return xy, bs


def _profiled(fn):
    """fn() and the library kernels it launched ({name: {"launches", "total_ms"}}, tb2_profile_*)."""
    import ctypes
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    _lib.check(lib.tb2_profile_begin())
    out = fn()
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(lib.tb2_profile_end(buf, len(buf)))
    return out, json.loads(buf.value.decode())


# ---------------------------------------------------------------------------------------------------------------------
# CPU: configuration and refusals that need no device
# ---------------------------------------------------------------------------------------------------------------------
def test_external_config_and_training_targets():
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import lstm_config
    from trajnetplusplusbaselines_b200.lstm import LSTM
    from trajnetplusplusbaselines_b200.lstm.external import is_external
    from trajnetplusplusbaselines_b200.lstm.trainer import check_trainable
    from trajnetplusplusbaselines_b200.lstm.training import _grad_targets
    pool = MixPool(out_dim=48)
    assert is_external(pool)
    cfg = lstm_config(128, 64, True, pool)
    assert cfg.pool_type == _lib.POOL_EXTERNAL and cfg.out_dim == 48
    model = LSTM(pool=pool)
    check_trainable(model)                              # accepted: autograd carries the module's gradients
    assert "pool_embedding_weight0" not in _grad_targets(model)
    with pytest.raises(NotImplementedError, match="goal_flag=True with an external"):
        from trajnetplusplusbaselines_b200.lstm.external import external_forward
        external_forward(LSTM(pool=pool, goal_flag=True), torch.zeros(9, 2, 2), None, torch.tensor([0, 2]), n_predict=12)


# ---------------------------------------------------------------------------------------------------------------------
# 1. forward against the fused path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("teacher", [True, False], ids=["teacher", "free"])
@pytest.mark.parametrize("kind", list(CLASSES))
def test_forward_matches_fused_module(monkeypatch, kind, teacher, tc):
    _tc(monkeypatch, tc)
    ext, fused = _models(kind)
    ext.eval()
    fused.eval()
    xy, bs = _scenes()
    M = xy.shape[1]
    obs = torch.from_numpy(xy[:9])
    kw = dict(prediction_truth=torch.from_numpy(xy[9:20]).clone()) if teacher else dict(n_predict=12)
    with torch.no_grad():
        (_, pred), prof = _profiled(lambda: ext(obs, torch.zeros(M, 2), torch.from_numpy(bs), **kw))
        _, want = fused(obs, torch.zeros(M, 2), torch.from_numpy(bs), **kw)
    assert "external_pooled" in prof and "pool_inputs_padded" in prof, prof.keys()
    assert not set(BUILTIN_KERNELS) & set(prof), prof.keys()
    pred, want = pred.numpy(), want.numpy()
    assert (np.isnan(pred) == np.isnan(want)).all()
    err = float(np.nanmax(np.abs(pred - want)))
    print("external %s %s [%s]: max |external - fused| = %.2e m" % (kind, "teacher" if teacher else "free",
                                                                   "tc" if tc else "no_tc", err))
    assert err <= (FWD_GATE_TC if tc else FWD_GATE), (kind, err)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", list(CLASSES))
def test_per_scene_layout_matches_fused_module(monkeypatch, kind, tc):
    """The evaluator's per-scene layout: predict_batch_xy (one padded forward per scene size) and __call__ of one
    scene, against the fused module's predict_batch_xy, including obs_length 2."""
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    _tc(monkeypatch, tc)
    ext, fused = _models(kind)
    xy, bs = _scenes(seed=5, n=10)
    xys = [xy[:, bs[i]:bs[i + 1]].astype(np.float64) for i in range(len(bs) - 1)]
    if kind == "traj_pool":       # sums over its whole batch: one scene per size keeps the groups per scene
        seen = {}
        xys = [seen.setdefault(x.shape[1], x) for x in xys if x.shape[1] not in seen]
    gate = FWD_GATE_TC if tc else FWD_GATE
    for obs_length in (9, 2):
        got = LSTMPredictor(ext).predict_batch_xy(xys, n_predict=12, obs_length=obs_length)
        want = LSTMPredictor(fused).predict_batch_xy(xys, n_predict=12, obs_length=obs_length)
        for g, w in zip(got, want):
            assert np.abs(g[0][0] - w[0][0]).max() <= gate
            assert (np.isnan(g[0][1]) == np.isnan(w[0][1])).all()
            if np.isfinite(w[0][1]).any():
                assert np.nanmax(np.abs(g[0][1] - w[0][1])) <= gate
    # the per-scene call (the reference's call) against the fused module's
    from trajnetplusplusbaselines_b200.data import TrackRow
    x = xys[-1]
    paths = [[TrackRow(100 + 10 * t, 7 + p, float(x[t, p, 0]), float(x[t, p, 1])) for t in range(x.shape[0])
              if not np.isnan(x[t, p, 0])] for p in range(x.shape[1])]
    one = LSTMPredictor(ext)(paths, np.zeros((len(paths), 2)), n_predict=12)
    want = LSTMPredictor(fused)(paths, np.zeros((len(paths), 2)), n_predict=12)
    assert np.abs(one[0][0] - want[0][0]).max() <= gate


# ---------------------------------------------------------------------------------------------------------------------
# 2. training against float64
# ---------------------------------------------------------------------------------------------------------------------
TRAIN_CASES = [(k, True) for k in CLASSES] + [("hiddenstatemlp", False), ("mix", True)]


def _train_scenes(obs_length):
    xy, bs = O.synthetic_scenes(6, 8, seed=31, ragged=True, nan_tracks=True, start_std=3.0)
    return xy[:obs_length + 12], bs


def _float64_step(pool, W, pool_to_input, xy, bs, obs_length):
    """Loss and gradients of the reference's LSTM, module and PredictionLoss in float64 on the CPU, fed fp32 inputs."""
    from trajnetbaselines.lstm.loss import PredictionLoss as RefLoss
    from trajnetbaselines.lstm.lstm import LSTM as RefLSTM
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        model = RefLSTM(pool=pool.double(), pool_to_input=pool_to_input)
        model.load_state_dict({k: v.double() for k, v in W.items()})
        model = model.double().train()
        scene = torch.from_numpy(xy).double()
        split = torch.from_numpy(bs)
        rel, _ = model(scene[:obs_length], torch.zeros(scene.shape[1], 2), split, scene[obs_length:-1].clone())
        assert rel.dtype == torch.float64
        targets = scene[obs_length:] - scene[obs_length - 1:-1]
        loss = RefLoss()(rel[-12:], targets, split) * (len(bs) - 1)
        loss.backward()
        return float(loss.detach()), {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    finally:
        torch.set_default_dtype(old)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("obs_length", [9, 2])
@pytest.mark.parametrize("kind,pool_to_input", TRAIN_CASES, ids=["%s-%s" % (k, "input" if p else "hidden")
                                                                   for k, p in TRAIN_CASES])
def test_training_matches_float64(monkeypatch, kind, pool_to_input, obs_length, tc):
    from trajnetplusplusbaselines_b200.lstm import LSTM, PredictionLoss
    _tc(monkeypatch, tc)
    _ref()
    if kind == "mix":
        torch.manual_seed(41)
        pool = MixPool(out_dim=32)
    else:
        kw = dict(KW[kind])
        if not pool_to_input:
            kw["out_dim"] = 128                  # h += pooled: out_dim == hidden_dim
        from trajnetbaselines.lstm import non_gridbased_pooling as NG
        torch.manual_seed(41)
        pool = getattr(NG, CLASSES[kind])(**kw)
    torch.manual_seed(42)
    model = LSTM(pool=copy.deepcopy(pool), pool_to_input=pool_to_input)
    W = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.cuda().train()
    xy, bs = _train_scenes(obs_length)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    rel, _ = model(scene[:obs_length], torch.zeros(scene.shape[1], 2).cuda(), split, scene[obs_length:-1].clone())
    targets = scene[obs_length:] - scene[obs_length - 1:-1]
    loss = PredictionLoss()(rel[-12:], targets, split.cuda()) * (len(bs) - 1)
    loss.backward()
    loss_ref, grads_ref = _float64_step(copy.deepcopy(pool), W, pool_to_input, xy, bs, obs_length)
    assert abs(float(loss) - loss_ref) <= 1e-5 * abs(loss_ref), (float(loss), loss_ref)
    got = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    assert set(got) == set(grads_ref), set(got) ^ set(grads_ref)
    assert any(k.startswith("pool.") for k in got)
    worst = ("", 0.0)
    for k, g in grads_ref.items():
        scale = max(float(g.abs().max()), 1e-12)
        e = float((got[k].double().cpu() - g).abs().max()) / scale
        worst = max(worst, (k, e), key=lambda t: t[1])
    print("train %s pool_to_input=%s obs %d [%s]: worst gradient error %.2e of max (%s)"
          % (kind, pool_to_input, obs_length, "tc" if tc else "no_tc", worst[1], worst[0]))
    assert worst[1] <= 1e-4, worst


# ---------------------------------------------------------------------------------------------------------------------
# 3. drop-in: the reference's unmodified Trainer.train_batch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_reference_trainer_drives_external_model():
    _ref()
    from trajnetbaselines.lstm import trainer as ref_trainer
    from trajnetbaselines.lstm.loss import PredictionLoss as RefLoss
    from trajnetbaselines.lstm.lstm import LSTM as RefLSTM
    from trajnetplusplusbaselines_b200.lstm import LSTM, PredictionLoss
    pool = _ref_module("hiddenstatemlp", 7)
    torch.manual_seed(8)
    model = LSTM(pool=copy.deepcopy(pool))
    ref_model = RefLSTM(pool=copy.deepcopy(pool))
    ref_model.load_state_dict(model.state_dict())
    model = model.cuda().train()
    ref_model.train()
    xy, bs = O.synthetic_scenes(8, 7, seed=17, ragged=True, nan_tracks=True)
    B = len(bs) - 1
    scene, goals, split = torch.from_numpy(xy), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs)
    lr = 0.05
    t_ref = ref_trainer.Trainer(model=ref_model, criterion=RefLoss(), optimizer=torch.optim.SGD(ref_model.parameters(), lr=lr),
                                device=torch.device("cpu"), batch_size=B, augment=False)
    t_mine = ref_trainer.Trainer(model=model, criterion=PredictionLoss(), optimizer=torch.optim.SGD(model.parameters(), lr=lr),
                                 device=torch.device("cuda"), batch_size=B, augment=False)
    before = {k: v.detach().clone() for k, v in ref_model.state_dict().items()}
    loss_ref = t_ref.train_batch(scene, goals, split)
    loss = t_mine.train_batch(scene.cuda(), goals.cuda(), split.cuda())
    assert abs(loss - loss_ref) <= 1e-4 * max(1.0, abs(loss_ref)), (loss, loss_ref)
    sd_ref, sd = ref_model.state_dict(), model.state_dict()
    worst = 0.0
    for k in sd_ref:
        step_ref = (sd_ref[k] - before[k]).numpy()
        step = (sd[k].cpu() - before[k]).numpy()
        scale = max(float(np.abs(step_ref).max()), 1e-6 * lr)
        worst = max(worst, float(np.abs(step - step_ref).max()) / scale)
    assert worst < 1e-3, worst


# ---------------------------------------------------------------------------------------------------------------------
# 4. a sync-free user module
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
def test_sync_free_module_runs_without_host_synchronisation(monkeypatch, tc):
    from trajnetplusplusbaselines_b200.lstm import LSTM
    _tc(monkeypatch, tc)
    torch.manual_seed(3)
    pool = MixPool(out_dim=32)
    model = LSTM(pool=pool).cuda().train()
    xy, bs = O.synthetic_scenes(5, 9, seed=4, ragged=True, nan_tracks=True)
    scene = torch.from_numpy(xy).cuda()
    split = torch.from_numpy(bs)
    goals = torch.zeros(xy.shape[1], 2, device="cuda")
    model(scene[:9], goals, split, scene[9:20].clone())       # warm-up: layouts, handles, workspaces
    torch.cuda.synchronize()
    pool.calls.clear()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rel, pred = model(scene[:9], goals, split, scene[9:20].clone())
        loss = torch.nan_to_num(rel).square().sum() + torch.nan_to_num(pred).sum()
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    B, n_pad = len(bs) - 1, int(np.diff(bs).max())
    assert pool.calls[0] == ("reset", B * n_pad, n_pad - 1, torch.device("cuda", torch.cuda.current_device()))
    fwd = pool.calls[1:]
    assert len(fwd) == 8 + 11
    assert all(c == ("forward", (B, n_pad, 128), (B, n_pad, 2), (B, n_pad, 2)) for c in fwd), fwd[0]
    assert pool.hidden.weight.grad is not None and float(pool.hidden.weight.grad.abs().sum()) > 0


# ---------------------------------------------------------------------------------------------------------------------
# 5. end to end: the native Trainer, then the evaluator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_native_trainer_and_evaluator_end_to_end(tmp_path):
    _ref()
    from oracle.ref_shim import reference_root
    from trajnetplusplusbaselines_b200 import evaluator
    from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, paths_to_xy, read_ndjson_scenes, trajnet_line
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor, PredictionLoss
    from trajnetplusplusbaselines_b200.lstm import trainer as TR
    path = os.path.join(reference_root(), "DATA_BLOCK", "trajdata", "train", "biwi_hotel.ndjson")
    scenes = []
    for sid, paths in read_ndjson_scenes(path):
        scenes.append((sid, paths))
        if len(scenes) == 24:
            break
    pool = _ref_module("hiddenstatemlp", 9)
    torch.manual_seed(10)
    model = LSTM(pool=pool)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
    trainer = TR.Trainer(model=model, criterion=PredictionLoss(), optimizer=opt,
                         lr_scheduler=torch.optim.lr_scheduler.StepLR(opt, 1), device=torch.device("cuda"), batch_size=8,
                         augment=False, val_flag=False)
    store = TR.SceneStore([("biwi_hotel", sid, paths_to_xy(p)) for sid, p in scenes[:20]])
    out = str(tmp_path / "ext.pkl")
    trainer.loop(store, None, None, None, out, epochs=2)
    predictor = LSTMPredictor.load(out)
    state = torch.load(out + ".state", weights_only=False)
    assert any(k.startswith("pool.") for k in state["state_dict"])
    infile = str(tmp_path / "test.ndjson")
    rows = {}
    with open(infile, "w") as f:
        for sid, paths in scenes[20:]:
            frames = [r.frame for r in paths[0]]
            f.write(trajnet_line(SceneRow(sid, paths[0][0].pedestrian, frames[0], frames[-1], 2.5, 1)) + "\n")
            for p in paths:
                for r in p:
                    rows[(r.frame, r.pedestrian)] = r
        for key in sorted(rows):
            r = rows[key]
            f.write(trajnet_line(TrackRow(r.frame, r.pedestrian, r.x, r.y)) + "\n")
    assert evaluator.evaluate_file(predictor, infile, str(tmp_path / "pred.ndjson")) == 4
    assert os.path.getsize(tmp_path / "pred.ndjson") > 0
    # the batched column pipeline against the per-scene call
    batched = predictor.predict_batch_xy([paths_to_xy(p) for _, p in scenes[20:]], n_predict=12)
    for (_, paths), b in zip(scenes[20:], batched):
        one = predictor(paths, np.zeros((len(paths), 2)), n_predict=12)
        assert np.abs(one[0][0] - b[0][0]).max() <= 1e-5
        if one[0][1].size:
            assert (np.isnan(one[0][1]) == np.isnan(b[0][1])).all()
            assert np.nanmax(np.abs(one[0][1] - b[0][1]), initial=0.0) <= 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals():
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor
    from trajnetplusplusbaselines_b200.lstm.sampling import SampledLSTMPredictor
    from trajnetplusplusbaselines_b200.sgan.sgan import LSTMGenerator, SGAN, SGANPredictor
    from trajnetplusplusbaselines_b200.vae.vae import VAE, VAEPredictor
    model = LSTM(pool=MixPool(out_dim=32)).cuda()
    xy, bs = O.synthetic_scenes(2, 4, seed=1)
    xys = [xy[:, bs[i]:bs[i + 1]].astype(np.float64) for i in range(2)]
    with pytest.raises(NotImplementedError, match="external interaction module"):
        SampledLSTMPredictor(model).predict_batch_xy(xys, n_predict=12, modes=3)
    with pytest.raises(NotImplementedError, match="external interaction module"):
        list(SampledLSTMPredictor(model)._mode_scenes(torch.from_numpy(xy[:9, :4]), None, torch.tensor([0, 4]), 12, 2))
    gen = LSTMGenerator(pool=MixPool(out_dim=32)).cuda()
    with pytest.raises(NotImplementedError, match="external interaction module"):
        SGANPredictor(SGAN(generator=gen)).predict_batch_xy(xys, n_predict=12, modes=2)
    with pytest.raises(NotImplementedError, match="external interaction module"):
        VAEPredictor(VAE(pool=MixPool(out_dim=32)).cuda()).predict_batch_xy(xys, n_predict=12, modes=2)
    with pytest.raises(NotImplementedError, match="goal_flag=True with an external"):
        LSTM(pool=MixPool(out_dim=32), goal_flag=True).cuda()(torch.from_numpy(xy[:9]), torch.zeros(8, 2),
                                                              torch.from_numpy(bs), n_predict=12)
    goal_model = LSTM(pool=MixPool(out_dim=32), goal_flag=True).cuda()
    with pytest.raises(NotImplementedError, match="goal_flag=True with an external"):
        LSTMPredictor(goal_model).predict_batch_xy(xys, [np.zeros((4, 2))] * 2, n_predict=12)
