"""The native trainer (trajnetplusplusbaselines_b200/lstm/trainer.py) against the reference's Trainer
(trajnetbaselines/lstm/trainer.py, imported unmodified through oracle/ref_shim.py):

  * the epoch plan consumes Python's and NumPy's generators as Trainer.train does (CPU);
  * tb2_scenes_gather_epoch builds every batch bit for bit as the reference's per-scene NumPy chain (GPU);
  * the native Trainer.loop and the reference's Trainer.loop driving the same GPU model agree bit for bit: batches, losses,
    parameters, optimizer state (GPU);
  * the CLI end to end, and its refusals before any file is read.
"""
import copy
import json
import math
import os
import random
import warnings

import numpy as np
import pytest
import torch

from trajnetplusplusbaselines_b200.lstm import trainer as TR

TRAIN_FILES = ("biwi_hotel", "crowds_students001", "crowds_students003", "crowds_zara01", "crowds_zara03", "lcas",
               "wildtrack")


def _reference():
    from oracle.ref_shim import import_reference
    return import_reference()


def _train_path(name):
    from oracle.ref_shim import reference_root
    return os.path.join(reference_root(), "DATA_BLOCK", "trajdata", "train", name + ".ndjson")


def _ref_scenes(name, limit=None):
    """[(filename, scene_id, paths)] of a training file, as the reference's prepare_data holds them."""
    from trajnetplusplusbaselines_b200.data import read_ndjson_scenes
    out = []
    for sid, paths in read_ndjson_scenes(_train_path(name)):
        out.append((name, sid, paths))
        if limit is not None and len(out) == limit:
            break
    return out


def _kept_counts(scenes):
    from trajnetplusplusbaselines_b200.data import paths_to_xy
    from trajnetplusplusbaselines_b200.lstm.lstm import drop_distant
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.array([int(drop_distant(paths_to_xy(p))[1].sum()) for _, _, p in scenes], dtype=np.int64)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the epoch plan against the reference's Trainer.train / val (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _record_reference_epochs(scenes, opts, epochs, batch_size, seeds):
    """Run the reference Trainer.train / val with recorders in place of train_batch / val_batch; record the scene order,
    random_rotation's theta, add_noise's draw and every batch split."""
    ref = _reference()
    from trajnetbaselines.lstm import trainer as ref_trainer
    from trajnetbaselines.lstm.lstm import LSTM as RefLSTM
    model = RefLSTM()
    t = ref_trainer.Trainer(model=model, optimizer=torch.optim.SGD(model.parameters(), lr=0.0), device=torch.device("cpu"),
                            batch_size=batch_size, augment=opts["augment"], normalize_scene=opts["normalize_scene"],
                            augment_noise=opts["augment_noise"], obs_dropout=opts["obs_dropout"])
    rec = dict(thetas=[], noise=[], splits=[], starts=[], val_splits=[], orders=[])

    def train_batch(batch_scene, batch_scene_goal, batch_split):
        if t.obs_dropout:
            t.start_length = random.randint(0, t.obs_length - 2)
            rec["starts"].append(t.start_length)
        rec["splits"].append(batch_split.tolist())
        return 0.0

    def val_batch(batch_scene, batch_scene_goal, batch_split):
        rec["val_splits"].append(batch_split.tolist())
        return 0.0, 0.0

    orig_rotation, orig_noise = ref_trainer.random_rotation, ref.augmentation.add_noise

    def random_rotation(xy, goals=None):
        state = random.getstate()
        rec["thetas"].append(random.random() * 2.0 * math.pi)
        random.setstate(state)
        return orig_rotation(xy, goals=goals)

    def add_noise(observation, thresh=0.005, obs_length=9, ped='primary'):
        state = np.random.get_state()
        rec["noise"].append(np.random.uniform(-thresh, thresh, observation[:obs_length, 1:].shape))
        np.random.set_state(state)
        return orig_noise(observation, thresh=thresh, obs_length=obs_length, ped=ped)

    t.train_batch, t.val_batch = train_batch, val_batch
    ref_trainer.random_rotation, ref.augmentation.add_noise = random_rotation, add_noise
    random.seed(seeds[0])
    np.random.seed(seeds[1])
    train = list(scenes)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for epoch in range(epochs):
                t.train(train, None, epoch)
                rec["orders"].append([(f, sid) for f, sid, _ in train])
                t.val(scenes[:5], None, epoch)
    finally:
        ref_trainer.random_rotation, ref.augmentation.add_noise = orig_rotation, orig_noise
    rec["after"] = (random.random(), np.random.random_sample())
    return rec


OPTION_SETS = [dict(augment=a, augment_noise=n, obs_dropout=d, normalize_scene=z)
               for a in (False, True) for n in (False, True) for d in (False, True) for z in (False, True)]


@pytest.mark.needs_reference
@pytest.mark.parametrize("opts", OPTION_SETS, ids=lambda o: "-".join(k for k, v in o.items() if v) or "plain")
def test_epoch_plan_consumes_generators_like_reference(opts):
    scenes = _ref_scenes("biwi_hotel", 50) + _ref_scenes("crowds_zara01", 51)     # 101 scenes: a partial last batch
    batch_size, epochs, seeds = 8, 2, (5, 9)
    rec = _record_reference_epochs(scenes, opts, epochs, batch_size, seeds)
    kept = _kept_counts(scenes)
    names = [(f, sid) for f, sid, _ in scenes]
    random.seed(seeds[0])
    np.random.seed(seeds[1])
    order = list(range(len(scenes)))
    thetas, noise, splits, starts = [], [], [], []
    for epoch in range(epochs):
        plan = TR.draw_epoch_plan(order, kept, batch_size, 21, 9, opts["augment"], opts["augment_noise"],
                                  opts["obs_dropout"])
        assert [names[i] for i in plan.order] == rec["orders"][epoch]
        if opts["augment"]:
            thetas += plan.thetas.tolist()
        else:
            assert plan.thetas is None
        if opts["augment_noise"]:
            for p, s in enumerate(plan.order):
                size = 9 * (kept[s] - 1) * 2
                noise.append(plan.noise[plan.noise_off[p]:plan.noise_off[p] + size].reshape(9, kept[s] - 1, 2))
            assert plan.noise_off[-1] + 9 * (kept[plan.order[-1]] - 1) * 2 == len(plan.noise)
        else:
            assert plan.noise is None
        starts += plan.start_lengths or []
        splits += [s.tolist() for s in plan.splits]
    assert thetas == rec["thetas"]
    assert len(noise) == len(rec["noise"])
    for a, b in zip(noise, rec["noise"]):
        assert a.shape == b.shape and np.array_equal(a, b)
    assert starts == rec["starts"]
    assert splits == rec["splits"] and len(splits[-1]) == 101 % 8 + 1
    assert (random.random(), np.random.random_sample()) == rec["after"]      # val draws nothing, on both sides


@pytest.mark.needs_reference
def test_one_noise_draw_equals_per_scene_draws():
    """add_noise draws uniform(-0.02, 0.02, [9, N - 1, 2]) per scene (N = 1 included); one draw of the concatenated size
    gives the same values."""
    shapes = [(9, k, 2) for k in (3, 0, 1, 7, 0, 12, 2)]
    np.random.seed(123)
    per_scene = [np.random.uniform(-0.02, 0.02, s) for s in shapes]
    after = np.random.random_sample()
    np.random.seed(123)
    flat = np.random.uniform(-0.02, 0.02, sum(int(np.prod(s)) for s in shapes))
    assert np.random.random_sample() == after
    assert np.array_equal(np.concatenate([a.reshape(-1) for a in per_scene]), flat)


# ---------------------------------------------------------------------------------------------------------------------
# 2. tb2_scenes_gather_epoch against the reference's per-scene chain (GPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_mixed_frame_counts_raise(tmp_path):
    xy = lambda T, n: np.zeros((T, n, 2))
    with pytest.raises(ValueError, match="fileB: scene 7 has 20 frames"):
        TR.SceneStore([("fileA", 1, xy(21, 3)), ("fileB", 7, xy(20, 2))])
    from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, trajnet_line
    fn = str(tmp_path / "mixed.ndjson")
    with open(fn, "w") as f:
        for sid, (s, e) in enumerate([(0, 20), (100, 190)]):
            f.write(trajnet_line(SceneRow(sid, 1, s, e, 2.5, 1)) + "\n")
        for frame in list(range(0, 21)) + list(range(100, 191, 10)):
            f.write(trajnet_line(TrackRow(frame, 1, 0.1 * frame, 0.0)) + "\n")
    with pytest.raises(ValueError, match="mixed.ndjson: scene 1 has 10 frames"):
        TR.SceneStore.from_files([fn])


def _reference_chain(ref, xy, obs_length, normalize, augment, noise):
    from trajnetbaselines.lstm import lstm as ref_lstm
    from trajnetbaselines.lstm import utils as ref_utils
    scene, _ = ref_lstm.drop_distant(xy)
    if normalize:
        scene, _, _ = ref_utils.center_scene(scene, obs_length)
    if augment:
        scene = ref_utils.random_rotation(scene)
    if noise:
        scene = ref.augmentation.add_noise(scene, thresh=0.02, ped='neigh')
    return scene


@pytest.mark.gpu
@pytest.mark.needs_reference
def test_gather_epoch_matches_reference_chain_bitwise():
    ref = _reference()
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.data import load_scenes_xy
    files = [_train_path(n) for n in TRAIN_FILES]
    store = TR.SceneStore.from_files(files)
    assert store.n > 10000 and store.T == 21
    xys = [xy for f in files for _, xy in load_scenes_xy(f)]
    assert len(xys) == store.n
    cases = [(9, z, a, n) for z in (False, True) for a in (False, True) for n in (False, True)] + [(5, True, True, True)]
    batch_size = 64
    for obs_length, normalize, augment, noise in cases:
        random.seed(11)
        np.random.seed(12)
        plan = TR.draw_epoch_plan(list(range(store.n)), store.kept, batch_size, store.T, obs_length, augment, noise)
        frame = store.frames(obs_length) if normalize else None
        before = _lib.load().tb2_launch_count()
        batches = store.gather(plan.order, batch_size, frame=frame, thetas=plan.thetas, noise=plan.noise,
                               noise_off=plan.noise_off)
        assert _lib.load().tb2_launch_count() == before + 1                  # the whole epoch in one launch
        random.seed(11)
        np.random.seed(12)
        order = list(range(store.n))
        random.shuffle(order)
        assert order == plan.order.tolist()
        prev_end = None
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for k, (view, split) in enumerate(batches):
                chain = [_reference_chain(ref, xys[s], obs_length, normalize, augment, noise)
                         for s in order[k * batch_size:(k + 1) * batch_size]]
                want = torch.Tensor(np.concatenate(chain, axis=1)).numpy()
                assert split.tolist() == np.cumsum([0] + [c.shape[1] for c in chain]).tolist()
                assert view.is_contiguous() and tuple(view.shape) == want.shape
                if prev_end is not None:
                    assert view.data_ptr() == prev_end                       # batches follow each other in one buffer
                prev_end = view.data_ptr() + view.numel() * 4
                assert _same(view.cpu().numpy(), want), (obs_length, normalize, augment, noise, k)


# ---------------------------------------------------------------------------------------------------------------------
# 3. the native loop against the reference's loop driving the same GPU model (GPU)
# ---------------------------------------------------------------------------------------------------------------------
LOOP_CONFIGS = {
    "vanilla": dict(pool=None, loss="pred", col_wt=0.0, opts=dict()),
    "directional_aug_norm": dict(pool=dict(type_="directional"), loss="pred", col_wt=0.0,
                                 opts=dict(augment=True, normalize_scene=True)),
    "social_noise_dropout": dict(pool=dict(type_="social"), loss="pred", col_wt=0.0,
                                 opts=dict(augment_noise=True, obs_dropout=True)),
    # the reference's val_batch calls the criterion without positions, which its collision term asserts on
    # (lstm/loss.py:118-119): with col_wt > 0 the reference trains without validation, and so does this check
    "directional_l2_col": dict(pool=dict(type_="directional"), loss="L2", col_wt=0.1, opts=dict(), val=False),
}


def _make_model(cfg):
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    torch.manual_seed(3)
    pool = None
    if cfg["pool"] is not None:
        pool = GridBasedPooling(hidden_dim=128, cell_side=0.6, n=12, out_dim=256, embedding_arch="one_layer", constant=0,
                                layer_dims=[512], latent_dim=16, **cfg["pool"])
    return LSTM(pool=pool, embedding_dim=64, hidden_dim=128).cuda()


def _criterion(cfg):
    from trajnetplusplusbaselines_b200.lstm import L2Loss, PredictionLoss
    return L2Loss(col_wt=cfg["col_wt"]) if cfg["loss"] == "L2" else PredictionLoss(col_wt=cfg["col_wt"])


def _record_forward(monkeypatch, holder):
    """Record what LSTM.forward receives into holder["rec"] (patched on the class: the loops pickle the model)."""
    from trajnetplusplusbaselines_b200.lstm import LSTM
    fwd = LSTM.forward

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None):
        holder["rec"]["forward"].append((observed.detach().cpu().numpy().copy(), [int(v) for v in batch_split],
                                         None if prediction_truth is None else prediction_truth.detach().cpu().numpy().copy(),
                                         n_predict))
        return fwd(self, observed, goals, batch_split, prediction_truth, n_predict)

    monkeypatch.setattr(LSTM, "forward", forward)


def _instrument(trainer, model):
    rec = dict(forward=[], train_loss=[], val_loss=[], after_epoch=[])
    tb, vb, tr = trainer.train_batch, trainer.val_batch, trainer.train

    def train_batch(*a):
        loss = tb(*a)
        rec["train_loss"].append(float(loss))
        return loss

    def val_batch(*a):
        loss, loss_test = vb(*a)
        rec["val_loss"].append((float(loss), float(loss_test)))
        return loss, loss_test

    def train(*a):
        tr(*a)
        rec["after_epoch"].append((copy.deepcopy({k: v.cpu() for k, v in model.state_dict().items()}),
                                   copy.deepcopy(trainer.optimizer.state_dict())))

    trainer.train_batch, trainer.val_batch, trainer.train = train_batch, val_batch, train
    return rec


def _same(a, b):
    """Bit for bit, except that a NaN equals any NaN: NumPy on the host keeps a NaN operand's sign through a product, the
    device returns the canonical NaN, and every consumer of a coordinate only asks isnan."""
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    nan = np.isnan(a)
    if not np.array_equal(nan, np.isnan(b)):
        return False
    return np.array_equal(a[~nan].view(np.uint8), b[~nan].view(np.uint8))


@pytest.mark.gpu
@pytest.mark.needs_reference
@pytest.mark.parametrize("name", list(LOOP_CONFIGS))
def test_native_loop_matches_reference_loop_bitwise(name, tmp_path, monkeypatch):
    _reference()
    from trajnetbaselines.lstm import trainer as ref_trainer
    from trajnetplusplusbaselines_b200.data import paths_to_xy
    cfg = LOOP_CONFIGS[name]
    opts = cfg["opts"]
    train_list = _ref_scenes("crowds_zara01", 24)
    val_list = _ref_scenes("biwi_hotel", 5)
    holder = {}
    _record_forward(monkeypatch, holder)
    records = []
    for native in (False, True):
        model = _make_model(cfg)
        opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
        sched = torch.optim.lr_scheduler.StepLR(opt, 1)
        kw = dict(model=model, criterion=_criterion(cfg), optimizer=opt, lr_scheduler=sched, device=torch.device("cuda"),
                  batch_size=8, augment=opts.get("augment", False), normalize_scene=opts.get("normalize_scene", False),
                  augment_noise=opts.get("augment_noise", False), obs_dropout=opts.get("obs_dropout", False),
                  val_flag=cfg.get("val", True))
        if native:
            trainer = TR.Trainer(**kw)
            train = TR.SceneStore([(f, sid, paths_to_xy(p)) for f, sid, p in train_list])
            val = TR.SceneStore([(f, sid, paths_to_xy(p)) for f, sid, p in val_list])
        else:
            trainer = ref_trainer.Trainer(**kw)
            train, val = list(train_list), list(val_list)
        rec = holder["rec"] = _instrument(trainer, model)
        random.seed(21)
        np.random.seed(22)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            trainer.loop(train, val, None, None, str(tmp_path / ("native" if native else "ref")), epochs=2)
        records.append(rec)
    ref, mine = records
    assert len(ref["forward"]) == len(mine["forward"]) == 2 * (3 + (2 if cfg.get("val", True) else 0))
    for i, (r, m) in enumerate(zip(ref["forward"], mine["forward"])):
        assert _same(r[0], m[0]), ("observed", i)
        assert r[1] == m[1], ("split", i)
        assert (r[2] is None) == (m[2] is None) and (r[2] is None or _same(r[2], m[2])), ("prediction_truth", i)
        assert r[3] == m[3]
    assert _same(np.array(ref["train_loss"], dtype=np.float64), np.array(mine["train_loss"], dtype=np.float64))
    assert _same(np.array(ref["val_loss"], dtype=np.float64), np.array(mine["val_loss"], dtype=np.float64))
    for (sd_r, opt_r), (sd_m, opt_m) in zip(ref["after_epoch"], mine["after_epoch"]):
        assert list(sd_r) == list(sd_m)
        for k in sd_r:
            assert _same(sd_r[k].numpy(), sd_m[k].numpy()), k
        assert opt_r["param_groups"] == opt_m["param_groups"]
        for idx, st in opt_r["state"].items():
            for k, v in st.items():
                assert _same(v.cpu().numpy(), opt_m["state"][idx][k].cpu().numpy()), (idx, k)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the CLI end to end (GPU; the data files come from the reference's DATA_BLOCK)
# ---------------------------------------------------------------------------------------------------------------------
def _write_dataset(root, val_scenes=5):
    import shutil
    from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, trajnet_line
    train = os.path.join(root, "DATA_BLOCK", "tiny", "train")
    val = os.path.join(root, "DATA_BLOCK", "tiny", "val")
    os.makedirs(train)
    os.makedirs(val)
    for name in ("biwi_hotel", "crowds_zara03"):
        shutil.copy(_train_path(name), train)
    rows = {}
    with open(os.path.join(val, "lcas_val.ndjson"), "w") as f:
        for _, sid, paths in _ref_scenes("lcas", val_scenes):
            frames = [r.frame for r in paths[0]]
            f.write(trajnet_line(SceneRow(sid, paths[0][0].pedestrian, frames[0], frames[-1], 2.5, 1)) + "\n")
            for path in paths:
                for r in path:
                    rows[(r.frame, r.pedestrian)] = r
        for key in sorted(rows):
            r = rows[key]
            f.write(trajnet_line(TrackRow(r.frame, r.pedestrian, r.x, r.y)) + "\n")


def _log_records(fn):
    with open(fn) as f:
        return [json.loads(line) for line in f if line.strip()]


@pytest.mark.gpu
@pytest.mark.needs_reference
def test_cli_end_to_end(tmp_path, monkeypatch):
    _reference()
    from trajnetbaselines.lstm.gridbased_pooling import GridBasedPooling as RefPool
    from trajnetbaselines.lstm.lstm import LSTM as RefLSTM
    from trajnetplusplusbaselines_b200 import evaluator
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    _write_dataset(str(tmp_path))
    monkeypatch.chdir(tmp_path)
    common = ["--path", "tiny", "--type", "directional", "--save_every", "1", "--step_size", "1", "--output", "t"]
    TR.main(common + ["--epochs", "2"])
    out = os.path.join("OUTPUT_BLOCK", "tiny")
    base = "lstm_directional_t.pkl"
    expect = {base, base + ".state", base + ".log"}
    for k in range(3):
        expect |= {base + ".epoch%d" % k, base + ".epoch%d.state" % k}
    assert set(os.listdir(out)) == expect
    records = _log_records(os.path.join(out, base + ".log"))
    types = [r["type"] for r in records]
    assert types[0] == "process" and types.count("train-epoch") == 2 and types.count("val-epoch") == 2
    assert "train" in types                                  # the two files hold more than 10 batches of 8 scenes
    keys = {"process": {"argv", "args", "version", "hostname"},
            "train": {"epoch", "batch", "n_batches", "time", "data_time", "lr", "loss"},
            "train-epoch": {"epoch", "loss", "time"}, "val-epoch": {"epoch", "loss", "test_loss", "time"}}
    for r in records:
        assert keys[r["type"]] | {"type", "message", "levelname", "name", "asctime"} == set(r), r
        if r["type"] != "process":
            assert r["name"] == "Trainer"
    assert [r["epoch"] for r in records if r["type"] == "train-epoch"] == [1, 2]
    assert all(math.isfinite(r["loss"]) for r in records if r["type"] in ("train-epoch", "val-epoch"))

    predictor = LSTMPredictor.load(os.path.join(out, base))
    predictor.model.to("cuda")
    infile = os.path.join("DATA_BLOCK", "tiny", "val", "lcas_val.ndjson")
    assert evaluator.evaluate_file(predictor, infile, str(tmp_path / "pred.ndjson")) == 5
    assert os.path.getsize(tmp_path / "pred.ndjson") > 0

    state = torch.load(os.path.join(out, base + ".state"), map_location="cpu")
    assert state["epoch"] == 2
    ref_model = RefLSTM(pool=RefPool(type_="directional", hidden_dim=128, cell_side=0.6, n=12, front=False, out_dim=256,
                                     embedding_arch="one_layer", constant=0, norm=0, layer_dims=[512], latent_dim=16),
                        embedding_dim=64, hidden_dim=128, goal_flag=False, goal_dim=64)
    ref_model.load_state_dict(state["state_dict"], strict=True)

    # --load-full-state: epoch, optimizer and scheduler come back; the re-saved .epoch1 equals the one it was loaded from
    first = torch.load(os.path.join(out, base + ".epoch1.state"), map_location="cpu")
    assert first["optimizer"]["param_groups"][0]["lr"] == pytest.approx(1e-4)
    os.rename(os.path.join(out, base + ".epoch1.state"), str(tmp_path / "resume.state"))
    TR.main(common + ["--epochs", "3", "--load-full-state", str(tmp_path / "resume.state")])
    again = torch.load(os.path.join(out, base + ".epoch1.state"), map_location="cpu")
    assert again["epoch"] == 1 and again["scheduler"] == first["scheduler"]
    assert again["optimizer"]["param_groups"] == first["optimizer"]["param_groups"]
    for k, v in first["state_dict"].items():
        assert torch.equal(v, again["state_dict"][k]), k
    for idx, st in first["optimizer"]["state"].items():
        for k, v in st.items():
            assert torch.equal(v, again["optimizer"]["state"][idx][k]), (idx, k)
    final = torch.load(os.path.join(out, base + ".state"), map_location="cpu")
    assert final["epoch"] == 3
    assert final["optimizer"]["param_groups"][0]["lr"] == pytest.approx(1e-6)
    steps = {float(st["step"]) for st in final["optimizer"]["state"].values()}
    assert steps == {3 * float(next(iter(first["optimizer"]["state"].values()))["step"])}
    records = _log_records(os.path.join(out, base + ".log"))          # appended to, like the reference
    assert [r["type"] for r in records].count("process") == 2
    assert [r["epoch"] for r in records if r["type"] == "train-epoch"] == [1, 2, 2, 3]


# ---------------------------------------------------------------------------------------------------------------------
# 5. refusals, before any file is read (CPU)
# ---------------------------------------------------------------------------------------------------------------------
REFUSALS = [
    (["--type", "hiddenstatemlp"], "training of HiddenStateMLPPooling is not built"),
    (["--type", "nn"], "training of NearestNeighborMLP is not built"),
    (["--type", "attentionmlp"], "training of AttentionMLPPooling is not built"),
    (["--type", "nn_lstm"], "training of NearestNeighborLSTM is not built"),
    (["--type", "traj_pool"], "training of TrajectronPooling is not built"),
    (["--goals"], "goal_flag=True is not built"),
    (["--type", "occupancy", "--embedding_arch", "two_layer"],
     "training backward supports one_layer grid embeddings with constant = 0"),
    (["--type", "directional", "--pool_constant", "1"],
     "training backward supports one_layer grid embeddings with constant = 0"),
    (["--type", "social", "--embedding_arch", "None"],
     "social training backward supports one_layer / two_layer embeddings with constant = 0"),
]


@pytest.mark.parametrize("argv,message", REFUSALS, ids=[" ".join(a) for a, _ in REFUSALS])
def test_cli_refuses_before_reading_data(argv, message, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                    # no DATA_BLOCK here: reading any data file would fail differently
    with pytest.raises(SystemExit) as e:
        TR.main(["--path", "nowhere"] + argv)
    assert message in str(e.value.code)
    assert os.listdir(tmp_path) == []             # no OUTPUT_BLOCK, no log


def test_prepare_data_folders(tmp_path, capsys):
    assert TR.prepare_data(str(tmp_path), subset="/val/") == (None, None, False)
    with pytest.raises(SystemExit):
        TR.prepare_data(str(tmp_path), subset="/train/")
    assert "Train folder does NOT exist" in capsys.readouterr().out


def test_json_log_records():
    import logging
    rec = logging.LogRecord("Trainer", logging.INFO, __file__, 1, {"type": "train-epoch", "epoch": 1, "loss": 0.5}, None,
                            None)
    out = json.loads(TR.JsonLineFormatter().format(rec))
    assert list(out) == ["message", "levelname", "name", "asctime", "type", "epoch", "loss"]
    assert out["message"] is None and out["name"] == "Trainer" and out["loss"] == 0.5
