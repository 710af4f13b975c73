"""Goal-conditioned LSTM inference: LSTM(goal_flag=True) (reference lstm.py:72-85,131-139) and goal files through the
evaluator (reference lstm/trajnet_evaluator.py:52-57, evaluator/write_utils.py:21-25).

CPU:
  * a float64 restatement of the goal-conditioned step / forward (below; pooling from torch_ref) against
    tests/golden/goal_golden.npz, made by the unmodified reference (oracle/make_goal_golden.py): vanilla at goal_dim 64
    and 32, occupancy, directional, social, hidden-state MLP and nearest-neighbour pooling, a zero-norm goal direction
    and absent tracks, free-running and teacher-forced;
  * refusals: the training forward, S-GAN / VAE with goal_flag=True; the evaluator's missing goal file / pedestrian id.
GPU:
  * one step of every interaction module at H = 32, 128, 256, goal_dim 64 (tensor-core gates where they apply) and 32
    (FFMA gates), with the tensor cores on and under TB2_DISABLE_TC=1, and pool_to_input=False; the kernel that ran
    is asserted from the profile timer names;
  * whole forwards in the padded and the per-scene layouts; the goal-taking C calls without goals;
  * a reference-pickled goal predictor against this package's; evaluator files from the column pipeline, the row
    pipeline and the per-scene call, byte-identical, with and without --normalize_scene.
"""
import argparse
import ctypes
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch_ref as TR  # noqa: E402
from oracle import lstm_oracle as O  # noqa: E402
from oracle.make_goal_golden import CASES, goal_inputs, goal_weights, model_kwargs  # noqa: E402
from test_hidden_dim import _nan_rel, _profiled, _set_tc  # noqa: E402
from test_step_forward import BF16_KERNELS, NONGRID, STEP_GATE, _cfg, _pool_module, _state, _step_scenes  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
NAN = float("nan")
PHASES = ("encoder", "decoder")


# ---------------------------------------------------------------------------------------------------------------------
# float64 restatement of the goal-conditioned step (lstm.py:118-168 with :131-139)
# ---------------------------------------------------------------------------------------------------------------------
def goal_embedding(W, obs2, goals, dtype):
    """cat(ReLU(W_g . 4 d + b_g), 0, 0), d = (obs2 - goal) / |obs2 - goal| (0 at norm 0), for every row."""
    diff = (obs2 - goals).to(dtype)
    norm = torch.sqrt((diff * diff).sum(dim=1, keepdim=True))
    d = torch.where(norm == 0, torch.zeros_like(diff), diff / norm)
    e = torch.relu((d * 4.0) @ W["goal_embedding.input_embeddings.0.weight"].T + W["goal_embedding.input_embeddings.0.bias"])
    return torch.cat([e, torch.zeros(e.shape[0], 2, dtype=dtype)], dim=1)


def goal_step(W, cfg, phase, h, c, obs1, obs2, goals, bs, H, dtype=F64, pool_to_input=True, pad_to_batch_max=True,
              pool_state=None):
    M = obs2.shape[0]
    mask = ~torch.isnan(obs1[:, 0]) & ~torch.isnan(obs2[:, 0])
    vel = (obs2 - obs1)[mask].to(dtype)
    e = torch.relu((vel * 4.0) @ W["input_embedding.input_embeddings.0.weight"].T + W["input_embedding.input_embeddings.0.bias"])
    x = torch.cat([e, torch.zeros(e.shape[0], 2, dtype=dtype), goal_embedding(W, obs2, goals, dtype)[mask]], dim=1)
    hm = h[mask]
    if getattr(cfg, "type_", None) in TR.NONGRID:
        pooled = TR.nongrid_pool_ragged(cfg, W, h, obs1, obs2, bs, pad_to_batch_max, dtype, pool_state)[mask]
    elif cfg is not None:
        pooled = TR._grid(cfg, W, TR._pad(obs1, bs, NAN), TR._pad(obs2, bs, NAN), TR._pad(h, bs, NAN), dtype, None,
                          primary_edges=phase == "decoder")[TR._pad(mask, bs, False).reshape(-1)]
    if cfg is not None:
        if pool_to_input:
            x = torch.cat([x, pooled], dim=1)
        else:
            hm = hm + pooled
    gates = x @ W[phase + ".weight_ih"].T + W[phase + ".bias_ih"] + hm @ W[phase + ".weight_hh"].T + W[phase + ".bias_hh"]
    i, f = torch.sigmoid(gates[:, :H]), torch.sigmoid(gates[:, H:2 * H])
    g, o = torch.tanh(gates[:, 2 * H:3 * H]), torch.sigmoid(gates[:, 3 * H:])
    c2 = f * c[mask] + i * g
    h2 = o * torch.tanh(c2)
    raw = h2 @ W["hidden2normal.linear.weight"].T + W["hidden2normal.linear.bias"]
    nrm = torch.cat([raw[:, :2], 0.01 + 0.2 * torch.sigmoid(raw[:, 2:4]), 0.7 * torch.sigmoid(raw[:, 4:5])], dim=1)
    idx = mask.nonzero().flatten()
    return (h.index_copy(0, idx, h2), c.index_copy(0, idx, c2),
            torch.full((M, 5), NAN, dtype=dtype).index_copy(0, idx, nrm))


def goal_forward(W, cfg, observed, goals, bs, H, prediction_truth=None, n_predict=None, pad_to_batch_max=True,
                 pool_to_input=True):
    """LSTM.forward (lstm.py:170-264) of a goal model in float64; positions fed back in float32 like the reference."""
    bs = [int(v) for v in bs]
    M = observed.shape[1]
    prim = torch.tensor(bs[:-1])
    h, c = torch.zeros(M, H, dtype=F64), torch.zeros(M, H, dtype=F64)
    state = TR.pool_state_zeros(cfg, M, F64)
    truth = [None] * (n_predict - 1) if n_predict is not None else [t.clone() for t in prediction_truth]
    normals, positions = [], []

    def step(phase, h, c, o1, o2):
        return goal_step(W, cfg, phase, h, c, o1, o2, goals, bs, H, F64, pool_to_input, pad_to_batch_max, state)

    for t in range(observed.shape[0] - 1):
        h, c, n = step("encoder", h, c, observed[t], observed[t + 1])
        normals.append(n)
        positions.append(observed[t + 1] + n[:, :2].to(observed.dtype))
    seq = [observed[-1].clone()] + truth
    for k in range(len(seq) - 1):
        o1, o2 = seq[k], seq[k + 1]
        if o1 is None:
            o1 = positions[-2]
        else:
            o1 = o1.clone()
            o1[prim] = positions[-2][prim]
        if o2 is None:
            o2 = positions[-1]
        else:
            o2 = o2.clone()
            o2[prim] = positions[-1][prim]
            seq[k + 1] = o2
        h, c, n = step("decoder", h, c, o1, o2)
        normals.append(n)
        positions.append(o2 + n[:, :2].to(o2.dtype))
    return torch.stack(normals).numpy(), torch.stack(positions).numpy()


def _w64(W):
    return {k: torch.tensor(v, dtype=F64) for k, v in W.items()}


def _case_cfg(kind):
    table, spec = model_kwargs(kind)
    if spec is None:
        return None
    cls = {id(O.NONGRID_SPECS): O.MlpPoolConfig, id(O.NN_SPECS): O.NnPoolConfig}.get(id(table), O.PoolConfig)
    return cls(**spec)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the restatement against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "goal_golden.npz"))


@pytest.mark.parametrize("case,kind,goal_dim,seed", CASES, ids=[c[0] for c in CASES])
def test_restatement_matches_reference(golden, case, kind, goal_dim, seed):
    xy, bs, goals = goal_inputs()
    assert np.array_equal(xy, golden["xy"], equal_nan=True) and np.array_equal(goals, golden["goals"])
    o2 = xy[8]
    assert ((o2 - goals) == 0).all(axis=1).any()                     # a zero-norm goal direction is covered
    assert np.isnan(xy[:9, :, 0]).any()                              # and absent tracks
    W, cfg = _w64(goal_weights(kind, goal_dim, seed)), _case_cfg(kind)
    with torch.no_grad():
        rel_f, pred_f = goal_forward(W, cfg, torch.from_numpy(xy[:9]), torch.from_numpy(goals), bs, 128, n_predict=12)
        rel_t, pred_t = goal_forward(W, cfg, torch.from_numpy(xy[:9]), torch.from_numpy(goals), bs, 128,
                                     prediction_truth=torch.from_numpy(xy[9:20]))
    for name, got in (("rel_free", rel_f), ("pred_free", pred_f), ("rel_teacher", rel_t), ("pred_teacher", pred_t)):
        assert _nan_rel(got, golden[case + "/" + name]) <= 2e-6, (case, name)


def _goal_model(kind, H, W, goal_dim, pool_to_input=True, cls=None):
    from trajnetplusplusbaselines_b200.lstm import LSTM
    cls = cls or LSTM
    model = cls(hidden_dim=H, pool=_pool_module(kind, H, None if pool_to_input else H), pool_to_input=pool_to_input,
                goal_flag=True, goal_dim=goal_dim)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    return model


def test_training_forward_refuses_goals():
    from trajnetplusplusbaselines_b200.lstm.trainer import GOALS_MESSAGE
    model = _goal_model("vanilla", 128, goal_weights("vanilla", 64, 1), 64)
    xy, bs, goals = goal_inputs()
    with pytest.raises(NotImplementedError, match="goal_flag=True is not built") as err:
        model(torch.from_numpy(xy[:9]), torch.from_numpy(goals), torch.from_numpy(bs),
              prediction_truth=torch.from_numpy(xy[9:20]))
    assert str(err.value) == GOALS_MESSAGE


def test_sgan_and_vae_refuse_goals():
    from trajnetplusplusbaselines_b200.sgan import SGAN, LSTMDiscriminator, LSTMGenerator
    from trajnetplusplusbaselines_b200.vae import VAE
    xy, bs, goals = goal_inputs()
    obs, g, split = torch.from_numpy(xy[:9]), torch.from_numpy(goals), torch.from_numpy(bs)
    gen = LSTMGenerator(goal_flag=True).eval()
    disc = LSTMDiscriminator(goal_flag=True).eval()
    vae = VAE(goal_flag=True).eval()
    with torch.no_grad():
        for call in (lambda: gen(obs, g, split, n_predict=12), lambda: SGAN(gen, disc)(obs, g, split, n_predict=12),
                     lambda: disc(obs, torch.from_numpy(xy[9:])[:12], g, split), lambda: vae(obs, g, split, n_predict=12)):
            with pytest.raises(NotImplementedError, match="goal"):
                call()


# ---------------------------------------------------------------------------------------------------------------------
# evaluator: goal files
# ---------------------------------------------------------------------------------------------------------------------
def _dataset(root, sizes, seed, drop=None, name="data"):
    """DATA_BLOCK/goals/test/<name>.ndjson (scenes with a late-appearing track) and its goal file, every pedestrian's
    goal at its last position in the file; drop: a pedestrian id left out of the goal file."""
    from test_classical_evaluator import _write_scenes
    from trajnetplusplusbaselines_b200.data import read_ndjson_scenes
    test_dir = os.path.join(root, "DATA_BLOCK", "goals", "test")
    os.makedirs(test_dir, exist_ok=True)
    infile = os.path.join(test_dir, name + ".ndjson")
    _write_scenes(infile, sizes, seed)
    goals = {}
    for _, paths in read_ndjson_scenes(infile):
        for path in paths:
            goals[path[0].pedestrian] = (path[-1].x, path[-1].y)
    goals.pop(drop, None)
    os.makedirs(os.path.join(root, "goal_files", "test_private"), exist_ok=True)
    with open(os.path.join(root, "goal_files", "test_private", name + ".pkl"), "wb") as f:
        pickle.dump(goals, f)
    return infile


class _GoalModel(torch.nn.Module):
    goal_flag = True


class _RecordingPredictor:
    """predict_batch_xy records the goals it gets (no device needed)."""

    def __init__(self):
        self.model = _GoalModel()
        self.goals = []

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None):
        self.goals.extend(scene_goals)
        return [{0: [np.zeros((n_predict, 2)), np.zeros((n_predict, xy.shape[1] - 1, 2))]} for xy in xys]


def _eval_args(path, **kw):
    args = argparse.Namespace(path=path, output=["model.pkl"], obs_length=9, pred_length=12, modes=1, chunk=4,
                              normalize_scene=False)
    args.__dict__.update(kw)
    return args


def test_evaluator_reads_goal_files_and_refuses_missing_ones(tmp_path, monkeypatch):
    from trajnetplusplusbaselines_b200 import evaluator
    monkeypatch.chdir(str(tmp_path))
    _dataset(str(tmp_path), [5, 3, 6, 4], seed=3)
    pred_dir = os.path.join("DATA_BLOCK", "goals", "test_pred") + os.sep
    rec = _RecordingPredictor()
    evaluator.get_predictions(_eval_args(pred_dir), load_predictor=lambda f: rec)
    with open(os.path.join("goal_files", "test_private", "data.pkl"), "rb") as f:
        table = pickle.load(f)
    scenes = evaluator.load_test_scenes_xy(os.path.join("DATA_BLOCK", "goals", "test", "data.ndjson"))
    assert len(rec.goals) == len(scenes)
    for g, (xy, meta) in zip(rec.goals, scenes):
        assert g.shape == (xy.shape[1], 2)                               # the tracks preprocess_test kept
        assert np.array_equal(g, np.array([table[p] for p in [meta.pedestrian] + meta.neigh_ids]))
    # a missing goal file: refused before the model folder is created
    os.remove(os.path.join("goal_files", "test_private", "data.pkl"))
    args = _eval_args(pred_dir, output=["other.pkl"])
    with pytest.raises(FileNotFoundError, match="goal_files/test_private/data.pkl"):
        evaluator.get_predictions(args, load_predictor=lambda f: _RecordingPredictor())
    assert not os.path.exists(os.path.join(pred_dir, "other_modes1"))


@pytest.mark.parametrize("drop", [101, 3], ids=["kept_track", "dropped_late_track"])
def test_evaluator_refuses_a_missing_pedestrian_id(tmp_path, monkeypatch, drop):
    """Two test files, the second one's goal file lacks an id: nothing is written, not even the model folder (a re-run
    would skip the model).  Like the reference, a track preprocess_test drops (pedestrian 3 enters after the
    observation) needs a goal too."""
    from trajnetplusplusbaselines_b200 import evaluator
    from trajnetplusplusbaselines_b200.data import read_ndjson_scenes
    monkeypatch.chdir(str(tmp_path))
    _dataset(str(tmp_path), [5, 3, 6], seed=4, name="a_first")
    second = _dataset(str(tmp_path), [5, 3, 6], seed=5, drop=drop, name="b_second")
    late = [p[0].pedestrian for _, paths in read_ndjson_scenes(second) for p in paths
            if p[0].frame > sorted(r.frame for r in paths[0])[8]]
    assert 3 in late and 101 not in late
    pred_dir = os.path.join("DATA_BLOCK", "goals", "test_pred") + os.sep
    rec = _RecordingPredictor()
    with pytest.raises(KeyError, match="b_second.pkl has no goal for pedestrian %d" % drop):
        evaluator.get_predictions(_eval_args(pred_dir), load_predictor=lambda f: rec)
    assert not os.path.exists(os.path.join(pred_dir, "model_modes1")) and not rec.goals


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
STEP_KINDS = ["vanilla", "occupancy", "directional", "social_default", "hiddenstatemlp", "attentionmlp", "nn", "nn_lstm",
              "traj_pool"]


def _gpu_goal_step(model, phase, obs1, obs2, goals, bs, h, c):
    def run():
        if model.pool is not None and getattr(model.pool, "stateful", False):
            handle = model._engine()
            handle.pool_state_reset(model._layouts.get(bs, device=handle.device))
        with torch.no_grad():
            (h2, c2), normal = model.step(getattr(model, phase), (torch.from_numpy(h).cuda(), torch.from_numpy(c).cuda()),
                                          torch.from_numpy(obs1), torch.from_numpy(obs2), torch.from_numpy(goals),
                                          torch.from_numpy(bs))
        return [t.cpu().numpy() for t in (h2, c2, normal)]
    return _profiled(run)


def _step_goals(obs2, seed):
    rng = np.random.RandomState(seed)
    goals = (np.nan_to_num(obs2) + rng.randn(*obs2.shape) * 3.0).astype(np.float32)
    present = np.nonzero(~np.isnan(obs2[:, 0]))[0]
    goals[present[0]] = obs2[present[0]]                                 # zero-norm direction
    return goals


def _check_goal_step(kind, H, goal_dim, tc, pool_to_input=True):
    W = goal_weights(kind, goal_dim, seed=H + goal_dim, hidden_dim=H, relu_bias=3.0,
                     **({} if pool_to_input else dict(out_dim=H, pool_to_input=False)))
    cfg = _cfg(kind, H, None if pool_to_input else H)
    model = _goal_model(kind, H, W, goal_dim, pool_to_input).cuda().eval()
    obs1, obs2, bs = _step_scenes(seed=H + 7)
    goals = _step_goals(obs2, seed=H)
    h, c = _state(obs2.shape[0], H, seed=H + 1)
    P = model.encoder.weight_ih.shape[1] - 64 - goal_dim
    tc_gates = tc and pool_to_input and H % 64 == 0 and P % 64 == 0 and (64 + goal_dim) % 64 == 0
    gate_kernel = "lstm_gates_tc" if tc_gates else "lstm_gates"
    for phase in PHASES:
        got, kernels = _gpu_goal_step(model, phase, obs1, obs2, goals, bs, h, c)
        assert gate_kernel in kernels and ({"lstm_gates", "lstm_gates_tc"} - {gate_kernel}).isdisjoint(kernels), sorted(kernels)
        # the grid pools' pool_prepare writes the [emb | goal_emb] operand itself; the other models launch embed_split
        grid = getattr(cfg, "type_", None) in ("occupancy", "directional", "social")
        assert ("embed_split" in kernels) == (tc_gates and not grid), sorted(kernels)
        with torch.no_grad():
            ref = goal_step(_w64(W), cfg, phase, torch.from_numpy(h).to(F64), torch.from_numpy(c).to(F64),
                            torch.from_numpy(obs1), torch.from_numpy(obs2), torch.from_numpy(goals), bs, H, F64,
                            pool_to_input, True, TR.pool_state_zeros(cfg, obs2.shape[0], F64))
        gate = STEP_GATE[bool(tc and kernels & BF16_KERNELS)]
        for name, g, r in zip(("h", "c", "normal"), got, ref):
            assert _nan_rel(g, r.numpy()) <= gate, (kind, H, goal_dim, tc, phase, name, _nan_rel(g, r.numpy()))


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("goal_dim", [64, 32])
@pytest.mark.parametrize("H", [32, 128, 256])
@pytest.mark.parametrize("kind", STEP_KINDS)
def test_goal_step_matches_float64(monkeypatch, kind, H, goal_dim, tc):
    _set_tc(monkeypatch, tc)
    _check_goal_step(kind, H, goal_dim, tc)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", ["occupancy", "social_default", "hiddenstatemlp", "nn_lstm"])
def test_goal_step_pool_added_to_h(monkeypatch, kind, tc):
    _set_tc(monkeypatch, tc)
    _check_goal_step(kind, 128, 64, tc, pool_to_input=False)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("layout", ["padded", "per_scene"])
@pytest.mark.parametrize("case,kind,goal_dim,seed", CASES, ids=[c[0] for c in CASES])
def test_goal_forward_matches_float64(monkeypatch, case, kind, goal_dim, seed, layout, tc):
    """Whole forwards, free-running and teacher-forced, with test_step_forward's position tolerances."""
    _set_tc(monkeypatch, tc)
    W = goal_weights(kind, goal_dim, seed)
    model = _goal_model(kind, 128, W, goal_dim).cuda().eval()
    xy, bs, goals = goal_inputs()
    padded = layout == "padded"
    obs, g, split = torch.from_numpy(xy[:9]), torch.from_numpy(goals), torch.from_numpy(bs)
    truth = torch.from_numpy(xy[9:20]).clone()
    with torch.no_grad():
        if padded:
            _, pred_f = model(obs, g, split, n_predict=12)
            _, pred_t = model(obs, g, split, prediction_truth=truth)
        else:
            _, pred_f = model._forward_nograd(obs, split, None, 12, pad_to_batch_max=False, goals=g)
            _, pred_t = model._forward_nograd(obs, split, truth, None, pad_to_batch_max=False, goals=g)
    cfg, W64 = _case_cfg(kind), _w64(W)
    with torch.no_grad():
        _, ref_f = goal_forward(W64, cfg, obs, g, bs, 128, n_predict=12, pad_to_batch_max=padded)
        _, ref_t = goal_forward(W64, cfg, obs, g, bs, 128, prediction_truth=truth, pad_to_batch_max=padded)
    tol = (3e-4 if kind.split("_")[0] in NONGRID else 1e-4) if tc else 2e-5
    for got, ref in ((pred_f, ref_f), (pred_t, ref_t)):
        got = got.cpu().numpy()
        assert (np.isnan(got) == np.isnan(ref)).all()
        assert float(np.nanmax(np.abs(got - ref))) <= tol, (case, layout, tc, float(np.nanmax(np.abs(got - ref))))


@pytest.mark.gpu
def test_goal_calls_without_goals_are_refused():
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import _ptr
    lib = _lib.load()
    model = _goal_model("vanilla", 128, goal_weights("vanilla", 64, 1), 64).cuda().eval()
    handle = model._engine()
    xy, bs, goals = goal_inputs()
    layout = model._layouts.get(bs, device=handle.device)
    ws, need = handle.workspace(layout)
    M = layout.num_tracks
    f32 = dict(dtype=torch.float32, device="cuda")
    obs = torch.from_numpy(xy[:9]).cuda()
    normals, positions = torch.empty((19, M, 5), **f32), torch.empty((19, M, 2), **f32)
    h, c = torch.empty((M, 128), **f32), torch.empty((M, 128), **f32)
    normal = torch.empty((M, 5), **f32)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.tb2_lstm_step_forward(handle.handle, layout.handle, 0, _ptr(obs[0]), _ptr(obs[1]), None, None, _ptr(h),
                                     _ptr(c), _ptr(h), _ptr(c), _ptr(normal), None, _ptr(ws), need, stream) == -1
    assert b"goals_dev" in lib.tb2_last_error()
    assert lib.tb2_lstm_forward_steps(handle.handle, layout.handle, _ptr(obs), 9, None, 11, None, None, 0, 19,
                                      _ptr(normals), _ptr(positions), _ptr(h), _ptr(c), None, None, 0, None, None, None,
                                      _ptr(ws), need, stream) == -1
    host_n, host_p = torch.empty((19, M, 5), pin_memory=True), torch.empty((19, M, 2), pin_memory=True)
    side = torch.cuda.Stream()
    assert lib.tb2_lstm_forward_steps(handle.handle, layout.handle, _ptr(obs), 9, None, 11, None, None, 0, 19,
                                      _ptr(normals), _ptr(positions), _ptr(h), _ptr(c), None, None, 0, _ptr(host_n),
                                      _ptr(host_p), ctypes.c_void_p(side.cuda_stream), _ptr(ws), need, stream) == -1
    with pytest.raises(ValueError, match="needs the goals"):
        with torch.no_grad():
            model(obs.cpu(), None, torch.from_numpy(bs), n_predict=12)


@pytest.mark.gpu
def test_device_scene_transform_of_goals_is_the_host_one():
    from trajnetplusplusbaselines_b200.lstm.lstm import center_scene
    from trajnetplusplusbaselines_b200.lstm.scene_ops import preprocess_scenes
    xy, bs, goals = goal_inputs()
    scenes = [xy[:, bs[i]:bs[i + 1]].astype(np.float64) for i in range(len(bs) - 1)]
    goals64 = goals.astype(np.float64) * 1.37
    out = preprocess_scenes([s[:9] for s in scenes], device="cuda", normalize_scene=True, goals=goals64)
    got = out[5].cpu().numpy()
    for i, s in enumerate(scenes):
        _, _, _, g = center_scene(s[:9].copy(), 9, goals=goals64[bs[i]:bs[i + 1]])
        assert np.array_equal(got[bs[i]:bs[i + 1]], torch.Tensor(g).numpy())        # bit for bit, like the positions


@pytest.mark.gpu
@pytest.mark.needs_reference
@pytest.mark.parametrize("kind,goal_dim", [("directional", 64), ("vanilla", 32)])
def test_reference_goal_predictor_drops_in(tmp_path, kind, goal_dim):
    """A goal predictor the reference pickled: the pickle names the reference's classes, so, as for the other reference
    checkpoints (INTEGRATION.md: checkpoints interchange through the state_dict), its model's state_dict and goal_dim
    build this package's LSTM(goal_flag=True); both predictors then predict the same scenes of a shipped data file."""
    from oracle.make_goal_golden import build_reference_model
    from oracle.ref_shim import import_reference
    import_reference()
    from trajnetbaselines.lstm import trajnet_evaluator as ref_eval
    from trajnetbaselines.lstm.lstm import LSTMPredictor as RefPredictor
    from trajnetplusplusbaselines_b200.data import read_ndjson_scenes, preprocess_test
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    W = goal_weights(kind, goal_dim, seed=9)
    ref_model = build_reference_model(kind, goal_dim, W)
    RefPredictor(ref_model).save({"state_dict": ref_model.state_dict()}, str(tmp_path / "ref.pkl"))
    with open(tmp_path / "ref.pkl", "rb") as f:
        saved = torch.load(f, weights_only=False)          # the reference pickles the whole predictor
    assert saved.model.goal_flag and saved.model.goal_dim == goal_dim
    from trajnetplusplusbaselines_b200.lstm import LSTM
    table, spec = model_kwargs(kind)
    model = LSTM(pool=_pool_module(kind, 128) if spec is not None else None, goal_flag=True, goal_dim=saved.model.goal_dim)
    model.load_state_dict(saved.model.state_dict(), strict=True)
    predictor = LSTMPredictor(model.cuda())
    from oracle.ref_shim import reference_root
    data = os.path.join(reference_root(), "DATA_BLOCK", "trajdata", "train", "biwi_hotel.ndjson")
    scenes = list(read_ndjson_scenes(data))[:6]
    last = {}
    for _, paths in read_ndjson_scenes(data):
        for p in paths:
            last[p[0].pedestrian] = (p[-1].x, p[-1].y)        # every pedestrian's last position in the file
    for normalize in (False, True):
        args = argparse.Namespace(obs_length=9, pred_length=12, modes=1, normalize_scene=normalize)
        for _, paths in scenes:
            paths = preprocess_test(paths, 9)
            goal = np.array([last[p[0].pedestrian] for p in paths])
            out_ref = ref_eval.predict_scene(RefPredictor(saved.model), "m", paths, goal, args)
            out = ref_eval.predict_scene(predictor, "m", paths, goal, args)
            assert np.abs(out[0][0] - out_ref[0][0]).max() < 1e-4
            if len(paths) > 1:
                assert np.nanmax(np.abs(out[0][1] - out_ref[0][1])) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("normalize", [False, True], ids=["raw", "normalize_scene"])
def test_goal_files_through_both_pipelines_byte_identical(tmp_path, monkeypatch, normalize):
    from trajnetplusplusbaselines_b200 import evaluator
    from trajnetplusplusbaselines_b200.data import load_goal_file
    from trajnetplusplusbaselines_b200.lstm import LSTMPredictor
    infile = _dataset(str(tmp_path), [5, 3, 6, 4, 7], seed=5)
    goals = load_goal_file(str(tmp_path / "goal_files" / "test_private" / "data.pkl"))
    model = _goal_model("directional", 128, goal_weights("directional", 64, seed=5), 64).cuda().eval()
    predictor = LSTMPredictor(model)
    args = argparse.Namespace(normalize_scene=normalize)
    cols, rows = str(tmp_path / "cols.ndjson"), str(tmp_path / "rows.ndjson")
    evaluator.evaluate_file(predictor, infile, cols, chunk=2, args=args, goals=goals)

    class PerScene:            # the row pipeline, scene by scene through LSTMPredictor.__call__
        def __init__(self, p):
            self.model = p.model
            self.p = p

        def __call__(self, *a, **kw):
            return self.p(*a, **kw)
    evaluator.evaluate_file(PerScene(predictor), infile, rows, args=args, goals=goals)
    batched_rows = str(tmp_path / "batched_rows.ndjson")
    scenes = evaluator.load_test_scenes(infile)
    scene_goals = [np.array([goals[p[0].pedestrian] for p in paths]) for _, _, paths in scenes]
    evaluator.write_predictions(evaluator.predict_scenes(predictor, scenes, chunk=3, args=args, goals=scene_goals),
                                scenes, batched_rows)
    with open(cols, "rb") as a, open(rows, "rb") as b, open(batched_rows, "rb") as c:
        ca, cb, cc = a.read(), b.read(), c.read()
    assert len(ca) > 1000 and ca == cb == cc
    # the goals change the predictions
    plain = str(tmp_path / "zero_goals.ndjson")
    zero = {k: (0.0, 0.0) for k in goals}
    evaluator.evaluate_file(predictor, infile, plain, args=args, goals=zero)
    with open(plain, "rb") as f:
        assert f.read() != ca
