"""Every mode of every scene in one batched decode (trajnetplusplusbaselines_b200/multimodal.py): SGANPredictor /
VAEPredictor.predict_batch_xy against the per-scene __call__ fed the same random vectors, the decoder-context kernels
(tb2_sgan_decoder_context / tb2_vae_decoder_context) against the per-mode kernels on a copy of the state, and the
evaluator's routing: S-GAN / VAE through the column pipeline at any `modes`, byte-identical files."""
import os
import socket
import types

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import lstm_oracle as O
from oracle import sgan_oracle as SO
from oracle.make_sgan_golden import SGAN_CASES
from oracle.make_vae_golden import VAE_CASES
from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, paths_to_xy, trajnet_line

PLAIN = types.SimpleNamespace(normalize_scene=False)
NORMALIZED = types.SimpleNamespace(normalize_scene=True)
SIZES = (1, 5, 60, 2, 13, 7, 30, 3)        # tracks per scene: a lone primary up to a crowd
WSEED = {c[1]: c[7] for c in SGAN_CASES}     # weight seeds of the golden fixtures
VSEED = {c[1]: c[7] for c in VAE_CASES}


# ------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------
def _scenes(sizes, seed, n_frames=9):
    """float64 [n_frames, N, 2] random walks; about one neighbour in five enters during the observation and one in
    seven leaves before its end (NaN rows), the primary is always present."""
    rng = np.random.RandomState(seed)
    xys = []
    for n in sizes:
        xy = rng.randn(n, 2)[None] * 2.0 + np.cumsum(rng.randn(n_frames, n, 2) * 0.3, axis=0)
        for p in range(1, n):
            u = rng.rand()
            if u < 0.2:
                xy[:rng.randint(1, n_frames - 1), p] = np.nan
            elif u < 0.35:
                xy[rng.randint(2, n_frames - 1):, p] = np.nan
        xys.append(xy)
    return xys


def _paths(xy):
    paths = [[TrackRow(10 * t, 100 + p, float(xy[t, p, 0]), float(xy[t, p, 1])) for t in range(xy.shape[0])
              if not np.isnan(xy[t, p, 0])] for p in range(xy.shape[1])]
    assert np.array_equal(paths_to_xy(paths), xy, equal_nan=True)
    return paths


def _pool(kind):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling, HiddenStateMLPPooling, NearestNeighborLSTM
    if kind in O.NONGRID_SPECS:
        return HiddenStateMLPPooling(**O.NONGRID_SPECS[kind])
    if kind in O.NN_LSTM_SPECS:
        return NearestNeighborLSTM(**O.NN_LSTM_SPECS[kind])
    spec = O.MODEL_SPECS[kind]
    return GridBasedPooling(**spec) if spec else None


def _load(module, W):
    sd = module.state_dict()
    sd.update({k: torch.from_numpy(v.copy()) for k, v in W.items() if k in sd})
    module.load_state_dict(sd)


def _sgan(kind, seed, no_noise=False, device="cuda"):
    from trajnetplusplusbaselines_b200.sgan import SGAN, LSTMGenerator, SGANPredictor
    gen = LSTMGenerator(pool=_pool(kind), no_noise=no_noise)
    _load(gen, SO.sgan_weights(kind, seed)[0])
    return SGANPredictor(SGAN(generator=gen, k=1, d_steps=0).to(device).eval())


def _vae(kind, seed):
    from trajnetplusplusbaselines_b200.vae import VAE, VAEPredictor
    model = VAE(pool=_pool(kind))
    _load(model, SO.vae_weights(kind, seed))
    return VAEPredictor(model.cuda().eval())


def _sgan_singles(predictor, xys, noise, modes, args):
    """The per-scene __call__ of every scene, decode q of scene b drawing noise[q, b]."""
    gen = predictor.model.generator
    outs = []
    try:
        for b, xy in enumerate(xys):
            draws = iter([torch.from_numpy(noise[q, b].copy()) for q in range(modes)])
            gen._draw_noise = lambda device, it=draws: next(it).to(device).contiguous()
            outs.append(predictor(_paths(xy), np.zeros((xy.shape[1], 2)), n_predict=12, modes=modes, obs_length=9,
                                  args=args))
            assert next(draws, None) is None
    finally:
        gen.__dict__.pop('_draw_noise', None)
    return outs


def _vae_singles(predictor, xys, z, modes, args):
    """The per-scene __call__ of every scene with the latent samples z[:, tracks of the scene]."""
    outs, lo = [], 0
    try:
        for xy in xys:
            hi = lo + xy.shape[1]
            predictor.model.fixed_z = torch.from_numpy(z[:, lo:hi].copy())
            outs.append(predictor(_paths(xy), np.zeros((xy.shape[1], 2)), n_predict=12, modes=modes, obs_length=9,
                                  args=args))
            lo = hi
    finally:
        predictor.model.fixed_z = None
    return outs


def _assert_same(singles, batched, modes):
    assert len(singles) == len(batched)
    for i, (s, b) in enumerate(zip(singles, batched)):
        assert sorted(s) == sorted(b) == list(range(modes))
        for q in range(modes):
            assert s[q][0].dtype == b[q][0].dtype and s[q][0].shape == b[q][0].shape == (12, 2)
            assert np.array_equal(s[q][0], b[q][0], equal_nan=True), (i, q)
        assert s[0][1].shape == b[0][1].shape and np.array_equal(s[0][1], b[0][1], equal_nan=True), i
        for q in range(1, modes):
            assert len(s[q][1]) == 0 and len(b[q][1]) == 0


# ------------------------------------------------------------------------------------------------------------------
# GPU: batched == per scene, bit for bit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalized"])
@pytest.mark.parametrize("kind", ["vanilla", "directional", "social", "social_small", "hiddenstatemlp"])
def test_sgan_batched_equals_per_scene(kind, normalize):
    predictor = _sgan(kind, WSEED.get(kind, 7))
    args = NORMALIZED if normalize else PLAIN
    xys = _scenes(SIZES, seed=len(kind))
    rng = np.random.RandomState(5)
    for modes in (1, 3, 20):
        noise = rng.standard_normal((modes, len(xys), 8)).astype(np.float32)
        batched = predictor.predict_batch_xy(xys, n_predict=12, obs_length=9, args=args, modes=modes, noise=noise)
        _assert_same(_sgan_singles(predictor, xys, noise, modes, args), batched, modes)


@pytest.mark.gpu
def test_sgan_no_noise_and_fixed_noise_batched_equal_per_scene():
    """no_noise (the golden fixture's case): the decoder starts from the encoder state; fixed_noise: every (scene, mode)
    decodes with that vector."""
    xys = _scenes((4, 1, 9), seed=3)
    predictor = _sgan("vanilla", 4, no_noise=True)
    singles = [predictor(_paths(xy), np.zeros((xy.shape[1], 2)), n_predict=12, modes=3, args=PLAIN) for xy in xys]
    _assert_same(singles, predictor.predict_batch_xy(xys, args=PLAIN, modes=3), 3)
    predictor = _sgan("directional", 2)
    predictor.model.generator.fixed_noise = torch.linspace(-1.0, 1.0, 8)
    singles = [predictor(_paths(xy), np.zeros((xy.shape[1], 2)), n_predict=12, modes=3, args=PLAIN) for xy in xys]
    _assert_same(singles, predictor.predict_batch_xy(xys, args=PLAIN, modes=3), 3)


@pytest.mark.gpu
@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalized"])
@pytest.mark.parametrize("kind", ["vanilla", "directional", "social", "social_small", "hiddenstatemlp"])
def test_vae_batched_equals_per_scene(kind, normalize):
    predictor = _vae(kind, VSEED.get(kind, 9))
    args = NORMALIZED if normalize else PLAIN
    xys = _scenes(SIZES, seed=10 + len(kind))
    M = sum(xy.shape[1] for xy in xys)
    rng = np.random.RandomState(6)
    for modes in (1, 3, 20):
        z = (rng.standard_normal((modes, M, 128)) * 1.6).astype(np.float32)
        batched = predictor.predict_batch_xy(xys, n_predict=12, obs_length=9, args=args, modes=modes, z=z)
        _assert_same(_vae_singles(predictor, xys, z, modes, args), batched, modes)
        predictor.model.fixed_z = torch.from_numpy(z)           # the model's fixed_z is the same hook
        again = predictor.predict_batch_xy(xys, n_predict=12, obs_length=9, args=args, modes=modes)
        predictor.model.fixed_z = None
        _assert_same(batched, again, modes)


@pytest.mark.gpu
def test_start_length_and_short_horizons_equal_per_scene():
    """The VAE observes xy[start_length:obs_length], the generator xy[:obs_length] (as their __call__ do); n_predict 1
    (no decoder step) and obs_length 2."""
    xys = _scenes((3, 6, 1), seed=21)
    vae = _vae("directional", 2)
    M = sum(xy.shape[1] for xy in xys)
    z = np.random.RandomState(1).standard_normal((3, M, 128)).astype(np.float32)
    for kw in (dict(start_length=2), dict(obs_length=2), dict(n_predict=1)):
        n_predict = kw.get("n_predict", 12)
        batched = vae.predict_batch_xy(xys, args=PLAIN, modes=3, z=z, **kw)
        lo = 0
        for xy, b in zip(xys, batched):
            hi = lo + xy.shape[1]
            vae.model.fixed_z = torch.from_numpy(z[:, lo:hi].copy())
            s = vae(_paths(xy), np.zeros((xy.shape[1], 2)), modes=3, args=PLAIN, **kw)
            vae.model.fixed_z = None
            for q in range(3):
                assert s[q][0].shape == (n_predict, 2) and np.array_equal(s[q][0], b[q][0], equal_nan=True), (kw, q)
            assert np.array_equal(s[0][1], b[0][1], equal_nan=True)
            lo = hi
    sgan = _sgan("social_small", 3)
    noise = np.random.RandomState(2).standard_normal((3, len(xys), 8)).astype(np.float32)
    for kw in (dict(start_length=2), dict(obs_length=2), dict(n_predict=1)):
        batched = sgan.predict_batch_xy(xys, args=PLAIN, modes=3, noise=noise, **kw)
        gen = sgan.model.generator
        for b, (xy, got) in enumerate(zip(xys, batched)):
            draws = iter([torch.from_numpy(noise[q, b].copy()) for q in range(3)])
            gen._draw_noise = lambda device, it=draws: next(it).to(device)
            s = sgan(_paths(xy), np.zeros((xy.shape[1], 2)), modes=3, args=PLAIN, **kw)
            gen.__dict__.pop('_draw_noise')
            for q in range(3):
                assert np.array_equal(s[q][0], got[q][0], equal_nan=True), (kw, q)
            assert np.array_equal(s[0][1], got[0][1], equal_nan=True)


# ------------------------------------------------------------------------------------------------------------------
# GPU: mode groups, random draws
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("model", ["sgan", "vae"])
def test_mode_grouping_is_invisible(model):
    """A row cap below k * M splits the modes into groups; the draws are made before the split, so the same seed gives
    the same arrays whatever the grouping."""
    predictor = _sgan("social", 7) if model == "sgan" else _vae("directional", 2)
    xys = _scenes((4, 11, 1, 6), seed=8)
    M = sum(xy.shape[1] for xy in xys)
    outs = []
    for max_rows in (None, 1, 2 * M, 3 * M + 5):              # one group; a mode per group; two; three per group
        torch.manual_seed(123)
        outs.append(predictor.predict_batch_xy(xys, args=NORMALIZED, modes=7, max_rows=max_rows))
    for other in outs[1:]:
        _assert_same(outs[0], other, 7)


@pytest.mark.gpu
def test_rows_per_decode_splits_large_chunks():
    """The default cap comes from the engine's workspace: a few rows per MB, far below the rows of 1024 scenes x 20
    tracks x 50 modes."""
    from trajnetplusplusbaselines_b200 import multimodal
    predictor = _sgan("social", 7)
    gen = predictor.model.generator
    split = np.arange(0, 20 * 1024 + 1, 20)
    layout = gen._layouts.get(split.tolist(), False, device=gen._device())
    cap = multimodal.rows_per_decode(gen._engine(), layout, 19, 9)
    assert 20 * 1024 <= cap < 50 * 20 * 1024


@pytest.mark.gpu
def test_draws_are_per_scene_and_mode():
    xy = _scenes((6,), seed=4)[0]
    for noise_type in ("gaussian", "uniform"):
        predictor = _sgan("directional", 2)
        predictor.model.generator.noise_type = noise_type
        torch.manual_seed(0)
        out = predictor.predict_batch_xy([xy, xy], args=PLAIN, modes=3)
        assert np.abs(out[0][0][0] - out[0][1][0]).max() > 1e-4          # two modes of one scene
        assert np.abs(out[0][0][0] - out[1][0][0]).max() > 1e-4          # two scenes of one mode
        assert np.abs(out[0][1][0] - out[1][2][0]).max() > 1e-4
    predictor.model.generator.no_noise = True
    out = predictor.predict_batch_xy([xy, xy], args=PLAIN, modes=3)
    for b in range(2):
        for q in range(3):
            assert np.array_equal(out[b][q][0], out[0][0][0])
    vae = _vae("vanilla", 1)
    torch.manual_seed(0)
    out = vae.predict_batch_xy([xy, xy], args=PLAIN, modes=3)
    assert np.abs(out[0][0][0] - out[0][1][0]).max() > 1e-4
    assert np.abs(out[0][0][0] - out[1][0][0]).max() > 1e-4
    torch.manual_seed(0)
    again = vae.predict_batch_xy([xy, xy], args=PLAIN, modes=3)
    _assert_same(out, again, 3)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ------------------------------------------------------------------------------------------------------------------
def _call(name, *args):
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import _ptr, _stream
    conv = [_ptr(a) if torch.is_tensor(a) or a is None else int(a) for a in args]
    return getattr(_lib.load(), name)(*conv, _stream(torch.device("cuda", torch.cuda.current_device())))


@pytest.mark.gpu
@pytest.mark.parametrize("H,nd", [(128, 8), (37, 6), (40, 7), (5, 0)])
def test_sgan_decoder_context_equals_add_noise_on_a_clone(H, nd):
    g = torch.Generator(device="cuda").manual_seed(H + nd)
    split = [0, 3, 4, 9, 13]
    M, B, k = split[-1], len(split) - 1, 5
    cuda = dict(device="cuda", dtype=torch.float32)
    W = torch.randn((H - nd, H), generator=g, **cuda) / np.sqrt(H)
    bias = torch.randn(H - nd, generator=g, **cuda) * 0.1
    h_enc, c_enc = torch.randn((M, H), generator=g, **cuda), torch.randn((M, H), generator=g, **cuda)
    noise = torch.randn((k, B, max(nd, 1)), generator=g, **cuda)[:, :, :nd].contiguous()
    groups = torch.tensor(np.repeat(np.arange(B), np.diff(split)), dtype=torch.int32, device="cuda")
    h_out, c_out = torch.full((k * M, H), np.nan, **cuda), torch.full((k * M, H), np.nan, **cuda)
    assert _call("tb2_sgan_decoder_context", W, bias, noise, groups, B, h_enc, c_enc, M, H, nd, k, h_out, c_out) == 0
    for q in range(k):
        for b in range(B):
            lo, hi = split[b], split[b + 1]
            h = h_enc[lo:hi].clone()
            assert _call("tb2_sgan_add_noise", W, bias, noise[q, b].contiguous(), h, hi - lo, H, nd) == 0
            assert torch.equal(h_out[q * M + lo:q * M + hi], h), (q, b)
        assert torch.equal(c_out[q * M:(q + 1) * M], c_enc)
    assert _call("tb2_sgan_decoder_context", W, bias, noise, groups, B, h_enc, c_enc, M, H, nd, 0, h_out, c_out) != 0
    assert _call("tb2_sgan_decoder_context", W, bias, noise, groups, B, h_enc, c_enc, M, H, H, k, h_out, c_out) != 0


@pytest.mark.gpu
@pytest.mark.parametrize("H,L", [(128, 128), (45, 37), (128, 3), (7, 130)])
def test_vae_decoder_context_equals_scale_hidden_on_a_clone(H, L):
    g = torch.Generator(device="cuda").manual_seed(H * L)
    M, k = 11, 4
    cuda = dict(device="cuda", dtype=torch.float32)
    W = torch.rand((H, L), generator=g, **cuda) / np.sqrt(L) - 0.02
    bias = torch.randn(H, generator=g, **cuda) * 0.1
    h_enc, c_enc = torch.randn((M, H), generator=g, **cuda), torch.randn((M, H), generator=g, **cuda)
    z = torch.randn((k * M, L), generator=g, **cuda)
    h_out, c_out = torch.full((k * M, H), np.nan, **cuda), torch.full((k * M, H), np.nan, **cuda)
    assert _call("tb2_vae_decoder_context", W, bias, z, h_enc, c_enc, M, H, L, k, h_out, c_out) == 0
    for q in range(k):
        h = h_enc.clone()
        assert _call("tb2_vae_scale_hidden", W, bias, z[q * M:(q + 1) * M].contiguous(), h, M, H, L) == 0
        assert torch.equal(h_out[q * M:(q + 1) * M], h), q
        assert torch.equal(c_out[q * M:(q + 1) * M], c_enc)
    assert _call("tb2_vae_decoder_context", W, bias, z, h_enc, c_enc, M, H, L, 0, h_out, c_out) != 0
    assert _call("tb2_vae_decoder_context", W, bias, None, h_enc, c_enc, M, H, L, k, h_out, c_out) != 0


# ------------------------------------------------------------------------------------------------------------------
# GPU: end to end through the evaluator
# ------------------------------------------------------------------------------------------------------------------
class _Rows:
    """Hides predict_batch_xy: the evaluator takes the row pipeline (one __call__ per scene)."""

    def __init__(self, predictor):
        self.predictor = predictor

    def __call__(self, *args, **kwargs):
        return self.predictor(*args, **kwargs)


def _injected_files(predictor, infile, cols, rows, modes, seed):
    """evaluate_file through the column pipeline into `cols` and through the row pipeline into `rows`, with the same
    per-(mode, scene) noise."""
    from trajnetplusplusbaselines_b200.data import load_test_scenes_xy
    from trajnetplusplusbaselines_b200.evaluator import _column_pipeline, evaluate_file
    B = len(load_test_scenes_xy(infile))
    noise = np.random.RandomState(seed).standard_normal((modes, B, 8)).astype(np.float32)
    plain = predictor.predict_batch_xy
    predictor.predict_batch_xy = lambda xys, modes=1, **kw: plain(xys, modes=modes, noise=noise, **kw)
    try:
        assert _column_pipeline(predictor, modes)
        assert evaluate_file(predictor, infile, cols, modes=modes, chunk=B, args=PLAIN) == B
    finally:
        del predictor.predict_batch_xy
    gen = predictor.model.generator
    draws = iter([torch.from_numpy(noise[q, b].copy()) for b in range(B) for q in range(modes)])
    gen._draw_noise = lambda device: next(draws).to(device)
    try:
        assert not _column_pipeline(_Rows(predictor), modes)
        assert evaluate_file(_Rows(predictor), infile, rows, modes=modes, args=PLAIN) == B
    finally:
        gen.__dict__.pop('_draw_noise')
    assert open(cols, "rb").read() == open(rows, "rb").read()


@pytest.mark.gpu
@pytest.mark.needs_reference
def test_evaluate_file_collision_test_modes3_byte_identical(tmp_path):
    """The reference's collision test scene (its ground truth holds the observation only: the evaluator runs the
    Pass / Fail collision test on it)."""
    from oracle.ref_shim import reference_root
    from trajnetplusplusbaselines_b200.scoring import collision_test
    infile = os.path.join(reference_root(), "DATA_BLOCK", "collision_test", "test", "collision_test.ndjson")
    os.makedirs(str(tmp_path / "cols"))
    cols = str(tmp_path / "cols" / "collision_test.ndjson")
    _injected_files(_sgan("social_small", 3), infile, cols, str(tmp_path / "rows.ndjson"), 3, seed=11)
    text = open(cols).read()
    assert '"prediction_number": 2' in text
    args = types.SimpleNamespace(path=str(tmp_path), pred_length=12)
    assert collision_test(["collision_test.ndjson"], "cols", args) in ("Pass", "Fail")


@pytest.mark.gpu
def test_evaluate_file_synthetic_modes3_byte_identical_and_scored(tmp_path):
    """Scenes with late / leaving neighbours through both pipelines of evaluate_file; the file scores with the Top-3
    columns against the full scenes."""
    from trajnetplusplusbaselines_b200.scoring import score_file
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 8, 2, 25, 4], seed=2)
    cols = str(tmp_path / "cols.ndjson")
    _injected_files(_sgan("directional", 2), infile, cols, str(tmp_path / "rows.ndjson"), 3, seed=12)
    metrics, _, _ = score_file(infile, cols)
    assert metrics.N == 6
    assert np.isfinite(metrics.topk_ade) and 0 < metrics.topk_ade <= metrics.average_l2
    assert np.isfinite(metrics.topk_fde) and 0 < metrics.topk_fde <= metrics.final_l2


# ------------------------------------------------------------------------------------------------------------------
# CPU: routing of the evaluator, byte-identical files at modes 3, sharded over gloo
# ------------------------------------------------------------------------------------------------------------------
def _write_scenes(filename, sizes, seed):
    rng = np.random.RandomState(seed)
    with open(filename, "w") as f:
        for sid, n in enumerate(sizes):
            frames = [1000 * sid + 10 * t for t in range(21)]
            start, vel = rng.randn(n, 2) * 3.0, rng.randn(n, 2) * 0.2
            f.write(trajnet_line(SceneRow(sid, 100 * sid, frames[0], frames[-1], 2.5, 1 + sid % 4)) + "\n")
            for p in range(n):
                t0, t1 = (0, 21) if p == 0 else [(0, 21), (3, 21), (0, 6), (12, 21)][p % 4]    # late, leaving, after obs
                for t in range(t0, t1):
                    f.write(trajnet_line(TrackRow(frames[t], 100 * sid + p, start[p, 0] + vel[p, 0] * t,
                                                  start[p, 1] + vel[p, 1] * t)) + "\n")


def _cv_modes(xy, n_predict, obs_length, modes):
    v = xy[obs_length - 1] - xy[obs_length - 2]
    out = {}
    for q in range(modes):
        pred = xy[obs_length - 1][None] + np.arange(1, n_predict + 1)[:, None, None] * v[None] * (1.0 + 0.37 * q)
        out[q] = [pred[:, 0], pred[:, 1:] if q == 0 else []]
    return out


class _ModesConstantVelocity:
    """Stand-in with the reference's predictor call signature (CPU): mode q moves 1 + 0.37 q times as fast."""

    def __call__(self, paths, scene_goal, n_predict=12, modes=1, predict_all=True, obs_length=9, start_length=0,
                 args=None):
        return _cv_modes(paths_to_xy(paths), n_predict, obs_length, modes)


class _ArrayModesConstantVelocity(_ModesConstantVelocity):
    """The same with the array entry point that takes `modes`: evaluate_file takes the column pipeline at any modes."""

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None, modes=1):
        return [_cv_modes(xy, n_predict, obs_length, modes) for xy in xys]


class _ArrayOneMode(_ModesConstantVelocity):
    """predict_batch_xy without `modes` (like LSTMPredictor): the column pipeline at modes 1 only."""

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None):
        return [_cv_modes(xy, n_predict, obs_length, 1) for xy in xys]


def test_routing_of_the_evaluator():
    from trajnetplusplusbaselines_b200.evaluator import _column_pipeline, batches_modes
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor
    for modes in (1, 3, 50):
        assert _column_pipeline(_ArrayModesConstantVelocity(), modes)
        assert not _column_pipeline(_ModesConstantVelocity(), modes)
        assert _column_pipeline(_ArrayOneMode(), modes) == (modes == 1)
        assert _column_pipeline(LSTMPredictor(LSTM()), modes) == (modes == 1)
        assert not batches_modes(LSTMPredictor(LSTM()))
    sgan = _sgan("vanilla", 1, device="cpu")
    assert batches_modes(sgan) and _column_pipeline(sgan, 3) and _column_pipeline(sgan, 1)
    # an interaction module with its own LSTM state is not replicated per mode: the row pipeline keeps it
    stateful = _sgan("nn_lstm", 1, device="cpu")
    assert not stateful.batch_decode_supported()
    assert not _column_pipeline(stateful, 3) and not _column_pipeline(stateful, 1)
    with pytest.raises(NotImplementedError):
        stateful.predict_batch_xy(_scenes((3,), seed=0), modes=3)


def test_column_pipeline_modes3_writes_the_row_pipelines_file(tmp_path):
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file, load_test_scenes, predict_scenes
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 7, 2, 5, 4], seed=4)
    rows, cols = str(tmp_path / "rows.ndjson"), str(tmp_path / "cols.ndjson")
    assert evaluate_file(_ModesConstantVelocity(), infile, rows, modes=3) == 6
    assert evaluate_file(_ArrayModesConstantVelocity(), infile, cols, modes=3, chunk=4) == 6
    text = open(rows, "rb").read()
    assert text == open(cols, "rb").read()
    assert b'"prediction_number": 2' in text
    # predict_scenes (the row loader) batches such a predictor too, with the same predictions
    scenes = load_test_scenes(infile)
    got = predict_scenes(_ArrayModesConstantVelocity(), scenes, modes=3, chunk=4)
    want = predict_scenes(_ModesConstantVelocity(), scenes, modes=3)
    for g, w in zip(got, want):
        assert sorted(g) == sorted(w) == [0, 1, 2]
        for q in range(3):
            assert np.array_equal(g[q][0], w[q][0])
            assert np.array_equal(np.asarray(g[q][1]), np.asarray(w[q][1]), equal_nan=True)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _eval_worker(rank, world, port, infile, outfile):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file
    assert evaluate_file(_ArrayModesConstantVelocity(), infile, outfile, modes=3, chunk=2) == 7
    assert os.path.exists(outfile) and not os.path.exists("%s.part%d" % (outfile, rank))
    dist.destroy_process_group()


def test_column_pipeline_modes3_sharded_world2_gloo(tmp_path):
    from trajnetplusplusbaselines_b200.evaluator import evaluate_file
    infile = str(tmp_path / "in.ndjson")
    _write_scenes(infile, [3, 1, 6, 2, 2, 9, 4], seed=5)
    single = str(tmp_path / "single.ndjson")
    assert evaluate_file(_ModesConstantVelocity(), infile, single, modes=3) == 7
    sharded = str(tmp_path / "sharded.ndjson")
    mp.spawn(_eval_worker, args=(2, _free_port(), infile, sharded), nprocs=2, join=True)
    assert open(sharded, "rb").read() == open(single, "rb").read()
