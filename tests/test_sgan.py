"""S-GAN generator / discriminator (SURVEY.md 8f rank 2) vs vectors the unmodified reference produced
with its noise source patched to a fixed vector (oracle/make_sgan_golden.py).
CPU: the numpy restatement (oracle/sgan_oracle.py); GPU: the package through the C ABI."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import lstm_oracle as O
from oracle import sgan_oracle as SO
from oracle.make_sgan_golden import NOISE, SGAN_CASES

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "sgan_golden.npz"))
IDS = [c[0] for c in SGAN_CASES]


def _inputs(case):
    name, kind, B, N, ragged, nan_tracks, dseed, wseed, no_noise = case
    xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
    Wg, Wd = SO.sgan_weights(kind, wseed)
    return name, kind, xy, bs, Wg, Wd, (None if no_noise else NOISE)


def _close(a, b, tol):
    assert (np.isnan(a) == np.isnan(b)).all()
    assert np.nanmax(np.abs(a - b)) < tol, float(np.nanmax(np.abs(a - b)))


@pytest.mark.parametrize("case", SGAN_CASES, ids=IDS)
def test_oracle_matches_reference(case):
    name, kind, xy, bs, Wg, Wd, noise = _inputs(case)
    cfg = O.pool_config(kind)
    rel, pred = SO.generator_forward(Wg, cfg, xy[:9], bs, n_predict=12, noise=noise)
    _close(rel, GOLD[name + "/rel"], 2e-5)
    _close(pred, GOLD[name + "/pred"], 2e-5)
    rel_tf, pred_tf = SO.generator_forward(Wg, cfg, xy[:9], bs, prediction_truth=xy[9:-1], noise=noise)
    _close(pred_tf, GOLD[name + "/pred_tf"], 2e-5)
    _close(SO.discriminator_forward(Wd, cfg, xy[:9], xy[9:21], bs), GOLD[name + "/scores_real"], 2e-5)
    _close(SO.discriminator_forward(Wd, cfg, xy[:9], GOLD[name + "/pred"][-12:], bs), GOLD[name + "/scores_fake"], 2e-5)


def test_state_dict_keys_are_the_references():
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling
    from trajnetplusplusbaselines_b200.sgan import LSTMDiscriminator, LSTMGenerator
    Wg, Wd = SO.sgan_weights("social_small", 3)
    spec = O.MODEL_SPECS["social_small"]
    gen = LSTMGenerator(pool=GridBasedPooling(**spec))
    dis = LSTMDiscriminator(pool=GridBasedPooling(**spec))
    strip = lambda sd: {k for k in sd if not k.startswith("goal_embedding.")}
    assert strip(gen.state_dict()) == strip(Wg)
    assert strip(dis.state_dict()) == strip(Wd)


def _models(kind, Wg, Wd, noise):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling
    from trajnetplusplusbaselines_b200.sgan import LSTMDiscriminator, LSTMGenerator
    spec = O.MODEL_SPECS[kind]
    gen = LSTMGenerator(pool=GridBasedPooling(**spec) if spec else None, no_noise=noise is None)
    dis = LSTMDiscriminator(pool=GridBasedPooling(**spec) if spec else None)
    for module, W in ((gen, Wg), (dis, Wd)):
        sd = module.state_dict()
        sd.update({k: torch.from_numpy(v.copy()) for k, v in W.items()})
        module.load_state_dict(sd)
    gen.fixed_noise = None if noise is None else torch.from_numpy(noise.copy())
    return gen.cuda().eval(), dis.cuda().eval()


@pytest.mark.gpu
@pytest.mark.parametrize("case", SGAN_CASES, ids=IDS)
def test_cuda_generator_and_discriminator_match_reference(case):
    name, kind, xy, bs, Wg, Wd, noise = _inputs(case)
    gen, dis = _models(kind, Wg, Wd, noise)
    scene, split = torch.from_numpy(xy), torch.from_numpy(bs)
    goals = torch.zeros(xy.shape[1], 2)
    with torch.no_grad():
        rel, pred = gen(scene[:9], goals, split, n_predict=12)
        rel, pred = rel.numpy().copy(), pred.numpy().copy()
        rel_tf, pred_tf = gen(scene[:9], goals, split, scene[9:-1].clone())
        pred_tf = pred_tf.numpy().copy()
        s_real = dis(scene[:9], scene[9:21], goals, split).numpy()
        s_fake = dis(scene[:9], torch.from_numpy(GOLD[name + "/pred"][-12:]), goals, split).numpy()
    _close(rel, GOLD[name + "/rel"], 1e-4)
    _close(pred, GOLD[name + "/pred"], 1e-4)            # the 1e-4 m gate of the LSTM path
    _close(pred_tf, GOLD[name + "/pred_tf"], 1e-4)
    _close(s_real, GOLD[name + "/scores_real"], 1e-4)
    _close(s_fake, GOLD[name + "/scores_fake"], 1e-4)


@pytest.mark.gpu
def test_sgan_modes_and_predictor():
    """k modes share one encoder pass; with a fixed noise vector all modes coincide with the golden
    run, with random noise they differ; SGANPredictor returns the reference's dictionary layout."""
    from trajnetplusplusbaselines_b200.data import TrackRow
    from trajnetplusplusbaselines_b200.sgan import SGAN, SGANPredictor
    name, kind, xy, bs, Wg, Wd, noise = _inputs(SGAN_CASES[1])
    gen, dis = _models(kind, Wg, Wd, noise)
    model = SGAN(generator=gen, discriminator=dis, k=3, d_steps=0)
    scene, split = torch.from_numpy(xy), torch.from_numpy(bs)
    with torch.no_grad():
        rel_list, pred_list, _, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), split, n_predict=12)
    assert len(pred_list) == 3
    for p in pred_list:
        _close(p.numpy(), GOLD[name + "/pred"], 1e-4)
    gen.fixed_noise = None
    torch.manual_seed(0)
    with torch.no_grad():
        _, pred_list, _, _ = model(scene[:9], torch.zeros(xy.shape[1], 2), split, n_predict=12)
    a, b = pred_list[0].numpy()[-12:, 0], pred_list[1].numpy()[-12:, 0]
    assert np.abs(a - b).max() > 1e-4                   # different noise, different futures
    assert np.abs(pred_list[0].numpy()[:8] - pred_list[1].numpy()[:8])[~np.isnan(pred_list[0].numpy()[:8])].max() == 0.0
    paths = [[TrackRow(10 * t, p, float(xy[t, p, 0]), float(xy[t, p, 1])) for t in range(9) if not np.isnan(xy[t, p, 0])]
             for p in range(bs[0], bs[1])]
    paths = [p for p in paths if p]
    out = SGANPredictor(model)(paths, np.zeros((len(paths), 2)), n_predict=12, modes=3, obs_length=9,
                               args=types.SimpleNamespace(normalize_scene=False))
    assert sorted(out) == [0, 1, 2]
    assert out[0][0].shape == (12, 2) and out[0][1].shape == (12, len(paths) - 1, 2) and out[1][1] == []


@pytest.mark.gpu
def test_discriminator_refuses_more_tracks_than_batch_split():
    """A batch_split that covers fewer tracks than observed is refused, as LSTM.forward refuses it."""
    name, kind, xy, bs, Wg, Wd, noise = _inputs(SGAN_CASES[0])
    _, dis = _models(kind, Wg, Wd, noise)
    scene = torch.from_numpy(np.concatenate([xy, xy[:, :1]], axis=1))         # one track more than bs[-1]
    with torch.no_grad(), pytest.raises(ValueError, match=r"batch_split\[-1\] != number of tracks"):
        dis(scene[:9], scene[9:21], torch.zeros(scene.shape[1], 2), torch.from_numpy(bs))


@pytest.mark.gpu
def test_sgan_training_fails_loudly():
    name, kind, xy, bs, Wg, Wd, noise = _inputs(SGAN_CASES[0])
    gen, _ = _models(kind, Wg, Wd, noise)
    gen.train()
    with pytest.raises(NotImplementedError):
        gen(torch.from_numpy(xy[:9]), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), n_predict=12)
