"""VAE forecaster at test time (SURVEY.md 8f rank 2) vs vectors the unmodified reference produced with
its latent sampler patched to fixed samples (oracle/make_vae_golden.py)."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import lstm_oracle as O
from oracle import sgan_oracle as SO
from oracle.make_vae_golden import VAE_CASES, fixed_z

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "vae_golden.npz"))
IDS = [c[0] for c in VAE_CASES]


def _close(a, b, tol):
    assert (np.isnan(a) == np.isnan(b)).all()
    assert np.nanmax(np.abs(a - b)) < tol, float(np.nanmax(np.abs(a - b)))


@pytest.mark.parametrize("case", VAE_CASES, ids=IDS)
def test_oracle_matches_reference(case):
    name, kind, B, N, ragged, nan_tracks, dseed, wseed, modes = case
    xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
    W = SO.vae_weights(kind, wseed)
    z = fixed_z(name, modes, xy.shape[1])
    for k in range(modes):
        rel, pred = SO.vae_forward(W, O.pool_config(kind), xy[:9], bs, n_predict=12, z=z[k])
        _close(rel, GOLD["%s/rel%d" % (name, k)], 2e-5)
        _close(pred, GOLD["%s/pred%d" % (name, k)], 2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("case", VAE_CASES, ids=IDS)
def test_cuda_vae_matches_reference(case):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling
    from trajnetplusplusbaselines_b200.vae import VAE
    name, kind, B, N, ragged, nan_tracks, dseed, wseed, modes = case
    xy, bs = O.synthetic_scenes(B, N, seed=dseed, ragged=ragged, nan_tracks=nan_tracks)
    W = SO.vae_weights(kind, wseed)
    spec = O.MODEL_SPECS[kind]
    model = VAE(pool=GridBasedPooling(**spec) if spec else None, num_modes=modes)
    sd = model.state_dict()
    assert {k for k in sd if not k.startswith("goal_embedding.")} == {k for k in W if not k.startswith("goal_embedding.")}
    sd.update({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model.load_state_dict(sd)
    model = model.cuda().eval()
    model.fixed_z = torch.from_numpy(fixed_z(name, modes, xy.shape[1]))
    with torch.no_grad():
        rel_list, pred_list, zxy, zx = model(torch.from_numpy(xy[:9]), torch.zeros(xy.shape[1], 2),
                                             torch.from_numpy(bs), n_predict=12)
        outs = [(r.numpy().copy(), p.numpy().copy()) for r, p in zip(rel_list, pred_list)]
    assert zxy is None and zx is None and len(outs) == modes
    for k, (rel, pred) in enumerate(outs):
        _close(rel, GOLD["%s/rel%d" % (name, k)], 1e-4)
        _close(pred, GOLD["%s/pred%d" % (name, k)], 1e-4)


@pytest.mark.gpu
def test_vae_refuses_more_tracks_than_batch_split():
    """A batch_split that covers fewer tracks than observed is refused, as LSTM.forward refuses it."""
    from trajnetplusplusbaselines_b200.vae import VAE
    xy, bs = O.synthetic_scenes(3, 5, seed=9)
    scene = torch.from_numpy(np.concatenate([xy, xy[:, :1]], axis=1))         # one track more than bs[-1]
    model = VAE().cuda().eval()
    with torch.no_grad(), pytest.raises(ValueError, match=r"batch_split\[-1\] != number of tracks"):
        model(scene[:9], torch.zeros(scene.shape[1], 2), torch.from_numpy(bs), n_predict=12)


@pytest.mark.gpu
def test_vae_predictor_and_training_guard():
    from trajnetplusplusbaselines_b200.data import TrackRow
    from trajnetplusplusbaselines_b200.vae import VAE, VAEPredictor
    xy, bs = O.synthetic_scenes(1, 5, seed=9)
    model = VAE().cuda()
    paths = [[TrackRow(10 * t, p, float(xy[t, p, 0]), float(xy[t, p, 1])) for t in range(9)] for p in range(5)]
    np.random.seed(0)
    out = VAEPredictor(model)(paths, np.zeros((5, 2)), n_predict=12, modes=3, obs_length=9,
                              args=types.SimpleNamespace(normalize_scene=False))
    assert sorted(out) == [0, 1, 2] and out[0][0].shape == (12, 2) and out[0][1].shape == (12, 4, 2)
    assert np.abs(out[0][0] - out[1][0]).max() > 0         # different latent samples
    model.train()
    with pytest.raises(NotImplementedError):
        model(torch.from_numpy(xy[:9]), torch.zeros(5, 2), torch.from_numpy(bs), n_predict=12)
