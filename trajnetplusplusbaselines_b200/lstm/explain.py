"""Explain LSTM forecasts: layer-wise relevance (LRP) of every neighbour to each predicted step of a scene's primary.

For each scene b and prediction t = 0 .. n_predict - 1 of the free-running forecast model(observed, None, batch_split,
n_predict) the explained scalar is y = |mu|, the norm of the primary's predicted mean velocity at step
s_t = obs_length - 2 + t (y = d . mu with d = mu / |mu| held fixed; y = 0 and every relevance 0 when mu is 0 or not finite).
Relevance goes backward with the eps-rule (Bach et al. 2015, z' = z + eps sign(z), sign(0) = +1) through the Linear layers
and the signal-take-all rule (Arras et al. 2017) through the LSTM cell:

  head      R_h[u] = h_u (d . W_n[0:2, u]) / y' * y
  cell      R_c = R_h (+ R_c_prev from the later step); R_c_prev = f c_prev / c' R_c, R_g = i g / c' R_c; i, f, o get nothing
  operand   z_g = W_g [emb | pooled | h_prev] + b_g:  R_X[k] = X_k sum_u W_g[u, k] R_g[u] / z_g[u]'; the h_prev part and
            R_c_prev continue at step s - 1, down to step 0
  own       the emb part through ReLU(Linear(2 -> E - 2)) of 4 vel, one eps-rule, summed over both velocity components:
            the primary's own relevance at step s
  grid      the pooled part through the grid embedding's ReLU(Linear) layers (one eps-rule each) to each cell value
            G[cell, ch]; a cell's relevance, summed over its channels, goes to the neighbour that won the cell at that step
            (the forward's last writer); overwritten writers and empty cells get nothing.  Cell values: occupancy 1,
            directional the winner's relative velocity, social the winner's latent W_enc h_j + b_enc (relevance stops
            there and does not enter the neighbour's own history)
  decoder   the inputs are the fed-back positions (the primary's and the neighbours' predictions): reported the same way
  absent    where the primary is absent its state is carried unchanged: relevance passes through and no input gets any

The residual y - sum(all reported relevance) is what the biases and eps absorbed.  The pass runs on the device
(csrc/relevance.cu, tb2_lstm_relevance) on the forward's saved states and the training backward's per-step records of the
primaries; results are bit-identical from run to run.

`python -m trajnetplusplusbaselines_b200.lstm.explain --model X.pkl --input test.ndjson --output rel.npz` explains every
test scene of an ndjson file (read and preprocessed as the evaluator's column pipeline does) and writes one npz.
"""
import collections
import ctypes

import numpy as np
import torch

from .. import _lib
from ..engine import _ptr, _stream
from .training import check_rollout

Relevance = collections.namedtuple('Relevance', 'relevance explained residual normals positions')
Relevance.__doc__ = """relevance [n_predict, S, M] float32: for prediction t, the relevance of each track's input at step s (the own
velocity column at the scene's primary, each neighbour's column elsewhere; S = obs_length - 1 + n_predict - 1);
explained [n_predict, B]: y = |mu| of each scene's primary at its step s_t; residual [n_predict, B]: y minus the scene's
summed relevance; normals / positions: the forecast, bit for bit model(observed, None, batch_split, n_predict)'s.
relevance / explained / residual are on the model's device, normals / positions on the device `observed` came from."""


def check_relevance(model):
    """NotImplementedError, before anything runs, for the models relevance() does not explain: S-GAN / VAE, goal models,
    the non-grid and user-defined interaction modules (check_rollout), and grid configurations the training backward does
    not take (trainer.check_trainable's grid rules: three_layer, constant != 0, pool_to_input=False, widths above 1024)."""
    from .trainer import check_trainable
    check_rollout(model)
    try:
        check_trainable(model)
    except RuntimeError as e:
        raise NotImplementedError("relevance: %s" % e)
    pool = model.pool
    if pool is not None and pool.type_ == 'social' and max(
            m.out_features for m in pool.embedding if isinstance(m, torch.nn.Linear)) > 1024:
        raise NotImplementedError("relevance: social grid embedding widths above 1024 are not built")


def relevance(model, observed, batch_split, n_predict=12, eps=1e-3, pad_to_batch_max=True):
    """Layer-wise relevance of the free-running forecast model(observed, None, batch_split, n_predict) (module docstring):
    observed [obs_length, M, 2] with the primary first in each scene of batch_split [B + 1]; pad_to_batch_max as in
    differentiable_rollout (True: the trainer's padded batch, False: every scene as if it were called on its own).
    Returns a Relevance."""
    check_relevance(model)
    if not (eps >= 0 and np.isfinite(eps)):
        raise ValueError("eps must be finite and >= 0, got %r" % (eps,))
    if int(n_predict) != n_predict or n_predict < 1:
        raise ValueError("n_predict must be an integer >= 1, got %r" % (n_predict,))
    n_predict = int(n_predict)
    lib = _lib.load()
    split = torch.as_tensor(batch_split, dtype=torch.int64).cpu()
    with torch.no_grad():
        normals, positions, states, (obs, _, layout, _) = model._forward_nograd(
            observed, split, None, n_predict, want_states=True, pad_to_batch_max=pad_to_batch_max)
    handle = model._engine()
    device = handle.device
    obs_length = int(obs.shape[0])
    S = obs_length - 1 + n_predict - 1
    B, M = int(split.numel()) - 1, layout.num_tracks
    rel = torch.empty((n_predict, S, M), dtype=torch.float32, device=device)
    explained = torch.empty((n_predict, B), dtype=torch.float32, device=device)
    w, keep = handle.weights_struct(model._weight_fields())
    need = int(lib.tb2_lstm_relevance_workspace_bytes(handle.handle, layout.handle, n_predict, obs_length))
    ws = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.tb2_lstm_relevance(handle.handle, layout.handle, ctypes.byref(w), _ptr(obs), obs_length,
                                          n_predict - 1, _ptr(positions[-S:].contiguous()), _ptr(states), float(eps),
                                          _ptr(rel), _ptr(explained), _ptr(ws), need, _stream(device)))
    del keep
    scene_of = torch.repeat_interleave(torch.arange(B, device=device), (split[1:] - split[:-1]).to(device))
    summed = torch.zeros((n_predict, B), dtype=torch.float64, device=device)
    summed.index_add_(1, scene_of, rel.double().sum(dim=1))
    residual = (explained.double() - summed).float()
    out_device = observed.device if torch.is_tensor(observed) else torch.device('cpu')
    return Relevance(rel, explained, residual, normals.to(out_device), positions.to(out_device))


def explain_scenes(model, xys, n_predict=12, obs_length=9, eps=1e-3, normalize_scene=False):
    """relevance() of every scene of `xys` (float64 [n_frames, N_i, 2], primary first, as data.load_test_scenes_xy gives
    them) in one batched call, each scene as if it were called on its own (LSTMPredictor.predict_batch_xy's layout).
    With normalize_scene every scene is first centred and rotated as the predictor does.  Returns per scene
    (relevance [n_predict, S, N_i], explained [n_predict], residual [n_predict]) as float32 numpy arrays."""
    check_relevance(model)
    model.eval()
    split = np.zeros(len(xys) + 1, dtype=np.int64)
    split[1:] = np.cumsum([xy.shape[1] for xy in xys])
    if not xys:
        return []
    if normalize_scene:
        from .scene_ops import preprocess_scenes
        observed = preprocess_scenes([xy[:obs_length] for xy in xys], device=model._device(), normalize_scene=True,
                                     obs_length=obs_length)[0]
    else:
        observed = torch.Tensor(np.concatenate([xy[:obs_length] for xy in xys], axis=1))
    res = relevance(model, observed, torch.from_numpy(split), n_predict, eps, pad_to_batch_max=False)
    rel, expl, resid = res.relevance.cpu().numpy(), res.explained.cpu().numpy(), res.residual.cpu().numpy()
    return [(rel[:, :, split[i]:split[i + 1]], expl[:, i], resid[:, i]) for i in range(len(xys))]


def main(argv=None):
    import argparse
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--model', required=True, help='saved LSTM model (.pkl)')
    parser.add_argument('--input', required=True, help='test scenes (.ndjson)')
    parser.add_argument('--output', required=True, help='relevance record (.npz)')
    parser.add_argument('--eps', default=1e-3, type=float, help='stabiliser of the eps-rule')
    parser.add_argument('--n_predict', default=12, type=int, help='predictions explained per scene')
    parser.add_argument('--obs_length', default=9, type=int)
    parser.add_argument('--normalize_scene', action='store_true')
    args = parser.parse_args(argv)
    if not (args.eps >= 0 and np.isfinite(args.eps)):
        raise SystemExit("explain: --eps must be finite and >= 0 (got %g)" % args.eps)
    if args.n_predict < 1:
        raise SystemExit("explain: --n_predict must be >= 1 (got %d)" % args.n_predict)
    if args.obs_length < 2:
        raise SystemExit("explain: --obs_length must be >= 2 (got %d)" % args.obs_length)
    from .lstm import LSTMPredictor
    predictor = LSTMPredictor.load(args.model)
    try:
        check_relevance(predictor.model)
    except NotImplementedError as e:
        raise SystemExit("explain: %s" % e)
    from ..data import load_test_scenes_xy
    scenes = load_test_scenes_xy(args.input, args.obs_length)
    predictor.model.to('cuda')
    results = explain_scenes(predictor.model, [xy for xy, _ in scenes], args.n_predict, args.obs_length, args.eps,
                             args.normalize_scene)
    arrays = {}
    for i, ((_, meta), (rel, expl, resid)) in enumerate(zip(scenes, results)):
        arrays['scene_id_%d' % i] = np.int64(meta.scene_id)
        arrays['ped_ids_%d' % i] = np.array([meta.pedestrian] + list(meta.neigh_ids), dtype=np.int64)
        arrays['relevance_%d' % i] = rel
        arrays['explained_%d' % i] = expl
        arrays['residual_%d' % i] = resid
    np.savez(args.output, num_scenes=np.int64(len(scenes)), **arrays)
    print("explained %d scenes x %d predictions into %s" % (len(scenes), args.n_predict, args.output))


if __name__ == '__main__':
    main()
