"""Attribute LSTM forecast errors to neighbours: exact Shapley values over every coalition of each scene's nearest neighbours.

Definition.  For each scene b (after the evaluator's preprocessing, primary first):

  players     the K nearest neighbours of the primary at the last observed frame, K = min(players, N_b - 1), players in
              0..12 (default 8).  Distance is the squared Euclidean distance in float64 of the float32 positions the model
              reads; a neighbour whose position there is not finite counts as +inf; ties go to the lower row.  Every other
              neighbour is background and is in every coalition.  Player r is the r-th nearest (rank r, bit r of a mask).
  instance    for each coalition S of the players (a mask over the ranks), the scene with the players outside S deleted:
              xy[:, rows] with the primary first and the remaining tracks in their original relative order (row order
              decides the grid pools' last-writer cells).  Deleting a row is the counterfactual, not NaN-masking it: the
              attention module's fill values and the nearest-neighbour padding would see NaN rows.
  values      v_ADE(S), v_FDE(S): the ADE / FDE in float64 of the primary's free-running mean forecast of instance (b, S)
              against its ground truth over the n_predict predicted frames, bit for bit what scoring.score_arrays returns
              for mode 0 of the same unrounded prediction.
  Shapley     phi_j = sum over S subset of P \\ {j} of |S|! (K - |S| - 1)! / K! (v(S u {j}) - v(S)), summed in float64 in
              ascending mask order without atomics; the weights are ratios of exact integer factorials (exact for K <= 12).
              A negative phi means the neighbour's presence lowers the error.  sum_j phi_j = v(P) - v(empty) up to rounding.
  normalize   center_scene depends only on the primary's observation, so every instance shares its scene's frame: scenes
              are normalised once, before the expansion, and the predictions go back to the world frame before they are
              scored; the values are those of predict_batch_xy(args.normalize_scene=True)'s world-frame predictions.

Device work, per chunk of scenes (at most `chunk` instances, a scene's 2^K instances never split): one launch of
tb2_shapley_expand builds every instance's observed rows (csrc/shapley.cu); the forecasts are one LSTM._forward_nograd
(pad_to_batch_max=False: each instance as if it ran alone) over the instance batch; one launch of tb2_shapley_values
scores every instance and sums the Shapley values, one CTA per scene.  The host computes the instances' batch_split from
the scene sizes, K and the popcounts of the masks, without reading anything back from the device.  Results do not depend
on `chunk`.

Every built-in interaction module is served in every configuration its inference forward takes.  Goal models, S-GAN /
VAE (stochastic, not an LSTM) and user-defined interaction modules are refused before anything runs.

`python -m trajnetplusplusbaselines_b200.lstm.shapley --path <dataset> --output <model.pkl>` attributes every scene of
DATA_BLOCK/<dataset>/test_private/*.ndjson and writes <model>_shapley_players<K>.npz beside the model.
"""
import collections
import os

import numpy as np
import torch

from .. import _lib
from ..engine import _ptr, _stream

MAX_PLAYERS = 12
MAX_SCENE_ROWS = 6144          # tb2_shapley_expand keeps one distance per row of a scene in shared memory

_POPCOUNT = np.array([bin(m).count('1') for m in range(1 << MAX_PLAYERS)], dtype=np.int64)

Shapley = collections.namedtuple('Shapley', 'phi_ade phi_fde player_rows num_players v_full_ade v_full_fde v_empty_ade '
                                            'v_empty_fde positions values')
Shapley.__doc__ = """phi_ade, phi_fde [B, 12] float64 (NaN past K); player_rows [B, 12] int64: the players' rows in their
scene by rank (-1 past K); num_players [B] int64: K; v_full_ade / v_full_fde / v_empty_ade / v_empty_fde [B] float64:
v(all players), v(no player); positions [F, M, 2] float32: the full scenes' forecast, bit for bit
_forward_nograd(observed, batch_split, None, n_predict, pad_to_batch_max=False)'s; values [I, 2] float64 (v_ADE, v_FDE of
every instance, scene b's 2^K rows in mask order after those of the scenes before it) or None when not asked for."""


def check_shapley(model):
    """NotImplementedError, before anything runs, for the models shapley() does not attribute: S-GAN / VAE (stochastic,
    not an LSTM), goal models and user-defined interaction modules (they run in torch, and a module that mixes the
    entries of its batch would couple the instances)."""
    from .external import is_external
    from .lstm import LSTM
    if type(model) is not LSTM:
        raise NotImplementedError("shapley serves LSTM models; %s (S-GAN / VAE) is not built" % type(model).__name__)
    if model.goal_flag:
        raise NotImplementedError("shapley of a goal-conditioned model (goal_flag=True) is not built")
    if is_external(model.pool):
        raise NotImplementedError("shapley of a user-defined interaction module (%s) is not built"
                                  % type(model.pool).__name__)


def _check_players(players):
    if isinstance(players, bool) or int(players) != players or not 0 <= players <= MAX_PLAYERS:
        raise ValueError("players must be an integer in 0..%d, got %r" % (MAX_PLAYERS, players))
    return int(players)


def _check_truth(truth, num_scenes, n_predict):
    """truth as float64 [B, n_predict, 2] host array; ValueError for a shape that does not match or a non-finite
    position of a primary."""
    if int(n_predict) != n_predict or n_predict < 1:
        raise ValueError("n_predict must be an integer >= 1, got %r" % (n_predict,))
    truth = truth.detach().cpu().numpy() if torch.is_tensor(truth) else np.asarray(truth)
    truth = np.ascontiguousarray(truth, dtype=np.float64)
    if truth.shape != (num_scenes, int(n_predict), 2):
        raise ValueError("truth must be [%d, %d, 2] (each scene's primary over the predicted frames), got %s"
                         % (num_scenes, int(n_predict), list(truth.shape)))
    bad = np.nonzero(~np.isfinite(truth).all(axis=(1, 2)))[0]
    if len(bad):
        raise ValueError("scene %d: the primary's truth has a non-finite position" % int(bad[0]))
    return truth


def num_players(sizes, players):
    """K per scene: min(players, N_b - 1)."""
    return np.minimum(int(players), np.maximum(np.asarray(sizes, dtype=np.int64) - 1, 0))


def instance_split(sizes, K):
    """batch_split [I + 1] of the instances of scenes of `sizes` rows with K players each: scene b's 2^K instances in
    mask order, instance (b, mask) of N_b - K_b + popcount(mask) rows."""
    parts = [n - k + _POPCOUNT[:1 << k] for n, k in zip(np.asarray(sizes, dtype=np.int64), np.asarray(K, dtype=np.int64))]
    split = np.zeros(sum(len(p) for p in parts) + 1, dtype=np.int64)
    if parts:
        np.cumsum(np.concatenate(parts), out=split[1:])
    return split


def chunks(K, chunk):
    """[(b0, b1)]: consecutive scenes whose instances (2^K each) add up to at most `chunk`."""
    out, b0, total = [], 0, 0
    for b, k in enumerate(np.asarray(K, dtype=np.int64)):
        n = 1 << int(k)
        if total + n > chunk:
            out.append((b0, b))
            b0, total = b, 0
        total += n
    if len(K):
        out.append((b0, len(K)))
    return out


def _i32(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)


def shapley(model, observed, truth, batch_split, players=8, n_predict=12, chunk=65536, scene_frames=None,
            return_values=False):
    """Shapley values of each scene's players for the ADE and FDE of its primary's forecast (module docstring).

    observed [obs_length, M, 2] (the model's input, primary first in each scene of batch_split [B + 1]); truth
    [B, n_predict, 2] the primaries' ground truth over the predicted frames; chunk: instances per forward.  scene_frames
    = (rotation [B], centre [B, 2]) of center_scene (scene_ops.preprocess_scenes returns them): `observed` is in the
    scenes' normalised frames, and the predictions go back to the world frame (inverse_scenes) before they are scored.
    Returns a Shapley of tensors on the model's device; return_values: also every instance's value."""
    check_shapley(model)
    players = _check_players(players)
    split = np.asarray(torch.as_tensor(batch_split, dtype=torch.int64).cpu().numpy(), dtype=np.int64)
    B = len(split) - 1
    truth = _check_truth(truth, B, n_predict)
    n_predict = int(n_predict)
    if isinstance(chunk, bool) or int(chunk) != chunk or chunk < 1:
        raise ValueError("chunk must be an integer >= 1, got %r" % (chunk,))
    sizes = np.diff(split)
    if tuple(observed.shape[1:]) != (int(split[-1]), 2):
        raise ValueError("observed must be [obs_length, %d, 2], got %s" % (int(split[-1]), list(observed.shape)))
    if B and (sizes < 1).any():
        raise ValueError("every scene needs its primary (batch_split must increase)")
    if B and sizes.max() > MAX_SCENE_ROWS:
        raise ValueError("scenes of more than %d tracks are not built" % MAX_SCENE_ROWS)
    K = num_players(sizes, players)
    if B and (1 << int(K.max())) > chunk:
        raise ValueError("chunk=%d is below a scene's 2^K = %d instances" % (chunk, 1 << int(K.max())))
    model.eval()
    handle = model._engine()
    device = handle.device
    lib = _lib.load()
    st = _stream(device)
    f64 = dict(dtype=torch.float64, device=device)
    obs = observed.detach().to(device=device, dtype=torch.float32).contiguous()
    T_obs = int(obs.shape[0])
    truth_d = torch.from_numpy(truth).to(device)
    frame_d = None
    if scene_frames is not None:
        from .scene_ops import _frame_table
        rotation, center = scene_frames
        frame_d = torch.from_numpy(_frame_table(np.asarray(center, dtype=np.float64).reshape(B, 2),
                                                -np.asarray(rotation, dtype=np.float64).reshape(B))).to(device)
    parts = collections.defaultdict(list)
    for b0, b1 in chunks(K, int(chunk)):
        nb, k = b1 - b0, K[b0:b1]
        first = np.zeros(nb + 1, dtype=np.int64)
        np.cumsum(1 << k, out=first[1:])
        isplit = instance_split(sizes[b0:b1], k)
        I, M_out = int(first[-1]), int(isplit[-1])
        # held until the launches are queued: a freed temporary's memory could take the next upload
        scene_off_d, first_d, isplit_d = _i32(split[b0:b1 + 1], device), _i32(first, device), _i32(isplit, device)
        expanded = torch.empty((T_obs, M_out, 2), dtype=torch.float32, device=device)
        rows = torch.empty((nb, MAX_PLAYERS), dtype=torch.int32, device=device)
        coalition = torch.empty(I, dtype=torch.int32, device=device)
        with torch.cuda.device(device):
            _lib.check(lib.tb2_shapley_expand(_ptr(obs), T_obs, int(obs.shape[1]), _ptr(scene_off_d),
                                              _ptr(first_d), _ptr(isplit_d), nb, I, int(sizes[b0:b1].max()), M_out,
                                              _ptr(expanded), _ptr(rows), _ptr(coalition), st))
        with torch.no_grad():
            _, pos = model._forward_nograd(expanded, torch.from_numpy(isplit), None, n_predict, pad_to_batch_max=False)
        pos = pos.contiguous()
        phi_a = torch.empty((nb, MAX_PLAYERS), **f64)
        phi_f = torch.empty((nb, MAX_PLAYERS), **f64)
        v = torch.empty((4, nb), **f64)
        values = torch.empty((I, 2), **f64) if return_values else None
        with torch.cuda.device(device):
            _lib.check(lib.tb2_shapley_values(_ptr(pos), int(pos.shape[0]), M_out, n_predict, _ptr(first_d),
                                              _ptr(isplit_d), nb, int(k.max()), _ptr(truth_d[b0:b1]),
                                              _ptr(frame_d[b0:b1]) if frame_d is not None else None, _ptr(phi_a),
                                              _ptr(phi_f), _ptr(v), _ptr(values) if values is not None else None, st))
        # the full coalition (the last mask) keeps every row in order: its rows are the scene's own forecast
        local = split[b0:b1] - split[b0]
        full = np.arange(int(sizes[b0:b1].sum())) + np.repeat(isplit[first[1:] - 1] - local, sizes[b0:b1])
        parts['positions'].append(pos[:, torch.from_numpy(full).to(device)])
        parts['phi_ade'].append(phi_a)
        parts['phi_fde'].append(phi_f)
        parts['rows'].append(rows)
        parts['v'].append(v)
        if values is not None:
            parts['values'].append(values)
    if not B:
        F = T_obs - 1 + n_predict - 1 + (1 if T_obs == 2 else 0)
        empty = torch.empty((0, MAX_PLAYERS), **f64)
        e = torch.empty(0, **f64)
        return Shapley(empty, empty.clone(), torch.empty((0, MAX_PLAYERS), dtype=torch.int64, device=device),
                       torch.empty(0, dtype=torch.int64, device=device), e, e.clone(), e.clone(), e.clone(),
                       torch.empty((F, 0, 2), dtype=torch.float32, device=device),
                       torch.empty((0, 2), **f64) if return_values else None)
    v = torch.cat(parts['v'], dim=1)
    return Shapley(torch.cat(parts['phi_ade']), torch.cat(parts['phi_fde']), torch.cat(parts['rows']).long(),
                   torch.from_numpy(K).to(device), v[0], v[1], v[2], v[3], torch.cat(parts['positions'], dim=1),
                   torch.cat(parts['values']) if return_values else None)


def shapley_scenes(model, xys, truths, players=8, n_predict=12, obs_length=9, normalize_scene=False, chunk=65536,
                   return_values=False):
    """shapley() of every scene of `xys` (float64 [n_frames, N_i, 2], primary first, as data.load_test_scenes_xy gives
    them; frames [0, obs_length) are observed) against truths (per scene the primary's [n_predict, 2] ground truth).
    With normalize_scene every scene is centred and rotated once, as LSTMPredictor.predict_batch_xy does, and the
    predictions are scored in the world frame.  Returns a Shapley of host arrays (positions in the model's frame)."""
    check_shapley(model)
    players = _check_players(players)
    truth = _check_truth(np.stack([np.asarray(t, dtype=np.float64) for t in truths]) if len(truths) else
                         np.zeros((0, int(n_predict), 2)), len(xys), n_predict)
    split = np.zeros(len(xys) + 1, dtype=np.int64)
    split[1:] = np.cumsum([xy.shape[1] for xy in xys])
    device = model._device()
    frames = None
    if normalize_scene and xys:
        from .scene_ops import preprocess_scenes
        observed, _, _, rotation, center = preprocess_scenes([xy[:obs_length] for xy in xys], device=device,
                                                             normalize_scene=True, obs_length=obs_length)[:5]
        frames = (rotation, center)
    elif xys:
        observed = torch.Tensor(np.concatenate([xy[:obs_length] for xy in xys], axis=1))
    else:
        observed = torch.empty((obs_length, 0, 2))
    res = shapley(model, observed, truth, split, players, n_predict, chunk, frames, return_values)
    return Shapley(*(f.cpu().numpy() if f is not None else None for f in res))


def summary(phi, v_full, v_empty, num_players):
    """For one metric over a set of scenes: (scenes, mean v(empty) - v(full) -- what the neighbours do to the error --,
    mean sum_j |phi_j|, and the share of the scenes with players where the nearest neighbour's |phi| is the largest and
    not 0).  NaN for a mean or share over no scene."""
    n = len(num_players)
    absphi = np.where(np.isnan(phi), 0.0, np.abs(phi))
    has = num_players > 0
    top = has & (absphi[:, 0] > 0) & (absphi[:, 0] == absphi.max(axis=1, initial=0.0))
    nan = float('nan')
    return (n, float(np.mean(v_empty - v_full)) if n else nan, float(np.mean(absphi.sum(axis=1))) if n else nan,
            float(top.sum()) / float(has.sum()) if has.any() else nan)


def format_line(label, ade, fde):
    """One printed summary line from summary() of the ADE and of the FDE attributions."""
    return "%-24s %7d %12.6f %12.6f %12.6f %12.6f %9.4f %9.4f" % (label, ade[0], ade[1], fde[1], ade[2], fde[2], ade[3],
                                                                  fde[3])


def _truths(private_file, scenes, obs_length, pred_length):
    """Per test scene the primary's ground truth [pred_length, 2]: the frames after the observation of the same scene
    id in data.load_scenes_xy of the file.  ValueError for a scene id without a match, too few frames, or an
    observation that differs."""
    from ..data import load_scenes_xy
    full = dict(load_scenes_xy(private_file))
    out = []
    for xy, meta in scenes:
        f = full.get(meta.scene_id)
        if f is None:
            raise ValueError("%s: scene %d has no ground truth" % (private_file, meta.scene_id))
        if f.shape[0] < obs_length + pred_length or not np.array_equal(f[:obs_length, 0], xy[:obs_length, 0],
                                                                       equal_nan=True):
            raise ValueError("%s: scene %d: the ground truth does not continue the observation over %d frames"
                             % (private_file, meta.scene_id, pred_length))
        out.append(f[obs_length:obs_length + pred_length, 0])
    return out


def main(argv=None):
    import argparse
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--path', default='trajdata', help='dataset under DATA_BLOCK (its test_private folder)')
    parser.add_argument('--output', required=True, help='saved LSTM model (.pkl)')
    parser.add_argument('--players', default=8, type=int, help='nearest neighbours attributed per scene (0..12)')
    parser.add_argument('--normalize_scene', action='store_true')
    parser.add_argument('--chunk', default=65536, type=int, help='counterfactual scenes per batched forward')
    parser.add_argument('--obs_length', default=9, type=int)
    parser.add_argument('--pred_length', default=12, type=int)
    args = parser.parse_args(argv)
    if not 0 <= args.players <= MAX_PLAYERS:
        raise SystemExit("shapley: --players must be in 0..%d (got %d)" % (MAX_PLAYERS, args.players))
    if args.chunk < (1 << args.players):
        raise SystemExit("shapley: --chunk must be >= 2^players = %d (got %d)" % (1 << args.players, args.chunk))
    if args.obs_length < 2:
        raise SystemExit("shapley: --obs_length must be >= 2 (got %d)" % args.obs_length)
    if args.pred_length < 1:
        raise SystemExit("shapley: --pred_length must be >= 1 (got %d)" % args.pred_length)
    from ..data import load_test_scenes_xy
    from .lstm import LSTMPredictor
    predictor = LSTMPredictor.load(args.output)
    try:
        check_shapley(predictor.model)
    except NotImplementedError as e:
        raise SystemExit("shapley: %s" % e)
    model = predictor.model.to('cuda')
    private_dir = os.path.join('DATA_BLOCK', args.path, 'test_private')
    files = sorted(f for f in os.listdir(private_dir) if not f.startswith('.') and f.endswith('.ndjson'))
    rec = collections.defaultdict(list)
    lines = []
    for name in files:
        path = os.path.join(private_dir, name)
        scenes = load_test_scenes_xy(path, args.obs_length)
        res = shapley_scenes(model, [xy for xy, _ in scenes], _truths(path, scenes, args.obs_length, args.pred_length),
                             args.players, args.pred_length, args.obs_length, args.normalize_scene, args.chunk)
        ids = np.full((len(scenes), MAX_PLAYERS), -1, dtype=np.int64)
        for i, (xy, meta) in enumerate(scenes):
            peds = [meta.pedestrian] + list(meta.neigh_ids)
            if len(peds) != xy.shape[1]:
                raise ValueError("%s: scene %d: %d pedestrian ids for %d tracks" % (path, meta.scene_id, len(peds),
                                                                                   xy.shape[1]))
            k = int(res.num_players[i])
            ids[i, :k] = [peds[r] for r in res.player_rows[i, :k]]
        key = name[:-len('.ndjson')]
        rec['dataset'] += [key] * len(scenes)
        rec['scene_id'].append(np.array([meta.scene_id for _, meta in scenes], dtype=np.int64))
        rec['player_ids'].append(ids)
        for field in ('num_players', 'phi_ade', 'phi_fde', 'v_full_ade', 'v_full_fde', 'v_empty_ade', 'v_empty_fde'):
            rec[field].append(getattr(res, field))
        lines.append((key, res._asdict()))
    fields = ('scene_id', 'player_ids', 'num_players', 'phi_ade', 'phi_fde', 'v_full_ade', 'v_full_fde', 'v_empty_ade',
              'v_empty_fde')
    empty = dict(scene_id=np.empty(0, dtype=np.int64), player_ids=np.empty((0, MAX_PLAYERS), dtype=np.int64),
                 num_players=np.empty(0, dtype=np.int64), phi_ade=np.empty((0, MAX_PLAYERS)),
                 phi_fde=np.empty((0, MAX_PLAYERS)))
    pooled = {k: np.concatenate(rec[k]) if rec[k] else empty.get(k, np.empty(0)) for k in fields}
    out = '%s_shapley_players%d.npz' % (os.path.splitext(args.output)[0], args.players)
    np.savez(out, dataset=np.array(rec['dataset'], dtype=str), **pooled)
    print("%-24s %7s %12s %12s %12s %12s %9s %9s" % ('file', 'scenes', 'dADE', 'dFDE', 'sum|phi|ADE', 'sum|phi|FDE',
                                                     'top1 ADE', 'top1 FDE'))
    for key, r in lines + [('pooled', pooled)]:
        print(format_line(key, summary(r['phi_ade'], r['v_full_ade'], r['v_empty_ade'], r['num_players']),
                          summary(r['phi_fde'], r['v_full_fde'], r['v_empty_fde'], r['num_players'])))
    print("wrote %s" % out)


if __name__ == '__main__':
    main()
