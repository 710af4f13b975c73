"""Collision attack on LSTM forecasts: how far must the primary's observed track move for the forecast to collide?

Per scene the attack perturbs the primary's observed positions by delta, one 2-vector per observed frame with
|delta_t| <= eps, to minimise D, the smallest distance between the primary's and a neighbour's predicted positions at
the points the scorer's Col-I test samples (D <= 0.2 m exactly when Col-I fires).  Projected gradient descent with
normalised per-frame steps of alpha = 2.5 eps / steps, on the gradient of the free-running forecast with nothing detached
(lstm.differentiable_rollout); a scene stops moving once its best D is <= 0.2 m.  The result is, per scene, the iterate
with the smallest D (the earlier one on ties).  Objective and step are one CUDA launch each (csrc/attack.cu).

`python -m trajnetplusplusbaselines_b200.attack --path <dataset> --output <model.pkl>` attacks every test scene of
DATA_BLOCK/<dataset>/test, writes the attacked predictions to test_pred/<model>_attack_eps<eps>_steps<steps>/ and
the per-scene delta and D to <that folder>.npz, and prints the evaluator's table for the clean and the attacked
predictions.
"""
import collections
import os
import shutil
import tempfile

import numpy as np
import torch

from . import _lib
from .engine import _ptr, _stream
from .lstm.training import check_rollout

COL_LIMIT = 0.2

AttackResult = collections.namedtuple('AttackResult', 'delta predictions clean_predictions d_clean d_attacked')
AttackResult.__doc__ = """delta [n, obs_length, 2] float64: the primary's perturbation per observed frame (world frame);
predictions / clean_predictions: per scene {0: [primary [pred_length, 2], neighbours [pred_length, N - 1, 2]]} as
LSTMPredictor.predict_batch_xy returns them; d_clean / d_attacked [n] float64: D before and after (+inf: no pair)."""


def _rotate(v, angle):
    """center_scene's rotation (lstm/utils.py:32-51) of [..., 2] vectors by `angle` [B] (broadcast over the scenes axis)."""
    ct, st = np.cos(angle), np.sin(angle)
    return np.stack([v[..., 0] * ct - v[..., 1] * st, v[..., 0] * st + v[..., 1] * ct], axis=-1)


def _attack_chunk(model, xys, eps, steps, obs_length, pred_length, normalize_scene):
    from .lstm.training import differentiable_rollout
    lib = _lib.load()
    device = model._device()
    split = np.zeros(len(xys) + 1, dtype=np.int64)
    split[1:] = np.cumsum([xy.shape[1] for xy in xys])
    B, M = len(xys), int(split[-1])
    if normalize_scene:
        # the frame is fixed by the clean observation: the attack runs in it, delta is rotated back at the end
        from .lstm.scene_ops import preprocess_scenes
        observed, _, _, rotation, center = preprocess_scenes([xy[:obs_length] for xy in xys], device=device,
                                                             normalize_scene=True, obs_length=obs_length)[:5]
    else:
        observed = torch.Tensor(np.concatenate([xy[:obs_length] for xy in xys], axis=1)).to(device)
    observed = observed.contiguous()
    layout = model._layouts.get(torch.from_numpy(split), pad_to_batch_max=False, device=device)
    f32 = dict(dtype=torch.float32, device=device)
    f64 = dict(dtype=torch.float64, device=device)
    delta = torch.zeros((obs_length, B, 2), **f32)
    best_delta = torch.zeros((obs_length, B, 2), **f32)
    best_D = torch.full((B,), float('inf'), **f64)
    D = torch.empty((B,), **f64)
    observed_adv = observed.clone()
    alpha = 2.5 * eps / steps
    st = _stream(device)
    for it in range(steps + 1):
        move = it < steps
        obs_in = observed_adv.clone().requires_grad_(move)
        with torch.enable_grad():
            _, positions = differentiable_rollout(model, obs_in, torch.from_numpy(split), pred_length,
                                                  pad_to_batch_max=False)
        positions = positions.contiguous()
        F = int(positions.shape[0])
        dpos = torch.empty_like(positions)
        with torch.cuda.device(device):
            _lib.check(lib.tb2_attack_objective(layout.handle, _ptr(positions), F, F - pred_length, _ptr(D), _ptr(dpos),
                                                st))
        d_obs = torch.autograd.grad(positions, obs_in, grad_outputs=dpos)[0].contiguous() if move else None
        if it == 0:           # iterate 0 also stays the best of a scene whose D is +inf on every iterate
            clean, d_clean, best_pos = positions.detach().clone(), D.clone(), positions.detach().clone()
        with torch.cuda.device(device):
            _lib.check(lib.tb2_attack_step(layout.handle, _ptr(d_obs), _ptr(observed), obs_length, _ptr(delta), _ptr(D), F,
                                           _ptr(positions), _ptr(best_D), _ptr(best_delta), _ptr(best_pos),
                                           _ptr(observed_adv), float(eps), float(alpha), int(move), st))
    if normalize_scene:
        from .lstm.scene_ops import inverse_scenes
        out, out_clean = inverse_scenes(best_pos, split, rotation, center), inverse_scenes(clean, split, rotation, center)
        delta_w = _rotate(best_delta.double().cpu().numpy(), -np.asarray(rotation, dtype=np.float64))
    else:
        out, out_clean = best_pos.cpu().numpy(), clean.cpu().numpy()
        delta_w = best_delta.double().cpu().numpy()

    def per_scene(arr):
        return [{0: [np.array(arr[-pred_length:, split[i]]), np.array(arr[-pred_length:, split[i] + 1:split[i + 1]])]}
                for i in range(B)]
    return (delta_w.transpose(1, 0, 2), per_scene(out), per_scene(out_clean), d_clean.cpu().numpy(),
            best_D.cpu().numpy())


def collision_attack(model, xys, eps=0.1, steps=20, obs_length=9, pred_length=12, normalize_scene=False, chunk=1024):
    """Attack every scene of `xys` (float64 [n_frames, N_i, 2] arrays, primary first, as data.load_test_scenes_xy gives
    them; frames [0, obs_length) are observed), `chunk` scenes per batched forward.  Each chunk takes steps + 1 forwards
    and `steps` backwards on the device.  eps = 0 gives the clean forecast (delta stays exactly 0).  With
    normalize_scene every scene is centred and rotated once, by the frame its CLEAN observation defines
    (scene_ops.preprocess_scenes); the attack runs in that frame (the ball is rotation-invariant), the predictions go back
    through inverse_scenes and delta is rotated back.  Returns an AttackResult."""
    if not eps >= 0:
        raise ValueError("eps must be >= 0, got %r" % (eps,))
    if int(steps) != steps or steps < 1:
        raise ValueError("steps must be an integer >= 1, got %r" % (steps,))
    check_rollout(model)
    model.eval()
    parts = [_attack_chunk(model, xys[i:i + chunk], eps, int(steps), obs_length, pred_length, normalize_scene)
             for i in range(0, len(xys), chunk)]
    if not parts:
        e = np.empty(0)
        return AttackResult(np.empty((0, obs_length, 2)), [], [], e, e)
    return AttackResult(np.concatenate([p[0] for p in parts]), sum((p[1] for p in parts), []),
                        sum((p[2] for p in parts), []), np.concatenate([p[3] for p in parts]),
                        np.concatenate([p[4] for p in parts]))


def main(argv=None):
    import argparse
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--path', default='trajdata', help='dataset under DATA_BLOCK (its test / test_private folders)')
    parser.add_argument('--output', required=True, help='saved LSTM model (.pkl)')
    parser.add_argument('--eps', default=0.1, type=float, help='radius of the per-frame L2 ball, metres')
    parser.add_argument('--steps', default=20, type=int, help='PGD steps')
    parser.add_argument('--normalize_scene', action='store_true')
    parser.add_argument('--obs_length', default=9, type=int)
    parser.add_argument('--pred_length', default=12, type=int)
    parser.add_argument('--chunk', default=1024, type=int, help='scenes per batched forward')
    args = parser.parse_args(argv)
    if not args.eps > 0:
        raise SystemExit("--eps must be > 0 (got %g)" % args.eps)
    if args.steps < 1:
        raise SystemExit("--steps must be >= 1 (got %d)" % args.steps)
    from .data import load_test_scenes_xy, write_predictions_xy
    from .lstm import LSTMPredictor
    from .scoring import format_table, score_file
    predictor = LSTMPredictor.load(args.output)
    try:
        check_rollout(predictor.model)
    except NotImplementedError as e:
        raise SystemExit("attack: %s" % e)
    predictor.model.to('cuda')
    root = os.path.join('DATA_BLOCK', args.path)
    test_dir, private_dir = os.path.join(root, 'test'), os.path.join(root, 'test_private')
    name = '%s_attack_eps%g_steps%d' % (os.path.basename(args.output).replace('.pkl', ''), args.eps, args.steps)
    out_dir = os.path.join(root, 'test_pred', name)
    if os.path.exists(out_dir):
        raise SystemExit("attack: %s already exists" % out_dir)
    datasets = sorted(f for f in os.listdir(test_dir) if not f.startswith('.') and f.endswith('.ndjson'))
    os.makedirs(out_dir)
    clean_dir = tempfile.mkdtemp()
    rec = collections.defaultdict(list)
    clean_results, attacked_results = {}, {}
    try:
        for dataset in datasets:
            scenes = load_test_scenes_xy(os.path.join(test_dir, dataset), args.obs_length)
            res = collision_attack(predictor.model, [xy for xy, _ in scenes], args.eps, args.steps, args.obs_length,
                                   args.pred_length, args.normalize_scene, args.chunk)
            metas = [meta for _, meta in scenes]
            for folder, preds in ((out_dir, res.predictions), (clean_dir, res.clean_predictions)):
                target = os.path.join(folder, dataset)
                open(target, 'w').close()
                if preds:
                    write_predictions_xy(preds, metas, target, obs_length=args.obs_length, pred_length=args.pred_length)
            key = dataset[:-len('.ndjson')]
            for results, folder in ((clean_results, clean_dir), (attacked_results, out_dir)):
                results[key] = score_file(os.path.join(private_dir, dataset), os.path.join(folder, dataset),
                                          obs_length=args.obs_length, pred_length=args.pred_length)
            rec['dataset'] += [key] * len(scenes)
            rec['scene_id'].append(np.array([meta.scene_id for meta in metas], dtype=np.int64))
            rec['delta'].append(res.delta)
            rec['d_clean'].append(res.d_clean)
            rec['d_attacked'].append(res.d_attacked)
    finally:
        shutil.rmtree(clean_dir)
    cat = {k: np.concatenate(v) if v else np.empty(0) for k, v in rec.items() if k != 'dataset'}
    np.savez(out_dir + '.npz', dataset=np.array(rec['dataset'], dtype=str), scene_id=cat.get('scene_id', np.empty(0)),
             delta=cat.get('delta', np.empty((0, args.obs_length, 2))), d_clean=cat.get('d_clean', np.empty(0)),
             d_attacked=cat.get('d_attacked', np.empty(0)))
    label = os.path.basename(args.output).replace('.pkl', '')
    print(format_table(label + ' clean', clean_results, 'NA'))
    print(format_table(label + ' attacked', attacked_results, 'NA'))
    d_att = cat.get('d_attacked', np.empty(0))
    print('attacked %d scenes, %d reached D <= %g m' % (len(d_att), int(np.sum(d_att <= COL_LIMIT)), COL_LIMIT))


if __name__ == '__main__':
    main()
