"""Social-force / ORCA parameter sweeps and the classical evaluation table, on the device.

Replaces trajnetbaselines/classical/socialforce_eval.py: `evaluate` is its table for one setting (Evaluator.aggregate,
:25-84: N, ORCA, SF and KF, ADE / FDE means over the scenes of a file), `fit` the hyper-parameter tuning it leaves to
re-running the whole tool once per setting (:236-258).  Every (scene, setting) pair of a file is one work item of one
launch (socialforce.sweep / orca.sweep); only the primary's ADE / FDE leave the GPU.

    python -m trajnetplusplusbaselines_b200.classical.sweep FILES... --tau 0.3 0.5 --vo 2.1 --sigma 0.2 0.3

Each parameter flag takes several values and the sweep runs their Cartesian product.  `--simulator kalman` is the
Kalman filter (the reference's `kf` branch, unreachable from its own `choices`).
"""
import argparse
import itertools
import os

import numpy as np

from .. import data
from . import kalman, orca, socialforce
from .common import initial_states_xy, to_device

SF_DEFAULT = (0.5, 2.1, 0.3)          # --tau --vo --sigma      (socialforce_eval.py:146-151)
ORCA_DEFAULT = (4.0, 4.0, 0.6)        # --min_dist --react_time --radius  (:153-158)


def _representable(cols):
    """Per scene of the parsed columns (load_scenes_xy's order): True when its xy array holds all of its rows, i.e.
    every row of a pedestrian that has one on the primary's frames lies on those frames, once per frame, with finite
    coordinates (NaN in the array means "no row")."""
    order = np.argsort(cols['frame'], kind='stable')
    f, p, x, y = cols['frame'][order], cols['ped'][order], cols['x'][order], cols['y'][order]
    los = np.searchsorted(f, cols['scene_start'], side='left')
    his = np.searchsorted(f, cols['scene_end'], side='right')
    ok = []
    for i in range(len(los)):
        lo, hi = int(los[i]), int(his[i])
        fs, ps = f[lo:hi], p[lo:hi]
        pf = np.unique(fs[ps == cols['scene_ped'][i]])
        if len(pf) == 0:
            continue                                    # no primary: the scene is skipped by both pipelines
        kept = np.isin(ps, np.unique(ps[np.isin(fs, pf)]))
        fk, pk = fs[kept], ps[kept]
        ok.append(bool(np.isin(fk, pf).all() and np.isfinite(x[lo:hi][kept]).all() and np.isfinite(y[lo:hi][kept]).all()
                       and len(np.unique(np.stack([pk, fk]), axis=1)[0]) == len(pk)))
    return ok


def load_scenes(path, dest_type='interp'):
    """[(scene_id, xy or paths)] of a file for initial_states_xy: xy arrays from the native column pipeline, the rows
    (paths) of every scene an xy array cannot represent, and of all scenes for dest_type 'true'."""
    cols = None if dest_type == 'true' else data.parse_ndjson_columns(path)
    if cols is None:
        return list(data.read_ndjson_scenes(path))
    scenes = data.load_scenes_xy(path)
    ok = _representable(cols)
    if not all(ok):
        rows = list(data.read_ndjson_scenes(path))
        scenes = [s if good else r for s, r, good in zip(scenes, rows, ok)]
    return scenes


def prepare_file(path, obs_length=9, pred_length=12, dest_type='interp', dest_dict=None, device=None):
    """initial_states_xy of every scene of an ndjson file, moved to the device once (common.PreparedScenes)."""
    scenes = load_scenes(path, dest_type)
    state, speeds, offsets, truth = initial_states_xy(scenes, obs_length, pred_length, dest_type, dest_dict)
    return to_device(state, speeds, offsets, truth, scenes=scenes, device=device)


def scene_paths(scene):
    """Track rows of a scene held as an xy array (frame = row index), for the per-scene predictors."""
    if not isinstance(scene, np.ndarray):
        return scene
    paths = []
    for j in range(scene.shape[1]):
        t = np.nonzero(~np.isnan(scene[:, j, 0]))[0]
        paths.append([data.TrackRow(int(f), j, float(scene[f, j, 0]), float(scene[f, j, 1])) for f in t])
    return paths


def score(truth, pred):
    """(ADE, FDE) of one predicted primary [pred_length, 2] against its truth, in the sweep kernels' order:
    distances summed sequentially in float64, ADE = sum / n, FDE = the last distance."""
    d = np.sqrt((truth[:, 0] - pred[:, 0]) * (truth[:, 0] - pred[:, 0]) + (truth[:, 1] - pred[:, 1]) * (truth[:, 1] - pred[:, 1]))
    s = 0.0
    for v in d:
        s += float(v)
    return s / len(d), float(d[-1])


def _mean(values):
    """Evaluator.aggregate's mean: sequential sum over the scenes / N (NaN propagates)."""
    s = 0.0
    for v in values:
        s += float(v)
    return s / len(values)


def evaluate(prepared, simulator='all', sf_params=SF_DEFAULT, orca_params=ORCA_DEFAULT, dest_type='interp',
             obs_length=9, kf_samples=5):
    """The reference's table for one file and one setting -> (average_l2, final_l2, nonfinite), dicts keyed as
    Evaluator.result() ('N', 'orca<dest_type>', 'sf<dest_type>', 'kf'); nonfinite[name] = scenes with a non-finite ADE.
    KF runs kalman.predict per scene, like aggregate, drawing from NumPy's global RNG."""
    B = int(prepared.truth.shape[0])
    avg, fin, bad = {'N': B}, {'N': B}, {}
    runs = []
    if simulator in ('all', 'orca'):
        runs.append(('orca' + dest_type, lambda: orca.sweep(prepared, [orca_params])))
    if simulator in ('all', 'sf'):
        runs.append(('sf' + dest_type, lambda: socialforce.sweep(prepared, [sf_params])))
    for name, run in runs:
        ade, fde = (t[0].cpu().numpy() for t in run())
        avg[name], fin[name], bad[name] = _mean(ade), _mean(fde), int((~np.isfinite(ade)).sum())
    if simulator in ('all', 'kalman'):
        if prepared.scenes is None:
            raise ValueError("KF needs the scenes' rows: prepare with sweep.prepare_file")
        truth = prepared.truth.cpu().numpy()
        pred_length = truth.shape[1]
        ade, fde = np.empty(B), np.empty(B)
        for b, (_, scene) in enumerate(prepared.scenes):
            pred = kalman.predict(scene_paths(scene), n_predict=pred_length, obs_length=obs_length,
                                  n_samples=kf_samples)[0][0]
            ade[b], fde[b] = score(truth[b], pred)
        avg['kf'], fin['kf'], bad['kf'] = _mean(ade), _mean(fde), int((~np.isfinite(ade)).sum())
    return avg, fin, bad


def fit(ades, fdes=None):
    """Best setting by mean ADE over the scenes with a finite ADE, per file and pooled over all files' scenes.

    ades: per file an ADE array [P, B_f] (CUDA or numpy) from socialforce.sweep / orca.sweep with the same P settings.
    Returns {'files': [...], 'pooled': {...}}, each {'best': index, 'ade': [P] means, 'fde': [P] means over the same
    scenes (fdes given), 'finite': [P] scene counts, 'skipped': [P] non-finite scenes}.  Ties go to the lowest index; a
    setting without a finite scene never wins."""
    host = lambda t: t.cpu().numpy() if hasattr(t, 'cpu') else np.asarray(t, dtype=np.float64)
    ades = [host(a) for a in ades]
    fdes = [host(f) for f in fdes] if fdes is not None else None

    def one(ade, fde):
        ok = np.isfinite(ade)
        n = ok.sum(axis=1)
        with np.errstate(invalid='ignore', divide='ignore'):
            mean = np.where(ok, ade, 0.0).sum(axis=1) / n
            r = {'ade': mean, 'finite': n, 'skipped': ade.shape[1] - n}
            if fde is not None:
                r['fde'] = np.where(ok, fde, 0.0).sum(axis=1) / n
        r['best'] = int(np.argmin(np.where(n > 0, mean, np.inf))) if (n > 0).any() else None
        return r

    files = [one(a, fdes[i] if fdes is not None else None) for i, a in enumerate(ades)]
    pooled = one(np.concatenate(ades, axis=1), np.concatenate(fdes, axis=1) if fdes is not None else None)
    return {'files': files, 'pooled': pooled}


def _table(title, results, columns):
    lines = ['## ' + title, '{:>30s} |   N  | '.format('') + ' | '.join(c for c, _ in columns)]
    for name, r, bad in results:
        cells = ''.join(' | {:.2f}'.format(r[k]) + (' ({} non-finite)'.format(bad[k]) if bad[k] else '') for _, k in columns)
        lines.append('{:>30s} | {:>4}{}'.format(name, r['N'], cells))
    return '\n'.join(lines)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    parser.add_argument('files', nargs='+', help='ndjson scene files (e.g. DATA_BLOCK/trajdata/train/*.ndjson)')
    parser.add_argument('--obs_length', default=9, type=int, help='observation length')
    parser.add_argument('--pred_length', default=12, type=int, help='prediction length')
    parser.add_argument('--simulator', default='all', choices=('all', 'orca', 'sf', 'kalman'))
    parser.add_argument('--tau', default=[SF_DEFAULT[0]], type=float, nargs='+', help='Tau of Social Force')
    parser.add_argument('--vo', default=[SF_DEFAULT[1]], type=float, nargs='+', help='V0 of Social Force')
    parser.add_argument('--sigma', default=[SF_DEFAULT[2]], type=float, nargs='+', help='sigma of Social Force')
    parser.add_argument('--min_dist', default=[ORCA_DEFAULT[0]], type=float, nargs='+', help='MinNeighDist of ORCA')
    parser.add_argument('--react_time', default=[ORCA_DEFAULT[1]], type=float, nargs='+', help='NeighReactTime of ORCA')
    parser.add_argument('--radius', default=[ORCA_DEFAULT[2]], type=float, nargs='+', help='agent radius of ORCA')
    args = parser.parse_args(argv)

    names = [os.path.basename(f).replace('.ndjson', '') for f in args.files]
    prepared = [prepare_file(f, args.obs_length, args.pred_length) for f in args.files]
    grids = {}
    if args.simulator in ('all', 'sf'):
        grids['sf'] = (socialforce.sweep, list(itertools.product(args.tau, args.vo, args.sigma)), 'tau, v0, sigma')
    if args.simulator in ('all', 'orca'):
        grids['orca'] = (orca.sweep, list(itertools.product(args.min_dist, args.react_time, args.radius)),
                         'min_dist, react_time, radius')
    best = {}
    for sim, (run, grid, labels) in grids.items():
        out = [run(p, grid) for p in prepared]
        f = fit([a for a, _ in out], [d for _, d in out])
        print('## %s: %d settings (%s), best by mean ADE over the scenes with a finite ADE' % (sim.upper(), len(grid), labels))
        for name, r in list(zip(names, f['files'])) + [('pooled', f['pooled'])]:
            b = r['best']
            if b is None:
                print('{:>30s} | no setting with a finite scene'.format(name))
                continue
            print('{:>30s} | {} | ADE {:.4f} | FDE {:.4f} | {} scenes, {} non-finite skipped'.format(
                name, ', '.join('%g' % v for v in grid[b]), r['ade'][b], r['fde'][b], r['finite'][b], r['skipped'][b]))
        print('')
        pb = f['pooled']['best']
        best[sim] = grid[pb if pb is not None else 0]

    results = [(name, *evaluate(p, args.simulator, sf_params=best.get('sf', SF_DEFAULT),
                                orca_params=best.get('orca', ORCA_DEFAULT), obs_length=args.obs_length))
               for name, p in zip(names, prepared)]
    columns = [(c, k) for c, k, s in (('ORCA', 'orcainterp', 'orca'), ('SF', 'sfinterp', 'sf'), ('KF', 'kf', 'kalman'))
               if args.simulator in ('all', s)]
    settings = ', '.join('%s at (%s)' % (s.upper(), ', '.join('%g' % v for v in best[s])) for s in best)
    if settings:
        print('# ' + settings)
    print(_table('Average L2 [m]', [(n, a, bad) for n, a, _, bad in results], columns))
    print('')
    print(_table('Final L2 [m]', [(n, f, bad) for n, _, f, bad in results], columns))


if __name__ == '__main__':
    main()
