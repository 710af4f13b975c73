"""Fit social-force parameters (tau, v0, sigma) by gradient, on the device.

The sweep tool (classical.sweep) finds the best cell of a grid; this module starts from the best cells of such a grid
and runs L-BFGS-B on the mean ADE (or FDE) with its exact gradient: one tb2_sf_sweep_grad launch per file and
function evaluation returns every scene's ADE / FDE with d/d(tau, v0, sigma), carried through the rollout in forward
mode (socialforce.sweep_grad).

    python -m trajnetplusplusbaselines_b200.classical.fit FILES... --tau 0.3 0.5 --vo 1.0 2.1 --sigma 0.2 0.3

The objective is sweep.fit's: the mean over the scenes with a finite ADE at the start setting, a scene set then held
fixed; an iterate at which one of those scenes is non-finite scores +inf, so the line search backs off.  Fits run per
file and pooled over all files.  The fitted setting is reported through socialforce.sweep, the value path, and the
reference's SF table (sweep.evaluate) is printed at the pooled fit.
"""
import argparse
import itertools
import os

import numpy as np

from . import socialforce, sweep

OBJECTIVES = ('ade', 'fde')
LOWER = (1e-6, 0.0, 1e-6)             # tau > 0, v0 >= 0, sigma > 0 (tb2_sf_sweep refuses tau, sigma <= 0)


def _host(t):
    return t.cpu().numpy() if hasattr(t, 'cpu') else np.asarray(t, dtype=np.float64)


def device_values(prepared, settings):
    """(ade, fde) numpy [P, B] of socialforce.sweep."""
    return tuple(_host(t) for t in socialforce.sweep(prepared, settings))


def device_grads(prepared, theta):
    """(ade [B], fde [B], dade [B, 3], dfde [B, 3]) numpy of one socialforce.sweep_grad launch at theta."""
    return tuple(_host(t)[0] for t in socialforce.sweep_grad(prepared, [theta]))


class Objective:
    """Mean ADE (objective 'ade') or FDE of the scenes of several prepared files with a finite ADE at theta0, and its
    gradient; grads(prepared, theta) is device_grads or a stand-in.  Calling it returns (value, gradient [3]); value
    +inf when a counted scene is non-finite.  Keeps the best finite point it has evaluated."""

    def __init__(self, prepared, theta0, objective='ade', grads=device_grads):
        if objective not in OBJECTIVES:
            raise ValueError("objective must be one of %s" % (OBJECTIVES,))
        self.prepared, self.objective, self.grads = list(prepared), objective, grads
        ades = [grads(p, tuple(theta0))[0] for p in self.prepared]
        self.masks = [np.isfinite(a) for a in ades]
        self.used = int(sum(m.sum() for m in self.masks))
        self.skipped = int(sum(len(m) for m in self.masks)) - self.used
        self.nfev = 0
        self.best = (np.inf, np.asarray(theta0, dtype=np.float64))
        self.bad = None                      # the last non-finite point evaluated

    def __call__(self, theta):
        theta = np.asarray(theta, dtype=np.float64)
        self.nfev += 1
        k = 0 if self.objective == 'ade' else 1
        outs = [self.grads(p, tuple(float(v) for v in theta)) for p in self.prepared]
        m = np.concatenate(self.masks)
        v = np.concatenate([o[k] for o in outs])
        d = np.concatenate([o[2 + k] for o in outs])
        if self.used == 0 or not (np.isfinite(v[m]).all() and np.isfinite(d[m]).all()):
            self.bad = theta.copy()
            return np.inf, np.zeros(3)
        value = masked_mean(v, m)
        if value < self.best[0]:
            self.best = (value, theta.copy())
        return value, np.where(m[:, None], d, 0.0).sum(axis=0) / self.used


def masked_mean(v, m):
    """sweep.fit's mean of v [B] over the scenes m [B]: a row sum with zeros elsewhere, over the count."""
    return float(np.where(m, v, 0.0)[None].sum(axis=1)[0] / m.sum())


def minimize(objective, theta0, max_iter=100, restarts=10):
    """L-BFGS-B from theta0 within LOWER -> (theta, value, nit).  SciPy's L-BFGS-B stops at the first +inf it meets;
    each time it does, the search restarts from the best point within a box of half the distance to the non-finite
    point, so it backs off from the region.  The best evaluated point is kept: the result is never worse than theta0."""
    from scipy.optimize import minimize as sp_minimize
    objective(theta0)
    radius, nit = np.inf, 0
    for _ in range(restarts + 1):
        x = objective.best[1]
        objective.bad = None
        bounds = [(max(lo, xi - radius), xi + radius if np.isfinite(radius) else None) for lo, xi in zip(LOWER, x)]
        res = sp_minimize(objective, x, jac=True, method='L-BFGS-B', bounds=bounds,
                          options={'maxiter': max(1, int(max_iter) - nit)})
        nit += int(res.nit)
        if objective.bad is None or nit >= max_iter:
            break
        radius = 0.5 * float(np.abs(objective.bad - objective.best[1]).max())
    value, theta = objective.best
    return theta, value, nit


def _starts(r, objective, k):
    """Indices of the k best grid cells of one sweep.fit entry by the objective's means (cells with a finite scene)."""
    mean = np.where(r['finite'] > 0, r[objective], np.inf)
    order = [int(i) for i in np.argsort(mean, kind='stable') if np.isfinite(mean[i])]
    return order[:k]


def fit_group(prepared, grid, fitted_cells, objective='ade', starts=1, max_iter=100, grads=device_grads,
              values=device_values):
    """One fit over the files `prepared` (a list) from the best `starts` cells of `fitted_cells` (one sweep.fit entry
    over those files) -> dict start / theta (tuples), start_ade / start_fde / ade / fde (socialforce.sweep means over the
    start's scene set), used / skipped scenes, nit / nfev summed over the starts; None without a finite cell."""
    cells = _starts(fitted_cells, objective, starts)
    if not cells:
        return None
    best, nit, nfev = None, 0, 0
    for c in cells:
        obj = Objective(prepared, grid[c], objective, grads)
        theta, value, it = minimize(obj, np.asarray(grid[c], dtype=np.float64), max_iter)
        nit, nfev = nit + it, nfev + obj.nfev
        if best is None or value < best[1]:
            best = (c, value, theta, obj)
    c, _, theta, obj = best
    r = {'start': tuple(float(v) for v in grid[c]), 'theta': tuple(float(v) for v in theta), 'used': obj.used,
         'skipped': obj.skipped, 'nit': nit, 'nfev': nfev}
    m = np.concatenate(obj.masks)
    for key, setting in (('start_', r['start']), ('', r['theta'])):
        outs = [values(p, [setting]) for p in prepared]
        r[key + 'ade'] = masked_mean(np.concatenate([a[0] for a, _ in outs]), m)
        r[key + 'fde'] = masked_mean(np.concatenate([f[0] for _, f in outs]), m)
    return r


def fit(prepared, grid, objective='ade', starts=1, max_iter=100, grads=device_grads, values=device_values):
    """Per file and pooled fits from a grid of settings [(tau, v0, sigma)] -> {'files': [...], 'pooled': ...}, each
    fit_group's dict (or None), plus 'grid': sweep.fit's result over the grid."""
    outs = [values(p, grid) for p in prepared]
    cells = sweep.fit([a for a, _ in outs], [f for _, f in outs])
    files = [fit_group([p], grid, r, objective, starts, max_iter, grads, values)
             for p, r in zip(prepared, cells['files'])]
    pooled = fit_group(prepared, grid, cells['pooled'], objective, starts, max_iter, grads, values)
    return {'files': files, 'pooled': pooled, 'grid': cells}


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    parser.add_argument('files', nargs='+', help='ndjson scene files (e.g. DATA_BLOCK/trajdata/train/*.ndjson)')
    parser.add_argument('--obs_length', default=9, type=int, help='observation length')
    parser.add_argument('--pred_length', default=12, type=int, help='prediction length')
    parser.add_argument('--tau', default=[sweep.SF_DEFAULT[0]], type=float, nargs='+', help='Tau of Social Force')
    parser.add_argument('--vo', default=[sweep.SF_DEFAULT[1]], type=float, nargs='+', help='V0 of Social Force')
    parser.add_argument('--sigma', default=[sweep.SF_DEFAULT[2]], type=float, nargs='+', help='sigma of Social Force')
    parser.add_argument('--starts', default=1, type=int, help='fits from the best K cells of the grid')
    parser.add_argument('--objective', default='ade', choices=OBJECTIVES, help='mean ADE or mean FDE')
    parser.add_argument('--max_iter', default=100, type=int, help='L-BFGS-B iterations per start')
    args = parser.parse_args(argv)
    if args.starts < 1 or args.max_iter < 1:
        parser.error('--starts and --max_iter must be >= 1')
    return args


def _setting(t):
    return ', '.join('%.4g' % v for v in t)


def main(argv=None):
    args = parse_args(argv)
    names = [os.path.basename(f).replace('.ndjson', '') for f in args.files]
    prepared = [sweep.prepare_file(f, args.obs_length, args.pred_length) for f in args.files]
    grid = list(itertools.product(args.tau, args.vo, args.sigma))
    f = fit(prepared, grid, args.objective, args.starts, args.max_iter)
    print('## SF fit: mean %s by L-BFGS-B from the best %d of %d grid settings (tau, v0, sigma)'
          % (args.objective.upper(), args.starts, len(grid)))
    for name, r in list(zip(names, f['files'])) + [('pooled', f['pooled'])]:
        if r is None:
            print('{:>30s} | no setting with a finite scene'.format(name))
            continue
        print('{:>30s} | start {} | ADE {:.4f} | FDE {:.4f}'.format(name, _setting(r['start']), r['start_ade'],
                                                                  r['start_fde']))
        print('{:>30s} | fit   {} | ADE {:.4f} | FDE {:.4f} | {} scenes, {} skipped | {} iterations, {} evaluations'
              .format('', _setting(r['theta']), r['ade'], r['fde'], r['used'], r['skipped'], r['nit'], r['nfev']))
    print('')
    theta = f['pooled']['theta'] if f['pooled'] is not None else sweep.SF_DEFAULT
    results = [(name, *sweep.evaluate(p, 'sf', sf_params=theta, obs_length=args.obs_length))
               for name, p in zip(names, prepared)]
    print('# SF at (%s)' % _setting(theta))
    print(sweep._table('Average L2 [m]', [(n, a, bad) for n, a, _, bad in results], [('SF', 'sfinterp')]))
    print('')
    print(sweep._table('Final L2 [m]', [(n, fi, bad) for n, _, fi, bad in results], [('SF', 'sfinterp')]))
    return f


if __name__ == '__main__':
    main()
