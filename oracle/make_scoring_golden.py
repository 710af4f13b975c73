"""Golden data of the prediction scorer (tests/test_scoring.py).  TEST INFRASTRUCTURE.

    python -m oracle.make_scoring_golden       (needs the reference: /root/reference or oracle/_ref)

Writes tests/golden/scoring_golden.npz:
  syn/<case>/*  synthetic scenes already on the primary's prediction frames (ties between modes, NaN and partly present
                neighbours, neighbours at exactly 2 x 0.1 m, 1 / 3 / 50 modes) with the expected per-scene values:
                ADE / FDE per mode (evaluator/eval_utils.py ade / fde), Top-3 (eval_utils.topk_ade / topk_fde), Col-I /
                Col-II (eval_utils.collision on the frames both tracks have), NLL (scipy.stats.gaussian_kde through
                oracle/metrics_oracle.py's skip / clip rules);
  kde/*         sample sets and query points with scipy.stats.gaussian_kde(...).logpdf (NaN where scipy cannot fit one),
                including near-degenerate sets;
  agg/<case>/*  ground-truth and prediction ndjson texts built from DATA_BLOCK scenes with their real tags, and the
                reference's TrajnetEvaluator.aggregate() / result() over them (oracle/metrics_oracle.py standing in for
                trajnetplusplustools.metrics), as a [9, 8] table: rows overall, the 4 categories, the 4 sub-categories;
                columns N, average_l2, final_l2, gt_col, pred_col, topk_ade, topk_fde, nll;
  collision_test/{test,test_private}  the texts of DATA_BLOCK/collision_test.
"""
import json
import os
import sys
import types
from collections import OrderedDict, defaultdict, namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import metrics_oracle as MO  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "scoring_golden.npz")
T = 12
OBS = 9
Row = namedtuple('Row', ['frame', 'pedestrian', 'x', 'y', 'prediction_number', 'scene_id'])
SceneRow = namedtuple('SceneRow', ['scene', 'pedestrian', 'start', 'end', 'fps', 'tag'])
FIELDS = ('N', 'average_l2', 'final_l2', 'gt_col', 'pred_col', 'topk_ade', 'topk_fde', 'nll')


def reference():
    """The reference's evaluator modules with trajnetplusplustools.metrics served by metrics_oracle."""
    from oracle import ref_shim
    ref_shim.import_reference()
    sys.modules['trajnetplusplustools'].metrics = MO
    sys.modules['trajnetplusplustools.metrics'] = MO
    if 'pandas' not in sys.modules:
        try:
            import pandas  # noqa: F401
        except ImportError:
            sys.modules['pandas'] = types.ModuleType('pandas')
    from evaluator import eval_utils, trajnet_evaluator
    return eval_utils, trajnet_evaluator


# ---------------------------------------------------------------------------------------------------------------------
# ndjson: a json.loads restatement of trajnetplusplustools.Reader(..., scene_type='paths')
# ---------------------------------------------------------------------------------------------------------------------
def read_paths(text, limit=None):
    """[(scene_id, paths)] of the first `limit` scenes (all by default) and the scene rows by id."""
    tracks_by_frame = defaultdict(list)
    scenes = OrderedDict()
    for line in text.splitlines():
        if not line.strip():
            continue
        d = json.loads(line)
        if 'track' in d:
            t = d['track']
            tracks_by_frame[t['f']].append(Row(t['f'], t['p'], t['x'], t['y'], t.get('prediction_number'), t.get('scene_id')))
        elif 'scene' in d:
            s = d['scene']
            scenes[s['id']] = SceneRow(s['id'], s['p'], s['s'], s['e'], s.get('fps'), s.get('tag'))
    out = []
    for sid, s in list(scenes.items())[:limit]:
        prim, others = [], OrderedDict()
        for f in range(s.start, s.end + 1):
            for r in tracks_by_frame.get(f, ()):
                if r.pedestrian == s.pedestrian:
                    prim.append(r)
                else:
                    others.setdefault(r.pedestrian, []).append(r)
        out.append((sid, [prim] + list(others.values())))
    return out, scenes


def subset_text(filename, n_scenes):
    """The first n_scenes scene rows of a DATA_BLOCK file and every track row up to their last frame."""
    scenes, tracks = [], []
    with open(filename) as f:
        for line in f:
            d = json.loads(line)
            (scenes if 'scene' in d else tracks).append((d, line.rstrip('\n')))
    scenes = scenes[:n_scenes]
    last = max(d['scene']['e'] for d, _ in scenes)
    return '\n'.join([l for _, l in scenes] + [l for d, l in tracks if d['track']['f'] <= last]) + '\n'


def prediction_text(gt_text, modes, rng, drop_neighbour_of=None):
    """Predictions in the reference writer's format: per scene the primary's last T frames per mode (ground truth plus
    seeded noise, some modes tied) and mode 0 of every neighbour seen before the end of the observation (NaN where it has
    no row); `drop_neighbour_of` = scene index whose last predicted neighbour is left out."""
    lines = []
    for i, (sid, paths) in enumerate(read_paths(gt_text)[0]):
        prim = paths[0]
        frames = [r.frame for r in prim][-T:]
        last_obs = prim[OBS - 1].frame
        lines.append(json.dumps({'scene': {'id': sid, 'p': prim[0].pedestrian, 's': prim[0].frame, 'e': prim[-1].frame,
                                           'fps': 2.5, 'tag': 0}}))
        gt = np.array([[r.x, r.y] for r in prim][-T:])
        for m in range(modes):
            noise = rng.randn(T, 2) * (0.05 + 0.1 * np.arange(T)[:, None] / T) * (1 + m % 4)
            if m > 0 and rng.rand() < 0.2:
                noise = prev                                                           # noqa: F821 -- a tied mode
            prev = noise
            xy = gt + noise
            lines += [json.dumps({'track': {'f': f, 'p': prim[0].pedestrian, 'x': round(float(x), 2), 'y': round(float(y), 2),
                                            'prediction_number': m, 'scene_id': sid}}) for f, (x, y) in zip(frames, xy)]
        neigh = [p for p in paths[1:] if p[0].frame <= last_obs]
        if drop_neighbour_of == i and neigh:
            neigh = neigh[:-1]
        for p in neigh:
            at = {r.frame: (r.x, r.y) for r in p}
            for f in frames:
                x, y = at.get(f, (float('nan'), float('nan')))
                dx, dy = rng.randn(2) * 0.1
                lines.append(json.dumps({'track': {'f': f, 'p': p[0].pedestrian, 'x': round(x + dx, 2), 'y': round(y + dy, 2),
                                                   'prediction_number': 0, 'scene_id': sid}}))
    return '\n'.join(lines) + '\n'


def run_reference(trajnet_evaluator, gt_text, pred_text, disable_collision=False):
    gt, scenes_by_id = read_paths(gt_text)
    pred, _ = read_paths(pred_text)
    indexes, sub_indexes = defaultdict(list), defaultdict(list)
    for sid, s in scenes_by_id.items():
        indexes[s.tag[0]].append(sid)
        for sub in s.tag[1]:
            sub_indexes[sub].append(sid)
    args = types.SimpleNamespace(pred_length=T, obs_length=OBS, disable_collision=disable_collision)
    ev = trajnet_evaluator.TrajnetEvaluator([p for _, p in gt], [sid for sid, _ in gt], [p for _, p in pred], indexes,
                                            sub_indexes, args)
    ev.aggregate()
    metrics, categories, sub_categories = ev.result()
    table = [metrics] + [getattr(categories, n) for n in ('static_scenes', 'linear_scenes', 'forced_non_linear_scenes',
                                                          'non_linear_scenes')]
    table += [getattr(sub_categories, n) for n in ('lf', 'ca', 'grp', 'others')]
    return np.array([[float(getattr(m, f)) for f in FIELDS] for m in table])


# ---------------------------------------------------------------------------------------------------------------------
# synthetic scenes on the prediction frames
# ---------------------------------------------------------------------------------------------------------------------
def synthetic(rng, S, K):
    r2 = lambda a: np.round(a, 2)
    gt = r2(np.cumsum(rng.randn(S, T, 2) * 0.3, axis=1) + rng.randn(S, 1, 2) * 3)
    modes = r2(gt[:, None] + rng.randn(S, K, T, 2) * rng.uniform(0.05, 0.6, (S, K, 1, 1)))
    for s in range(S):
        # ties, but never a timestep whose modes take exactly two distinct positions: such a set lies on a line, and
        # whether its covariance factors is decided by the rounding of the mean (see DESIGN.md section 2)
        if K > 1 and s % 5 == 1:
            t = rng.randint(T)
            modes[s, :, t] = modes[s, 0, t]                                      # a timestep where every mode ties
        if K > 3 and s % 3 == 0:
            modes[s, rng.randint(1, K)] = modes[s, 0]                           # a mode identical to mode 0
    if K > 1:
        modes[0] = modes[0, :1]                                                  # every timestep identical: NLL skipped
        # on the line y = 0: the deviations in y are exactly 0 in any summation order, so the covariance is singular on
        # every implementation (samples exactly on another line are singular or not by the rounding of the mean)
        modes[2, :, :, 1] = 0.0
        modes[4, rng.randint(K), 5] = np.nan                                      # a NaN mode at one timestep
    if K > 3:                                            # with 3 modes the 3 offsets are often equal: a line again
        modes[3, :, :, 1] = gt[3, None, :, 1] + rng.randint(-1, 2, (K, T)) * 0.01       # near-degenerate in y
    gt_off, pr_off, nbs = [0], [0], {'gt': ([], []), 'pred': ([], [])}
    for s in range(S):
        for kind, off in (('gt', gt_off), ('pred', pr_off)):
            n = rng.randint(0, 5)
            for j in range(n):
                xy = modes[s, 0] + rng.randn(1, 2) * 0.4 + rng.randn(T, 2) * 0.05
                if j == 0 and s % 4 == 0:
                    xy = modes[s, 0] + np.array([0.2, 0.0])                      # exactly at the collision distance
                xy = r2(xy)
                mask = np.ones(T, dtype=np.uint8)
                style = rng.randint(5)
                if style == 1:
                    mask[:rng.randint(1, T)] = 0                                  # enters late
                elif style == 2:
                    mask[rng.randint(1, T):] = 0                                  # leaves early
                elif style == 3:
                    xy[rng.randint(T):] = np.nan                                  # rows with NaN coordinates
                elif style == 4:
                    mask[rng.rand(T) < 0.4] = 0                                   # gaps
                xy[mask == 0] = np.nan
                nbs[kind][0].append(xy)
                nbs[kind][1].append(mask)
            off.append(off[-1] + n)
        if s == 5:
            pr_off[-1] = pr_off[-2] + 0                                           # no predicted neighbour at all
            del nbs['pred'][0][pr_off[-1]:], nbs['pred'][1][pr_off[-1]:]
    stack = lambda v, shape, dt: np.array(v, dtype=dt).reshape(shape)
    d = dict(gt_primary=gt, pred_primary=modes, num_modes=np.full(S, K, dtype=np.int32),
             gt_neigh_off=np.array(gt_off, dtype=np.int32), pred_neigh_off=np.array(pr_off, dtype=np.int32),
             gt_neigh=stack(nbs['gt'][0], (-1, T, 2), np.float64), gt_neigh_mask=stack(nbs['gt'][1], (-1, T), np.uint8),
             pred_neigh=stack(nbs['pred'][0], (-1, T, 2), np.float64),
             pred_neigh_mask=stack(nbs['pred'][1], (-1, T), np.uint8))
    return d


def expected(eval_utils, d):
    S, K = d['pred_primary'].shape[:2]
    ade = np.array([[eval_utils.ade(d['pred_primary'][s, m][None], d['gt_primary'][s][None]) for m in range(K)] for s in range(S)])
    fde = np.array([[eval_utils.fde(d['pred_primary'][s, m][None], d['gt_primary'][s][None]) for m in range(K)] for s in range(S)])
    topk_ade = np.array([eval_utils.topk_ade([p[None] for p in d['pred_primary'][s, :3]], d['gt_primary'][s][None]) for s in range(S)])
    topk_fde = np.array([eval_utils.topk_fde([p[None] for p in d['pred_primary'][s, :3]], d['gt_primary'][s][None]) for s in range(S)])

    def col(kind, s):
        off, nb, mask = d[kind + '_neigh_off'], d[kind + '_neigh'], d[kind + '_neigh_mask']
        prim = d['pred_primary'][s, 0]
        for j in range(off[s], off[s + 1]):
            keep = mask[j] == 1                                                   # the frames both tracks have
            if keep.any() and eval_utils.collision(prim[keep], nb[j][keep]):
                return 1
        return 0
    col_gt = np.array([col('gt', s) for s in range(S)], dtype=np.int32)
    col_pred = np.array([col('pred', s) for s in range(S)], dtype=np.int32)
    nll = np.full(S, np.nan)
    for s in range(S):
        kept = [MO.timestep_logpdf(d['pred_primary'][s, :, t], d['gt_primary'][s, t]) for t in range(T)]
        kept = [v for v in kept if v is not None]
        if kept:
            nll[s] = -(sum(kept) / len(kept))
    return dict(ade=ade, fde=fde, topk_ade=topk_ade, topk_fde=topk_fde, col_gt=col_gt, col_pred=col_pred, nll=nll)


def kde_cases(rng):
    sets, points = [], []
    for K in (3, 4, 10, 50, 50, 50):
        sets.append(np.round(rng.randn(K, 2) * rng.uniform(0.1, 2.0), 2))
        points.append(np.round(rng.randn(2), 2))
    base = np.round(rng.randn(50, 2), 2)
    sets.append(np.stack([base[:, 0], base[:, 0] * 0.5 + 0.01 * rng.randint(-1, 2, 50)], axis=1))    # almost a line
    points.append(np.array([0.1, 0.05]))
    sets.append(np.stack([base[:, 0], np.zeros(50)], axis=1))                                         # y = 0: singular
    points.append(np.array([0.0, 0.0]))
    sets.append(np.concatenate([np.zeros((48, 2)), [[0.01, 0.0], [0.0, 0.01]]]))                     # two points apart
    points.append(np.array([0.0, 0.0]))
    sets.append(np.round(rng.randn(50, 2) * 0.02, 2))                                                  # many ties
    points.append(np.array([5.0, -5.0]))                                                               # far: clipped
    Kmax = max(len(s) for s in sets)
    samples = np.full((len(sets), Kmax, 2), np.nan)
    for i, s in enumerate(sets):
        samples[i, :len(s)] = s
    logpdf = np.array([np.nan if (v := MO.kde_logpdf(s, p)) is None else v for s, p in zip(sets, points)])
    return dict(samples=samples, count=np.array([len(s) for s in sets], dtype=np.int32), point=np.array(points), logpdf=logpdf)


def main():
    from oracle.ref_shim import reference_root
    eval_utils, trajnet_evaluator = reference()
    rng = np.random.RandomState(2024)
    out = {}
    for case, (S, K) in (('modes1', (24, 1)), ('modes3', (24, 3)), ('modes50', (12, 50))):
        d = synthetic(rng, S, K)
        for k, v in d.items():
            out['syn/%s/%s' % (case, k)] = v
        for k, v in expected(eval_utils, d).items():
            out['syn/%s/expect_%s' % (case, k)] = v
    for k, v in kde_cases(rng).items():
        out['kde/' + k] = v
    data = os.path.join(reference_root(), 'DATA_BLOCK')
    texts = {'zara': subset_text(os.path.join(data, 'trajdata', 'train', 'crowds_zara01.ndjson'), 60),
             'zara_small': subset_text(os.path.join(data, 'trajdata', 'train', 'crowds_zara01.ndjson'), 14),
             'hotel': subset_text(os.path.join(data, 'trajdata', 'train', 'biwi_hotel.ndjson'), 40)}
    cases = (('zara_modes1_mismatch', 'zara', 1, 30, False), ('zara_modes1_nocol', 'zara', 1, 30, True),
             ('zara_modes3', 'zara', 3, None, False), ('hotel_modes1', 'hotel', 1, None, False),
             ('zara_modes50', 'zara_small', 50, None, False))
    for case, gt_name, modes, drop, nocol in cases:
        gt_text = texts[gt_name]
        pred_text = prediction_text(gt_text, modes, np.random.RandomState(len(case) * 7 + modes), drop_neighbour_of=drop)
        out['agg/%s/gt' % case] = np.frombuffer(gt_text.encode(), dtype=np.uint8)
        out['agg/%s/pred' % case] = np.frombuffer(pred_text.encode(), dtype=np.uint8)
        out['agg/%s/disable_collision' % case] = np.array(nocol)
        out['agg/%s/result' % case] = run_reference(trajnet_evaluator, gt_text, pred_text, disable_collision=nocol)
    for part in ('test', 'test_private'):
        with open(os.path.join(data, 'collision_test', part, 'collision_test.ndjson'), 'rb') as f:
            out['collision_test/' + part] = np.frombuffer(f.read(), dtype=np.uint8)
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
