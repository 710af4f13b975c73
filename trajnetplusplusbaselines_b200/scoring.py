"""Scoring of TrajNet++ prediction files: the metric half of the reference's evaluator (evaluator/trajnet_evaluator.py,
evaluator/evaluator_helpers.py) with the per-scene metrics computed by one CUDA launch per file (csrc/metrics.cu,
tb2_score_scenes).

    metrics, categories, sub_categories = score_file('test_private/x.ndjson', 'test_pred/model_modes1/x.ndjson')

The host side reads both files (csrc/ndjson.cu tb2_ndjson_parse_meta, json.loads for a file the native parser refuses)
and assembles what TrajnetEvaluator.aggregate reads from trajnetplusplustools.Reader(..., scene_type='paths'): scenes
paired by position in the files, prediction rows filtered by scene_id, every track placed on the ground truth's last
pred_length frames of the primary with a presence mask.  The accumulation over scenes (categories, the Col-I rule, Top-3
and NLL switched by the number of predicted modes) follows aggregate scene by scene.
"""
import ctypes
import dataclasses
import json
import os
from dataclasses import dataclass, field

import numpy as np

from . import _lib

CATEGORY_FIELDS = ('static_scenes', 'linear_scenes', 'forced_non_linear_scenes', 'non_linear_scenes')    # tag 1..4
SUB_CATEGORY_FIELDS = ('lf', 'ca', 'grp', 'others')                                                   # sub-tag 1..4
TOPK = 3                        # Top-3 ADE / FDE over modes 0..2
TOPK_MIN_PREDICTIONS = 1        # Top-k is scored when the file holds more than this prediction_number
NLL_MIN_PREDICTIONS = 48        # NLL likewise


@dataclass
class Metrics:
    """Sums over scenes (average_l2 = ADE, final_l2 = FDE, gt_col = Col-II, pred_col = Col-I, -1 once the neighbour counts
    of a scene differ); avg_vals() turns them into means, the collisions into percentages."""
    N: int = 0
    average_l2: float = 0
    final_l2: float = 0
    gt_col: float = 0
    pred_col: float = 0
    topk_ade: float = 0
    topk_fde: float = 0
    nll: float = 0

    def __iadd__(self, other):
        for name in ('N', 'average_l2', 'final_l2', 'gt_col', 'topk_ade', 'topk_fde', 'nll'):
            setattr(self, name, getattr(self, name) + getattr(other, name))
        self.pred_col = -1 if -1 in (self.pred_col, other.pred_col) else self.pred_col + other.pred_col
        return self

    def avg_vals(self):
        if self.N == 0:
            return
        n = self.N
        self.average_l2 /= n
        self.final_l2 /= n
        self.gt_col /= 0.01 * n
        if self.pred_col != -1:
            self.pred_col /= 0.01 * n
        self.topk_ade /= n
        self.topk_fde /= n
        self.nll /= n

    def to_list(self):
        return [self.N, self.average_l2, self.final_l2, self.pred_col, self.gt_col, self.topk_ade, self.topk_fde, self.nll]

    def avg_vals_to_list(self):
        self.avg_vals()
        return self.to_list()


@dataclass
class Categories:
    static_scenes: Metrics = field(default_factory=Metrics)
    linear_scenes: Metrics = field(default_factory=Metrics)
    forced_non_linear_scenes: Metrics = field(default_factory=Metrics)
    non_linear_scenes: Metrics = field(default_factory=Metrics)


@dataclass
class Sub_categories:  # noqa: N801 -- the reference's name
    lf: Metrics = field(default_factory=Metrics)
    ca: Metrics = field(default_factory=Metrics)
    grp: Metrics = field(default_factory=Metrics)
    others: Metrics = field(default_factory=Metrics)


# ----------------------------------------------------------------------------------------------------------------------
# Reading
# ----------------------------------------------------------------------------------------------------------------------
def _parse_meta_native(text):
    """Columns of parse_ndjson_meta through tb2_ndjson_parse_meta, or None when it refuses a line."""
    max_rows = text.count(b'\n') + 1
    i64 = lambda: np.empty(max_rows, dtype=np.int64)
    cols = dict(frame=i64(), ped=i64(), x=np.empty(max_rows), y=np.empty(max_rows), prediction_number=i64(),
                track_scene_id=i64(), scene_id=i64(), scene_ped=i64(), scene_start=i64(), scene_end=i64(),
                scene_tag=i64(), scene_subs=i64())
    counts = np.zeros(3, dtype=np.int64)                    # tracks, scenes, refused line
    ptr = lambda a: ctypes.c_void_p(a.ctypes.data)
    _lib.check(_lib.load().tb2_ndjson_parse_meta(
        ctypes.cast(ctypes.c_char_p(text), ctypes.c_void_p), len(text), max_rows,
        ptr(cols['frame']), ptr(cols['ped']), ptr(cols['x']), ptr(cols['y']), ptr(cols['prediction_number']),
        ptr(cols['track_scene_id']), ptr(counts[0:1]), ptr(cols['scene_id']), ptr(cols['scene_ped']),
        ptr(cols['scene_start']), ptr(cols['scene_end']), ptr(cols['scene_tag']), ptr(cols['scene_subs']),
        ptr(counts[1:2]), ptr(counts[2:3])))
    if counts[2] >= 0:
        return None
    nt, ns = int(counts[0]), int(counts[1])
    return {k: (v[:ns] if k.startswith('scene_') else v[:nt]) for k, v in cols.items()}


def parse_ndjson_meta(filename, native=True):
    """Columns of an ndjson file with the metadata the scorer reads: track rows (frame, ped, x, y, prediction_number,
    scene_id; -1 where absent) in file order and scene rows (scene_id, scene_ped, scene_start, scene_end, scene_tag = main
    type or -1, scene_subs = bitmask of the sub-types).  The native parser reads the file; where it refuses a line the
    whole file goes through json.loads, which gives the same columns."""
    with open(filename, 'rb') as f:
        text = f.read()
    cols = _parse_meta_native(text) if native else None
    if cols is not None:
        return cols
    tracks, scenes = [], []
    lines = [line for line in text.decode().splitlines() if line.strip()]
    for d in json.loads('[' + ','.join(lines) + ']') if lines else ():
        if 'track' in d:
            t = d['track']
            pn, sid = t.get('prediction_number'), t.get('scene_id')
            tracks.append((t['f'], t['p'], t['x'], t['y'], -1 if pn is None else pn, -1 if sid is None else sid))
        elif 'scene' in d:
            s = d['scene']
            tag = s.get('tag')
            if tag is None:
                main, subs = -1, 0
            elif isinstance(tag, int):
                main, subs = tag, 0
            else:
                main, subs = tag[0], sum(1 << k for k in set(tag[1]))
            scenes.append((s['id'], s['p'], s['s'], s['e'], main, subs))
    tr = np.array(tracks, dtype=object).reshape(-1, 6)
    sc = np.array(scenes, dtype=np.int64).reshape(-1, 6)
    out = {k: tr[:, i].astype(np.int64) for i, k in enumerate(('frame', 'ped'))}
    out.update(x=tr[:, 2].astype(np.float64), y=tr[:, 3].astype(np.float64), prediction_number=tr[:, 4].astype(np.int64),
               track_scene_id=tr[:, 5].astype(np.int64))
    out.update({k: sc[:, i].copy() for i, k in enumerate(('scene_id', 'scene_ped', 'scene_start', 'scene_end', 'scene_tag',
                                                          'scene_subs'))})
    return out


class SceneReader:
    """trajnetplusplustools.Reader(..., scene_type='paths') over parsed columns: scenes keyed by id in order of first
    appearance (a repeated id keeps its first position and its last row), the rows of a scene are those with a frame in
    [start, end], by frame and in file order within a frame."""

    def __init__(self, cols):
        sid = cols['scene_id']
        _, first = np.unique(sid, return_index=True)
        _, last_rev = np.unique(sid[::-1], return_index=True)
        rows = (len(sid) - 1 - last_rev)[np.argsort(first, kind='stable')]
        self.scene_id, self.ped = sid[rows], cols['scene_ped'][rows]
        self.tag, self.subs = cols['scene_tag'][rows], cols['scene_subs'][rows]
        order = np.argsort(cols['frame'], kind='stable')
        self.f = cols['frame'][order]
        self.p = cols['ped'][order]
        self.xy = np.stack([cols['x'][order], cols['y'][order]], axis=1)
        self.pn = cols['prediction_number'][order]
        self.sid = cols['track_scene_id'][order]
        self.lo = np.searchsorted(self.f, cols['scene_start'][rows], side='left')
        self.hi = np.searchsorted(self.f, cols['scene_end'][rows], side='right')

    def __len__(self):
        return len(self.scene_id)

    def window(self, i):
        return slice(int(self.lo[i]), int(self.hi[i]))


def tracks_on_frames(frames, peds, xy, keep_peds, want):
    """[len(keep_peds), len(want), 2] positions + [.., len(want)] masks of the rows of each pedestrian in keep_peds."""
    n, T = len(keep_peds), len(want)
    nb = np.full((n, T, 2), np.nan)
    mask = np.zeros((n, T), dtype=np.uint8)
    if n == 0 or T == 0 or len(frames) == 0:
        return nb, mask
    order = np.argsort(keep_peds, kind='stable')
    j = np.minimum(np.searchsorted(keep_peds[order], peds), n - 1)
    t = np.minimum(np.searchsorted(want, frames), T - 1)
    ok = (keep_peds[order][j] == peds) & (want[t] == frames)
    nb[order[j[ok]], t[ok]] = xy[ok]
    mask[order[j[ok]], t[ok]] = 1
    return nb, mask


def first_appearance(frames, peds, exclude):
    """Pedestrians other than `exclude` in order of first appearance (trajnetplusplustools track_rows_to_paths), with the
    frame of their first row."""
    idx = np.flatnonzero(peds != exclude)
    uniq, first = np.unique(peds[idx], return_index=True)
    order = np.argsort(first, kind='stable')
    return uniq[order], frames[idx[first[order]]]


def assemble(gt_file, pred_file, obs_length=9, pred_length=12):
    """The arrays tb2_score_scenes reads, for the scenes of gt_file paired by position with those of pred_file.
    Raises Exception('frame numbers are not consistent') where mode 0 of a scene's primary is not on the ground truth's
    last pred_length frames."""
    gt, pr = SceneReader(parse_ndjson_meta(gt_file)), SceneReader(parse_ndjson_meta(pred_file))
    S, T = len(gt), pred_length
    if len(pr) < S:
        raise IndexError('%s: %d scenes, the ground truth has %d' % (pred_file, len(pr), S))
    num_predictions = 0
    if S:
        w = pr.window(0)
        pn0 = pr.pn[w][pr.p[w] == pr.ped[0]]
        num_predictions = max(0, int(pn0.max())) if len(pn0) else 0
    gt_prim = np.empty((S, T, 2))
    modes_per_scene = []
    n_modes = np.empty(S, dtype=np.int32)
    gt_nb, gt_mask, pr_nb, pr_mask = [], [], [], []
    gt_count, pr_count = np.zeros(S, dtype=np.int32), np.zeros(S, dtype=np.int32)
    for i in range(S):
        w = gt.window(i)
        f, p, xy = gt.f[w], gt.p[w], gt.xy[w]
        prim = p == gt.ped[i]
        pf = f[prim]
        frame_gt = pf[-T:]
        # prediction side: rows of the paired scene that carry this scene's id
        v = pr.window(i)
        keep = pr.sid[v] == gt.scene_id[i]
        qf, qp, qxy, qn = pr.f[v][keep], pr.p[v][keep], pr.xy[v][keep], pr.pn[v][keep]
        qprim = qp == pr.ped[i]
        m0 = qprim & (qn == 0)
        if len(frame_gt) != T or not np.array_equal(qf[m0], frame_gt):
            raise Exception('frame numbers are not consistent')
        gt_prim[i] = xy[prim][-T:]
        K = int(qn[qprim].max()) + 1
        n_modes[i] = K
        modes = np.full((K, T, 2), np.nan)
        sel = qprim & (qn >= 0)
        k = np.minimum(np.searchsorted(frame_gt, qf[sel]), T - 1)
        hit = frame_gt[k] == qf[sel]
        modes[qn[sel][hit], k[hit]] = qxy[sel][hit]
        modes_per_scene.append(modes)
        # ground-truth neighbours that appear before the end of the observation (drop_post_obs)
        peds, first_frame = first_appearance(f, p, gt.ped[i])
        peds = peds[first_frame < pf[obs_length]]
        nb, mask = tracks_on_frames(f, p, xy, peds, frame_gt)
        gt_nb.append(nb)
        gt_mask.append(mask)
        gt_count[i] = len(peds)
        # predicted neighbours (every pedestrian with a row of this scene), mode 0 on the same frames
        qpeds = first_appearance(qf, qp, pr.ped[i])[0]
        sel = qn == 0
        nb, mask = tracks_on_frames(qf[sel], qp[sel], qxy[sel], qpeds, frame_gt)
        pr_nb.append(nb)
        pr_mask.append(mask)
        pr_count[i] = len(qpeds)
    K = int(n_modes.max()) if S else 1
    pred_prim = np.full((S, K, T, 2), np.nan)
    for i, modes in enumerate(modes_per_scene):
        pred_prim[i, :len(modes)] = modes
    cat = lambda parts, shape, dt: np.concatenate(parts) if parts else np.empty(shape, dtype=dt)
    off = lambda c: np.concatenate([[0], np.cumsum(c)]).astype(np.int32)
    main = np.zeros(S, dtype=np.int64)
    subs = np.zeros(S, dtype=np.int64)
    # categories by scene id over ALL scene rows of the ground truth (Reader.scenes_by_id), first key 1..4
    tag_of = dict(zip(gt.scene_id.tolist(), zip(gt.tag.tolist(), gt.subs.tolist())))
    for i in range(S):
        main[i], subs[i] = tag_of[int(gt.scene_id[i])]
    return dict(num_predictions=num_predictions, gt_primary=gt_prim, pred_primary=pred_prim, num_modes=n_modes,
                gt_neigh_off=off(gt_count), gt_neigh=cat(gt_nb, (0, T, 2), np.float64), gt_neigh_mask=cat(gt_mask, (0, T), np.uint8),
                pred_neigh_off=off(pr_count), pred_neigh=cat(pr_nb, (0, T, 2), np.float64),
                pred_neigh_mask=cat(pr_mask, (0, T), np.uint8), scene_id=gt.scene_id.copy(), tag=main, subs=subs)


# ----------------------------------------------------------------------------------------------------------------------
# Scoring
# ----------------------------------------------------------------------------------------------------------------------
def score_arrays(a, with_nll):
    """One tb2_score_scenes launch over assembled arrays -> dict(ade, fde [S, K] per mode, nll [S], flags [S]).

    `a` holds gt_primary [S, T, 2], pred_primary [S, K, T, 2], num_modes [S] (1..K), {gt,pred}_neigh_off [S + 1]
    (non-decreasing from 0), {gt,pred}_neigh [N, T, 2] and {gt,pred}_neigh_mask [N, T] with N = the last offset.  The
    arrays are converted to the dtypes the kernel reads (float64 / int32 / uint8); a shape that does not fit raises."""
    import torch
    _lib.require_cuda()
    pred_primary = np.asarray(a['pred_primary'], dtype=np.float64)
    if pred_primary.ndim != 4 or pred_primary.shape[3] != 2:
        raise ValueError('pred_primary must be [S, K, T, 2], got %s' % (pred_primary.shape,))
    S, K, T = pred_primary.shape[:3]
    cast = dict(gt_primary=((S, T, 2), np.float64), pred_primary=((S, K, T, 2), np.float64), num_modes=((S,), np.int32),
                gt_neigh_off=((S + 1,), np.int32), pred_neigh_off=((S + 1,), np.int32))
    arrays = {}
    for k, (shape, dt) in cast.items():
        v = np.asarray(a[k])
        if v.shape != shape:
            raise ValueError('%s must have shape %s, got %s' % (k, shape, v.shape))
        arrays[k] = np.ascontiguousarray(v, dtype=dt)
    if S and ((arrays['num_modes'] < 1) | (arrays['num_modes'] > K)).any():
        raise ValueError('num_modes must be in 1..%d' % K)
    for kind in ('gt', 'pred'):
        off = arrays[kind + '_neigh_off']
        if off[0] != 0 or (np.diff(off) < 0).any():
            raise ValueError('%s_neigh_off must start at 0 and not decrease' % kind)
        n = int(off[-1])
        for k, shape, dt in ((kind + '_neigh', (n, T, 2), np.float64), (kind + '_neigh_mask', (n, T), np.uint8)):
            v = np.asarray(a[k])
            if v.shape != shape:
                raise ValueError('%s must have shape %s, got %s' % (k, shape, v.shape))
            arrays[k] = np.ascontiguousarray(v, dtype=dt)
    dev = torch.device('cuda', torch.cuda.current_device())
    ins = {k: torch.from_numpy(v).to(dev) for k, v in arrays.items()}          # torch allocations are 512-byte aligned
    ade = torch.empty((S, K), dtype=torch.float64, device=dev)
    fde = torch.empty_like(ade)
    nll = torch.empty(S, dtype=torch.float64, device=dev)
    flags = torch.empty(S, dtype=torch.int32, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(_lib.load().tb2_score_scenes(
        S, T, K, p(ins['gt_primary']), p(ins['pred_primary']), p(ins['num_modes']), p(ins['gt_neigh_off']), p(ins['gt_neigh']),
        p(ins['gt_neigh_mask']), p(ins['pred_neigh_off']), p(ins['pred_neigh']), p(ins['pred_neigh_mask']), 1 if with_nll else 0,
        p(ade), p(fde), p(nll), p(flags), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    out = dict(ade=ade.cpu().numpy(), fde=fde.cpu().numpy(), flags=flags.cpu().numpy())
    out['nll'] = nll.cpu().numpy() if with_nll else np.full(S, np.nan)
    return out


def score_scenes(gt_file, pred_file, obs_length=9, pred_length=12):
    """Per-scene records of a prediction file: (assembled arrays, dict(ade, fde [S, K] per mode, nll [S], flags [S] of
    _lib.SCORE_* bits)).  NLL is computed when the file's first scene holds more than 48 predictions."""
    a = assemble(gt_file, pred_file, obs_length, pred_length)
    return a, score_arrays(a, a['num_predictions'] > NLL_MIN_PREDICTIONS)


def _topk(values):
    """eval_utils.topk_ade / topk_fde: the smallest value over modes 0..2, 1e10 when none is a number."""
    best = 1e10
    for v in values[:TOPK]:
        if v < best:
            best = float(v)
    return best


def aggregate(a, rec, disable_collision=False):
    """(metrics, categories, sub_categories) of one file from its per-scene records, accumulated scene by scene as
    TrajnetEvaluator.aggregate does.  Col-I: once a scene's neighbour counts differ, Col-I is -1 for the whole file and for
    that scene's categories, and no further Col-I collision is counted."""
    S = len(a['scene_id'])
    metrics = Metrics(S, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
    score = {k: Metrics() for k in range(1, 5)}
    sub_score = {k: Metrics() for k in range(1, 5)}
    num_predictions = a['num_predictions']
    enable_col1 = True
    totals = dict(average_l2=0.0, final_l2=0.0, topk_ade=0.0, topk_fde=0.0, nll=0.0)
    for i in range(S):
        main = int(a['tag'][i])
        if main not in score:
            raise KeyError('scene %d: main type %d is not one of 1..4' % (int(a['scene_id'][i]), main))
        targets = [score[main]] + [sub_score[k] for k in range(1, 5) if (int(a['subs'][i]) >> k) & 1]
        flags = int(rec['flags'][i])
        for m in targets:
            m.N += 1
        if not disable_collision:
            if flags & _lib.SCORE_COL_GT:
                metrics.gt_col += 1
                for m in targets:
                    m.gt_col += 1
            if flags & _lib.SCORE_NEIGH_COUNT_DIFFERS:
                enable_col1 = False
                for m in [metrics] + targets:
                    m.pred_col = -1
            if enable_col1 and flags & _lib.SCORE_COL_PRED:
                for m in [metrics] + targets:
                    m.pred_col += 1
        values = dict(average_l2=float(rec['ade'][i, 0]), final_l2=float(rec['fde'][i, 0]))
        if num_predictions > TOPK_MIN_PREDICTIONS:
            values.update(topk_ade=_topk(rec['ade'][i]), topk_fde=_topk(rec['fde'][i]))
        if num_predictions > NLL_MIN_PREDICTIONS:
            if flags & _lib.SCORE_NLL_ALL_SKIPPED:
                raise Exception('All Predictions are Identical')
            values['nll'] = float(rec['nll'][i])
        for name, v in values.items():
            totals[name] += v
            for m in targets:
                setattr(m, name, getattr(m, name) + v)
    for name, v in totals.items():
        setattr(metrics, name, v)
    return (metrics, Categories(*(score[k] for k in range(1, 5))), Sub_categories(*(sub_score[k] for k in range(1, 5))))


def score_file(gt_file, pred_file, obs_length=9, pred_length=12, disable_collision=False):
    """(metrics, categories, sub_categories) of a prediction file against its ground truth: the result of the reference's
    evaluator.trajnet_evaluator.eval(gt, pred, args) with the per-scene metrics computed on the GPU."""
    a, rec = score_scenes(gt_file, pred_file, obs_length, pred_length)
    return aggregate(a, rec, disable_collision)


def collision_test(list_sub, name, args):
    """The simple collision test of the reference's evaluator: "Fail" when the primary of the first scene of the model's
    collision_test.ndjson collides with its first neighbour, "Pass" otherwise, "NA" without that file."""
    if 'collision_test.ndjson' not in list_sub:
        return "NA"
    r = SceneReader(parse_ndjson_meta(os.path.join(args.path, name, 'collision_test.ndjson')))
    T = args.pred_length
    w = r.window(0)
    f, p, xy = r.f[w], r.p[w], r.xy[w]
    prim = p == r.ped[0]
    frames, prim_xy = f[prim][-T:], xy[prim][-T:]
    if len(frames) != T:
        raise IndexError('collision_test.ndjson: the primary has %d rows, %d needed' % (len(frames), T))
    neigh = first_appearance(f, p, r.ped[0])[0][:1]
    nb, mask = tracks_on_frames(f, p, xy, neigh, frames)
    a = dict(gt_primary=prim_xy[None], pred_primary=prim_xy[None, None], num_modes=np.ones(1, dtype=np.int32),
             gt_neigh_off=np.zeros(2, dtype=np.int32), gt_neigh=np.empty((0, T, 2)), gt_neigh_mask=np.empty((0, T), np.uint8),
             pred_neigh_off=np.array([0, len(neigh)], dtype=np.int32), pred_neigh=nb, pred_neigh_mask=mask)
    return "Fail" if score_arrays(a, False)['flags'][0] & _lib.SCORE_COL_PRED else "Pass"


# ----------------------------------------------------------------------------------------------------------------------
# Table
# ----------------------------------------------------------------------------------------------------------------------
COLUMNS = ('No.', 'ADE', 'FDE', 'Col I', 'Col II', 'Top3 ADE', 'Top3 FDE', 'NLL')
# rows of the results table: (type, sub-type, where the values come from)
TYPE_ROWS = (('I', '', ('categories', 'static_scenes')), ('II', '', ('categories', 'linear_scenes')),
             ('III', '', ('categories', 'forced_non_linear_scenes')), ('III', 'LF', ('sub_categories', 'lf')),
             ('III', 'CA', ('sub_categories', 'ca')), ('III', 'Grp', ('sub_categories', 'grp')),
             ('III', 'Oth', ('sub_categories', 'others')), ('IV', '', ('categories', 'non_linear_scenes')))


def _line(label, cells):
    return '%-24s' % label[:24] + ''.join('%10s' % c for c in cells)


def _cells(values):
    return ['%d' % values[0]] + [format(v, '.2f') for v in values[1:]]


def summarize(results):
    """Sums of per-dataset results {dataset: (metrics, categories, sub_categories)} -> {'overall': Metrics,
    'categories': Categories, 'sub_categories': Sub_categories} (not yet averaged)."""
    total = dict(overall=Metrics(), categories=Categories(), sub_categories=Sub_categories())
    for metrics, categories, sub_categories in results.values():
        total['overall'] += metrics
        for name in CATEGORY_FIELDS:
            getattr(total['categories'], name).__iadd__(getattr(categories, name))
        for name in SUB_CATEGORY_FIELDS:
            getattr(total['sub_categories'], name).__iadd__(getattr(sub_categories, name))
    return total


def format_table(label, results, col_result):
    """Text table of one model: one row per dataset, the overall row with the collision test, one row per scene type."""
    lines = [_line(label, COLUMNS), _line('', ['-' * 8] * len(COLUMNS))]
    for dataset, (metrics, _, _) in sorted(results.items()):
        lines.append(_line(dataset, _cells(dataclasses.replace(metrics).avg_vals_to_list())))
    total = summarize(results)
    lines.append(_line('Overall', _cells(total['overall'].avg_vals_to_list())) + '   Col_test: %s' % col_result)
    for type_, sub, (group, name) in TYPE_ROWS:
        lines.append(_line('Type %s %s' % (type_, sub), _cells(getattr(total[group], name).avg_vals_to_list())))
    return '\n'.join(lines)


def trajnet_evaluate(args, out=print):
    """Scores <args.path>/<model>_modes<k>/*.ndjson (<model>_sample_modes<k> with args.sample) against the ground truth
    in the sibling test_private folder and prints
    one table per model.  Returns {label: {dataset: (metrics, categories, sub_categories)}}."""
    pred_root = args.path.rstrip(os.sep)
    private_root = (pred_root[:-len('_pred')] if pred_root.endswith('_pred') else pred_root) + '_private'
    from .evaluator import prediction_folder
    model_names = [prediction_folder(model, args) for model in args.output]
    labels = args.labels if getattr(args, 'labels', None) is not None else model_names
    disable_collision = getattr(args, 'disable_collision', False)
    everything = {}
    for label, model_name in zip(labels, model_names):
        files = sorted(f for f in os.listdir(os.path.join(pred_root, model_name)) if not f.startswith('.'))
        col_result = collision_test(files, model_name, args)
        results = {f[:-len('.ndjson')] if f.endswith('.ndjson') else f:
                   score_file(os.path.join(private_root, f), os.path.join(pred_root, model_name, f), obs_length=args.obs_length,
                              pred_length=args.pred_length, disable_collision=disable_collision)
                   for f in files if f != 'collision_test.ndjson'}
        out(format_table(label, results, col_result))
        everything[label] = results
    return everything
