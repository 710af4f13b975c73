"""Minimal stand-ins for the trajnetplusplustools types the predictor boundary touches.

The reference imports `trajnetplusplustools` (not vendored, absent from this image) for
`TrackRow` and `Reader.paths_to_xy` (lstm/lstm.py:289, classical/*.py).  The on-disk format is
visible in the reference's DATA_BLOCK/*.ndjson; these helpers implement just that.
"""
import json
import os
import pickle
from collections import namedtuple, defaultdict

import numpy as np

TrackRow = namedtuple('TrackRow', ['frame', 'pedestrian', 'x', 'y', 'prediction_number', 'scene_id'])
TrackRow.__new__.__defaults__ = (None, None, None, None, None, None)
SceneRow = namedtuple('SceneRow', ['scene', 'pedestrian', 'start', 'end', 'fps', 'tag'])
SceneRow.__new__.__defaults__ = (None, None, None, None, None, None)


def paths_to_xy(paths):
    """list of paths (primary first) -> xy [n_frames, n_peds, 2] float64, NaN where absent.

    Same contract as trajnetplusplustools.Reader.paths_to_xy: the frames are the SORTED set of the
    primary pedestrian's frames, and a pedestrian without a single row in those frames is dropped (it
    would be an all-NaN column that the writer later emits as NaN track rows).
    """
    if paths and paths[0] and not isinstance(paths[0][0], tuple):     # rows with attributes only: normalise to tuples
        paths = [[(r.frame, r.pedestrian, r.x, r.y) for r in path] for path in paths]
    frames = sorted({r[0] for r in paths[0]})              # TrackRow is a tuple: (frame, pedestrian, x, y, ...)
    frame_index = {f: i for i, f in enumerate(frames)}
    n_frames = len(frames)
    nan = float('nan')
    columns = []                                            # one flat [x0, y0, x1, y1, ...] list per kept pedestrian
    for path in paths:
        col = None
        for r in path:
            i = frame_index.get(r[0])
            if i is not None:
                if col is None:
                    col = [nan] * (2 * n_frames)
                col[2 * i] = r[2]
                col[2 * i + 1] = r[3]
        if col is not None:
            columns.append(col)
    if not columns:
        return np.full((n_frames, 0, 2), np.nan)
    xy = np.array(columns, dtype=np.float64).reshape(len(columns), n_frames, 2)
    return np.ascontiguousarray(xy.transpose(1, 0, 2))


def read_ndjson_scenes(filename):
    """Yield (scene_id, paths) with the primary pedestrian first (TrajNet++ ndjson)."""
    tracks_by_frame = defaultdict(list)
    scenes = []
    with open(filename) as f:
        lines = [line for line in f if line.strip()]
    # one C-level parse of the whole file instead of a json.loads call per line
    for d in json.loads('[' + ','.join(lines) + ']') if lines else ():
        if 'track' in d:
            t = d['track']
            row = TrackRow(t['f'], t['p'], t['x'], t['y'], t.get('prediction_number'), t.get('scene_id'))
            tracks_by_frame[row.frame].append(row)
        elif 'scene' in d:
            s = d['scene']
            scenes.append(SceneRow(s['id'], s['p'], s['s'], s['e'], s.get('fps'), s.get('tag')))
    for s in scenes:
        by_ped = defaultdict(list)
        for frame in range(s.start, s.end + 1):
            for r in tracks_by_frame.get(frame, ()):
                by_ped[r.pedestrian].append(r)
        if s.pedestrian not in by_ped:
            continue
        paths = [by_ped[s.pedestrian]] + [p for pid, p in by_ped.items() if pid != s.pedestrian]
        yield s.scene, paths


def preprocess_test(scene, obs_len):
    """Drop tracks that only appear after the observation period (evaluator/write_utils.py:31-39)."""
    obs_frames = [row.frame for row in scene[0]][:obs_len]
    last_obs_frame = obs_frames[-1]
    return [[row for row in ped if row.frame <= last_obs_frame]
            for ped in scene if ped[0].frame <= last_obs_frame]


def goal_file(dataset_file):
    """Where the reference's evaluator reads the goals of a test file (evaluator/write_utils.py:21-25): relative to the
    working directory, goal_files/test_private/<file stem>.pkl."""
    stem = os.path.splitext(os.path.basename(dataset_file))[0]
    return os.path.join('goal_files', 'test_private', stem + '.pkl')


def load_goal_file(path):
    """The goals of a test file: dict pedestrian id -> (x, y), as written by the reference's get_dest.py."""
    if not os.path.exists(path):
        raise FileNotFoundError("goal file %s not found (a goal-conditioned model reads the goals of every test file "
                                "from goal_files/test_private/<file>.pkl)" % path)
    with open(path, 'rb') as f:
        return pickle.load(f)


def scene_pedestrians(filename):
    """The pedestrian ids with a row inside some scene of an ndjson file (the scenes read_ndjson_scenes yields, before
    preprocess_test): the ids whose goals the reference's evaluator looks up (evaluator/write_utils.py:21-25)."""
    cols = parse_ndjson_columns(filename)
    if cols is None:                                        # the row pipeline is the definition
        return {path[0].pedestrian for _, paths in read_ndjson_scenes(filename) for path in paths}
    order = np.argsort(cols['frame'], kind='stable')
    f, p = cols['frame'][order], cols['ped'][order]
    los = np.searchsorted(f, cols['scene_start'], side='left')
    his = np.searchsorted(f, cols['scene_end'], side='right')
    ids = set()
    for lo, hi, primary in zip(los, his, cols['scene_ped']):
        peds = np.unique(p[lo:hi])
        if primary in peds:                                 # read_ndjson_scenes skips a scene without its primary
            ids.update(peds.tolist())
    return ids


def check_goal_ids(goals, filename, path='goal file'):
    """Raise KeyError naming the first pedestrian of a scene of `filename` that has no goal in `goals`.  Like the
    reference, every track of a scene needs one, including the tracks preprocess_test then drops."""
    missing = sorted(ped for ped in scene_pedestrians(filename) if ped not in goals)
    if missing:
        raise KeyError("%s has no goal for pedestrian %s (%d pedestrian(s) of %s without a goal)"
                       % (path, missing[0], len(missing), filename))


def scene_goals(goals, ped_ids, path='goal file'):
    """float64 [len(ped_ids), 2]: the goals of a scene's tracks in track order (primary first), looked up by pedestrian
    id.  The tracks are those the predictor gets, so a track preprocess_test drops has no goal row."""
    out = np.empty((len(ped_ids), 2), dtype=np.float64)
    for i, ped in enumerate(ped_ids):
        g = goals.get(ped, goals.get(int(ped))) if hasattr(goals, 'get') else None
        if g is None:
            raise KeyError("%s has no goal for pedestrian %s" % (path, ped))
        out[i] = (float(g[0]), float(g[1]))
    return out


def trajnet_line(row):
    """One ndjson line for a SceneRow / TrackRow (the trajnetplusplustools.writers.trajnet format as it
    appears in the reference's DATA_BLOCK files: coordinates rounded to 2 decimals)."""
    if isinstance(row, SceneRow):
        return json.dumps({'scene': {'id': row.scene, 'p': row.pedestrian, 's': row.start, 'e': row.end,
                                     'fps': row.fps, 'tag': row.tag}})
    x, y = round(float(row.x), 2), round(float(row.y), 2)
    if row.prediction_number is None:
        return json.dumps({'track': {'f': row.frame, 'p': row.pedestrian, 'x': x, 'y': y}})
    return json.dumps({'track': {'f': row.frame, 'p': row.pedestrian, 'x': x, 'y': y,
                                 'prediction_number': row.prediction_number, 'scene_id': row.scene_id}})


def write_predictions(pred_list, scenes, filename, obs_length=9, pred_length=12):
    """Append the predictions of a list of scenes to an ndjson file -- same records, in the same
    order, as evaluator/write_utils.py:42-81 (which goes through trajnetplusplustools.writers).

    pred_list : per scene {mode: [primary [pred_length, 2], neighbours [pred_length, K, 2] or []]}
    scenes    : per scene (anything, scene_id, paths) as the reference evaluator holds them
    """
    seq_length = obs_length + pred_length

    def track_line(frame, ped, x, y, mode, scene_id):
        # same text as trajnet_line(TrackRow(...)) without building the dict / calling json.dumps per row
        x, y = round(float(x), 2), round(float(y), 2)
        if (type(frame) is int and type(ped) is int and type(mode) is int and type(scene_id) is int
                and x - x == 0.0 and y - y == 0.0):          # finite
            return '{"track": {"f": %d, "p": %d, "x": %r, "y": %r, "prediction_number": %d, "scene_id": %d}}\n' % (
                frame, ped, x, y, mode, scene_id)
        return trajnet_line(TrackRow(frame, ped, x, y, mode, scene_id)) + '\n'

    with open(filename, "a") as out:
        for predictions, (_, scene_id, paths) in zip(pred_list, scenes):
            observed_path = paths[0]
            frame_diff = observed_path[1].frame - observed_path[0].frame
            first_frame = observed_path[obs_length - 1].frame + frame_diff
            ped_id = observed_path[0].pedestrian
            neigh_ids = [p[0].pedestrian for p in paths[1:]]
            out.write(trajnet_line(SceneRow(scene_id, ped_id, observed_path[0].frame,
                                            observed_path[0].frame + (seq_length - 1) * frame_diff, 2.5, 0)))
            out.write('\n')
            for m in range(len(predictions)):
                prediction, neigh_predictions = predictions[m]
                rows = [track_line(first_frame + i * frame_diff, ped_id, prediction[i][0], prediction[i][1], m, scene_id)
                        for i in range(len(prediction))]
                if len(neigh_predictions):
                    neigh = np.asarray(neigh_predictions).tolist()          # python floats once, not per element
                    for n in range(len(neigh[0])):
                        rows.extend(track_line(first_frame + j * frame_diff, neigh_ids[n], neigh[j][n][0], neigh[j][n][1],
                                               m, scene_id) for j in range(len(neigh)))
                out.write(''.join(rows))


# ------------------------------------------------------------------------------------------------------------------
# Column pipeline of the batched evaluator (SURVEY.md 8f rank 1).  Same results as the row pipeline above
# (read_ndjson_scenes -> preprocess_test -> paths_to_xy ... write_predictions), without one Python object per track row:
# the text passes are native (csrc/ndjson.cu: tb2_ndjson_parse / tb2_ndjson_format), the per-scene assembly is NumPy.
# The row pipeline stays the definition: a file the native parser refuses goes through it, and tests/test_data_io.py
# holds the two against each other (arrays equal, output files byte-identical).
# ------------------------------------------------------------------------------------------------------------------
SceneMeta = namedtuple('SceneMeta', ['scene_id', 'pedestrian', 'first_frame', 'frame_diff', 'last_obs_frame', 'neigh_ids'])


def parse_ndjson_columns(filename):
    """Track / scene columns of an ndjson file through the native parser, or None when it refuses a line.

    Returns dict(frame, ped, x, y: track rows in file order; scene_id, scene_ped, scene_start, scene_end)."""
    import ctypes
    from . import _lib
    with open(filename, 'rb') as f:
        text = f.read()
    max_rows = text.count(b'\n') + 1
    i64 = lambda: np.empty(max_rows, dtype=np.int64)
    cols = dict(frame=i64(), ped=i64(), x=np.empty(max_rows), y=np.empty(max_rows),
                scene_id=i64(), scene_ped=i64(), scene_start=i64(), scene_end=i64())
    counts = np.zeros(3, dtype=np.int64)                    # tracks, scenes, refused line
    ptr = lambda a: ctypes.c_void_p(a.ctypes.data)
    _lib.check(_lib.load().tb2_ndjson_parse(
        ctypes.cast(ctypes.c_char_p(text), ctypes.c_void_p), len(text), max_rows,            # the bytes object's own buffer
        ptr(cols['frame']), ptr(cols['ped']), ptr(cols['x']), ptr(cols['y']),
        ptr(counts[0:1]), ptr(cols['scene_id']), ptr(cols['scene_ped']), ptr(cols['scene_start']), ptr(cols['scene_end']),
        ptr(counts[1:2]), ptr(counts[2:3])))
    if counts[2] >= 0:
        return None
    nt, ns = int(counts[0]), int(counts[1])
    return {k: (v[:ns] if k.startswith('scene_') else v[:nt]) for k, v in cols.items()}


def _scene_meta_from_paths(scene_id, paths, obs_length):
    observed_path = paths[0]
    return SceneMeta(scene_id, observed_path[0].pedestrian, observed_path[0].frame,
                     observed_path[1].frame - observed_path[0].frame, observed_path[obs_length - 1].frame,
                     [p[0].pedestrian for p in paths[1:]])


def load_scenes_xy(filename):
    """[(scene_id, xy float64 [n_frames, n_peds, 2])] of EVERY scene of an ndjson file over its whole frame range: per scene
    exactly paths_to_xy(paths) of read_ndjson_scenes (what the reference's trainer loop starts from,
    lstm/trainer.py:98-99) -- the input of lstm.scene_ops.preprocess_scenes."""
    cols = parse_ndjson_columns(filename)
    if cols is None:
        return [(scene_id, paths_to_xy(paths)) for scene_id, paths in read_ndjson_scenes(filename)]
    return [(meta.scene_id, xy) for xy, meta in _assemble_scenes(cols, None)]


def load_test_scenes_xy(filename, obs_length=9):
    """[(xy float64 [n_frames, n_peds, 2], SceneMeta)] of the test scenes of an ndjson file: per scene exactly
    paths_to_xy(preprocess_test(paths, obs_length)) and what write_predictions reads off those paths."""
    cols = parse_ndjson_columns(filename)
    if cols is None:                                        # the row pipeline is the definition
        out = []
        for scene_id, paths in read_ndjson_scenes(filename):
            paths = preprocess_test(paths, obs_length)
            out.append((paths_to_xy(paths), _scene_meta_from_paths(scene_id, paths, obs_length)))
        return out
    return _assemble_scenes(cols, obs_length)


def _assemble_scenes(cols, obs_length):
    """Per scene the xy array and SceneMeta from the parsed columns; obs_length None = the whole scene (no preprocess_test,
    the frame fields of the SceneMeta then describe the primary's first two frames and its last one)."""
    order = np.argsort(cols['frame'], kind='stable')        # by frame, file order within a frame (tracks_by_frame)
    f, p, x, y = cols['frame'][order], cols['ped'][order], cols['x'][order], cols['y'][order]
    los = np.searchsorted(f, cols['scene_start'], side='left')
    his = np.searchsorted(f, cols['scene_end'], side='right')
    out = []
    for i in range(len(los)):
        lo, hi = int(los[i]), int(his[i])
        fs, ps = f[lo:hi], p[lo:hi]
        primary = int(cols['scene_ped'][i])
        pf = fs[ps == primary]                              # the primary's rows, ascending frames
        if len(pf) == 0:
            continue                                        # read_ndjson_scenes skips a scene without its primary
        last = pf[:obs_length][-1] if obs_length is not None else fs[-1]      # preprocess_test: last frame of the observation
        cut = int(np.searchsorted(fs, last, side='right'))
        fs, ps, xs, ys = fs[:cut], ps[:cut], x[lo:lo + cut], y[lo:lo + cut]
        observed = pf[pf <= last]
        need = 1 if obs_length is None else max(obs_length, 2)
        if len(observed) < need:
            raise IndexError("scene %d: the primary has %d observed rows, %d needed" % (int(cols['scene_id'][i]), len(observed), need))
        uniq, first, inv = np.unique(ps, return_index=True, return_inverse=True)
        by_first = np.argsort(first, kind='stable')         # pedestrians in order of first appearance
        peds = uniq[by_first]
        k = int(np.nonzero(peds == primary)[0][0])
        peds = np.concatenate([peds[k:k + 1], peds[:k], peds[k + 1:]])           # primary first
        rank = np.empty(len(uniq), dtype=np.int64)
        rank[np.searchsorted(uniq, peds)] = np.arange(len(peds))
        col = rank[inv]
        frames = np.unique(observed)                        # paths_to_xy: sorted set of the primary's frames
        fi = np.minimum(np.searchsorted(frames, fs), len(frames) - 1)
        valid = frames[fi] == fs
        present = np.zeros(len(peds), dtype=bool)
        present[col[valid]] = True                          # a pedestrian without a row in those frames is dropped
        newcol = np.cumsum(present) - 1
        xy = np.full((len(frames), int(present.sum()), 2), np.nan)
        xy[fi[valid], newcol[col[valid]], 0] = xs[valid]
        xy[fi[valid], newcol[col[valid]], 1] = ys[valid]
        meta = SceneMeta(int(cols['scene_id'][i]), primary, int(observed[0]), int(observed[1] - observed[0]) if len(observed) > 1 else 0,
                         int(observed[obs_length - 1] if obs_length is not None else observed[-1]), peds[1:].tolist())
        out.append((xy, meta))
    return out


def write_predictions_xy(pred_list, metas, filename, obs_length=9, pred_length=12):
    """write_predictions for the column pipeline: same records, same bytes (one native formatting pass per call)."""
    import ctypes
    from . import _lib
    seq_length = obs_length + pred_length
    n = len(metas)
    sid = np.empty(n, dtype=np.int64)
    sped, sstart, send, nrows = (np.empty(n, dtype=np.int64) for _ in range(4))
    frames, peds, xs, ys, modes = [], [], [], [], []
    for i, (predictions, m) in enumerate(zip(pred_list, metas)):
        first_frame = m.last_obs_frame + m.frame_diff
        sid[i], sped[i], sstart[i], send[i] = m.scene_id, m.pedestrian, m.first_frame, m.first_frame + (seq_length - 1) * m.frame_diff
        rows = 0
        for mode in range(len(predictions)):
            prediction, neigh = predictions[mode]
            prediction = np.asarray(prediction, dtype=np.float64)
            T = len(prediction)
            f_prim = first_frame + np.arange(T, dtype=np.int64) * m.frame_diff
            frames.append(f_prim)
            peds.append(np.full(T, m.pedestrian, dtype=np.int64))
            xs.append(prediction[:, 0])
            ys.append(prediction[:, 1])
            count = T
            if len(neigh):
                neigh = np.asarray(neigh, dtype=np.float64)                    # [T', K, 2]
                Tn, K = neigh.shape[0], neigh.shape[1]
                ids = np.asarray(m.neigh_ids[:K], dtype=np.int64)
                if len(ids) != K:
                    raise IndexError("scene %d: %d neighbour predictions, %d neighbour ids" % (m.scene_id, K, len(ids)))
                frames.append(np.tile(first_frame + np.arange(Tn, dtype=np.int64) * m.frame_diff, K))
                peds.append(np.repeat(ids, Tn))
                xs.append(neigh[:, :, 0].T.reshape(-1))
                ys.append(neigh[:, :, 1].T.reshape(-1))
                count += Tn * K
            modes.append(np.full(count, mode, dtype=np.int64))
            rows += count
        nrows[i] = rows
    cat = lambda parts, dt: np.ascontiguousarray(np.concatenate(parts)) if parts else np.empty(0, dtype=dt)
    frames, peds, modes = cat(frames, np.int64), cat(peds, np.int64), cat(modes, np.int64)
    xs, ys = cat(xs, np.float64), cat(ys, np.float64)
    capacity = 160 * (n + len(frames)) + 16
    buf = ctypes.create_string_buffer(capacity)
    ptr = lambda a: ctypes.c_void_p(a.ctypes.data)
    used = _lib.load().tb2_ndjson_format(n, ptr(sid), ptr(sped), ptr(sstart), ptr(send), ptr(nrows), ptr(frames), ptr(peds),
                                         ptr(xs), ptr(ys), ptr(modes), ctypes.cast(buf, ctypes.c_void_p), capacity)
    if used < 0:
        _lib.check(int(used))
    if used > capacity:
        raise RuntimeError("tb2_ndjson_format needs %d bytes, %d provided" % (used, capacity))
    with open(filename, "ab") as out:
        out.write(memoryview(buf)[:used])
