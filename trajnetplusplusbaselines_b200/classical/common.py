"""Host-side scene preparation shared by the classical adapters (NumPy, O(scene)).

Mirrors the adapter code around the third-party simulators in the reference
(trajnetbaselines/classical/socialforce.py:15-72, orca.py:14-82): which pedestrians are
simulated, their initial velocity (stride-3 finite difference) and their destination (linear
extrapolation of the observed path).
"""
import ctypes
from collections import namedtuple

import numpy as np

FPS = 20                                   # simulation steps per second (socialforce.py:71, orca.py:86)


def sampling_rate(fps):
    """Simulation steps per observed frame: the scenes are sampled at 2.5 Hz (socialforce.py:72, orca.py:87)."""
    return int(fps / 2.5)


SAMPLING_RATE = sampling_rate(FPS)


def _velocity(cx, cy, px, py, stride):
    """Initial velocity and speed from the position `stride` rows back (socialforce.py:28-38): scalar NumPy calls, so
    the path and xy preparations round identically."""
    if stride == 0:
        return 0.0, 0.0, 0.0
    diff = np.array([cx - px, cy - py])
    theta = np.arctan2(diff[1], diff[0])
    speed = np.linalg.norm(diff) / (stride * 0.4)
    return speed * np.cos(theta), speed * np.sin(theta), speed


def initial_states(input_paths, start_frame, pred_length, dest_dict=None, dest_type='interp'):
    """-> (state [K, 6] float64: x, y, vx, vy, dx, dy; speeds [K]) for the K pedestrians present at
    `start_frame`, in path order (socialforce.py:15-55 / orca.py:14-58)."""
    rows, speeds = [], []
    for path in input_paths:
        ped_id = path[0].pedestrian
        past_path = [t for t in path if t.frame <= start_frame]
        future_path = [t for t in path if t.frame > start_frame]
        past_frames = [t.frame for t in past_path]
        len_path = len(past_path)
        if start_frame not in past_frames:
            continue
        curr = past_path[-1]
        if len_path >= 4:
            stride, prev = 3, past_path[-4]
        else:
            stride, prev = len_path - 1, past_path[-len_path]
        v_x, v_y, speed = _velocity(curr.x, curr.y, prev.x, prev.y, stride)
        if dest_type == 'true':
            if dest_dict is None:
                raise ValueError
            d_x, d_y = dest_dict[ped_id]
        elif dest_type == 'interp':
            if len_path == 1:
                d_x, d_y = curr.x, curr.y
            else:   # interp1d(..., fill_value='extrapolate') evaluated at len-1+pred_length
                p1, p0 = past_path[-1], past_path[-2]
                d_x = p1.x + (p1.x - p0.x) * pred_length
                d_y = p1.y + (p1.y - p0.y) * pred_length
        elif dest_type == 'vel':
            d_x, d_y = pred_length * v_x, pred_length * v_y
        elif dest_type == 'pred_end':
            d_x, d_y = future_path[-1].x, future_path[-1].y
        else:
            raise NotImplementedError
        rows.append([curr.x, curr.y, v_x, v_y, d_x, d_y])
        speeds.append(speed)
    return np.array(rows, dtype=np.float64).reshape(-1, 6), np.array(speeds, dtype=np.float64)


def xy_representable(xy):
    """False where NaN cannot stand for "no row": the xy arrays of load_scenes_xy hold every row of a scene only when
    each pedestrian's rows fall on the primary's frames, once per frame, with finite coordinates.  The caller knows the
    rows; this checks what the array itself shows (the primary present at every frame)."""
    return xy.shape[1] > 0 and not np.isnan(xy[:, 0]).any()


def initial_states_xy(xy_list, obs_length=9, pred_length=12, dest_type='interp', dest_dict=None, truth=True):
    """initial_states for every scene of a list, from xy arrays instead of track rows.

    xy_list: [(scene_id, scene)] as data.load_scenes_xy returns it, `scene` an xy array [n_frames, n_peds, 2] (NaN =
    no row, primary first, frames = the primary's) -- or the scene's paths (rows), which go through initial_states.  A
    scene whose rows an xy array cannot represent (rows off the primary's frames, repeated frames, non-finite
    coordinates) must be passed as paths; so must every scene for dest_type 'true', which needs pedestrian ids.

    Per scene the result is bit-identical to initial_states(paths, primary[obs_length - 1].frame, pred_length, ...),
    including the reference's row-count semantics: the stride counts past ROWS (prev = past_path[-4]) and 'interp'
    extrapolates from the last two rows.

    Returns numpy arrays: state [A, 6] float64, speeds [A], agent_offsets [B + 1] int64 (scene b owns rows
    agent_offsets[b] .. agent_offsets[b + 1] - 1, its primary first), truth [B, pred_length, 2] float64 (the primary's
    last pred_length rows, what metrics.average_l2(paths[0], prediction) compares against).  truth=False: None instead
    (test scenes, which hold the observation only).
    """
    if dest_type not in ('interp', 'vel', 'pred_end', 'true'):
        raise NotImplementedError(dest_type)
    want_truth = truth
    states, speeds, counts, truth = [], [], [], []
    t0 = obs_length - 1
    for _, scene in xy_list:
        if not isinstance(scene, np.ndarray):                   # rows: the definition
            paths = scene
            st, sp = initial_states(paths, paths[0][t0].frame, pred_length, dest_dict, dest_type)
            tr = np.array([[r.x, r.y] for r in paths[0][-pred_length:]], dtype=np.float64)
        else:
            if dest_type == 'true':
                raise ValueError("dest_type 'true' needs pedestrian ids: pass the scene's paths")
            if not xy_representable(scene):
                raise ValueError("xy array without its primary at every frame: pass the scene's paths")
            st, sp = _initial_states_xy_scene(scene, t0, pred_length, dest_type)
            tr = scene[-pred_length:, 0]
        if want_truth and len(tr) < pred_length:
            raise ValueError("the primary has %d rows, %d needed for the truth" % (len(tr), pred_length))
        states.append(st)
        speeds.append(sp)
        counts.append(len(st))
        truth.append(tr)
    offsets = np.zeros(len(counts) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum(counts)
    return (np.concatenate(states).reshape(-1, 6) if states else np.zeros((0, 6)),
            np.concatenate(speeds) if speeds else np.zeros(0), offsets,
            np.array(truth, dtype=np.float64).reshape(len(truth), pred_length, 2) if want_truth else None)


def _initial_states_xy_scene(xy, t0, pred_length, dest_type):
    present = ~np.isnan(xy[:, :, 0])                           # [n_frames, n_peds]: a row at that frame
    rows, speeds = [], []
    for j in np.nonzero(present[t0])[0]:                         # present at start_frame, in path order
        past = np.nonzero(present[:t0 + 1, j])[0]                # frame indices of past_path
        len_path = len(past)
        curr = xy[past[-1], j]
        if len_path >= 4:
            stride, prev = 3, xy[past[-4], j]
        else:
            stride, prev = len_path - 1, xy[past[0], j]
        v_x, v_y, speed = _velocity(curr[0], curr[1], prev[0], prev[1], stride)
        if dest_type == 'interp':
            if len_path == 1:
                d_x, d_y = curr[0], curr[1]
            else:
                p1, p0 = curr, xy[past[-2], j]
                d_x = p1[0] + (p1[0] - p0[0]) * pred_length
                d_y = p1[1] + (p1[1] - p0[1]) * pred_length
        elif dest_type == 'vel':
            d_x, d_y = pred_length * v_x, pred_length * v_y
        else:                                                    # 'pred_end': the last row after start_frame
            future = np.nonzero(present[t0 + 1:, j])[0]
            if len(future) == 0:
                raise IndexError("pred_end: pedestrian %d has no row after the observation" % j)
            d_x, d_y = xy[t0 + 1 + future[-1], j]
        rows.append([curr[0], curr[1], v_x, v_y, d_x, d_y])
        speeds.append(speed)
    return np.array(rows, dtype=np.float64).reshape(-1, 6), np.array(speeds, dtype=np.float64)


# Scenes on the device for the sweeps (socialforce.sweep / orca.sweep): state [A, 6] float64, speeds [A] float64 and
# truth [B, pred_length, 2] float64 CUDA tensors, layout the SceneLayout of agent_offsets [B + 1] (numpy).  `scenes` is
# the host list initial_states_xy read (None when built from arrays).
PreparedScenes = namedtuple('PreparedScenes', ['state', 'speeds', 'truth', 'agent_offsets', 'layout', 'scenes'])


def to_device(state, speeds, agent_offsets, truth, scenes=None, device=None):
    """initial_states_xy's arrays -> PreparedScenes on `device` (default: the current CUDA device)."""
    import torch
    from ..engine import SceneLayout, _device_of
    device = _device_of(device)
    state = np.asarray(state, dtype=np.float64).reshape(-1, 6)
    speeds = np.asarray(speeds, dtype=np.float64).reshape(-1)
    offsets = np.asarray(agent_offsets, dtype=np.int64).reshape(-1)
    truth = np.asarray(truth, dtype=np.float64)
    B = len(offsets) - 1
    if B < 1 or offsets[0] != 0 or (np.diff(offsets) < 1).any() or offsets[-1] != len(state) or len(speeds) != len(state):
        raise ValueError("agent_offsets must start at 0, grow by >= 1 pedestrian per scene and end at len(state)")
    if truth.ndim != 3 or truth.shape[0] != B or truth.shape[2] != 2:
        raise ValueError("truth must be [B, pred_length, 2], got %s for B = %d" % (truth.shape, B))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return PreparedScenes(t(state), t(speeds), t(truth), offsets, SceneLayout(offsets, device=device), scenes)


def sweep_params(params, dtype, names, positive, B):
    """[P, 3] settings checked before any launch: P >= 1, P x B < 2^31, finite, and the columns `positive` > 0."""
    with np.errstate(over='ignore'):                      # too large for float32: inf, refused below
        arr = np.asarray(params, dtype=dtype)
    if arr.ndim == 1:
        arr = arr.reshape(1, -1)
    if arr.ndim != 2 or arr.shape[1] != 3 or arr.shape[0] < 1:
        raise ValueError("params must be [P, 3] (%s) with P >= 1, got shape %s" % (", ".join(names), np.shape(params)))
    if arr.shape[0] * B >= 2 ** 31:
        raise ValueError("P x B = %d x %d must stay below 2^31" % (arr.shape[0], B))
    if not np.isfinite(arr).all():
        raise ValueError("non-finite sweep parameter")
    for c in positive:
        if not (arr[:, c] > 0).all():
            raise ValueError("%s must be > 0" % names[c])
    return np.ascontiguousarray(arr)


# ---- the one driver of tb2_sf_* / tb2_orca_* (socialforce.py and orca.py state what is their own) -------------------
def simulate(sim, params, inputs, batch_split, n_samples, out_dtype, device=None):
    """One tb2_<sim>_simulate launch over every scene of batch_split.  inputs: [(array, torch dtype)] in the entry
    point's order, one row per pedestrian; params: the ctypes parameter struct.  -> sampled positions
    [n_samples, A, 2] of out_dtype on `device` (default: the current CUDA device)."""
    import torch
    from .. import _lib
    from ..engine import SceneLayout, _device_of, _ptr, _stream
    _lib.require_cuda()
    lib = _lib.load()
    device = _device_of(device)
    tensors = [torch.as_tensor(x, dtype=dtype).to(device).contiguous() for x, dtype in inputs]
    layout = SceneLayout(batch_split, device=device)
    if layout.num_tracks != tensors[0].shape[0]:
        raise ValueError("batch_split[-1] != number of pedestrians")
    out = torch.empty((n_samples, tensors[0].shape[0], 2), dtype=out_dtype, device=device)
    with torch.cuda.device(device):
        _lib.check(getattr(lib, "tb2_%s_simulate" % sim)(layout.handle, ctypes.byref(params), *map(_ptr, tensors),
                                                          _ptr(out), _stream(device)))
    return out


def sweep(sim, prepared, settings, params, inputs, grad=False):
    """One tb2_<sim>_sweep launch: settings [P, 3] (checked by sweep_params), params the ctypes struct of the fields
    the settings leave alone, inputs the device tensors of prepared in the entry point's order -> (ade, fde) CUDA
    float64 [P, B].  grad: tb2_<sim>_sweep_grad instead -> (ade, fde, dade, dfde), the derivatives [P, B, 3] with
    respect to the three settings."""
    import torch
    from .. import _lib
    from ..engine import _ptr, _stream
    _lib.require_cuda()
    lib = _lib.load()
    B, T = int(prepared.truth.shape[0]), int(prepared.truth.shape[1])
    device = prepared.state.device
    prm = torch.from_numpy(settings).to(device)
    outs = [torch.empty((len(settings), B), dtype=torch.float64, device=device) for _ in range(2)]
    if grad:
        outs += [torch.empty((len(settings), B, 3), dtype=torch.float64, device=device) for _ in range(2)]
    with torch.cuda.device(device):
        _lib.check(getattr(lib, "tb2_%s_sweep%s" % (sim, "_grad" if grad else ""))(
            prepared.layout.handle, ctypes.byref(params), _ptr(prm), len(settings), *map(_ptr, inputs),
            _ptr(prepared.truth), T, *map(_ptr, outs), _stream(device)))
    return tuple(outs)


def predict(rollout, input_paths, dest_dict, dest_type, predict_all, n_predict, obs_length, stationary=False):
    """The reference adapters' `predict` around a simulator (socialforce.py:74-111, orca.py:84-134).  rollout(state,
    speeds, offsets, pred_length) -> positions [pred_length, K, 2] float64 (host) of the K pedestrians present at the
    last observed frame, primary first.  stationary: with none present, the primary stays where it was last seen
    (socialforce.py:96-99; the ORCA adapter has no such case)."""
    start_frame = input_paths[0][obs_length - 1].frame
    state, speeds = initial_states(input_paths, start_frame, n_predict, dest_dict, dest_type)
    if stationary and len(state) == 0:
        past_path = [t for t in input_paths[0] if t.frame == start_frame]
        states = np.stack([[[past_path[0].x, past_path[0].y]] for _ in range(n_predict)])
    else:
        states = rollout(state, speeds, [0, len(state)], n_predict)
    primary_track = states[:, 0, 0:2]
    neighbours_tracks = states[:, 1:, 0:2]
    if not predict_all:
        neighbours_tracks = []
    return {0: (primary_track, neighbours_tracks)}
