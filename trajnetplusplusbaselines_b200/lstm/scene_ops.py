"""Batched scene preprocessing on the device (SURVEY.md 8f rank 3).

The reference prepares every scene on the host in NumPy before it joins a batch: `drop_distant`
(lstm/lstm.py:16-22), `center_scene` (lstm/utils.py:32-51), `random_rotation` (lstm/utils.py:10-17) in the trainer loop
(lstm/trainer.py:107-116), `center_scene` / `inverse_scene` (augmentation.py:65-68) around the predictor
(lstm/lstm.py:292-309).  Here the O(T * M) passes of a whole ragged batch run as three kernels of libtrajnet_b200
(csrc/scene_ops.cu: tb2_scenes_drop_distant / _transform / _inverse) in float64 with the reference's operation order, so the
float32 batch that reaches the model is bit-identical to the host path.  What stays on the host is O(B) scalar work: the
centre and the rotation angle of a scene come from two positions of its primary and go through the same libm calls
(`numpy.arctan2`, `math.cos`, `math.sin`) as the reference's.

There is no CPU implementation of the batched passes in this module: without a CUDA device the calls raise.  The
per-scene NumPy functions of the reference's API (`drop_distant`, `center_scene`, ...) live in lstm/lstm.py.
"""
import math

import numpy as np
import torch

from .. import _lib
from ..engine import _device_of, _ptr, _stream


def scene_frames(xy, split, obs_length=9):
    """Per scene the (centre [B, 2], rotation [B]) `center_scene` derives from its primary (lstm/utils.py:36-48):
    centre = primary's last observation, rotation = -arctan2 of the last observed displacement + pi / 2.  Host, O(B)."""
    first = np.asarray(split[:-1], dtype=np.int64)
    center = xy[obs_length - 1, first]                                         # [B, 2]
    last_obs = xy[obs_length - 1, first] - center
    second_last_obs = xy[obs_length - 2, first] - center
    diff = last_obs - second_last_obs
    rotation = -np.arctan2(diff[:, 1], diff[:, 0]) + np.pi / 2
    return center, rotation


def _frame_table(center, angle):
    """[B, 4] float64 rows (cx, cy, cos(angle), sin(angle)); math.cos / math.sin like theta_rotation (lstm/utils.py:24-30)."""
    table = np.empty((len(angle), 4), dtype=np.float64)
    table[:, 0:2] = center
    table[:, 2] = [math.cos(a) for a in angle]
    table[:, 3] = [math.sin(a) for a in angle]
    return table


def preprocess_scenes(scenes, device=None, r=None, normalize_scene=False, obs_length=9, thetas=None, goals=None):
    """Build one model batch from `scenes` (list of float64 arrays [T, N_i, 2], primary first, as Reader.paths_to_xy
    returns them), doing per scene what the reference's trainer loop does (lstm/trainer.py:107-116):

      r              -> drop_distant(xy, r)        (None: keep every track)
      normalize_scene -> center_scene(xy, obs_length)
      thetas [B]     -> random_rotation with these angles (the caller draws them: `random.random() * 2 * pi`)

    Returns (xy float32 CUDA tensor [T, M', 2], batch_split int64 CPU tensor [B + 1], keep mask bool ndarray [M],
    rotation ndarray [B], centre ndarray [B, 2]); rotation / centre are zeros without normalize_scene.

    goals: float64 [M, 2], one goal per track of the concatenated scenes.  They go through the same transform as the
    positions (center_scene / random_rotation with goals, lstm/utils.py:10-51), a track that drop_distant removes takes
    its goal with it, and float32 goals [M', 2] on the device are appended to the returned tuple."""
    _lib.require_cuda()
    lib = _lib.load()
    device = _device_of(device)
    B = len(scenes)
    split = np.zeros(B + 1, dtype=np.int64)
    split[1:] = np.cumsum([s.shape[1] for s in scenes])
    M = int(split[-1])
    host = np.ascontiguousarray(np.concatenate(scenes, axis=1), dtype=np.float64) if B else np.zeros((0, 0, 2))
    T = host.shape[0]
    rotation = np.zeros(B)
    center = np.zeros((B, 2))
    with torch.cuda.device(device):
        st = _stream(device)
        xy = torch.from_numpy(host).to(device)
        off = torch.from_numpy(split.astype(np.int32)).to(device)
        keep_dev, out_off, new_split, keep = None, off, split, np.ones(M, dtype=bool)
        if r is not None and M:
            keep_dev = torch.empty(M, dtype=torch.uint8, device=device)
            counts = torch.empty(B, dtype=torch.int32, device=device)
            _lib.check(lib.tb2_scenes_drop_distant(_ptr(xy), _ptr(off), T, M, B, float(r) ** 2, _ptr(keep_dev), _ptr(counts), st))
            new_split = np.zeros(B + 1, dtype=np.int64)
            new_split[1:] = np.cumsum(counts.cpu().numpy())
            out_off = torch.from_numpy(new_split.astype(np.int32)).to(device)
            keep = keep_dev.cpu().numpy().astype(bool)
        frame = aug = None
        if normalize_scene and B:
            center, rotation = scene_frames(host, split, obs_length)
            frame = torch.from_numpy(_frame_table(center, rotation)).to(device)
        if thetas is not None and B:
            thetas = np.asarray(thetas, dtype=np.float64)
            aug = torch.from_numpy(np.ascontiguousarray(_frame_table(np.zeros((B, 2)), thetas)[:, 2:4])).to(device)
        M_out = int(new_split[-1])
        out = torch.empty((T, M_out, 2), dtype=torch.float32, device=device)
        _lib.check(lib.tb2_scenes_transform(_ptr(xy), _ptr(off), _ptr(keep_dev), _ptr(out_off), T, M, M_out, B, _ptr(frame),
                                            _ptr(aug), _ptr(out), st))
        if goals is not None:           # one more "frame" of points through the same per-point transform
            goals = np.ascontiguousarray(goals, dtype=np.float64)
            if goals.shape != (M, 2):
                raise ValueError("goals must be [%d, 2] (one per track), got %s" % (M, list(goals.shape)))
            goals_in = torch.from_numpy(goals).to(device)
            goals_out = torch.empty((M_out, 2), dtype=torch.float32, device=device)
            _lib.check(lib.tb2_scenes_transform(_ptr(goals_in), _ptr(off), _ptr(keep_dev), _ptr(out_off), 1, M, M_out, B,
                                                _ptr(frame), _ptr(aug), _ptr(goals_out), st))
            return out, torch.from_numpy(new_split), keep, rotation, center, goals_out
    return out, torch.from_numpy(new_split), keep, rotation, center


def inverse_scenes(pred, batch_split, rotation, center):
    """`inverse_scene(output_scenes, rotation, center)` (augmentation.py:65-68, lstm/lstm.py:303-304) for every scene of a
    batch: pred float32 CUDA tensor [S, M, 2] -> float64 ndarray [S, M, 2]."""
    _lib.require_cuda()
    lib = _lib.load()
    if pred.device.type != 'cuda' or pred.dtype != torch.float32:
        raise RuntimeError("inverse_scenes needs the model's float32 CUDA output")
    pred = pred.contiguous()
    S, M = int(pred.shape[0]), int(pred.shape[1])
    split = np.asarray(batch_split, dtype=np.int64)
    B = len(split) - 1
    device = pred.device
    with torch.cuda.device(device):
        off = torch.from_numpy(split.astype(np.int32)).to(device)
        frame = torch.from_numpy(_frame_table(np.asarray(center, dtype=np.float64), -np.asarray(rotation, dtype=np.float64))).to(device)
        out = torch.empty((S, M, 2), dtype=torch.float64, device=device)
        _lib.check(lib.tb2_scenes_inverse(_ptr(pred), _ptr(off), S, M, B, _ptr(frame), _ptr(out), _stream(device)))
    return out.cpu().numpy()
