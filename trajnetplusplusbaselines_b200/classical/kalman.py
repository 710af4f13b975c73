"""Kalman predictor with the reference's `predict` signature (CPU: BASELINE configs[0]).

Mirrors trajnetbaselines/classical/kalman.py:6-73.  pykalman's em / smooth / sample are replaced
by tb2_kalman_predict (host C++ in csrc/kalman.cu, float64).  The reference averages 5 noisy
`kf.sample` draws from the unseeded global NumPy RNG; `n_samples=5` reproduces that (same RNG
source, noise drawn from the fitted Q, R), `n_samples=0` returns the expectation.

predict_tracks_device runs the same EM / smoother code on the GPU (tb2_kalman_predict_device, one thread per track):
the expectation bit-identical to the host's, the sampled mean drawn on the device from torch's generator.
"""
import ctypes

import numpy as np

from .. import _lib

_A = np.array([[1, 1, 0, 0], [0, 1, 0, 0], [0, 0, 1, 1], [0, 0, 0, 1]], dtype=np.float64)
_C = np.array([[1, 0, 0, 0], [0, 0, 1, 0]], dtype=np.float64)


def concat_tracks(tracks):
    """Tracks [T_i, 2] -> (obs [sum T_i, 2] float64, offsets [n + 1] int64): the layout of the Kalman entry points."""
    tracks = [np.asarray(t, dtype=np.float64).reshape(-1, 2) for t in tracks]
    offsets = np.zeros(len(tracks) + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(t) for t in tracks])
    return (np.ascontiguousarray(np.concatenate(tracks)) if tracks else np.zeros((0, 2))), offsets


def predict_tracks(tracks, n_predict=12, n_samples=5, em_iterations=10):
    """tracks: list of [T_i, 2] arrays -> [n_tracks, n_predict, 2] float64."""
    lib = _lib.load()
    obs, offs = concat_tracks(tracks)
    n = len(offs) - 1
    pred = np.zeros((n, n_predict, 2), dtype=np.float64)
    q = np.zeros((n, 4, 4), dtype=np.float64)
    r = np.zeros((n, 2, 2), dtype=np.float64)
    last = np.zeros((n, 4), dtype=np.float64)
    _lib.check(lib.tb2_kalman_predict(obs.ctypes.data, offs.ctypes.data, n, n_predict, em_iterations,
                                      pred.ctypes.data, q.ctypes.data, r.ctypes.data, last.ctypes.data))
    if n_samples:
        for i in range(n):   # kalman.py:53-60: mean of n_samples x kf.sample(n_predict + 1)[observations][1:]
            acc = np.zeros((n_predict, 2))
            for _ in range(n_samples):
                x = last[i].copy()
                np.random.multivariate_normal(np.zeros(2), r[i])          # z_0 is drawn, then dropped
                for k in range(n_predict):
                    x = _A @ x + np.random.multivariate_normal(np.zeros(4), q[i])
                    acc[k] += _C @ x + np.random.multivariate_normal(np.zeros(2), r[i])
            pred[i] = acc / n_samples
    return pred


def predict_concat_device(obs, offsets, n_predict=12, n_samples=5, em_iterations=10, generator=None, eps=None,
                          device=None):
    """predict_tracks_device on tracks given concatenated: obs [total_obs, 2] float64 (host), offsets [n_tracks + 1]
    int64 (host).  Returns CUDA float64 tensors (pred [n, n_predict, 2], q [n, 4, 4], r [n, 2, 2], last [n, 4])."""
    import torch
    from ..engine import _device_of, _ptr, _stream
    _lib.require_cuda()
    lib = _lib.load()
    device = _device_of(device)
    offs = np.ascontiguousarray(offsets, dtype=np.int64)
    n = len(offs) - 1
    f64 = dict(dtype=torch.float64, device=device)
    pred, q, r, last = (torch.empty(s, **f64) for s in ((n, n_predict, 2), (n, 4, 4), (n, 2, 2), (n, 4)))
    if n_samples and eps is None:
        eps = torch.randn((n, n_predict, 6), generator=generator, **f64)
    if eps is not None:
        eps = torch.as_tensor(eps, **f64).contiguous()
        if tuple(eps.shape) != (n, n_predict, 6):
            raise ValueError("eps must be [n_tracks, n_predict, 6], got %s" % (tuple(eps.shape),))
    obs_t = torch.from_numpy(np.ascontiguousarray(obs, dtype=np.float64).reshape(-1, 2)).to(device)
    offs_t = torch.from_numpy(offs).to(device)
    ws = torch.empty(int(lib.tb2_kalman_workspace_bytes(offs.ctypes.data, n)), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.tb2_kalman_predict_device(_ptr(obs_t), offs.ctypes.data, _ptr(offs_t), n, n_predict, em_iterations,
                                                 n_samples, _ptr(eps), _ptr(pred), _ptr(q), _ptr(r), _ptr(last), _ptr(ws),
                                                 ws.numel(), _stream(device)))
    return pred, q, r, last


def predict_tracks_device(tracks, n_predict=12, n_samples=5, em_iterations=10, generator=None, eps=None, device=None):
    """predict_tracks on the device (tb2_kalman_predict_device): tracks list of [T_i, 2] arrays -> pred CUDA float64
    [n_tracks, n_predict, 2].  n_samples = 0: the expectation, bit-identical to predict_tracks(n_samples=0).
    n_samples >= 1: the mean of n_samples sampled rollouts, drawn as one rollout driven by Q / n_samples and
    R / n_samples from eps [n_tracks, n_predict, 6] standard normals (default: torch.randn on the device from
    `generator`).  The random stream is torch's, not NumPy's global one (DESIGN §8)."""
    obs, offs = concat_tracks(tracks)
    return predict_concat_device(obs, offs, n_predict=n_predict, n_samples=n_samples, em_iterations=em_iterations,
                                 generator=generator, eps=eps, device=device)[0]


def predict(paths, predict_all=True, n_predict=12, obs_length=9, n_samples=5):
    neighbours_tracks = []
    primary = paths[0]
    start_frame = primary[obs_length - 1].frame
    if not predict_all:
        paths = paths[0:1]
    tracks, is_primary = [], []
    for i, path in enumerate(paths):
        past_path = [t for t in path if t.frame <= start_frame]
        past_frames = [t.frame for t in past_path]
        if start_frame not in past_frames or len(past_path) < 2:
            continue
        tracks.append(np.array([(r.x, r.y) for r in past_path], dtype=np.float64))
        is_primary.append(i == 0)
    pred = predict_tracks(tracks, n_predict=n_predict, n_samples=n_samples)
    primary_track = None
    for p, prim in zip(pred, is_primary):
        if prim:
            primary_track = p
        else:
            neighbours_tracks.append(p)
    if len(neighbours_tracks):
        neighbours_tracks = np.array(neighbours_tracks).transpose(1, 0, 2)
    return {0: (primary_track, neighbours_tracks)}
