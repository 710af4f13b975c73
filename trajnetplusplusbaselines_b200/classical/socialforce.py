"""Social-force predictor with the reference's `predict` signature, simulated on the GPU.

Mirrors trajnetbaselines/classical/socialforce.py:10-111.  The 96 x Simulator.step() loop of
the un-vendored `socialforce` package is replaced by tb2_sf_simulate (csrc/classical.cu): one
persistent kernel, one CTA per scene, float64 like upstream.  `simulate_batch` exposes the same
kernel for many scenes per launch (the evaluator's joblib fan-out collapses into one call).
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from ..engine import SceneLayout, _ptr, _stream
from .common import initial_states, sweep_params


def simulate_batch(states, batch_split, sf_params=(0.5, 2.1, 0.3), n_steps=96, sample_every=8, fps=20,
                   device=None):
    """states [A, 6] float64 (x, y, vx, vy, dx, dy) of all scenes, batch_split [B+1] ->
    sampled positions [ceil(n_steps / sample_every), A, 2] float64 (CUDA tensor)."""
    _lib.require_cuda()
    lib = _lib.load()
    device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    st = torch.as_tensor(states, dtype=torch.float64).to(device).contiguous()
    layout = SceneLayout(batch_split, device=device)
    if layout.num_tracks != st.shape[0]:
        raise ValueError("batch_split[-1] != number of pedestrians")
    p = _lib.SfParams()
    p.delta_t = 1.0 / fps
    p.tau, p.v0, p.sigma = float(sf_params[0]), float(sf_params[1]), float(sf_params[2])
    p.n_steps, p.sample_every = int(n_steps), int(sample_every)
    n_samples = (n_steps + sample_every - 1) // sample_every
    out = torch.empty((n_samples, st.shape[0], 2), dtype=torch.float64, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.tb2_sf_simulate(layout.handle, ctypes.byref(p), _ptr(st), _ptr(out), _stream(device)))
    return out


def sweep(prepared, params, fps=20):
    """ADE / FDE of the primary of every scene of `prepared` (common.PreparedScenes) under every setting of params
    [P, 3] (tau, v0, sigma) -> (ade, fde) CUDA float64 [P, B], one launch (tb2_sf_sweep).  Row s equals
    simulate_batch(state, agent_offsets, params[s], n_steps=pred_length * sampling_rate, sample_every=sampling_rate)
    scored against prepared.truth: distances in sample order summed in float64, ADE = sum / pred_length, FDE = the
    last distance.  The trajectories never reach device memory."""
    B, T = int(prepared.truth.shape[0]), int(prepared.truth.shape[1])
    prm = sweep_params(params, np.float64, ("tau", "v0", "sigma"), (0, 2), B)
    _lib.require_cuda()
    lib = _lib.load()
    sampling_rate = int(fps / 2.5)
    p = _lib.SfParams()
    p.delta_t = 1.0 / fps
    p.tau, p.v0, p.sigma = (float(v) for v in prm[0])
    p.n_steps, p.sample_every = T * sampling_rate, sampling_rate
    device = prepared.state.device
    prm_t = torch.from_numpy(prm).to(device)
    ade = torch.empty((len(prm), B), dtype=torch.float64, device=device)
    fde = torch.empty_like(ade)
    with torch.cuda.device(device):
        _lib.check(lib.tb2_sf_sweep(prepared.layout.handle, ctypes.byref(p), _ptr(prm_t), len(prm), _ptr(prepared.state),
                                    _ptr(prepared.truth), T, _ptr(ade), _ptr(fde), _stream(device)))
    return ade, fde


def predict(input_paths, dest_dict=None, dest_type='interp', sf_params=[0.5, 2.1, 0.3],
            predict_all=True, n_predict=12, obs_length=9):
    pred_length = n_predict
    primary = input_paths[0]
    start_frame = primary[obs_length - 1].frame
    initial_state, _ = initial_states(input_paths, start_frame, pred_length, dest_dict, dest_type)
    fps = 20
    sampling_rate = int(fps / 2.5)
    if len(initial_state) != 0:
        states = simulate_batch(initial_state, [0, len(initial_state)], sf_params,
                                n_steps=pred_length * sampling_rate, sample_every=sampling_rate, fps=fps)
        states = states.cpu().numpy()
    else:   # stationary (socialforce.py:96-99)
        past_path = [t for t in input_paths[0] if t.frame == start_frame]
        states = np.stack([[[past_path[0].x, past_path[0].y]] for _ in range(pred_length)])
    primary_track = states[:, 0, 0:2]
    neighbours_tracks = states[:, 1:, 0:2]
    if not predict_all:
        neighbours_tracks = []
    return {0: (primary_track, neighbours_tracks)}
