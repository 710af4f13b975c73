"""ORCA predictor with the reference's `predict` signature, simulated on the GPU.

Mirrors trajnetbaselines/classical/orca.py:10-134.  rvo2.PyRVOSimulator + the per-agent
doStep / getAgentPosition / setAgentPrefVelocity loop (3 FFI calls per agent per step) is
replaced by tb2_orca_simulate (csrc/classical.cu): one persistent kernel, one CTA per scene,
float arithmetic like RVO2.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from ..engine import SceneLayout, _ptr, _stream
from .common import initial_states, sweep_params

MAX_SPEED_MULTIPLIER = 1.3   # applied inside the kernel (orca.py:8,36)


def simulate_batch(pos, vel, goals, speeds, batch_split, orca_params=(1.5, 1.5, 0.4), n_steps=97,
                   sample_every=8, fps=20, max_neighbors=10, end_range=0.05, device=None):
    """pos, vel [A, 2]; goals [A, 2]; speeds [A]; -> [n_steps // sample_every, A, 2] float32."""
    _lib.require_cuda()
    lib = _lib.load()
    device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    pos_t = torch.as_tensor(np.asarray(pos), dtype=torch.float32).to(device).contiguous()
    vel_t = torch.as_tensor(np.asarray(vel), dtype=torch.float32).to(device).contiguous()
    goal_t = torch.as_tensor(np.asarray(goals), dtype=torch.float64).to(device).contiguous()
    speed_t = torch.as_tensor(np.asarray(speeds), dtype=torch.float64).to(device).contiguous()
    layout = SceneLayout(batch_split, device=device)
    if layout.num_tracks != pos_t.shape[0]:
        raise ValueError("batch_split[-1] != number of agents")
    p = _lib.OrcaParams()
    p.time_step = 1.0 / fps
    p.neighbor_dist = float(orca_params[0])
    p.max_neighbors = int(max_neighbors)
    p.time_horizon = float(orca_params[1])
    p.radius = float(orca_params[2])
    p.end_range = float(end_range)
    p.n_steps, p.sample_every = int(n_steps), int(sample_every)
    out = torch.empty((n_steps // sample_every, pos_t.shape[0], 2), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.tb2_orca_simulate(layout.handle, ctypes.byref(p), _ptr(pos_t), _ptr(vel_t),
                                         _ptr(goal_t), _ptr(speed_t), _ptr(out), _stream(device)))
    return out


def sweep(prepared, params, fps=20, max_neighbors=10, end_range=0.05):
    """ADE / FDE of the primary of every scene of `prepared` (common.PreparedScenes) under every setting of params
    [P, 3] (neighbor_dist, time_horizon, radius; float32 like RVO2) -> (ade, fde) CUDA float64 [P, B], one launch
    (tb2_orca_sweep).  Row s equals simulate_batch(...(params[s]), n_steps=sampling_rate * pred_length + 1) with the
    float positions widened to double and scored against prepared.truth: distances in sample order summed in float64,
    ADE = sum / pred_length, FDE = the last distance."""
    B, T = int(prepared.truth.shape[0]), int(prepared.truth.shape[1])
    prm = sweep_params(params, np.float32, ("neighbor_dist", "time_horizon", "radius"), (1, 2), B)
    _lib.require_cuda()
    lib = _lib.load()
    sampling_rate = int(fps / 2.5)
    p = _lib.OrcaParams()
    p.time_step = 1.0 / fps
    p.neighbor_dist, p.time_horizon, p.radius = (float(v) for v in prm[0])
    p.max_neighbors = int(max_neighbors)
    p.end_range = float(end_range)
    p.n_steps, p.sample_every = sampling_rate * T + 1, sampling_rate
    device = prepared.state.device
    st = prepared.state
    pos = st[:, 0:2].to(torch.float32).contiguous()
    vel = st[:, 2:4].to(torch.float32).contiguous()
    goal = st[:, 4:6].contiguous()
    prm_t = torch.from_numpy(prm).to(device)
    ade = torch.empty((len(prm), B), dtype=torch.float64, device=device)
    fde = torch.empty_like(ade)
    with torch.cuda.device(device):
        _lib.check(lib.tb2_orca_sweep(prepared.layout.handle, ctypes.byref(p), _ptr(prm_t), len(prm), _ptr(pos), _ptr(vel),
                                      _ptr(goal), _ptr(prepared.speeds), _ptr(prepared.truth), T, _ptr(ade), _ptr(fde),
                                      _stream(device)))
    return ade, fde


def predict(input_paths, dest_dict=None, dest_type='interp', orca_params=[1.5, 1.5, 0.4],
            predict_all=True, n_predict=12, obs_length=9):
    pred_length = n_predict
    primary = input_paths[0]
    start_frame = primary[obs_length - 1].frame
    state, speeds = initial_states(input_paths, start_frame, pred_length, dest_dict, dest_type)
    fps = 20
    sampling_rate = int(fps / 2.5)
    n_steps = sampling_rate * pred_length + 1          # orca.py:99
    states = simulate_batch(state[:, 0:2], state[:, 2:4], state[:, 4:6], speeds, [0, len(state)],
                            orca_params, n_steps=n_steps, sample_every=sampling_rate, fps=fps)
    states = states.cpu().numpy().astype(np.float64)
    primary_track = states[:, 0, 0:2]
    neighbours_tracks = states[:, 1:, 0:2]
    if not predict_all:
        neighbours_tracks = []
    return {0: (primary_track, neighbours_tracks)}
