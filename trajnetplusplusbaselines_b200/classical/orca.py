"""ORCA predictor with the reference's `predict` signature, simulated on the GPU.

Mirrors trajnetbaselines/classical/orca.py:10-134.  rvo2.PyRVOSimulator + the per-agent
doStep / getAgentPosition / setAgentPrefVelocity loop (3 FFI calls per agent per step) is
replaced by tb2_orca_simulate (csrc/classical.cu): one persistent kernel, one CTA per scene,
float arithmetic like RVO2.
"""
import numpy as np
import torch

from .. import _lib
from . import common
from .common import FPS, SAMPLING_RATE, sampling_rate, sweep_params

MAX_SPEED_MULTIPLIER = 1.3   # applied inside the kernel (orca.py:8,36)


def steps_for(pred_length, rate=SAMPLING_RATE):
    """Simulation steps for pred_length observed frames (orca.py:99): one more than social force's."""
    return rate * pred_length + 1


def _params(orca_params, steps, sample_every, fps, max_neighbors, end_range):
    p = _lib.OrcaParams()
    p.time_step = 1.0 / fps
    p.neighbor_dist, p.time_horizon, p.radius = float(orca_params[0]), float(orca_params[1]), float(orca_params[2])
    p.max_neighbors = int(max_neighbors)
    p.end_range = float(end_range)
    p.n_steps, p.sample_every = int(steps), int(sample_every)
    return p


def simulate_batch(pos, vel, goals, speeds, batch_split, orca_params=(1.5, 1.5, 0.4), n_steps=steps_for(12),
                   sample_every=SAMPLING_RATE, fps=FPS, max_neighbors=10, end_range=0.05, device=None):
    """pos, vel [A, 2]; goals [A, 2]; speeds [A]; -> [n_steps // sample_every, A, 2] float32."""
    p = _params(orca_params, n_steps, sample_every, fps, max_neighbors, end_range)
    inputs = [(pos, torch.float32), (vel, torch.float32), (goals, torch.float64), (speeds, torch.float64)]
    return common.simulate("orca", p, inputs, batch_split, n_steps // sample_every, torch.float32, device)


def rollout(state, speeds, batch_split, orca_params, pred_length, device=None):
    """simulate_batch as `predict` runs it -> positions [pred_length, A, 2] widened to float64 (host)."""
    out = simulate_batch(state[:, 0:2], state[:, 2:4], state[:, 4:6], speeds, batch_split, orca_params,
                         n_steps=steps_for(pred_length), device=device)
    return out.cpu().numpy().astype(np.float64)


def sweep(prepared, params, fps=FPS, max_neighbors=10, end_range=0.05):
    """ADE / FDE of the primary of every scene of `prepared` (common.PreparedScenes) under every setting of params
    [P, 3] (neighbor_dist, time_horizon, radius; float32 like RVO2) -> (ade, fde) CUDA float64 [P, B], one launch
    (tb2_orca_sweep).  Row s equals simulate_batch(...(params[s]), n_steps=steps_for(pred_length, rate),
    sample_every=rate) with rate = sampling_rate(fps), the float positions widened to double and scored against
    prepared.truth: distances in sample order summed in float64, ADE = sum / pred_length, FDE = the last distance."""
    prm = sweep_params(params, np.float32, ("neighbor_dist", "time_horizon", "radius"), (1, 2),
                       int(prepared.truth.shape[0]))
    rate = sampling_rate(fps)
    p = _params(prm[0], steps_for(int(prepared.truth.shape[1]), rate), rate, fps, max_neighbors, end_range)
    st = prepared.state
    inputs = [st[:, 0:2].to(torch.float32).contiguous(), st[:, 2:4].to(torch.float32).contiguous(),
              st[:, 4:6].contiguous(), prepared.speeds]
    return common.sweep("orca", prepared, prm, p, inputs)


def predict(input_paths, dest_dict=None, dest_type='interp', orca_params=[1.5, 1.5, 0.4],
            predict_all=True, n_predict=12, obs_length=9):
    run = lambda state, speeds, batch_split, pred_length: rollout(state, speeds, batch_split, orca_params, pred_length)
    return common.predict(run, input_paths, dest_dict, dest_type, predict_all, n_predict, obs_length)
