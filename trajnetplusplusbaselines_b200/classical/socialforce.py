"""Social-force predictor with the reference's `predict` signature, simulated on the GPU.

Mirrors trajnetbaselines/classical/socialforce.py:10-111.  The 96 x Simulator.step() loop of
the un-vendored `socialforce` package is replaced by tb2_sf_simulate (csrc/classical.cu): one
persistent kernel, one CTA per scene, float64 like upstream.  `simulate_batch` exposes the same
kernel for many scenes per launch (the evaluator's joblib fan-out collapses into one call).
"""
import numpy as np
import torch

from .. import _lib
from . import common
from .common import FPS, SAMPLING_RATE, sampling_rate, sweep_params


MAX_GRAD_SCENE = 256         # tb2_sf_sweep_grad's largest scene (kSfGradMaxScene, csrc/classical.cu)


def steps_for(pred_length, rate=SAMPLING_RATE):
    """Simulation steps for pred_length observed frames (socialforce.py:93)."""
    return pred_length * rate


def _params(sf_params, steps, sample_every, fps):
    p = _lib.SfParams()
    p.delta_t = 1.0 / fps
    p.tau, p.v0, p.sigma = float(sf_params[0]), float(sf_params[1]), float(sf_params[2])
    p.n_steps, p.sample_every = int(steps), int(sample_every)
    return p


def simulate_batch(states, batch_split, sf_params=(0.5, 2.1, 0.3), n_steps=steps_for(12), sample_every=SAMPLING_RATE,
                   fps=FPS, device=None):
    """states [A, 6] float64 (x, y, vx, vy, dx, dy) of all scenes, batch_split [B+1] ->
    sampled positions [ceil(n_steps / sample_every), A, 2] float64 (CUDA tensor)."""
    return common.simulate("sf", _params(sf_params, n_steps, sample_every, fps), [(states, torch.float64)],
                           batch_split, (n_steps + sample_every - 1) // sample_every, torch.float64, device)


def rollout(state, speeds, batch_split, sf_params, pred_length, device=None):
    """simulate_batch as `predict` runs it -> positions [pred_length, A, 2] float64 (host)."""
    return simulate_batch(state, batch_split, sf_params, n_steps=steps_for(pred_length), device=device).cpu().numpy()


def _sweep(prepared, params, fps, grad):
    prm = sweep_params(params, np.float64, ("tau", "v0", "sigma"), (0, 2), int(prepared.truth.shape[0]))
    rate = sampling_rate(fps)
    p = _params(prm[0], steps_for(int(prepared.truth.shape[1]), rate), rate, fps)
    return common.sweep("sf", prepared, prm, p, [prepared.state], grad=grad)


def sweep(prepared, params, fps=FPS):
    """ADE / FDE of the primary of every scene of `prepared` (common.PreparedScenes) under every setting of params
    [P, 3] (tau, v0, sigma) -> (ade, fde) CUDA float64 [P, B], one launch (tb2_sf_sweep).  Row s equals
    simulate_batch(state, agent_offsets, params[s], n_steps=steps_for(pred_length, rate), sample_every=rate) with
    rate = sampling_rate(fps), scored against prepared.truth: distances in sample order summed in float64,
    ADE = sum / pred_length, FDE = the last distance.  The trajectories never reach device memory."""
    return _sweep(prepared, params, fps, False)


def sweep_grad(prepared, params, fps=FPS):
    """sweep with derivatives -> (ade, fde, dade, dfde) CUDA float64; ade / fde [P, B] equal sweep's bit for bit,
    dade / dfde [P, B, 3] are d/d(tau, v0, sigma) of them, carried through the rollout in forward mode
    (tb2_sf_sweep_grad).  The field-of-view weight and the speed clip are piecewise: the derivative is that of the
    branch taken.  The library refuses a scene of more than MAX_GRAD_SCENE pedestrians before any launch; the
    parameters are checked as in sweep."""
    return _sweep(prepared, params, fps, True)


def predict(input_paths, dest_dict=None, dest_type='interp', sf_params=[0.5, 2.1, 0.3],
            predict_all=True, n_predict=12, obs_length=9):
    run = lambda state, speeds, batch_split, pred_length: rollout(state, speeds, batch_split, sf_params, pred_length)
    return common.predict(run, input_paths, dest_dict, dest_type, predict_all, n_predict, obs_length, stationary=True)
