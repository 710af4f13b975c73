"""The handcrafted baselines on the evaluator's column pipeline: one predictor object per model of
classical/trajnet_evaluator.py (kf, sf, sf_opt, orca, orca_opt, cv) with `predict_batch_xy`.

The reference calls each model's `predict(paths, ...)` once per scene under joblib (classical/trajnet_evaluator.py:91).
Here a chunk of scenes goes through one call: social force and ORCA simulate every pedestrian of the chunk in one
`simulate_batch` launch (their `rollout`), the Kalman filter fits every track of the chunk in one device launch
(kalman.predict_concat_device), constant velocity is one NumPy expression.  Per scene the result equals the
per-scene `predict` on the preprocessed paths (kalman.predict(..., n_samples=0) for kf without noise), so
evaluator.evaluate_file writes the bytes the row pipeline writes from those per-scene results.

The reference's classical predict_scene ignores `modes`: every predictor returns {0: (primary, neighbours)} per scene,
so only mode 0 is written (into the `_modes<k>` folder), at any `modes`.
"""
import numpy as np

from . import kalman, orca, socialforce
from .common import initial_states_xy


def _split(out, offsets):
    """[T, A, 2] positions of all pedestrians -> per scene {0: (primary [T, 2], neighbours [T, K, 2])}."""
    return [{0: (out[:, lo, 0:2], out[:, lo + 1:hi, 0:2])} for lo, hi in zip(offsets[:-1], offsets[1:])]


class SimulatorBatch:
    """simulator.predict(paths, params) for every scene of a chunk, `simulator` the socialforce or orca module: one
    simulator.rollout launch."""

    def __init__(self, simulator, params, device=None):
        self.simulator = simulator
        self.params = [float(v) for v in params]
        self.device = device

    def predict_batch_xy(self, xys, n_predict=12, obs_length=9, args=None, modes=1):
        if not xys:
            return []
        state, speeds, offsets, _ = initial_states_xy([(None, xy) for xy in xys], obs_length, n_predict, truth=False)
        out = self.simulator.rollout(state, speeds, offsets, self.params, n_predict, device=self.device)
        return _split(out, offsets)


class SocialForceBatch(SimulatorBatch):
    def __init__(self, sf_params=(0.5, 2.1, 0.3), device=None):
        super().__init__(socialforce, sf_params, device)
        self.sf_params = self.params


class OrcaBatch(SimulatorBatch):
    def __init__(self, orca_params=(1.5, 1.5, 0.4), device=None):
        super().__init__(orca, orca_params, device)
        self.orca_params = self.params


def kalman_tracks_xy(xy, obs_length):
    """The tracks kalman.predict fits for one scene (kalman.py:25-29): the pedestrians present at the last observed
    frame with at least 2 past rows, in path order.  -> (columns [K], rows [sum T_i, 2], lengths [K])."""
    t0 = obs_length - 1
    present = ~np.isnan(xy[:t0 + 1, :, 0])                    # [t0 + 1, N]
    cols = np.nonzero(present[t0] & (present.sum(axis=0) >= 2))[0]
    mask = present[:, cols].T                                  # [K, t0 + 1]: each track's rows in frame order
    rows = xy[:t0 + 1, cols].transpose(1, 0, 2)[mask]
    return cols, rows, mask.sum(axis=1)


class KalmanBatch:
    """kalman.predict(paths, n_samples=...) for every scene of a chunk: the tracks of all scenes in one device launch
    (tb2_kalman_predict_device).  n_samples = 0: the expectation, bit-identical to the host path; n_samples >= 1: the
    mean of n_samples sampled rollouts from torch's generator `generator` (DESIGN §8)."""

    def __init__(self, n_samples=5, em_iterations=10, generator=None, device=None):
        self.n_samples = int(n_samples)
        self.em_iterations = int(em_iterations)
        self.generator = generator
        self.device = device

    def predict_batch_xy(self, xys, n_predict=12, obs_length=9, args=None, modes=1):
        per_scene = [kalman_tracks_xy(xy, obs_length) for xy in xys]
        counts = np.array([len(c) for c, _, _ in per_scene], dtype=np.int64)
        tracks = [t for _, rows, n in per_scene if len(n) for t in np.split(rows, np.cumsum(n)[:-1])]
        obs, offsets = kalman.concat_tracks(tracks)
        pred = kalman.predict_concat_device(obs, offsets, n_predict=n_predict, n_samples=self.n_samples,
                                            em_iterations=self.em_iterations, generator=self.generator,
                                            device=self.device)[0].cpu().numpy()
        out, lo = [], 0
        for (cols, _, _), k in zip(per_scene, counts):
            tracks = pred[lo:lo + k]
            lo += k
            primary, first = (tracks[0], 1) if k and cols[0] == 0 else (None, 0)
            neighbours = tracks[first:].transpose(1, 0, 2) if k > first else []
            out.append({0: (primary, neighbours)})
        return out


class ConstantVelocityBatch:
    """constant_velocity.predict for every scene of a chunk, one NumPy expression with the same float64 operations:
    last + i * (last - previous), i = 1 .. n_predict."""

    def predict_batch_xy(self, xys, n_predict=12, obs_length=9, args=None, modes=1):
        if not xys:
            return []
        last = np.concatenate([xy[-1] for xy in xys])              # [A, 2]
        velocity = last - np.concatenate([xy[-2] for xy in xys])
        out = last + np.array([i * velocity for i in range(1, n_predict + 1)])
        offsets = np.cumsum([0] + [xy.shape[1] for xy in xys])
        return _split(out, offsets)


# the models of classical/trajnet_evaluator.py, in the reference's order, and their settings (predict_scene, :14-28)
MODELS = ('kf', 'sf', 'sf_opt', 'orca', 'orca_opt', 'cv')


def load_predictor(model_name, kf_samples=5, generator=None, device=None):
    """The batched predictor of a model name as the reference's load_predictor / predict_scene resolve it
    ('kf' / 'sf_opt' / 'orca_opt' / 'sf' / 'orca' / 'cv', with or without the `_modes<k>` suffix or `.pkl`)."""
    if 'kf' in model_name:
        return KalmanBatch(n_samples=kf_samples, generator=generator, device=device)
    if 'sf_opt' in model_name:
        return SocialForceBatch([0.5, 5.0, 0.3], device=device)
    if 'orca_opt' in model_name:
        return OrcaBatch([0.4, 1.0, 0.3], device=device)
    if 'sf' in model_name:
        return SocialForceBatch(device=device)
    if 'orca' in model_name:
        return OrcaBatch(device=device)
    if 'cv' in model_name:
        return ConstantVelocityBatch()
    raise NotImplementedError(model_name)
