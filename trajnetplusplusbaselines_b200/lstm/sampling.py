"""Multi-modal predictions of an LSTM model: every mode after the first samples its trajectory from the model's own
per-step bivariate normal instead of following the mean.

This goes beyond the reference, whose LSTMPredictor (lstm/lstm.py:266-313) returns k identical copies of the mean
trajectory at `modes` k (every step feeds back obs2 + mu, lstm.py:232,255).  Each step already predicts the density
PredictionLoss trains, N(mu, [[sx^2, rho sx sy], [rho sx sy, sy^2]]); Social-LSTM (Alahi et al. 2016) draws its
test-time trajectories from it.  Here, for mode q >= 1, every predicted position (the last encoder step's output and
every decoder step's, of every present track) is

    pos = obs2 + mu + (sx e1, sy (rho e1 + sqrt(1 - rho^2) e2)),   (e1, e2) ~ N(0, I),

and that draw is what the next step is fed back.  Mode 0 is the mean trajectory (e = 0), bit for bit that of
LSTMPredictor; rows with NaN normals stay NaN.  The pairs are one float32 tensor eps [n_predict, k * M, 2], mode-major,
drawn per call on the model's device with torch.randn (mode 0 zeroed) before any split of the modes into decode groups,
so the results do not depend on the grouping.  `fixed_eps` (argument or attribute) replaces the draw.
"""
import torch

from .. import multimodal

GOALS_MESSAGE = "sampled predictions of a goal-conditioned LSTM (goal_flag=True) are not built"


def draw_eps(device, rows, modes, n_predict, fixed_eps=None):
    """eps float32 [n_predict, modes * rows, 2] on `device`: fixed_eps as given, else standard normal draws with mode 0
    (the first `rows` columns) zeroed."""
    if fixed_eps is not None:
        eps = torch.as_tensor(fixed_eps, dtype=torch.float32).to(device)
        if tuple(eps.shape) != (n_predict, modes * rows, 2):
            raise ValueError("fixed_eps must be [n_predict, modes * M, 2] = [%d, %d, 2], got %s"
                             % (n_predict, modes * rows, list(eps.shape)))
        return eps.contiguous()
    eps = torch.randn((n_predict, modes * rows, 2), dtype=torch.float32, device=device)
    eps[:, :rows] = 0.0
    return eps


class SampledLSTMPredictor(multimodal.ModesPredictor):
    """Sampled multi-modal predictor of an LSTM model (see the module docstring).

    predict_batch_xy decodes every mode of many scenes at once (the evaluator's column pipeline: the encoder once over
    the chunk, then one sampled decode of k * M rows per mode group); __call__ runs one sampled forward per mode of one
    scene, the path of interaction modules with their own LSTM state (nn_lstm, traj_pool), which the batched decode does
    not replicate.  Neighbours are returned in mode 0 only.  `fixed_eps` ([n_predict, modes * N, 2] of the call's N
    tracks) replaces the random draw of every call while set."""
    _model_noun = 'LSTM model'

    def __init__(self, model):
        super().__init__(model)
        self.fixed_eps = None
        self._refuse_goals()

    def _refuse_goals(self):
        if getattr(self.model, 'goal_flag', False):
            raise NotImplementedError(GOALS_MESSAGE)

    def _lstm_model(self):
        return self.model

    def _mode_scenes(self, observed, scene_goal, batch_split, n_predict, modes):
        self._refuse_goals()
        body = self.model
        seq = body._sequence(observed, batch_split, None, n_predict)
        M = seq.layout.num_tracks
        eps = draw_eps(seq.handle.device, M, modes, n_predict, self.fixed_eps)
        for q in range(modes):        # one sampled forward per mode, each mode's outputs handled before the next forward
            if q > 0:
                seq = body._sequence(observed, batch_split, None, n_predict)
            seq.handle.forward_steps_sampled(seq.layout, seq.obs, None, seq.n_decode, 0, seq.S,
                                             eps[:, q * M:(q + 1) * M].contiguous(), seq.normals, seq.positions, seq.h,
                                             seq.c)
            yield body._results(seq, seq.normals, seq.positions)[1]

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None, modes=1,
                         fixed_eps=None, max_rows=None):
        """Every mode of many scenes in one batched decode (multimodal.predict_modes).

        xys: list of float64 [n_frames, N_i, 2] as paths_to_xy returns them.  Returns per scene the dictionary of
        __call__, {mode: [primary [n_predict, 2], neighbours if mode == 0 else []]}.  fixed_eps: [n_predict, modes * M,
        2] pairs of the chunk's M tracks (mode-major) instead of the draw.  max_rows: rows of one decode (default:
        multimodal.rows_per_decode); more modes are decoded in groups."""
        self._refuse_goals()
        fixed = fixed_eps if fixed_eps is not None else self.fixed_eps

        def make_eps(device, rows, modes):
            return draw_eps(device, rows, modes, int(n_predict), fixed)

        return self._predict_batch_xy(xys, n_predict, obs_length, start_length, args, modes, max_rows,
                                      lambda device, split, modes: multimodal.replicated_context, make_eps)

