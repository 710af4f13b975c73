"""VAE forecaster + predictor with the reference's API, inference side (SURVEY.md 8f rank 2).

Mirrors trajnetbaselines/vae/vae.py: VAE :26-315, VAEEncoder :317-332, VAEDecoder :334-345,
VAEPredictor :347-398, utils.sample_multivariate_distribution (vae/utils.py:4-24).  The step is the
LSTM step of lstm/lstm.py (same kernels, `obs_encoder` in the encoder slot); at test time the latent
sample rescales the encoder state, h <- h * ReLU(fc z) (add_noise :87-106 -> tb2_vae_scale_hidden),
and each of the num_modes decodes from that state.  The observation encoder runs once.  Same
constructor arguments and state_dict keys.  Training (prediction encoder, KL term) is not built:
model.train() + forward raises.  VAEPredictor.predict_batch_xy decodes every mode of many scenes at
once (the evaluator's path, ../multimodal.py).
"""
import numpy as np
import torch

from .. import _lib, multimodal
from ..engine import _ptr, _stream, linear_on
from ..lstm.lstm import LSTM, center_scene, drop_distant, inverse_scene  # noqa: F401
from ..lstm.modules import Hidden2Normal, InputEmbedding


def sample_multivariate_distribution(mean, var_log):
    """vae/utils.py:4-24: one N(mean, diag(exp(var_log))) sample per track (numpy RNG, like the reference)."""
    mean = mean.detach().cpu().numpy()
    std = np.exp(0.5 * var_log.detach().cpu().numpy())
    return torch.from_numpy((mean + std * np.random.standard_normal(mean.shape)).astype(np.float32))


class VAEEncoder(torch.nn.Module):
    """vae.py:317-332 (parameters; used by the reference at training time only when desire=True)."""

    def __init__(self, input_dim, output_dim):
        super().__init__()
        self.input_dim, self.output_dim = input_dim, output_dim
        self.fc_mu = torch.nn.Linear(self.input_dim, self.output_dim // 2)
        self.fc_var = torch.nn.Linear(self.input_dim, self.output_dim // 2)
        self.relu = torch.nn.ReLU()

    def forward(self, inputs):
        inputs = torch.reshape(torch.stack(list(inputs)) if isinstance(inputs, (list, tuple)) else inputs,
                               (-1, self.input_dim))
        return self.relu(self.fc_mu(inputs)), 0.01 + self.relu(self.fc_var(inputs))


class VAEDecoder(torch.nn.Module):
    """vae.py:334-345."""

    def __init__(self, input_dim, output_dim):
        super().__init__()
        self.input_dim, self.output_dim = input_dim, output_dim
        self.fc = torch.nn.Linear(self.input_dim, self.output_dim)
        self.relu = torch.nn.ReLU()

    def forward(self, inputs):
        return self.relu(self.fc(torch.reshape(inputs, (-1, self.input_dim))))


class VAE(torch.nn.Module):
    """vae.py:26-315.  `fixed_z` (tensor [num_modes, M, latent_dim]) replaces the random draws when set."""

    def __init__(self, embedding_dim=64, hidden_dim=128, pool=None, pool_to_input=True, goal_dim=None,
                 goal_flag=False, num_modes=1, latent_dim=128):
        super().__init__()
        body = LSTM(embedding_dim, hidden_dim, pool, pool_to_input, goal_dim, goal_flag)
        self._body = [body]                    # engine owner; its modules are registered below under the reference's names
        self.hidden_dim = hidden_dim
        self.embedding_dim = embedding_dim
        self.pool = pool
        self.pool_to_input = pool_to_input
        self.input_embedding = body.input_embedding
        self.goal_flag = goal_flag
        self.goal_dim = body.goal_dim
        self.goal_embedding = body.goal_embedding
        self.obs_encoder = body.encoder
        in_dim = body.encoder.weight_ih.shape[1]
        self.pred_encoder = torch.nn.LSTMCell(in_dim, hidden_dim)
        self.decoder = body.decoder
        self.hidden2normal = body.hidden2normal
        self.latent_dim = latent_dim
        self.num_modes = num_modes
        self.desire = True
        self.vae_encoder_xy = VAEEncoder(2 * hidden_dim, 2 * latent_dim)
        self.vae_encoder_x = VAEEncoder(hidden_dim, 2 * latent_dim)
        self.vae_decoder = VAEDecoder(latent_dim, hidden_dim)
        self.fixed_z = None

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None):
        """(rel_pred_scene list, pred_scene list, z_distr_xy, z_distr_x), vae.py:188-315 in eval mode."""
        assert ((prediction_truth is None) + (n_predict is None)) == 1
        multimodal.refuse_goals(self)
        if self.training or (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("VAE training (prediction encoder, KL term) is not built; use "
                                      "model.eval() under torch.no_grad()")
        multimodal.refuse_input_grad(self, observed, prediction_truth)
        if not self.desire:
            raise NotImplementedError("desire=False (latent prior from vae_encoder_x) is not built")
        body = self._body[0]
        seq = body._encode(body._sequence(observed, batch_split, prediction_truth, n_predict))
        device, M = seq.handle.device, seq.layout.num_tracks
        lib = _lib.load()
        w, b = linear_on(self.vae_decoder.fc, device)
        rel_list, pred_list = [], []
        for k in range(self.num_modes):
            if self.fixed_z is not None:
                z = torch.as_tensor(self.fixed_z[k], dtype=torch.float32)
            else:      # prior N(0, exp(1) I): z_mu_obs = 0, z_var_log_obs = 1 (vae.py:277-278)
                z = sample_multivariate_distribution(torch.zeros(M, self.latent_dim), torch.ones(M, self.latent_dim))
            z = z.to(device).contiguous()

            def scale_hidden(h, c):
                with torch.cuda.device(device):
                    _lib.check(lib.tb2_vae_scale_hidden(_ptr(w), _ptr(b), _ptr(z), _ptr(h), M, int(self.hidden_dim),
                                                        int(self.latent_dim), _stream(device)))
            normals, positions = body._decode(seq, scale_hidden, seed=False)
            rel_list.append(normals)
            pred_list.append(positions)
        return rel_list, pred_list, None, None


class VAEPredictor(multimodal.ModesPredictor):
    """vae.py:347-398."""

    def _lstm_model(self):
        return self.model._body[0]

    def _mode_scenes(self, observed, scene_goal, batch_split, n_predict, modes):
        self.model.num_modes = modes
        return self.model(observed, scene_goal, batch_split, n_predict=n_predict)[1]

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None, modes=1,
                         z=None, max_rows=None):
        """Every mode of many scenes in one batched decode (the evaluator's column pipeline, multimodal.py).

        xys: list of float64 [n_frames, N_i, 2] as paths_to_xy returns them.  Returns per scene the dictionary of
        __call__, {mode: [primary [n_predict, 2], neighbours if mode == 0 else []]}.  The latent samples are drawn once
        per call, on the device, one per (mode, track) from the prior N(0, e I) as in __call__; the model's `fixed_z`
        ([modes, M, latent_dim] over the M tracks of all scenes) replaces the draw, and so does z (same shape).
        max_rows: rows of one decode (default: multimodal.rows_per_decode); more modes are decoded in groups."""
        if not self.model.desire:
            raise NotImplementedError("desire=False (latent prior from vae_encoder_x) is not built")

        def context(device, split, modes):
            M, L = int(split[-1]), int(self.model.latent_dim)
            draws = self.model.fixed_z if z is None else z
            if draws is not None:
                draws = torch.as_tensor(draws, dtype=torch.float32).to(device).reshape(modes, M, L).contiguous()
            else:      # prior N(0, exp(1) I): z_mu_obs = 0, z_var_log_obs = 1 (vae.py:277-278)
                draws = torch.randn((modes, M, L), device=device).mul_(float(np.exp(0.5)))
            w, b = linear_on(self.model.vae_decoder.fc, device)
            return multimodal.vae_context(w, b, draws, L)
        return self._predict_batch_xy(xys, n_predict, obs_length, start_length, args, modes, max_rows, context)
