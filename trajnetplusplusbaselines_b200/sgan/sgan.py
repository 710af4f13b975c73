"""S-GAN generator / discriminator / predictor with the reference's API, inference side, backed by
libtrajnet_b200 (SURVEY.md 8f rank 2).

Mirrors trajnetbaselines/sgan/sgan.py: get_noise :27-32, make_mlp :34-45, SGAN :47-133,
LSTMGenerator :135-394, LSTMDiscriminator :396-581, SGANPredictor :583-630.  The generator's step
is the LSTM step of lstm/lstm.py (same kernels); what differs is the noise injection between
encoder and decoder (adding_noise :200-221 -> tb2_sgan_add_noise) and the k-mode loop.  The encoder
is deterministic, so it runs ONCE and every mode restarts from a copy of its state
(tb2_lstm_forward_steps); the reference re-runs it per mode.  Same constructor arguments and
state_dict keys (reference checkpoints load verbatim).  GAN training (variety loss, discriminator
steps) is not built: forward under grad mode raises.  SGANPredictor.predict_batch_xy decodes every mode
of many scenes at once (the evaluator's path, ../multimodal.py).
"""
import torch
from torch import nn

from .. import _lib, multimodal
from ..engine import _ptr, _stream, linear_on
from ..lstm.lstm import LSTM, center_scene, drop_distant, inverse_scene  # noqa: F401


def get_noise(shape, noise_type, device):
    """sgan.py:27-32."""
    if noise_type == 'gaussian':
        return torch.randn(*shape, device=device)
    if noise_type == 'uniform':
        return torch.rand(*shape, device=device).sub_(0.5).mul_(2.0)
    raise ValueError('Unrecognized noise type "%s"' % noise_type)


def make_mlp(dim_list, activation='relu', batch_norm=True, dropout=0):
    """sgan.py:34-45 (an activation follows every Linear, the last one included)."""
    layers = []
    for dim_in, dim_out in zip(dim_list[:-1], dim_list[1:]):
        layers.append(nn.Linear(dim_in, dim_out))
        if activation == 'relu':
            layers.append(nn.ReLU())
        elif activation == 'leakyrelu':
            layers.append(nn.LeakyReLU())
        if dropout > 0:
            layers.append(nn.Dropout(p=dropout))
    return nn.Sequential(*layers)


class LSTMGenerator(LSTM):
    """sgan.py:135-394.  `fixed_noise` (tensor [noise_dim]) replaces the random draw when set."""

    def __init__(self, embedding_dim=64, hidden_dim=128, pool=None, pool_to_input=True, goal_dim=None,
                 goal_flag=False, noise_dim=8, no_noise=False, noise_type='gaussian'):
        super().__init__(embedding_dim, hidden_dim, pool, pool_to_input, goal_dim, goal_flag)
        self.noise_dim = noise_dim
        self.no_noise = no_noise
        self.noise_type = noise_type
        self.mlp_decoder_context = make_mlp([self.hidden_dim, self.hidden_dim - self.noise_dim])
        self.fixed_noise = None

    def _draw_noise(self, device):
        if self.fixed_noise is not None:
            return torch.as_tensor(self.fixed_noise, dtype=torch.float32).to(device).contiguous()
        return get_noise((self.noise_dim,), self.noise_type, device=device).float().contiguous()

    def encode(self, observed, batch_split, prediction_truth, n_predict):
        """Encoder steps only; returns the sequence every mode's decoder starts from."""
        multimodal.refuse_goals(self)
        if prediction_truth is not None:
            # sgan.py:367-369 chains (observed[-1:], prediction_truth[:-1]): the last frame is unused
            prediction_truth = prediction_truth[:-1]
        return self._encode(self._sequence(observed, batch_split, prediction_truth, n_predict))

    def decode(self, seq):
        """One mode: noise into a copy of the encoder state, then the decoder steps."""
        return self._decode(seq, self._add_noise)

    def _add_noise(self, h, c):
        """h <- [ReLU(mlp_decoder_context(h)), noise] in place, one noise draw for every track (sgan.py:200-221)."""
        if self.no_noise:
            return
        device = h.device
        noise = self._draw_noise(device)
        w, b = linear_on(self.mlp_decoder_context[0], device)
        with torch.cuda.device(device):
            _lib.check(_lib.load().tb2_sgan_add_noise(_ptr(w), _ptr(b), _ptr(noise), _ptr(h), int(h.shape[0]),
                                                      int(self.hidden_dim), int(self.noise_dim), _stream(device)))

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None):
        """sgan.py:301-394: (rel_pred_scene [S, M, 5], pred_scene [S, M, 2])."""
        assert ((prediction_truth is None) + (n_predict is None)) == 1
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("S-GAN training (variety loss / discriminator steps) is not built; "
                                      "call the generator under torch.no_grad()")
        multimodal.refuse_input_grad(self, observed, prediction_truth)
        return self.decode(self.encode(observed, batch_split, prediction_truth, n_predict))


class LSTMDiscriminator(torch.nn.Module):
    """sgan.py:396-581: encoder-only LSTM over [observed; prediction], an MLP scores the primaries."""

    def __init__(self, embedding_dim=64, hidden_dim=128, pool=None, pool_to_input=True, goal_dim=None,
                 goal_flag=False):
        super().__init__()
        # the recurrence is the LSTM step; decoder / head slots of the engine are never read here
        self._lstm = [LSTM(embedding_dim, hidden_dim, pool, pool_to_input, goal_dim, goal_flag)]
        body = self._lstm[0]
        self.hidden_dim = hidden_dim
        self.embedding_dim = embedding_dim
        self.pool = pool
        self.pool_to_input = pool_to_input
        self.input_embedding = body.input_embedding
        self.goal_flag = goal_flag
        self.goal_dim = body.goal_dim
        self.goal_embedding = body.goal_embedding
        self.encoder = body.encoder
        self.real_classifier = make_mlp([hidden_dim, int(hidden_dim / 2), int(hidden_dim / 4), 1])

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        body = self._lstm[0]       # decoder / hidden2normal of the shared body are not registered here
        body.decoder._apply(fn)
        body.hidden2normal._apply(fn)
        return out

    def forward(self, observed, prediction, goals, batch_split):
        """scores [batch_size, 1] of the primary tracks (sgan.py:524-581)."""
        multimodal.refuse_goals(self)
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("S-GAN training is not built; score under torch.no_grad()")
        multimodal.refuse_input_grad(self, observed, prediction)
        body = self._lstm[0]
        # n_predict = 1: no decoder step, every frame of [observed; prediction] goes through the encoder
        seq = body._encode(body._sequence(torch.cat([observed, prediction], dim=0), batch_split, None, 1))
        device = seq.handle.device
        prim = torch.as_tensor(seq.layout.offsets[:-1], device=device)
        scores = self.real_classifier(seq.h[prim])
        return scores if observed.device == device else scores.to(observed.device)


class SGAN(torch.nn.Module):
    """sgan.py:47-133 (inference side: k generator modes, discriminator scores when asked for)."""

    def __init__(self, generator=None, discriminator=None, k=1, d_steps=1, g_steps=1):
        super().__init__()
        self.generator = generator if generator is not None else LSTMGenerator()
        self.g_steps = g_steps
        self.discriminator = discriminator if discriminator is not None else LSTMDiscriminator()
        self.d_steps = d_steps
        self.k = k

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None, step_type='g',
                pred_length=12):
        assert ((prediction_truth is None) + (n_predict is None)) == 1
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("S-GAN training is not built; call under torch.no_grad()")
        multimodal.refuse_input_grad(self, observed, prediction_truth)
        rel_pred_list, pred_list = [], []
        seq = self.generator.encode(observed, batch_split, prediction_truth, n_predict)   # shared by all modes
        for _ in range(self.k):
            rel_pred_scene, pred_scene = self.generator.decode(seq)
            rel_pred_list.append(rel_pred_scene)
            pred_list.append(pred_scene)
            if step_type == 'd':
                break
        if self.d_steps and (prediction_truth is not None):
            scores_real = self.discriminator(observed, prediction_truth, goals, batch_split)
            scores_fake = self.discriminator(observed, pred_scene[-pred_length:], goals, batch_split)
            return rel_pred_list, pred_list, scores_real, scores_fake
        return rel_pred_list, pred_list, None, None


class SGANPredictor(multimodal.ModesPredictor):
    """sgan.py:583-630."""
    start_length_applies = False     # sgan.py:603 feeds xy[:obs_length]
    _model_noun = 'generator'

    def _lstm_model(self):
        return self.model.generator

    def _mode_scenes(self, observed, scene_goal, batch_split, n_predict, modes):
        self.model.d_steps = 0
        if modes is not None:
            self.model.k = modes
        return self.model(observed, scene_goal, batch_split, n_predict=n_predict)[1]

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None, modes=1,
                         noise=None, max_rows=None):
        """Every mode of many scenes in one batched decode (the evaluator's column pipeline, multimodal.py).

        xys: list of float64 [n_frames, N_i, 2] as paths_to_xy returns them.  Returns per scene the dictionary of
        __call__, {mode: [primary [n_predict, 2], neighbours if mode == 0 else []]}.  The noise is drawn once per call,
        on the device, one vector per (mode, scene) like the per-scene decodes draw it; `fixed_noise` and `no_noise`
        of the generator apply as in __call__.  noise: explicit [modes, B, noise_dim] vectors instead of the draw.
        max_rows: rows of one decode (default: multimodal.rows_per_decode); more modes are decoded in groups."""
        gen = self.model.generator

        def context(device, split, modes):
            B, nd = len(split) - 1, int(gen.noise_dim)
            if gen.no_noise:
                draws = None
            elif noise is not None:
                draws = torch.as_tensor(noise, dtype=torch.float32).to(device).reshape(modes, B, nd).contiguous()
            elif gen.fixed_noise is not None:
                fixed = torch.as_tensor(gen.fixed_noise, dtype=torch.float32).to(device).reshape(1, 1, nd)
                draws = fixed.expand(modes, B, nd).contiguous()
            else:
                draws = get_noise((modes, B, nd), gen.noise_type, device=device).float().contiguous()
            w, b = linear_on(gen.mlp_decoder_context[0], device)
            return multimodal.sgan_context(w, b, draws, multimodal.group_of_rows(split, device), B, nd)
        return self._predict_batch_xy(xys, n_predict, obs_length, start_length, args, modes, max_rows, context)
