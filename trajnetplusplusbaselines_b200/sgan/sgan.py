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
import ctypes

import numpy as np
import torch
from torch import nn

from .. import _lib, multimodal
from ..data import paths_to_xy
from ..engine import _ptr, _stream
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
        """Encoder steps only; returns the context every mode's decoder starts from."""
        handle = self._engine()
        device = handle.device
        layout = self._layouts.get(batch_split.tolist() if torch.is_tensor(batch_split) else batch_split,
                                   device=self._device())
        M = layout.num_tracks
        if observed.shape[1] != M:
            raise ValueError("batch_split[-1] != number of tracks")
        obs = self._to_device(observed, device)
        obs_length = int(obs.shape[0])
        truth = None
        if prediction_truth is not None:
            if isinstance(prediction_truth, (list, tuple)):
                prediction_truth = torch.stack(list(prediction_truth))
            # sgan.py:367-369 chains (observed[-1:], prediction_truth[:-1]): the last frame is unused
            truth = self._to_device(prediction_truth, device)[:-1].contiguous()
            n_decode = int(truth.shape[0])
            if n_decode == 0:
                truth = None
        else:
            n_decode = int(n_predict) - 1
        S = obs_length - 1 + n_decode
        f32 = dict(dtype=torch.float32, device=device)
        ctx = dict(handle=handle, layout=layout, obs=obs, truth=truth, n_decode=n_decode, S=S, S_enc=obs_length - 1,
                   normals=torch.empty((S, M, 5), **f32), positions=torch.empty((S, M, 2), **f32),
                   h=torch.empty((M, self.hidden_dim), **f32), c=torch.empty((M, self.hidden_dim), **f32),
                   out_device=observed.device)
        handle.forward_steps(layout, obs, truth, n_decode, 0, ctx['S_enc'], ctx['normals'], ctx['positions'],
                             ctx['h'], ctx['c'])
        return ctx

    def decode(self, ctx):
        """One mode: noise into a copy of the encoder state, then the decoder steps."""
        handle, device = ctx['handle'], ctx['handle'].device
        h, c = ctx['h'].clone(), ctx['c'].clone()
        normals, positions = ctx['normals'].clone(), ctx['positions'].clone()
        if not self.no_noise:
            lin = self.mlp_decoder_context[0]
            noise = self._draw_noise(device)
            lib = _lib.load()
            w = lin.weight.detach().to(device=device, dtype=torch.float32).contiguous()
            b = lin.bias.detach().to(device=device, dtype=torch.float32).contiguous()
            with torch.cuda.device(device):
                _lib.check(lib.tb2_sgan_add_noise(_ptr(w), _ptr(b), _ptr(noise), _ptr(h), int(h.shape[0]),
                                                  int(self.hidden_dim), int(self.noise_dim), _stream(device)))
        handle.forward_steps(ctx['layout'], ctx['obs'], ctx['truth'], ctx['n_decode'], ctx['S_enc'], ctx['S'],
                             normals, positions, h, c)
        if int(ctx['obs'].shape[0]) == 2:        # sgan.py:353-354: positions seeded with observed[-1]
            positions = torch.cat([ctx['obs'][-1:].clone(), positions], dim=0)
        if ctx['out_device'] != device:
            normals, positions = self._to_host(normals, positions)
        return normals, positions

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None):
        """sgan.py:301-394: (rel_pred_scene [S, M, 5], pred_scene [S, M, 2])."""
        assert ((prediction_truth is None) + (n_predict is None)) == 1
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("S-GAN training (variety loss / discriminator steps) is not built; "
                                      "call the generator under torch.no_grad()")
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
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("S-GAN training is not built; score under torch.no_grad()")
        body = self._lstm[0]
        handle = body._engine()
        device = handle.device
        seq = torch.cat([body._to_device(observed, device), body._to_device(prediction, device)], dim=0)
        layout = body._layouts.get(batch_split.tolist() if torch.is_tensor(batch_split) else batch_split,
                                   device=body._device())
        M = layout.num_tracks
        S = int(seq.shape[0]) - 1
        f32 = dict(dtype=torch.float32, device=device)
        normals, positions = torch.empty((S, M, 5), **f32), torch.empty((S, M, 2), **f32)
        h, c = torch.empty((M, self.hidden_dim), **f32), torch.empty((M, self.hidden_dim), **f32)
        handle.forward_steps(layout, seq, None, 0, 0, S, normals, positions, h, c)
        prim = torch.as_tensor(layout.offsets[:-1], device=device)
        scores = self.real_classifier(h[prim])
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
        rel_pred_list, pred_list = [], []
        ctx = self.generator.encode(observed, batch_split, prediction_truth, n_predict)   # shared by all modes
        for _ in range(self.k):
            rel_pred_scene, pred_scene = self.generator.decode(ctx)
            rel_pred_list.append(rel_pred_scene)
            pred_list.append(pred_scene)
            if step_type == 'd':
                break
        if self.d_steps and (prediction_truth is not None):
            scores_real = self.discriminator(observed, prediction_truth, goals, batch_split)
            scores_fake = self.discriminator(observed, pred_scene[-pred_length:], goals, batch_split)
            return rel_pred_list, pred_list, scores_real, scores_fake
        return rel_pred_list, pred_list, None, None


class SGANPredictor(object):
    """sgan.py:583-630."""

    def __init__(self, model):
        self.model = model

    def save(self, state, filename):
        with open(filename, 'wb') as f:
            torch.save(self, f)
        with open(filename + '.state', 'wb') as f:
            torch.save(state, f)

    @staticmethod
    def load(filename):
        with open(filename, 'rb') as f:
            return torch.load(f, weights_only=False)

    def __call__(self, paths, scene_goal, n_predict=12, modes=1, predict_all=True, obs_length=9, start_length=0,
                 args=None):
        self.model.eval()
        self.model.d_steps = 0
        if modes is not None:
            self.model.k = modes
        with torch.no_grad():
            xy = paths_to_xy(paths)
            batch_split = [0, xy.shape[1]]
            normalize = bool(getattr(args, 'normalize_scene', False))
            if normalize:
                xy, rotation, center, scene_goal = center_scene(xy, obs_length, goals=np.asarray(scene_goal))
            xy = torch.Tensor(xy)
            scene_goal = torch.Tensor(np.asarray(scene_goal))
            batch_split = torch.Tensor(batch_split).long()
            multimodal_outputs = {}
            _, output_scenes_list, _, _ = self.model(xy[:obs_length], scene_goal, batch_split, n_predict=n_predict)
            for num_p, output_scenes in enumerate(output_scenes_list):
                output_scenes = output_scenes.cpu().numpy()
                if normalize:
                    output_scenes = inverse_scene(output_scenes, rotation, center)
                output_primary = output_scenes[-n_predict:, 0]
                output_neighs = output_scenes[-n_predict:, 1:]
                multimodal_outputs[num_p] = [output_primary, output_neighs if num_p == 0 else []]
        return multimodal_outputs

    def batch_decode_supported(self):
        """predict_batch_xy serves every generator except those whose interaction module carries its own LSTM state
        (NearestNeighborLSTM, TrajectronPooling): that state is not replicated per mode."""
        return not multimodal.stateful_pool(self.model.generator)

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None, modes=1,
                         noise=None, max_rows=None):
        """Every mode of many scenes in one batched decode (the evaluator's column pipeline, multimodal.py).

        xys: list of float64 [n_frames, N_i, 2] as paths_to_xy returns them.  Returns per scene the dictionary of
        __call__, {mode: [primary [n_predict, 2], neighbours if mode == 0 else []]}.  The noise is drawn once per call,
        on the device, one vector per (mode, scene) like the per-scene decodes draw it; `fixed_noise` and `no_noise`
        of the generator apply as in __call__.  noise: explicit [modes, B, noise_dim] vectors instead of the draw.
        max_rows: rows of one decode (default: multimodal.rows_per_decode); more modes are decoded in groups."""
        gen = self.model.generator
        if not self.batch_decode_supported():
            raise NotImplementedError("batched decoding of a generator whose interaction module keeps an LSTM state "
                                      "is not built; call the predictor scene by scene")
        self.model.eval()
        modes = int(modes)
        if modes < 1:
            raise ValueError("modes must be >= 1")
        if not xys:
            return []
        normalize = bool(getattr(args, 'normalize_scene', False))
        with torch.no_grad():
            # sgan.py:603 feeds xy[:obs_length]: start_length does not apply to the generator
            observed, split, rotation, center = multimodal.observed_batch(gen, xys, obs_length, 0, normalize)
            device = observed.device
            B, nd = len(xys), int(gen.noise_dim)
            if gen.no_noise:
                noise = None
            elif noise is not None:
                noise = torch.as_tensor(noise, dtype=torch.float32).to(device).reshape(modes, B, nd).contiguous()
            elif gen.fixed_noise is not None:
                fixed = torch.as_tensor(gen.fixed_noise, dtype=torch.float32).to(device).reshape(1, 1, nd)
                noise = fixed.expand(modes, B, nd).contiguous()
            else:
                noise = get_noise((modes, B, nd), gen.noise_type, device=device).float().contiguous()
            lin = gen.mlp_decoder_context[0]
            w = lin.weight.detach().to(device=device, dtype=torch.float32).contiguous()
            b = lin.bias.detach().to(device=device, dtype=torch.float32).contiguous()
            context = multimodal.sgan_context(w, b, noise, multimodal.group_of_rows(split, device), B, nd)
            pred = multimodal.predict_modes(gen, observed, split, n_predict, modes, context, max_rows)
            return multimodal.scene_results(pred, split, modes, n_predict, normalize, rotation, center)
