"""Every mode of every scene in one batched decode: the evaluator path of the multi-modal predictors (S-GAN, VAE, and the
sampled LSTM modes of lstm/sampling.py, whose decode draws every predicted position from its step's normal).

The per-scene predictors (SGANPredictor / VAEPredictor.__call__) run one encoder pass and then k decoder passes of
pred_length - 1 steps each over the 5-50 tracks of one scene.  Here the encoder runs once over the B scenes of a chunk
(M tracks) and the k decoders run as ONE decode over k * M rows, laid out mode-major: row q * M + m is track m in mode
q, and replica q * B + b is scene b of mode q, a separate scene of one layout.  The layouts use per-scene semantics
(tb2_layout_set_padding(0)), so no pooling ever mixes two modes or two scenes, and every row computes what the
per-scene call computes.  The decoder's starting state comes from one kernel over the encoder state
(tb2_sgan_decoder_context / tb2_vae_decoder_context, csrc/sgan.cu); the replicated observations and encoder positions
are torch copies on the device.

One decode is capped at `rows_per_decode` rows (the engine's workspace per row plus the replicated state per row,
within DECODE_BYTES); above the cap the modes are split into groups.  The random draws are made for all modes before
the split, so the results do not depend on the grouping.
"""
import numpy as np
import torch

from . import _lib
from .engine import _ptr, _stream
from .lstm.lstm import Predictor

# device memory one decode may take: the engine's workspace for its rows plus their replicated state
DECODE_BYTES = 2 << 30


def stateful_pool(body):
    """True for interaction modules that carry an LSTM state of their own through the time loop (NearestNeighborLSTM,
    TrajectronPooling): that state lives in the engine's workspace and is not replicated per mode."""
    return bool(getattr(body.pool, 'stateful', False))


def replicated_split(split, k):
    """batch_split of k mode-major replicas of the scenes `split` (int64 [B + 1]) -> int64 [k * B + 1]."""
    split = np.asarray(split, dtype=np.int64)
    M = int(split[-1])
    out = np.empty(k * (len(split) - 1) + 1, dtype=np.int64)
    out[:-1] = (split[:-1][None, :] + M * np.arange(k, dtype=np.int64)[:, None]).reshape(-1)
    out[-1] = k * M
    return out


def rows_per_decode(handle, layout, num_steps, obs_length, budget=DECODE_BYTES):
    """Rows of one decode: `budget` over the bytes one row takes, i.e. its share of the engine's workspace (which
    grows linearly with the rows of a layout of the same largest scene) plus its replicated observations, normals,
    positions and (h, c) state."""
    M = max(layout.num_tracks, 1)
    ws = int(_lib.load().tb2_lstm_workspace_bytes(handle.handle, layout.handle))
    state = 4 * (num_steps * 7 + obs_length * 2 + 2 * int(handle.config.hidden_dim))
    return max(int(budget // (ws / M + state)), 1)


def observed_batch(body, xys, obs_length, start_length, normalize):
    """(observed float32 [obs_length - start_length, M, 2] on the model's device, batch_split int64 [B + 1],
    rotation [B], centre [B, 2]): the inputs of the per-scene call for every scene, centred / rotated on the device
    (lstm/scene_ops.py) when `normalize`."""
    split = np.zeros(len(xys) + 1, dtype=np.int64)
    split[1:] = np.cumsum([xy.shape[1] for xy in xys])
    device = body._device()
    if normalize:
        from .lstm.scene_ops import preprocess_scenes
        observed, _, _, rotation, center = preprocess_scenes([xy[:obs_length] for xy in xys], device=device,
                                                             normalize_scene=True, obs_length=obs_length)
        return observed[start_length:].contiguous(), split, rotation, center
    host = np.concatenate([xy[start_length:obs_length] for xy in xys], axis=1)
    return torch.from_numpy(host.astype(np.float32)).to(device), split, None, None


GOALS_MESSAGE = "S-GAN / VAE with goal_flag=True are not built (goal-conditioned decoding); goal_flag=True is built for LSTM"


def refuse_goals(model):
    """S-GAN / VAE decode without goals: a goal-conditioned one is refused rather than run on missing inputs."""
    if getattr(model, 'goal_flag', False):
        raise NotImplementedError(GOALS_MESSAGE)


def refuse_input_grad(model, *inputs):
    """S-GAN / VAE have no backward: an input that asks for a gradient is refused rather than left without one."""
    if torch.is_grad_enabled() and any(torch.is_tensor(t) and t.requires_grad for t in inputs):
        raise NotImplementedError("gradients wrt the inputs of %s are not built (it has no backward); call it under "
                                  "torch.no_grad() or detach the inputs" % type(model).__name__)


def sample_positions(normals, positions, eps):
    """positions [rows, 2] += the offset of the normals [rows, 5] at the standard normal pairs eps [rows, 2], in place on
    the device (tb2_lstm_sample_positions)."""
    device = positions.device
    with torch.cuda.device(device):
        _lib.check(_lib.load().tb2_lstm_sample_positions(_ptr(normals), _ptr(positions), _ptr(eps),
                                                         int(positions.shape[0]), _stream(device)))


def predict_modes(body, observed, split, n_predict, modes, context, max_rows=None, eps=None):
    """Encoder once over the scenes of `split`, then the decoders of all `modes` modes.

    context(h_enc, c_enc, q0, q1, h_out, c_out) writes the decoder starting state of modes [q0, q1) into
    h_out / c_out [(q1 - q0) * M, H].  eps: float32 [n_predict, modes * M, 2] on the device, mode-major: every predicted
    position of the decode is drawn from its step's normal (tb2_lstm_forward_steps with eps_dev), the first one, the
    encoder's last output, on the replicated rows before the decoder starts.  Returns the positions of the last
    n_predict steps, float32 [n_predict, modes * M, 2] on the device, mode-major."""
    refuse_goals(body)
    enc = body._encode(body._sequence(observed, split, None, n_predict, pad_to_batch_max=False))
    handle, device, M, S_enc, S = enc.handle, enc.handle.device, enc.layout.num_tracks, enc.S_enc, enc.S
    H = int(body.hidden_dim)
    f32 = dict(dtype=torch.float32, device=device)
    cap = rows_per_decode(handle, enc.layout, S, int(enc.obs.shape[0])) if max_rows is None else int(max_rows)
    per_group = max(1, min(modes, cap // max(M, 1)))
    out = torch.empty((n_predict, modes * M, 2), **f32)
    for q0 in range(0, modes, per_group):
        q1 = min(q0 + per_group, modes)
        kq = q1 - q0
        rows = kq * M
        rep = body._layouts.get(replicated_split(split, kq), False, device=device)
        obs_rep = enc.obs.repeat(1, kq, 1)
        normals, positions = torch.empty((S, rows, 5), **f32), torch.empty((S, rows, 2), **f32)
        positions[:S_enc] = enc.positions[:S_enc].repeat(1, kq, 1)      # the decoder's first inputs
        h, c = torch.empty((rows, H), **f32), torch.empty((rows, H), **f32)
        context(enc.h, enc.c, q0, q1, h, c)
        if eps is None:
            handle.forward_steps(rep, obs_rep, None, enc.n_decode, S_enc, S, normals, positions, h, c)
        else:
            part = eps[:, q0 * M:q1 * M].contiguous()
            sample_positions(enc.normals[S_enc - 1].repeat(kq, 1), positions[S_enc - 1], part[0])
            handle.forward_steps_sampled(rep, obs_rep, None, enc.n_decode, S_enc, S, part, normals, positions, h, c)
        out[:, q0 * M:q1 * M] = positions[S - n_predict:]
    return out


class ModesPredictor(Predictor):
    """Base of the multi-modal predictors (SGANPredictor, VAEPredictor): the per-scene call returns the neighbours in
    mode 0 only, and predict_batch_xy decodes every mode of many scenes at once through _predict_batch_xy."""
    neighbours_every_mode = False
    _model_noun = 'model'       # what the refusal of batched decoding calls the model

    def _lstm_model(self):
        """The LSTM whose engine runs the model."""
        raise NotImplementedError

    def batch_decode_supported(self):
        """predict_batch_xy serves every model except those whose interaction module carries its own LSTM state
        (NearestNeighborLSTM, TrajectronPooling): that state is not replicated per mode."""
        return not stateful_pool(self._lstm_model())

    def _predict_batch_xy(self, xys, n_predict, obs_length, start_length, args, modes, max_rows, make_context,
                          make_eps=None):
        """predict_batch_xy: make_context(device, split, modes) draws the random inputs of every mode and returns the
        context() of predict_modes; make_eps(device, M, modes), if given, returns its eps."""
        body = self._lstm_model()
        if not self.batch_decode_supported():
            raise NotImplementedError("batched decoding of a %s whose interaction module keeps an LSTM state is not "
                                      "built; call the predictor scene by scene" % self._model_noun)
        self.model.eval()
        modes = int(modes)
        if modes < 1:
            raise ValueError("modes must be >= 1")
        if not xys:
            return []
        normalize = bool(getattr(args, 'normalize_scene', False))
        first = start_length if self.start_length_applies else 0
        with torch.no_grad():
            observed, split, rotation, center = observed_batch(body, xys, obs_length, first, normalize)
            context = make_context(observed.device, split, modes)
            eps = make_eps(observed.device, int(split[-1]), modes) if make_eps is not None else None
            pred = predict_modes(body, observed, split, n_predict, modes, context, max_rows, eps)
            return scene_results(pred, split, modes, n_predict, normalize, rotation, center)


def scene_results(pred, split, modes, n_predict, normalize, rotation=None, center=None):
    """Per scene {mode: [primary [n_predict, 2], neighbours [n_predict, N - 1, 2] if mode == 0 else []]} -- the
    dictionary of the per-scene __call__ -- from the mode-major positions of predict_modes."""
    B = len(split) - 1
    M = int(split[-1])
    if normalize:
        from .lstm.scene_ops import inverse_scenes
        pred = inverse_scenes(pred, replicated_split(split, modes), np.tile(rotation, modes),
                              np.tile(np.asarray(center).reshape(B, 2), (modes, 1)))
    else:
        pred = pred.cpu().numpy()
    pred = pred.reshape(n_predict, modes, M, 2)
    results = []
    for i in range(B):
        lo, hi = int(split[i]), int(split[i + 1])
        out = {q: [np.array(pred[:, q, lo]), []] for q in range(modes)}
        out[0][1] = np.array(pred[:, 0, lo + 1:hi])
        results.append(out)
    return results


def group_of_rows(split, device):
    """Scene index of every track, int32 [M] on `device`."""
    split = np.asarray(split, dtype=np.int64)
    return torch.from_numpy(np.repeat(np.arange(len(split) - 1, dtype=np.int32), np.diff(split))).to(device)


def replicated_context(h_enc, c_enc, q0, q1, h_out, c_out):
    """context() of predict_modes where every mode's decoder starts from the encoder state itself."""
    h_out.copy_(h_enc.repeat(q1 - q0, 1))
    c_out.copy_(c_enc.repeat(q1 - q0, 1))


def sgan_context(weight, bias, noise, groups, num_groups, noise_dim):
    """context() of predict_modes for the S-GAN generator: noise [k, num_groups, noise_dim] (None: no noise)."""
    lib = _lib.load()

    def run(h_enc, c_enc, q0, q1, h_out, c_out):
        kq = q1 - q0
        if noise is None:                      # no_noise: the decoder starts from the encoder state (sgan.py:200-204)
            replicated_context(h_enc, c_enc, q0, q1, h_out, c_out)
            return
        part = noise[q0:q1].contiguous()
        device = h_enc.device
        with torch.cuda.device(device):
            _lib.check(lib.tb2_sgan_decoder_context(
                _ptr(weight), _ptr(bias), _ptr(part), _ptr(groups), int(num_groups), _ptr(h_enc), _ptr(c_enc),
                int(h_enc.shape[0]), int(h_enc.shape[1]), int(noise_dim), int(kq), _ptr(h_out), _ptr(c_out),
                _stream(device)))
    return run


def vae_context(weight, bias, z, latent_dim):
    """context() of predict_modes for the VAE: z [k, M, latent_dim], one latent sample per (mode, track)."""
    lib = _lib.load()

    def run(h_enc, c_enc, q0, q1, h_out, c_out):
        part = z[q0:q1].contiguous()
        device = h_enc.device
        with torch.cuda.device(device):
            _lib.check(lib.tb2_vae_decoder_context(
                _ptr(weight), _ptr(bias), _ptr(part), _ptr(h_enc), _ptr(c_enc), int(h_enc.shape[0]),
                int(h_enc.shape[1]), int(latent_dim), int(q1 - q0), _ptr(h_out), _ptr(c_out), _stream(device)))
    return run
