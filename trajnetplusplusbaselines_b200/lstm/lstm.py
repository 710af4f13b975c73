"""LSTM forecaster + predictor with the reference's API, backed by libtrajnet_b200.

Mirrors trajnetbaselines/lstm/lstm.py: drop_distant :16-22, LSTM :45-264, LSTMPredictor
:266-313.  Same constructor arguments, same state_dict keys (SURVEY.md 8b/B2), same
forward signature and return shapes; the time loop, the per-step mask / embed / pool /
LSTMCell / Gaussian head and the decoder feedback rule all run on the GPU through
tb2_lstm_forward_steps (csrc/capi.cu).  There is no torch or CPU implementation of the
step in this package: without the CUDA library the calls raise.
"""
import math
from collections import namedtuple

import numpy as np
import torch

from .. import _lib
from ..data import paths_to_xy
from ..engine import LayoutCache, ModelHandle, lstm_config, weights_key
from .external import EXTERNAL_GOALS_MESSAGE, external_forward, external_step, is_external, scene_size_groups
from .modules import Hidden2Normal, InputEmbedding

NAN = float('nan')

# the fused sequence calls (S-GAN / VAE decoding, sampled modes) read a built-in module's configuration; a module of the
# caller's runs only through LSTM.forward / LSTM.step
EXTERNAL_FUSED_MESSAGE = ("%s is an external interaction module (it has no fill_config): LSTM.forward, LSTM.step and "
                          "LSTMPredictor run it; S-GAN / VAE and sampled predictions with it are not built")

# one forward set up by LSTM._sequence
Sequence = namedtuple('Sequence', 'handle layout obs truth n_decode S_enc S normals positions h c out_device goals')


def drop_distant(xy, r=6.0):
    """Drops pedestrians more than r meters away from the primary ped (lstm.py:16-22)."""
    distance_2 = np.sum(np.square(xy - xy[:, 0:1]), axis=2)
    mask = np.nanmin(distance_2, axis=0) < r**2
    return xy[:, mask], mask


def theta_rotation(xy, theta):
    """Reference lstm/utils.py:24-30 (math.cos / math.sin of the scalar angle, like the reference)."""
    ct, st = math.cos(theta), math.sin(theta)
    r = np.array([[ct, st], [-st, ct]])
    return np.einsum('ptc,ci->pti', xy, r)


def center_scene(xy, obs_length=9, ped_id=0, goals=None):
    """Host-side scene normalisation (reference lstm/utils.py:32-51)."""
    if goals is not None:
        goals = goals[np.newaxis, :, :]
    center = xy[obs_length - 1, ped_id]
    xy = xy - center[np.newaxis, np.newaxis, :]
    if goals is not None:
        goals = goals - center[np.newaxis, np.newaxis, :]
    last_obs = xy[obs_length - 1, ped_id]
    second_last_obs = xy[obs_length - 2, ped_id]
    diff = np.array([last_obs[0] - second_last_obs[0], last_obs[1] - second_last_obs[1]])
    thet = np.arctan2(diff[1], diff[0])
    rotation = -thet + np.pi / 2
    xy = theta_rotation(xy, rotation)
    if goals is not None:
        goals = theta_rotation(goals, rotation)
        return xy, rotation, center, goals[0]
    return xy, rotation, center


def inverse_scene(xy, rotation, center):
    """Reference augmentation.py:65-68."""
    xy = theta_rotation(xy, -rotation)
    return xy + center[np.newaxis, np.newaxis, :]


class LSTM(torch.nn.Module):
    def __init__(self, embedding_dim=64, hidden_dim=128, pool=None, pool_to_input=True, goal_dim=None, goal_flag=False):
        """Same arguments as the reference (lstm.py:46-60)."""
        super().__init__()
        self.hidden_dim = hidden_dim
        self.embedding_dim = embedding_dim
        self.pool = pool
        self.pool_to_input = pool_to_input

        scale = 4.0
        self.input_embedding = InputEmbedding(2, self.embedding_dim, scale)

        self.goal_flag = goal_flag
        self.goal_dim = goal_dim or embedding_dim
        self.goal_embedding = InputEmbedding(2, self.goal_dim, scale)
        goal_rep_dim = self.goal_dim if self.goal_flag else 0

        pooling_dim = 0
        if pool is not None and self.pool_to_input:
            pooling_dim = self.pool.out_dim

        self.encoder = torch.nn.LSTMCell(self.embedding_dim + goal_rep_dim + pooling_dim, self.hidden_dim)
        self.decoder = torch.nn.LSTMCell(self.embedding_dim + goal_rep_dim + pooling_dim, self.hidden_dim)
        self.hidden2normal = Hidden2Normal(self.hidden_dim)

        self._handle = None
        self._layouts = LayoutCache()
        self._pinned = {}

    # -- engine plumbing ---------------------------------------------------------------------
    def _device(self):
        return self.hidden2normal.linear.weight.device

    def _engine(self, force_repack=False):
        """force_repack: re-upload / repack the weights even if (data_ptr, _version, optimizer epoch) did
        not change.  The training forward passes True: updates through `p.data` (manual SGD, EMA,
        `.data.clamp_`) change none of the three."""
        device = self._device()
        if device.type != 'cuda':
            _lib.require_cuda()
            raise RuntimeError("LSTM parameters are on %s: move the model to a CUDA device (model.to('cuda')); "
                               "there is no CPU path" % device)
        if self._handle is None or self._handle.device != device:
            cfg = lstm_config(self.hidden_dim, self.embedding_dim, self.pool_to_input, self.pool,
                              self.goal_dim if self.goal_flag else 0)
            self._handle = ModelHandle(cfg, device)
        key = weights_key(self)
        if force_repack or key != self._handle._weights_key:
            self._handle.set_weights(self._weight_fields(), key=key, force=force_repack)
        return self._handle

    def _weight_fields(self):
        lin = self.input_embedding.input_embeddings[0]
        fields = dict(
            input_embedding_weight=lin.weight, input_embedding_bias=lin.bias,
            encoder_weight_ih=self.encoder.weight_ih, encoder_weight_hh=self.encoder.weight_hh,
            encoder_bias_ih=self.encoder.bias_ih, encoder_bias_hh=self.encoder.bias_hh,
            decoder_weight_ih=self.decoder.weight_ih, decoder_weight_hh=self.decoder.weight_hh,
            decoder_bias_ih=self.decoder.bias_ih, decoder_bias_hh=self.decoder.bias_hh,
            hidden2normal_weight=self.hidden2normal.linear.weight,
            hidden2normal_bias=self.hidden2normal.linear.bias)
        if self.goal_flag:
            goal = self.goal_embedding.input_embeddings[0]
            fields.update(goal_embedding_weight=goal.weight, goal_embedding_bias=goal.bias)
        if self.pool is not None and not is_external(self.pool):      # an external module's weights stay in torch
            fields.update(self.pool.weight_fields())
        return fields

    def _goals_on(self, goals, num_tracks, device):
        """The goals [M, 2] a goal-conditioned model reads, fp32 on `device`; None for a model without goal input (which
        ignores them, like the reference)."""
        if not self.goal_flag:
            return None
        if goals is None:
            raise ValueError("goal_flag=True: the model needs the goals of the tracks ([M, 2])")
        if not torch.is_tensor(goals):
            goals = torch.as_tensor(np.asarray(goals, dtype=np.float64))
        if tuple(goals.shape) != (num_tracks, 2):
            raise ValueError("goals must be [%d, 2] (one per track), got %s" % (num_tracks, list(goals.shape)))
        return self._to_device(goals, device, 'goals')

    def _to_device(self, t, device, slot):
        """Host tensors go through pinned staging (H2D inside the caller's timed region).  slot names the argument: each
        argument of a call has its own staging buffer, and a buffer is refilled only once its previous asynchronous copy
        to the device has completed."""
        if t is None:
            return None
        t = t.detach()
        if t.device.type == 'cuda':
            return t.to(device=device, dtype=torch.float32).contiguous()
        t = t.to(dtype=torch.float32).contiguous()
        if t.is_pinned():
            return t.to(device, non_blocking=True)
        key = (tuple(t.shape), 'in', slot)
        staged = self._pinned.get(key)
        if staged is None:
            staged = (torch.empty(t.shape, dtype=torch.float32, pin_memory=True), torch.cuda.Event())
            self._pinned[key] = staged
        buf, copied = staged
        copied.synchronize()              # the previous copy out of this buffer has been read (no-op before the first)
        # plain single-threaded memcpy: torch's CPU copy_ may go through the intra-op thread pool,
        # whose wake-up latency showed rare 10-50 ms tails on the (virtualised) GPU hosts
        np.copyto(buf.numpy(), t.numpy())
        out = buf.to(device, non_blocking=True)
        copied.record(torch.cuda.current_stream(device))
        return out

    # -- reference API -----------------------------------------------------------------------
    def step(self, lstm, hidden_cell_state, obs1, obs2, goals, batch_split):
        """One step (lstm.py:91-168).  hidden_cell_state = (h [M, H], c [M, H]) flat CUDA tensors
        (the reference's per-track Python lists are also accepted and converted)."""
        phase = _lib.PHASE_ENCODER if lstm is self.encoder else _lib.PHASE_DECODER
        if is_external(self.pool):
            return external_step(self, hidden_cell_state, phase, obs1, obs2, batch_split)
        handle = self._engine()
        device = handle.device
        h, c = hidden_cell_state
        was_list = isinstance(h, (list, tuple))
        if was_list:
            h, c = torch.stack(list(h)), torch.stack(list(c))
        h = h.detach().to(device=device, dtype=torch.float32).contiguous().clone()
        c = c.detach().to(device=device, dtype=torch.float32).contiguous().clone()
        layout = self._layouts.get(batch_split, device=device)
        o1 = self._to_device(obs1, device, 'obs1')
        o2 = self._to_device(obs2, device, 'obs2')
        g = self._goals_on(goals, layout.num_tracks, device)
        normal, _ = handle.step_forward(layout, phase, o1, o2, h, c, goals=g)
        if was_list:
            return (list(h), list(c)), normal
        return (h, c), normal

    def forward(self, observed, goals, batch_split, prediction_truth=None, n_predict=None):
        """Forecast the entire sequence (lstm.py:170-264).

        observed [obs_length, M, 2]; batch_split [B + 1]; prediction_truth [pred_length - 1, M, 2]
        (teacher forcing) xor n_predict.  Returns rel_pred_scene [S, M, 5], pred_scene [S, M, 2]
        on the device `observed` came from.
        """
        assert ((prediction_truth is None) + (n_predict is None)) == 1
        if is_external(self.pool):        # the module runs in torch between the step's kernels (lstm/external.py)
            return external_forward(self, observed, goals, batch_split, prediction_truth, n_predict)
        # the graph path: parameter gradients, and / or d observed (a model with frozen parameters serves input gradients)
        if torch.is_grad_enabled() and ((torch.is_tensor(observed) and observed.requires_grad) or
                                        any(p.requires_grad for p in self.parameters())):
            from .training import sequence_with_grad
            return sequence_with_grad(self, observed, batch_split, prediction_truth, n_predict)
        return self._forward_nograd(observed, batch_split, prediction_truth, n_predict, goals=goals)

    def _sequence(self, observed, batch_split, prediction_truth, n_predict, pad_to_batch_max=True, force_repack=False,
                  goals=None):
        """A forward of `observed` [obs_length, M, 2] set up on the model's device: the inputs there and empty outputs
        and (h, c) state.  Launches nothing.  The steps are [0, S_enc) for the encoder and [S_enc, S) for the decoder;
        truth is None when there is no teacher forcing.  goals [M, 2]: read by a goal-conditioned model only."""
        if is_external(self.pool):
            raise NotImplementedError(EXTERNAL_FUSED_MESSAGE % type(self.pool).__name__)
        handle = self._engine(force_repack)
        device = handle.device
        layout = self._layouts.get(batch_split, pad_to_batch_max, device=device)
        M = layout.num_tracks
        if observed.shape[1] != M:
            raise ValueError("batch_split[-1] != number of tracks")
        obs = self._to_device(observed, device, 'observed')
        goals = self._goals_on(goals, M, device)
        truth = None
        if prediction_truth is not None:
            if isinstance(prediction_truth, (list, tuple)):
                prediction_truth = torch.stack(list(prediction_truth))
            truth = self._to_device(prediction_truth, device, 'truth')
            n_decode = int(truth.shape[0])
            if n_decode == 0:
                truth = None
        else:
            n_decode = int(n_predict) - 1
        S_enc = int(obs.shape[0]) - 1
        S = S_enc + n_decode
        f32 = dict(dtype=torch.float32, device=device)
        return Sequence(handle, layout, obs, truth, n_decode, S_enc, S,
                        normals=torch.empty((S, M, 5), **f32), positions=torch.empty((S, M, 2), **f32),
                        h=torch.empty((M, self.hidden_dim), **f32), c=torch.empty((M, self.hidden_dim), **f32),
                        out_device=observed.device, goals=goals)

    def _encode(self, seq):
        """The encoder steps [0, S_enc) of `seq`, into its own outputs and state."""
        seq.handle.forward_steps(seq.layout, seq.obs, seq.truth, seq.n_decode, 0, seq.S_enc, seq.normals,
                                 seq.positions, seq.h, seq.c, goals=seq.goals)
        return seq

    def _decode(self, seq, context, seed=True):
        """One decode from a copy of the encoder state and outputs of `seq`: context(h, c) edits the copied state, then
        the decoder steps [S_enc, S) run.  Returns the outputs as _results does."""
        h, c = seq.h.clone(), seq.c.clone()
        normals, positions = seq.normals.clone(), seq.positions.clone()
        context(h, c)
        seq.handle.forward_steps(seq.layout, seq.obs, seq.truth, seq.n_decode, seq.S_enc, seq.S, normals, positions,
                                 h, c, goals=seq.goals)
        return self._results(seq, normals, positions, seed)

    def _results(self, seq, normals, positions, seed=True):
        """(normals, positions) on the device `observed` came from.  seed: at obs_length 2 the positions start with
        observed[-1] (lstm.py:222-223, sgan.py:353-354; the VAE has no such rule)."""
        if seed and seq.obs.shape[0] == 2:
            positions = torch.cat([seq.obs[-1:].clone(), positions], dim=0)
        if seq.out_device != seq.handle.device:
            normals, positions = self._to_host(normals, positions)
        return normals, positions

    def _forward_nograd(self, observed, batch_split, prediction_truth, n_predict, want_states=False,
                        pad_to_batch_max=True, force_repack=False, goals=None):
        seq = self._sequence(observed, batch_split, prediction_truth, n_predict, pad_to_batch_max, force_repack, goals)
        handle, layout, device = seq.handle, seq.layout, seq.handle.device
        inputs = (layout, seq.obs, seq.truth, seq.n_decode, 0, seq.S, seq.normals, seq.positions, seq.h, seq.c)
        if want_states:
            # training forward: the outputs stay on the device; the per-step states are kept for the backward, and
            # so are the grid-embedding records the social backward reads (0 bytes: not a social model, no cache)
            states = torch.empty((seq.S, 2, layout.num_tracks, self.hidden_dim), dtype=torch.float32, device=device)
            cache_bytes = handle.train_cache_bytes(layout, seq.S)
            cache = torch.empty(cache_bytes, dtype=torch.uint8, device=device) if cache_bytes > 0 else None
            handle.forward_steps(*inputs, goals=seq.goals, states=states, cache=cache)
            normals, positions = self._results(seq._replace(out_device=device), seq.normals, seq.positions)
            return normals, positions, states, (seq.obs, seq.truth, layout, cache)
        if seq.out_device != device and seq.obs.shape[0] > 2:
            # host caller: every step's slice of the results is copied to pinned host memory on a second stream
            # while the later steps compute; one synchronisation of that stream at the end
            normals_h, positions_h = self._host_buffers(seq.normals, seq.positions)
            copy_stream = self._copy_stream(device)
            handle.forward_steps(*inputs, goals=seq.goals, host=(normals_h, positions_h, copy_stream))
            copy_stream.synchronize()
            return normals_h.view(normals_h.shape), positions_h.view(positions_h.shape)
        handle.forward_steps(*inputs, goals=seq.goals)
        return self._results(seq, seq.normals, seq.positions)

    def _host_buffers(self, *tensors):
        """Pinned host buffers shaped like `tensors`, from a pool (no per-call allocation: fresh host
        pages cost ~2 ms per result under the box's virtualisation).  A buffer is reused only once
        nothing derived from an earlier result (views, .numpy() arrays) is alive any more, which the
        storage use-count tells."""
        outs = []
        for i, t in enumerate(tensors):
            key = (tuple(t.shape), 'out', i)
            pool = self._pinned.setdefault(key, [])
            buf = None
            for cand in pool:
                if torch._C._storage_Use_Count(cand.untyped_storage()._cdata) <= 2:
                    buf = cand
                    break
            if buf is None:
                buf = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
                pool.append(buf)
            outs.append(buf)
        return outs

    def _copy_stream(self, device):
        st = self._pinned.get(('copy_stream', device.index))
        if st is None:
            st = torch.cuda.Stream(device=device)
            self._pinned[('copy_stream', device.index)] = st
        return st

    def _to_host(self, *tensors):
        """D2H into pooled pinned buffers; VIEWS of them are handed out."""
        outs = []
        for buf, t in zip(self._host_buffers(*tensors), tensors):
            buf.copy_(t, non_blocking=True)
            outs.append(buf.view(buf.shape))
        torch.cuda.current_stream(tensors[0].device).synchronize()
        return outs

    def __getstate__(self):
        # handles / pinned staging are per-process; never pickled (LSTMPredictor.save pickles the model)
        state = self.__dict__.copy()
        state['_handle'] = None
        state['_layouts'] = LayoutCache()
        state['_pinned'] = {}
        return state


class Predictor(object):
    """What the LSTM, S-GAN and VAE predictors share (reference lstm.py:266-313, sgan.py:583-630, vae.py:347-398):
    save / load and the per-scene call.  A subclass supplies `_mode_scenes` and the two class attributes below."""
    start_length_applies = True      # the model is fed xy[start_length:obs_length], else xy[:obs_length]
    neighbours_every_mode = True     # every mode returns the neighbours' predictions, else mode 0 only

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
            return torch.load(f, weights_only=False)   # torch >= 2.6 default would reject the pickle

    def _mode_scenes(self, observed, scene_goal, batch_split, n_predict, modes):
        """The predicted positions [S, N, 2] of every mode, in order (an iterable)."""
        raise NotImplementedError

    def __call__(self, paths, scene_goal, n_predict=12, modes=1, predict_all=True, obs_length=9, start_length=0,
                 args=None):
        self.model.eval()
        with torch.no_grad():
            xy = paths_to_xy(paths)
            batch_split = [0, xy.shape[1]]
            normalize = bool(getattr(args, 'normalize_scene', False))
            if normalize:
                xy, rotation, center, scene_goal = center_scene(xy, obs_length, goals=np.asarray(scene_goal))
            xy = torch.Tensor(xy)
            scene_goal = torch.Tensor(np.asarray(scene_goal))
            batch_split = torch.Tensor(batch_split).long()
            first = start_length if self.start_length_applies else 0
            multimodal_outputs = {}
            for num_p, output_scenes in enumerate(self._mode_scenes(xy[first:obs_length], scene_goal, batch_split,
                                                                    n_predict, modes)):
                output_scenes = output_scenes.cpu().numpy()
                if normalize:
                    output_scenes = inverse_scene(output_scenes, rotation, center)
                output_primary = output_scenes[-n_predict:, 0]
                output_neighs = output_scenes[-n_predict:, 1:]
                multimodal_outputs[num_p] = [output_primary,
                                             output_neighs if num_p == 0 or self.neighbours_every_mode else []]
        return multimodal_outputs


class LSTMPredictor(Predictor):
    """Reference lstm.py:266-313."""

    def _mode_scenes(self, observed, scene_goal, batch_split, n_predict, modes):
        for _ in range(modes):        # one forward per mode, each mode's outputs handled before the next forward
            yield self.model(observed, scene_goal, batch_split, n_predict=n_predict)[1]

    def predict_batch(self, scenes, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None):
        """Many scenes in ONE forward call (SURVEY.md 8f rank 1: replaces the evaluator's
        joblib.Parallel(n_jobs=12) over predict_scene, lstm/trajnet_evaluator.py:61).

        scenes: list of `paths` (each as for __call__).  Returns a list of {0: [primary, neighbours]}
        in the same order, equal to calling the predictor scene by scene: the scene layout is created
        with tb2_layout_set_padding(0), so a scene does not see the padding slots a batched call of
        the reference would add (those clobber grid cell 0, gridbased_pooling.py:281-293)."""
        return self.predict_batch_xy([paths_to_xy(paths) for paths in scenes], scene_goals, n_predict, obs_length,
                                     start_length, args)

    def predict_batch_xy(self, xys, scene_goals=None, n_predict=12, obs_length=9, start_length=0, args=None):
        """predict_batch on arrays: xys = list of float64 [n_frames, N_i, 2] as paths_to_xy returns them (the column
        pipeline of the evaluator, data.load_test_scenes_xy, builds them without TrackRow objects).  scene_goals: per
        scene the goals [N_i, 2] of its tracks, read by a goal-conditioned model (goal_flag=True) only.

        With an external interaction module (lstm/external.py) the scenes run in one padded forward per distinct
        scene size: a group has no padding, so each scene is seen as in a per-scene call by any module whose batch
        entries do not interact, and a stateful module keeps one state per forward.  A module that mixes the entries of
        its batch (a sum over the whole batch, like TrajectronPooling's) matches per-scene calls only in __call__."""
        if is_external(self.model.pool):
            if self.model.goal_flag:
                raise NotImplementedError(EXTERNAL_GOALS_MESSAGE)
            results = [None] * len(xys)
            for idx in scene_size_groups(xys):
                part = self._predict_batch_xy([xys[i] for i in idx], None, n_predict, obs_length, start_length, args)
                for i, r in zip(idx, part):
                    results[i] = r
            return results
        return self._predict_batch_xy(xys, scene_goals, n_predict, obs_length, start_length, args)

    def _predict_batch_xy(self, xys, scene_goals, n_predict, obs_length, start_length, args):
        self.model.eval()
        normalize = bool(getattr(args, 'normalize_scene', False))
        split = np.zeros(len(xys) + 1, dtype=np.int64)
        split[1:] = np.cumsum([xy.shape[1] for xy in xys])
        goals = None
        if self.model.goal_flag:
            if scene_goals is None or len(scene_goals) != len(xys):
                raise ValueError("goal_flag=True: predict_batch_xy needs one goal array per scene (scene_goals)")
            goals = np.concatenate([np.asarray(g, dtype=np.float64).reshape(-1, 2) for g in scene_goals], axis=0)
        with torch.no_grad():
            if normalize:
                # center_scene / inverse_scene of every scene on the device (lstm/scene_ops.py, SURVEY.md 8f rank 3)
                from .scene_ops import inverse_scenes, preprocess_scenes
                prepared = preprocess_scenes([xy[:obs_length] for xy in xys], device=self.model._device(),
                                             normalize_scene=True, obs_length=obs_length, goals=goals)
                observed, _, _, rotation, center = prepared[:5]
                goals = prepared[5] if goals is not None else None
                observed = observed[start_length:]
            else:
                observed = torch.Tensor(np.concatenate([xy[start_length:obs_length] for xy in xys], axis=1))
                goals = torch.Tensor(goals) if goals is not None else None
            if is_external(self.model.pool):
                _, output_scenes = self.model(observed, goals, torch.from_numpy(split), n_predict=n_predict)
            else:
                _, output_scenes = self.model._forward_nograd(observed, torch.from_numpy(split), None, n_predict,
                                                              pad_to_batch_max=False, goals=goals)
            if normalize:
                output_scenes = inverse_scenes(output_scenes, split, rotation, center)
            else:
                output_scenes = output_scenes.cpu().numpy()
        results = []
        for i in range(len(xys)):
            out = output_scenes[:, split[i]:split[i + 1]]
            results.append({0: [np.array(out[-n_predict:, 0]), np.array(out[-n_predict:, 1:])]})
        return results
