"""LSTM models with an external interaction module: any `torch.nn.Module` that follows the reference's pool plug.

The plug (reference lstm/lstm.py:25-42, 141-151, 212-216) is

    pool.reset(num_tracks, max_num_neigh, device)          once per forward
    pool(hidden [B, N, H], obs1 [B, N, 2], obs2 [B, N, 2]) -> [B * N, out_dim]
    pool.out_dim

A module without `fill_config` (not one of this package's built-in modules, whose forward is fused into the library's
kernels) runs here: the library runs the LSTM step on the device and torch runs the module, step by step, on the
current stream, with no host synchronisation in between.  Per step:

    tb2_pool_inputs_padded        ragged obs1 / obs2 / h -> [B, n_pad, .], NaN padding (generate_pooling_inputs)
    pool(h_pad, obs1_pad, obs2_pad)
    tb2_lstm_step_forward         with pooled_padded_dev: the module's row of every present track into the gate
                                  operand, then the step

n_pad is the largest scene of the batch, and every track's hidden state goes in, absent tracks included, as in the
reference.  Under grad mode each of the two library calls is a torch.autograd.Function (backward:
tb2_pool_inputs_padded_backward and tb2_lstm_step_backward), so autograd carries the gradient through the user's
module into its parameters and into every track's hidden state, and, when `observed` requires grad, into the
positions the encoder steps read (the velocity input, the module's position inputs and pos = obs2 + mu).
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from ..engine import _ptr, _stream

EXTERNAL_GOALS_MESSAGE = "goal_flag=True with an external interaction module (one without fill_config) is not built"


def is_external(pool):
    """The module runs in torch between the step's kernels (it is not one of the built-in, fused modules)."""
    return pool is not None and not hasattr(pool, 'fill_config')


def _f32(t):
    return t if (t.dtype == torch.float32 and t.is_contiguous()) else t.to(torch.float32).contiguous()


def _primaries(layout):
    """The scenes' first rows (batch_split[:-1]) as an int64 device tensor, kept with the layout (copied once, without
    synchronising: pinned memory, non-blocking)."""
    rows = getattr(layout, '_primary_rows', None)
    if rows is None:
        host = torch.tensor(layout.offsets[:-1], dtype=torch.int64).pin_memory()
        rows = host.to(layout.device, non_blocking=True)
        layout._primary_rows = rows
    return rows


class _PaddedInputs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layout, obs1, obs2, h):
        B, n_pad, H = layout.num_scenes, layout.max_scene, int(h.shape[1])
        f32 = dict(dtype=torch.float32, device=h.device)
        o1p, o2p = torch.empty((B, n_pad, 2), **f32), torch.empty((B, n_pad, 2), **f32)
        hp = torch.empty((B, n_pad, H), **f32)
        with torch.cuda.device(h.device):
            _lib.check(_lib.load().tb2_pool_inputs_padded(layout.handle, _ptr(obs1), _ptr(obs2), _ptr(h), H, _ptr(o1p),
                                                          _ptr(o2p), _ptr(hp), _stream(h.device)))
        ctx.layout = layout
        ctx.shape = tuple(h.shape)
        if not (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            ctx.mark_non_differentiable(o1p, o2p)
        return o1p, o2p, hp

    @staticmethod
    def _unpad(layout, d_pad, width, device):
        """[M, width] += the track slots of d_pad [B, n_pad, width]; None when nothing flowed back."""
        d = torch.zeros((layout.num_tracks, width), dtype=torch.float32, device=device)
        if d_pad is not None:
            with torch.cuda.device(device):
                _lib.check(_lib.load().tb2_pool_inputs_padded_backward(layout.handle, _ptr(_f32(d_pad)), width, _ptr(d),
                                                                       _stream(device)))
        return d

    @staticmethod
    def backward(ctx, d_o1p, d_o2p, d_hp):
        device = next(t.device for t in (d_hp, d_o1p, d_o2p) if t is not None)
        d_o1 = _PaddedInputs._unpad(ctx.layout, d_o1p, 2, device) if ctx.needs_input_grad[1] else None
        d_o2 = _PaddedInputs._unpad(ctx.layout, d_o2p, 2, device) if ctx.needs_input_grad[2] else None
        d_h = _PaddedInputs._unpad(ctx.layout, d_hp, ctx.shape[1], device) if d_hp is not None else None
        return None, d_o1, d_o2, d_h


def _lstm_params(model):
    from .training import _GRAD_FIELDS
    return tuple(f(model) for f in _GRAD_FIELDS.values())


class _PooledStep(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, handle, layout, phase, obs1, obs2, pooled, h, c, *params):
        h_out, c_out = torch.empty_like(h), torch.empty_like(c)
        normal, pos = handle.step_forward(layout, phase, obs1, obs2, h, c, pooled=pooled, h_out=h_out, c_out=c_out)
        ctx.model, ctx.handle, ctx.layout, ctx.phase, ctx.params = model, handle, layout, phase, params
        ctx.save_for_backward(obs1, obs2, pooled, h, c)
        return h_out, c_out, normal, pos

    @staticmethod
    def backward(ctx, d_h_out, d_c_out, d_normal, d_pos):
        from .training import _GRAD_FIELDS
        obs1, obs2, pooled, h, c = ctx.saved_tensors
        model, handle, layout, phase = ctx.model, ctx.handle, ctx.layout, ctx.phase
        device = h.device
        f32 = dict(dtype=torch.float32, device=device)
        M, H = h.shape
        d_h_out = torch.zeros((M, H), **f32) if d_h_out is None else _f32(d_h_out)
        d_c_out = torch.zeros((M, H), **f32) if d_c_out is None else _f32(d_c_out)
        dn = torch.zeros((M, 5), **f32)
        if d_normal is not None:
            dn += torch.nan_to_num(d_normal.to(torch.float32))
        if d_pos is not None:            # pos = obs2 + mu (lstm.py:232,255); obs2 is data / detached
            dn[:, :2] += torch.nan_to_num(d_pos.to(torch.float32))
        d_h_in, d_c_in, d_pooled = torch.empty((M, H), **f32), torch.empty((M, H), **f32), torch.empty_like(pooled)
        want_obs = ctx.needs_input_grad[4] or ctx.needs_input_grad[5]
        d_obs1 = torch.zeros((M, 2), **f32) if want_obs else None
        d_obs2 = torch.zeros((M, 2), **f32) if want_obs else None
        cell = "encoder_" if phase == _lib.PHASE_ENCODER else "decoder_"
        fields = [k for k in _GRAD_FIELDS if not k.startswith(("encoder_", "decoder_")) or k.startswith(cell)]
        grads = {k: torch.zeros(tuple(_GRAD_FIELDS[k](model).shape), **f32) for k in fields}
        g = _lib.LstmGrads()
        for k, t in grads.items():
            setattr(g, k, t.data_ptr())
        if want_obs:
            g.d_obs1, g.d_obs2 = d_obs1.data_ptr(), d_obs2.data_ptr()
        w, keep = handle.weights_struct(model._weight_fields())
        lib = _lib.load()
        need = int(lib.tb2_lstm_step_backward_workspace_bytes(handle.handle, layout.handle))
        bws = torch.empty(need, dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            _lib.check(lib.tb2_lstm_step_backward(
                handle.handle, layout.handle, ctypes.byref(w), phase, _ptr(obs1), _ptr(obs2), _ptr(pooled), _ptr(h),
                _ptr(c), _ptr(d_h_out), _ptr(d_c_out), _ptr(dn), _ptr(d_h_in), _ptr(d_c_in), _ptr(d_pooled),
                ctypes.byref(g), _ptr(bws), need, _stream(device)))
        del keep
        if want_obs and d_pos is not None:      # pos = obs2 + mu
            d_obs2 += torch.nan_to_num(d_pos.to(torch.float32))
        out = []
        for k, p in zip(_GRAD_FIELDS, ctx.params):
            gr = grads.get(k)
            out.append(gr.to(p.dtype) if (gr is not None and p.requires_grad) else None)
        return (None, None, None, None, d_obs1, d_obs2, d_pooled, d_h_in, d_c_in) + tuple(out)


def pooled_step(model, handle, layout, phase, obs1, obs2, h, c):
    """One recurrence step with the external module: padded inputs, the module, the step.  Returns
    (h, c, normal [M, 5], pos [M, 2]) on the device; differentiable under grad mode."""
    o1p, o2p, hp = _PaddedInputs.apply(layout, obs1, obs2, h)
    pooled = model.pool(hp, o1p, o2p)
    B, n_pad, out_dim = layout.num_scenes, layout.max_scene, int(model.pool.out_dim)
    if not torch.is_tensor(pooled) or tuple(pooled.shape) != (B * n_pad, out_dim):
        raise ValueError("%s returned %s; the pool plug returns [batch_size * num_tracks, out_dim] = [%d, %d] "
                         "(reference lstm.py:147)" % (type(model.pool).__name__,
                                                      list(pooled.shape) if torch.is_tensor(pooled) else type(pooled),
                                                      B * n_pad, out_dim))
    if pooled.device != h.device:
        raise ValueError("%s returned a tensor on %s; the model runs on %s" % (type(model.pool).__name__, pooled.device,
                                                                              h.device))
    return _PooledStep.apply(model, handle, layout, phase, obs1, obs2, _f32(pooled), h, c, *_lstm_params(model))


def _truth_frames(model, prediction_truth, device):
    if prediction_truth is None:
        return None
    if isinstance(prediction_truth, (list, tuple)):
        prediction_truth = torch.stack(list(prediction_truth))
    return model._to_device(prediction_truth, device, 'truth')


def external_forward(model, observed, goals, batch_split, prediction_truth=None, n_predict=None):
    """LSTM.forward (lstm.py:170-264) with an external module: the reference's time loop, step by step."""
    if model.goal_flag:
        raise NotImplementedError(EXTERNAL_GOALS_MESSAGE)
    grad = torch.is_grad_enabled()
    handle = model._engine(force_repack=grad)     # a graph-recording forward repacks, as the fused training forward does
    device = handle.device
    layout = model._layouts.get(batch_split, device=device)
    M = layout.num_tracks
    if observed.shape[1] != M:
        raise ValueError("batch_split[-1] != number of tracks")
    if grad and torch.is_tensor(observed) and observed.requires_grad:      # d observed flows back through the copy
        obs = observed.to(device=device, dtype=torch.float32).contiguous()
    else:
        obs = model._to_device(observed, device, 'observed')
    truth = _truth_frames(model, prediction_truth, device)
    n_decode = int(truth.shape[0]) if truth is not None else int(n_predict) - 1
    H = int(model.hidden_dim)
    h = torch.zeros((M, H), dtype=torch.float32, device=device)
    c = torch.zeros((M, H), dtype=torch.float32, device=device)
    B, n_pad = layout.num_scenes, layout.max_scene
    model.pool.reset(B * n_pad, n_pad - 1, device=device)              # lstm.py:212-216

    normals = []
    positions = [obs[-1]] if obs.shape[0] == 2 else []
    for s in range(int(obs.shape[0]) - 1):                            # encoder (lstm.py:226-232)
        h, c, normal, pos = pooled_step(model, handle, layout, _lib.PHASE_ENCODER, obs[s], obs[s + 1], h, c)
        normals.append(normal)
        positions.append(pos)
    primaries = _primaries(layout) if n_decode > 0 else None
    # seq[0] = observed[-1] is a tensor in every forward: its primary rows take the fed-back position too.  It is the
    # reference's deep copy (lstm.py:235): no gradient flows back through it
    seq = [obs[-1].detach()] + ([truth[k] for k in range(n_decode)] if truth is not None else [None] * n_decode)
    for k in range(n_decode):                                         # decoder: the feedback rule of lstm.py:240-250
        o1, o2 = seq[k], seq[k + 1]
        if o1 is None:
            o1 = positions[-2].detach()
        else:
            o1 = o1.clone()
            o1[primaries] = positions[-2].detach()[primaries]
        if o2 is None:
            o2 = positions[-1].detach()
        else:
            o2 = o2.clone()
            o2[primaries] = positions[-1].detach()[primaries]
        h, c, normal, pos = pooled_step(model, handle, layout, _lib.PHASE_DECODER, o1.contiguous(), o2.contiguous(), h, c)
        normals.append(normal)
        positions.append(pos)
    rel_pred_scene = torch.stack(normals, dim=0)
    pred_scene = torch.stack(positions, dim=0)
    if observed.device != device and not grad:
        rel_pred_scene, pred_scene = model._to_host(rel_pred_scene, pred_scene)
    return rel_pred_scene, pred_scene


def external_step(model, hidden_cell_state, phase, obs1, obs2, batch_split):
    """LSTM.step (lstm.py:91-168) with an external module: one step, the module called on the padded inputs."""
    if model.goal_flag:
        raise NotImplementedError(EXTERNAL_GOALS_MESSAGE)
    handle = model._engine()
    device = handle.device
    layout = model._layouts.get(batch_split, device=device)
    h, c = hidden_cell_state
    was_list = isinstance(h, (list, tuple))
    if was_list:
        h, c = torch.stack(list(h)), torch.stack(list(c))
    h, c = _f32(h.to(device)), _f32(c.to(device))
    o1 = model._to_device(obs1, device, 'obs1')
    o2 = model._to_device(obs2, device, 'obs2')
    h, c, normal, _ = pooled_step(model, handle, layout, phase, o1, o2, h, c)
    if was_list:
        return (list(h), list(c)), normal
    return (h, c), normal


def scene_size_groups(xys):
    """Indices of the scenes of each distinct size, in order of first appearance: a padded forward of one group has
    no padding, so every scene in it is seen as in a call on that scene alone."""
    groups = {}
    for i, xy in enumerate(xys):
        groups.setdefault(int(xy.shape[1]), []).append(i)
    return [np.asarray(v, dtype=np.int64) for v in groups.values()]
