"""Autograd bridge for training: LSTM.forward under grad mode.

The forward is the same fused CUDA time loop as inference (with the per-step states kept);
the backward is tb2_lstm_sequence_backward (csrc/train.cu): BPTT restricted to the tracks that
actually receive gradient (all tracks for social pooling, whose hidden-state scatter couples the
tracks of a scene).  Mirrors what autograd computes for the reference's
Trainer.train_batch (trajnetbaselines/lstm/trainer.py:229-269).

When `observed` requires grad, the same backward also returns d observed: through the encoder steps'
velocity inputs, the directional grid's relative velocities and the hidden states social pooling
reads, plus pred = obs2 + mu of the encoder steps.  The decoder's inputs are detached, as in the
reference (its deep copy of observed[-1] and prediction_truth, and the fed-back positions).
"""
import ctypes

import torch

from .. import _lib
from ..engine import _ptr, _stream

_GRAD_FIELDS = {
    "input_embedding_weight": lambda m: m.input_embedding.input_embeddings[0].weight,
    "input_embedding_bias": lambda m: m.input_embedding.input_embeddings[0].bias,
    "encoder_weight_ih": lambda m: m.encoder.weight_ih,
    "encoder_weight_hh": lambda m: m.encoder.weight_hh,
    "encoder_bias_ih": lambda m: m.encoder.bias_ih,
    "encoder_bias_hh": lambda m: m.encoder.bias_hh,
    "decoder_weight_ih": lambda m: m.decoder.weight_ih,
    "decoder_weight_hh": lambda m: m.decoder.weight_hh,
    "decoder_bias_ih": lambda m: m.decoder.bias_ih,
    "decoder_bias_hh": lambda m: m.decoder.bias_hh,
    "hidden2normal_weight": lambda m: m.hidden2normal.linear.weight,
    "hidden2normal_bias": lambda m: m.hidden2normal.linear.bias,
}


def _refuse_goals(model):
    if model.goal_flag:       # goal-conditioned models are built for inference only
        from .trainer import GOALS_MESSAGE
        raise NotImplementedError(GOALS_MESSAGE)


def _grad_targets(model):
    """field name -> parameter, for every parameter the backward kernel produces a gradient for."""
    _refuse_goals(model)
    out = {k: f(model) for k, f in _GRAD_FIELDS.items()}
    pool = model.pool
    if pool is not None and not hasattr(pool, 'fill_config'):
        return out         # an external module: autograd carries its own gradients (lstm/external.py)
    if pool is not None and not hasattr(pool, 'embedding_arch'):        # only GridBasedPooling has a backward
        raise NotImplementedError("training of %s is not built (inference only); use torch.no_grad()" % type(pool).__name__)
    if pool is not None and pool.embedding is not None:
        linears = [m for m in pool.embedding if isinstance(m, torch.nn.Linear)]
        out["pool_embedding_weight0"] = linears[0].weight
        out["pool_embedding_bias0"] = linears[0].bias
        if len(linears) > 1:
            out["pool_embedding_weight1"] = linears[1].weight
            out["pool_embedding_bias1"] = linears[1].bias
    if pool is not None and getattr(pool, 'type_', None) == 'social':
        out["pool_encoding_weight"] = pool.hidden_dim_encoding.weight
        out["pool_encoding_bias"] = pool.hidden_dim_encoding.bias
    return out


def _save_forward(ctx, model, observed, params, forward_out):
    """Keep what the backward of a training forward (model._forward_nograd with want_states) needs."""
    normals, positions, states, (obs, truth, layout, cache) = forward_out
    ctx.model, ctx.layout, ctx.obs, ctx.truth, ctx.states, ctx.cache = model, layout, obs, truth, states, cache
    ctx.num_steps = normals.shape[0]
    ctx.observed_meta = (observed.device, observed.dtype) if torch.is_tensor(observed) else None
    ctx.params = params
    ctx.save_for_backward(positions)
    return normals, positions


def _run_backward(ctx, active, d_obs, launch):
    """One backward call over the rows `active` (int32 on the device): zeroed parameter gradients and d_obs (or None) go
    into the gradient struct, `launch(lib, handle, weights, grads, workspace, bytes, bwd_workspace, bytes, positions of
    the steps, cache bytes, device)` issues the call.  Returns autograd's tuple for the forward's arguments (model,
    observed, three more, *params)."""
    model, layout = ctx.model, ctx.layout
    (positions,) = ctx.saved_tensors
    handle = model._engine()
    device = handle.device
    lib = _lib.load()
    S = ctx.num_steps
    R = int(active.numel())
    targets = _grad_targets(model)
    grads = {k: torch.zeros_like(p, dtype=torch.float32, device=device).contiguous() for k, p in targets.items()}
    if R > 0:
        g = _lib.LstmGrads()
        for k, t in grads.items():
            setattr(g, k, t.data_ptr())
        if d_obs is not None:
            g.d_observed = d_obs.data_ptr()
        w, keep = handle.weights_struct(model._weight_fields())
        ws, need = handle.workspace(layout)
        bneed = int(lib.tb2_lstm_backward_workspace_bytes(handle.handle, layout.handle, R, S))
        bws = torch.empty(bneed, dtype=torch.uint8, device=device)
        pos_steps = positions[-S:].contiguous()
        cache_bytes = 0 if ctx.cache is None else int(ctx.cache.numel())      # no cache: not a social model
        with torch.cuda.device(device):
            _lib.check(launch(lib, handle, w, g, ws, need, bws, bneed, pos_steps, cache_bytes, device))
        del keep
    # a sequence without a decoder step (pred_length 1) never uses the decoder cell: like autograd on the
    # reference, its parameters get no gradient (None), so optimizers leave them alone
    unused = ("decoder_",) if S == int(ctx.obs.shape[0]) - 1 else ()
    by_param = {id(p): grads[k] for k, p in targets.items() if not k.startswith(unused)}
    out = []
    for p in ctx.params:
        gr = by_param.get(id(p))
        out.append(gr.to(p.dtype) if (gr is not None and p.requires_grad) else None)
    d_in = None
    if d_obs is not None and ctx.needs_input_grad[1]:
        device_in, dtype_in = ctx.observed_meta
        d_in = d_obs.to(device=device_in, dtype=dtype_in)
    return (None, d_in, None, None, None) + tuple(out)


class _SequenceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, observed, batch_split, prediction_truth, n_predict, *params):
        # grad mode is off inside autograd.Function.forward, so "is this a training forward" cannot be asked
        # in LSTM._engine: every forward that records a graph repacks the weights (a few tens of
        # microseconds), which also covers parameter updates that bypass version counters and optimizer hooks
        return _save_forward(ctx, model, observed, params, model._forward_nograd(
            observed, batch_split, prediction_truth, n_predict, want_states=True, force_repack=True))

    @staticmethod
    def backward(ctx, d_normals, d_positions):
        device = ctx.model._engine().device
        S = ctx.num_steps
        M = ctx.layout.num_tracks
        obs_length = int(ctx.obs.shape[0])
        dn = torch.zeros((S, M, 5), dtype=torch.float32, device=device)
        if d_normals is not None:
            dn += torch.nan_to_num(d_normals.to(device=device, dtype=torch.float32))
        d_obs = None
        if ctx.needs_input_grad[1]:
            d_obs = torch.zeros((obs_length, M, 2), dtype=torch.float32, device=device)
        if d_positions is not None:       # pred = obs2 + mu (lstm.py:232,255)
            dp_all = torch.nan_to_num(d_positions.to(device=device, dtype=torch.float32))
            dp = dp_all[-S:]
            dn[:, :, :2] += dp
            if d_obs is not None:         # obs2 of the encoder steps is observed[s + 1]; the decoder's are detached
                if dp_all.shape[0] > S:   # obs_length 2: positions[0] is observed[-1] itself (lstm.py:222-223)
                    d_obs[-1] += dp_all[0]
                d_obs[1:obs_length] += dp[:obs_length - 1]
        dn = dn.contiguous()
        social = ctx.model.pool is not None and getattr(ctx.model.pool, 'type_', None) == 'social'
        if social:      # the hidden-state scatter couples all tracks of a scene: every row is active
            active = torch.arange(M, dtype=torch.int32, device=device)
        else:
            active = (dn != 0).any(dim=2).any(dim=0).nonzero().flatten().to(torch.int32).contiguous()

        def launch(lib, handle, w, g, ws, need, bws, bneed, pos_steps, cache_bytes, device):
            return lib.tb2_lstm_sequence_backward(
                handle.handle, ctx.layout.handle, ctypes.byref(w), _ptr(ctx.obs), obs_length, _ptr(ctx.truth),
                S - (obs_length - 1), _ptr(pos_steps), _ptr(ctx.states), _ptr(dn), _ptr(active), int(active.numel()),
                ctypes.byref(g), _ptr(ws), need, _ptr(bws), bneed, _ptr(ctx.cache), cache_bytes, _stream(device))
        return _run_backward(ctx, active, d_obs, launch)


def sequence_with_grad(model, observed, batch_split, prediction_truth, n_predict):
    _refuse_goals(model)
    if torch.is_tensor(observed) and observed.requires_grad:
        _grad_targets(model)          # refuses the modules without a backward before anything runs
    params = tuple(model.parameters())
    return _SequenceFn.apply(model, observed, batch_split, prediction_truth, n_predict, *params)


class _RolloutFn(torch.autograd.Function):
    """The free-running forward of LSTM.forward, differentiated with nothing detached: tb2_lstm_rollout_backward."""

    @staticmethod
    def forward(ctx, model, observed, batch_split, n_predict, pad_to_batch_max, *params):
        return _save_forward(ctx, model, observed, params, model._forward_nograd(
            observed, batch_split, None, n_predict, want_states=True, pad_to_batch_max=pad_to_batch_max,
            force_repack=True))

    @staticmethod
    def backward(ctx, d_normals, d_positions):
        (positions,) = ctx.saved_tensors
        device = ctx.model._engine().device
        S, M = ctx.num_steps, ctx.layout.num_tracks
        obs_length = int(ctx.obs.shape[0])

        def upstream(d, shape):
            out = torch.zeros(shape, dtype=torch.float32, device=device)
            if d is not None:
                out += torch.nan_to_num(d.to(device=device, dtype=torch.float32))
            return out.contiguous()
        dn = upstream(d_normals, (S, M, 5))
        dp = upstream(d_positions, tuple(positions.shape))
        d_obs = torch.zeros((obs_length, M, 2), dtype=torch.float32, device=device)
        # every row: picking the rows with a gradient would read the upstream gradients back to the host, a
        # synchronisation on every call (an attack's loop makes one per iteration); rows without one add exact zeros
        active = torch.arange(M, dtype=torch.int32, device=device)

        def launch(lib, handle, w, g, ws, need, bws, bneed, pos_steps, cache_bytes, device):
            return lib.tb2_lstm_rollout_backward(
                handle.handle, ctx.layout.handle, ctypes.byref(w), _ptr(ctx.obs), obs_length, S - (obs_length - 1),
                _ptr(pos_steps), _ptr(ctx.states), _ptr(dn), _ptr(dp), _ptr(active), M, ctypes.byref(g), _ptr(ws), need,
                _ptr(bws), bneed, _ptr(ctx.cache), cache_bytes, _stream(device))
        return _run_backward(ctx, active, d_obs, launch)


def check_rollout(model):
    """NotImplementedError for the models differentiable_rollout (and the collision attack built on it) cannot
    differentiate: S-GAN / VAE, goal models, user-defined and the built-in non-grid interaction modules."""
    from .lstm import LSTM
    from .external import is_external
    if type(model) is not LSTM:
        raise NotImplementedError("differentiable_rollout serves LSTM models; %s (S-GAN / VAE) is not built"
                                  % type(model).__name__)
    _refuse_goals(model)
    if is_external(model.pool):
        raise NotImplementedError("differentiable_rollout of a user-defined interaction module (%s) is not built"
                                  % type(model.pool).__name__)
    _grad_targets(model)              # refuses the non-grid modules


def differentiable_rollout(model, observed, batch_split, n_predict, pad_to_batch_max=True):
    """(normals, positions) of the free-running forecast model(observed, None, batch_split, n_predict=n_predict), bit for
    bit, differentiable with nothing detached: unlike LSTM.forward's graph (the reference's, whose decoder inputs are
    detached), the gradient follows every fed-back position into the decoder's velocity inputs, the directional grid's
    relative velocities and pos = obs2 + mu, down to `observed` and the parameters.  Parameters may be frozen or
    trainable.  pad_to_batch_max=False: every scene as if it were called on its own (LSTMPredictor.predict_batch_xy's
    layout).  Vanilla, occupancy, directional and social models; NotImplementedError (check_rollout) for goal models,
    the non-grid and user-defined interaction modules, S-GAN and VAE, before anything runs.  The backward makes no host
    synchronisation."""
    check_rollout(model)
    params = tuple(model.parameters())
    return _RolloutFn.apply(model, observed, batch_split, n_predict, pad_to_batch_max, *params)
