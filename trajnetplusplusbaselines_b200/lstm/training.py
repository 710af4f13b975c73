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


class _SequenceFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, model, observed, batch_split, prediction_truth, n_predict, *params):
        # grad mode is off inside autograd.Function.forward, so "is this a training forward" cannot be asked
        # in LSTM._engine: every forward that records a graph repacks the weights (a few tens of
        # microseconds), which also covers parameter updates that bypass version counters and optimizer hooks
        normals, positions, states, (obs, truth, layout, cache) = model._forward_nograd(
            observed, batch_split, prediction_truth, n_predict, want_states=True, force_repack=True)
        ctx.model = model
        ctx.layout = layout
        ctx.obs = obs
        ctx.truth = truth
        ctx.states = states
        ctx.cache = cache
        ctx.num_steps = normals.shape[0]
        ctx.observed_meta = (observed.device, observed.dtype) if torch.is_tensor(observed) else None
        ctx.params = params
        ctx.save_for_backward(positions)
        return normals, positions

    @staticmethod
    def backward(ctx, d_normals, d_positions):
        model, layout = ctx.model, ctx.layout
        (positions,) = ctx.saved_tensors
        handle = model._engine()
        device = handle.device
        lib = _lib.load()
        S = ctx.num_steps
        M = layout.num_tracks
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
        social = model.pool is not None and getattr(model.pool, 'type_', None) == 'social'
        if social:      # the hidden-state scatter couples all tracks of a scene: every row is active
            active = torch.arange(M, dtype=torch.int32, device=device)
        else:
            active = (dn != 0).any(dim=2).any(dim=0).nonzero().flatten().to(torch.int32).contiguous()
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
            n_decode = S - (int(ctx.obs.shape[0]) - 1)
            cache_bytes = 0 if ctx.cache is None else int(ctx.cache.numel())      # no cache: not a social model
            with torch.cuda.device(device):
                _lib.check(lib.tb2_lstm_sequence_backward(
                    handle.handle, layout.handle, ctypes.byref(w), _ptr(ctx.obs), int(ctx.obs.shape[0]),
                    _ptr(ctx.truth), n_decode, _ptr(pos_steps), _ptr(ctx.states), _ptr(dn), _ptr(active), R,
                    ctypes.byref(g), _ptr(ws), need, _ptr(bws), bneed, _ptr(ctx.cache), cache_bytes, _stream(device)))
            del keep
        # a sequence without a decoder step (pred_length 1) never uses the decoder cell: like autograd on the
        # reference, its parameters get no gradient (None), so optimizers leave them alone
        unused = ("decoder_",) if S == int(ctx.obs.shape[0]) - 1 else ()
        by_param = {id(p): grads[k] for k, p in targets.items() if not k.startswith(unused)}
        out = []
        for p in ctx.params:
            gr = by_param.get(id(p))
            out.append(gr.to(p.dtype) if (gr is not None and p.requires_grad) else None)
        if d_obs is not None:
            device_in, dtype_in = ctx.observed_meta
            d_obs = d_obs.to(device=device_in, dtype=dtype_in)
        return (None, d_obs, None, None, None) + tuple(out)


def sequence_with_grad(model, observed, batch_split, prediction_truth, n_predict):
    _refuse_goals(model)
    if torch.is_tensor(observed) and observed.requires_grad:
        _grad_targets(model)          # refuses the modules without a backward before anything runs
    params = tuple(model.parameters())
    return _SequenceFn.apply(model, observed, batch_split, prediction_truth, n_predict, *params)
