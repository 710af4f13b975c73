"""Losses with the reference's API (trajnetbaselines/lstm/loss.py: PredictionLoss :6-91, L2Loss
:93-135, CollisionLoss term :138-162).

The loss acts on the [pred_length x batch_size] primary rows only.  The per-(frame, scene) value and
its analytic derivative come from one kernel each (tb2_prediction_loss / tb2_l2_loss /
tb2_collision_loss, csrc/loss.cu) behind a torch.autograd.Function, so autograd chains them into the
CUDA BPTT of lstm/training.py.  There is no torch / CPU implementation of the loss expressions in this
package: predictions that are not CUDA fp32 tensors raise.
"""
import ctypes

import torch

from .. import _lib
from ..engine import LayoutCache, _ptr, _stream

_layouts = LayoutCache(capacity=8)


def _require_cuda_f32(t, what):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32):
        _lib.require_cuda()
        raise RuntimeError("%s must be a CUDA float32 tensor (got %s on %s): the losses run on the GPU only, "
                           "there is no CPU path" % (what, getattr(t, 'dtype', type(t)), getattr(t, 'device', '?')))


class _PrimaryLossFn(torch.autograd.Function):
    """values [T, B] of the primaries; backward scatters d value / d inputs into [T, M, 5].
    kind 0: PredictionLoss (bivariate Gaussian + background), kind 1: L2Loss.  Both depend on targets - mu only, so
    d targets = -d mu of the primaries (the Trainer's first target, xy[obs] - xy[obs - 1], depends on observed)."""

    @staticmethod
    def forward(ctx, inputs, targets, prim, background_rate, kind):
        lib = _lib.load()
        inputs = inputs.contiguous()
        targets = targets.contiguous()
        T, M = int(inputs.shape[0]), int(inputs.shape[1])
        B = int(prim.numel())
        values = torch.empty((T, B), dtype=torch.float32, device=inputs.device)
        dinputs = torch.empty((T, B, 5), dtype=torch.float32, device=inputs.device)
        with torch.cuda.device(inputs.device):
            if kind == 0:
                _lib.check(lib.tb2_prediction_loss(_ptr(inputs), _ptr(targets), _ptr(prim), T, M, B,
                                                   ctypes.c_float(background_rate), _ptr(values), _ptr(dinputs),
                                                   _stream(inputs.device)))
            else:
                _lib.check(lib.tb2_l2_loss(_ptr(inputs), _ptr(targets), _ptr(prim), T, M, B, _ptr(values),
                                           _ptr(dinputs), _stream(inputs.device)))
        ctx.save_for_backward(dinputs, prim)
        ctx.shape = (T, M)
        return values

    @staticmethod
    def backward(ctx, grad_values):
        dinputs, prim = ctx.saved_tensors
        T, M = ctx.shape
        grad = torch.zeros((T, M, 5), dtype=torch.float32, device=dinputs.device)
        grad[:, prim.long()] = dinputs * grad_values.unsqueeze(-1)
        d_targets = -grad[..., :2] if ctx.needs_input_grad[1] else None
        return grad, d_targets, None, None, None


class _CollisionLossFn(torch.autograd.Function):
    """CollisionLoss (loss.py:138-162) summed over frames, scenes and colliding neighbours."""

    @staticmethod
    def forward(ctx, positions, batch_split, col_wt, col_distance):
        lib = _lib.load()
        positions = positions.contiguous()
        layout = _layouts.get(batch_split, device=positions.device)
        T, M = int(positions.shape[0]), int(positions.shape[1])
        B = layout.num_scenes
        per = torch.empty((T, B), dtype=torch.float32, device=positions.device)
        dprim = torch.empty((T, B, 2), dtype=torch.float32, device=positions.device)
        with torch.cuda.device(positions.device):
            _lib.check(lib.tb2_collision_loss(layout.handle, _ptr(positions), T, ctypes.c_float(col_wt),
                                              ctypes.c_float(col_distance), _ptr(per), _ptr(dprim),
                                              _stream(positions.device)))
        ctx.save_for_backward(dprim)
        ctx.prim = [int(v) for v in batch_split[:-1]]
        ctx.shape = (T, M)
        return per.sum()

    @staticmethod
    def backward(ctx, grad_out):
        (dprim,) = ctx.saved_tensors
        T, M = ctx.shape
        grad = torch.zeros((T, M, 2), dtype=torch.float32, device=dprim.device)
        grad[:, torch.as_tensor(ctx.prim, device=dprim.device)] = dprim * grad_out
        return grad, None, None, None


def collision_loss(predictions, batch_split, col_wt=10.0, col_distance=0.2):
    """loss.py:138-162.  predictions [pred_length, num_tracks, 2]: the primary of each scene is
    penalised for coming within col_distance of a neighbour (neighbours are constants; NaN
    coordinates count as -1000)."""
    _require_cuda_f32(predictions, "predictions")
    batch_split = [int(v) for v in batch_split]
    return _CollisionLossFn.apply(predictions[..., :2], batch_split, float(col_wt), float(col_distance))


class _PrimaryLoss(torch.nn.Module):
    _kind = 0

    def _values(self, inputs, targets, batch_split, background_rate=0.0):
        _require_cuda_f32(inputs, "inputs")
        prim = batch_split[:-1].to(device=inputs.device, dtype=torch.int32)
        return _PrimaryLossFn.apply(inputs, targets.to(device=inputs.device, dtype=torch.float32), prim,
                                    float(background_rate), self._kind)

    def _reduce(self, values, col_loss):
        if self.keep_batch_dim:
            return values.mean(dim=0) * self.loss_multiplier
        if self.col_wt:
            return torch.mean(values) * self.loss_multiplier + col_loss * self.loss_multiplier
        return torch.mean(values) * self.loss_multiplier

    def _col(self, batch_split, positions):
        if not self.col_wt:
            return 0
        assert positions is not None, "Prediction positions required to calculate collision loss"
        return collision_loss(positions, batch_split.tolist(), self.col_wt, self.col_distance)


class PredictionLoss(_PrimaryLoss):
    """2D Gaussian with a flat background: -log(0.01 + bg N(x|mu, 3) + (0.99 - bg) N(x|mu, sigma, rho))
    (loss.py:6-91); evaluated by tb2_prediction_loss."""
    _kind = 0

    def __init__(self, keep_batch_dim=False, background_rate=0.2, col_wt=0.0, col_distance=0.2):
        super().__init__()
        self.keep_batch_dim = keep_batch_dim
        self.background_rate = background_rate
        self.loss_multiplier = 1
        self.col_wt = col_wt
        self.col_distance = col_distance

    def forward(self, inputs, targets, batch_split, positions=None):
        """inputs [pred_length, num_tracks, 5], targets [pred_length, num_tracks, 2] (loss.py:52-91)."""
        batch_split = torch.as_tensor(batch_split)
        col_loss = self._col(batch_split, positions)
        return self._reduce(self._values(inputs, targets, batch_split, self.background_rate), col_loss)


class L2Loss(_PrimaryLoss):
    """Deterministic variant (loss.py:93-135): 100 x MSE on the primaries' mean prediction; evaluated
    by tb2_l2_loss."""
    _kind = 1

    def __init__(self, keep_batch_dim=False, col_wt=0.0, col_distance=0.2):
        super().__init__()
        self.keep_batch_dim = keep_batch_dim
        self.loss_multiplier = 100
        self.col_wt = col_wt
        self.col_distance = col_distance

    def forward(self, inputs, targets, batch_split, positions=None):
        batch_split = torch.as_tensor(batch_split)
        col_loss = self._col(batch_split, positions)
        return self._reduce(self._values(inputs, targets, batch_split), col_loss)
