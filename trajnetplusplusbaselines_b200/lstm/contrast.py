"""Social-NCE (Liu, Yan & Alahi, ICCV 2021): a contrastive training term that asks the primary's hidden state at the
end of the observation to tell its own future position from places where it would collide with a neighbour.  This
package's definition is DESIGN.md §1 A24; in short, per scene b and horizon step d = 1 .. horizon (frame
f = obs_length - 1 + d, coordinates relative to the primary's last observed position x0):

  * positive: the primary at f, plus sigma * eps;
  * negatives: for every neighbour with a finite position at f and k = 0 .. 7, that position shifted by
    rho (cos k pi/4, sin k pi/4), plus sigma * eps;
  * keys = normalize(phi(x, y, d)), query = normalize(psi(h)), with phi and psi two-layer ReLU MLPs;
  * term = logsumexp(q . keys / temperature) - q . key_positive / temperature, for each pair whose positive is finite;
    L_nce is the mean over those pairs (0 without any).

eps [B, horizon, 1 + 8 (n_max - 1), 2] is one torch.randn draw on the model's device per call (`fixed_eps` replaces
it).  The term and its gradients are two launches (csrc/contrast.cu): a per-scene forward that also writes the
scene's gradient partials, and a reduction that sums them in scene order and scales them by d loss / count, the count
of finite pairs read on the device.  Neither synchronises with the host.
"""
import torch

from .. import _lib
from ..engine import LayoutCache, _ptr, _stream

_layouts = LayoutCache(capacity=8)

MLP_DIMS = (16, 32, 64)
HEAD_DIMS = (4, 8, 16)


class _SocialNCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, scene, hidden, layout, obs_frame, eps, *params):
        lib = _lib.load()
        device = hidden.device
        B, H = layout.num_scenes, module.hidden_dim
        theta = torch.cat([p.detach().reshape(-1) for p in params]).to(torch.float32).contiguous()
        f32 = dict(dtype=torch.float32, device=device)
        terms = torch.empty((B, module.horizon), **f32)
        valid = torch.empty((B, module.horizon), **f32)
        dh_part = torch.empty((B, H), **f32)
        dp_part = torch.empty((B, theta.numel()), **f32)
        with torch.cuda.device(device):
            _lib.check(lib.tb2_snce_forward(
                layout.handle, _ptr(scene), int(scene.shape[0]), obs_frame, module.horizon, _ptr(hidden), H,
                _ptr(theta), module.mlp_dim, module.head_dim, module.temperature, module.rho, module.sigma, _ptr(eps),
                _ptr(terms), _ptr(valid), _ptr(dh_part), _ptr(dp_part), _stream(device)))
        count = valid.sum()
        loss = terms.sum() / count.clamp(min=1.0)
        ctx.layout, ctx.hidden_shape, ctx.hidden_dim = layout, tuple(hidden.shape), H
        ctx.shapes = [p.shape for p in params]
        ctx.save_for_backward(count, dh_part, dp_part)
        ctx.mark_non_differentiable(terms, valid)
        return loss, terms, valid

    @staticmethod
    def backward(ctx, d_loss, d_terms, d_valid):
        count, dh_part, dp_part = ctx.saved_tensors
        device = dh_part.device
        lib = _lib.load()
        d_hidden = torch.zeros(ctx.hidden_shape, dtype=torch.float32, device=device)
        d_params = torch.empty(dp_part.shape[1], dtype=torch.float32, device=device)
        d_loss = d_loss.to(device=device, dtype=torch.float32).contiguous()
        with torch.cuda.device(device):
            _lib.check(lib.tb2_snce_backward(ctx.layout.handle, _ptr(d_loss), _ptr(count), ctx.hidden_dim,
                                             int(d_params.numel()), _ptr(dh_part), _ptr(dp_part), _ptr(d_hidden),
                                             _ptr(d_params), _stream(device)))
        grads, at = [], 0
        for shape in ctx.shapes:
            n = shape.numel()
            grads.append(d_params[at:at + n].view(shape))
            at += n
        return (None, None, d_hidden, None, None, None) + tuple(grads)


class SocialNCE(torch.nn.Module):
    """The event encoder phi(x, y, d) = W2 relu(W1 [x, y, d] + b1) + b2 and the projection head
    psi(h) = V2 relu(V1 h + c1) + c2 of the Social-NCE term, and the term itself (module docstring).

    hidden_dim: the LSTM's width; mlp_dim in (16, 32, 64) and head_dim in (4, 8, 16): the MLPs' hidden and output
    widths; horizon >= 1 future steps; temperature > 0; rho >= 0 and sigma >= 0 in metres."""

    def __init__(self, hidden_dim, mlp_dim=32, head_dim=8, horizon=4, temperature=0.1, rho=0.2, sigma=0.05):
        super().__init__()
        if not 1 <= int(hidden_dim) <= 1024:
            raise ValueError("hidden_dim must be in 1..1024, got %r" % (hidden_dim,))
        if mlp_dim not in MLP_DIMS or head_dim not in HEAD_DIMS:
            raise ValueError("Social-NCE is built for mlp_dim in %s and head_dim in %s, got %r, %r"
                             % (MLP_DIMS, HEAD_DIMS, mlp_dim, head_dim))
        if int(horizon) != horizon or horizon < 1:
            raise ValueError("horizon must be an integer >= 1, got %r" % (horizon,))
        if not temperature > 0:
            raise ValueError("temperature must be > 0, got %r" % (temperature,))
        if not (rho >= 0 and sigma >= 0):
            raise ValueError("rho and sigma must be >= 0, got %r, %r" % (rho, sigma))
        self.hidden_dim, self.mlp_dim, self.head_dim, self.horizon = int(hidden_dim), mlp_dim, head_dim, int(horizon)
        self.temperature, self.rho, self.sigma = float(temperature), float(rho), float(sigma)
        self.event_encoder = torch.nn.Sequential(torch.nn.Linear(3, mlp_dim), torch.nn.ReLU(),
                                                 torch.nn.Linear(mlp_dim, head_dim))
        self.head = torch.nn.Sequential(torch.nn.Linear(hidden_dim, mlp_dim), torch.nn.ReLU(),
                                        torch.nn.Linear(mlp_dim, head_dim))
        self.fixed_eps = None       # a tensor of eps_shape: used instead of the call's draw (tests)

    def eps_shape(self, batch_split):
        """The shape of one call's eps: [B, horizon, 1 + 8 (n_max - 1), 2]."""
        sizes = [int(b) - int(a) for a, b in zip(batch_split[:-1], batch_split[1:])]
        n_max = max(sizes) if sizes else 1
        return (len(sizes), self.horizon, 1 + 8 * (n_max - 1), 2)

    def forward(self, scene, hidden, batch_split, obs_length, return_terms=False, layouts=None):
        """L_nce (0-dim) of the scenes of `batch_split` (a host sequence or tensor).

        scene [T, M, 2] float32 on the device: observed and future positions (the trainer's batch_scene);
        hidden [M, H]: every track's hidden state after the step that consumed frame obs_length - 1 (the query is
        each scene's first row).  return_terms: also the per-pair terms and finiteness [B, horizon] (not
        differentiable).  layouts: the LayoutCache to take the batch's layout from (the trainer passes the model's, so a
        training step builds one layout per batch, not two); None: the module's own.  The call draws eps with
        torch.randn unless `fixed_eps` is set, and makes no host synchronisation."""
        if not (torch.is_tensor(scene) and scene.is_cuda and scene.dtype == torch.float32):
            _lib.require_cuda()
            raise RuntimeError("scene must be a CUDA float32 tensor: Social-NCE runs on the GPU only")
        device = scene.device
        obs_frame = int(obs_length) - 1
        if obs_frame < 0 or obs_frame + self.horizon >= scene.shape[0]:
            raise ValueError("scene has %d frames: obs_length %d + horizon %d do not fit"
                             % (scene.shape[0], obs_length, self.horizon))
        layout = (_layouts if layouts is None else layouts).get(batch_split, device=device)
        if scene.shape[1] != layout.num_tracks or tuple(hidden.shape) != (layout.num_tracks, self.hidden_dim):
            raise ValueError("scene [T, M, 2] and hidden [M, %d] must match batch_split (M = %d)"
                             % (self.hidden_dim, layout.num_tracks))
        shape = self.eps_shape(layout.offsets)
        if self.fixed_eps is not None:
            if tuple(self.fixed_eps.shape) != shape:
                raise ValueError("fixed_eps has shape %s, this call needs %s" % (tuple(self.fixed_eps.shape), shape))
            eps = self.fixed_eps.to(device=device, dtype=torch.float32).contiguous()
        else:
            eps = torch.randn(shape, dtype=torch.float32, device=device)
        loss, terms, valid = _SocialNCEFn.apply(self, scene.contiguous(), hidden.to(torch.float32).contiguous(),
                                                layout, obs_frame, eps, *self.parameters())
        return (loss, terms, valid) if return_terms else loss


def check_contrast(model):
    """NotImplementedError (or the training path's own error) for a model the Social-NCE term cannot train: the
    refusals of check_trainable first, then S-GAN / VAE and user-defined interaction modules."""
    from .external import is_external
    from .lstm import LSTM
    from .trainer import check_trainable
    check_trainable(model)
    if type(model) is not LSTM:
        raise NotImplementedError("Social-NCE training of %s (S-GAN / VAE) is not built" % type(model).__name__)
    if is_external(model.pool):
        raise NotImplementedError("Social-NCE training with a user-defined interaction module (%s) is not built"
                                  % type(model.pool).__name__)
