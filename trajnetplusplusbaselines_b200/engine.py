"""Thin host-side owner of the C-ABI handles (model weights, scene layout, scratch).

PyTorch is plumbing here: it owns device memory and streams; every computation on the hot
path happens inside libtrajnet_b200.so.
"""
import ctypes
import weakref
from collections import OrderedDict

import torch

from . import _lib


# Parameter changes are detected through (data_ptr, _version) of every parameter.  Fused / foreach
# optimizers (torch.optim.Adam(fused=True)) update parameters without bumping `_version`, so every
# optimizer step additionally advances this epoch, which is part of the weight key.
_optimizer_epoch = [0]


def _on_optimizer_step(optimizer, args, kwargs):
    _optimizer_epoch[0] += 1


try:
    from torch.optim.optimizer import register_optimizer_step_post_hook
    register_optimizer_step_post_hook(_on_optimizer_step)
except Exception:      # very old torch: training forwards re-upload unconditionally (see LSTM._engine)
    pass


def weights_key(module):
    """Changes whenever a parameter of `module` may have changed."""
    return (_optimizer_epoch[0],) + tuple((p.data_ptr(), p._version) for p in module.parameters())


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def linear_on(linear, device):
    """(weight, bias) of a torch.nn.Linear as fp32 contiguous tensors on `device`, for a kernel that reads them."""
    return tuple(t.detach().to(device=device, dtype=torch.float32).contiguous() for t in (linear.weight, linear.bias))


def _device_of(device):
    """Resolved CUDA device (the current one when `device` is None or an index-less 'cuda')."""
    device = torch.device('cuda' if device is None else device)
    if device.type != 'cuda':
        raise RuntimeError("scene layouts live in device memory: got device %s" % device)
    if device.index is None:
        device = torch.device('cuda', torch.cuda.current_device())
    return device


class SceneLayout:
    """tb2_layout wrapper: the `batch_split` partition of tracks into scenes.  The handle owns device
    buffers, allocated on `device` (default: the current CUDA device); a layout must only be used with
    models / tensors of that device."""

    def __init__(self, batch_split, pad_to_batch_max=True, device=None):
        _lib.require_cuda()
        lib = _lib.load()
        self.device = _device_of(device)
        offs = [int(v) for v in batch_split]
        self.offsets = offs
        arr = (ctypes.c_int64 * len(offs))(*offs)
        handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_layout_create(arr, len(offs) - 1, ctypes.byref(handle)))
        self.handle = handle
        self.num_scenes = len(offs) - 1
        self.num_tracks = offs[-1]
        self.max_scene = int(lib.tb2_layout_max_scene(handle))
        self.pad_to_batch_max = bool(pad_to_batch_max)
        if not pad_to_batch_max:     # evaluator semantics: every scene as if called on its own
            _lib.check(lib.tb2_layout_set_padding(handle, 0))
        self._finalizer = weakref.finalize(self, lib.tb2_layout_destroy, handle)


class LayoutCache:
    def __init__(self, capacity=8):
        self.capacity = capacity
        self._items = OrderedDict()

    def get(self, batch_split, pad_to_batch_max=True, device=None):
        """batch_split: a sequence, tensor or array of offsets."""
        device = _device_of(device)
        if hasattr(batch_split, 'tolist'):       # one conversion instead of a 0-d tensor per element
            batch_split = batch_split.tolist()
        key = tuple(int(v) for v in batch_split) + (bool(pad_to_batch_max), device.index)
        item = self._items.get(key)
        if item is None:
            item = SceneLayout(key[:-2], pad_to_batch_max, device)
            self._items[key] = item
            if len(self._items) > self.capacity:
                self._items.popitem(last=False)
        else:
            self._items.move_to_end(key)
        return item


def lstm_config(hidden_dim, embedding_dim, pool_to_input, pool, goal_dim=0):
    """tb2_lstm_config of an LSTM of these widths around the interaction module `pool` (None: no pooling); goal_dim > 0:
    the LSTM input carries a goal embedding of that width (LSTM(goal_flag=True))."""
    cfg = _lib.LstmConfig()
    cfg.hidden_dim = int(hidden_dim)
    cfg.embedding_dim = int(embedding_dim)
    cfg.goal_dim = int(goal_dim)
    cfg.pool_to_input = int(bool(pool_to_input))
    cfg.pool_type = _lib.POOL_NONE
    cfg.pool_size = cfg.blur_size = 1
    if pool is not None and hasattr(pool, 'fill_config'):
        pool.fill_config(cfg)
    elif pool is not None:       # a module of the caller's, run in torch between the step's kernels (lstm/external.py)
        cfg.pool_type = _lib.POOL_EXTERNAL
        cfg.out_dim = int(pool.out_dim)
    return cfg


class PoolPlug(torch.nn.Module):
    """Base of the interaction modules (GridBasedPooling and the non-grid modules).

    Inside `LSTM.forward` a module is not called: the fused sequence entry point reads its configuration
    (`fill_config`) and parameters (`weight_fields`).  Called on its own, the module is the reference's pool plug,
    `(hidden_states [B, N, H], obs1 [B, N, 2], obs2 [B, N, 2]) -> [B * N, width]`, run through a model handle of its
    own (tb2_pool_forward) whose LSTM-cell slots hold zeros: tb2_lstm_set_weights requires them, the pool never
    reads them."""
    _reads_hidden = False       # the plug reads hidden states (and its handle's LSTM width is theirs)
    stateful = False            # carries an LSTM state of its own through the time loop, kept in the engine's workspace

    def __init__(self):
        super().__init__()
        self._handle = None
        self._layouts = LayoutCache()

    def __getstate__(self):
        """The per-process device handles of the plug (model handle, layouts, zero LSTM-cell weights,
        interaction-encoder state bookkeeping) are never pickled (LSTMPredictor.save pickles the whole model,
        lstm.py:270-277); they are rebuilt lazily after loading."""
        state = self.__dict__.copy()
        state.pop('_compiled_call_impl', None)         # like torch.nn.Module.__getstate__
        state['_handle'] = None
        state['_layouts'] = LayoutCache()
        state.pop('_standalone_dummy', None)
        state.pop('_state_tracks', None)
        if '_reset_pending' in state:
            state['_reset_pending'] = True
        return state

    def weights_version(self):
        return weights_key(self)

    def reset(self, num_tracks, max_num_neigh, device):
        """The reference resets per-call pool state here; a stateless module keeps none."""
        self.track_mask = None

    def _plug_width(self):
        """LSTM width of the plug's handle: that of the hidden states it reads, else any supported width."""
        return int(self.hidden_dim) if self._reads_hidden else 128

    def _plug_out_dim(self):
        """Width of the plug's output."""
        return int(self.out_dim)

    def _plug_device(self, obs1):
        device = next(self.parameters()).device
        if device.type != 'cuda':
            raise RuntimeError("%s runs on CUDA only: move the module to the GPU (module.cuda())" % type(self).__name__)
        return device

    def _plug_state(self, handle, layout):
        """Bookkeeping of a stateful module before a plug call."""

    def _plug_handle(self, device):
        """The plug's model handle on `device` with the module's current weights."""
        if self._handle is None or self._handle.device != device:
            self._handle = ModelHandle(lstm_config(self._plug_width(), 64, True, self), device)
            self._standalone_dummy = None
        if getattr(self, '_standalone_dummy', None) is None:
            z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
            H, in_dim = self._plug_width(), 64 + self._plug_out_dim()
            self._standalone_dummy = dict(
                input_embedding_weight=z(62, 2), input_embedding_bias=z(62),
                encoder_weight_ih=z(4 * H, in_dim), encoder_weight_hh=z(4 * H, H),
                encoder_bias_ih=z(4 * H), encoder_bias_hh=z(4 * H),
                decoder_weight_ih=z(4 * H, in_dim), decoder_weight_hh=z(4 * H, H),
                decoder_bias_ih=z(4 * H), decoder_bias_hh=z(4 * H),
                hidden2normal_weight=z(5, H), hidden2normal_bias=z(5))
        fields = dict(self._standalone_dummy)
        fields.update(self.weight_fields())
        self._handle.set_weights(fields, key=self.weights_version())
        return self._handle

    def forward(self, hidden_states, obs1, obs2):
        """[B, N, H], [B, N, 2], [B, N, 2] -> [B * N, width] on the device of obs1."""
        _lib.require_cuda()
        batch_size, num_tracks = obs1.size(0), obs1.size(1)
        device = self._plug_device(obs1)
        if self._reads_hidden and hidden_states.size(-1) != self.hidden_dim:
            raise ValueError("hidden_states width != hidden_dim")
        handle = self._plug_handle(device)
        layout = self._layouts.get(range(0, batch_size * num_tracks + 1, num_tracks), device=device)
        self._plug_state(handle, layout)
        f32 = dict(device=device, dtype=torch.float32)
        o1 = obs1.detach().to(**f32).reshape(-1, 2).contiguous()
        o2 = obs2.detach().to(**f32).reshape(-1, 2).contiguous()
        hid = None
        if self._reads_hidden:
            hid = hidden_states.detach().to(**f32).reshape(batch_size * num_tracks, -1).contiguous()
        out = handle.pool_forward(layout, hid, o1, o2, self._plug_out_dim())
        return out.to(obs1.device) if obs1.device != device else out


class ModelHandle:
    """tb2_lstm wrapper: configuration + repacked weights on one device."""

    def __init__(self, config, device):
        _lib.require_cuda()
        lib = _lib.load()
        self.device = torch.device(device)
        self.config = config
        handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_lstm_create(ctypes.byref(config), ctypes.byref(handle)))
        self.handle = handle
        self._finalizer = weakref.finalize(self, lib.tb2_lstm_destroy, handle)
        self._weights_key = None
        self._workspace = None

    def weights_struct(self, named):
        """tb2_lstm_weights from a dict field name -> tensor (or list of 3 for the MLP)."""
        w = _lib.LstmWeights()
        keep = []
        for field, value in named.items():
            if isinstance(value, (list, tuple)):
                arr = getattr(w, field)
                for i, t in enumerate(value):
                    if t is not None:
                        t = self._prep(t)
                        keep.append(t)
                        arr[i] = t.data_ptr()
            elif value is not None:
                t = self._prep(value)
                keep.append(t)
                setattr(w, field, t.data_ptr())
        return w, keep

    def set_weights(self, named, key=None, force=False):
        """named: dict field name -> CUDA fp32 contiguous tensor (or list of 3 for the MLP)."""
        if not force and key is not None and key == self._weights_key:
            return
        lib = _lib.load()
        w, keep = self.weights_struct(named)
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_lstm_set_weights(self.handle, ctypes.byref(w), _stream(self.device)))
        # the repack kernels read `keep` asynchronously on the current stream; record usage
        for t in keep:
            t.record_stream(torch.cuda.current_stream(self.device))
        self._weights_key = key

    def _prep(self, t):
        t = t.detach()
        if t.device != self.device or t.dtype != torch.float32 or not t.is_contiguous():
            t = t.to(device=self.device, dtype=torch.float32).contiguous()
        return t

    def workspace(self, layout):
        lib = _lib.load()
        need = int(lib.tb2_lstm_workspace_bytes(self.handle, layout.handle))
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._workspace, need

    # -- compute entry points ---------------------------------------------------------------
    def grid_indices(self, layout, obs):
        lib = _lib.load()
        nm1 = max(layout.max_scene - 1, 0)
        cells = torch.empty((layout.num_tracks, nm1), dtype=torch.int32, device=self.device)
        flags = torch.empty((layout.num_tracks, nm1), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_grid_indices(self.handle, layout.handle, _ptr(obs), _ptr(cells),
                                            _ptr(flags), _stream(self.device)))
        return cells, flags

    def pool_forward(self, layout, hidden, obs1, obs2, out_dim):
        lib = _lib.load()
        ws, need = self.workspace(layout)
        out = torch.empty((layout.num_tracks, out_dim), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_pool_forward(self.handle, layout.handle, _ptr(hidden), _ptr(obs1),
                                            _ptr(obs2), _ptr(out), _ptr(ws), need, _stream(self.device)))
        return out

    def pool_state_reset(self, layout):
        """tb2_pool_state_reset: zero the interaction-encoder LSTM state of a stateful pool in this handle's workspace."""
        lib = _lib.load()
        ws, need = self.workspace(layout)
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_pool_state_reset(self.handle, layout.handle, _ptr(ws), need, _stream(self.device)))

    # goals: [M, 2] fp32 device tensor of a goal-conditioned model (None for any other; the library refuses a goal model
    # without them)
    def step_forward(self, layout, phase, obs1, obs2, h, c, goals=None, pooled=None, h_out=None, c_out=None):
        """One step (tb2_lstm_step_forward); without h_out / c_out, h and c are updated in place.  pooled: the external
        interaction module's output [B * n_pad, out_dim] (TB2_POOL_EXTERNAL models only).  Returns (normal [M,5],
        pos [M,2])."""
        lib = _lib.load()
        ws, need = self.workspace(layout)
        M = layout.num_tracks
        normal = torch.empty((M, 5), dtype=torch.float32, device=self.device)
        pos = torch.empty((M, 2), dtype=torch.float32, device=self.device)
        h_out = h if h_out is None else h_out
        c_out = c if c_out is None else c_out
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_lstm_step_forward(self.handle, layout.handle, phase, _ptr(obs1), _ptr(obs2), _ptr(goals),
                                                 _ptr(pooled), _ptr(h), _ptr(c), _ptr(h_out), _ptr(c_out), _ptr(normal),
                                                 _ptr(pos), _ptr(ws), need, _stream(self.device)))
        return normal, pos

    def forward_steps(self, layout, observed, truth, n_decode, first_step, last_step, normals, positions, h, c,
                      goals=None, eps=None, states=None, cache=None, host=None):
        """Steps [first_step, last_step) of the time loop on caller-owned state (tb2_lstm_forward_steps).
        eps [n_decode + 1, M, 2]: every predicted position is drawn from its step's normal at these standard normal
        pairs.  states [S, 2, M, H]: the state after every step.  cache: uint8 device tensor of train_cache_bytes,
        where the social pooling keeps its per-step records for tb2_lstm_sequence_backward.  host = (normals_host,
        positions_host, copy_stream): every step's results are copied to the pinned host tensors on copy_stream,
        which the caller synchronises before reading them."""
        lib = _lib.load()
        ws, need = self.workspace(layout)
        normals_host, positions_host, copy_stream = host if host is not None else (None, None, None)
        with torch.cuda.device(self.device):
            _lib.check(lib.tb2_lstm_forward_steps(
                self.handle, layout.handle, _ptr(observed), int(observed.shape[0]), _ptr(truth), int(n_decode),
                _ptr(goals), _ptr(eps), int(first_step), int(last_step), _ptr(normals), _ptr(positions), _ptr(h),
                _ptr(c), _ptr(states), _ptr(cache), 0 if cache is None else int(cache.numel()), _ptr(normals_host),
                _ptr(positions_host), ctypes.c_void_p(copy_stream.cuda_stream if copy_stream is not None else 0),
                _ptr(ws), need, _stream(self.device)))

    def forward_steps_sampled(self, layout, observed, truth, n_decode, first_step, last_step, eps, normals, positions, h,
                              c):
        """forward_steps with every predicted position drawn from its step's normal at the standard normal pairs
        eps [n_decode + 1, M, 2]."""
        self.forward_steps(layout, observed, truth, n_decode, first_step, last_step, normals, positions, h, c, eps=eps)

    def train_cache_bytes(self, layout, num_steps):
        return int(_lib.load().tb2_lstm_train_cache_bytes(self.handle, layout.handle, int(num_steps)))
