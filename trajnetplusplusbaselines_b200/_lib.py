"""ctypes binding of libtrajnet_b200.so (C ABI declared in include/trajnet_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails the
caller gets a RuntimeError.  CUDA is never initialised at import time (fork safety: the
reference evaluator forks joblib workers around the predictor, lstm/trajnet_evaluator.py:61).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtrajnet_b200.so")

POOL_NONE, POOL_OCCUPANCY, POOL_DIRECTIONAL, POOL_SOCIAL, POOL_HIDDEN_MLP, POOL_NN_MLP, POOL_ATTN_MLP, POOL_NN_LSTM, POOL_TRAJECTRON = 0, 1, 2, 3, 4, 5, 6, 7, 8
POOL_EXTERNAL = 16      # any other interaction module: torch runs it between the step's kernels (lstm/external.py)
PHASE_ENCODER, PHASE_DECODER = 0, 1
# LSTM widths the kernels are built for, and tb2_lstm_create's refusal of any other (kHiddenDimMessage, csrc/common.cuh)
HIDDEN_DIMS = tuple(range(32, 257, 32))
HIDDEN_DIM_MESSAGE = "hidden_dim must be a multiple of 32 from 32 to 256 (32, 64, 96, ..., 256)"
SCORE_COL_GT, SCORE_COL_PRED, SCORE_NEIGH_COUNT_DIFFERS, SCORE_NLL_ALL_SKIPPED = 1, 2, 4, 8     # tb2_score_scenes flags

_c_float_p = ctypes.c_void_p   # device pointers travel as integers


class LstmConfig(ctypes.Structure):
    _fields_ = [
        ("hidden_dim", ctypes.c_int32),
        ("embedding_dim", ctypes.c_int32),
        ("pool_type", ctypes.c_int32),
        ("pool_to_input", ctypes.c_int32),
        ("n", ctypes.c_int32),
        ("cell_side", ctypes.c_float),
        ("pool_size", ctypes.c_int32),
        ("blur_size", ctypes.c_int32),
        ("front", ctypes.c_int32),
        ("constant", ctypes.c_float),
        ("latent_dim", ctypes.c_int32),
        ("num_layers", ctypes.c_int32),
        ("layer_dims", ctypes.c_int32 * 2),
        ("out_dim", ctypes.c_int32),
        ("mlp_dim_spatial", ctypes.c_int32),
        ("mlp_dim_vel", ctypes.c_int32),
        ("mlp_dim_hidden", ctypes.c_int32),
        ("attn_fill", ctypes.c_float),
        ("goal_dim", ctypes.c_int32),
    ]


class LstmWeights(ctypes.Structure):
    _fields_ = [
        ("input_embedding_weight", ctypes.c_void_p),
        ("input_embedding_bias", ctypes.c_void_p),
        ("encoder_weight_ih", ctypes.c_void_p),
        ("encoder_weight_hh", ctypes.c_void_p),
        ("encoder_bias_ih", ctypes.c_void_p),
        ("encoder_bias_hh", ctypes.c_void_p),
        ("decoder_weight_ih", ctypes.c_void_p),
        ("decoder_weight_hh", ctypes.c_void_p),
        ("decoder_bias_ih", ctypes.c_void_p),
        ("decoder_bias_hh", ctypes.c_void_p),
        ("hidden2normal_weight", ctypes.c_void_p),
        ("hidden2normal_bias", ctypes.c_void_p),
        ("pool_encoding_weight", ctypes.c_void_p),
        ("pool_encoding_bias", ctypes.c_void_p),
        ("pool_embedding_weight", ctypes.c_void_p * 3),
        ("pool_embedding_bias", ctypes.c_void_p * 3),
        ("pool_spatial_weight", ctypes.c_void_p),
        ("pool_spatial_bias", ctypes.c_void_p),
        ("pool_vel_weight", ctypes.c_void_p),
        ("pool_vel_bias", ctypes.c_void_p),
        ("pool_hidden_weight", ctypes.c_void_p),
        ("pool_hidden_bias", ctypes.c_void_p),
        ("pool_out_weight", ctypes.c_void_p),
        ("pool_out_bias", ctypes.c_void_p),
        ("pool_attn_wq", ctypes.c_void_p),
        ("pool_attn_wk", ctypes.c_void_p),
        ("pool_attn_wv", ctypes.c_void_p),
        ("pool_attn_in_proj_weight", ctypes.c_void_p),
        ("pool_attn_in_proj_bias", ctypes.c_void_p),
        ("pool_attn_out_proj_weight", ctypes.c_void_p),
        ("pool_attn_out_proj_bias", ctypes.c_void_p),
        ("pool_lstm_weight_ih", ctypes.c_void_p),
        ("pool_lstm_weight_hh", ctypes.c_void_p),
        ("pool_lstm_bias_ih", ctypes.c_void_p),
        ("pool_lstm_bias_hh", ctypes.c_void_p),
        ("goal_embedding_weight", ctypes.c_void_p),
        ("goal_embedding_bias", ctypes.c_void_p),
    ]


class LstmGrads(ctypes.Structure):
    _fields_ = [(name, ctypes.c_void_p) for name in (
        "input_embedding_weight", "input_embedding_bias",
        "encoder_weight_ih", "encoder_weight_hh", "encoder_bias_ih", "encoder_bias_hh",
        "decoder_weight_ih", "decoder_weight_hh", "decoder_bias_ih", "decoder_bias_hh",
        "hidden2normal_weight", "hidden2normal_bias",
        "pool_embedding_weight0", "pool_embedding_bias0", "pool_embedding_weight1", "pool_embedding_bias1",
        "pool_encoding_weight", "pool_encoding_bias", "d_observed", "d_obs1", "d_obs2")]


class SfParams(ctypes.Structure):
    _fields_ = [
        ("delta_t", ctypes.c_double),
        ("tau", ctypes.c_double),
        ("v0", ctypes.c_double),
        ("sigma", ctypes.c_double),
        ("n_steps", ctypes.c_int32),
        ("sample_every", ctypes.c_int32),
    ]


class OrcaParams(ctypes.Structure):
    _fields_ = [
        ("time_step", ctypes.c_float),
        ("neighbor_dist", ctypes.c_float),
        ("max_neighbors", ctypes.c_int32),
        ("time_horizon", ctypes.c_float),
        ("radius", ctypes.c_float),
        ("end_range", ctypes.c_double),
        ("n_steps", ctypes.c_int32),
        ("sample_every", ctypes.c_int32),
    ]


_vp = ctypes.c_void_p
_i32 = ctypes.c_int32
_sz = ctypes.c_size_t

# name -> (restype, argtypes); must list every symbol include/trajnet_b200.h declares
PROTOTYPES = {
    "tb2_last_error": (ctypes.c_char_p, []),
    "tb2_version": (ctypes.c_int, []),
    "tb2_launch_count": (ctypes.c_uint64, []),
    "tb2_profile_begin": (ctypes.c_int, []),
    "tb2_profile_end": (ctypes.c_int, [ctypes.c_char_p, _sz]),
    "tb2_lstm_create": (ctypes.c_int, [ctypes.POINTER(LstmConfig), ctypes.POINTER(_vp)]),
    "tb2_lstm_destroy": (ctypes.c_int, [_vp]),
    "tb2_lstm_set_weights": (ctypes.c_int, [_vp, ctypes.POINTER(LstmWeights), _vp]),
    "tb2_layout_create": (ctypes.c_int, [ctypes.POINTER(ctypes.c_int64), _i32, ctypes.POINTER(_vp)]),
    "tb2_layout_destroy": (ctypes.c_int, [_vp]),
    "tb2_layout_num_tracks": (_i32, [_vp]),
    "tb2_layout_max_scene": (_i32, [_vp]),
    "tb2_layout_set_padding": (ctypes.c_int, [_vp, _i32]),
    "tb2_lstm_workspace_bytes": (_sz, [_vp, _vp]),
    "tb2_grid_indices": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "tb2_pool_forward": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "tb2_lstm_step_forward": (ctypes.c_int, [_vp, _vp, _i32] + [_vp] * 11 + [_sz, _vp]),
    "tb2_lstm_forward_steps": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp,
                                              _vp, _sz, _vp, _vp, _vp, _vp, _sz, _vp]),
    "tb2_lstm_sample_positions": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp]),
    "tb2_lstm_backward_workspace_bytes": (_sz, [_vp, _vp, _i32, _i32]),
    "tb2_lstm_sequence_backward": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(LstmWeights), _vp, _i32, _vp, _i32,
                                                  _vp, _vp, _vp, _vp, _i32, ctypes.POINTER(LstmGrads),
                                                  _vp, _sz, _vp, _sz, _vp, _sz, _vp]),
    "tb2_lstm_rollout_backward": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(LstmWeights), _vp, _i32, _i32, _vp, _vp, _vp,
                                                 _vp, _vp, _i32, ctypes.POINTER(LstmGrads), _vp, _sz, _vp, _sz, _vp, _sz,
                                                 _vp]),
    "tb2_lstm_relevance_workspace_bytes": (_sz, [_vp, _vp, _i32, _i32]),
    "tb2_lstm_relevance": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(LstmWeights), _vp, _i32, _i32, _vp, _vp, ctypes.c_float,
                                          _vp, _vp, _vp, _sz, _vp]),
    "tb2_shapley_expand": (ctypes.c_int, [_vp, _i32, _i32, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "tb2_shapley_values": (ctypes.c_int, [_vp, _i32, _i32, _i32, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                          _vp]),
    "tb2_attack_objective": (ctypes.c_int, [_vp, _vp, _i32, _i32, _vp, _vp, _vp]),
    "tb2_attack_step": (ctypes.c_int, [_vp, _vp, _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp,
                                       ctypes.c_float, ctypes.c_float, _i32, _vp]),
    "tb2_pool_state_reset": (ctypes.c_int, [_vp, _vp, _vp, _sz, _vp]),
    "tb2_pool_inputs_padded": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp]),
    "tb2_pool_inputs_padded_backward": (ctypes.c_int, [_vp, _vp, _i32, _vp, _vp]),
    "tb2_lstm_step_backward_workspace_bytes": (_sz, [_vp, _vp]),
    "tb2_lstm_step_backward": (ctypes.c_int, [_vp, _vp, ctypes.POINTER(LstmWeights), _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                              _vp, _vp, _vp, _vp, _vp, ctypes.POINTER(LstmGrads), _vp, _sz, _vp]),
    "tb2_lstm_train_cache_bytes": (_sz, [_vp, _vp, _i32]),
    "tb2_sgan_add_noise": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "tb2_vae_scale_hidden": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _vp]),
    "tb2_sgan_decoder_context": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "tb2_vae_decoder_context": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp]),
    "tb2_prediction_loss": (ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, ctypes.c_float, _vp, _vp, _vp]),
    "tb2_l2_loss": (ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "tb2_collision_loss": (ctypes.c_int, [_vp, _vp, _i32, ctypes.c_float, ctypes.c_float, _vp, _vp, _vp]),
    "tb2_scenes_drop_distant": (ctypes.c_int, [_vp, _vp, _i32, _i32, _i32, ctypes.c_double, _vp, _vp, _vp]),
    "tb2_scenes_transform": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "tb2_scenes_inverse": (ctypes.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp]),
    "tb2_scenes_gather_epoch": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i32, _i32, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp,
                                               _vp, _i32, _vp, _vp]),
    "tb2_ndjson_parse": (ctypes.c_int, [_vp, _sz, ctypes.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "tb2_ndjson_format": (ctypes.c_int64, [ctypes.c_int64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int64]),
    "tb2_ndjson_parse_meta": (ctypes.c_int, [_vp, _sz, ctypes.c_int64] + [_vp] * 15),
    "tb2_score_scenes": (ctypes.c_int, [_i32, _i32, _i32] + [_vp] * 9 + [_i32] + [_vp] * 5),
    "tb2_sf_simulate": (ctypes.c_int, [_vp, ctypes.POINTER(SfParams), _vp, _vp, _vp]),
    "tb2_kalman_predict": (ctypes.c_int, [_vp, _vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp]),
    "tb2_kalman_workspace_bytes": (_sz, [_vp, _i32]),
    "tb2_kalman_predict_device": (ctypes.c_int, [_vp, _vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp,
                                                 _sz, _vp]),
    "tb2_orca_simulate": (ctypes.c_int, [_vp, ctypes.POINTER(OrcaParams), _vp, _vp, _vp, _vp, _vp, _vp]),
    "tb2_sf_sweep": (ctypes.c_int, [_vp, ctypes.POINTER(SfParams), _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp]),
    "tb2_sf_sweep_grad": (ctypes.c_int, [_vp, ctypes.POINTER(SfParams), _vp, _i32, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "tb2_orca_sweep": (ctypes.c_int, [_vp, ctypes.POINTER(OrcaParams), _vp, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp]),
}

_lib = None


def load():
    """Load the shared library (once) and attach the prototypes.  Raises if it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libtrajnet_b200.so is not built (%s). Run `python -m trajnetplusplusbaselines_b200.build`; "
            "there is no CPU fallback for the hot path." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in PROTOTYPES.items():
        fn = getattr(lib, name)     # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        msg = load().tb2_last_error()
        raise RuntimeError("libtrajnet_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("trajnetplusplusbaselines_b200 needs a CUDA device (sm_90a); there is no CPU path")
