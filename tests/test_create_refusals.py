"""tb2_lstm_create refuses every invalid configuration with a fixed return code and message, before any CUDA call
(so the table runs with or without a GPU).  Each pool type's own checks come before the shared `pool_to_input` rule,
and nn_lstm's velocity / width check before the nearest-neighbour check it shares with nn."""
import ctypes

import pytest

INVALID, UNSUPPORTED = -1, -3
I = "invalid argument: "
GRID_POOL_SIZE = "pool_size / blur_size != 1 are not built (the reference CLI never sets them)"
NN = I + "nearest-neighbour pooling needs 1 <= n <= 32 and out_dim == n * mlp_dim_spatial"
NN_LSTM = I + "nearest-neighbour LSTM pooling needs 1 <= hidden_dim <= 512, out_dim <= 1024 and velocities"
TRAJ = I + "Trajectron pooling needs 1 <= hidden_dim <= 512 and out_dim <= 1024"
ATTN = I + "attention pooling needs mlp_dim <= 128 (kernel specialisation)"
HIDDEN = I + "hidden-state MLP pooling widths"
POOL_TO_INPUT = I + "pool_to_input=0 needs out_dim == hidden_dim"

# an accepted configuration of every pool type (the reference trainer's defaults), hidden_dim = 128
VALID = {
    "vanilla": dict(pool_type=0),
    "occupancy": dict(pool_type=1, n=4, cell_side=2.0, num_layers=1, out_dim=128),
    "directional": dict(pool_type=2, n=4, cell_side=2.0, num_layers=1, out_dim=128),
    "social": dict(pool_type=3, n=16, cell_side=0.6, latent_dim=16, num_layers=2, layer_dims=(1024, 0), out_dim=256),
    "hiddenstatemlp": dict(pool_type=4, out_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, mlp_dim_hidden=64),
    "nn": dict(pool_type=5, n=4, out_dim=32, mlp_dim_spatial=8, mlp_dim_vel=1),
    "attentionmlp": dict(pool_type=6, out_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, mlp_dim_hidden=64),
    "nn_lstm": dict(pool_type=7, n=4, out_dim=32, mlp_dim_spatial=8, mlp_dim_vel=1, mlp_dim_hidden=256),
    "traj_pool": dict(pool_type=8, n=4, out_dim=32, mlp_dim_spatial=32, mlp_dim_vel=1, mlp_dim_hidden=256),
}

# (kind, changes to its valid configuration, return code, tb2_last_error())
REFUSALS = [
    ("vanilla", dict(hidden_dim=100), UNSUPPORTED,
     "hidden_dim must be a multiple of 32 from 32 to 256 (32, 64, 96, ..., 256)"),
    ("vanilla", dict(embedding_dim=3), INVALID, I + "embedding_dim out of range"),
    ("social", dict(embedding_dim=1025), INVALID, I + "embedding_dim out of range"),
    ("vanilla", dict(pool_type=-1), INVALID, I + "bad pool_type"),
    ("vanilla", dict(pool_type=9), INVALID, I + "bad pool_type"),
    # grids
    ("occupancy", dict(pool_size=2), UNSUPPORTED, GRID_POOL_SIZE),
    ("social", dict(blur_size=3), UNSUPPORTED, GRID_POOL_SIZE),
    ("directional", dict(pool_size=2, n=0, pool_to_input=0, out_dim=64), UNSUPPORTED, GRID_POOL_SIZE),
    ("occupancy", dict(n=0), INVALID, I + "grid size"),
    ("directional", dict(n=65), INVALID, I + "grid size"),
    ("social", dict(cell_side=0.0), INVALID, I + "grid size"),
    ("occupancy", dict(num_layers=4), INVALID, I + "num_layers"),
    ("directional", dict(num_layers=-1), INVALID, I + "num_layers"),
    ("social", dict(latent_dim=12), UNSUPPORTED, "social latent_dim must be 4, 8, 16 or 32"),
    ("social", dict(latent_dim=64, pool_to_input=0), UNSUPPORTED, "social latent_dim must be 4, 8, 16 or 32"),
    ("social", dict(layer_dims=(0, 0)), INVALID, I + "MLP width"),
    ("occupancy", dict(num_layers=3, layer_dims=(64, -1)), INVALID, I + "MLP width"),
    ("occupancy", dict(out_dim=0, pool_to_input=0), INVALID, I + "MLP width"),
    # nearest-neighbour MLP / LSTM
    ("nn", dict(n=0), INVALID, NN),
    ("nn", dict(n=33, out_dim=33 * 8), INVALID, NN),
    ("nn", dict(mlp_dim_spatial=0, out_dim=0), INVALID, NN),
    ("nn", dict(out_dim=31), INVALID, NN),
    ("nn", dict(n=0, pool_to_input=0), INVALID, NN),
    ("nn_lstm", dict(mlp_dim_vel=0), INVALID, NN_LSTM),
    ("nn_lstm", dict(mlp_dim_vel=0, n=0), INVALID, NN_LSTM),
    ("nn_lstm", dict(mlp_dim_hidden=0), INVALID, NN_LSTM),
    ("nn_lstm", dict(mlp_dim_hidden=513), INVALID, NN_LSTM),
    ("nn_lstm", dict(n=32, mlp_dim_spatial=33, out_dim=32 * 33), INVALID, NN_LSTM),
    ("nn_lstm", dict(n=0), INVALID, NN),
    ("nn_lstm", dict(out_dim=36, pool_to_input=0), INVALID, NN),
    # Trajectron
    ("traj_pool", dict(mlp_dim_hidden=0), INVALID, TRAJ),
    ("traj_pool", dict(mlp_dim_hidden=513), INVALID, TRAJ),
    ("traj_pool", dict(out_dim=0), INVALID, TRAJ),
    ("traj_pool", dict(out_dim=1025, pool_to_input=0), INVALID, TRAJ),
    # attention / hidden-state MLP
    ("attentionmlp", dict(mlp_dim_hidden=65), INVALID, ATTN),
    ("attentionmlp", dict(mlp_dim_spatial=0), INVALID, ATTN),
    ("attentionmlp", dict(mlp_dim_vel=-1), INVALID, ATTN),
    ("attentionmlp", dict(out_dim=0, pool_to_input=0), INVALID, ATTN),
    ("hiddenstatemlp", dict(mlp_dim_spatial=0), INVALID, HIDDEN),
    ("hiddenstatemlp", dict(mlp_dim_hidden=-1), INVALID, HIDDEN),
    ("hiddenstatemlp", dict(mlp_dim_hidden=4096 - 63), INVALID, HIDDEN),
    ("hiddenstatemlp", dict(out_dim=0), INVALID, HIDDEN),
] + [
    # pool_to_input = 0 adds the pool output to the hidden state: its width must be hidden_dim, for every pool type
    (kind, dict(pool_to_input=0, **changes), INVALID, POOL_TO_INPUT) for kind, changes in [
        ("occupancy", dict(num_layers=0)),
        ("directional", dict(out_dim=64)),
        ("social", dict()),
        ("hiddenstatemlp", dict(out_dim=64)),
        ("nn", dict()),
        ("attentionmlp", dict(out_dim=256)),
        ("nn_lstm", dict()),
        ("traj_pool", dict(out_dim=129)),
    ]
]


def _config(kind, changes):
    from trajnetplusplusbaselines_b200 import _lib
    cfg = _lib.LstmConfig()
    cfg.hidden_dim, cfg.embedding_dim, cfg.pool_to_input = 128, 64, 1
    cfg.pool_size = cfg.blur_size = 1
    for field, value in dict(VALID[kind], **changes).items():
        if field == "layer_dims":
            cfg.layer_dims[0], cfg.layer_dims[1] = value
        else:
            setattr(cfg, field, value)
    return cfg


@pytest.mark.parametrize("kind,changes,rc,message", REFUSALS,
                         ids=["%s-%s" % (k, "-".join("%s=%s" % kv for kv in c.items())) for k, c, _, _ in REFUSALS])
def test_create_refuses_invalid_configuration(kind, changes, rc, message):
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    handle = ctypes.c_void_p()
    got = lib.tb2_lstm_create(ctypes.byref(_config(kind, changes)), ctypes.byref(handle))
    assert (got, lib.tb2_last_error().decode()) == (rc, message)
    assert not handle.value
