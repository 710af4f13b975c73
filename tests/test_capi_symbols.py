"""The C-ABI library loads and exports every symbol include/trajnet_b200.h declares (CPU only;
no compute calls)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "trajnet_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tb2_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_header_symbols():
    from trajnetplusplusbaselines_b200 import build, _lib
    build.build()
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 15
    for name in names:
        assert hasattr(lib, name), "missing export: " + name
        assert name in _lib.PROTOTYPES, "ctypes prototype missing for " + name
    assert lib.tb2_version() >= 100


# size_t and uint64_t are the same 64-bit unsigned type on the platforms the library builds for (ctypes.c_size_t is
# ctypes.c_uint64 there)
_C_KINDS = {"int": "int32", "int32_t": "int32", "int64_t": "int64", "size_t": "size_t", "uint64_t": "size_t",
            "float": "float", "double": "double"}


def _c_kind(c_type):
    return "pointer" if "*" in c_type else _C_KINDS[c_type.replace("const", "").strip()]


def _ctypes_kind(t):
    import ctypes
    if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
        return "pointer"
    for kind, c in (("int32", ctypes.c_int32), ("int64", ctypes.c_int64), ("size_t", ctypes.c_size_t),
                    ("float", ctypes.c_float), ("double", ctypes.c_double)):
        if t is c:
            return kind
    return repr(t)


def test_prototypes_match_header_declarations():
    """Every ctypes prototype passes its function's arguments, and takes its result, as the header declares them: the
    same number, and per position a pointer or a scalar of the same width and type.  A shifted argument would reach
    the library as a garbage pointer."""
    from trajnetplusplusbaselines_b200 import _lib
    text = open(os.path.join(ROOT, "include", "trajnet_b200.h")).read()
    text = re.sub(r"^#.*$", "", re.sub(r"/\*.*?\*/", "", text, flags=re.S), flags=re.M)
    decls = re.findall(r"([^;{}()]*?)\b(tb2_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", text)
    assert sorted(name for _, name, _ in decls) == _declared()
    for ret, name, params in decls:
        params = [] if params.strip() == "void" else [re.sub(r"\w+\s*$", "", p) for p in params.split(",")]
        restype, argtypes = _lib.PROTOTYPES[name]
        assert len(argtypes) == len(params), (name, len(argtypes), len(params))
        assert _ctypes_kind(restype) == _c_kind(ret), name
        for i, (t, p) in enumerate(zip(argtypes, params)):
            assert _ctypes_kind(t) == _c_kind(p), (name, i, p)


def test_no_cpu_fallback_without_cuda():
    import torch
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from trajnetplusplusbaselines_b200.lstm import LSTM
    import numpy as np
    model = LSTM()
    obs = torch.zeros(9, 4, 2)
    with torch.no_grad(), pytest.raises(RuntimeError):
        model(obs, torch.zeros(4, 2), torch.tensor([0, 4]), n_predict=12)


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "trajnetplusplusbaselines_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_state_dict_keys_match_reference_layout():
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    pool = GridBasedPooling(type_='social', hidden_dim=128, cell_side=0.6, n=16, out_dim=256,
                            embedding_arch='two_layer', layer_dims=[1024], latent_dim=16)
    sd = LSTM(pool=pool).state_dict()
    expect = {  # SURVEY.md 8b/B2 (probe of the reference's own state_dict)
        'pool.hidden_dim_encoding.weight': (16, 128), 'pool.embedding.0.weight': (1024, 4096),
        'pool.embedding.2.weight': (256, 1024), 'input_embedding.input_embeddings.0.weight': (62, 2),
        'goal_embedding.input_embeddings.0.weight': (62, 2), 'encoder.weight_ih': (512, 320),
        'encoder.weight_hh': (512, 128), 'decoder.weight_ih': (512, 320),
        'hidden2normal.linear.weight': (5, 128),
    }
    for k, shape in expect.items():
        assert tuple(sd[k].shape) == shape, k


def test_header_is_plain_c_and_links(tmp_path):
    """The boundary is a C ABI: a C translation unit (gcc, not nvcc / g++) includes the header, takes the
    address of every entry point and links against the shared library."""
    import re
    import subprocess
    header = open(os.path.join(ROOT, "include", "trajnet_b200.h")).read()
    names = sorted(set(re.findall(r"\b(tb2_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 20
    src = os.path.join(tmp_path, "abi.c")
    with open(src, "w") as f:
        f.write('#include "trajnet_b200.h"\n#include <stdio.h>\ntypedef void (*fn_t)(void);\n'
                'int main(void) {\n    fn_t fns[] = {\n')
        f.write("".join("        (fn_t)%s,\n" % n for n in names))
        f.write('    };\n    printf("%d %d\\n", (int)(sizeof(fns) / sizeof(fns[0])), tb2_version());\n    return 0;\n}\n')
    libdir = os.path.join(ROOT, "trajnetplusplusbaselines_b200")
    exe = os.path.join(tmp_path, "abi")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                    "-L", libdir, "-l:libtrajnet_b200.so", "-Wl,-rpath," + libdir], check=True)
    out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()
    assert int(out[0]) == len(names) and int(out[1]) > 0


def test_weight_key_follows_optimizer_steps():
    """engine.weights_key must change after ANY optimizer step (fused optimizers do not bump the
    parameters' version counters) and stay put otherwise."""
    import torch
    from trajnetplusplusbaselines_b200.engine import weights_key
    lin = torch.nn.Linear(4, 3)
    k0 = weights_key(lin)
    assert weights_key(lin) == k0
    opt = torch.optim.SGD(lin.parameters(), lr=0.1)
    lin(torch.ones(2, 4)).sum().backward()
    opt.step()
    k1 = weights_key(lin)
    assert k1 != k0
    with torch.no_grad():
        lin.weight.add_(1.0)            # plain in-place update: version counter
    assert weights_key(lin) != k1


def _all_model_kinds():
    from oracle import lstm_oracle as O
    kinds = [k for k in O.MODEL_SPECS]
    for table in (O.NONGRID_SPECS, O.NN_SPECS, O.ATTN_SPECS, O.NN_LSTM_SPECS, O.TRAJ_SPECS):
        kinds += list(table)
    return kinds


def _build_pool(kind):
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import lstm as L
    if kind in O.TRAJ_SPECS:
        return L.TrajectronPooling(**O.TRAJ_SPECS[kind])
    if kind in O.NN_LSTM_SPECS:
        return L.NearestNeighborLSTM(**O.NN_LSTM_SPECS[kind])
    if kind in O.NN_SPECS:
        return L.NearestNeighborMLP(**O.NN_SPECS[kind])
    if kind in O.ATTN_SPECS:
        return L.AttentionMLPPooling(**O.ATTN_SPECS[kind])
    if kind in O.NONGRID_SPECS:
        return L.HiddenStateMLPPooling(**O.NONGRID_SPECS[kind])
    spec = O.MODEL_SPECS[kind]
    return L.GridBasedPooling(**spec) if spec is not None else None


@pytest.mark.parametrize("kind", _all_model_kinds())
def test_create_accepts_every_model_configuration(kind):
    """tb2_lstm_create validates the configuration before its first CUDA call: on a box without a GPU every model kind
    must get PAST the validation (TB2_ERR_CUDA from the first allocation), never TB2_ERR_INVALID / _UNSUPPORTED."""
    import ctypes
    import torch
    if torch.cuda.is_available():
        pytest.skip("CPU-side check of the argument validation")
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    cfg = _lib.LstmConfig()
    cfg.hidden_dim, cfg.embedding_dim, cfg.pool_to_input = 128, 64, 1
    cfg.pool_type = _lib.POOL_NONE
    cfg.pool_size = cfg.blur_size = 1
    pool = _build_pool(kind)
    if pool is not None:
        pool.fill_config(cfg)
    handle = ctypes.c_void_p()
    rc = lib.tb2_lstm_create(ctypes.byref(cfg), ctypes.byref(handle))
    assert rc == -2, (kind, rc, lib.tb2_last_error())


@pytest.mark.parametrize("kind", ["social_small", "hiddenstatemlp_small", "nn_small", "attentionmlp_small", "nn_lstm_small",
                                  "traj_pool_small"])
def test_predictor_pickle_drops_device_handles(kind, tmp_path):
    """LSTMPredictor.save pickles the whole model (lstm.py:270-277): the per-process handles a pooling module holds after its
    stand-alone plug was used (ctypes pointers, layouts) must not reach the pickle."""
    import torch
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200.lstm import LSTM, LSTMPredictor
    model = LSTM(pool=_build_pool(kind))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(kind, seed=3).items()})
    unpicklable = lambda: None                       # stands for a ModelHandle / ctypes pointer
    model.pool._handle = unpicklable
    model.pool._layouts._items[("fake",)] = unpicklable
    model.pool._standalone_dummy = {"x": unpicklable}
    model.pool._state_tracks = 5
    if hasattr(model.pool, "_reset_pending"):
        model.pool._reset_pending = False
    fn = str(tmp_path / "m.pkl")
    LSTMPredictor(model).save({"epoch": 0}, fn)
    again = LSTMPredictor.load(fn)
    assert again.model.pool._handle is None and len(again.model.pool._layouts._items) == 0
    assert getattr(again.model.pool, "_standalone_dummy", None) is None
    if hasattr(model.pool, "_reset_pending"):
        assert again.model.pool._reset_pending is True
    for k, v in model.state_dict().items():
        assert torch.equal(v, again.model.state_dict()[k]), k
