"""Generate tests/golden/step_golden.npz from the UNMODIFIED reference (build container).

    python -m oracle.make_step_golden

One LSTM.step and one stand-alone GridBasedPooling call where no other fixture pins them:
  * LSTM.step of the encoder and of the decoder from non-zero (h, c) (h uniform in +-1, c in +-3) at H = 32, 160
    and 224, for a directional and a social model, on ragged scenes with tracks absent at obs1 or at obs2;
  * LSTM(pool_to_input=False) steps (the pooled vector added to h, lstm.py:151) with occupancy, social and
    hiddenstatemlp pools of out_dim = hidden_dim, at H = 32;
  * GridBasedPooling outputs of an occupancy grid with n = 36, a directional grid with n = 26 (first Linears too
    large for the forward's row kernel) and an occupancy grid without embedding (embedding_arch='None').
The grid embedding's biases are +-3 (random_weights(relu_bias=3)), so no ReLU pre-activation sits near 0.
TEST INFRASTRUCTURE: tests/test_step_forward.py pins oracle/lstm_oracle.py and tests/torch_ref.py to this file.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O          # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

RELU_BIAS = 3.0
STEP_CASES = [(kind, H) for H in (32, 160, 224) for kind in ("directional", "social_small")]
ADD_TO_H_CASES = [(kind, 32) for kind in ("occupancy", "social_default", "hiddenstatemlp")]
POOL_KINDS = ["occupancy_n36", "directional_n26", "occupancy_raw"]
PHASES = ("encoder", "decoder")


def pool_spec(kind, H, pool_to_input=True):
    """Constructor arguments of the kind's interaction module at LSTM width H (None: no pooling); without
    pool_to_input the module's output is added to h, so its out_dim is H."""
    table = O.NONGRID_SPECS if kind in O.NONGRID_SPECS else O.MODEL_SPECS
    spec = table[kind]
    if spec is None:
        return None
    spec = dict(spec, hidden_dim=H)
    return spec if pool_to_input else dict(spec, out_dim=H)


def pool_config(kind, H, pool_to_input=True):
    spec = pool_spec(kind, H, pool_to_input)
    if spec is None:
        return None
    return O.MlpPoolConfig(**spec) if kind in O.NONGRID_SPECS else O.PoolConfig(**spec)


def weights(kind, H, seed, pool_to_input=True):
    return O.random_weights(kind, seed=seed, hidden_dim=H, relu_bias=RELU_BIAS, pool_to_input=pool_to_input,
                            out_dim=None if pool_to_input else H)


def step_inputs(H, seed):
    """Ragged scenes, one step: obs1 / obs2 [M, 2] fp32 with rows absent at obs1 only and at obs2 only, the
    batch_split, and random non-zero h [M, H] in +-1 and c in +-3 (absent rows included)."""
    xy, bs = O.synthetic_scenes(4, 5, seed=seed, ragged=True)
    obs1, obs2 = xy[7].copy(), xy[8].copy()
    M = obs2.shape[0]
    obs1[1] = np.nan
    obs2[M - 2] = np.nan
    rng = np.random.RandomState(seed + 1)
    h = rng.uniform(-1.0, 1.0, size=(M, H)).astype(np.float32)
    c = rng.uniform(-3.0, 3.0, size=(M, H)).astype(np.float32)
    return obs1, obs2, bs, h, c


def pool_inputs(kind, seed):
    """[B, N, 2] positions with a padded scene and tracks absent at obs1 / obs2, for a stand-alone grid call."""
    rng = np.random.RandomState(seed)
    B, N = 3, 9
    obs2 = (rng.randn(B, N, 2) * 2.0).astype(np.float32)
    obs1 = obs2 - (rng.randn(B, N, 2) * 0.3).astype(np.float32)
    hid = (rng.randn(B, N, 128) * 0.5).astype(np.float32)
    obs1[1, 5:] = obs2[1, 5:] = hid[1, 5:] = np.nan
    obs1[2, 3] = np.nan
    obs2[0, 6] = np.nan
    return hid, obs1, obs2


def build_reference_model(kind, W, H, pool_to_input=True):
    from trajnetbaselines.lstm import LSTM, GridBasedPooling
    from trajnetbaselines.lstm.non_gridbased_pooling import HiddenStateMLPPooling
    spec = pool_spec(kind, H, pool_to_input)
    pool = None
    if spec is not None:
        pool = HiddenStateMLPPooling(**spec) if kind in O.NONGRID_SPECS else GridBasedPooling(**spec)
    model = LSTM(hidden_dim=H, pool=pool, pool_to_input=pool_to_input)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    return model.eval()


def reference_step(model, phase, obs1, obs2, bs, h, c):
    """LSTM.step of the reference on the per-track lists it keeps: (h', c', normal) as arrays."""
    M = obs2.shape[0]
    if model.pool is not None:
        model.pool.reset(M, int((bs[1:] - bs[:-1]).max()) - 1, device=torch.device("cpu"))
    state = ([torch.from_numpy(r.copy()) for r in h], [torch.from_numpy(r.copy()) for r in c])
    with torch.no_grad():
        (h2, c2), normal = model.step(getattr(model, phase), state, torch.from_numpy(obs1), torch.from_numpy(obs2),
                                      torch.zeros(M, 2), torch.from_numpy(bs))
    return torch.stack(h2).numpy(), torch.stack(c2).numpy(), normal.numpy()


def main():
    torch.set_num_threads(1)
    import_reference()
    from trajnetbaselines.lstm import GridBasedPooling
    out = {}
    for cases, pti in ((STEP_CASES, True), (ADD_TO_H_CASES, False)):
        for kind, H in cases:
            model = build_reference_model(kind, weights(kind, H, seed=H + 3, pool_to_input=pti), H, pti)
            obs1, obs2, bs, h, c = step_inputs(H, seed=H)
            for phase in PHASES:
                key = "step/%s/%d/%s/%s/" % (kind, H, "input" if pti else "add_to_h", phase)
                out[key + "h"], out[key + "c"], out[key + "normal"] = reference_step(model, phase, obs1, obs2, bs, h, c)
    for kind in POOL_KINDS:
        W = O.random_weights(kind, seed=17, relu_bias=RELU_BIAS)
        pool = GridBasedPooling(**O.MODEL_SPECS[kind])
        pool.load_state_dict({k[len("pool."):]: torch.from_numpy(v.copy()) for k, v in W.items()
                              if k.startswith("pool.")}, strict=True)
        hid, obs1, obs2 = pool_inputs(kind, seed=19)
        with torch.no_grad():
            out["pool/%s" % kind] = pool(torch.from_numpy(hid), torch.from_numpy(obs1), torch.from_numpy(obs2)).numpy()
    path = os.path.join(ROOT, "tests", "golden", "step_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
