"""Generate tests/golden/hidden_dim_golden.npz from the UNMODIFIED reference (build container).

    python -m oracle.make_hidden_dim_golden

LSTMs at hidden widths other than the default 128 (`--hidden-dim` of the reference trainers), at H = 64 and 256:
  * LSTM.forward, free-running and teacher-forced, for vanilla, directional, social_small and hiddenstatemlp, on
    ragged scenes with entering / leaving tracks;
  * Trainer.train_batch (trainer.py:229-269, plain SGD at lr 0 so the gradients stay in .grad) for directional
    and social (the reference trainer's --type social defaults): the loss and every parameter gradient.
The grid embedding's biases are +-3 (random_weights(relu_bias=3)), so no ReLU pre-activation sits near 0.
TEST INFRASTRUCTURE: tests/test_hidden_dim.py pins oracle/lstm_oracle.py and tests/torch_ref.py to this file.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import lstm_oracle as O          # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402
from oracle.make_train_golden import summarize  # noqa: E402

WIDTHS = [64, 256]
FORWARD_KINDS = ["vanilla", "directional", "social_small", "hiddenstatemlp"]
TRAIN_KINDS = ["directional", "social_default"]
RELU_BIAS = 3.0


def pool_spec(kind, H):
    """Constructor arguments of the kind's interaction module at LSTM width H (None: no pooling)."""
    if kind in O.NONGRID_SPECS:
        return dict(O.NONGRID_SPECS[kind], hidden_dim=H)
    spec = O.MODEL_SPECS[kind]
    return None if spec is None else dict(spec, hidden_dim=H)


def pool_config(kind, H):
    """oracle / restatement configuration of the kind at width H."""
    spec = pool_spec(kind, H)
    if spec is None:
        return None
    return O.MlpPoolConfig(**spec) if kind in O.NONGRID_SPECS else O.PoolConfig(**spec)


def weights(kind, H, seed):
    return O.random_weights(kind, seed=seed, hidden_dim=H, relu_bias=RELU_BIAS)


def forward_inputs(H):
    return O.synthetic_scenes(7, 8, seed=40 + H // 32, ragged=True, nan_tracks=True)


def train_inputs(H):
    return O.synthetic_scenes(5, 7, seed=50 + H // 32, ragged=True, nan_tracks=True)


def build_reference_model(kind, W, H):
    from trajnetbaselines.lstm import LSTM, GridBasedPooling
    from trajnetbaselines.lstm.non_gridbased_pooling import HiddenStateMLPPooling
    spec = pool_spec(kind, H)
    pool = None
    if spec is not None:
        pool = HiddenStateMLPPooling(**spec) if kind in O.NONGRID_SPECS else GridBasedPooling(**spec)
    model = LSTM(hidden_dim=H, pool=pool)
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    return model


def main():
    torch.set_num_threads(1)
    import_reference()
    from trajnetbaselines.lstm import trainer as ref_trainer
    from trajnetbaselines.lstm.loss import PredictionLoss
    out = {}
    for H in WIDTHS:
        xy, bs = forward_inputs(H)
        M = xy.shape[1]
        for kind in FORWARD_KINDS:
            model = build_reference_model(kind, weights(kind, H, seed=H + 1), H).eval()
            with torch.no_grad():
                rel_f, pred_f = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs), n_predict=12)
                rel_t, pred_t = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs),
                                      prediction_truth=torch.from_numpy(xy[9:20]).clone())
            key = "fwd/%s/%d/" % (kind, H)
            out[key + "rel_free"] = rel_f.numpy()
            out[key + "pred_free"] = pred_f.numpy()
            out[key + "rel_teacher"] = rel_t.numpy()
            out[key + "pred_teacher"] = pred_t.numpy()
        xy, bs = train_inputs(H)
        B = len(bs) - 1
        for kind in TRAIN_KINDS:
            model = build_reference_model(kind, weights(kind, H, seed=H + 2), H).train()
            t = ref_trainer.Trainer(model=model, criterion=PredictionLoss(),
                                    optimizer=torch.optim.SGD(model.parameters(), lr=0.0),
                                    device=torch.device("cpu"), batch_size=B, augment=False)
            loss = t.train_batch(torch.from_numpy(xy), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs))
            key = "train/%s/%d/" % (kind, H)
            out[key + "loss"] = np.array([loss], dtype=np.float64)
            for pname, p in model.named_parameters():
                if p.grad is not None:
                    summarize(key + pname, p.grad.numpy(), out)
            print(kind, H, "loss %.6f" % loss)
    path = os.path.join(ROOT, "tests", "golden", "hidden_dim_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
