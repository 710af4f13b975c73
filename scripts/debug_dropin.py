"""Per-parameter gradient comparison: CUDA backward vs the unmodified reference (oracle/_ref) autograd."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from oracle import lstm_oracle as O
from oracle.ref_shim import import_reference
import_reference()
from oracle.make_golden import build_reference_model
from trajnetbaselines.lstm.loss import PredictionLoss as RefLoss
from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
torch.set_num_threads(8)

def grads(kind, B, N, seed, ragged, nan_tracks, wseed=11):
    W = O.random_weights(kind, seed=wseed)
    ref = build_reference_model(kind, W); ref.train()
    mine = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind])); mine.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}); mine = mine.cuda().train()
    xy, bs = O.synthetic_scenes(B, N, seed=seed, ragged=ragged, nan_tracks=nan_tracks)
    scene = torch.from_numpy(xy); split = torch.from_numpy(bs); M = xy.shape[1]
    out = {}
    for name, model, crit, dev in (("ref", ref, RefLoss(), "cpu"), ("b200", mine, PredictionLoss(), "cuda")):
        s = scene.to(dev)
        rel, _ = model(s[:9], torch.zeros(M, 2).to(dev), split.to(dev), s[9:-1].clone())
        loss = crit(rel[-12:], s[9:21] - s[8:20], split.to(dev)) * (len(bs) - 1)
        model.zero_grad(); loss.backward()
        out[name] = (float(loss), {k: (p.grad.detach().cpu().numpy() if p.grad is not None else None) for k, p in model.named_parameters()})
    print("%s B=%d N=%d seed=%d ragged=%d nan=%d  loss ref %.6f b200 %.6f" % (kind, B, N, seed, ragged, nan_tracks, out["ref"][0], out["b200"][0]))
    for k, g in out["ref"][1].items():
        gb = out["b200"][1][k]
        if g is None or gb is None:
            continue
        rel = np.abs(gb - g).max() / max(np.abs(g).max(), 1e-12)
        if rel > 1e-4:
            print("    %-40s rel err %.3e  (max |g| %.3e)" % (k, rel, np.abs(g).max()))

print("env TB2_DISABLE_TC=%s" % os.environ.get("TB2_DISABLE_TC"))
grads("social", 10, 7, 17, False, False)
grads("social", 5, 7, 17, False, False)
grads("social", 10, 7, 18, False, False)
grads("social", 12, 9, 5, False, False)
