"""evaluate_file of the multi-modal predictors: the batched decode of every mode of every scene (column pipeline,
multimodal.py) against the per-scene row pipeline (one encoder pass and `modes` decoder passes per scene), on the same
files.  S-GAN and VAE, directional pooling, modes 1 / 3 / 50, on 1024 synthetic scenes (2-20 pedestrians, some entering
during the observation) and on DATA_BLOCK/collision_test/test.  Every (model, file, modes, path) is warmed up, then
timed over --runs calls between CUDA events with a device synchronise on both sides; one JSON line each with the
median, min and max time, scenes/s and modes * scenes/s of the median.

    python scripts/multimodal_bench.py [--scenes 1024] [--runs 3] [--row-runs 1] [--modes 1 3 50]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from oracle import lstm_oracle as O
from oracle import sgan_oracle as SO
from oracle.ref_shim import reference_root
from trajnetplusplusbaselines_b200.data import SceneRow, TrackRow, trajnet_line
from trajnetplusplusbaselines_b200.evaluator import _column_pipeline, evaluate_file
from trajnetplusplusbaselines_b200.lstm import GridBasedPooling
from trajnetplusplusbaselines_b200.sgan import SGAN, LSTMGenerator, SGANPredictor
from trajnetplusplusbaselines_b200.vae import VAE, VAEPredictor

KIND = "directional"


def write_scenes(filename, n_scenes, seed=0):
    rng = np.random.RandomState(seed)
    with open(filename, "w") as f:
        for sid in range(n_scenes):
            n = int(rng.randint(2, 21))
            frames = [1000 * sid + 10 * t for t in range(21)]
            start, vel = rng.randn(n, 2) * 3.0, rng.randn(n, 2) * 0.3
            f.write(trajnet_line(SceneRow(sid, 100 * sid, frames[0], frames[-1], 2.5, 0)) + "\n")
            for p in range(n):
                t0 = 0 if p == 0 or rng.rand() > 0.15 else int(rng.randint(1, 8))
                for t in range(t0, 21):
                    f.write(trajnet_line(TrackRow(frames[t], 100 * sid + p, float(start[p, 0] + vel[p, 0] * t),
                                                  float(start[p, 1] + vel[p, 1] * t))) + "\n")


def load(module, W):
    sd = module.state_dict()
    sd.update({k: torch.from_numpy(v.copy()) for k, v in W.items() if k in sd})
    module.load_state_dict(sd)


def predictors():
    gen = LSTMGenerator(pool=GridBasedPooling(**O.MODEL_SPECS[KIND]))
    load(gen, SO.sgan_weights(KIND, 2)[0])
    vae = VAE(pool=GridBasedPooling(**O.MODEL_SPECS[KIND]))
    load(vae, SO.vae_weights(KIND, 2))
    return {"sgan": SGANPredictor(SGAN(generator=gen, k=1, d_steps=0).cuda().eval()),
            "vae": VAEPredictor(vae.cuda().eval())}


class RowPipeline:
    """The predictor behind the reference's call signature only: evaluate_file calls it scene by scene."""

    def __init__(self, predictor):
        self.predictor = predictor

    def __call__(self, *args, **kwargs):
        return self.predictor(*args, **kwargs)


def timed(fn, runs):
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) * 1e-3)
    return times


def device_info():
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                               text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        limit = "unknown"
    return torch.cuda.get_device_name(0), limit


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--scenes", type=int, default=1024)
    parser.add_argument("--runs", type=int, default=3, help="timed calls of the batched path")
    parser.add_argument("--row-runs", type=int, default=1, help="timed calls of the per-scene row path")
    parser.add_argument("--modes", type=int, nargs="+", default=[1, 3, 50])
    args = parser.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.manual_seed(0)
    np.random.seed(0)
    gpu, power = device_info()
    plain = types.SimpleNamespace(normalize_scene=False)
    tmp = tempfile.mkdtemp(prefix="multimodal_bench_")
    files = {}
    files["synthetic_%d" % args.scenes] = os.path.join(tmp, "synthetic.ndjson")
    write_scenes(files["synthetic_%d" % args.scenes], args.scenes)
    root = reference_root()
    if root is not None:
        files["collision_test"] = os.path.join(root, "DATA_BLOCK", "collision_test", "test", "collision_test.ndjson")
    warm = os.path.join(tmp, "warm.ndjson")
    write_scenes(warm, 16, seed=1)
    out = os.path.join(tmp, "out.ndjson")
    for name, predictor in predictors().items():
        for fname, infile in files.items():
            n_scenes = sum(1 for line in open(infile) if line.startswith('{"scene"'))
            for modes in args.modes:
                for path, p, runs in (("batched", predictor, args.runs), ("row", RowPipeline(predictor), args.row_runs)):
                    assert _column_pipeline(p, modes) == (path == "batched")
                    run = lambda f=infile: evaluate_file(p, f, out, modes=modes, args=plain)
                    evaluate_file(p, warm if path == "row" else infile, out, modes=modes, args=plain)     # warm-up
                    times = timed(run, runs)
                    med = statistics.median(times)
                    print(json.dumps({"model": name, "pool": KIND, "file": fname, "scenes": n_scenes, "modes": modes,
                                      "path": path, "runs": runs, "s_median": round(med, 4),
                                      "s_min": round(min(times), 4), "s_max": round(max(times), 4),
                                      "scenes_per_s": round(n_scenes / med, 1),
                                      "mode_scenes_per_s": round(modes * n_scenes / med, 1),
                                      "gpu": gpu, "power_limit": power}), flush=True)
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)


if __name__ == "__main__":
    main()
