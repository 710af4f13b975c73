"""evaluate_file with sampled LSTM modes (the evaluator's --sample, lstm/sampling.py): the batched decode of every mode
of every scene (column pipeline) against the per-scene path (one sampled forward per mode and scene), directional
pooling, modes 3 and 50, on 1024 synthetic scenes of 2-20 pedestrians (some entering during the observation).  Every
(modes, path) is warmed up, then timed over --runs calls between CUDA events with a device synchronise on both sides; one
JSON line each with the median, min and max time and scenes/s of the median.

Then the kernels of one sampled batched decode of the file's first --chunk scenes, by tb2_profile_*: launches and time
per launch of sample_positions next to the other kernels of the step.

    python scripts/sampling_bench.py [--scenes 1024] [--runs 3] [--row-runs 1] [--modes 3 50]
"""
import argparse
import ctypes
import json
import os
import statistics
import sys
import tempfile
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

from multimodal_bench import KIND, RowPipeline, device_info, timed, write_scenes
from oracle import lstm_oracle as O
from trajnetplusplusbaselines_b200 import _lib
from trajnetplusplusbaselines_b200.data import load_test_scenes_xy
from trajnetplusplusbaselines_b200.evaluator import _column_pipeline, evaluate_file
from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, SampledLSTMPredictor


def predictor():
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[KIND]))
    sd = model.state_dict()
    sd.update({k: torch.from_numpy(v.copy()) for k, v in O.random_weights(KIND, seed=2).items() if k in sd})
    model.load_state_dict(sd)
    return SampledLSTMPredictor(model.cuda().eval())


def kernel_profile(p, infile, modes, chunk, plain):
    """{kernel: {launches, total_ms, us_per_launch}} of one batched sampled decode of the first `chunk` scenes."""
    lib = _lib.load()
    xys = [xy for xy, _ in load_test_scenes_xy(infile)[:chunk]]
    p.predict_batch_xy(xys, modes=modes, args=plain)
    torch.cuda.synchronize()
    buf = ctypes.create_string_buffer(1 << 16)
    lib.tb2_profile_begin()
    p.predict_batch_xy(xys, modes=modes, args=plain)
    _lib.check(lib.tb2_profile_end(buf, len(buf)))
    prof = json.loads(buf.value.decode())
    for v in prof.values():
        v["us_per_launch"] = round(1e3 * v["total_ms"] / v["launches"], 2)
        v["total_ms"] = round(v["total_ms"], 3)
    return prof


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--scenes", type=int, default=1024)
    parser.add_argument("--runs", type=int, default=3, help="timed calls of the batched path")
    parser.add_argument("--row-runs", type=int, default=1, help="timed calls of the per-scene path")
    parser.add_argument("--modes", type=int, nargs="+", default=[3, 50])
    parser.add_argument("--chunk", type=int, default=1024, help="scenes of the profiled decode")
    args = parser.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.manual_seed(0)
    gpu, power = device_info()
    plain = types.SimpleNamespace(normalize_scene=False)
    tmp = tempfile.mkdtemp(prefix="sampling_bench_")
    infile = os.path.join(tmp, "synthetic.ndjson")
    write_scenes(infile, args.scenes)
    warm = os.path.join(tmp, "warm.ndjson")
    write_scenes(warm, 16, seed=1)
    out = os.path.join(tmp, "out.ndjson")
    p = predictor()
    for modes in args.modes:
        for path, q, runs in (("batched", p, args.runs), ("per_scene", RowPipeline(p), args.row_runs)):
            assert _column_pipeline(q, modes) == (path == "batched")
            run = lambda: evaluate_file(q, infile, out, modes=modes, args=plain)
            evaluate_file(q, warm if path == "per_scene" else infile, out, modes=modes, args=plain)     # warm-up
            times = timed(run, runs)
            med = statistics.median(times)
            print(json.dumps({"model": "lstm_sample", "pool": KIND, "scenes": args.scenes, "modes": modes, "path": path,
                              "runs": runs, "s_median": round(med, 4), "s_min": round(min(times), 4),
                              "s_max": round(max(times), 4), "scenes_per_s": round(args.scenes / med, 1),
                              "gpu": gpu, "power_limit": power}), flush=True)
        print(json.dumps({"model": "lstm_sample", "pool": KIND, "modes": modes, "profile_scenes": args.chunk,
                          "kernels": kernel_profile(p, infile, modes, args.chunk, plain), "gpu": gpu,
                          "power_limit": power}), flush=True)
    for f in os.listdir(tmp):
        os.remove(os.path.join(tmp, f))
    os.rmdir(tmp)


if __name__ == "__main__":
    main()
