"""What bounds the step's two wgmma kernels, dense_layer_tc (grid layer 2) and lstm_gates_tc: each timed with one part
of its mainloop taken out.

    python scripts/step_gemm_ablate.py [--dir DIR] [--rounds 3] [--build-only]
    python scripts/step_gemm_ablate.py --time [--lib OTHER.so] [--scenes 256] [--forwards 5]

Compiles csrc/gemm_tc.cu and csrc/gates_tc.cu again with -DTB2_GEMM_ABLATE=<n> and links them with the package's
other objects into DIR/libgemm_ablate<n>.so (DIR defaults to a temporary directory; a library already there is kept),
then times each with `--time --lib`, alternating with the package's own library, `--rounds` times each.  The ablated
kernels compute wrong results; only their times mean anything (csrc/wgmma.cuh lists the variants).

--time runs the Social-LSTM inference of bench.py (same seeded weights and scenes, 256 scenes x 20 pedestrians:
dense_layer_tc at M = 5120, K = 1024, N = 256; lstm_gates_tc at M = 5120, K = 448, N = 512, H = 128) with an L2 flush
between forwards, and times every launch of both kernels with CUDA events (tb2_profile_*).  Beside the times it
prints the FLOPs and operand bytes of one CTA computed from the shapes.  Prints one JSON line per run with the GPU's
name and power limit, and a summary line with the range of each variant.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {1: "no wgmma", 2: "one stage, no operand stream", 3: "no epilogue stores", 4: "one wgmma group in flight"}
KERNELS = ("dense_layer_tc", "lstm_gates_tc")
SOURCES = ("gemm_tc.cu", "gates_tc.cu")
PEDS, OBS, PRED = 20, 9, 12


def build_variant(n, out_dir):
    from trajnetplusplusbaselines_b200 import build as b
    lib = os.path.join(out_dir, "libgemm_ablate%d.so" % n)
    if os.path.exists(lib):
        return lib
    b.build()                                   # the other objects
    objdir = os.path.join(b.HERE, "build")
    objs = []
    for src in SOURCES:
        obj = os.path.join(out_dir, "%s_ablate%d.o" % (src[:-3], n))
        subprocess.check_call([b._nvcc()] + b.NVCC_FLAGS + ["-DTB2_GEMM_ABLATE=%d" % n, "-c",
                                                            os.path.join(b.CSRC, src), "-o", obj])
        objs.append(obj)
    others = [os.path.join(objdir, os.path.basename(s)[:-3] + ".o") for s in b.sources()
              if os.path.basename(s) not in SOURCES]
    subprocess.check_call([b._nvcc(), "-shared", "-o", lib] + objs + others +
                          ["-gencode", "arch=compute_90a,code=sm_90a", "-ldl"])
    return lib


def cta_work(M=5120):
    """FLOPs and operand bytes of one CTA of each kernel at the benchmark's shape (3 bf16 passes, hi / lo operands)."""
    dense = {"ctas": (M // 128) * (256 // 128), "flop": 3 * 2 * 128 * 128 * 1024,
             "operand_bytes": 2 * 2 * (128 + 128) * 1024}
    gates = {"ctas": (M // 128) * 2, "flop": 3 * 2 * 128 * 256 * 448, "operand_bytes": 2 * 2 * (128 + 256) * 448}
    return {"dense_layer_tc": dense, "lstm_gates_tc": gates}


def time_lib(args):
    import torch
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    assert torch.cuda.is_available(), "step_gemm_ablate.py --time needs a CUDA device"
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    W = O.random_weights("social", seed=1)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS["social"]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.to(dev).eval()
    xy, bs = O.synthetic_scenes(args.scenes, PEDS, n_frames=OBS + PRED, seed=0)      # bench.py's inputs
    M = xy.shape[1]
    obs = torch.from_numpy(xy[:OBS]).to(dev)
    goals, split = torch.zeros(M, 2), torch.from_numpy(bs)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    with torch.no_grad():
        for _ in range(3):
            model(obs, goals, split, n_predict=PRED)
        torch.cuda.synchronize(dev)
        lib.tb2_profile_begin()
        for _ in range(args.forwards):
            flush.zero_()
            model(obs, goals, split, n_predict=PRED)
        buf = ctypes.create_string_buffer(1 << 16)
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
    prof = json.loads(buf.value.decode())
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu, "lib": _lib.LIB_PATH, "tracks": M}
    work = cta_work(M)
    for k in KERNELS:
        us = 1e3 * prof[k]["total_ms"] / prof[k]["launches"]
        out[k + "_us"] = us
        out[k] = dict(work[k], launches=prof[k]["launches"],
                      cta_tflop_s=work[k]["flop"] / (us * 1e-6) / 1e12,
                      operand_stream_tb_s=work[k]["ctas"] * work[k]["operand_bytes"] / (us * 1e-6) / 1e12)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--time", action="store_true", help="time one library (a child run of the ablation)")
    ap.add_argument("--lib", help="with --time: this build of the library instead of the package's")
    ap.add_argument("--scenes", type=int, default=256)
    ap.add_argument("--forwards", type=int, default=5)
    args = ap.parse_args()
    if args.time:
        return time_lib(args)
    out_dir = args.dir or tempfile.mkdtemp(prefix="step_gemm_ablate_")
    os.makedirs(out_dir, exist_ok=True)
    libs = {0: None}
    for n in VARIANTS:
        libs[n] = build_variant(n, out_dir)
    if args.build_only:
        return
    times = {n: {k: [] for k in KERNELS} for n in libs}
    gpu = None
    for _ in range(args.rounds):
        for n, lib in libs.items():
            cmd = [sys.executable, os.path.abspath(__file__), "--time", "--scenes", str(args.scenes),
                   "--forwards", str(args.forwards)]
            out = subprocess.run(cmd + (["--lib", lib] if lib else []), capture_output=True, text=True, check=True)
            res = json.loads(out.stdout.strip().splitlines()[-1])
            gpu = res["gpu"]
            for k in KERNELS:
                times[n][k].append(res[k + "_us"])
            print(json.dumps({"ablate": n, "what": VARIANTS.get(n, "the library as built"),
                              **{k + "_us": res[k + "_us"] for k in KERNELS}, "gpu": gpu}), flush=True)
    print(json.dumps({"gpu": gpu, "us_min_max": {
        VARIANTS.get(n, "the library as built"): {k: [min(t[k]), max(t[k])] for k in KERNELS}
        for n, t in times.items()}}))


if __name__ == "__main__":
    main()
