"""What bounds sparse_layer1_mma: the kernel timed with one of its parts taken out.

    python scripts/layer1_ablate.py [--dir DIR] [--rounds 3] [--build-only]

Compiles csrc/pool.cu again with -DTB2_L1_ABLATE=<n> and links it with the package's other objects into
DIR/libablate<n>.so (DIR defaults to a temporary directory; a library already there is kept), then times each with
scripts/layer1_bench.py --lib, alternating with the package's own library, `--rounds` times each.  The ablated
kernels compute wrong results; only their times mean anything:
  1  accumulators summed in registers: no shared-memory accumulator loads or stores
  2  every tile reads cell 0's weights: the same requests, always L2 hits on one slab per column chunk
  3  no mma.sync: the products replaced by a few integer operations on the same fragments
  4  every tile reads cell 0's weights from a copy each warp makes in shared memory before the loop: no L2 weight
     traffic at all (2 keeps the same L2 requests in flight)
Prints one JSON line per run and a summary line with the range of each variant.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = {1: "no accumulator traffic", 2: "weights from cell 0", 3: "no mma", 4: "weights from shared memory"}


def build_variant(n, out_dir):
    from trajnetplusplusbaselines_b200 import build as b
    lib = os.path.join(out_dir, "libablate%d.so" % n)
    if os.path.exists(lib):
        return lib
    b.build()                                   # the other objects
    objdir = os.path.join(b.HERE, "build")
    obj = os.path.join(out_dir, "pool_ablate%d.o" % n)
    subprocess.check_call([b._nvcc()] + b.NVCC_FLAGS + ["-DTB2_L1_ABLATE=%d" % n, "-c", os.path.join(b.CSRC, "pool.cu"),
                           "-o", obj])
    others = [os.path.join(objdir, os.path.basename(s)[:-3] + ".o") for s in b.sources()
              if os.path.basename(s) != "pool.cu"]
    subprocess.check_call([b._nvcc(), "-shared", "-o", lib, obj] + others +
                          ["-gencode", "arch=compute_90a,code=sm_90a", "-ldl"])
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--build-only", action="store_true")
    args = ap.parse_args()
    out_dir = args.dir or tempfile.mkdtemp(prefix="layer1_ablate_")
    os.makedirs(out_dir, exist_ok=True)
    libs = {0: None}
    for n in VARIANTS:
        libs[n] = build_variant(n, out_dir)
    if args.build_only:
        return
    times = {n: [] for n in libs}
    gpu = None
    for _ in range(args.rounds):
        for n, lib in libs.items():
            cmd = [sys.executable, os.path.join(ROOT, "scripts", "layer1_bench.py"), "--time-only"]
            out = subprocess.run(cmd + (["--lib", lib] if lib else []), capture_output=True, text=True, check=True)
            res = json.loads(out.stdout.strip().splitlines()[-1])
            gpu = res["gpu"]
            times[n].append(res["sparse_layer1_mma_us"])
            print(json.dumps({"ablate": n, "what": VARIANTS.get(n, "the library as built"),
                              "sparse_layer1_mma_us": res["sparse_layer1_mma_us"], "gpu": gpu}), flush=True)
    print(json.dumps({"gpu": gpu, "sparse_layer1_mma_us_min_max": {
        VARIANTS.get(n, "the library as built"): [min(t), max(t)] for n, t in times.items()}}))


if __name__ == "__main__":
    main()
