"""In-tree build of libtrajnet_b200.so (hand-written sm_90a CUDA behind a C ABI).

`python -m trajnetplusplusbaselines_b200.build` or `__graft_entry__.build()`.  nvcc
cross-compiles without a GPU; the .so and the object files are build products (git-ignored).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(ROOT, "include")
LIB_NAME = "libtrajnet_b200.so"
LIB_PATH = os.path.join(HERE, LIB_NAME)

NVCC_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
    "-I", INCLUDE, "-I", CSRC,
]


# classical.cu is compared operation-by-operation with the CPU restatement (oracle/), metrics.cu decides collisions at a
# distance threshold like numpy does, kalman.cu runs one EM / smoother code on the host (no FMA on baseline x86-64) and
# on the device with bit-identical results: no FMA contraction
PER_FILE_FLAGS = {"classical.cu": ["-fmad=false"], "metrics.cu": ["-fmad=false"], "kalman.cu": ["-fmad=false"]}


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found (needed to build %s)" % LIB_NAME)
    return exe


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    deps.append(os.path.join(INCLUDE, "trajnet_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        extra = PER_FILE_FLAGS.get(os.path.basename(src), [])
        cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s" % src)
    cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-ldl"]
    subprocess.check_call(cmd)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
