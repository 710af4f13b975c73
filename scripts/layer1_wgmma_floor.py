"""Lower bound for a wgmma formulation of the social grid's first Linear, against the kernel that runs it.

    python scripts/layer1_wgmma_floor.py [--scenes 256] [--iters 50]

A wgmma version of sparse_layer1 puts the tracks on the 64-row side and accumulates one K = 16 product per grid cell
over all 256 cells.  That is the dense product [M, 4096] x [4096, 1024] on the tensor cores, 3 bf16 passes (hi/lo
split, as every tensor kernel of the library), plus building the zero-padded per-cell A tiles.  The first part alone
is exactly what dense_layer_tc_kernel (wgmma + TMA) computes at that shape, so its time is a floor for that design.
This script times it with CUDA events at the BASELINE track count and, in the same process, the per-step time of the
layer's current kernel (sparse_layer1_mma, warp-level mma.sync over the occupied cells only) inside a Social-LSTM
forward.  Prints one JSON line with the GPU's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    lib = _lib.load()
    dense = getattr(lib, "_ZN3tb215launch_dense_tcEPKvS1_S1_S1_PKfPfPvS5_iiiiP11CUstream_st")   # tb2::launch_dense_tc
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    dense.restype = i32
    dense.argtypes = [vp] * 8 + [i32] * 4 + [vp]
    dev = torch.device("cuda", 0)
    M, K, N = args.scenes * 20, 4096, 1024
    g = torch.Generator(device=dev).manual_seed(0)
    a = torch.randn(M, K, device=dev, generator=g) * (torch.rand(M, K, device=dev, generator=g) < 0.08)
    w = torch.randn(N, K, device=dev, generator=g) * 0.02
    a_hi = a.bfloat16(); a_lo = (a - a_hi.float()).bfloat16()
    w_hi = w.bfloat16(); w_lo = (w - w_hi.float()).bfloat16()
    bias = torch.zeros(N, device=dev)
    y = torch.empty(M, N, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def launch():
        _lib.check(dense(a_hi.data_ptr(), a_lo.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(), bias.data_ptr(),
                         y.data_ptr(), None, None, M, K, N, 1, st))

    for _ in range(5):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        launch()
    e1.record()
    torch.cuda.synchronize(dev)
    dense_us = 1e3 * e0.elapsed_time(e1) / args.iters
    ref = torch.relu(a_hi.float() @ w_hi.float().T + a_hi.float() @ w_lo.float().T + a_lo.float() @ w_hi.float().T)
    err = float((y - ref).abs().max())

    W = O.random_weights("social", seed=1)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS["social"]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.to(dev).eval()
    xy, bs = O.synthetic_scenes(args.scenes, 20, n_frames=21, seed=1000)
    obs = torch.from_numpy(xy[:9]).to(dev)
    goals, split = torch.zeros(M, 2), torch.from_numpy(bs)
    with torch.no_grad():
        for _ in range(3):
            model(obs, goals, split, n_predict=12)
        lib.tb2_profile_begin()
        for _ in range(3):
            model(obs, goals, split, n_predict=12)
        buf = ctypes.create_string_buffer(1 << 16)
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
    prof = json.loads(buf.value.decode())["sparse_layer1_mma"]
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    flop = 3 * 2.0 * M * K * N
    print(json.dumps({"gpu": gpu, "tracks": M,
                      "wgmma_dense_floor_us": dense_us, "wgmma_dense_tflops": flop / (dense_us * 1e-6) / 1e12,
                      "wgmma_dense_max_abs_err_vs_fp32_of_split": err,
                      "sparse_layer1_mma_us": 1e3 * prof["total_ms"] / prof["launches"]}))


if __name__ == "__main__":
    main()
