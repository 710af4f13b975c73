"""The social grid's first Linear (sparse_layer1_mma) at the benchmark's shape: time, weight stream, occupancy.

    python scripts/layer1_bench.py [--scenes 256] [--forwards 5]

Runs the Social-LSTM inference of bench.py (same seeded weights and scenes, an L2 flush between forwards) and times
every sparse_layer1_mma launch with CUDA events (tb2_profile_*).  Beside the time it prints what the launch moves and
does, computed from the shapes:
  * L2 weight bytes per call: every CTA walks every cell's (cell, column chunk) slab of the hi/lo weight image, so
    groups x chunks x cells x slab bytes;
  * the weight stream those bytes make at the measured time;
  * MMA tiles per CTA: 16-row mma.sync tiles of one scene group summed over the cells, from the winners of the
    observed frames 0, 8 and 20 (the model's own predictions replace them later in the forward);
  * CTAs per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor), hence the number of waves.
Prints one JSON line with the GPU's name and power limit.
"""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEDS, OBS, PRED = 20, 9, 12
GROUP_CAP = 160            # rows of a scene group at the benchmark's shape (tb2_layout_create)
SLAB_BYTES_PER_COL = 64    # 16 latent channels x (hi, lo) bf16


def winners_per_cell(xy, bs, cfg):
    """[rows, cells] bool: row i has a winning (in-range) writer in the cell at the frame xy [M, 2]."""
    from oracle import lstm_oracle as O
    B = len(bs) - 1
    obs = xy.reshape(B, PEDS, 2)
    oi, in_range = O.grid_cells(obs, cfg)
    cells = cfg.n * cfg.n
    rows = B * PEDS
    oi, in_range = oi.reshape(rows, PEDS - 1), in_range.reshape(rows, PEDS - 1)
    last = np.full((rows, cells), -1, dtype=np.int64)        # last writer per cell (out of range writes cell 0)
    for jj in range(PEDS - 1):
        last[np.arange(rows), oi[:, jj]] = jj
    win = last >= 0
    r = np.arange(rows)[:, None]
    win &= in_range[r, np.maximum(last, 0)]
    return win


def tiles_per_cta(xy_frames, bs, cfg):
    groups = GROUP_CAP // PEDS
    out = []
    for xy in xy_frames:
        win = winners_per_cell(xy, bs, cfg)
        per_group = win.reshape(-1, groups * PEDS, win.shape[1]).sum(axis=1)      # [groups, cells] pairs
        out.append(float(np.ceil(per_group / 16.0).sum(axis=1).mean()))
    return float(np.mean(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=256)
    ap.add_argument("--forwards", type=int, default=5)
    args = ap.parse_args()
    import torch
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    assert torch.cuda.is_available(), "layer1_bench.py needs a CUDA device"
    lib = _lib.load()
    info = getattr(lib, "_ZN3tb215layer1_mma_infoEiiiPiS0_S0_")      # tb2::layer1_mma_info
    info.restype = ctypes.c_int
    info.argtypes = [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3
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
    prof = json.loads(buf.value.decode())["sparse_layer1_mma"]
    us = 1e3 * prof["total_ms"] / prof["launches"]

    cfg = O.pool_config("social")
    cells, d1, nm1 = cfg.n * cfg.n, O.MODEL_SPECS["social"]["layer_dims"][0], PEDS - 1
    chunk, threads, per_sm = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(info(GROUP_CAP, cells, nm1, ctypes.byref(chunk), ctypes.byref(threads), ctypes.byref(per_sm)))
    groups = math.ceil(args.scenes * PEDS / GROUP_CAP)
    chunks = math.ceil(d1 / chunk.value)
    wbytes = groups * chunks * cells * chunk.value * SLAB_BYTES_PER_COL
    ctas = groups * chunks
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "gpu": gpu, "scenes": args.scenes, "tracks": M,
        "sparse_layer1_mma_us": us, "launches": prof["launches"],
        "grid": {"groups": groups, "chunks": chunks, "chunk_cols": chunk.value, "threads": threads.value, "ctas": ctas},
        "l2_weight_bytes_per_call": wbytes, "weight_stream_tb_s": wbytes / (us * 1e-6) / 1e12,
        "mma_tiles_per_cta": tiles_per_cta([xy[f] for f in (0, 8, 20)], bs, cfg),
        "ctas_per_sm": per_sm.value, "sms": sms, "waves": math.ceil(ctas / (per_sm.value * sms))}))


if __name__ == "__main__":
    main()
