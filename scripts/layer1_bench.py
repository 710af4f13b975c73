"""The social grid's first Linear (sparse_layer1_mma) at the benchmark's shape: time, weight stream, occupancy.

    python scripts/layer1_bench.py [--scenes 256] [--forwards 5] [--lib OTHER.so] [--time-only]

--lib times another build of the library (same C ABI) instead of the package's; --time-only skips the wavefront models.

Runs the Social-LSTM inference of bench.py (same seeded weights and scenes, an L2 flush between forwards) and times
every sparse_layer1_mma launch with CUDA events (tb2_profile_*).  Beside the time it prints what the launch moves and
does, computed from the shapes:
  * L2 weight bytes per call: every CTA reads the (cell, column chunk) slab of the hi/lo weight image once per
    16-row tile of its tile list (a cell without pairs is skipped, a cell of several tiles is read once per tile),
    so groups x chunks x tiles per CTA x slab bytes;
  * the weight stream those bytes make at the measured time;
  * MMA tiles per CTA: 16-row mma.sync tiles of one scene group summed over the cells, from the winners of the
    observed frames 0, 8 and 20 (the model's own predictions replace them later in the forward), and the real and
    padded row slots of those tiles;
  * a model (not a measurement) of the shared-memory wavefronts of one CTA's tile loop, from the same winners.  A warp
    access costs, per group of lanes the hardware serves together, the larger of the distinct 4-byte words over 32 and
    the most distinct words in one bank; times the warps of a CTA (16, or 8 for the 32-column layouts).  "before_tile_list" and "tile_list" take all 32 lanes as one
    group (the tile layout before the flat tile list: padding rows load the zero latent row and read-modify-write
    dummy accumulator rows, 32-bit A loads from separate hi / lo rows; and the flat tile list: padding rows touch no
    accumulator, one 128-bit (hi, lo) A load per row, two 32-bit slot words, two 64-bit loads and stores per
    accumulator row at a 264-float stride).  "phased" serves a 64-bit access a half-warp (tile rows 4h .. 4h + 3) and
    a 128-bit access a quarter-warp (rows 2q, 2q + 1) at a time, which is where two accumulator rows of a tile collide:
    "tile_list_64bit_stride264" is the flat tile list again, "packed_128bit_stride<S>" the current layout (one slot
    word, one 128-bit load and store per accumulator row, the warp's 16 columns of a row contiguous) at row strides of
    264, 272 and 280 floats, "warp32_128bit_stride<S>" the kernel's layout (8 warps of 32 columns: a tile's slot word
    and A rows loaded once per warp, two adjacent 128-bit words per accumulator row and lane) at strides of 256 to 280
    floats (the kernel's is 260);
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


def winners_per_cell(xy, bs, cfg, with_writer=False):
    """[rows, cells] bool: row i has a winning (in-range) writer in the cell at the frame xy [M, 2].  with_writer:
    also the winner's scene-local pedestrian index [rows, cells]."""
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
    if with_writer:
        i = np.arange(rows)[:, None] % PEDS
        return win, last + (last >= i)                         # neighbour slot jj -> pedestrian j (diagonal removed)
    return win


def tiles_per_cta(xy_frames, bs, cfg):
    groups = GROUP_CAP // PEDS
    out = []
    for xy in xy_frames:
        win = winners_per_cell(xy, bs, cfg)
        per_group = win.reshape(-1, groups * PEDS, win.shape[1]).sum(axis=1)      # [groups, cells] pairs
        out.append(float(np.ceil(per_group / 16.0).sum(axis=1).mean()))
    return float(np.mean(out))


def tile_slots_per_cta(xy_frames, bs, cfg):
    """(real, padded) row slots of one CTA's 16-row tiles, averaged over the groups and frames."""
    groups = GROUP_CAP // PEDS
    real, padded = [], []
    for xy in xy_frames:
        per_group = winners_per_cell(xy, bs, cfg).reshape(-1, groups * PEDS, cfg.n * cfg.n).sum(axis=1)
        real.append(per_group.sum(axis=1).mean())
        padded.append((16 * np.ceil(per_group / 16.0)).sum(axis=1).mean())
    return float(np.mean(real)), float(np.mean(padded))


def _wavefronts(words):
    """Modelled wavefronts of one warp access touching the 4-byte shared-memory words `words`."""
    if not words:
        return 0
    words = set(words)
    return max(-(-len(words) // 32), int(np.bincount([w % 32 for w in words], minlength=32).max()))


def wavefronts_per_cta(xy_frames, bs, cfg):
    """(before, after) modelled shared-memory wavefronts of one CTA's tile loop (see the module docstring)."""
    stride, cap, cells = 264, GROUP_CAP, cfg.n * cfg.n
    rows_per_group = GROUP_CAP // PEDS * PEDS
    tot = np.zeros(2)
    n = 0
    for xy in xy_frames:
        win, writer = winners_per_cell(xy, bs, cfg, with_writer=True)
        lat_row = writer + (np.arange(len(win)) // PEDS * PEDS % rows_per_group)[:, None]    # group-local row of j
        for grp in range(len(win) // rows_per_group):
            sl = slice(grp * rows_per_group, (grp + 1) * rows_per_group)
            w, lr = win[sl], lat_row[sl]
            for cell in range(cells):
                rows = np.nonzero(w[:, cell])[0]
                for e0 in range(0, len(rows), 16):
                    slot = [(int(r), int(lr[r, cell])) for r in rows[e0:e0 + 16]]
                    slot += [None] * (16 - len(slot))
                    ent = 2                                      # two 32-bit slot-word loads, 8 words each
                    old_a = new_a = old_acc = new_acc = 0
                    for half in (0, 1):
                        s8 = slot[8 * half:8 * half + 8]
                        lat_old = [cap + 1 if e is None else e[1] for e in s8]
                        for base in (0, (cap + 2) * 8):         # lat_hi, lat_lo: words 2t, 2t + 1 of 8-word rows
                            for c in (0, 1):
                                old_a += _wavefronts([base + 8 * l + 2 * t + c for l in lat_old for t in range(4)])
                        # (hi, lo) of a row and lane t in 16 bytes: 16-word rows, one 128-bit load per row
                        new_a += _wavefronts([16 * l + 4 * t + c for l in lat_old for t in range(4) for c in range(4)])
                        for j in (0, 1):
                            acc_old = [cap + 8 * half + g if e is None else e[0] for g, e in enumerate(s8)]
                            acc_new = [e[0] for e in s8 if e is not None]
                            old_acc += 2 * _wavefronts([r * stride + 8 * j + 2 * t + c for r in acc_old
                                                        for t in range(4) for c in (0, 1)])
                            new_acc += 2 * _wavefronts([r * stride + 8 * j + 2 * t + c for r in acc_new
                                                        for t in range(4) for c in (0, 1)])
                    tot += (ent + old_a + old_acc, ent + new_a + new_acc)
            n += 1
    return tuple(float(v) * 16 / n for v in tot)


ACC_STRIDES = (264, 272, 280)
ACC_STRIDES_32 = (256, 260, 264, 268, 272, 276, 280)


def phased_wavefronts_per_cta(xy_frames, bs, cfg):
    """Modelled shared-memory wavefronts of one CTA's tile loop with 64-bit accesses served per half-warp and 128-bit
    accesses per quarter-warp (see the module docstring): {layout: wavefronts}."""
    cap, cells = GROUP_CAP, cfg.n * cfg.n
    rows_per_group = GROUP_CAP // PEDS * PEDS
    names = (["tile_list_64bit_stride264"] + ["packed_128bit_stride%d" % s for s in ACC_STRIDES] +
             ["warp32_128bit_stride%d" % s for s in ACC_STRIDES_32])
    n16 = 1 + len(ACC_STRIDES)
    warps = np.array([16] * n16 + [8] * len(ACC_STRIDES_32))      # warps of a CTA walking the whole tile list
    slot_words = np.array([2] + [1] * (len(names) - 1))
    tot = np.zeros(len(names))
    n = 0
    for xy in xy_frames:
        win, writer = winners_per_cell(xy, bs, cfg, with_writer=True)
        lat_row = writer + (np.arange(len(win)) // PEDS * PEDS % rows_per_group)[:, None]
        for grp in range(len(win) // rows_per_group):
            sl = slice(grp * rows_per_group, (grp + 1) * rows_per_group)
            w, lr = win[sl], lat_row[sl]
            for cell in range(cells):
                rows = np.nonzero(w[:, cell])[0]
                for e0 in range(0, len(rows), 16):
                    slot = [(int(r), int(lr[r, cell])) for r in rows[e0:e0 + 16]]
                    slot += [None] * (16 - len(slot))
                    a = 0
                    acc = np.zeros(len(names))
                    for half in (0, 1):
                        s8 = slot[8 * half:8 * half + 8]
                        lat = [cap + 1 if e is None else e[1] for e in s8]
                        for q in range(4):                      # 128-bit A loads: two rows per quarter-warp
                            a += _wavefronts([16 * l + 4 * t + c for l in lat[2 * q:2 * q + 2]
                                              for t in range(4) for c in range(4)])
                        for h in (0, 1):                        # 64-bit: rows 4h .. 4h + 3, both n-tiles, load + store
                            r4 = [e[0] for e in s8[4 * h:4 * h + 4] if e is not None]
                            acc[0] += 2 * 2 * _wavefronts([r * 264 + 2 * t + c for r in r4
                                                           for t in range(4) for c in (0, 1)])
                        for q in range(4):                      # 128-bit: rows 2q, 2q + 1, load + store
                            r2 = [e[0] for e in s8[2 * q:2 * q + 2] if e is not None]
                            for i, stride in enumerate(ACC_STRIDES):
                                acc[1 + i] += 2 * _wavefronts([r * stride + 4 * t + c for r in r2
                                                               for t in range(4) for c in range(4)])
                            for i, stride in enumerate(ACC_STRIDES_32):     # 32 columns: words 8t and 8t + 4
                                for h in (0, 1):
                                    acc[n16 + i] += 2 * _wavefronts([r * stride + 8 * t + 4 * h + c for r in r2
                                                                     for t in range(4) for c in range(4)])
                    tot += warps * (a + acc + slot_words)
            n += 1
    return {k: float(v) / n for k, v in zip(names, tot)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=256)
    ap.add_argument("--forwards", type=int, default=5)
    ap.add_argument("--lib", help="time this build of the library instead of the package's")
    ap.add_argument("--time-only", action="store_true", help="skip the shared-memory wavefront models")
    args = ap.parse_args()
    import torch
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    assert torch.cuda.is_available(), "layer1_bench.py needs a CUDA device"
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
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
    frames = [xy[f] for f in (0, 8, 20)]
    tiles = tiles_per_cta(frames, bs, cfg)
    wbytes = groups * chunks * tiles * chunk.value * SLAB_BYTES_PER_COL
    ctas = groups * chunks
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    slots = tile_slots_per_cta(frames, bs, cfg)
    wf = (None, None) if args.time_only else wavefronts_per_cta(frames, bs, cfg)
    phased = None if args.time_only else phased_wavefronts_per_cta(frames, bs, cfg)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "gpu": gpu, "lib": _lib.LIB_PATH, "scenes": args.scenes, "tracks": M,
        "sparse_layer1_mma_us": us, "launches": prof["launches"],
        "grid": {"groups": groups, "chunks": chunks, "chunk_cols": chunk.value, "threads": threads.value, "ctas": ctas},
        "l2_weight_bytes_per_call": wbytes, "weight_stream_tb_s": wbytes / (us * 1e-6) / 1e12,
        "mma_tiles_per_cta": tiles,
        "tile_slots_per_cta": {"real": slots[0], "padded": slots[1]},
        "smem_wavefronts_per_cta_model": {"before_tile_list": wf[0], "tile_list": wf[1], "phased": phased},
        "ctas_per_sm": per_sm.value, "sms": sms, "waves": math.ceil(ctas / (per_sm.value * sms))}))


if __name__ == "__main__":
    main()
