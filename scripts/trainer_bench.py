"""Seconds per training epoch of the native trainer loop (lstm/trainer.py) against the reference's `Trainer.train` loop
driving the same GPU model.

Data: the seven DATA_BLOCK/trajdata/train files of the reference (through oracle/ref_shim.py: the reference tree or the
oracle/_ref copy build() makes).  Cells: directional (D-LSTM) and social (one_layer) models as the CLI builds them by
default, batch size 8 (the CLI default) and 64, `--augment --normalize_scene`, PredictionLoss, Adam.  Per cell and loop:
one warm-up epoch, then `--epochs` timed epochs (host clock around a whole `train` call, which ends in a device
synchronise on both sides), reported as the list and its median, and scenes/s of the median.  Then one extra native
epoch under tb2_profile_* gives the CUDA-event time of its one tb2_scenes_gather_epoch launch (a separate epoch: the
profiler's events are not part of the timed ones).

Prints one JSON line per cell, then one with the GPU's name, power limit and SM clocks (read in the same call).

    python scripts/trainer_bench.py [--epochs 3] [--cells directional:8,directional:64,social:8,social:64]
"""
import argparse
import ctypes
import json
import logging
import os
import random
import subprocess
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from trajnetplusplusbaselines_b200 import _lib
from trajnetplusplusbaselines_b200.data import read_ndjson_scenes
from trajnetplusplusbaselines_b200.lstm import PredictionLoss
from trajnetplusplusbaselines_b200.lstm import trainer as TR


def emit(**kw):
    print(json.dumps(kw), flush=True)


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return torch.cuda.get_device_name(0), q


def make_trainer(kind, batch_size, trainer_cls, state=None):
    args = TR.build_parser().parse_args(["--type", kind])
    torch.manual_seed(0)
    model = TR.build_model(args).cuda()
    if state is not None:
        model.load_state_dict(state)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
    sched = torch.optim.lr_scheduler.StepLR(opt, 10)
    return trainer_cls(model, criterion=PredictionLoss(), optimizer=opt, lr_scheduler=sched, device=torch.device("cuda"),
                       batch_size=batch_size, augment=True, normalize_scene=True)


def time_epochs(trainer, scenes, epochs):
    times = []
    for epoch in range(epochs + 1):                      # epoch 0 warms up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        trainer.train(scenes, None, epoch)
        torch.cuda.synchronize()
        if epoch:
            times.append(time.perf_counter() - t0)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--cells", default="directional:8,directional:64,social:8,social:64")
    args = ap.parse_args()
    _lib.require_cuda()
    from oracle.ref_shim import import_reference, reference_root
    import_reference()
    from trajnetbaselines.lstm import trainer as ref_trainer
    logging.getLogger().setLevel(logging.WARNING)
    warnings.simplefilter("ignore")
    folder = os.path.join(reference_root(), "DATA_BLOCK", "trajdata", "train")
    files = sorted(os.path.join(folder, f) for f in os.listdir(folder) if f.endswith(".ndjson"))
    t0 = time.perf_counter()
    store = TR.SceneStore.from_files(files)
    torch.cuda.synchronize()
    load_s = time.perf_counter() - t0
    ref_scenes = [(os.path.basename(f).split(".")[-2], sid, paths) for f in files for sid, paths in read_ndjson_scenes(f)]
    assert len(ref_scenes) == store.n
    emit(scenes=store.n, tracks=int(store.split[-1]), kept_tracks=int(store.kept.sum()), frames=store.T,
         store_load_s=round(load_s, 3))
    lib = _lib.load()
    for cell in args.cells.split(","):
        kind, bs = cell.split(":")
        bs = int(bs)
        random.seed(1)
        np.random.seed(1)
        native = make_trainer(kind, bs, TR.Trainer)
        state = {k: v.detach().clone() for k, v in native.model.state_dict().items()}
        native_s = time_epochs(native, store, args.epochs)
        lib.tb2_profile_begin()
        native.train(store, None, args.epochs + 1)
        torch.cuda.synchronize()
        buf = ctypes.create_string_buffer(1 << 16)
        _lib.check(lib.tb2_profile_end(buf, len(buf)))
        gather = json.loads(buf.value.decode()).get("scenes_gather_epoch", {})
        random.seed(1)
        np.random.seed(1)
        ref = make_trainer(kind, bs, ref_trainer.Trainer, state)
        ref_s = time_epochs(ref, list(ref_scenes), args.epochs)
        med_n, med_r = float(np.median(native_s)), float(np.median(ref_s))
        emit(model=kind, batch_size=bs, augment=True, normalize_scene=True,
             native_epoch_s=[round(v, 3) for v in native_s], native_median_s=round(med_n, 3),
             native_scenes_per_s=round(store.n / med_n, 1),
             reference_epoch_s=[round(v, 3) for v in ref_s], reference_median_s=round(med_r, 3),
             reference_scenes_per_s=round(store.n / med_r, 1), reference_over_native=round(med_r / med_n, 2),
             gather_kernel_ms=gather.get("total_ms"), gather_launches=gather.get("launches"))
        del native, ref
        torch.cuda.empty_cache()
    name, q = device_info()
    emit(gpu=name, nvidia_smi_name_power_limit_max_sm_clock_sm_clock=q)


if __name__ == "__main__":
    main()
