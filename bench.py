#!/usr/bin/env python
"""Benchmark of the TrajNet++ hot path on one or more H100 GPUs.

    python bench.py --gpus N --steps K --warmup W            # CUDA arm
    python bench.py --impl reference --gpus N --steps K --warmup W   # CPU arm: the unmodified reference (oracle/_ref)
    python bench.py ... --dump-outputs DIR    # also write the last timed step's outputs as DIR/<name>.npy

A "step" is one pass of the hot path over one batch of synthetic scenes: one call of
LSTM.forward = (obs-1) + (pred-1) = 19 recurrence steps for every track of the batch.
Metric: pedestrian-steps / second = tracks x 19 x K / time (SURVEY.md section 8d).
Workload at every N: BASELINE.json configs[2] -- Social-LSTM (--type social --n 16
--embedding_arch two_layer --layer_dims 1024), 256 scenes x 20 pedestrians PER GPU (weak
scaling: scenes are independent, no data-path collective), T = 9 observed + 12 predicted.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KIND = "social"
SCENES_PER_GPU = 256
PEDS = 20
OBS, PRED = 9, 12
STEPS_PER_FORWARD = (OBS - 1) + (PRED - 1)       # 19
STATE_BYTES_PER_PED_STEP = 2092                   # SURVEY.md 8d: xy 16 + h,c in 1024 + h,c out 1024 + normal 20 + pos 8
DENSE_FLOP_PER_PED_STEP = {                       # SURVEY.md 8d, dense-equivalent forward FLOPs
    "sparse_layer1": 2 * 4096 * 1024,             # first Linear of the grid embedding (4096 -> 1024)
    "sparse_layer1_mma": 2 * 4096 * 1024,
    "dense_layer": 2 * 1024 * 256,
    "dense_layer_tc": 2 * 1024 * 256,
    "lstm_gates": 2 * (64 + 256 + 128) * 512 + 2 * 128 * 5,
    "lstm_gates_tc": 2 * (64 + 256 + 128) * 512 + 2 * 128 * 5,
}


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        d = json.load(open(path))
        return d["hbm_gbs"], d["bf16_tflops"], d.get("bf16_tflops_sustained", d["bf16_tflops"]), "measured"
    return 3350.0, 989.0, 989.0, "H100 SXM data sheet (dense bf16)"


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    QUERY = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
             "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index = index
        self.proc = None
        self.lines = []

    def run(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.QUERY,
                 "--format=csv,noheader,nounits", "-lms", "100"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                self.lines.append(line.strip())
        except Exception:
            pass

    def stop(self):
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()
        sm, smax, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            parts = [p.strip() for p in ln.split(",")]
            if len(parts) < 9:
                continue
            try:
                sm.append(float(parts[1]))
                smax.append(float(parts[2]))
            except ValueError:
                continue
            for name, val in zip(names, parts[5:9]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"], "samples": 0}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(np.max(smax)),
                "reasons": sorted(reasons), "samples": len(sm)}


def make_inputs(rank, scenes, seed=0):
    from oracle import lstm_oracle as O      # synthetic generator only (shared with the tests)
    xy, bs = O.synthetic_scenes(scenes, PEDS, n_frames=OBS + PRED, seed=seed + 1000 * rank)
    return xy, bs


def workload_config(scenes, world):
    """`config` of the JSON line -- identical for the CUDA arm and the reference arm."""
    return {"workload": "Social-LSTM inference (BASELINE configs[2]): type=social n=16 cell_side=0.6 "
                        "two_layer 1024 -> 256, latent 16, hidden 128",
            "scenes_per_gpu": scenes, "peds_per_scene": PEDS, "obs": OBS, "pred": PRED,
            "recurrence_steps_per_step": STEPS_PER_FORWARD, "parallelism": "scenes sharded x%d, no collective" % world,
            "l2": "256 MiB memset between timed iterations (untimed); inputs are smaller than L2"}


def cpu_oracle_run(scenes):
    """Fallback CPU leg when the reference install is absent: the numpy oracle port on `scenes` scenes."""
    from oracle import lstm_oracle as O
    W = O.random_weights(KIND, seed=1)
    xy, bs = make_inputs(0, scenes)
    cfg = O.pool_config(KIND)
    t0 = time.perf_counter()
    O.forward(W, cfg, xy[:OBS], bs, n_predict=PRED)
    dt = time.perf_counter() - t0
    return scenes * PEDS * STEPS_PER_FORWARD / dt, dt


class ReferenceCpu:
    """The UNMODIFIED reference (oracle/_ref, see oracle/build_ref.py) on the host cores: its own
    `trajnetbaselines.lstm.LSTM` + `GridBasedPooling`, torch CPU, same seeded weights and synthetic scenes as the
    CUDA arm, `LSTM.forward(observed, goals, batch_split, n_predict=12)` under torch.no_grad()."""

    def __init__(self):
        import torch
        from oracle import lstm_oracle as O
        from oracle.ref_shim import import_reference, reference_root
        import_reference()
        from oracle.make_golden import build_reference_model
        self.torch = torch
        self.root = reference_root()
        self.model = build_reference_model(KIND, O.random_weights(KIND, seed=1))
        self._inputs = {}
        # "all the host threads it can use": torch's intra-op pool at os.cpu_count() threads is the natural choice,
        # but on a many-core virtualised host the reference's thousands of tiny ops per forward get SLOWER with
        # more threads (measured on a 128-core GPU box: 64 scenes in 62 s at 128 threads, ~1 s at 8).  The thread
        # count is therefore calibrated on a small forward and the fastest setting is used and reported.
        self.host_cores = os.cpu_count()
        best = None
        for n in sorted({c for c in (4, 8, 16, 32, 64, self.host_cores) if c <= self.host_cores}):
            torch.set_num_threads(n)
            self.forward_seconds(8)
            t = min(self.forward_seconds(8) for _ in range(2))
            if best is None or t < best[0]:
                best = (t, n)
            if t > 4.0 * best[0]:
                break                              # far past the optimum: larger pools only get worse
        self.cores = best[1]
        torch.set_num_threads(self.cores)

    def forward_seconds(self, scenes):
        torch = self.torch
        if scenes not in self._inputs:
            xy, bs = make_inputs(0, scenes)
            self._inputs[scenes] = (torch.from_numpy(xy[:OBS].copy()), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs))
        obs, goals, split = self._inputs[scenes]
        t0 = time.perf_counter()
        with torch.no_grad():
            self.model(obs, goals, split, n_predict=PRED)
        return time.perf_counter() - t0


def run_reference(args):
    """--impl reference: the reference's own CPU implementation of the path, all host threads, same metric /
    config.  A step is one forward of the full workload (256 scenes x 20 pedestrians) unless that would not
    finish in a few minutes on this host, in which case a step is a 64-scene sample (stated in cpu_baseline)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    try:
        ref = ReferenceCpu()
        kind = "reference"
    except Exception as exc:                      # reference not importable: the numpy restatement, labelled as such
        ref, kind = None, "port"
        note = "reference install not importable (%s: %s); numpy fp32 oracle port instead" % (type(exc).__name__, exc)
    cores = os.cpu_count()
    full = args.scenes
    if ref is not None:
        ref.forward_seconds(8)
        probe = ref.forward_seconds(64)                       # untimed probe: does the full workload fit the budget?
        sample = full if probe * (full / 64.0) * (args.steps + 1) < 240.0 else 64
        for i in range(args.warmup):
            ref.forward_seconds(sample if i == 0 else 8)
        per_step = [ref.forward_seconds(sample) for _ in range(args.steps)]
        cores = ref.cores
        how = ("unmodified reference (%s) torch %s CPU, torch.set_num_threads(%d) = fastest of a calibration sweep on this "
               "%d-core host, LSTM.forward under no_grad"
               % (os.path.relpath(ref.root, ROOT) if ref.root.startswith(ROOT) else ref.root, ref.torch.__version__, cores,
                  ref.host_cores))
    else:
        sample = 64
        for _ in range(args.warmup):
            cpu_oracle_run(8)
        per_step = [cpu_oracle_run(sample)[1] for _ in range(args.steps)]
        how = note
    t_total = float(sum(per_step))
    value = sample * PEDS * STEPS_PER_FORWARD * args.steps / t_total
    med = float(np.median(per_step))
    line = {
        "impl": "reference", "metric": "pedestrian-steps/sec", "value": value, "unit": "ped-steps/s",
        "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * t_total / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": workload_config(full, max(args.gpus, 1)),
        "cpu_baseline": {"value": value, "unit": "ped-steps/s", "cores": cores, "kind": kind,
                         "sample": "%d scenes x %d peds x %d steps per step (%s); %s; median step %.2f s, "
                                   "best step = %.0f ped-steps/s"
                                   % (sample, PEDS, STEPS_PER_FORWARD, "the full workload" if sample == full else
                                      "bounded sample of the %d-scene workload" % full, how, med,
                                      sample * PEDS * STEPS_PER_FORWARD / min(per_step))},
        "e2e": {"value": value, "unit": "ped-steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def train_record(torch, dist, device, world, rank, steps, warmup=3):
    """BASELINE configs[3] under the same launch: D-LSTM `Trainer.train_batch` work (teacher-forced forward,
    PredictionLoss x batch, CUDA BPTT, Adam) on 256 scenes per GPU, plus ONE flat-bucket all-reduce of the
    gradients per step when world > 1.  Device-timed, max over ranks (reference lstm/trainer.py:229-269)."""
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss
    from trajnetplusplusbaselines_b200.parallel import allreduce_gradients
    kind = "directional"
    B = SCENES_PER_GPU
    W = O.random_weights(kind, seed=1)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.to(device).train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4, fused=True)   # trainer.py:497 hyper-parameters
    crit = PredictionLoss()
    xy, bs = O.synthetic_scenes(B, PEDS, seed=100 + rank)
    scene = torch.from_numpy(xy).to(device)
    bs_t = torch.from_numpy(bs)
    targets = scene[OBS:OBS + PRED] - scene[OBS - 1:OBS + PRED - 1]
    goals = torch.zeros(xy.shape[1], 2)
    ar_events = []
    bucket = [0]

    def step(timed):
        rel, _ = model(scene[:OBS], goals, bs_t, scene[OBS:-1])
        loss = crit(rel[-PRED:], targets, bs_t) * B
        opt.zero_grad()
        loss.backward()
        if world > 1:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            bucket[0] = allreduce_gradients(model.parameters())
            e1.record()
            if timed:
                ar_events.append((e0, e1))
        opt.step()
        return loss

    for _ in range(warmup):
        step(False)
    torch.cuda.synchronize(device)
    if world > 1:
        dist.barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        loss = step(True)
    b.record()
    torch.cuda.synchronize(device)
    if world > 1:
        dist.barrier()
    ar_ms = sum(e0.elapsed_time(e1) for e0, e1 in ar_events)
    t = torch.tensor([a.elapsed_time(b), ar_ms], dtype=torch.float64, device=device)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ar_ms = t.tolist()
    M = xy.shape[1]
    return {"workload": "D-LSTM Trainer.train_batch (BASELINE configs[3]): directional n=12 one_layer 256, teacher-forced, "
                        "PredictionLoss, CUDA BPTT, fused Adam; %d scenes x %d peds per GPU" % (B, PEDS),
            "n_gpus": world, "steps": steps, "warmup": warmup, "ms_per_step": ms / steps,
            "value": M * STEPS_PER_FORWARD * world * steps / (ms * 1e-3), "unit": "ped-steps/s", "scaling": "weak",
            "collective": None if world == 1 else
            {"op": "one NCCL all-reduce(SUM) of a flat fp32 bucket per step", "floats": int(bucket[0]),
             "ms_per_step": ar_ms / steps, "share_of_step": ar_ms / ms,
             "note": "CUDA events around bucket build + ncclAllReduce + scatter back, max over ranks"},
            "loss": float(loss.item())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--scenes", type=int, default=SCENES_PER_GPU, help="scenes per GPU")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-train", action="store_true", help="skip the D-LSTM training sub-record")
    ap.add_argument("--dump-outputs", metavar="DIR",
                    help="write the (rel, pred) arrays of the last timed inference step as DIR/<name>.npy (float32)")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)
    args.warmup = max(args.warmup, 3)

    import torch
    import torch.distributed as dist
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench.py needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
    lib = _lib.load()

    def barrier():
        torch.cuda.synchronize(device)
        if world > 1:
            dist.barrier()

    # model: random-init weights of the BASELINE architecture (seeded, same as the CPU arm)
    W = O.random_weights(KIND, seed=1)
    model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[KIND]))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
    model = model.to(device).eval()

    xy, bs = make_inputs(rank, args.scenes)
    M = xy.shape[1]
    observed_host = torch.from_numpy(xy[:OBS]).pin_memory()
    observed_dev = observed_host.to(device)
    goals = torch.zeros(M, 2)
    bs_t = torch.from_numpy(bs)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=device)     # > 50 MB L2

    def step_resident():
        with torch.no_grad():
            return model(observed_dev, goals, bs_t, n_predict=PRED)

    def step_e2e():
        with torch.no_grad():
            return model(observed_host, goals, bs_t, n_predict=PRED)      # H2D in, D2H out inside

    # ---- device-resident arm ---------------------------------------------------------------
    for _ in range(args.warmup):
        step_resident()
    barrier()
    sampler = ClockSampler(local_rank)
    sampler.start()
    time.sleep(0.25)
    launches0 = int(lib.tb2_launch_count())
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]
    stops = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]
    barrier()
    t_wall0 = time.perf_counter()
    last = None
    for i in range(args.steps):
        flush.zero_()                       # L2 flush between timed iterations (untimed)
        starts[i].record()
        last = step_resident()
        stops[i].record()
    barrier()
    t_wall = time.perf_counter() - t_wall0
    launches = int(lib.tb2_launch_count()) - launches0
    ms = sum(s.elapsed_time(e) for s, e in zip(starts, stops))
    clocks = sampler.stop()
    if args.dump_outputs and rank == 0:
        # inputs and weights are seeded, so two builds can be compared output for output (5120 tracks: ~2.7 MB).
        # Above 64 MB in all, a fixed seeded sample of tracks (axis 1) is written, with its indices as track_index.npy.
        os.makedirs(args.dump_outputs, exist_ok=True)
        arrs = {name: arr.detach().cpu().numpy().astype(np.float32) for name, arr in zip(("rel", "pred"), last)}
        per_track = sum(a.nbytes // a.shape[1] for a in arrs.values())
        if per_track * M > (64 << 20):
            keep = (64 << 20) // (per_track + 8)          # + 8 bytes per track for its float64 index
            idx = np.sort(np.random.RandomState(0).choice(M, keep, replace=False))
            arrs = {name: np.ascontiguousarray(a[:, idx]) for name, a in arrs.items()}
            arrs["track_index"] = idx.astype(np.float64)
        for name, a in arrs.items():
            np.save(os.path.join(args.dump_outputs, name + ".npy"), a)
    last = None

    # ---- end-to-end arm (host buffers, copies inside the timed region) -----------------------
    keep = None
    for _ in range(args.warmup):
        keep = step_e2e()      # held across the next call like in the timed loop, so the pinned result pool reaches
    barrier()                  # its steady state (two buffer sets) during warm-up: a cudaHostAlloc costs ~50 ms here
    keep = None
    import gc
    gc.collect()
    per_step = []
    for i in range(args.steps):
        flush.zero_()
        torch.cuda.synchronize(device)
        t0 = time.perf_counter()
        rel, pred = step_e2e()             # returns host tensors after the copies have completed
        per_step.append(1e3 * (time.perf_counter() - t0))
    e2e_ms = sum(per_step)                 # every step counts (no re-measurement): median / p95 are reported beside it
    barrier()
    h2d = observed_host.numel() * 4 + bs_t.numel() * 8
    d2h = (rel.numel() + pred.numel()) * 4

    # ---- per-kernel CUDA-event timing for the roofline (separate pass, events on the launch stream)
    prof_iters = 3
    lib.tb2_profile_begin()
    for _ in range(prof_iters):
        flush.zero_()
        step_resident()
    buf = ctypes.create_string_buffer(1 << 16)
    _lib.check(lib.tb2_profile_end(buf, len(buf)))
    prof = json.loads(buf.value.decode())

    t = torch.tensor([ms, e2e_ms], dtype=torch.float64, device=device)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_max, e2e_ms_max = t.tolist()

    # ---- training sub-record: the one workload with a collective (BASELINE configs[3]) ------------------
    train = None
    if not args.no_train:
        train = train_record(torch, dist, device, world, rank, args.steps)

    if rank == 0:
        ped_steps = M * STEPS_PER_FORWARD * world          # every rank runs the same shape
        value = ped_steps * args.steps / (ms_max * 1e-3)
        e2e_value = ped_steps * args.steps / (e2e_ms_max * 1e-3)
        hbm, tf_burst, tf_sust, how = peaks()
        total_ms = sum(v["total_ms"] for v in prof.values()) or 1.0
        dom = max(prof, key=lambda k: prof[k]["total_ms"])
        dom_avg_ms = prof[dom]["total_ms"] / prof[dom]["launches"]
        kern = {}
        for name, v in prof.items():
            avg = v["total_ms"] / v["launches"]
            kern[name] = {"avg_us": 1e3 * avg, "launches_per_forward": v["launches"] / prof_iters,
                          "share": v["total_ms"] / total_ms}
        if dom in DENSE_FLOP_PER_PED_STEP:
            flops = DENSE_FLOP_PER_PED_STEP[dom] * M
            achieved = flops / (dom_avg_ms * 1e-3) / 1e12
            roofline = {"kernel": dom, "bound": "tensor", "achieved": achieved, "peak": tf_sust,
                        "unit": "TFLOP/s", "frac": achieved / tf_sust,
                        "peak_source": how + " bf16 sustained (kernel timed inside a long step)",
                        "note": "achieved = dense algorithmic FLOPs of the 4096->1024 grid Linear (SURVEY 8d: "
                                "2*4096*1024 per ped-step) / CUDA-event time; the kernel issues 3 bf16 passes "
                                "(hi/lo split for the 1e-4 m gate), so 1/3 of peak is its ceiling"}
        else:
            bytes_ = STATE_BYTES_PER_PED_STEP * M
            achieved = bytes_ / (dom_avg_ms * 1e-3) / 1e9
            roofline = {"kernel": dom, "bound": "hbm", "achieved": achieved, "peak": hbm, "unit": "GB/s",
                        "frac": achieved / hbm, "peak_source": how}
        # state-streaming view of the whole step (all kernels of one recurrence step)
        step_ms = total_ms / prof_iters / STEPS_PER_FORWARD
        roofline["step_hbm"] = {"achieved": STATE_BYTES_PER_PED_STEP * M / (step_ms * 1e-3) / 1e9,
                                "peak": hbm, "unit": "GB/s",
                                "frac": STATE_BYTES_PER_PED_STEP * M / (step_ms * 1e-3) / 1e9 / hbm}
        roofline["kernels"] = kern
        cpu = None
        if world == 1 and not args.no_cpu_baseline:
            n_cpu = min(args.scenes, SCENES_PER_GPU)
            try:
                ref = ReferenceCpu()
                ref.forward_seconds(8)
                probe = ref.forward_seconds(64)
                sample = n_cpu if probe * (n_cpu / 64.0) < 40.0 else 64          # bounded: about 10-30 s of CPU work
                dt = min(ref.forward_seconds(sample) for _ in range(2)) if sample * probe / 64.0 < 12.0 else ref.forward_seconds(sample)
                cpu = {"value": sample * PEDS * STEPS_PER_FORWARD / dt, "unit": "ped-steps/s", "cores": ref.cores, "kind": "reference",
                       "sample": "one forward of %d scenes x %d peds x %d steps (%s, %.1f s); unmodified reference from %s, torch %s "
                                 "CPU, torch.set_num_threads(%d) (fastest of a calibration sweep on this %d-core host); "
                                 "64-scene forward: %.0f ped-steps/s"
                                 % (sample, PEDS, STEPS_PER_FORWARD, "the full workload" if sample == n_cpu else "bounded sample",
                                    dt, os.path.relpath(ref.root, ROOT) if ref.root.startswith(ROOT) else ref.root,
                                    torch.__version__, ref.cores, ref.host_cores, 64 * PEDS * STEPS_PER_FORWARD / probe)}
            except Exception as exc:
                cpu_oracle_run(8)
                v, dt = cpu_oracle_run(64)
                cpu = {"value": v, "unit": "ped-steps/s", "cores": os.cpu_count(), "kind": "port",
                       "sample": "one forward of 64 scenes x 20 peds x 19 steps (%.1f s), numpy fp32 oracle port, BLAS threads=all "
                                 "(reference install not importable: %s)" % (dt, exc)}
        line = {
            "metric": "pedestrian-steps/sec", "value": value, "unit": "ped-steps/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_max / args.steps,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": workload_config(args.scenes, world),
            "e2e": {"value": e2e_value, "unit": "ped-steps/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                    "ms_per_step": e2e_ms_max / args.steps, "ms_median": float(np.median(per_step)),
                    "ms_p95": float(np.percentile(per_step, 95)), "ms_max": float(max(per_step)),
                    "note": "wall clock per call of LSTM.forward with host tensors in and out (rank 0's distribution; "
                            "value = all steps, none dropped or re-measured)"},
            "gpu_launches": launches,
            "clocks": clocks,
            "roofline": roofline,
            "cpu_baseline": cpu,
            "train": train,
            "wall_s_timed_region": t_wall,
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
