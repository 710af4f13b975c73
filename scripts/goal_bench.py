"""Inference rate of goal-conditioned LSTM models (LSTM(goal_flag=True), goal_dim 64) next to the same models without the
goal input, on bench.py's synthetic batch (256 scenes x 20 tracks, 9 observed + 12 predicted frames) with its seeded
weights: S-LSTM (social n=16 two_layer 1024 -> 256, latent 16) and D-LSTM (directional n=12 one_layer 256), H = 128.
The goal embedding widens the gate GEMM's K by 64 (E + P + H = 448 -> 512); this measures what that costs.

For every (model, goals) it prints one JSON line with the device-resident forward rate in pedestrian-steps/s (CUDA
events around each call, inputs on the device), the per-step kernel times of one forward (tb2_profile_begin / end, a
separate run) and the gate kernel that ran.  The forward rate is the figure to compare: the kernels are launched with
programmatic dependent launch, so a kernel's timer window includes its wait for the previous kernel and the per-kernel
times do not add up to the forward.  Prints the card's name and power limit first.

    python scripts/goal_bench.py [--iters 30] [--rounds 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBS, PRED, SCENES, PEDS = 9, 12, 256, 20
STEPS = OBS - 1 + PRED - 1          # recurrence steps of a free-running forward (n_predict = 12)
KINDS = {"S-LSTM": "social", "D-LSTM": "directional"}
GOAL_DIM = 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3, help="alternating rounds of (without, with) goals")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)                        # oracle/: seeded weights and scenes
    import numpy as np
    import torch
    from oracle import lstm_oracle as O
    from oracle.make_goal_golden import goal_weights
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling

    if not torch.cuda.is_available():
        raise SystemExit("goal_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print("# card: %s" % (card[0] if card else "unknown"))
    lib = _lib.load()
    xy, bs = O.synthetic_scenes(SCENES, PEDS, n_frames=OBS + PRED, seed=1000)
    M = xy.shape[1]
    scene = torch.from_numpy(xy).cuda()
    bs_t = torch.from_numpy(bs)
    goals = torch.from_numpy((np.nan_to_num(xy[-1]) + 1.5).astype(np.float32)).cuda()

    for name, kind in KINDS.items():
        models = {}
        for with_goals in (False, True):
            W = goal_weights(kind, GOAL_DIM, seed=1) if with_goals else O.random_weights(kind, seed=1)
            model = LSTM(pool=GridBasedPooling(**O.MODEL_SPECS[kind]), goal_flag=with_goals, goal_dim=GOAL_DIM)
            model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
            models[with_goals] = model.cuda().eval()

        def fwd(with_goals):
            with torch.no_grad():
                return models[with_goals](scene[:OBS], goals, bs_t, n_predict=PRED)

        for g in (False, True):
            for _ in range(3):
                fwd(g)
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for _ in range(args.rounds):                 # alternate, so both see the same host / clock conditions
            for g in (False, True):
                ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
                for a, b in ev:
                    a.record()
                    fwd(g)
                    b.record()
                torch.cuda.synchronize()
                times[g].append(sum(a.elapsed_time(b) for a, b in ev) / args.iters)
        for g in (False, True):
            ms = sorted(times[g])[len(times[g]) // 2]
            buf = ctypes.create_string_buffer(1 << 16)
            lib.tb2_profile_begin()
            fwd(g)
            _lib.check(lib.tb2_profile_end(buf, len(buf)))
            prof = json.loads(buf.value.decode())
            gate = "lstm_gates_tc" if "lstm_gates_tc" in prof else "lstm_gates"
            print(json.dumps(dict(model=name, goals=g, goal_dim=GOAL_DIM if g else 0, scenes=SCENES, tracks=M,
                                  forward_ms_median=round(ms, 4), forward_ms_rounds=[round(t, 4) for t in times[g]],
                                  forward_ped_steps_per_s=round(M * STEPS / (ms * 1e-3)), gate_kernel=gate,
                                  kernel_us_per_step={k: round(1e3 * v["total_ms"] / STEPS, 2) for k, v in prof.items()})))


if __name__ == "__main__":
    main()
