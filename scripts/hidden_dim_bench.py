"""LSTM throughput at hidden widths 64, 128 and 256, at the BASELINE shape (256 scenes x 20 tracks, 9 observed + 12
predicted frames), for Social-LSTM (BASELINE configs[2]: social n=16 two_layer 1024 -> 256, latent 16) and D-LSTM
(directional n=12 one_layer 256), with the seeded weights and scenes bench.py uses.  For every (model, H) it prints one
JSON line with
  * the device-resident forward rate in pedestrian-steps/s (CUDA events around each call, inputs already on the device);
  * the per-step kernel times of one forward (tb2_profile_begin / end, a separate run);
  * the time of one Trainer.train_batch step (teacher-forced forward, PredictionLoss x batch, backward, Adam);
  * the gate kernel's achieved TFLOP/s: 2 (E + P + H) 4H FLOPs per pedestrian-step over its profiled time.
Prints the card's name and power limit first.

    python scripts/hidden_dim_bench.py [--iters 20] [--tree DIR] [--label NAME]

--tree imports the package from another checkout (built in place); a build that refuses a width reports it and goes on.
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
KINDS = {"social": "social", "directional": "directional"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--label", default=None)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)                        # oracle/: seeded weights and scenes
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling, PredictionLoss

    if not torch.cuda.is_available():
        raise SystemExit("hidden_dim_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print("# card: %s" % (card[0] if card else "unknown"))
    lib = _lib.load()
    label = args.label or os.path.basename(os.path.abspath(args.tree))
    xy, bs = O.synthetic_scenes(SCENES, PEDS, n_frames=OBS + PRED, seed=1000)
    M = xy.shape[1]
    scene = torch.from_numpy(xy).cuda()
    bs_t = torch.from_numpy(bs)
    goals = torch.zeros(M, 2)
    for name, kind in KINDS.items():
        for H in (64, 128, 256):
            row = dict(label=label, model=name, hidden_dim=H, scenes=SCENES, tracks=M)
            W = O.random_weights(kind, seed=1, hidden_dim=H)
            model = LSTM(hidden_dim=H, pool=GridBasedPooling(**dict(O.MODEL_SPECS[kind], hidden_dim=H)))
            model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()})
            model = model.cuda().eval()

            def fwd():
                with torch.no_grad():
                    return model(scene[:OBS], goals, bs_t, n_predict=PRED)
            try:
                for _ in range(3):
                    fwd()
            except RuntimeError as e:
                print(json.dumps(dict(row, refused=str(e))))
                continue
            torch.cuda.synchronize()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
            for a, b in ev:
                a.record()
                fwd()
                b.record()
            torch.cuda.synchronize()
            ms = sum(a.elapsed_time(b) for a, b in ev) / args.iters
            row["forward_ms"] = round(ms, 4)
            row["forward_ped_steps_per_s"] = M * STEPS / (ms * 1e-3)
            buf = ctypes.create_string_buffer(1 << 16)
            lib.tb2_profile_begin()
            fwd()
            _lib.check(lib.tb2_profile_end(buf, len(buf)))
            prof = json.loads(buf.value.decode())
            row["kernel_us_per_step"] = {k: round(1e3 * v["total_ms"] / STEPS, 2) for k, v in prof.items()}
            gate = "lstm_gates_tc" if "lstm_gates_tc" in prof else "lstm_gates"
            E, P = 64, 256
            flops = 2.0 * (E + P + H) * 4 * H * M * STEPS
            row["gate_kernel"] = gate
            row["gate_tflops"] = round(flops / (prof[gate]["total_ms"] * 1e-3) / 1e12, 2)

            model.train()
            opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-4)
            crit = PredictionLoss()
            targets = scene[OBS:OBS + PRED] - scene[OBS - 1:OBS + PRED - 1]

            def train_step():
                rel, _ = model(scene[:OBS], goals, bs_t, scene[OBS:-1])
                loss = crit(rel[-PRED:], targets, bs_t) * SCENES
                opt.zero_grad()
                loss.backward()
                opt.step()
            try:
                for _ in range(2):
                    train_step()
            except (RuntimeError, NotImplementedError) as e:
                row["train_refused"] = str(e)
                print(json.dumps(row))
                continue
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n = max(1, args.iters // 4)
            a.record()
            for _ in range(n):
                train_step()
            b.record()
            torch.cuda.synchronize()
            row["train_batch_ms"] = round(a.elapsed_time(b) / n, 3)
            print(json.dumps(row))


if __name__ == "__main__":
    main()
