"""Kernel times of the non-grid interaction modules (csrc/mlp_pool.cu) through the stand-alone plug, from CUDA events
(tb2_profile_begin / end): hidden_mlp_pool, attn_mlp_pool, nn_mlp_pool, traj_scene_sum + traj_feat and pool_lstm_cell,
at the reference trainer's widths (pool_dim 256, hidden 128, spatial / velocity 32), on 256 scenes x 20 tracks and on one
93-track scene.  Prints the card's name and power limit, then one JSON line per (module, shape).

    python scripts/nongrid_bench.py [--iters 200] [--tree DIR] [--label NAME]

--tree imports the package from another checkout (built in place), so that two builds can be timed alternately from one
shell command, e.g. for t in new old new old; do python scripts/nongrid_bench.py --tree $t; done.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--label", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import numpy as np
    import torch
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200 import lstm as L

    if not torch.cuda.is_available():
        raise SystemExit("nongrid_bench needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print("# card: %s" % (card[0] if card else "unknown"))
    lib = _lib.load()
    modules = {
        "hiddenstatemlp": lambda: L.HiddenStateMLPPooling(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256),
        "attentionmlp": lambda: L.AttentionMLPPooling(hidden_dim=128, mlp_dim=128, mlp_dim_spatial=32, mlp_dim_vel=32, out_dim=256),
        "nn": lambda: L.NearestNeighborMLP(n=4, out_dim=256),
        "nn_lstm": lambda: L.NearestNeighborLSTM(n=4, hidden_dim=128, out_dim=256),
        "traj_pool": lambda: L.TrajectronPooling(hidden_dim=128, out_dim=256),
    }
    for B, N in ((256, 20), (1, 93)):
        rng = np.random.RandomState(0)
        obs2 = torch.from_numpy((rng.rand(B, N, 2) * 10).astype(np.float32)).cuda()
        obs1 = obs2 - torch.from_numpy((rng.randn(B, N, 2) * 0.3).astype(np.float32)).cuda()
        hid = torch.from_numpy((rng.randn(B, N, 128) * 0.5).astype(np.float32)).cuda()
        for name, make in modules.items():
            torch.manual_seed(0)
            m = make().cuda()
            row = dict(label=args.label or os.path.basename(os.path.abspath(args.tree)), module=name, scenes=B, tracks=N)
            with torch.no_grad():
                try:
                    for _ in range(10):
                        m(hid, obs1, obs2)
                except RuntimeError as e:          # a launcher refusing the scene size (checked on the host)
                    print(json.dumps(dict(row, refused=str(e))))
                    continue
                torch.cuda.synchronize()
                buf = ctypes.create_string_buffer(1 << 16)
                lib.tb2_profile_begin()
                for _ in range(args.iters):
                    m(hid, obs1, obs2)
                _lib.check(lib.tb2_profile_end(buf, len(buf)))
            prof = json.loads(buf.value.decode())
            print(json.dumps(dict(row, kernel_us={k: round(1e3 * v["total_ms"] / v["launches"], 2) for k, v in prof.items()})))


if __name__ == "__main__":
    main()
