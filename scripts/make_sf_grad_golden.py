"""Writes tests/golden/sf_grad_golden.npz: complex-step ADE / FDE derivatives of real scenes for tb2_sf_sweep_grad.

Scenes of the reference's DATA_BLOCK/trajdata/train files, prepared as the sweep prepares them (sweep.load_scenes +
initial_states_xy, obs_length 9, pred_length 12): crowds_students001's largest scene, finite scenes of several sizes,
and one scene with a NaN destination (a pedestrian with a single observed row stands on its destination, so every
ADE of the scene is NaN).  The scenes' xy arrays (NaN = no row) are kept too, so a test can write them back to an
ndjson file.  For each of SETTINGS, tests/sf_cs_oracle.score_grad gives ADE / FDE and their derivatives.

    python scripts/make_sf_grad_golden.py [DATA_BLOCK/trajdata/train]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sf_cs_oracle as CS                                                          # noqa: E402
from oracle.ref_shim import reference_root                                         # noqa: E402
from trajnetplusplusbaselines_b200 import data                                     # noqa: E402
from trajnetplusplusbaselines_b200.classical import sweep                          # noqa: E402
from trajnetplusplusbaselines_b200.classical.common import initial_states_xy       # noqa: E402

SETTINGS = [(0.5, 2.1, 0.3), (0.3, 1.0, 0.6), (1.0, 5.0, 0.2)]
PICKS = {"crowds_students001.ndjson": 6, "biwi_hotel.ndjson": 3}               # finite scenes besides the largest


def _scenes(path, n_finite):
    loaded = sweep.load_scenes(path)
    state, _, off, truth = initial_states_xy(loaded)
    sizes = np.diff(off)
    nan_dest = (state[:, 4] == state[:, 0]) & (state[:, 5] == state[:, 1])
    finite = np.array([not nan_dest[off[b]:off[b + 1]].any() for b in range(len(sizes))])
    picks = [int(np.argmax(sizes))]
    by_size = [b for b in np.argsort(sizes, kind="stable") if finite[b] and sizes[b] > 1]
    picks += [int(by_size[i]) for i in np.linspace(0, len(by_size) - 1, n_finite).astype(int)]
    nan_scenes = [b for b in range(len(sizes)) if not finite[b] and 2 <= sizes[b] <= 6]
    if nan_scenes:
        picks.append(nan_scenes[0])
    picks = list(dict.fromkeys(picks))
    xy = lambda s: s if isinstance(s, np.ndarray) else data.paths_to_xy(s)
    return [(state[off[b]:off[b + 1]], truth[b], xy(loaded[b][1])) for b in picks]


def main():
    src = sys.argv[1] if len(sys.argv) > 1 else os.path.join(reference_root() or "", "DATA_BLOCK", "trajdata", "train")
    scenes = []
    for fn, k in PICKS.items():
        scenes += _scenes(os.path.join(src, fn), k)
    B, S = len(scenes), len(SETTINGS)
    ade, fde = np.empty((S, B)), np.empty((S, B))
    dade, dfde = np.empty((S, B, 3)), np.empty((S, B, 3))
    for s, prm in enumerate(SETTINGS):
        for b, (st, tr, _) in enumerate(scenes):
            ade[s, b], fde[s, b], dade[s, b], dfde[s, b] = CS.score_grad(st, tr[-12:], *prm)
    sizes = [len(st) for st, _, _ in scenes]
    out = {"state": np.concatenate([st for st, _, _ in scenes]), "offsets": np.concatenate([[0], np.cumsum(sizes)]),
           "truth": np.stack([tr for _, tr, _ in scenes]), "settings": np.array(SETTINGS, dtype=np.float64),
           "xy": np.concatenate([xy for _, _, xy in scenes], axis=1),
           "xy_offsets": np.concatenate([[0], np.cumsum([xy.shape[1] for _, _, xy in scenes])]),
           "ade": ade, "fde": fde, "dade": dade, "dfde": dfde}
    path = os.path.join(ROOT, "tests", "golden", "sf_grad_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d scenes (sizes %s), %d settings, %d non-finite" % (path, B, sizes, S, int((~np.isfinite(ade[0])).sum())))


if __name__ == "__main__":
    main()
