"""Golden vectors for the per-scene preprocessing functions, produced by the UNMODIFIED reference
(trajnetbaselines/lstm/lstm.py drop_distant, lstm/utils.py center_scene / theta_rotation,
augmentation.py inverse_scene) imported through oracle/ref_shim.py.

    python -m oracle.make_scene_ops_golden   -> tests/golden/scene_ops_golden.npz

Inputs are the seeded scenes of tests/test_scene_ops.py (_scenes([1, 4, 9, 33], seed=5)); they are
stored beside the outputs so the test checks that it regenerates the same scenes.
"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES, SEED, THETA = (1, 4, 9, 33), 5, 1.234


def main():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    from oracle.ref_shim import import_reference
    from test_scene_ops import _scenes
    import_reference()
    from trajnetbaselines import augmentation
    from trajnetbaselines.lstm import lstm as ref_lstm
    from trajnetbaselines.lstm import utils as ref_utils
    out = {}
    for i, xy in enumerate(_scenes(list(SIZES), seed=SEED)):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            dropped, mask = ref_lstm.drop_distant(xy)
        centered, rot, cen = ref_utils.center_scene(xy, 9)
        out["xy%d" % i] = xy
        out["drop%d" % i] = dropped
        out["mask%d" % i] = mask
        out["center%d" % i] = centered
        out["rot%d" % i] = np.float64(rot)
        out["cen%d" % i] = np.asarray(cen)
        out["theta%d" % i] = ref_utils.theta_rotation(xy, THETA)
        out["inverse%d" % i] = augmentation.inverse_scene(centered.astype(np.float32), rot, cen)
    path = os.path.join(ROOT, "tests", "golden", "scene_ops_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
