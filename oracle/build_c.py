"""Compile the oracle's plain-C parts (gcc) into oracle/_build/.  TEST INFRASTRUCTURE."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_build")
LIB = os.path.join(OUT_DIR, "liborca_oracle.so")


def build(force=False):
    src = os.path.join(HERE, "orca_oracle.c")
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= os.path.getmtime(src):
        return LIB
    os.makedirs(OUT_DIR, exist_ok=True)
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", LIB, src, "-lm"])
    return LIB


def load():
    import ctypes
    lib = ctypes.CDLL(build())
    lib.orca_simulate_scene.restype = ctypes.c_int
    lib.orca_simulate_scene.argtypes = [
        ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
        ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_double,
        ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return lib


ORCA_COUNTERS = ("at_cap", "collision_lines", "lp3", "end_range_stops")


def orca_simulate(pos, vel, goal, speed, time_step=0.05, neighbor_dist=1.5, max_neighbors=10,
                  time_horizon=1.5, radius=0.4, end_range=0.05, n_steps=97, sample_every=8, counters=None):
    """numpy front-end: pos, vel [n,2] float32; goal [n,2], speed [n] float64 -> [n_steps//8, n, 2].
    counters: None, or a dict that gets ORCA_COUNTERS added to it: (agent, step) pairs with a full neighbour list,
    ORCA lines from the collision branch, linearProgram3 calls, (agent, step) pairs whose preferred velocity is
    zeroed within end_range of the goal."""
    import numpy as np
    lib = load()
    pos = np.ascontiguousarray(pos, dtype=np.float32)
    vel = np.ascontiguousarray(vel, dtype=np.float32)
    goal = np.ascontiguousarray(goal, dtype=np.float64)
    speed = np.ascontiguousarray(speed, dtype=np.float64)
    n = len(pos)
    out = np.zeros((n_steps // sample_every, n, 2), dtype=np.float32)
    cnt = np.zeros(len(ORCA_COUNTERS), dtype=np.int64)
    rc = lib.orca_simulate_scene(n, pos.ctypes.data, vel.ctypes.data, goal.ctypes.data, speed.ctypes.data,
                                 time_step, neighbor_dist, max_neighbors, time_horizon, radius, end_range,
                                 n_steps, sample_every, out.ctypes.data,
                                 None if counters is None else cnt.ctypes.data)
    assert rc == 0
    if counters is not None:
        for k, v in zip(ORCA_COUNTERS, cnt):
            counters[k] = counters.get(k, 0) + int(v)
    return out


if __name__ == "__main__":
    print(build(force=True))
