"""The grid embedding's first Linear against a float64 product of its own operands, per element, in every kernel.

The first Linear runs as one of four kernels (csrc/pool.cu): sparse_layer1_mma (social grid, 16 latent channels, 3-pass
bf16 mma.sync), sparse_layer1<C, SOCIAL> (FFMA: other latent widths, occupancy / directional grids too wide for
pool_rows, and C = 16 under TB2_DISABLE_TC=1), pool_rows (occupancy / directional weights in shared memory) and
dense_grid (no embedding).  Each computes, for every row i,

    out[i] = ReLU(base + sum over the winning pairs (cell, j) of i of (payload_j - constant) . W1[:, cell slab])

with base = b1 + constant . sum_k W1[:, k].  The test gives the kernels operands whose bits it knows:

  * social: hidden_dim_encoding is a 0/1 selection with a non-zero bias, so lat = fl32(h[:, sel] + b_enc) whatever
    order pool_prepare sums in (fast_lat path at H = 128 / C = 16 and the generic one), and a padded slot's latent row
    is b_enc itself; occupancy's payload is 1, directional's nan_to_num(fl32(v_j - v_i)), v = fl32(obs2 - obs1);
  * what the kernel multiplies is v = fl32(payload - constant): split into hi = rn_bf16(v), lo = rn_bf16(v - hi) for
    the mma kernel (the weights split the same way), the fp32 values themselves for the FFMA kernels;
  * base[o] = fl32(b1[o] + fl32(constant . s)), s the sequential fp32 sum of W1[o, :] (lstm_step.cu's k order);
  * the winners come from the restatement's last-writer rule (tests/torch_ref.py); its cells and in-range flags are
    asserted equal to the kernel's own (tb2_grid_indices), so no cell-boundary disagreement can pose as arithmetic.

The gate is per element.  sparse_layer1_mma: |Y - Y64| <= C_ACC . S, Y64 the float64 sum of hi_a.hi_w + hi_a.lo_w +
lo_a.hi_w over the row's winning pairs plus the base, S the same sum of absolute values plus |base|.  The FFMA kernels:
(terms + 1) u S with fp32 operands, terms = winners x C fused multiply-adds into the row.  dense_grid: bit for bit.
One_layer models, so the output is ReLU(layer 1); every case runs with (W1, b1) and with (-W1, -b1): rounding to nearest
is sign-symmetric and the base negates exactly, so every pre-activation is seen on the positive side of the ReLU once;
where the float64 value is below -gate the output must be exactly 0.

Probe rows (pair scenes: an observer with one neighbour in a chosen cell other than cell 0, all else out of range)
have exactly one winning pair, so their output is base + slab(cell) . lat_j and a fault confined to one tile, one pass,
one ring slot, one n-tile or one lane moves a probe by a large part of its own S.

CPU (no device needed):
  * test_case_table_coverage: the table's own coverage (kernels x constants, cell runs, tiles per CTA mod kMmaDepth,
    groupings, OUTs, column chunks, CH of pool_rows, probes, benc rows, nm1 <= 0) from the restatement's winners and a
    restatement of the host's launch choices;
  * test_mma_emulation_inside_gate: a numpy emulation of sparse_layer1_mma's arithmetic (per tile the 3-pass product
    from +0 in fp32, rounded to nearest and truncated, tiles added in ascending cell order) stays within a quarter of
    the gate on every case of the GPU table; test_ffma_emulation_inside_gate: the FFMA kernels' fma chains, in ascending
    cell order and in winner-list order, stay inside theirs (a worst-case bound, which short chains can approach);
  * test_mma_emulated_faults_fail_gate / test_ffma_emulated_faults_fail_gate: each emulated fault fails by >= 4x;
  * test_operand_restatement: lat, payloads and base as the kernels form them;
  * test_oracle_constant_matches_reference: the oracle's pool_constant pinned to the reference (needs_reference).

GPU, each case with the tensor cores on and with TB2_DISABLE_TC=1:
  * test_layer1_matches_float64: the kernel by name (tb2_profile_*), the winners, the per-element gate, both signs,
    a bit-identical rerun;
  * test_layer1_rows_move_bit_identical: a scene's rows keep their bits in another group, at another position in its
    group and under the other grouping;
  * test_layer1_writes_stay_inside_output: tb2_pool_forward through ctypes into an oversized NaN-sentinel buffer;
  * test_forward_with_pool_constant: LSTM.forward against the oracle at 1e-4 m with pool_constant = 1.
"""
import ctypes
import functools
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_hidden_dim import _profiled, _set_tc  # noqa: E402
from test_wgmma_kernels import SENTINEL, bf16_rn, split  # noqa: E402

F32, F64 = np.float32, np.float64
U = 2.0 ** -24                  # fp32 unit roundoff
C_ACC = 2.0 ** -16              # per-element gate of sparse_layer1_mma's fp32 accumulation, relative to S
MARGIN = 4.0
MMA_DEPTH = 8                   # kMmaDepth: B fragment sets in flight
SMEM_LIMIT = 227 * 1024
LAYER1_KERNELS = {"sparse_layer1_mma", "sparse_layer1", "pool_rows", "dense_grid"}


# ---------------------------------------------------------------------------------------------------------------------
# the host's launch choices (pool.cu: launch_pool_mlp, l1_mma_smem_bytes, l1_smem_bytes, pool_rows_chunk)
# ---------------------------------------------------------------------------------------------------------------------
def mma_smem(cap, cells, nm1):
    tiles = (cap * nm1 + 15 * cells) // 16
    b = cap * 260 * 4 + (cap + 2) * 64 + (2 * cells + 1) * 4 + ((tiles + 1) & ~1) * 2 + (16 * tiles + 16 * 10) * 2
    return b + cap * nm1 * 4 + cap * 8 + 16


def ffma_smem(cap, C, social, cells, nm1):
    b = cap * 256 * 4 + ((cap + 1) * C * 4 if social else 0) + (4 * cells + 1) * 4
    b += (cap * nm1 * 4 + 15) & ~15
    if not social:
        b += cap * nm1 * C * 4
    return b + cap * nm1 * 4 + cap * 8 + 16


def rows_chunk(m):
    if m["type"] == "social" or m["C"] > 2:
        return 0
    KW = m["cells"] * m["C"]
    for ch in (256, 128, 64, 32):
        if ch > 32 and ch // 2 >= m["OUT"]:
            continue
        if KW * ch * 4 <= 160 * 1024:
            return ch
    return 0


def kernel_of(m, tc):
    if m["arch"] is None:
        return "dense_grid"
    if rows_chunk(m):
        return "pool_rows"
    if m["type"] == "social" and m["C"] == 16 and tc:
        return "sparse_layer1_mma"
    return "sparse_layer1"


def groups_of(sizes, cap):
    """Scene groups of the layout at one cap (capi.cu: tb2_layout_create): lists of scene indices."""
    cap = max(cap, max(sizes))
    out, cur, rows = [], [], 0
    for b, n in enumerate(sizes):
        if rows + n > cap and cur:
            out.append(cur)
            cur, rows = [], 0
        cur.append(b)
        rows += n
    out.append(cur)
    return out, cap


def ffma_refuses(m, sizes):
    """sparse_layer1 (FFMA) refuses a batch whose scene groups do not fit its shared memory."""
    n_max = max(sizes)
    cap = grouping(m, sizes, "sparse_layer1")[1]
    return ffma_smem(cap, m["C"], m["type"] == "social", m["cells"], max(n_max - 1, 1)) > SMEM_LIMIT


def grouping(m, sizes, kernel):
    """(groups, cap, which) of the scene grouping the kernel runs on."""
    n_max = max(sizes)
    nm1 = max(n_max - 1, 1)
    if kernel == "sparse_layer1_mma":
        which = 0 if mma_smem(max(160, n_max), m["cells"], nm1) <= SMEM_LIMIT else 1
    else:
        which = 0 if -(-m["OUT"] // 256) >= 4 else 1
        if which == 0 and ffma_smem(max(160, n_max), m["C"], m["type"] == "social", m["cells"], nm1) > SMEM_LIMIT:
            which = 1
    groups, cap = groups_of(sizes, (160, 40)[which])
    return groups, cap, which


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def model(type_, n, side, OUT, C=None, H=128, arch="one_layer", front=False):
    C = {"occupancy": 1, "directional": 2}.get(type_, C)
    return dict(type=type_, n=n, side=side, OUT=OUT, C=C, H=H, arch=arch, front=front, cells=n * n)


def cell_offset(m, a, b):
    """The relative position that lands in the middle of cell (a, b)."""
    offy = 0.0 if m["front"] else m["n"] / 2
    return np.array([(a + 0.5 - m["n"] / 2) * m["side"], (b + 0.5 - offy) * m["side"]])


def _probe_cells(m):
    """Cells (a, b) for pair scenes: neither the cell, its mirror, cell 0 nor the centre cell (where absent
    pedestrians' padded slots land) repeat."""
    n = m["n"]
    taken = {(0, 0), (n // 2, n // 2), (n // 2 - 1, n // 2 - 1)}
    out = []
    for a in range(1, n - 1):
        for b in range(1, n - 1):
            mirror = (n - 1 - a, n - 1 - b)
            if (a, b) in taken or mirror in taken or (a, b) == mirror:
                continue
            taken |= {(a, b), mirror}
            out.append((a, b))
    return out


class Batch:
    """Scenes as [n_s, 2] obs1 / obs2 arrays; `kind` of each scene for the coverage checks."""

    def __init__(self, m, seed):
        self.m, self.rng = m, np.random.default_rng(seed)
        self.obs1, self.obs2, self.kinds = [], [], []
        self.far = 4.0 * m["n"] * m["side"] + 10.0          # out of range of each other
        self.where = 0

    def _origin(self):
        self.where += 1
        return np.array([self.where * 3.7 % 97.0 - 48.0, self.where * 7.3 % 89.0 - 44.0])

    def _add(self, o2, kind, absent=()):
        o2 = np.asarray(o2, F64)
        o1 = o2 - self.rng.normal(0, 0.3, size=o2.shape)
        o2, o1 = o2.astype(F32), o1.astype(F32)
        for r in absent:
            o2[r] = np.nan
        self.obs1.append(o1)
        self.obs2.append(o2)
        self.kinds.append(kind)

    def pair(self, cell, count=1):
        """count scenes of an observer and one neighbour in the middle of `cell` (the neighbour sees the observer
        in the mirror cell): a run of `count` pairs in each of the two cells, every row a probe."""
        off = cell_offset(self.m, *cell)
        for _ in range(count):
            p = self._origin()
            self._add([p, p + off], "pair")

    def crowd(self, k, absent=0, spread=0.7):
        p = self._origin()
        w = self.m["n"] * self.m["side"] * spread
        self._add(p + self.rng.uniform(-w / 2, w / 2, size=(k, 2)), "crowd", absent=range(1, 1 + absent))

    def inert(self, k):
        p = self._origin()
        self._add([p + [q * self.far, 0.0] for q in range(k)], "inert")

    def absent_single(self):
        self._add([[0.0, 0.0]], "absent", absent=[0])

    def fill(self, rows, cap, n_max):
        """inert scenes of <= n_max tracks up to `cap` rows since the last multiple of cap."""
        left = cap - rows
        while left > 0:
            k = min(left, n_max)
            self.inert(k)
            left -= k

    @property
    def sizes(self):
        return [len(o) for o in self.obs2]


def batch_mix(m, seed, n_max=12):
    """Cap-160 groups: cell runs of 1, 15, 16, 17 / 32, 33 / 48 pairs; crowds with absent pedestrians (benc rows);
    16 groups of exactly t tiles, t = 0 .. 15 (pair scenes at distinct cells, two tiles each, and an absent
    pedestrian's padded-slot winner at the centre cell for odd t); groups filled to 160 rows with inert scenes."""
    bt = Batch(m, seed)
    cells = _probe_cells(m)
    take = iter(cells)
    for runs in ((1, 15, 16, 17), (32, 33), (48,)):
        for r in runs:
            bt.pair(next(take), r)
        bt.fill(2 * sum(runs), 160, n_max)
    for _ in range(2):
        rows = 0
        for k in (n_max, 9, 11, n_max, 7, 10, n_max, 8, 12, 6, n_max, 5, 9):
            k = min(k, n_max)
            bt.crowd(k, absent=2 if k < n_max else 0)
            rows += k
        bt.fill(rows, 160, n_max)
    for t in range(16):
        cs = cells[len(cells) - t // 2:]
        for c in cs:
            bt.pair(c)
        if t % 2:
            bt.absent_single()
        bt.fill(2 * len(cs) + t % 2, 160, n_max)
    bt.crowd(n_max)
    return bt


def batch_wide(m, seed, n_max=60):
    """A scene of n_max tracks: the mma kernel's shared memory no longer fits cap-160 groups (cap = n_max)."""
    bt = Batch(m, seed)
    bt.crowd(n_max, absent=0, spread=1.2)
    cells = _probe_cells(m)
    bt.pair(cells[0], 17)
    bt.pair(cells[1], 1)
    for k in (9, 12, 5):
        bt.crowd(k, absent=1)
    bt.absent_single()
    bt.crowd(n_max - 1, absent=3, spread=0.9)
    bt.inert(7)
    return bt


def batch_single(m, seed):
    """Every scene one track (nm1 <= 0): every output is ReLU(base)."""
    bt = Batch(m, seed)
    for i in range(37):
        bt._add([bt._origin()], "single", absent=[0] if i % 5 == 2 else [])
    return bt


def batch_big(m, seed, n_max):
    """The largest scene the launch takes next to pair scenes, crowds and absent pedestrians."""
    bt = Batch(m, seed)
    bt.crowd(n_max, absent=4, spread=1.5)
    cells = _probe_cells(m)
    bt.pair(cells[2], 16)
    bt.pair(cells[3], 3)
    for k in (20, 11, 3):
        bt.crowd(k, absent=1)
    bt.absent_single()
    return bt


def batch_rows(m, seed, n_max=120):
    """Many rows with long winner lists: pool_rows's rows per CTA bounded by its shared memory."""
    bt = Batch(m, seed)
    for k in (n_max, 90, n_max, 70, n_max, 100, n_max, 60, n_max, 110, 40, 30):
        bt.crowd(k, absent=2, spread=1.0)
    cells = _probe_cells(m)
    bt.pair(cells[0], 5)
    bt.absent_single()
    return bt


def batch_small(m, seed):
    """Crowds of 6 .. 12 with absent pedestrians, pair scenes and an absent pedestrian alone."""
    bt = Batch(m, seed)
    cells = _probe_cells(m)
    for i, k in enumerate((12, 9, 11, 6, 12, 8, 10, 7, 12, 5, 11, 12)):
        bt.crowd(k, absent=1 + i % 2 if k < 12 else 0)
        bt.pair(cells[i % len(cells)], 1 + i % 3)
    bt.absent_single()
    return bt


BATCHES = {"mix": batch_mix, "wide": batch_wide, "single": batch_single, "small": batch_small,
           "rows": batch_rows, "big": lambda m, seed: batch_big(m, seed, largest_mma_scene(m["cells"]))}


def largest_mma_scene(cells):
    """The largest scene sparse_layer1_mma takes: cap-40 grouping (cap = n_max) within shared memory and 254 rows."""
    return max(n for n in range(2, 255) if mma_smem(max(40, n), cells, n - 1) <= SMEM_LIMIT)


# ---------------------------------------------------------------------------------------------------------------------
# case table
# ---------------------------------------------------------------------------------------------------------------------
SOC12 = dict(type_="social", n=12, side=0.6, C=16)
CASES = [
    # sparse_layer1_mma (sparse_layer1<16, true> without the tensor cores): every column chunk shape
    dict(m=model(OUT=8, **SOC12), batch="mix", const=0.0),
    dict(m=model(OUT=100, **SOC12), batch="mix", const=1.0),
    dict(m=model(OUT=203, **SOC12), batch="mix", const=-1.0),
    dict(m=model(OUT=256, **SOC12), batch="mix", const=0.0),
    dict(m=model(OUT=257, **SOC12), batch="mix", const=1.0),
    dict(m=model(OUT=520, **SOC12), batch="mix", const=-1.0),
    dict(m=model(OUT=256, **SOC12), batch="wide", const=1.0),
    dict(m=model(OUT=257, **SOC12), batch="wide", const=-1.0),
    dict(m=model(OUT=256, **SOC12), batch="single", const=1.0),
    dict(m=model(OUT=256, type_="social", n=16, side=0.5, C=16), batch="big", const=-1.0),
    dict(m=model(OUT=128, type_="social", n=12, side=0.6, C=16, H=64), batch="small", const=1.0),   # generic lat
    # sparse_layer1<C, true>
    dict(m=model(OUT=128, type_="social", n=12, side=0.6, C=4), batch="small", const=1.0),
    dict(m=model(OUT=203, type_="social", n=10, side=0.6, C=8), batch="small", const=-1.0),
    dict(m=model(OUT=520, type_="social", n=8, side=0.7, C=32), batch="small", const=0.0),
    dict(m=model(OUT=1024, type_="social", n=8, side=0.7, C=4), batch="small", const=-1.0),     # cap-160 groups
    # sparse_layer1<C, false>
    dict(m=model(OUT=64, type_="occupancy", n=36, side=0.3), batch="small", const=1.0),
    dict(m=model(OUT=64, type_="occupancy", n=36, side=0.3), batch="wide", const=-1.0),
    dict(m=model(OUT=64, type_="directional", n=26, side=0.4), batch="small", const=-1.0),
    dict(m=model(OUT=257, type_="directional", n=26, side=0.4), batch="small", const=0.0),
    dict(m=model(OUT=64, type_="directional", n=26, side=0.4), batch="single", const=1.0),
    # pool_rows: CH 256 / 128 / 64 / 32, OUT % 4 != 0, rows per CTA bounded by shared memory
    dict(m=model(OUT=256, type_="occupancy", n=12, side=0.6), batch="small", const=1.0),
    dict(m=model(OUT=203, type_="occupancy", n=12, side=0.6), batch="small", const=-1.0),
    dict(m=model(OUT=256, type_="directional", n=12, side=0.6), batch="small", const=-1.0),
    dict(m=model(OUT=256, type_="directional", n=16, side=0.6), batch="small", const=0.0),
    dict(m=model(OUT=256, type_="directional", n=24, side=0.6), batch="rows", const=1.0),
    dict(m=model(OUT=99, type_="occupancy", n=4, side=0.6, front=True), batch="small", const=1.0),
    # dense_grid
    dict(m=model(OUT=0, type_="social", n=8, side=0.6, C=8, arch=None), batch="small", const=1.0),
    dict(m=model(OUT=0, type_="occupancy", n=8, side=0.6, arch=None), batch="small", const=-1.0),
    dict(m=model(OUT=0, type_="directional", n=6, side=0.6, arch=None), batch="single", const=0.0),
]


def case_id(c):
    m = c["m"]
    return "%s-n%d-C%d-H%d-OUT%d-%s-c%+d" % (m["type"], m["n"], m["C"], m["H"], m["OUT"], c["batch"], c["const"])


def case_seed(c):
    return sum(ord(ch) * (i + 1) for i, ch in enumerate(case_id(c))) % 100003


# ---------------------------------------------------------------------------------------------------------------------
# operands and the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
def restated_pairs(obs2, m):
    """(oi, ok, win) [N, N-1] of one padded scene: cells binned in fp32 like torch_ref._grid, last writer wins."""
    N = len(obs2)
    if N <= 1:
        z = np.zeros((N, 0), np.int64)
        return z, z.astype(bool), z.astype(bool)
    obs = obs2.copy()
    obs[np.isnan(obs).any(-1)] = -500.0
    keep = ~np.eye(N, dtype=bool)
    rel = (obs[None, :, :] - obs[:, None, :])[keep].reshape(N, N - 1, 2)
    off = np.array([m["n"] / 2, 0.0 if m["front"] else m["n"] / 2], F32)
    oij = rel / F32(m["side"]) + off
    assert oij.dtype == F32
    ok = ~((oij < 0) | (oij >= m["n"])).any(-1)
    o = np.where(ok[..., None], oij, 0).astype(np.int64)
    oi = o[..., 0] * m["n"] + o[..., 1]
    later = np.triu(np.ones((N - 1, N - 1), bool), 1)
    win = ~((oi[:, :, None] == oi[:, None, :]) & later).any(-1)
    return oi, ok, win & ok


class Operands:
    """Everything one case multiplies, as the kernels form it."""

    def __init__(self, case, sign=1.0, pad=True):
        m = self.m = case["m"]
        bt = BATCHES[case["batch"]](m, case_seed(case))
        self.kinds = bt.kinds
        self.sizes = sizes = bt.sizes
        self.off = np.concatenate([[0], np.cumsum(sizes)])
        self.M = M = int(self.off[-1])
        self.n_max = n_max = max(sizes)
        self.nm1 = max(n_max - 1, 1)
        self.const = F32(case["const"])
        self.obs1 = np.concatenate(bt.obs1)
        self.obs2 = np.concatenate(bt.obs2)
        rng = np.random.default_rng(case_seed(case) + 1)
        C, H, cells = m["C"], m["H"], m["cells"]
        self.C, self.cells = C, cells
        # weights
        self.W = {}
        if m["type"] == "social":
            sel = rng.choice(H, C, replace=False)
            We = np.zeros((C, H), F32)
            We[np.arange(C), sel] = 1
            self.benc = (rng.choice([-1, 1], C) * rng.uniform(0.3, 1.5, C)).astype(F32)
            self.W["hidden_dim_encoding.weight"], self.W["hidden_dim_encoding.bias"] = We, self.benc
            self.hidden = (rng.choice([-1, 1], (M, H)) * rng.uniform(0.25, 2.0, (M, H))).astype(F32)
            self.lat = (self.hidden[:, sel] + self.benc).astype(F32)
        else:
            self.hidden = None
        self.OUT = m["OUT"] if m["arch"] else C * cells
        if m["arch"]:
            K = C * cells
            self.W1 = (rng.standard_normal((self.OUT, K)) * (sign * 0.5 / math.sqrt(C))).astype(F32)
            self.b1 = (rng.standard_normal(self.OUT) * sign * 0.3).astype(F32)
            self.W["embedding.0.weight"], self.W["embedding.0.bias"] = self.W1, self.b1
            s = np.zeros(self.OUT, F32)
            for k in range(K):              # lstm_step.cu repack_layer1_kernel: sequential fp32 sum in k order
                s = (s + self.W1[:, k]).astype(F32)
            self.base = (self.b1 + (self.const * s).astype(F32)).astype(F32)
            self.Wt = np.ascontiguousarray(self.W1.reshape(self.OUT, C, cells).transpose(2, 1, 0))   # [cell, c, o]
        # winners in the kernel's row tables: slot jj of row i is neighbour jj + (jj >= i) of its padded scene
        nm1 = self.nm1
        self.pair_cell = np.zeros((M, nm1), np.int32)
        self.pair_flag = np.zeros((M, nm1), np.uint8)
        rows_w = []
        vel = (self.obs2 - self.obs1).astype(F32)
        for b, n_s in enumerate(sizes):
            r0 = self.off[b]
            N = n_max if pad else n_s
            o2 = np.full((N, 2), np.nan, F32)
            o2[:n_s] = self.obs2[r0:r0 + n_s]
            oi, ok, win = restated_pairs(o2, m)
            w = N - 1
            self.pair_cell[r0:r0 + n_s, :w] = np.where(ok[:n_s], oi[:n_s], 0)
            self.pair_flag[r0:r0 + n_s, :w] = ok[:n_s]
            for i in range(n_s):
                lst = []
                for jj in np.nonzero(win[i])[0]:
                    j = jj + (jj >= i)
                    lst.append((int(oi[i, jj]), int(r0 + j) if j < n_s else -1, r0 + i))
                rows_w.append(lst)
        self.Wmax = Wmax = max(1, max(len(x) for x in rows_w))
        self.count = np.array([len(x) for x in rows_w])
        self.wcell = np.full((M, Wmax), -1, np.int64)     # winners in the kernel's jj order
        self.wsrc = np.full((M, Wmax), -2, np.int64)      # global row of the neighbour, -1: padded slot (benc)
        self.pay = np.zeros((M, Wmax, C), F32)            # payload (lat / 1 / relative velocity)
        for i, lst in enumerate(rows_w):
            for k, (cell, j, _) in enumerate(lst):
                self.wcell[i, k], self.wsrc[i, k] = cell, j
                if m["type"] == "social":
                    self.pay[i, k] = self.benc if j < 0 else self.lat[j]
                elif m["type"] == "occupancy":
                    self.pay[i, k] = 1
                else:
                    vj = vel[j] if j >= 0 else np.full(2, np.nan, F32)
                    with np.errstate(invalid="ignore"):
                        self.pay[i, k] = np.nan_to_num((vj - vel[i]).astype(F32))
        self.has = self.wcell >= 0
        self.v = np.where(self.has[..., None], (self.pay - self.const).astype(F32), 0).astype(F32)
        # the same winners in ascending cell order (the order sparse_layer1 / sparse_layer1_mma accumulate in)
        order = np.argsort(np.where(self.has, self.wcell, 1 << 30), axis=1, kind="stable")
        self.cell_order = order
        self.probes = np.nonzero((self.count == 1) & (self.wcell[:, 0] > 0))[0]

    # -- the float64 oracle ----------------------------------------------------------------------------------------
    def dense_grid(self):
        """The grid itself [M, C * cells] (embedding None): constant, winners' payloads (lat unshifted)."""
        g = np.full((self.M, self.C, self.cells), self.const, F32)
        rows, ks = np.nonzero(self.has)
        g[rows, :, self.wcell[rows, ks]] = self.pay[rows, ks]
        return g.reshape(self.M, -1)

    def oracle(self, mma, dev="cpu"):
        """float64 (Y64, S) [M, OUT] of the pre-activation; mma: of the bf16 (hi, lo) 3-pass product."""
        M, C, cells = self.M, self.C, self.cells
        rows, ks = np.nonzero(self.has)
        cols = self.wcell[rows, ks]
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev).double()     # noqa: E731
        W = t(self.W1)
        base = t(self.base)

        def grid(v):
            g = torch.zeros(M, C, cells, dtype=torch.float64, device=dev)
            g[torch.from_numpy(rows).to(dev), :, torch.from_numpy(cols).to(dev)] = t(v[rows, ks])
            return g.reshape(M, -1)
        if mma:
            vh, vl = split(self.v)
            wh, wl = (t(x) for x in split(self.W1))
            gh, gl = grid(vh), grid(vl)
            y = gh @ wh.T + gh @ wl.T + gl @ wh.T + base
            s = gh.abs() @ wh.abs().T + gh.abs() @ wl.abs().T + gl.abs() @ wh.abs().T + base.abs()
        else:
            g = grid(self.v)
            y, s = g @ W.T + base, g.abs() @ W.abs().T + base.abs()
        return y, s

    def gate(self, S, mma):
        if mma:
            return C_ACC * S
        terms = torch.from_numpy(self.count * self.C).to(S.device).double()[:, None]
        return (terms + 1) * U * S


# ---------------------------------------------------------------------------------------------------------------------
# numpy emulations of the kernels' arithmetic
# ---------------------------------------------------------------------------------------------------------------------
def _round(s, rounding):
    r = s.astype(F32)
    if rounding == "rz":
        over = np.abs(r.astype(F64)) > np.abs(s)
        r[over] = np.nextafter(r[over], F32(0))
    return r


def tile_lists(op, kernel):
    """Per CTA (scene group): its tiles in the kernel's order as (cell, [rows]) -- the cell's pairs in 16-row tiles in
    ascending cell order (the order of pairs inside a cell is not fixed; rows ascending here)."""
    groups, _, _ = grouping(op.m, op.sizes, kernel)
    out = []
    for g in groups:
        r0, r1 = op.off[g[0]], op.off[g[-1] + 1]
        by_cell = {}
        for r in range(r0, r1):
            for k in range(op.count[r]):
                by_cell.setdefault(int(op.wcell[r, k]), []).append(r)
        tiles = []
        for c in sorted(by_cell):
            rs = by_cell[c]
            tiles += [(c, rs[i:i + 16]) for i in range(0, len(rs), 16)]
        out.append(tiles)
    return out


def emulate_mma(op, rows, rounding="rn", fault=None):
    """sparse_layer1_mma on `rows`: per winning pair (one tile row) the 3-pass product summed from +0 in fp32, the
    tiles added to the row's accumulator (from the base) in ascending cell order; ReLU.  fault: (name, arg)."""
    name, arg = fault if fault else (None, None)
    v = op.v[rows].copy()
    if name == "benc_zero_row":            # a padded neighbour's slot reads the zero row instead of b_enc
        v[op.wsrc[rows] == -1] = 0
    if name == "benc_no_constant":         # b_enc staged without - constant
        v[op.wsrc[rows] == -1] = op.benc
    vh, vl = split(v)
    wh, wl = split(op.Wt)
    base = op.b1 if name == "base_no_constant" else op.base
    acc = np.broadcast_to(base, (len(rows), op.OUT)).astype(F32)
    for kk in range(op.Wmax):
        k = op.cell_order[rows, kk]
        ri = np.arange(len(rows))
        cell = op.wcell[rows, k]
        live = cell >= 0
        cw = np.where(live, cell, 0)
        wc = cw.copy()
        if name == "stale_ring":           # tile (cell, rows) reads the slab of the cell eight tiles earlier
            cell_t, rows_t, prev = arg
            hit = live & (cell == cell_t) & np.isin(rows, rows_t)
            wc[hit] = prev
        a_h, a_l = vh[ri, k], vl[ri, k]
        d = np.zeros((len(rows), op.OUT), F32)
        for p, (a, w) in enumerate(((a_h, wh), (a_h, wl), (a_l, wh))):
            prod = np.einsum("mc,mco->mo", a.astype(F64), w[wc].astype(F64))
            if name == "no_lo_a" and p == 2:
                cell_t, rows_t = arg
                prod[live & (cell == cell_t) & np.isin(rows, rows_t)] = 0
            d = _round(d.astype(F64) + prod, rounding)
        if name == "drop_pair":
            d[live & (cell == arg[0]) & (rows == arg[1])] = 0
        d[~live] = 0
        acc = _round(acc.astype(F64) + d, rounding)
    y = np.maximum(acc, 0)
    if name == "chunk_shift":              # the last partial chunk's columns read one column further
        c0 = (op.OUT - 1) // 256 * 256
        y[:, c0:op.OUT - 1] = y[:, c0 + 1:op.OUT]
        y[:, op.OUT - 1] = 0
    return y


def emulate_ffma(op, rows, order="cell", fault=None):
    """The FFMA kernels on `rows`: from the base, one fp32 fma per (winner, channel); winners in ascending cell order
    (sparse_layer1) or in the row's list order (pool_rows); ReLU."""
    name, arg = fault if fault else (None, None)
    acc = np.broadcast_to(op.base, (len(rows), op.OUT)).astype(F32)
    ri = np.arange(len(rows))
    for kk in range(op.Wmax):
        k = op.cell_order[rows, kk] if order == "cell" else np.full(len(rows), kk)
        cell = op.wcell[rows, k]
        live = cell >= 0
        if name == "skip_winner":
            live = live & ~((rows == arg) & (kk == 0))
        w = op.Wt[np.where(live, cell, 0)]
        for c in range(op.C):
            prod = op.v[rows, k, c].astype(F64)[:, None] * w[:, c].astype(F64)
            acc = np.where(live[:, None], (acc.astype(F64) + prod).astype(F32), acc)
    if name == "row_at_base":              # a parity half left one row at its base
        acc[rows == arg] = op.base
    return np.maximum(acc, 0)


def gate_ratio(op, rows, y, mma):
    ref, S = op.oracle(mma)
    ref, S = ref.numpy()[rows], S.numpy()[rows]
    gate = op.gate(torch.from_numpy(S), mma).numpy() if mma else \
        ((op.count[rows] * op.C + 1)[:, None] * U * S)
    return float(np.max(np.abs(y.astype(F64) - np.maximum(ref, 0)) / gate))


def emulation_rows(op, limit=400):
    """Rows to emulate: every probe, every row with a padded-slot winner, the busiest rows, and some more."""
    busy = np.argsort(-op.count, kind="stable")[:limit // 2]
    benc = np.nonzero((op.wsrc == -1).any(1))[0]
    rest = np.arange(0, op.M, max(1, op.M // (limit // 4)))
    return np.unique(np.concatenate([op.probes[:limit // 4], benc, busy, rest]))


@functools.lru_cache(maxsize=None)
def operands(i, sign=1.0, pad=True):
    return Operands(CASES[i], sign, pad)


EMB = [i for i, c in enumerate(CASES) if c["m"]["arch"]]
MMA = [i for i in EMB if kernel_of(CASES[i]["m"], True) == "sparse_layer1_mma"]


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_case_table_coverage():
    kc = {}
    for c in CASES:
        for tc in (True, False):
            kc.setdefault(kernel_of(c["m"], tc), set()).add(c["const"])
    assert set(kc) == LAYER1_KERNELS
    for k, consts in kc.items():
        assert consts == {0.0, 1.0, -1.0}, (k, consts)
    runs, residues, groupings, outs = set(), set(), set(), set()
    empty_group = benc = single = False
    for i in MMA:
        op = operands(i)
        outs.add(op.OUT)
        _, _, which = grouping(op.m, op.sizes, "sparse_layer1_mma")
        groupings.add(which)
        for tiles in tile_lists(op, "sparse_layer1_mma"):
            residues.add(len(tiles) if len(tiles) < MMA_DEPTH else MMA_DEPTH + len(tiles) % MMA_DEPTH)
            cnt = {}
            for cell, rs in tiles:
                cnt[cell] = cnt.get(cell, 0) + len(rs)
            runs |= set(cnt.values())
            empty_group |= not tiles
        benc |= bool((op.wsrc == -1).any())
        single |= op.n_max == 1
        assert len(op.probes) >= 1 or op.n_max == 1
    assert {1, 15, 16, 17, 32, 33} <= runs and max(runs) >= 48, sorted(runs)
    assert set(range(MMA_DEPTH)) <= residues and {MMA_DEPTH + r for r in range(MMA_DEPTH)} <= residues, residues
    assert empty_group and benc and single and groupings == {0, 1}
    assert {8, 100, 203, 256, 257, 520} <= outs
    big = [operands(i) for i in MMA if CASES[i]["batch"] == "big"]
    assert big and big[0].cells == 256 and big[0].n_max == largest_mma_scene(256)
    assert ffma_refuses(big[0].m, big[0].sizes)           # without the tensor cores the same batch is refused
    assert mma_smem(largest_mma_scene(256) + 1, 256, largest_mma_scene(256)) > SMEM_LIMIT
    assert any(CASES[i]["m"]["H"] != 128 for i in MMA)                       # pool_prepare's generic latent path
    # sparse_layer1<C, true> / <C, false>, pool_rows
    ffma_social = {(c["m"]["C"], c["m"]["OUT"]) for c in CASES
                   if c["m"]["type"] == "social" and kernel_of(c["m"], False) == "sparse_layer1"}
    assert {4, 8, 16, 32} <= {C for C, _ in ffma_social}
    assert any(o % 2 for _, o in ffma_social) and any(o > 512 for _, o in ffma_social)
    assert any(-(-o // 256) >= 4 for _, o in ffma_social)                      # cap-160 groups
    payload = {(c["m"]["type"], c["m"]["n"]) for c in CASES if kernel_of(c["m"], True) == "sparse_layer1"
               and c["m"]["type"] != "social"}
    assert {("occupancy", 36), ("directional", 26)} <= payload
    rows = [c for c in CASES if kernel_of(c["m"], True) == "pool_rows"]
    assert {rows_chunk(c["m"]) for c in rows} == {256, 128, 64, 32}
    assert any(c["m"]["OUT"] % 4 for c in rows)
    big_rows = [operands(CASES.index(c)) for c in rows if c["batch"] == "rows"]
    assert big_rows and big_rows[0].M > _rows_per_cta(big_rows[0])
    dense = {c["m"]["type"] for c in CASES if c["m"]["arch"] is None}
    assert {"social", "occupancy"} <= dense


def _rows_per_cta(op):
    ch = rows_chunk(op.m)
    chunks = -(-op.OUT // ch)
    groups = -(-148 // chunks)
    rows = -(-op.M // groups)
    per_row = 4 + op.nm1 * 12
    return max(1, min(rows, (220 * 1024 - op.cells * op.C * ch * 4) // per_row))


def test_operand_restatement():
    """lat, payloads and base as the kernels form them: a 0/1 encoding sums exactly in any order, fl32(v - constant)
    splits into bf16 (hi, lo) exactly, and the base's constant term is exact at constant = +-1."""
    op = operands(MMA[1])
    H = op.m["H"]
    We = op.W["hidden_dim_encoding.weight"]
    lat = np.zeros((op.M, op.C), F32)
    for k in range(H):                      # any summation order gives h[sel]
        lat = (lat + op.hidden[:, k:k + 1] * We[:, k]).astype(F32)
    assert np.array_equal((lat + op.benc).astype(F32), op.lat)
    hi, lo = split(op.v)
    assert (np.abs(op.v.astype(F64) - hi - lo) <= np.abs(op.v) * 2.0 ** -16).all()
    assert np.array_equal(bf16_rn(hi), hi) and np.array_equal(bf16_rn(lo), lo)
    assert op.const == 1 and not np.array_equal(op.base, op.b1)
    neg = Operands(CASES[MMA[1]], sign=-1.0)
    assert np.array_equal(neg.base, -op.base)
    assert np.array_equal(neg.v, op.v) and np.array_equal(neg.W1, -op.W1)


@pytest.mark.parametrize("rounding", ["rn", "rz"])
def test_mma_emulation_inside_gate(rounding):
    for i in MMA:
        op = operands(i)
        rows = emulation_rows(op)
        r = gate_ratio(op, rows, emulate_mma(op, rows, rounding), True)
        print("mma emulation [%s] %s: err / gate %.3f" % (rounding, case_id(CASES[i]), r))
        assert r * MARGIN <= 1.0, (case_id(CASES[i]), r)


@pytest.mark.parametrize("order", ["cell", "list"])
def test_ffma_emulation_inside_gate(order):
    for i in EMB:
        op = operands(i)
        rows = emulation_rows(op, 200)
        r = gate_ratio(op, rows, emulate_ffma(op, rows, order), False)
        print("ffma emulation [%s] %s: err / gate %.3f" % (order, case_id(CASES[i]), r))
        # (terms + 1) u S bounds any order of the row's fma chain; a short chain (a probe's C terms) can come close
        assert r <= 1.0, (case_id(CASES[i]), r)


def _fault_case():
    """The mma case with a partial last chunk, pool_constant 1 and cap-160 groups of >= 9 tiles."""
    i = next(i for i in MMA if CASES[i]["batch"] == "mix" and CASES[i]["const"] == 1.0 and CASES[i]["m"]["OUT"] % 256)
    return i, operands(i)


def test_mma_emulated_faults_fail_gate():
    i, op = _fault_case()
    lists = tile_lists(op, "sparse_layer1_mma")
    probe = int(op.probes[0])
    pc = int(op.wcell[probe, 0])
    tiles = next(t for t in lists if len(t) > MMA_DEPTH and any(pc == c for c, _ in t))
    k = next(k for k, (c, rs) in enumerate(tiles) if c == pc and probe in rs)
    if k < MMA_DEPTH or tiles[k - MMA_DEPTH][0] == pc:
        k = next(k for k in range(MMA_DEPTH, len(tiles)) if tiles[k][0] != tiles[k - MMA_DEPTH][0])
    stale_cell, stale_rows = tiles[k]
    run = next(rs for c, rs in tiles if len(rs) >= 9)
    g8 = run[8]
    faults = {
        "no_lo_a": ("no_lo_a", (pc, [probe])),
        "drop_pair": ("drop_pair", (int(op.wcell[g8][op.wcell[g8] >= 0][0]) if op.count[g8] == 1 else
                                    next(int(c) for c in op.wcell[g8] if c >= 0), g8)),
        "stale_ring": ("stale_ring", (stale_cell, stale_rows, tiles[k - MMA_DEPTH][0])),
        "benc_zero_row": ("benc_zero_row", None),
        "benc_no_constant": ("benc_no_constant", None),
        "base_no_constant": ("base_no_constant", None),
        "chunk_shift": ("chunk_shift", None),
    }
    rows = emulation_rows(op)
    rows = np.unique(np.concatenate([rows, [probe, g8], stale_rows]))
    for name, fault in faults.items():
        r = gate_ratio(op, rows, emulate_mma(op, rows, "rn", fault), True)
        print("mma fault %-16s %s: err = %.0f x gate" % (name, case_id(CASES[i]), r))
        assert r >= MARGIN, (name, r)


# occupancy at constant 1: every winner's v = 1 - 1 is 0 (an occupied cell holds the constant), no winner to lose
FFMA_FAULT_CASES = [i for i in EMB if CASES[i]["batch"] != "single" and
                    not (CASES[i]["m"]["type"] == "occupancy" and CASES[i]["const"] == 1.0)][::3]


@pytest.mark.parametrize("i", FFMA_FAULT_CASES, ids=[case_id(CASES[i]) for i in FFMA_FAULT_CASES])
def test_ffma_emulated_faults_fail_gate(i):
    op = operands(i)
    probe = int(op.probes[0])
    rows = np.unique(np.concatenate([emulation_rows(op, 100), [probe]]))
    for name in ("skip_winner", "row_at_base"):
        r = gate_ratio(op, rows, emulate_ffma(op, rows, "cell", (name, probe)), False)
        print("ffma fault %-12s %s: err = %.0f x gate" % (name, case_id(CASES[i]), r))
        assert r >= MARGIN, (name, r)


E2E_KINDS = ("social_default", "social", "occupancy_n36", "occupancy_raw")


def _pool_config_const(kind, constant):
    from oracle import lstm_oracle as O
    return O.PoolConfig(**dict(O.MODEL_SPECS[kind], constant=constant))


@pytest.mark.needs_reference
@pytest.mark.parametrize("kind", E2E_KINDS)
def test_oracle_constant_matches_reference(kind):
    """The oracle's pool_constant (out-of-range and empty cells hold it) against the reference, on ragged scenes with
    NaN tracks."""
    from oracle import lstm_oracle as O
    from oracle.ref_shim import import_reference
    import_reference()
    from trajnetbaselines.lstm import LSTM as RefLSTM, GridBasedPooling as RefPool
    xy, bs = O.synthetic_scenes(6, 9, seed=41, ragged=True, nan_tracks=True)
    W = O.random_weights(kind, seed=7, relu_bias=3.0)
    model = RefLSTM(embedding_dim=64, pool=RefPool(**dict(O.MODEL_SPECS[kind], constant=1)))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    model.eval()
    with torch.no_grad():
        _, pred = model(torch.from_numpy(xy[:9]), torch.zeros(xy.shape[1], 2), torch.from_numpy(bs), n_predict=12)
    _, pred_o = O.forward(W, _pool_config_const(kind, 1.0), xy[:9], bs, n_predict=12)
    _, pred_0 = O.forward(W, _pool_config_const(kind, 0.0), xy[:9], bs, n_predict=12)
    assert (np.isnan(pred.numpy()) == np.isnan(pred_o)).all()
    assert np.nanmax(np.abs(pred.numpy() - pred_o)) < 2e-5
    assert np.nanmax(np.abs(pred_0 - pred_o)) > 1e-3           # the constant changes the forecast


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _pool(op, dev):
    from trajnetplusplusbaselines_b200.lstm import GridBasedPooling
    m = op.m
    kw = dict(type_=m["type"], n=m["n"], cell_side=m["side"], hidden_dim=m["H"], front=m["front"],
              embedding_arch=m["arch"] if m["arch"] else "None", constant=float(op.const))
    if m["arch"]:
        kw["out_dim"] = m["OUT"]
    if m["type"] == "social":
        kw["latent_dim"] = m["C"]
    pool = GridBasedPooling(**kw)
    pool.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in op.W.items()}, strict=True)
    return pool.to(dev)


def _inputs(op, dev):
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)     # noqa: E731
    return (f(op.hidden) if op.hidden is not None else None), f(op.obs1), f(op.obs2)


def _run(op, pool, layout, dev):
    handle = pool._plug_handle(dev)
    hid, o1, o2 = _inputs(op, dev)
    out, kernels = _profiled(lambda: handle.pool_forward(layout, hid, o1, o2, op.OUT))
    torch.cuda.synchronize(dev)
    return out, kernels & LAYER1_KERNELS


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("i", range(len(CASES)), ids=[case_id(c) for c in CASES])
def test_layer1_matches_float64(monkeypatch, i, tc):
    from trajnetplusplusbaselines_b200.engine import SceneLayout
    _set_tc(monkeypatch, tc)
    dev = torch.device("cuda", 0)
    op = operands(i)
    kernel = kernel_of(op.m, tc)
    mma = kernel == "sparse_layer1_mma"
    layout = SceneLayout([int(x) for x in op.off], device=dev)
    pool = _pool(op, dev)
    # the kernel's winners: the restatement's cells and in-range flags
    if op.n_max > 1:
        cells, flags = pool._plug_handle(dev).grid_indices(layout, _inputs(op, dev)[2])
        assert np.array_equal(flags.cpu().numpy(), op.pair_flag)
        assert np.array_equal(cells.cpu().numpy(), op.pair_cell)
    if kernel == "sparse_layer1" and ffma_refuses(op.m, op.sizes):
        # the largest scene of the tensor-core kernel: the FFMA kernel's groups do not fit, refused before any launch
        with pytest.raises(RuntimeError, match="does not fit in shared memory"):
            _run(op, pool, layout, dev)
        return
    out, kernels = _run(op, pool, layout, dev)
    assert kernels == {kernel}, (kernel, kernels)
    again, _ = _run(op, pool, layout, dev)
    assert torch.equal(_bits(out), _bits(again))
    if kernel == "dense_grid":
        assert torch.equal(_bits(out.cpu()), _bits(torch.from_numpy(op.dense_grid())))
        print("%s [%s]: bit for bit" % (case_id(CASES[i]), kernel))
        return
    ref, S = op.oracle(mma, dev)
    gate = op.gate(S, mma)
    with torch.no_grad():
        for p in pool.embedding[0].parameters():
            p.neg_()
    neg, _ = _run(op, pool, layout, dev)
    worst, old = 0.0, 0.0
    for y, r in ((out, ref), (neg, -ref)):
        y = y.double()
        e = (y - r.clamp_min(0)).abs()
        assert bool((e <= gate).all()), (kernel, float((e / gate).max()))
        assert bool((y[r < -gate] == 0).all())
        worst = max(worst, float((e / gate).max()))
        old = max(old, float(e.max() / r.clamp_min(0).abs().max().clamp_min(1e-30)))
    probes = torch.from_numpy(op.probes).to(dev)
    pw = float(((out.double() - ref.clamp_min(0)).abs() / gate)[probes].max()) if len(op.probes) else 0.0
    print("%s [%s]: err / gate %.3f (probes %.3f), old measure %.2e; M %d, winners %d, probes %d"
          % (case_id(CASES[i]), kernel, worst, pw, old, op.M, int(op.count.sum()), len(op.probes)))


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
def test_layer1_rows_move_bit_identical(monkeypatch, tc):
    """Per-scene layout (no padded slots), so a scene's winners do not depend on the batch: its rows keep their bits
    when the scene moves to another group, another position in its group, and the other grouping."""
    from trajnetplusplusbaselines_b200.engine import SceneLayout
    _set_tc(monkeypatch, tc)
    dev = torch.device("cuda", 0)
    case = dict(m=model(OUT=257, **SOC12), batch="wide", const=1.0)
    op = Operands(case, pad=False)
    pool = _pool(op, dev)
    handle = pool._plug_handle(dev)
    hid, o1, o2 = _inputs(op, dev)
    sizes = op.sizes

    def run(order):
        idx = np.concatenate([np.arange(op.off[b], op.off[b + 1]) for b in order])
        t = torch.from_numpy(idx).to(dev)
        off = np.concatenate([[0], np.cumsum([sizes[b] for b in order])])
        layout = SceneLayout([int(x) for x in off], pad_to_batch_max=False, device=dev)
        out = handle.pool_forward(layout, hid[t].contiguous(), o1[t].contiguous(), o2[t].contiguous(), op.OUT)
        res = torch.full((op.M, op.OUT), float("nan"), device=dev)
        res[t] = out
        return res
    B = len(sizes)
    small = [b for b in range(B) if sizes[b] < 50]
    base = run(list(range(B)))
    for order in (list(reversed(range(B))), small, small[::-1], small[1:] + small[:1]):
        moved = run(order)
        rows = torch.from_numpy(np.concatenate([np.arange(op.off[b], op.off[b + 1]) for b in order])).to(dev)
        assert torch.equal(_bits(base[rows]), _bits(moved[rows])), order
    kern = kernel_of(op.m, tc)
    assert grouping(op.m, sizes, kern)[1] != grouping(op.m, [sizes[b] for b in small], kern)[1]


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("i", [i for i in range(len(CASES)) if CASES[i]["batch"] != "rows"][::4])
def test_layer1_writes_stay_inside_output(monkeypatch, i, tc):
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import SceneLayout
    _set_tc(monkeypatch, tc)
    dev = torch.device("cuda", 0)
    op = operands(i)
    layout = SceneLayout([int(x) for x in op.off], device=dev)
    pool = _pool(op, dev)
    handle = pool._plug_handle(dev)
    hid, o1, o2 = _inputs(op, dev)
    ref = handle.pool_forward(layout, hid, o1, o2, op.OUT)
    n = op.M * op.OUT
    buf = torch.full((n + 3 * op.OUT + 61,), SENTINEL, dtype=torch.int32, device=dev)
    ws, need = handle.workspace(layout)
    p = lambda t: ctypes.c_void_p(t.data_ptr() if t is not None else 0)      # noqa: E731
    lib = _lib.load()
    _lib.check(lib.tb2_pool_forward(handle.handle, layout.handle, p(hid), p(o1), p(o2), p(buf), p(ws), need,
                                    ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    torch.cuda.synchronize(dev)
    assert bool((buf[n:] == SENTINEL).all())
    assert torch.equal(buf[:n], _bits(ref).reshape(-1))


@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False], ids=["tc", "no_tc"])
@pytest.mark.parametrize("kind", E2E_KINDS)
def test_forward_with_pool_constant(monkeypatch, kind, tc):
    from oracle import lstm_oracle as O
    from trajnetplusplusbaselines_b200.lstm import LSTM, GridBasedPooling
    _set_tc(monkeypatch, tc)
    W = O.random_weights(kind, seed=13, relu_bias=3.0)
    model = LSTM(pool=GridBasedPooling(**dict(O.MODEL_SPECS[kind], constant=1)))
    model.load_state_dict({k: torch.from_numpy(v.copy()) for k, v in W.items()}, strict=True)
    model = model.cuda().eval()
    xy, bs = O.synthetic_scenes(7, 9, seed=61, ragged=True, nan_tracks=True)
    M = xy.shape[1]
    with torch.no_grad():
        _, pred = model(torch.from_numpy(xy[:9]), torch.zeros(M, 2), torch.from_numpy(bs), n_predict=12)
    _, pred_o = O.forward(W, _pool_config_const(kind, 1.0), xy[:9], bs, n_predict=12)
    pred = pred.cpu().numpy()
    assert (np.isnan(pred) == np.isnan(pred_o)).all()
    err = float(np.nanmax(np.abs(pred - pred_o)))
    print("forward %s constant 1 [%s]: max |pos - oracle| %.2e m" % (kind, "tc" if tc else "no_tc", err))
    assert err <= 1e-4, err
