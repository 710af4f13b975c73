"""The step's two wgmma kernels against a float64 product of their own bf16 operands.

dense_layer_tc (the social grid's second Linear and the row GEMMs of the social backward) and lstm_gates_tc (the LSTM
gate GEMM with the cell update and the Gaussian head in its epilogue) multiply bf16 (hi, lo) operand pairs in three
tensor-core passes and accumulate in fp32.  Given operands whose bits the test knows, the float64 value of
hi_a.hi_w + hi_a.lo_w + lo_a.hi_w (+ bias) is what the kernel computes up to the order and rounding of its fp32
accumulation.  So the gate is per element:

    |Y - Y64| <= C_ACC * S,   S = sum_k (|hi_a hi_w| + |hi_a lo_w| + |lo_a hi_w|) + |bias|   (float64)

and the gate kernel's h, c, normal and position carry that bound through the cell update and the head to first order,
plus SFU_ABS per fast-math activation.  The test data mixes dense rows with probe rows that are non-zero in one k-block
only, so a fault confined to one k-block moves a probe row's result by a large fraction of its own S.

CPU (no device needed):
  * test_dense_emulation_* / test_gates_emulation_*: a numpy emulation of each kernel's arithmetic (fp32 accumulation
    of exact k16 chunk products in the kernel's k order, rounded to nearest and, since the tensor cores' accumulator
    rounding is not documented, truncated) passes C_ACC with 4x margin at every shape of the GPU tables; each emulated
    fault (one k16 step skipped, last k-block dropped, a stage read stale, the lo_a.hi_w pass lost in one k-block, the
    tail tile's rows shifted, a bias pair swapped; for the gate kernel also c read from the neighbouring unit and one
    cluster rank's head partial lost) fails it by 4x;
  * the shape tables assert their coverage: every residue of k-blocks mod ring depth (3 at BN = 128, 4 at BN = 64),
    the first h k-block of the gate kernel at each of its 3 stages, tail tiles, and launches of >= 3 waves of 132 SMs;
  * tb2::launch_dense_tc is exported under the mangled name the tests and scripts/layer1_wgmma_floor.py call.

GPU:
  * test_dense_matches_float64: dense_layer_tc called directly, every K at N = 64 / 256, every N at K = 64 / 448 /
    1024, an M sweep up to a 3-wave launch, and every shape the library calls it at; Y within the gate, the bf16 split
    bit for bit, rows past M untouched, a rerun and a row moved to another tile position bit-identical;
  * test_dense_refuses_unsupported_shapes: K or N not a multiple of 64 is refused before any launch;
  * test_gates_match_float64: lstm_gates_tc through tb2_lstm_step_forward at H = 64 .. 256 with no pool, an external
    pooled operand of P = 64 .. 1024 or a goal embedding; h, c, normal and position within the propagated gate, absent
    rows bit for bit, in-place and separate outputs bit-identical, a track's bits the same at M = 1 and inside a 3-wave
    launch, rows past M untouched; the same oracle with an fp32 FFMA bound for lstm_gates (TB2_DISABLE_TC=1, P = 40).
Every case prints its worst err / S (or err / gate) next to the error in the older measure, relative to the tensor's
largest entry, which the whole-step tests gate at 5e-5.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_hidden_dim import _profiled, _set_tc  # noqa: E402

F32, F64 = np.float32, np.float64
U = 2.0 ** -24                  # fp32 unit roundoff
C_ACC = 2.0 ** -16              # per-element gate of the fp32 accumulation, relative to S
SFU_ABS = 3e-7                  # |error| of one __expf / __fdividef sigmoid or tanh (gates_tc.cu)
OLD_GATE = 5e-5                 # the step tests' gate, relative to the tensor's largest entry
MARGIN = 4.0
SMS = 132                       # SMs of an H100 SXM: one resident CTA each for both kernels
DENSE_SYMBOL = "_ZN3tb215launch_dense_tcEPKvS1_S1_S1_PKfPfPvS5_iiiiP11CUstream_st"     # tb2::launch_dense_tc
SENTINEL = 0x7FBADBAD          # a NaN no kernel writes (its high half, 0x7FBA, is a bf16 NaN)


# ---------------------------------------------------------------------------------------------------------------------
# bf16 arithmetic of the kernels
# ---------------------------------------------------------------------------------------------------------------------
def bf16_rn(x):
    """float32 -> the float32 value of its bf16 rounding (to nearest even, __float2bfloat16_rn); finite inputs."""
    b = np.ascontiguousarray(x, F32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(F32)


def split(x):
    hi = bf16_rn(x)
    return hi, bf16_rn(np.asarray(x, F32) - hi)


def three_pass(a_hi, a_lo, w_hi, w_lo, bias, xp=np):
    """Float64 (Y64, S) of the 3-pass product + bias; numpy arrays or torch tensors (xp = torch)."""
    if xp is np:
        cat, f64 = np.concatenate, (lambda t: t.astype(F64))
    else:
        cat, f64 = torch.cat, (lambda t: t.double())
    A3 = cat([f64(a_hi), f64(a_hi), f64(a_lo)], 1)
    W3 = cat([f64(w_hi), f64(w_lo), f64(w_hi)], 1)
    b = f64(bias)
    return A3 @ W3.T + b, abs(A3) @ abs(W3).T + abs(b)


def emulate_gemm(A, W, bias, bk, depth, rounding="rn", fault=None):
    """fp32 accumulator of the kernels' mainloop: k-blocks of bk columns, 16-column steps, per step the passes
    hi.hi, hi.lo, lo.hi, each step's exact product added to the fp32 accumulator (rounded to nearest or truncated).
    Then + bias in fp32 (no ReLU).  fault: None or (name, arg) of an emulated kernel error."""
    a_hi, a_lo = split(A)
    w_hi, w_lo = split(W)
    M, K = A.shape
    nkb = K // bk
    name, arg = fault if fault else (None, None)
    acc = np.zeros((M, W.shape[0]), F32)
    for kb in range(nkb):
        if name == "drop_last" and kb == nkb - 1:
            break
        src = kb - depth if name == "stale" and kb == arg else kb          # the stage still holds k-block kb - depth
        for k in range(bk // 16):
            if name == "skip_k16" and (kb, k) == arg:
                continue
            cols = slice(src * bk + 16 * k, src * bk + 16 * k + 16)
            for a, w in ((a_hi, w_hi), (a_hi, w_lo), (a_lo, w_hi)):
                prod = a[:, cols].astype(F64) @ w[:, cols].astype(F64).T
                if a is a_lo and name == "no_lo_a" and kb == arg:
                    prod[:] = 0
                if a is a_lo and name == "no_lo_a_tail" and kb == arg:      # the last row tile's only
                    prod[(M - 1) // 128 * 128:] = 0
                s = acc.astype(F64) + prod
                r = s.astype(F32)
                if rounding == "rz":
                    over = np.abs(r.astype(F64)) > np.abs(s)
                    r[over] = np.nextafter(r[over], F32(0))
                acc = r
    b = np.array(bias, F32)
    if name == "bias_swap":
        b[[arg, arg + 1]] = b[[arg + 1, arg]]
    y = acc + b
    if name == "tail_shift":          # the last row tile's rows read one row further (the last one the zero fill)
        m0 = (M - 1) // 128 * 128
        y[m0:M - 1] = y[m0 + 1:M]
        y[M - 1] = b
    return y


# ---------------------------------------------------------------------------------------------------------------------
# dense_layer_tc: operands and shape table
# ---------------------------------------------------------------------------------------------------------------------
def dense_bn(N):
    return 128 if N % 128 == 0 else 64


def dense_depth(N):
    return 3 if dense_bn(N) == 128 else 4


def dense_operands(M, K, N, seed, bias_kind, tail_scale=1.0):
    """fp32 A [M, K], W [N, K], bias [N]: odd rows of A are probes, non-zero in k-block (r // 2) mod (K / 64) only; the
    rows of the last row tile (M > 128) scaled by tail_scale."""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(F32)
    nkb = K // 64
    for r in range(1, M, 2):
        kb = (r // 2) % nkb
        A[r, :kb * 64] = 0
        A[r, kb * 64 + 64:] = 0
    if M > 128:
        A[(M - 1) // 128 * 128:] *= F32(tail_scale)
    W = (rng.standard_normal((N, K)) * 0.05).astype(F32)
    bias = (rng.standard_normal(N) * 0.5 if bias_kind == "rand" else np.zeros(N)).astype(F32)
    return A, W, bias


OUTPUTS = ("y", "split", "both")


def _dense_cases():
    shapes = []
    for N in (64, 256):
        shapes += [(K, N, 300) for K in (64, 128, 192, 256, 320, 448, 512, 1024, 4096)]
    for K in (64, 448, 1024):
        shapes += [(K, N, 300) for N in (64, 192, 320, 256, 512, 1024)]
    for K, N in ((1024, 256), (512, 320)):
        shapes += [(K, N, M) for M in (1, 64, 127, 128, 129, 5120, 5121, 33000)]
    # the library's calls: forward layer 2 of the BASELINE grid (K = d1 = 1024, N = P = 256) and of social_c32 (128,
    # 64); the social backward at H = 128 / 256 (E = 64, P = 256, d1 = 1024): gate pre-activations of all steps
    # (K = E + P + H, N = 4H, M = steps x rows), d h = dgates . W_hh (4H -> H), d x = dgates . W_ih (4H -> E + P),
    # d hidden1 = dz2 . W2 (P -> d1)
    shapes += [(1024, 256, 5120), (128, 64, 5120), (448, 512, 12 * 2560), (576, 1024, 4 * 2560), (512, 128, 5120),
               (1024, 256, 5121), (512, 320, 5121), (1024, 320, 5120), (256, 1024, 5120)]
    cases, seen = [], set()
    for K, N, M in shapes:
        if (K, N, M) in seen:
            continue
        seen.add((K, N, M))
        i = len(cases)
        cases.append(dict(K=K, N=N, M=M, relu=i % 2, out=OUTPUTS[i % 3], bias="zero" if i % 4 == 3 else "rand"))
    return cases


DENSE_CASES = _dense_cases()


def _dense_id(c):
    return "K%d-N%d-M%d-relu%d-%s-%s" % (c["K"], c["N"], c["M"], c["relu"], c["out"], c["bias"])


def test_dense_table_coverage():
    # every case gates its fp32 output against the oracle (the split-only ones through a Y-only launch), so the
    # coverage below is coverage by oracle-checked cases
    bn ={dense_bn(c["N"]) for c in DENSE_CASES}
    assert bn == {64, 128}
    for depth in (3, 4):
        nkb = {c["K"] // 64 for c in DENSE_CASES if dense_depth(c["N"]) == depth}
        assert {n % depth for n in nkb} == set(range(depth)), (depth, nkb)
        assert {1, depth - 1, depth, depth + 1} <= nkb and max(nkb) >= 16 * depth, (depth, nkb)
    for key, values in (("relu", {0, 1}), ("out", set(OUTPUTS)), ("bias", {"rand", "zero"})):
        assert {c[key] for c in DENSE_CASES} == values, key
    Ms = {c["M"] for c in DENSE_CASES}
    assert {1, 127, 128, 129, 5121} <= Ms
    assert max(-(-c["M"] // 128) * (c["N"] // dense_bn(c["N"])) for c in DENSE_CASES) >= 3 * SMS
    shapes = {(c["K"], c["N"]) for c in DENSE_CASES}
    assert {(1024, 256), (128, 64), (448, 512), (576, 1024), (512, 128), (1024, 256), (512, 320), (1024, 320),
            (256, 1024)} <= shapes


def _emulation_shapes():
    """Distinct (K, N, relu, bias) of the table.  Columns are computed independently and rows only select a tile, so
    the emulation takes up to 128 columns and 2 K / 64 + 5 rows (every k-block probed, a tail tile)."""
    out = {}
    for c in DENSE_CASES:
        out[(c["K"], min(c["N"], 128), c["relu"], c["bias"])] = c
    return sorted(out)


def _dense_emulated(K, N, relu, bias_kind, seed, rounding="rn", fault=None, M=None, tail_scale=1.0):
    M = M or 2 * (K // 64) + 5
    A, W, bias = dense_operands(M, K, N, seed, bias_kind, tail_scale)
    y = emulate_gemm(A, W, bias, 64, dense_depth(N), rounding, fault)
    a_hi, a_lo = split(A)
    w_hi, w_lo = split(W)
    ref, S = three_pass(a_hi, a_lo, w_hi, w_lo, bias)
    if relu:
        y, ref = np.maximum(y, 0), np.maximum(ref, 0)
    return float(np.max(np.abs(y - ref) / S)), float(np.max(np.abs(y - ref)) / max(np.max(np.abs(ref)), 1e-30))


@pytest.mark.parametrize("rounding", ["rn", "rz"])
def test_dense_emulation_inside_gate(rounding):
    for K, N, relu, bias_kind in _emulation_shapes():
        err, old = _dense_emulated(K, N, relu, bias_kind, seed=K + N, rounding=rounding)
        print("dense emulation [%s] K=%d N=%d relu=%d bias=%s: err/S %.2e (gate %.2e), old measure %.2e"
              % (rounding, K, N, relu, bias_kind, err, C_ACC, old))
        assert err * MARGIN <= C_ACC, (K, N, relu, bias_kind, err)


def _dense_faults(K):
    nkb = K // 64
    faults = {"skip_k16": ("skip_k16", (nkb // 2, 2)), "drop_last": ("drop_last", None),
              "no_lo_a": ("no_lo_a", nkb - 1), "tail_shift": ("tail_shift", None), "bias_swap": ("bias_swap", 6)}
    return faults


@pytest.mark.parametrize("K,N", [(64, 64), (192, 256), (256, 64), (448, 320), (1024, 256), (4096, 64), (4096, 256)])
def test_dense_emulated_faults_fail_gate(K, N):
    faults = _dense_faults(K)
    depth = dense_depth(N)
    if K // 64 > depth:
        faults["stale"] = ("stale", K // 64 - 1)
    for name, fault in faults.items():
        err, old = _dense_emulated(K, N, 0, "rand", seed=K + 2 * N, fault=fault)
        print("dense fault %-10s K=%d N=%d: err/S %.2e = %.0f x gate, old measure %.2e"
              % (name, K, N, err, err / C_ACC, old))
        assert err >= MARGIN * C_ACC, (name, K, N, err)


@pytest.mark.parametrize("K,N", [(448, 320), (1024, 256), (4096, 64), (4096, 256)])
def test_dense_gate_catches_what_the_old_gate_misses(K, N):
    """A fault the older measure cannot see: the last row tile's rows are 2^-6 the size of the others (small
    activations or gradients in the tail of a batch), and the lo_a.hi_w pass is lost for that tile in the k-block of
    its first probe row.  The tensor stays within 5e-5 of its largest entry, the probe row fails the per-element gate
    by 4x or more; without the fault it passes with 4x margin."""
    nkb = K // 64
    M = 128 + 2 * nkb + 5
    kb = (129 // 2) % nkb
    for rounding in ("rn", "rz"):
        err, old = _dense_emulated(K, N, 0, "zero", seed=K + 3 * N, rounding=rounding, M=M, tail_scale=2.0 ** -6)
        assert err * MARGIN <= C_ACC and old <= OLD_GATE, (rounding, err, old)
    err, old = _dense_emulated(K, N, 0, "zero", seed=K + 3 * N, fault=("no_lo_a_tail", kb), M=M, tail_scale=2.0 ** -6)
    print("dense fault no_lo_a in the small tail tile K=%d N=%d: err/S %.2e = %.0f x gate, old measure %.2e (gate %.0e)"
          % (K, N, err, err / C_ACC, old, OLD_GATE))
    assert err >= MARGIN * C_ACC, err
    assert old <= OLD_GATE, old


# ---------------------------------------------------------------------------------------------------------------------
# lstm_gates_tc: operands, oracle and shape table
# ---------------------------------------------------------------------------------------------------------------------
GATE_BK, GATE_DEPTH = 32, 3


def gate_layout(H, P, G):
    """(k-blocks of [emb | goal_emb], of pooled, of h) of the gate kernel's K = 64 + G + P + H."""
    return (64 + G) // GATE_BK, P // GATE_BK, H // GATE_BK


def _gate_cases():
    cases = []
    for H in (64, 128, 192, 256):
        cases += [dict(H=H, P=P, G=0, M=129, tc=True) for P in (0, 64, 128, 192, 256, 1024)]
        cases.append(dict(H=H, P=0, G=64, M=129, tc=True))
    cases += [dict(H=128, P=256, G=0, M=M, tc=True) for M in (1, 127, 128, 5121)]
    cases += [dict(H=256, P=0, G=64, M=M, tc=True) for M in (1, 5121)]
    # >= 3 waves of 132 SMs: ceil(M / 128) row tiles x H / 64 CTAs
    cases += [dict(H=64, P=128, G=0, M=52000, tc=True), dict(H=192, P=0, G=64, M=17000, tc=True),
              dict(H=256, P=1024, G=0, M=13000, tc=True)]
    # the FFMA lstm_gates: with TB2_DISABLE_TC=1, and at a pooled width the wgmma kernel does not take (P = 40)
    cases += [dict(H=128, P=256, G=0, M=129, tc=False), dict(H=64, P=0, G=64, M=129, tc=False),
              dict(H=256, P=1024, G=0, M=5121, tc=False), dict(H=128, P=40, G=0, M=129, tc=True),
              dict(H=256, P=40, G=0, M=129, tc=True)]
    return cases


GATE_CASES = _gate_cases()


def _gate_id(c):
    return "H%d-P%d-G%d-M%d-%s" % (c["H"], c["P"], c["G"], c["M"], "tc" if c["tc"] else "no_tc")


def _gate_kernel(c):
    return "lstm_gates_tc" if c["tc"] and c["P"] % 64 == 0 else "lstm_gates"


def test_gate_table_coverage():
    tc = [c for c in GATE_CASES if _gate_kernel(c) == "lstm_gates_tc"]
    assert {c["H"] for c in tc} == {64, 128, 192, 256}
    assert {c["P"] for c in tc} >= {0, 64, 128, 256, 1024} and all(c["G"] == 0 or c["P"] == 0 for c in GATE_CASES)
    # the first h k-block (the pooled -> h or emb -> h switch) at each ring stage; the emb -> pooled switch is at
    # k-block 2 in every model the library builds (E = 64), stage 2
    h_stage = {sum(gate_layout(c["H"], c["P"], c["G"])[:2]) % GATE_DEPTH for c in tc}
    assert h_stage == {0, 1, 2}, h_stage
    assert {sum(gate_layout(c["H"], c["P"], c["G"])) % GATE_DEPTH for c in tc} == {0, 1, 2}
    assert {c["M"] for c in tc} >= {1, 127, 128, 129, 5121}
    for H in (64, 192, 256):
        assert any(c["H"] == H and -(-c["M"] // 128) * (H // 64) >= 3 * SMS for c in tc), H
    assert {c["G"] for c in tc} == {0, 64}
    assert {_gate_kernel(c) for c in GATE_CASES} == {"lstm_gates", "lstm_gates_tc"}


def dyadic(rng, shape, scale_bits, limit):
    """Multiples of 2^-scale_bits in [-limit, limit] as float32."""
    n = int(limit * 2 ** scale_bits)
    return (rng.integers(-n, n + 1, size=shape) / 2.0 ** scale_bits).astype(F32)


def gate_inputs(H, P, G, M, seed):
    """Weights (fp32 numpy, state_dict layout) and step inputs whose emb / goal_emb are exact in fp32: obs multiples of
    2^-6 in +-4 (steps up to 0.5), embedding weights and biases multiples of 2^-8 in +-1, axis-aligned goal directions.
    Odd rows are probes: they stand still, and pooled and h are zero outside one of their k-blocks.  Absent rows at
    the tile edges and the last row, and some rows with NaN only in obs1 or only in obs2."""
    rng = np.random.default_rng(seed)
    in_dim = 64 + G + P
    W = {"input_embedding_weight": dyadic(rng, (62, 2), 8, 1), "input_embedding_bias": dyadic(rng, (62,), 8, 1),
         "hidden2normal_weight": (rng.standard_normal((5, H)) * 0.3).astype(F32),
         "hidden2normal_bias": (rng.standard_normal(5) * 0.1).astype(F32)}
    for ph in ("encoder", "decoder"):
        W[ph + "_weight_ih"] = (rng.standard_normal((4 * H, in_dim)) * 0.08).astype(F32)
        W[ph + "_weight_hh"] = (rng.standard_normal((4 * H, H)) * 0.08).astype(F32)
        W[ph + "_bias_ih"] = (rng.standard_normal(4 * H) * 0.3).astype(F32)
        W[ph + "_bias_hh"] = (rng.standard_normal(4 * H) * 0.3).astype(F32)
    if G:
        W["goal_embedding_weight"] = dyadic(rng, (G - 2, 2), 8, 1)
        W["goal_embedding_bias"] = dyadic(rng, (G - 2,), 8, 1)
    obs1 = dyadic(rng, (M, 2), 6, 4)
    obs2 = obs1 + dyadic(rng, (M, 2), 6, 0.5)
    obs2[1::2] = obs1[1::2]               # probe rows stand still: emb = ReLU(b_e)
    goals = obs2.copy()
    axis = rng.integers(0, 2, size=M)
    off = dyadic(rng, (M,), 6, 4)
    goals[np.arange(M), axis] += off          # off = 0 on some rows: zero direction
    pooled = rng.standard_normal((M, P)).astype(F32)
    h = rng.uniform(-1, 1, size=(M, H)).astype(F32)
    c = rng.uniform(-3, 3, size=(M, H)).astype(F32)
    nkb = (P + H) // GATE_BK
    for r in range(1, M, 2):
        both = np.concatenate([pooled[r], h[r]])
        kb = (r // 2) % nkb
        keep = both[kb * GATE_BK:(kb + 1) * GATE_BK].copy()
        both[:] = 0
        both[kb * GATE_BK:(kb + 1) * GATE_BK] = keep
        pooled[r], h[r] = both[:P], both[P:]
    if M > 1:
        absent = [r for r in (0, 63, 64, 127, 128, M - 1) if r < M]
        obs2[absent] = np.nan
        obs1[[r for r in range(5, M, 17)]] = np.nan
        obs2[[r for r in range(11, M, 17)]] = np.nan
    return W, dict(obs1=obs1, obs2=obs2, goals=goals, pooled=pooled, h=h, c=c)


def gate_operand(W, x, G):
    """fp32 [emb | goal_emb | pooled | h] as the kernels form it (0 for absent rows); asserts emb / goal_emb exact."""
    o1, o2 = x["obs1"].astype(F64), x["obs2"].astype(F64)
    absent = np.isnan(o1[:, 0]) | np.isnan(o2[:, 0])
    v = np.where(absent[:, None], 0.0, 4.0 * (o2 - o1))
    We, be = W["input_embedding_weight"].astype(F64), W["input_embedding_bias"].astype(F64)
    emb = np.maximum(v @ We.T + be, 0.0)
    emb[absent] = 0
    parts = [emb, np.zeros((len(v), 2))]
    if G:
        d = np.where(absent[:, None], 0.0, o2 - x["goals"].astype(F64))
        n = np.sqrt((d ** 2).sum(1, keepdims=True))
        d = np.divide(d, n, out=np.zeros_like(d), where=n != 0)
        ge = np.maximum(4.0 * d @ W["goal_embedding_weight"].astype(F64).T + W["goal_embedding_bias"].astype(F64), 0.0)
        ge[absent] = 0
        parts += [ge, np.zeros((len(v), 2))]
    exact = np.concatenate(parts, 1)
    assert np.array_equal(exact.astype(F32).astype(F64), exact)
    pooled = np.where(absent[:, None], 0.0, x["pooled"]).astype(F32)
    return np.concatenate([exact.astype(F32), pooled, x["h"]], 1), absent


def gate_weights(W, phase):
    """fp32 [W_ih | W_hh] and the library's bias float32(b_ih + b_hh)."""
    Wc = np.concatenate([W[phase + "_weight_ih"], W[phase + "_weight_hh"]], 1)
    return Wc, (W[phase + "_bias_ih"] + W[phase + "_bias_hh"]).astype(F32)


def gate_oracle(Z, eZ, c_in, obs2, Wn, bn, H, xp=np):
    """float64 h, c, normal, pos of the cell update and head from the pre-activations Z [M, 4H] (gate order i, f, g, o)
    with per-element first-order error bounds from eZ, SFU_ABS per activation and fp32 rounding of each operation."""
    if xp is np:
        Z, eZ, c, o2, Wn, bn = (np.asarray(t, F64) for t in (Z, eZ, c_in, obs2, Wn, bn))
        sig, tanh, cat = (lambda t: 1 / (1 + np.exp(-t))), np.tanh, (lambda ts: np.concatenate(ts, 1))
    else:
        dev = Z.device
        c, o2, Wn, bn = (torch.as_tensor(np.asarray(t), device=dev).double() for t in (c_in, obs2, Wn, bn))
        sig, tanh, cat = torch.sigmoid, torch.tanh, (lambda ts: torch.cat(ts, 1))
    zi, zf, zg, zo = (Z[:, q * H:(q + 1) * H] for q in range(4))
    ei, ef, eg, eo = (eZ[:, q * H:(q + 1) * H] for q in range(4))
    i, f, g, o = sig(zi), sig(zf), tanh(zg), sig(zo)
    ei = i * (1 - i) * ei + SFU_ABS
    ef = f * (1 - f) * ef + SFU_ABS
    eo = o * (1 - o) * eo + SFU_ABS
    eg = (1 - g * g) * eg + SFU_ABS
    c1 = f * c + i * g
    ec = abs(c) * ef + abs(g) * ei + abs(i) * eg + 2 * U * (abs(f * c) + abs(i * g))
    tc = tanh(c1)
    etc = (1 - tc * tc) * ec + SFU_ABS
    h1 = o * tc
    eh = abs(tc) * eo + abs(o) * etc + U * abs(h1)
    s = h1 @ Wn.T + bn
    es = eh @ abs(Wn).T + (H + 2) * U * (abs(h1) @ abs(Wn).T + abs(bn))
    s2, s3, s4 = (sig(s[:, q:q + 1]) for q in (2, 3, 4))
    normal = cat([s[:, :2], 0.01 + 0.2 * s2, 0.01 + 0.2 * s3, 0.7 * s4])
    en = cat([es[:, :2],
              0.2 * (s2 * (1 - s2) * es[:, 2:3] + SFU_ABS) + 3 * U * abs(normal[:, 2:3]),
              0.2 * (s3 * (1 - s3) * es[:, 3:4] + SFU_ABS) + 3 * U * abs(normal[:, 3:4]),
              0.7 * (s4 * (1 - s4) * es[:, 4:5] + SFU_ABS) + 2 * U * abs(normal[:, 4:5])])
    pos = o2 + s[:, :2]
    epos = es[:, :2] + U * abs(pos)
    return (h1, c1, normal, pos), (eh, ec, en, epos)


def emulate_gate_epilogue(acc, bg, c_in, obs2, Wn, bn, H, fault=None):
    """fp32 cell update and head of the kernel's epilogue from the fp32 accumulator (exact libm activations)."""
    name, arg = fault if fault else (None, None)
    z = acc + bg
    sig = lambda t: (F32(1) / (F32(1) + np.exp(-t))).astype(F32)       # noqa: E731
    i, f, g, o = sig(z[:, :H]), sig(z[:, H:2 * H]), np.tanh(z[:, 2 * H:3 * H]), sig(z[:, 3 * H:])
    c = c_in.copy()
    if name == "c_neighbour":
        c[:, arg] = c_in[:, arg ^ 1]
    c1 = (f * c + i * g).astype(F32)
    h1 = (o * np.tanh(c1)).astype(F32)
    hw = h1.copy()
    if name == "rank_partial":
        hw[:, arg * 64:(arg + 1) * 64] = 0
    s = (hw @ Wn.T + bn).astype(F32)
    normal = np.concatenate([s[:, :2], F32(0.01) + F32(0.2) * sig(s[:, 2:4]), F32(0.7) * sig(s[:, 4:5])], 1)
    return h1, c1, normal, (obs2 + s[:, :2]).astype(F32)


def _gate_emulated(H, P, G, seed, rounding="rn", fault=None):
    """Largest err / gate and old-measure error of the emulated gate kernel over h, c, normal, pos (present rows)."""
    M = 2 * ((P + H) // GATE_BK) + 5
    W, x = gate_inputs(H, P, G, M, seed)
    A, absent = gate_operand(W, x, G)
    Wc, bg = gate_weights(W, "decoder")
    gemm_fault = fault if fault and fault[0] not in ("c_neighbour", "rank_partial") else None
    bias = bg.copy()
    if gemm_fault and gemm_fault[0] == "bias_swap":
        bias[[gemm_fault[1], gemm_fault[1] + 1]] = bias[[gemm_fault[1] + 1, gemm_fault[1]]]
        gemm_fault = None
    acc = emulate_gemm(A, Wc, np.zeros(4 * H, F32), GATE_BK, GATE_DEPTH, rounding, gemm_fault)
    got = emulate_gate_epilogue(acc, bias, x["c"], x["obs2"], W["hidden2normal_weight"], W["hidden2normal_bias"], H,
                                fault if fault and fault[0] in ("c_neighbour", "rank_partial") else None)
    a_hi, a_lo = split(A)
    w_hi, w_lo = split(Wc)
    Z, S = three_pass(a_hi, a_lo, w_hi, w_lo, bg)
    ref, bound = gate_oracle(Z, C_ACC * S, x["c"], x["obs2"], W["hidden2normal_weight"], W["hidden2normal_bias"], H)
    keep = ~absent
    worst, old = 0.0, 0.0
    for g, r, b in zip(got, ref, bound):
        e = np.abs(g[keep].astype(F64) - r[keep])
        worst = max(worst, float(np.max(e / b[keep])))
        old = max(old, float(np.max(e) / np.max(np.abs(r[keep]))))
    return worst, old


def _gate_shapes():
    return sorted({(c["H"], c["P"], c["G"]) for c in GATE_CASES if _gate_kernel(c) == "lstm_gates_tc"})


@pytest.mark.parametrize("rounding", ["rn", "rz"])
def test_gates_emulation_inside_gate(rounding):
    for H, P, G in _gate_shapes():
        worst, old = _gate_emulated(H, P, G, seed=H + P + G, rounding=rounding)
        print("gates emulation [%s] H=%d P=%d G=%d: err / gate %.2e, old measure %.2e"
              % (rounding, H, P, G, worst, old))
        assert worst * MARGIN <= 1.0, (H, P, G, worst)


@pytest.mark.parametrize("H,P,G", [(64, 0, 0), (128, 256, 0), (192, 64, 0), (256, 0, 64), (256, 1024, 0)])
def test_gates_emulated_faults_fail_gate(H, P, G):
    kb_e, kb_p, kb_h = gate_layout(H, P, G)
    nkb = kb_e + kb_p + kb_h
    faults = {"skip_k16": ("skip_k16", (nkb - 2, 1)), "drop_last": ("drop_last", None),
              "stale": ("stale", max(kb_e + kb_p, GATE_DEPTH)),       # at the first h k-block where it can be stale
              "no_lo_a": ("no_lo_a", kb_e + kb_p), "tail_shift": ("tail_shift", None), "bias_swap": ("bias_swap", 6),
              "c_neighbour": ("c_neighbour", 5)}
    if H > 64:
        faults["rank_partial"] = ("rank_partial", H // 64 - 1)
    for name, fault in faults.items():
        worst, old = _gate_emulated(H, P, G, seed=H + P + G + 1, fault=fault)
        print("gates fault %-12s H=%d P=%d G=%d: err = %.0f x gate, old measure %.2e" % (name, H, P, G, worst, old))
        assert worst >= MARGIN, (name, H, P, G, worst)


def test_gate_operand_emulation_is_exact():
    """emb and goal_emb of the test inputs: the kernels' fp32 fmaf order gives the float64 values (asserted inside
    gate_operand); an fp32 emulation of that order agrees bit for bit."""
    W, x = gate_inputs(128, 0, 64, 300, seed=5)
    A, absent = gate_operand(W, x, 64)
    o1, o2 = x["obs1"], x["obs2"]
    vx, vy = (o2[:, 0] - o1[:, 0]) * F32(4), (o2[:, 1] - o1[:, 1]) * F32(4)
    We, be = W["input_embedding_weight"], W["input_embedding_bias"]
    emb = np.maximum(We[:, 1][None] * vy[:, None] + (We[:, 0][None] * vx[:, None] + be[None]), 0).astype(F32)
    assert np.array_equal(emb[~absent], A[~absent, :62])


def test_dense_symbol_exported():
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    assert hasattr(lib, DENSE_SYMBOL)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: dense_layer_tc called directly
# ---------------------------------------------------------------------------------------------------------------------
def _dense_fn():
    from trajnetplusplusbaselines_b200 import _lib
    fn = getattr(_lib.load(), DENSE_SYMBOL)
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p] * 8 + [ctypes.c_int] * 4 + [ctypes.c_void_p]
    return fn


def _sentinel(shape, dtype, dev):
    """A buffer filled with the sentinel's bits (fp32), or with its high half, a bf16 NaN (bf16)."""
    if dtype == torch.float32:
        return torch.full(shape, SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)
    return torch.full(shape, int(SENTINEL >> 16), dtype=torch.int16, device=dev).view(torch.bfloat16)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _dense_run(fn, ops, M, K, N, relu, out, pad=3):
    """One launch on the first M rows of the operands into fresh sentinel-filled buffers with `pad` extra rows."""
    a_hi, a_lo, w_hi, w_lo, bias = ops
    dev = a_hi.device
    Y = _sentinel((M + pad, N), torch.float32, dev)
    Y_hi, Y_lo = _sentinel((M + pad, N), torch.bfloat16, dev), _sentinel((M + pad, N), torch.bfloat16, dev)
    p = lambda t, on: t.data_ptr() if on else None     # noqa: E731
    from trajnetplusplusbaselines_b200 import _lib
    st = torch.cuda.current_stream(dev).cuda_stream
    _lib.check(fn(a_hi.data_ptr(), a_lo.data_ptr(), w_hi.data_ptr(), w_lo.data_ptr(), bias.data_ptr(),
                  p(Y, out != "split"), p(Y_hi, out != "y"), p(Y_lo, out != "y"), M, K, N, relu, st))
    torch.cuda.synchronize(dev)
    return Y, Y_hi, Y_lo


@pytest.mark.gpu
@pytest.mark.parametrize("case", DENSE_CASES, ids=[_dense_id(c) for c in DENSE_CASES])
def test_dense_matches_float64(case):
    K, N, M, relu, out = case["K"], case["N"], case["M"], case["relu"], case["out"]
    dev = torch.device("cuda", 0)
    A, W, bias = dense_operands(M, K, N, seed=K * 7 + N + M, bias_kind=case["bias"])
    a_hi, a_lo = (torch.from_numpy(t).to(dev).bfloat16() for t in split(A))
    w_hi, w_lo = (torch.from_numpy(t).to(dev).bfloat16() for t in split(W))
    b = torch.from_numpy(bias).to(dev)
    ops = (a_hi, a_lo, w_hi, w_lo, b)
    fn = _dense_fn()
    (Y, Y_hi, Y_lo), kernels = _profiled(lambda: _dense_run(fn, ops, M, K, N, relu, out))
    assert kernels == {"dense_layer_tc"}, kernels
    ref, S = three_pass(a_hi, a_lo, w_hi, w_lo, b, xp=torch)
    if relu:
        ref = ref.clamp_min(0)
    for t, on in ((Y, out != "split"), (Y_hi, out != "y"), (Y_lo, out != "y")):
        # rows past M keep the sentinel, and so does an output not asked for
        assert bool((_bits(t[M if on else 0:]) == _bits(_sentinel((1,), t.dtype, dev))).all())
    # every mode is gated against the oracle: split only through a Y-only launch of the same operands, whose fp32
    # output the split must then be, bit for bit
    y32 = Y[:M] if out != "split" else _dense_run(fn, ops, M, K, N, relu, "y")[0][:M]
    y = y32.double()
    err = float(((y - ref).abs() / S.clamp_min(1e-300)).max())
    old = float((y - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
    print("dense %s: err/S %.2e (gate %.2e), old measure %.2e (gate %.0e)" % (_dense_id(case), err, C_ACC, old,
                                                                             OLD_GATE))
    assert bool(((y - ref).abs() <= C_ACC * S).all()), (err, C_ACC)
    assert old <= OLD_GATE, old
    if out != "y":
        hi = y32.bfloat16()
        assert torch.equal(_bits(Y_hi[:M]), _bits(hi))
        assert torch.equal(_bits(Y_lo[:M]), _bits((y32 - hi.float()).bfloat16()))
    again = _dense_run(fn, ops, M, K, N, relu, out)
    for t, u in zip((Y, Y_hi, Y_lo), again):
        assert torch.equal(_bits(t), _bits(u))
    if M > 128:
        # every row at another tile position: rows rolled by 61, and single rows at M = 1
        roll = torch.roll(torch.arange(M, device=dev), 61)
        moved = _dense_run(fn, (a_hi[roll].contiguous(), a_lo[roll].contiguous(), w_hi, w_lo, b), M, K, N, relu, out)
        for t, u in zip((Y, Y_hi, Y_lo), moved):
            assert torch.equal(_bits(t[:M][roll]), _bits(u[:M]))
        for r in sorted({0, 63, 64, 127, 128, M // 2, M - 1}):
            one = _dense_run(fn, (a_hi[r:r + 1].contiguous(), a_lo[r:r + 1].contiguous(), w_hi, w_lo, b), 1, K, N, relu,
                             out)
            for t, u in zip((Y, Y_hi, Y_lo), one):
                assert torch.equal(_bits(t[r:r + 1]), _bits(u[:1])), r


@pytest.mark.gpu
@pytest.mark.parametrize("K,N", [(32, 64), (96, 64), (64, 32), (64, 96), (96, 96)])
def test_dense_refuses_unsupported_shapes(K, N):
    from trajnetplusplusbaselines_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    a = torch.zeros(256, 256, dtype=torch.bfloat16, device=dev)
    y = torch.zeros(256, 256, device=dev)
    before = int(lib.tb2_launch_count())
    rc = _dense_fn()(a.data_ptr(), a.data_ptr(), a.data_ptr(), a.data_ptr(), y.data_ptr(), y.data_ptr(), None, None,
                     128, K, N, 0, torch.cuda.current_stream(dev).cuda_stream)
    assert rc != 0
    assert "K % 64 == 0 and N % 64 == 0" in lib.tb2_last_error().decode()
    torch.cuda.synchronize(dev)
    assert int(lib.tb2_launch_count()) == before


# ---------------------------------------------------------------------------------------------------------------------
# GPU: lstm_gates_tc through tb2_lstm_step_forward
# ---------------------------------------------------------------------------------------------------------------------
def _gate_model(W, H, P, G, dev):
    from trajnetplusplusbaselines_b200 import _lib
    from trajnetplusplusbaselines_b200.engine import ModelHandle, lstm_config
    cfg = lstm_config(H, 64, True, None, goal_dim=G)
    if P:
        cfg.pool_type, cfg.out_dim = _lib.POOL_EXTERNAL, P
    handle = ModelHandle(cfg, dev)
    handle.set_weights({k: torch.from_numpy(v).to(dev) for k, v in W.items()})
    return handle


class _Step:
    """tb2_lstm_step_forward on the caller's buffers: outputs with `pad` sentinel rows past M."""

    def __init__(self, handle, M, dev):
        from trajnetplusplusbaselines_b200.engine import SceneLayout
        self.handle, self.M, self.dev = handle, M, dev
        self.layout = SceneLayout(range(M + 1), device=dev)         # one track per scene: pooled_padded row m = track m

    def __call__(self, phase, x, inplace, pad=3):
        from trajnetplusplusbaselines_b200 import _lib
        lib = _lib.load()
        M, dev, H = self.M, self.dev, self.handle.config.hidden_dim
        t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in x.items()}
        ws, need = self.handle.workspace(self.layout)
        normal, pos = _sentinel((M + pad, 5), torch.float32, dev), _sentinel((M + pad, 2), torch.float32, dev)
        h_out, c_out = _sentinel((M + pad, H), torch.float32, dev), _sentinel((M + pad, H), torch.float32, dev)
        h_out[:M], c_out[:M] = t["h"], t["c"]
        h_in, c_in = (h_out, c_out) if inplace else (t["h"], t["c"])
        if not inplace:
            h_out, c_out = _sentinel((M + pad, H), torch.float32, dev), _sentinel((M + pad, H), torch.float32, dev)
        p = lambda v: ctypes.c_void_p(v.data_ptr() if v is not None else 0)     # noqa: E731
        goals = t["goals"] if self.handle.config.goal_dim else None
        pooled = t["pooled"] if self.handle.config.pool_type == _lib.POOL_EXTERNAL else None
        _lib.check(lib.tb2_lstm_step_forward(self.handle.handle, self.layout.handle, phase, p(t["obs1"]), p(t["obs2"]),
                                             p(goals), p(pooled), p(h_in), p(c_in), p(h_out), p(c_out), p(normal),
                                             p(pos), p(ws), need, ctypes.c_void_p(torch.cuda.current_stream(dev)
                                                                                 .cuda_stream)))
        torch.cuda.synchronize(dev)
        return h_out, c_out, normal, pos


def _rows(x, rows):
    return {k: v[rows] for k, v in x.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("case", GATE_CASES, ids=[_gate_id(c) for c in GATE_CASES])
def test_gates_match_float64(monkeypatch, case):
    H, P, G, M = case["H"], case["P"], case["G"], case["M"]
    _set_tc(monkeypatch, case["tc"])
    kernel = _gate_kernel(case)
    dev = torch.device("cuda", 0)
    W, x = gate_inputs(H, P, G, M, seed=H * 31 + P + G + M)
    handle = _gate_model(W, H, P, G, dev)
    step = _Step(handle, M, dev)
    A, absent = gate_operand(W, x, G)
    At = torch.from_numpy(A).to(dev)
    absent_t = torch.from_numpy(absent).to(dev)
    sent = _bits(_sentinel((1,), torch.float32, dev))
    report = []
    for phase, name in enumerate(("encoder", "decoder")):
        (h, c, normal, pos), kernels = _profiled(lambda: step(phase, x, inplace=False))
        assert kernel in kernels and not ({"lstm_gates", "lstm_gates_tc"} - {kernel}) & kernels, sorted(kernels)
        Wc, bg = gate_weights(W, name)
        Wt, bt = torch.from_numpy(Wc).to(dev), torch.from_numpy(bg).to(dev)
        if kernel == "lstm_gates_tc":
            Z, S = three_pass(At.bfloat16(), (At - At.bfloat16().float()).bfloat16(), Wt.bfloat16(),
                              (Wt - Wt.bfloat16().float()).bfloat16(), bt, xp=torch)
            eZ = C_ACC * S
        else:           # fp32 FFMA dot products of the fp32 operands: |error| <= (K + 1) u S
            Z = At.double() @ Wt.double().T + bt.double()
            eZ = (A.shape[1] + 1) * U * (At.double().abs() @ Wt.double().abs().T + bt.double().abs())
        ref, bound = gate_oracle(Z, eZ, x["c"], x["obs2"], W["hidden2normal_weight"], W["hidden2normal_bias"], H,
                                 xp=torch)
        keep = ~absent_t
        worst, old = 0.0, 0.0
        for label, got, r, b in zip(("h", "c", "normal", "pos"), (h, c, normal, pos), ref, bound):
            assert bool((_bits(got[M:]) == sent).all()), label           # rows past M untouched
            g = got[:M].double()
            e = (g[keep] - r[keep]).abs()
            assert bool((e <= b[keep]).all()), (label, float((e / b[keep]).max()))
            worst = max(worst, float((e / b[keep]).max()))
            old = max(old, float(e.max() / r[keep].abs().max()))
        # absent rows: state through bit for bit, NaN normal and position
        ab = absent_t
        assert torch.equal(_bits(h[:M][ab]), _bits(torch.from_numpy(x["h"]).to(dev)[ab]))
        assert torch.equal(_bits(c[:M][ab]), _bits(torch.from_numpy(x["c"]).to(dev)[ab]))
        assert bool(normal[:M][ab].isnan().all()) and bool(pos[:M][ab].isnan().all())
        # in place (h_out = h_in, c_out = c_in) gives the same bits
        for u, v in zip((h, c, normal, pos), step(phase, x, inplace=True)):
            assert torch.equal(_bits(u), _bits(v))
        report.append("%s err / gate %.2e, old measure %.2e" % (name, worst, old))
        if M > 5000 and phase == 0:
            # a track's bits at M = 1 equal its bits inside the large launch (present rows at several tile positions)
            one = _Step(handle, 1, dev)
            picks = [r for r in (1, 62, 65, 126, 129, 2 * 128 + 3, M // 2 + 1, M - 2) if not absent[r]]
            assert len(picks) >= 4
            for r in picks:
                for u, v in zip((h, c, normal, pos), one(phase, _rows(x, [r]), inplace=False)):
                    assert torch.equal(_bits(u[r:r + 1]), _bits(v[:1])), r
    print("gates %s [%s]: %s" % (_gate_id(case), kernel, "; ".join(report)))
