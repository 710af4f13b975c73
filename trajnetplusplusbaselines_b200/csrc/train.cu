// Backward of the recurrence (BPTT) for training -- reference: what autograd does for
// Trainer.train_batch (trajnetbaselines/lstm/trainer.py:229-269) through LSTM.forward
// (lstm/lstm.py:170-264).
//
// Gradient structure exploited (SURVEY.md 8a/A12, probe-verified on the reference): fed-back
// positions are detached (lstm.py:242-250), and for vanilla / occupancy / directional pooling the
// pooled vector does not depend on any hidden state, so a track's gradient never leaves its own
// LSTM chain.  The caller passes the list of ACTIVE rows (tracks that receive a non-zero upstream
// gradient: the scene primaries for PredictionLoss, loss.py:57,67) and the whole backward runs
// on those R rows only, in phases:
//   (A) per step: winners (pool_prepare) and the gather of X = [emb | pooled | h_prev], the pooled
//       rows recomputed from the winner list, plus the dense grid row of each active track;
//   (B) gate pre-activations of all steps in one GEMM per cell (encoder / decoder weights);
//   (C) the sequential chain, ONE kernel per step: cell + head backward with the recurrent
//       dgates(s+1) . W_hh mat-vec fused in;
//   (D) input gradients of all steps in one GEMM;  (E) every parameter gradient as one reduction
//       over all S * R (step, row) records, rows split over CTAs with the partial sums added in a
//       fixed order.  No floating-point atomics: results are bit-identical from run to run.
// Social pooling couples the tracks of a scene through lat_j = W_enc h_j: every track receives
// gradient, so social_backward (further down) runs on all M rows, with its own (A) (this step's
// forward records, from the training cache) and its own (C), which adds the
// backward of the grid MLP and of the hidden-state scatter to the chain.  Both drivers keep the
// same per-(step, row) records (RowRecords) and share phase (B) (gate_preactivations) and the
// LSTM / head / input-embedding weight gradients (lstm_weight_grads).
#include <cublas_v2.h>
#include <dlfcn.h>
#include <mutex>
#include <cuda_bf16.h>
#include <math_constants.h>

#include "common.cuh"

namespace tb2 {

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// X[r] = [emb(vel) | pooled | h_prev] for the active rows (one CTA per row).  The pooled part is
// recomputed from the step's winner list: pooled = relu(base + sum_winners Wt1[cell, c, :] * val)
// (one_layer embedding, constant = 0) -- R rows instead of re-running the first Linear on all M.
__global__ void __launch_bounds__(256) bwd_gather_kernel(
    const int* __restrict__ rows, int R, const float2* __restrict__ obs1, const float2* __restrict__ obs2,
    const float* __restrict__ We, const float* __restrict__ be, const float* __restrict__ h_prev,
    const int* __restrict__ win_count, const uint32_t* __restrict__ win_ent, const float* __restrict__ win_val,
    const float* __restrict__ Wt1, const float* __restrict__ base1, int nm1, int C, int cells,
    const float* __restrict__ pooled_src, float* __restrict__ X, float* __restrict__ G, float* __restrict__ vel,
    int* __restrict__ masked, int E, int P, int K, int H) {
    __shared__ uint32_t ent_s[64];
    __shared__ float val_s[64][2];
    const int r = blockIdx.x;
    if (r >= R) return;
    const int m = rows[r];
    const float2 a = obs1[m], b = obs2[m];
    const bool msk = isnan(a.x) || isnan(b.x);
    const float vx = msk ? 0.f : (b.x - a.x) * 4.0f, vy = msk ? 0.f : (b.y - a.y) * 4.0f;
    if (threadIdx.x == 0) {
        masked[r] = msk ? 1 : 0;
        vel[2 * r] = vx;
        vel[2 * r + 1] = vy;
    }
    float* x = X + (size_t)r * K;
    float* grow = G ? G + (size_t)r * C * cells : nullptr;     // the reference's grid row [C * n * n]
    if (grow)
        for (int k = threadIdx.x; k < C * cells; k += blockDim.x) grow[k] = 0.f;
    if (msk) {
        for (int k = threadIdx.x; k < K; k += blockDim.x) x[k] = 0.f;
        return;
    }
    for (int k = threadIdx.x; k < E; k += blockDim.x)
        x[k] = k < E - 2 ? fmaxf(fmaf(We[2 * k + 1], vy, fmaf(We[2 * k], vx, be[k])), 0.f) : 0.f;
    for (int k = threadIdx.x; k < H; k += blockDim.x)
        x[E + P + k] = h_prev ? h_prev[(size_t)m * H + k] : 0.f;
    if (pooled_src) {      // pooled vector of this row as the forward kernels produced it
        for (int o = threadIdx.x; o < P; o += blockDim.x) x[E + o] = pooled_src[(size_t)m * P + o];
    } else if (P > 0) {
        const int cnt = win_count[m];
        float acc[4];     // up to 4 output columns per thread (P <= 1024)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int o = threadIdx.x + q * blockDim.x;
            acc[q] = o < P ? base1[o] : 0.f;
        }
        for (int e0 = 0; e0 < cnt; e0 += 64) {
            const int n = min(64, cnt - e0);
            __syncthreads();
            if (threadIdx.x < n) {
                const size_t g = (size_t)m * nm1 + e0 + threadIdx.x;
                ent_s[threadIdx.x] = win_ent[g];
                val_s[threadIdx.x][0] = win_val[g * 2];
                val_s[threadIdx.x][1] = win_val[g * 2 + 1];
            }
            __syncthreads();
            if (threadIdx.x < n)      // a cell has one winner per row: plain stores (after the zero fill above)
                for (int c = 0; c < C; ++c)
                    grow[c * cells + (ent_s[threadIdx.x] >> 16)] = val_s[threadIdx.x][c];
            for (int e = 0; e < n; ++e) {
                const int cell = ent_s[e] >> 16;
                for (int c = 0; c < C; ++c) {
                    const float v = val_s[e][c];
                    const float* wrow = Wt1 + ((size_t)cell * C + c) * P;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int o = threadIdx.x + q * blockDim.x;
                        if (o < P) acc[q] = fmaf(wrow[o], v, acc[q]);
                    }
                }
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int o = threadIdx.x + q * blockDim.x;
            if (o < P) x[E + o] = fmaxf(acc[q], 0.f);
        }
    }
}

// Backward of LSTMCell + Hidden2Normal for one active row per CTA (4H threads; the first H, one per unit, do the cell
// and head math): the only kernel on the sequential chain of the BPTT.
//   in : gates_pre [R,4H] of this step (with bias), c_prev (state before the step, null = zeros),
//        incoming dh = dg_next[r] . Whh_next (recurrent part of the LATER step's gate gradient,
//        W_hh in torch layout [4H, H]) + pass_prev[r] (what by-passed the cell there); both null
//        at the last step.  dc [R,H] in place; upstream dnormal [M,5] (row-indexed by track)
//        dh_ext [M,H] (row-indexed by track, null = none): an upstream gradient wrt this step's output h, added to the
//        incoming dh before the masked-row branch, so an absent track's passes through its carried state
//   out: dgates [R,4H], dc (gradient wrt c_prev), hs [R,H] (h of this step), dn_raw [R,8],
//        pass_cur [R,H] (masked rows: dh goes straight through, lstm.py:158-166)
template <int H>
__global__ void __launch_bounds__(4 * H) bwd_cell_head_kernel(
    const int* __restrict__ rows, const int* __restrict__ masked, const float* __restrict__ gates_pre,
    const float* __restrict__ c_prev, const float* __restrict__ dg_next, const float* __restrict__ Whh_next,
    const float* __restrict__ dh_rec, const float* __restrict__ pass_prev, float* __restrict__ pass_cur,
    float* __restrict__ dc,
    const float* __restrict__ dnormal, const float* __restrict__ Wn, const float* __restrict__ bn,
    float* __restrict__ dgates, float* __restrict__ hs, float* __restrict__ dn_raw, const float* __restrict__ dh_ext,
    int R) {
    constexpr int kPow2 = H <= 32 ? 32 : H <= 64 ? 64 : H <= 128 ? 128 : 256;     // tree width of the head sums
    __shared__ float red[5][H];
    __shared__ float dn_s[5];
    __shared__ __align__(16) float dgn_s[4 * H];
    __shared__ float part_s[4][H];
    const int r = blockIdx.x, u = threadIdx.x % H, quarter = threadIdx.x / H;
    const int m = rows[r];
    float* dg = dgates + (size_t)r * 4 * H;
    float dh_in = 0.f;
    if (dh_rec) {       // many rows: dg_next . W_hh was done as one GEMM
        dh_in = dh_rec[(size_t)r * H + u] + pass_prev[(size_t)r * H + u];
    } else if (dg_next) {      // 4 x H threads: each quarter of the CTA reduces one gate block of the mat-vec
        dgn_s[threadIdx.x] = dg_next[(size_t)r * 4 * H + threadIdx.x];
        __syncthreads();
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        const float* wq = Whh_next + (size_t)quarter * H * H + u;
        const float* dq = dgn_s + quarter * H;
#pragma unroll 4
        for (int g = 0; g < H; g += 4) {
            a0 = fmaf(dq[g + 0], wq[(size_t)(g + 0) * H], a0);
            a1 = fmaf(dq[g + 1], wq[(size_t)(g + 1) * H], a1);
            a2 = fmaf(dq[g + 2], wq[(size_t)(g + 2) * H], a2);
            a3 = fmaf(dq[g + 3], wq[(size_t)(g + 3) * H], a3);
        }
        part_s[quarter][u] = (a0 + a1) + (a2 + a3);
        __syncthreads();
        dh_in = (part_s[0][u] + part_s[1][u]) + (part_s[2][u] + part_s[3][u]) + pass_prev[(size_t)r * H + u];
    }
    if (quarter != 0) return;       // the cell / head math below is one thread per unit (warps 0 .. H/32 - 1)
    if (dh_ext) dh_in += dh_ext[(size_t)m * H + u];
    if (masked[r]) {   // absent track: state passes through, no parameter gradient
#pragma unroll
        for (int g = 0; g < 4; ++g) dg[g * H + u] = 0.f;
        hs[(size_t)r * H + u] = 0.f;
        if (u < 8) dn_raw[r * 8 + u] = 0.f;
        pass_cur[(size_t)r * H + u] = dh_in;
        return;        // dc stays as it is
    }
    pass_cur[(size_t)r * H + u] = 0.f;
    const float* gp = gates_pre + (size_t)r * 4 * H;
    const float ig = sigm(gp[u]), fg = sigm(gp[H + u]), gg = tanhf(gp[2 * H + u]), og = sigm(gp[3 * H + u]);
    const float cp = c_prev ? c_prev[(size_t)m * H + u] : 0.f;
    const float cn = fg * cp + ig * gg;
    const float tc = tanhf(cn);
    const float hn = og * tc;
    hs[(size_t)r * H + u] = hn;
    // head: n_raw = Wn h + bn (modules.py:57); recomputed for the sigmoid derivatives
#pragma unroll
    for (int o = 0; o < 5; ++o) red[o][u] = Wn[o * H + u] * hn;
    asm volatile("bar.sync 1, %0;" ::"n"(H) : "memory");
    for (int s = kPow2 / 2; s > 0; s >>= 1) {
        if (u < s && u + s < H) {
#pragma unroll
            for (int o = 0; o < 5; ++o) red[o][u] += red[o][u + s];
        }
        asm volatile("bar.sync 1, %0;" ::"n"(H) : "memory");
    }
    if (u < 8) {
        float d = 0.f;
        if (u < 5) {
            const float raw = red[u][0] + bn[u];
            d = dnormal[(size_t)m * 5 + u];
            if (isnan(d)) d = 0.f;
            if (u >= 2) {
                const float sg = sigm(raw);
                d *= (u == 4 ? 0.7f : 0.2f) * sg * (1.f - sg);     // modules.py:60-62
            }
            dn_s[u] = d;
        }
        dn_raw[r * 8 + u] = d;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(H) : "memory");
    float dht = dh_in;
#pragma unroll
    for (int o = 0; o < 5; ++o) dht = fmaf(Wn[o * H + u], dn_s[o], dht);
    float dct = dc[(size_t)r * H + u] + dht * og * (1.f - tc * tc);
    const float dog = dht * tc;
    const float dig = dct * gg, dgg = dct * ig, dfg = dct * cp;
    dg[u] = dig * ig * (1.f - ig);
    dg[H + u] = dfg * fg * (1.f - fg);
    dg[2 * H + u] = dgg * (1.f - gg * gg);
    dg[3 * H + u] = dog * og * (1.f - og);
    dc[(size_t)r * H + u] = dct * fg;
}

// ------------------------------------------------------------------------------------------
// Tiled fp32 GEMMs (64 x 64 tiles, 32-deep slices, register prefetch of the next slice so one
// global-load latency is paid per slice instead of per 16 products).
//   gemm_kernel    :  C[M,N] = act(A[M,K] . B[K,N] (+ bias[n])), act = ReLU or none; one fmaf chain
//                     per output in ascending k from +0, bias added last (the backward's row GEMMs
//                     and the grid MLP's forward layers >= 2, launch_gemm_ffma)
//   gemm_tn_kernel :  C[n][k] (+)= sum_r A[r][n] * B[r][k]   (weight gradients; one CTA owns a
//                     tile of C and walks all rows of its slice: deterministic)
// ------------------------------------------------------------------------------------------
constexpr int kGT = 64, kGK = 32;

__device__ __forceinline__ float4 ld4(const float* base, size_t row, int ld, int col, int rows, int cols,
                                      bool vec) {
    // 4 consecutive elements of a row-major matrix, zero outside [rows, cols)
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if ((int)row >= rows) return v;
    const float* p = base + row * (size_t)ld + col;
    if (vec && col + 3 < cols) return *reinterpret_cast<const float4*>(p);
    if (col < cols) v.x = p[0];
    if (col + 1 < cols) v.y = p[1];
    if (col + 2 < cols) v.z = p[2];
    if (col + 3 < cols) v.w = p[3];
    return v;
}

template <int TM>
__global__ void __launch_bounds__(TM * 4) gemm_kernel(const float* __restrict__ A, int lda,
                                                      const float* __restrict__ B, int ldb,
                                                      float* __restrict__ Cm, int ldc, int M, int N, int K,
                                                      const float* __restrict__ bias, int relu, int vec) {
    constexpr int NT = TM * 4;                 // threads; each owns a 4 x 4 micro-tile of TM x 64
    constexpr int LA = TM * 8 / NT;            // float4 loads per thread for the A slice (TM x 32) = 2
    constexpr int LB = 64 * 8 / NT;            // ... for the B slice (64 x 32): 2 (TM = 64) or 4 (TM = 32)
    __shared__ __align__(16) float As[kGK][TM + 4];
    __shared__ __align__(16) float Bs[kGK][kGT + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * TM, n0 = blockIdx.x * kGT;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 ra[LA], rb[LB];
    auto load = [&](int k0) {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            const int f = tid + i * NT, row = f >> 3, kq = (f & 7) * 4;      // TM rows x 32 k
            ra[i] = ld4(A, (size_t)(m0 + row), lda, k0 + kq, M, K, vec);
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int f = tid + i * NT, kk = f >> 4, nq = (f & 15) * 4;     // 32 k x 64 n
            rb[i] = ld4(B, (size_t)(k0 + kk), ldb, n0 + nq, K, N, vec);
        }
    };
    auto store = [&]() {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            const int f = tid + i * NT, row = f >> 3, kq = (f & 7) * 4;
            As[kq + 0][row] = ra[i].x; As[kq + 1][row] = ra[i].y; As[kq + 2][row] = ra[i].z; As[kq + 3][row] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int f = tid + i * NT, kk = f >> 4, nq = (f & 15) * 4;
            *reinterpret_cast<float4*>(&Bs[kk][nq]) = rb[i];
        }
    };
    load(0);
    store();
    __syncthreads();
    for (int k0 = 0; k0 < K; k0 += kGK) {
        const bool more = k0 + kGK < K;
        if (more) load(k0 + kGK);
#pragma unroll
        for (int kk = 0; kk < kGK; ++kk) {
            const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
        if (more) {
            store();
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j] + (bias ? bias[n] : 0.f);
            if (relu) v = fmaxf(v, 0.f);
            Cm[(size_t)m * ldc + n] = v;
        }
    }
}

// SPLIT: rows split over gridDim.z, slice z writes its partial tile sums to C + z * N * Kc (dense
// N x Kc, ldc = Kc) and reduce_partials_kernel adds the slices in a fixed order; otherwise a single
// slice (rows_per_slice = R) adds its sums to C.
template <int TN, bool SPLIT>
__global__ void __launch_bounds__(TN * 4) gemm_tn_kernel(const float* __restrict__ A, int lda,
                                                         const float* __restrict__ B, int ldb,
                                                         float* __restrict__ Cm, int ldc, int R, int N, int Kc,
                                                         int rows_per_slice, int vec) {
    constexpr int NT = TN * 4;
    constexpr int LA = TN * 8 / NT;            // A slice: 32 rows x TN cols
    constexpr int LB = 64 * 8 / NT;            // B slice: 32 rows x 64 cols
    __shared__ __align__(16) float As[kGK][TN + 4];
    __shared__ __align__(16) float Bs[kGK][kGT + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int n0 = blockIdx.y * TN, k0c = blockIdx.x * kGT;
    const int rbeg = blockIdx.z * rows_per_slice, rend = min(R, rbeg + rows_per_slice);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float4 ra[LA], rb[LB];
    auto load = [&](int r0) {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            const int f = tid + i * NT, rr = f / (TN / 4), cq = (f % (TN / 4)) * 4;
            ra[i] = ld4(A, (size_t)(r0 + rr), lda, n0 + cq, rend, N, vec);
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int f = tid + i * NT, rr = f >> 4, cq = (f & 15) * 4;
            rb[i] = ld4(B, (size_t)(r0 + rr), ldb, k0c + cq, rend, Kc, vec);
        }
    };
    auto store = [&]() {
#pragma unroll
        for (int i = 0; i < LA; ++i) {
            const int f = tid + i * NT, rr = f / (TN / 4), cq = (f % (TN / 4)) * 4;
            *reinterpret_cast<float4*>(&As[rr][cq]) = ra[i];
        }
#pragma unroll
        for (int i = 0; i < LB; ++i) {
            const int f = tid + i * NT, rr = f >> 4, cq = (f & 15) * 4;
            *reinterpret_cast<float4*>(&Bs[rr][cq]) = rb[i];
        }
    };
    if (rbeg < rend) {
        load(rbeg);
        store();
    }
    __syncthreads();
    for (int r0 = rbeg; r0 < rend; r0 += kGK) {
        const bool more = r0 + kGK < rend;
        if (more) load(r0 + kGK);
#pragma unroll
        for (int rr = 0; rr < kGK; ++rr) {
            const float4 a = *reinterpret_cast<const float4*>(&As[rr][ty * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[rr][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
        if (more) {
            store();
            __syncthreads();
        }
    }
    float* out = SPLIT ? Cm + (size_t)blockIdx.z * N * Kc : Cm;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int n = n0 + ty * 4 + i;
        if (n >= N) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0c + tx * 4 + j;
            if (k >= Kc) continue;
            if (SPLIT) out[(size_t)n * ldc + k] = acc[i][j];
            else out[(size_t)n * ldc + k] += acc[i][j];
        }
    }
}

// C[n][k] (ldc) += sum_z part[z][n][k];  also used for column sums (N = 1)
__global__ void reduce_partials_kernel(const float* __restrict__ part, int Z, int N, int Kc, float* __restrict__ C,
                                       int ldc, float* __restrict__ C2) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)N * Kc) return;
    float s = 0.f;
    for (int z = 0; z < Z; ++z) s += part[(size_t)z * N * Kc + idx];
    const size_t n = idx / Kc, k = idx - n * Kc;
    if (C) C[n * ldc + k] += s;
    if (C2) C2[n * ldc + k] += s;
}

// part[z][n] = sum over the rows of slice z of A[r][n]
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ A, int lda, int R, int N,
                                                             int rows_per_slice, float* __restrict__ part) {
    __shared__ float sm[8][33];
    const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
    const int n = blockIdx.x * 32 + cx;
    const int rbeg = blockIdx.y * rows_per_slice, rend = min(R, rbeg + rows_per_slice);
    float s = 0.f;
    if (n < N)
        for (int r = rbeg + ry; r < rend; r += 8) s += A[(size_t)r * lda + n];
    sm[ry][cx] = s;
    __syncthreads();
    if (ry == 0 && n < N) {
        float t = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) t += sm[q][cx];
        part[(size_t)blockIdx.y * N + n] = t;
    }
}

// dst[r][o] = ref[r][o] > 0 ? src[r][o] : 0   (row strides given; dst may alias src)
__global__ void masked_copy_kernel(const float* __restrict__ ref, int ld_ref, const float* src, int ld_src,
                                   float* dst, int ld_dst, int rows, int cols) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)rows * cols) return;
    const size_t r = idx / cols;
    const int o = (int)(idx - r * cols);
    dst[r * ld_dst + o] = ref[r * ld_ref + o] > 0.f ? src[r * ld_src + o] : 0.f;
}

// dz = dX_pooled * (pooled > 0) in place (one_layer: pooled = relu(W1 grid + b1))
__global__ void relu_mask_kernel(const float* __restrict__ X, int ldx, float* __restrict__ dX, int ldd, int rows,
                                 int E, int P) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)rows * P) return;
    const size_t r = idx / P;
    const int o = (int)(idx - r * P);
    if (!(X[r * ldx + E + o] > 0.f)) dX[r * ldd + E + o] = 0.f;
}

// InputEmbedding backward (modules.py:24-30) over all saved (step, row) pairs: one CTA per
// embedding unit k, d pre[k] = dX[k] * (emb[k] > 0), fixed-order tree reduction.
__global__ void __launch_bounds__(256) bwd_embed_kernel(const float* __restrict__ X, int ldx,
                                                        const float* __restrict__ dXe, int ldd,
                                                        const float* __restrict__ vel, int rows_total,
                                                        float* __restrict__ dWe, float* __restrict__ dbe) {
    __shared__ float red[3][256];
    const int k = blockIdx.x, t = threadIdx.x;
    float gx = 0.f, gy = 0.f, gb = 0.f;
    for (int r = t; r < rows_total; r += 256) {
        if (X[(size_t)r * ldx + k] > 0.f) {
            const float d = dXe[(size_t)r * ldd + k];
            gx = fmaf(d, vel[2 * r], gx);
            gy = fmaf(d, vel[2 * r + 1], gy);
            gb += d;
        }
    }
    red[0][t] = gx; red[1][t] = gy; red[2][t] = gb;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (t < s) {
            red[0][t] += red[0][t + s]; red[1][t] += red[1][t + s]; red[2][t] += red[2][t + s];
        }
        __syncthreads();
    }
    if (t == 0 && dWe) {
        dWe[2 * k] += red[0][0];
        dWe[2 * k + 1] += red[1][0];
    }
    if (t == 0 && dbe) dbe[k] += red[2][0];
}


// ------------------------------------------------------------------------------------------
// Social pooling backward (gridbased_pooling.py:145-170 through autograd).  The grid of observer i
// holds lat_j = W_enc h_j + b_enc of the winning neighbour of each occupied cell.
//   * d W1 sees the grid as it was written: winners only.
//   * d lat follows what autograd's index_put_ backward does for `occ[rows, oi] = other_values`
//     (gridbased_pooling.py:290-293): grad_values = grad_occ[oi] for EVERY written pair, so each
//     IN-RANGE pair (i, j) receives d grid_i[cell(i, j), :] = W1[:, cell-slab]^T dz1_i -- also the
//     pairs a later writer of the same cell overwrote; out-of-range pairs were replaced by the
//     constant before the write (:281-282) and receive nothing.
// In-range pairs are bucketed by cell with a stable counting sort (scene by scene, slots
// ascending), so every reduction below runs in a fixed order: results are run-to-run identical,
// no float atomics.  A slot is row * nm1 + jj (neighbour slot jj <-> j = jj + (jj >= i)).
// ------------------------------------------------------------------------------------------
__global__ void pair_count_kernel(const int* __restrict__ scene_off, const int* __restrict__ masked,
                                  const int* __restrict__ pair_cell, const uint8_t* __restrict__ pair_flag,
                                  int nm1, int cells, int* __restrict__ counts) {
    extern __shared__ int hist_s[];
    const int b = blockIdx.x, row0 = scene_off[b], n_s = scene_off[b + 1] - row0;
    for (int c = threadIdx.x; c < cells; c += blockDim.x) hist_s[c] = 0;
    __syncthreads();
    for (int idx = threadIdx.x; idx < n_s * nm1; idx += blockDim.x) {
        const int r = idx / nm1;
        const size_t slot = (size_t)row0 * nm1 + idx;
        if (pair_flag[slot] && !masked[row0 + r]) atomicAdd(&hist_s[pair_cell[slot]], 1);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < cells; c += blockDim.x) counts[(size_t)b * cells + c] = hist_s[c];
}

// base[b][c] = pairs of cell c in scenes before b;  start[c] = pairs in cells before c
__global__ void pair_offsets_kernel(const int* __restrict__ counts, int B, int cells, int* __restrict__ base,
                                    int* __restrict__ start) {
    extern __shared__ int total_s[];
    for (int c = threadIdx.x; c < cells; c += blockDim.x) {
        int run = 0;
        for (int b = 0; b < B; ++b) {
            base[(size_t)b * cells + c] = run;
            run += counts[(size_t)b * cells + c];
        }
        total_s[c] = run;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int c = 0; c < cells; ++c) {
            start[c] = run;
            run += total_s[c];
        }
        start[cells] = run;
    }
}

// sorted[start[c] + base[b][c] + rank] = slot id, bit 31 set when the pair is NOT the winner of its
// cell (it then takes part in d lat but not in d W1); rank = earlier slots of the scene in cell c.
// Bit 30 ("dead"): an in-range pair of cell 0 whose observer's LAST writer of cell 0 is an out-of-range
// neighbour (or a padding slot).  The cell then holds the constant 0, and the reference's
// lp_pool2d(occ, 1, pool_size = 1) = sign(x) relu(|x|) has derivative sign(0)^2 = 0 at exactly 0
// (gridbased_pooling.py:304): no gradient reaches any writer of that cell.  (Found by the drop-in test
// against the unmodified Trainer.train_batch; a cell overwritten by a later IN-RANGE writer holds a non-zero
// latent vector and all its writers do receive gradient.)
__global__ void pair_place_kernel(const int* __restrict__ scene_off, const int* __restrict__ masked,
                                  const int* __restrict__ pair_cell, const uint8_t* __restrict__ pair_flag,
                                  const int* __restrict__ win_count, const uint32_t* __restrict__ win_ent, int nm1,
                                  int cells, const int* __restrict__ base, const int* __restrict__ start,
                                  int pad_to_max, unsigned* __restrict__ sorted) {
    extern __shared__ short cell_s[];         // [n_s * nm1] cell of the in-range pairs, -1 otherwise
    const int b = blockIdx.x, row0 = scene_off[b], n_s = scene_off[b + 1] - row0;
    for (int idx = threadIdx.x; idx < n_s * nm1; idx += blockDim.x) {
        const size_t slot = (size_t)row0 * nm1 + idx;
        cell_s[idx] = (short)((pair_flag[slot] && !masked[row0 + idx / nm1]) ? pair_cell[slot] : -1);
    }
    __syncthreads();
    const int n_slots = pad_to_max ? nm1 : n_s - 1;      // neighbour slots that write at all
    for (int idx = threadIdx.x; idx < n_s * nm1; idx += blockDim.x) {
        const int cell = cell_s[idx];
        if (cell < 0) continue;
        int rank = 0;
        for (int q = 0; q < idx; ++q) rank += cell_s[q] == cell;
        const int r = idx / nm1, jj = idx - r * nm1, j = jj + (jj >= r);
        const uint32_t want = ((uint32_t)cell << 16) | (uint32_t)j;
        bool winner = false;
        const int cnt = win_count[row0 + r];
        for (int e = 0; e < cnt; ++e) winner |= win_ent[(size_t)(row0 + r) * nm1 + e] == want;
        bool dead = false;
        if (cell == 0) {
            // last writer of cell 0 for this observer: in-range pairs of cell 0 and every out-of-range slot write it
            for (int q = n_slots - 1; q >= 0; --q) {
                const int cq = cell_s[r * nm1 + q];
                if (cq == 0) break;                                   // an in-range pair wrote last: the cell is alive
                if (cq < 0) { dead = true; break; }                   // out of range (or padding): constant
            }
        }
        sorted[start[cell] + base[(size_t)b * cells + cell] + rank] =
            (unsigned)((size_t)row0 * nm1 + idx) | (winner ? 0u : 0x80000000u) | (dead ? 0x40000000u : 0u);
    }
}

// dgrid[slot][ch] = sum_o dz1[row(slot)][o] * Wt1[cell][ch][o]  for the pairs of one cell
// (64 pairs x C channels per CTA, 64-deep slices of o through shared memory)
constexpr int kDgPairs = 64, kDgK = 64;

template <int C>
__global__ void __launch_bounds__(256) social_dgrid_kernel(const unsigned* __restrict__ sorted,
                                                           const int* __restrict__ start,
                                                           const float* __restrict__ dz1, int d1,
                                                           const float* __restrict__ Wt1, int nm1,
                                                           float* __restrict__ dgrid) {
    constexpr int CQ = C / 4;                       // channels per thread
    __shared__ __align__(16) float As[kDgPairs][kDgK + 4];
    __shared__ __align__(16) float Bs[C][kDgK + 4];
    __shared__ int slot_s[kDgPairs];
    const int cell = blockIdx.x;
    const int tid = threadIdx.x;
    const int pr = tid >> 2, cq = tid & 3;
    // a cell can hold more pairs than gridDim.y * 64 (several neighbours of one observer in the same cell, all
    // scenes of the batch): every CTA walks its chunks with stride gridDim.y
    for (int p0 = start[cell] + blockIdx.y * kDgPairs; p0 < start[cell + 1]; p0 += gridDim.y * kDgPairs) {
    const int p1 = min(start[cell + 1], p0 + kDgPairs);
    const int np = p1 - p0;
    __syncthreads();
    if (tid < kDgPairs) slot_s[tid] = tid < np ? (int)(sorted[p0 + tid] & 0x7fffffffu) : -1;       // bit 30 (dead) kept
    __syncthreads();
    float acc[CQ];
#pragma unroll
    for (int q = 0; q < CQ; ++q) acc[q] = 0.f;
    const float* Wc = Wt1 + (size_t)cell * C * d1;
    for (int k0 = 0; k0 < d1; k0 += kDgK) {
        for (int idx = tid; idx < kDgPairs * (kDgK / 4); idx += 256) {
            const int r = idx / (kDgK / 4), c4 = (idx % (kDgK / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            const int slot = slot_s[r] < 0 ? -1 : (slot_s[r] & 0x3fffffff);
            if (slot >= 0) {
                const float* src = dz1 + (size_t)(slot / nm1) * d1 + k0 + c4;
                if (k0 + c4 + 3 < d1) v = *reinterpret_cast<const float4*>(src);
                else {
                    if (k0 + c4 < d1) v.x = src[0];
                    if (k0 + c4 + 1 < d1) v.y = src[1];
                    if (k0 + c4 + 2 < d1) v.z = src[2];
                }
            }
            *reinterpret_cast<float4*>(&As[r][c4]) = v;
        }
        for (int idx = tid; idx < C * (kDgK / 4); idx += 256) {
            const int r = idx / (kDgK / 4), c4 = (idx % (kDgK / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            const float* src = Wc + (size_t)r * d1 + k0 + c4;
            if (k0 + c4 + 3 < d1) v = *reinterpret_cast<const float4*>(src);
            else {
                if (k0 + c4 < d1) v.x = src[0];
                if (k0 + c4 + 1 < d1) v.y = src[1];
                if (k0 + c4 + 2 < d1) v.z = src[2];
            }
            *reinterpret_cast<float4*>(&Bs[r][c4]) = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int o = 0; o < kDgK; o += 4) {
            const float4 a = *reinterpret_cast<const float4*>(&As[pr][o]);
#pragma unroll
            for (int q = 0; q < CQ; ++q) {
                const float4 w = *reinterpret_cast<const float4*>(&Bs[cq * CQ + q][o]);
                acc[q] = fmaf(a.x, w.x, fmaf(a.y, w.y, fmaf(a.z, w.z, fmaf(a.w, w.w, acc[q]))));
            }
        }
        __syncthreads();
    }
    if (pr < np) {
        const bool dead = (slot_s[pr] & 0x40000000) != 0;             // its cell holds the constant: zero gradient
        float* out = dgrid + (size_t)(slot_s[pr] & 0x3fffffff) * C + cq * CQ;
#pragma unroll
        for (int q = 0; q < CQ; ++q) out[q] = dead ? 0.f : acc[q];
    }
    }
}


// ------------------------------------------------------------------------------------------
// social_dgrid on the tensor cores (warp-level mma.sync, 3-pass bf16 split, fp32 accumulation): per grid cell the
// pairs of the cell form a GEMM  dgrid[pairs, 16] = dz1[rows of the pairs, d1] . Wt1[cell]^T[d1, 16]  whose A rows are
// gathered.  One CTA = one cell (its weight slab as bf16 hi | lo in shared memory, loaded once), 64 pairs per chunk:
// warp = (16-pair tile, half of the d1 range); the A fragments come straight from global memory (a quad reads 32
// contiguous bytes of a dz1 row per load) and are split into (hi, lo) in registers.  The FFMA version above needed
// five shared-memory loads per 16 FMAs and ran at 8.6 TFLOP/s.
// ------------------------------------------------------------------------------------------
constexpr int kDmPairs = 64, kDmYs = 8;
static size_t dgrid_mma_smem(int d1) { return (size_t)2 * 16 * (d1 + 8) * sizeof(__nv_bfloat16) + 4 * 16 * 16 * sizeof(float) + kDmPairs * sizeof(int); }

__global__ void __launch_bounds__(256) social_dgrid_mma_kernel(const unsigned* __restrict__ sorted, const int* __restrict__ start,
                                                               const float* __restrict__ dz1, int d1,
                                                               const __nv_bfloat16* __restrict__ w_hi,
                                                               const __nv_bfloat16* __restrict__ w_lo, int nm1,
                                                               float* __restrict__ dgrid) {
    extern __shared__ __align__(16) unsigned char smem_dm[];
    const int ldw = d1 + 8;                                       // bf16 elements per weight row (+8: conflict-free fragments)
    __nv_bfloat16* Bh = reinterpret_cast<__nv_bfloat16*>(smem_dm);
    __nv_bfloat16* Bl = Bh + 16 * ldw;
    float* red = reinterpret_cast<float*>(Bl + 16 * ldw);         // [4 pair tiles][16 rows][16 channels]
    int* slot_s = reinterpret_cast<int*>(red + 4 * 16 * 16);
    const int cell = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int p_begin = start[cell] + blockIdx.y * kDmPairs, p_end = start[cell + 1];
    if (p_begin >= p_end) return;
    for (int idx = tid; idx < 16 * (d1 / 8); idx += 256) {
        const int r = idx / (d1 / 8), c8 = (idx - r * (d1 / 8)) * 8;
        *reinterpret_cast<uint4*>(Bh + r * ldw + c8) = *reinterpret_cast<const uint4*>(w_hi + ((size_t)cell * 16 + r) * d1 + c8);
        *reinterpret_cast<uint4*>(Bl + r * ldw + c8) = *reinterpret_cast<const uint4*>(w_lo + ((size_t)cell * 16 + r) * d1 + c8);
    }
    const int pt = warp & 3, kh = warp >> 2, g = lane >> 2, t = lane & 3;
    const int khalf = d1 / 2;
    for (int p0 = p_begin; p0 < p_end; p0 += gridDim.y * kDmPairs) {
        const int np = min(kDmPairs, p_end - p0);
        __syncthreads();
        if (tid < kDmPairs) slot_s[tid] = tid < np ? (int)(sorted[p0 + tid] & 0x7fffffffu) : -1;
        __syncthreads();
        const int s0 = slot_s[pt * 16 + g], s1 = slot_s[pt * 16 + g + 8];
        const float* a0p = s0 < 0 ? nullptr : dz1 + (size_t)((s0 & 0x3fffffff) / nm1) * d1 + kh * khalf + 2 * t;
        const float* a1p = s1 < 0 ? nullptr : dz1 + (size_t)((s1 & 0x3fffffff) / nm1) * d1 + kh * khalf + 2 * t;
        float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        const float2 z2 = make_float2(0.f, 0.f);
        const uint32_t* bh0 = reinterpret_cast<const uint32_t*>(Bh + g * ldw + kh * khalf + 2 * t);
        const uint32_t* bl0 = reinterpret_cast<const uint32_t*>(Bl + g * ldw + kh * khalf + 2 * t);
        const int ldw2 = 8 * ldw / 2;                              // 32-bit words between channel g and g + 8
#pragma unroll 4
        for (int k0 = 0; k0 < khalf; k0 += 16) {
            const float2 v00 = a0p ? *reinterpret_cast<const float2*>(a0p + k0) : z2;
            const float2 v10 = a1p ? *reinterpret_cast<const float2*>(a1p + k0) : z2;
            const float2 v01 = a0p ? *reinterpret_cast<const float2*>(a0p + k0 + 8) : z2;
            const float2 v11 = a1p ? *reinterpret_cast<const float2*>(a1p + k0 + 8) : z2;
            uint32_t ah[4], al[4];
            split_bf16x2(v00, ah[0], al[0]); split_bf16x2(v10, ah[1], al[1]);
            split_bf16x2(v01, ah[2], al[2]); split_bf16x2(v11, ah[3], al[3]);
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                const uint32_t h0 = bh0[nt * ldw2 + k0 / 2], h1 = bh0[nt * ldw2 + k0 / 2 + 4];
                const uint32_t l0 = bl0[nt * ldw2 + k0 / 2], l1 = bl0[nt * ldw2 + k0 / 2 + 4];
                mma_bf16_16816(acc[nt], ah, h0, h1);
                mma_bf16_16816(acc[nt], al, h0, h1);
                mma_bf16_16816(acc[nt], ah, l0, l1);
            }
        }
        // the two halves of the d1 range: warps 4..7 hand their sums to warps 0..3
        float* rp = red + pt * 256;
        if (kh == 1) {
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                rp[g * 16 + nt * 8 + 2 * t] = acc[nt][0]; rp[g * 16 + nt * 8 + 2 * t + 1] = acc[nt][1];
                rp[(g + 8) * 16 + nt * 8 + 2 * t] = acc[nt][2]; rp[(g + 8) * 16 + nt * 8 + 2 * t + 1] = acc[nt][3];
            }
        }
        __syncthreads();
        if (kh == 0) {
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int sl = half ? s1 : s0;
                if (sl < 0) continue;
                const bool dead = (sl & 0x40000000) != 0;          // its cell holds the constant: zero gradient
                float* out = dgrid + (size_t)(sl & 0x3fffffff) * 16;
                const int r = g + 8 * half;
#pragma unroll
                for (int nt = 0; nt < 2; ++nt) {
                    const float x = acc[nt][2 * half] + rp[r * 16 + nt * 8 + 2 * t];
                    const float y = acc[nt][2 * half + 1] + rp[r * 16 + nt * 8 + 2 * t + 1];
                    *reinterpret_cast<float2*>(out + nt * 8 + 2 * t) = dead ? make_float2(0.f, 0.f) : make_float2(x, y);
                }
            }
        }
    }
}

// per scene: dlat[j] = sum over the observers i (rows ascending) whose pair (i, j) is in range of
// that pair's dgrid slot; then the social part of d h_prev[j] = W_enc^T dlat[j] is added to the
// by-pass buffer that the next (earlier) step's cell kernel reads.
__global__ void __launch_bounds__(256) social_scene_reduce_kernel(
    const int* __restrict__ scene_off, const int* __restrict__ masked, const uint8_t* __restrict__ pair_flag,
    int nm1, int C, const float* __restrict__ dgrid, const float* __restrict__ Wenc, float* __restrict__ dlat,
    float* __restrict__ dh_add, int H) {
    extern __shared__ float dl_s[];       // [n_s][C]
    const int b = blockIdx.x, row0 = scene_off[b], n_s = scene_off[b + 1] - row0;
    for (int idx = threadIdx.x; idx < n_s * C; idx += blockDim.x) {
        const int j = idx / C, ch = idx - j * C;
        float sum = 0.f;
        for (int r = 0; r < n_s; ++r) {
            if (r == j || masked[row0 + r]) continue;
            const size_t slot = (size_t)(row0 + r) * nm1 + (j - (j > r));
            if (pair_flag[slot]) sum += dgrid[slot * C + ch];
        }
        dl_s[idx] = sum;
        dlat[(size_t)(row0 + j) * C + ch] = sum;
    }
    __syncthreads();
    if (dh_add) {
        for (int idx = threadIdx.x; idx < n_s * H; idx += blockDim.x) {
            const int j = idx / H, u = idx - j * H;
            float a = 0.f;
            for (int ch = 0; ch < C; ++ch) a = fmaf(dl_s[j * C + ch], Wenc[ch * H + u], a);
            dh_add[(size_t)(row0 + j) * H + u] += a;
        }
    }
}


// dWt1 on the tensor cores (warp-level mma.sync, 3-pass bf16 split): per cell
//   dWt1[cell][16 ch][d1] += lat^T [16 ch x pairs] . dz1[rows of the pairs][d1]
// M = the 16 latent channels, K = the pairs of the cell (16 per k-step), N = 32 output columns per warp (4 n-tiles).
// The A fragments (latent vectors of the winning pairs, zero for overwritten ones) come from shared memory, the B
// fragments straight from the gathered dz1 rows (lane (g, t) reads column o0 + g of the rows of pairs 2t, 2t+1, 2t+8,
// 2t+9); one CTA = (cell, 256 columns).  The FFMA kernel below it is kept for C != 16.
__global__ void __launch_bounds__(256) social_dw1_mma_kernel(const unsigned* __restrict__ sorted, const int* __restrict__ start,
                                                             int nm1, const int* __restrict__ row_scene,
                                                             const int* __restrict__ scene_off, const float* __restrict__ lat,
                                                             const float* __restrict__ dz1, int d1, float* __restrict__ dWt1) {
    __shared__ float lat_s[32][17];          // [pair][channel], +1: conflict-free column reads
    __shared__ int row_s[32];
    const int cell = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int p0 = start[cell], p1 = start[cell + 1];
    if (p0 >= p1) return;
    const int obase = blockIdx.y * 256 + warp * 32;
    const bool active = obase < d1;          // d1 % 32 == 0: a warp is entirely inside or outside
    float acc[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[nt][k] = 0.f;
    for (int pb = p0; pb < p1; pb += 32) {
        const int nb = min(32, p1 - pb);
        __syncthreads();
        for (int idx = tid; idx < 32 * 16; idx += 256) {
            const int tt = idx >> 4, ch = idx & 15;
            float v = 0.f;
            int rowi = 0;
            if (tt < nb) {
                const unsigned sv = sorted[pb + tt];
                const int slot = (int)(sv & 0x3fffffffu);
                const int i = slot / nm1, jj = slot - i * nm1;
                const int s0 = scene_off[row_scene[i]];
                const int j = jj + (jj >= i - s0);
                // overwritten pairs are not in the grid: they contribute to d lat only
                v = (sv & 0x80000000u) ? 0.f : lat[(size_t)(s0 + j) * 16 + ch];
                rowi = i;
            }
            lat_s[tt][ch] = v;
            if (ch == 0) row_s[tt] = rowi;       // padded pairs read row 0 with a zero latent vector
        }
        __syncthreads();
        if (!active) continue;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            if (ks * 16 >= nb) break;
            const int kb = ks * 16;
            uint32_t ah[4], al[4];
            split_bf16x2(make_float2(lat_s[kb + 2 * t][g], lat_s[kb + 2 * t + 1][g]), ah[0], al[0]);
            split_bf16x2(make_float2(lat_s[kb + 2 * t][g + 8], lat_s[kb + 2 * t + 1][g + 8]), ah[1], al[1]);
            split_bf16x2(make_float2(lat_s[kb + 2 * t + 8][g], lat_s[kb + 2 * t + 9][g]), ah[2], al[2]);
            split_bf16x2(make_float2(lat_s[kb + 2 * t + 8][g + 8], lat_s[kb + 2 * t + 9][g + 8]), ah[3], al[3]);
            const float* r0 = dz1 + (size_t)row_s[kb + 2 * t] * d1 + obase + g;
            const float* r1 = dz1 + (size_t)row_s[kb + 2 * t + 1] * d1 + obase + g;
            const float* r2 = dz1 + (size_t)row_s[kb + 2 * t + 8] * d1 + obase + g;
            const float* r3 = dz1 + (size_t)row_s[kb + 2 * t + 9] * d1 + obase + g;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                uint32_t bh0, bl0, bh1, bl1;
                split_bf16x2(make_float2(__ldg(r0 + nt * 8), __ldg(r1 + nt * 8)), bh0, bl0);
                split_bf16x2(make_float2(__ldg(r2 + nt * 8), __ldg(r3 + nt * 8)), bh1, bl1);
                mma_bf16_16816(acc[nt], ah, bh0, bh1);
                mma_bf16_16816(acc[nt], al, bh0, bh1);
                mma_bf16_16816(acc[nt], ah, bl0, bl1);
            }
        }
    }
    if (active) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            float* d0 = dWt1 + ((size_t)cell * 16 + g) * d1 + obase + nt * 8 + 2 * t;
            float* d8 = dWt1 + ((size_t)cell * 16 + g + 8) * d1 + obase + nt * 8 + 2 * t;
            float2 v0 = *reinterpret_cast<float2*>(d0), v8 = *reinterpret_cast<float2*>(d8);
            v0.x += acc[nt][0]; v0.y += acc[nt][1]; v8.x += acc[nt][2]; v8.y += acc[nt][3];
            *reinterpret_cast<float2*>(d0) = v0;
            *reinterpret_cast<float2*>(d8) = v8;
        }
    }
}

// dWt1[cell][ch][o] += sum over the cell's pairs (sorted order) of dz1[i][o] * lat_j[ch]
template <int C>
__global__ void __launch_bounds__(256) social_dw1_kernel(const unsigned* __restrict__ sorted,
                                                         const int* __restrict__ start, int nm1,
                                                         const int* __restrict__ row_scene,
                                                         const int* __restrict__ scene_off,
                                                         const float* __restrict__ lat,
                                                         const float* __restrict__ dz1, int d1,
                                                         float* __restrict__ dWt1) {
    __shared__ float lat_s[32][C];
    __shared__ int row_s[32];
    const int cell = blockIdx.x, o = blockIdx.y * 256 + threadIdx.x;
    const int p0 = start[cell], p1 = start[cell + 1];
    if (p0 >= p1) return;
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.f;
    for (int pb = p0; pb < p1; pb += 32) {
        const int nb = min(32, p1 - pb);
        __syncthreads();
        for (int idx = threadIdx.x; idx < nb * C; idx += 256) {
            const int t = idx / C, ch = idx - t * C;
            const unsigned sv = sorted[pb + t];
            const int slot = (int)(sv & 0x3fffffffu);
            const int i = slot / nm1, jj = slot - i * nm1;
            const int s0 = scene_off[row_scene[i]];
            const int j = jj + (jj >= i - s0);
            // overwritten pairs are not in the grid: they contribute to d lat only
            lat_s[t][ch] = (sv & 0x80000000u) ? 0.f : lat[(size_t)(s0 + j) * C + ch];
            if (ch == 0) row_s[t] = i;
        }
        __syncthreads();
        if (o < d1) {
#pragma unroll 4
            for (int t = 0; t < nb; ++t) {
                const float dz = dz1[(size_t)row_s[t] * d1 + o];
#pragma unroll
                for (int c = 0; c < C; ++c) acc[c] = fmaf(dz, lat_s[t][c], acc[c]);
            }
        }
    }
    if (o < d1) {
#pragma unroll
        for (int c = 0; c < C; ++c) dWt1[((size_t)cell * C + c) * d1 + o] += acc[c];
    }
}

// dW1[o][ch * cells + cell] += dWt1[cell][ch][o]   (back to the reference's parameter layout)
__global__ void untranspose_add_kernel(const float* __restrict__ dWt1, float* __restrict__ dW1, int cells, int C,
                                       int d1) {
    const size_t total = (size_t)cells * C * d1;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (size_t)gridDim.x * blockDim.x) {
        const int o = (int)(idx % d1);
        const size_t cc = idx / d1;
        const int ch = (int)(cc % C), cell = (int)(cc / C);
        dW1[(size_t)o * C * cells + (size_t)ch * cells + cell] += dWt1[idx];
    }
}

// a forward record (hidden1 or the pooled vector of a step) as fp32: from the bf16 (hi, lo) pair, or a copy
__global__ void merge_split_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                                   const float* __restrict__ src, float* __restrict__ dst, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = hi ? __bfloat162float(hi[i]) + __bfloat162float(lo[i]) : src[i];
}

__global__ void iota_kernel(int* __restrict__ p, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i;
}

// row_of[rows[r]] = r (the caller fills row_of with -1 first)
__global__ void row_of_kernel(const int* __restrict__ rows, int R, int* __restrict__ row_of) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < R) row_of[rows[r]] = r;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    return v;
}

// Gradient wrt the positions of one step's inputs, vel = obs2 - obs1 (lstm.py:123-125): one CTA per scene, one warp per
// track t, every sum in a fixed order (no atomics: run-to-run identical).
//   d vel_t  = 4 We^T (relu mask (.) dX_emb[t])            the input embedding (modules.py:24-30), record row of t
//   PAIRS (directional grid, gridbased_pooling.py:118-140): rel_ij = vel_j - vel_i of every IN-RANGE pair (i, j) of an
//   observer i with a record receives d grid_i[cell(i, j), c] = Wt1[cell][c]^T dz_i, like index_put_'s backward gives
//   it to every writer, overwritten ones included.  Nothing reaches a channel whose cell holds exactly 0 (lp_pool2d's
//   sign(0)^2 = 0, :304: an out-of-range pair wrote the cell last, or the winner's value is 0) or a component of rel
//   that is not finite (nan_to_num, :140).  Track t collects + d rel_it as neighbour and - d rel_tj as observer, in
//   ascending observer order.
//   d obs2[t] += d vel_t,  d obs1[t] -= d vel_t
// X / DXIN / G are the step's records (row r = row_of[track]), DXIN's pooled columns already ReLU-masked (dz).
template <bool PAIRS>
__global__ void __launch_bounds__(256) input_grad_kernel(
    const int* __restrict__ scene_off, const int* __restrict__ row_of, const float2* __restrict__ obs1,
    const float2* __restrict__ obs2, const float* __restrict__ X, int ldx, const float* __restrict__ DXIN, int EP, int E,
    const float* __restrict__ We, const int* __restrict__ pair_cell, const uint8_t* __restrict__ pair_flag, int nm1,
    const float* __restrict__ G, int cells, const float* __restrict__ Wt1, float* __restrict__ d_obs1,
    float* __restrict__ d_obs2) {
    const int b = blockIdx.x, row0 = scene_off[b], n_s = scene_off[b + 1] - row0;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int P = EP - E;
    for (int t = warp; t < n_s; t += blockDim.x >> 5) {
        const int mt = row0 + t, rt = row_of[mt];
        float ax = 0.f, ay = 0.f;
        if (rt >= 0) {
            for (int k = lane; k < E - 2; k += 32) {
                if (X[(size_t)rt * ldx + k] > 0.f) {
                    const float d = DXIN[(size_t)rt * EP + k];
                    ax = fmaf(We[2 * k], d, ax);
                    ay = fmaf(We[2 * k + 1], d, ay);
                }
            }
            ax = 4.f * warp_sum(ax);
            ay = 4.f * warp_sum(ay);
        }
        if (PAIRS) {
            float px = 0.f, py = 0.f;
            const float2 at = obs1[mt], bt = obs2[mt];
            const float vtx = bt.x - at.x, vty = bt.y - at.y;
            for (int i = 0; i < n_s; ++i) {
                const int ri = row_of[row0 + i];
                if (ri < 0) continue;
                const float2 ai = obs1[row0 + i], bi = obs2[row0 + i];
                const float vix = bi.x - ai.x, viy = bi.y - ai.y;
                const float* dz = DXIN + (size_t)ri * EP + E;
                const float* gi = G + (size_t)ri * 2 * cells;
                const int jj0 = i == t ? 0 : t - (t > i), jj1 = i == t ? n_s - 1 : jj0 + 1;
                for (int jj = jj0; jj < jj1; ++jj) {
                    const size_t slot = (size_t)(row0 + i) * nm1 + jj;
                    if (!pair_flag[slot]) continue;
                    const int j = jj + (jj >= i), cell = pair_cell[slot];
                    float vjx = vtx, vjy = vty;
                    if (i == t) {
                        const float2 aj = obs1[row0 + j], bj = obs2[row0 + j];
                        vjx = bj.x - aj.x;
                        vjy = bj.y - aj.y;
                    }
                    const bool live_x = gi[cell] != 0.f && isfinite(vjx - vix);
                    const bool live_y = gi[cells + cell] != 0.f && isfinite(vjy - viy);
                    if (!live_x && !live_y) continue;
                    const float* w0 = Wt1 + (size_t)cell * 2 * P;
                    float sx = 0.f, sy = 0.f;
                    for (int o = lane; o < P; o += 32) {
                        sx = fmaf(w0[o], dz[o], sx);
                        sy = fmaf(w0[P + o], dz[o], sy);
                    }
                    sx = live_x ? warp_sum(sx) : 0.f;
                    sy = live_y ? warp_sum(sy) : 0.f;
                    if (i == t) {
                        px -= sx;
                        py -= sy;
                    } else {
                        px += sx;
                        py += sy;
                    }
                }
            }
            ax += px;
            ay += py;
        }
        if (lane == 0) {
            d_obs2[2 * (size_t)mt] += ax;
            d_obs2[2 * (size_t)mt + 1] += ay;
            d_obs1[2 * (size_t)mt] -= ax;
            d_obs1[2 * (size_t)mt + 1] -= ay;
        }
    }
}

// ------------------------------------------------------------------------------------------
// Position chain of the rollout backward (tb2_lstm_rollout_backward): step s outputs pos[s] = obs2_s + mu_s, and a
// decoder step reads obs2_s = pos[s - 1] and obs1_s = pos[s - 2] (its first step: observed[-1], primaries pos[s - 2]).
// dp [S][M][2] collects d pos[s] from the caller and from the later steps' inputs; dn [S][M][5] is the caller's
// d_normals that the cell kernel of step s reads.
// ------------------------------------------------------------------------------------------
// before step s's cell kernel: d mu_s += d pos[s], and d obs2_s += d pos[s] (dp[s - 1] or observed[s + 1]: `up`)
__global__ void rollout_fold_kernel(const float2* __restrict__ dp_s, float* __restrict__ dn_s, float2* __restrict__ up,
                                    int M) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    const float2 d = dp_s[m];
    dn_s[(size_t)m * 5] += d.x;
    dn_s[(size_t)m * 5 + 1] += d.y;
    up[m].x += d.x;
    up[m].y += d.y;
}

// the first decoder step's d obs1 (`d1`): the primaries read pos[s - 2] (dp_m2; null when that is observed[-1]), every
// other track observed[-1]
__global__ void rollout_route_kernel(const float2* __restrict__ d1, const int* __restrict__ row_scene,
                                     const int* __restrict__ scene_off, float2* __restrict__ dp_m2,
                                     float2* __restrict__ d_last, int M) {
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    float2* t = (dp_m2 && scene_off[row_scene[m]] == m) ? dp_m2 + m : d_last + m;
    t->x += d1[m].x;
    t->y += d1[m].y;
}

__global__ void add_kernel(float* __restrict__ dst, const float* __restrict__ src, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] += src[i];
}

}  // namespace tb2

using namespace tb2;

namespace tb2 {
int resolve_step_inputs(const tb2_layout* l, const float* observed, int obs_length, const float* truth,
                        const float* positions, int s, Workspace* ws, const float** o1, const float** o2,
                        int* phase, cudaStream_t st);

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }


// ------------------------------------------------------------------------------------------
// Large plain GEMMs of the all-row (social) backward: cuBLAS in fp32 (CUBLAS_COMPUTE_32F) -- library code for
// plain library GEMMs; everything with a gather, a mask or a fused epilogue stays in the kernels of this file.
// ------------------------------------------------------------------------------------------
// cuBLAS is bound at run time (dlopen): inside a torch process the already loaded libcublas.so.12 is used, whatever
// its minor version.  Without the library, or when a call fails, the FFMA kernels below do the work.
struct CublasApi {
    cublasStatus_t (*create)(cublasHandle_t*) = nullptr;
    cublasStatus_t (*set_stream)(cublasHandle_t, cudaStream_t) = nullptr;
    cublasStatus_t (*gemm_ex)(cublasHandle_t, cublasOperation_t, cublasOperation_t, int, int, int, const void*, const void*,
                              cudaDataType, int, const void*, cudaDataType, int, const void*, void*, cudaDataType, int,
                              cublasComputeType_t, cublasGemmAlgo_t) = nullptr;
    bool ok = false;
};
static const CublasApi& cublas_api() {
    static CublasApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* lib = dlopen("libcublas.so.12", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libcublas.so", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) return;
        api.create = reinterpret_cast<decltype(api.create)>(dlsym(lib, "cublasCreate_v2"));
        api.set_stream = reinterpret_cast<decltype(api.set_stream)>(dlsym(lib, "cublasSetStream_v2"));
        api.gemm_ex = reinterpret_cast<decltype(api.gemm_ex)>(dlsym(lib, "cublasGemmEx"));
        api.ok = api.create && api.set_stream && api.gemm_ex;
    });
    return api;
}

static cublasHandle_t cublas_for_device() {
    static std::mutex mu;
    static cublasHandle_t handles[64] = {nullptr};
    if (!cublas_api().ok) return nullptr;
    std::lock_guard<std::mutex> lock(mu);
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
    cublasHandle_t& h = handles[dev & 63];
    if (!h && cublas_api().create(&h) != CUBLAS_STATUS_SUCCESS) h = nullptr;
    return h;
}

// column-major view: C(m x n) = alpha * op(A)(m x k) . op(B)(k x n) + beta * C; false = not taken (caller falls back)
static bool cublas_gemm(cublasOperation_t ta, cublasOperation_t tb, int m, int n, int k, const float* A, int lda,
                        const float* B, int ldb, float beta, float* C, int ldc, const char* name, cudaStream_t st) {
    if ((double)m * n * k < 3.2e7) return false;            // small problems: the FFMA kernels (deterministic split order)
    cublasHandle_t h = cublas_for_device();
    if (!h) return false;
    const CublasApi& api = cublas_api();
    const float alpha = 1.f;
    KernelTimer kt(name, st);
    if (api.set_stream(h, st) != CUBLAS_STATUS_SUCCESS) return false;
    return api.gemm_ex(h, ta, tb, m, n, k, &alpha, A, CUDA_R_32F, lda, B, CUDA_R_32F, ldb, &beta, C, CUDA_R_32F, ldc,
                       CUBLAS_COMPUTE_32F, CUBLAS_GEMM_DEFAULT) == CUBLAS_STATUS_SUCCESS;
}

__global__ void fill_bias_rows_kernel(float* __restrict__ C, int ldc, int M, int N, const float* __restrict__ bias) {
    const size_t total = (size_t)M * (N / 4);
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t r = idx / (N / 4);
        const int c4 = (int)(idx - r * (N / 4)) * 4;
        *reinterpret_cast<float4*>(C + r * ldc + c4) = *reinterpret_cast<const float4*>(bias + c4);
    }
}

int launch_gemm_ffma(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K,
                     const float* bias, int relu, const char* name, cudaStream_t st) {
    const int vec = (lda % 4 == 0 && ldb % 4 == 0 && aligned16(A) && aligned16(B)) ? 1 : 0;
    const bool small = (size_t)((M + 63) / 64) * ((N + kGT - 1) / kGT) < 148;     // few tiles: halve them
    {
        KernelTimer kt(name, st);
        if (small)
            gemm_kernel<32><<<dim3((N + kGT - 1) / kGT, (M + 31) / 32), 128, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K,
                                                                                   bias, relu, vec);
        else
            gemm_kernel<64><<<dim3((N + kGT - 1) / kGT, (M + 63) / 64), 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K,
                                                                                   bias, relu, vec);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// C = A . B (+bias), B [K, N] row-major; large products on cuBLAS
static int gemm_nn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K,
                   const float* bias, cudaStream_t st) {
    {   // row-major C = A . B  <=>  column-major C^T (N x M) = B^T-view (N x K) . A^T-view (K x M)
        const bool bias_ok = !bias || (N % 4 == 0 && ldc % 4 == 0 && aligned16(C) && aligned16(bias));
        if (bias_ok && (double)M * N * K >= 3.2e7) {
            if (bias) {
                fill_bias_rows_kernel<<<1184, 256, 0, st>>>(C, ldc, M, N, bias);
                TB2_LAUNCH_CHECK();
            }
            if (cublas_gemm(CUBLAS_OP_N, CUBLAS_OP_N, N, M, K, B, ldb, A, lda, bias ? 1.f : 0.f, C, ldc, "bwd_gemm_cublas", st))
                return TB2_OK;
        }
    }
    return launch_gemm_ffma(A, lda, B, ldb, C, ldc, M, N, K, bias, 0, "bwd_gemm", st);
}

// C[n][k] += sum_r A[r][n] B[r][k]; rows are split over CTAs when the output has few tiles
// (partials in `scratch`, summed in a fixed order: run-to-run deterministic).  C = NULL: a gradient the caller did not
// ask for (tb2_lstm_grads), nothing runs.
static int gemm_tn(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int R, int N, int Kc,
                   float* scratch, size_t scratch_floats, cudaStream_t st) {
    if (R <= 0 || !C) return TB2_OK;
    // row-major C (N x Kc) += A^T . B  <=>  column-major C^T (Kc x N) += B-view (Kc x R) . (A-view (N x R))^T
    if (cublas_gemm(CUBLAS_OP_N, CUBLAS_OP_T, Kc, N, R, B, ldb, A, lda, 1.f, C, ldc, "bwd_gemm_tn_cublas", st)) return TB2_OK;
    const int vec = (lda % 4 == 0 && ldb % 4 == 0 && aligned16(A) && aligned16(B)) ? 1 : 0;
    const int tiles32 = ((N + 31) / 32) * ((Kc + kGT - 1) / kGT);
    int Z = (2 * 148 + tiles32 - 1) / tiles32;
    if (Z > (R + 127) / 128) Z = (R + 127) / 128;
    while (Z > 1 && (size_t)Z * N * Kc > scratch_floats) --Z;
    if (Z <= 1) {
        KernelTimer kt("bwd_gemm_tn", st);
        gemm_tn_kernel<32, false><<<dim3((Kc + kGT - 1) / kGT, (N + 31) / 32), 128, 0, st>>>(A, lda, B, ldb, C, ldc, R, N,
                                                                                         Kc, R, vec);
    } else {
        int rps = (R + Z - 1) / Z;
        rps = (rps + kGK - 1) / kGK * kGK;
        Z = (R + rps - 1) / rps;
        KernelTimer kt("bwd_gemm_tn", st);
        gemm_tn_kernel<32, true><<<dim3((Kc + kGT - 1) / kGT, (N + 31) / 32, Z), 128, 0, st>>>(A, lda, B, ldb, scratch, Kc,
                                                                                           R, N, Kc, rps, vec);
        reduce_partials_kernel<<<(unsigned)(((size_t)N * Kc + 255) / 256), 256, 0, st>>>(scratch, Z, N, Kc, C, ldc,
                                                                                      nullptr);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// out (and out2, when set) += the column sums of A; either may be NULL, nothing runs when both are
static int colsum(const float* A, int lda, int R, int N, float* out, float* out2, float* scratch,
                  size_t scratch_floats, cudaStream_t st) {
    if (R <= 0 || (!out && !out2)) return TB2_OK;
    int Z = (R + 63) / 64;
    if (Z > 64) Z = 64;
    while (Z > 1 && (size_t)Z * N > scratch_floats) --Z;
    const int rps = (R + Z - 1) / Z;
    Z = (R + rps - 1) / rps;
    colsum_partial_kernel<<<dim3((N + 31) / 32, Z), 256, 0, st>>>(A, lda, R, N, rps, scratch);
    reduce_partials_kernel<<<(N + 255) / 256, 256, 0, st>>>(scratch, Z, 1, N, out, N, out2);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// bwd_cell_head_kernel at the model's width (4H threads per row)
template <typename... Args>
static int launch_cell_head(int H, int rows, cudaStream_t st, Args... args) {
    switch (H) {
        case 32: bwd_cell_head_kernel<32><<<rows, 4 * 32, 0, st>>>(args...); break;
        case 64: bwd_cell_head_kernel<64><<<rows, 4 * 64, 0, st>>>(args...); break;
        case 96: bwd_cell_head_kernel<96><<<rows, 4 * 96, 0, st>>>(args...); break;
        case 128: bwd_cell_head_kernel<128><<<rows, 4 * 128, 0, st>>>(args...); break;
        case 160: bwd_cell_head_kernel<160><<<rows, 4 * 160, 0, st>>>(args...); break;
        case 192: bwd_cell_head_kernel<192><<<rows, 4 * 192, 0, st>>>(args...); break;
        case 224: bwd_cell_head_kernel<224><<<rows, 4 * 224, 0, st>>>(args...); break;
        case 256: bwd_cell_head_kernel<256><<<rows, 4 * 256, 0, st>>>(args...); break;
        default: set_error(kHiddenDimMessage); return TB2_ERR_UNSUPPORTED;
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// Carving of the backward workspace in floats, every array 16-byte aligned; a null base only counts the bytes
struct Carve {
    void* base;
    size_t off = 0;
    float* take(size_t n) {
        float* p = base ? reinterpret_cast<float*>(base) + off : nullptr;
        off += (n + 3) & ~(size_t)3;
        return p;
    }
    size_t bytes() const { return off * sizeof(float) + 256; }
};

// Per (step, row) records of both backward drivers (rows = the active rows, or all M tracks with social pooling),
// kept so that every weight gradient is one reduction over all S * rows records after the time loop.
struct RowRecords {
    float *X, *GP, *DG, *HS, *DN, *VEL, *DXIN;     // [S][rows][K | G4 | G4 | H | 8 | 2 | E+P]
    float *pass[2], *dc;                           // [rows][H] chain state
    float* scratch;                                // partial sums of the row-split reductions
    size_t scratch_floats;
    int* masked;                                   // [S][rows]
};

// extra_grad: floats of the largest weight gradient the driver reduces besides the LSTM's own (sizes `scratch`)
static void carve_records(const tb2_lstm* m, size_t rows, size_t S, size_t extra_grad, Carve& c, RowRecords* o) {
    const size_t K = (size_t)m->K_gate, EP = (size_t)(m->E + m->P), H = (size_t)m->H, G4 = 4 * H;
    o->X = c.take(S * rows * K);
    o->GP = c.take(S * rows * G4);
    o->DG = c.take(S * rows * G4);
    o->HS = c.take(S * rows * H);
    o->DN = c.take(S * rows * 8);
    o->VEL = c.take(S * rows * 2);
    o->DXIN = c.take(S * rows * EP);
    o->pass[0] = c.take(rows * H);
    o->pass[1] = c.take(rows * H);
    o->dc = c.take(rows * H);
    o->scratch_floats = 8 * (extra_grad > G4 * K ? extra_grad : G4 * K);
    o->scratch = c.take(o->scratch_floats);
    o->masked = reinterpret_cast<int*>(c.take(S * rows));
}

// The rollout backward's position chain (rollout_fold_kernel): dn [S][M][5], dp [S][M][2], d1 [M][2]
struct RolloutBuffers {
    float *dn, *dp, *d1;
};

static void carve_rollout(size_t S, size_t M, Carve& c, RolloutBuffers* o) {
    o->dn = c.take(S * M * 5);
    o->dp = c.take(S * M * 2);
    o->d1 = c.take(M * 2);
}

struct BwdBuffers : RowRecords {
    float* G;                                      // [S][R][C n n] grid rows
    int* row_of;                                   // [M] record row of each track, -1: none (d observed)
    RolloutBuffers ro;
};

static size_t carve_bwd(const tb2_lstm* m, size_t R, size_t S, size_t M, void* base, BwdBuffers* b) {
    const size_t P = (size_t)m->P, CG = (size_t)m->C * (size_t)m->cells;
    BwdBuffers tmp;
    BwdBuffers* o = b ? b : &tmp;
    Carve c{base};
    carve_records(m, R, S, P * CG, c, o);
    o->G = c.take(P ? S * R * CG : 4);
    o->row_of = reinterpret_cast<int*>(c.take(M));
    carve_rollout(S, M, c, &o->ro);
    return c.bytes();
}


// src [R x Cc] row-major -> bf16 (hi, lo) of its transpose [Cc x R] (weights: a few hundred KB, once per backward)
__global__ void transpose_split_kernel(const float* __restrict__ src, int R, int Cc, __nv_bfloat16* __restrict__ hi,
                                       __nv_bfloat16* __restrict__ lo) {
    const size_t total = (size_t)R * Cc;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t c = idx / R;
        const int r = (int)(idx - c * R);
        split_bf16(src[(size_t)r * Cc + c], hi[idx], lo[idx]);
    }
}
// fp32 window [rows x cols] (leading dimension ld_src) -> bf16 (hi, lo) at column col_off of a [rows x ld_dst] matrix
static int split2d(const float* src, int ld_src, size_t rows, int cols, __nv_bfloat16* hi, __nv_bfloat16* lo, int ld_dst,
                   int col_off, cudaStream_t st) {
    KernelTimer kt("bwd_split", st);
    return launch_split_bf16_rows(src, ld_src, rows, cols, hi + col_off, lo + col_off, ld_dst, 148 * 16, st);
}

struct SocBuffers : RowRecords {
    float *H1, *DH1, *DLAT, *DGRID, *dWt1;
    int *rows, *counts, *base, *start;
    unsigned* sorted;
    __nv_bfloat16 *Wt1_hi, *Wt1_lo;                       // bf16 split of the cell-major first-layer weights (dgrid on mma.sync)
    // 3-pass wgmma versions of the row GEMMs (dense_layer_tc_kernel): bf16 (hi, lo) operands
    __nv_bfloat16 *X_hi, *X_lo;                           // [S][M][K]
    __nv_bfloat16 *DG_hi[2], *DG_lo[2];                   // [M][G4], steps s and s + 1
    __nv_bfloat16 *DZ2_hi, *DZ2_lo;                       // [M][P]
    __nv_bfloat16 *Wcat_hi[2], *Wcat_lo[2];               // [G4][K] = [W_ih | W_hh] per phase
    __nv_bfloat16 *WhhT_hi[2], *WhhT_lo[2];               // [H][G4]
    __nv_bfloat16 *WihT_hi[2], *WihT_lo[2];               // [E + P][G4]
    __nv_bfloat16 *W2T_hi, *W2T_lo;                       // [d1][P]
    float* zero_bias;                                     // [max(d1, G4)]
    RolloutBuffers ro;
};

static size_t carve_social(const tb2_lstm* m, const tb2_layout* l, size_t S, void* basep, SocBuffers* b) {
    const size_t M = (size_t)l->M, K = (size_t)m->K_gate, E = (size_t)m->E, P = (size_t)m->P;
    const size_t d1 = (size_t)m->mlp_dims[1], C = (size_t)m->C, cells = (size_t)m->cells;
    const size_t nm1 = (size_t)(l->n_max > 1 ? l->n_max - 1 : 1);
    const size_t H = (size_t)m->H, G4 = 4 * H;
    SocBuffers tmp;
    SocBuffers* o = b ? b : &tmp;
    Carve c{basep};
    carve_records(m, M, S, P * d1, c, o);
    o->H1 = c.take(m->n_mlp == 2 ? S * M * d1 : 4);
    o->DH1 = c.take(M * (d1 > H ? d1 : H));     // also holds the [M,H] recurrent d h of a step
    o->DLAT = c.take(S * M * C);
    o->DGRID = c.take(M * nm1 * C);
    o->dWt1 = c.take(cells * C * d1);
    o->rows = reinterpret_cast<int*>(c.take(M));
    o->sorted = reinterpret_cast<unsigned*>(c.take(M * nm1));
    o->counts = reinterpret_cast<int*>(c.take((size_t)l->B * cells));
    o->base = reinterpret_cast<int*>(c.take((size_t)l->B * cells));
    o->start = reinterpret_cast<int*>(c.take(cells + 1));
    o->Wt1_hi = reinterpret_cast<__nv_bfloat16*>(c.take((cells * C * d1 + 1) / 2));
    o->Wt1_lo = reinterpret_cast<__nv_bfloat16*>(c.take((cells * C * d1 + 1) / 2));
    auto take_bf16 = [&](size_t n) { return reinterpret_cast<__nv_bfloat16*>(c.take((n + 1) / 2)); };
    o->X_hi = take_bf16(S * M * K);
    o->X_lo = take_bf16(S * M * K);
    for (int i = 0; i < 2; ++i) {
        o->DG_hi[i] = take_bf16(M * G4);
        o->DG_lo[i] = take_bf16(M * G4);
        o->Wcat_hi[i] = take_bf16(G4 * K);
        o->Wcat_lo[i] = take_bf16(G4 * K);
        o->WhhT_hi[i] = take_bf16(H * G4);
        o->WhhT_lo[i] = take_bf16(H * G4);
        o->WihT_hi[i] = take_bf16((E + P) * G4);
        o->WihT_lo[i] = take_bf16((E + P) * G4);
    }
    o->DZ2_hi = take_bf16(M * P);
    o->DZ2_lo = take_bf16(M * P);
    o->W2T_hi = take_bf16(d1 * P);
    o->W2T_lo = take_bf16(d1 * P);
    o->zero_bias = c.take(d1 > G4 ? d1 : G4);
    carve_rollout(S, M, c, &o->ro);
    return c.bytes();
}

// (B) gate pre-activations of all steps: one GEMM per cell (encoder / decoder weights).  wgmma (the social backward,
// when its row GEMMs run on the tensor cores): the 3-pass wgmma kernel on the bf16 splits of X and [W_ih | W_hh]
// there; otherwise gemm_nn.
// row_exact: the FFMA kernel whatever the size (launch_gemm_ffma, never cuBLAS), so every row's bits are independent of
// how many rows the call has (the relevance pass).
static int gate_preactivations(const tb2_lstm* m, const RowRecords& b, int rows, int S, int S_enc,
                               const SocBuffers* wgmma, cudaStream_t st, bool row_exact = false) {
    const int K = m->K_gate, G4 = 4 * m->H;
    for (int phase = 0; phase < 2; ++phase) {
        const int s0 = phase == TB2_PHASE_ENCODER ? 0 : S_enc;
        const int ns = phase == TB2_PHASE_ENCODER ? S_enc : S - S_enc;
        if (ns <= 0) continue;
        const size_t x0 = (size_t)s0 * rows * K;
        float* GP = b.GP + (size_t)s0 * rows * G4;
        const int rc = wgmma ? launch_dense_tc(wgmma->X_hi + x0, wgmma->X_lo + x0, wgmma->Wcat_hi[phase],
                                               wgmma->Wcat_lo[phase], m->bg[phase], GP, nullptr, nullptr, ns * rows, K,
                                               G4, 0, st)
                     : row_exact ? launch_gemm_ffma(b.X + x0, K, m->WgT[phase], G4, GP, G4, ns * rows, G4, K, m->bg[phase], 0,
                                                    "bwd_gemm", st)
                                 : gemm_nn(b.X + x0, K, m->WgT[phase], G4, GP, G4, ns * rows, G4, K, m->bg[phase], st);
        if (rc) return rc;
    }
    return TB2_OK;
}

int launch_gate_preactivations(const tb2_lstm* m, const float* X, float* GP, int rows, int S, int S_enc,
                               cudaStream_t st) {
    RowRecords r{};
    r.X = const_cast<float*>(X);
    r.GP = GP;
    return gate_preactivations(m, r, rows, S, S_enc, nullptr, st, true);
}

int launch_bwd_gather(const tb2_lstm* m, const int* rows, int R, const float* obs1, const float* obs2,
                      const float* h_prev, const Workspace* winners, const float* pooled_src, int nm1, float* X, float* G,
                      float* vel, int* masked, cudaStream_t st) {
    {
        KernelTimer kt("bwd_gather", st);
        bwd_gather_kernel<<<R, 256, 0, st>>>(rows, R, (const float2*)obs1, (const float2*)obs2, m->We, m->be, h_prev,
                                             winners ? winners->win_count : nullptr, winners ? winners->win_ent : nullptr,
                                             winners ? winners->win_val : nullptr, m->Wt1, m->base1, nm1, m->C, m->cells,
                                             pooled_src, X, G, vel, masked, m->E, m->P, m->K_gate, m->H);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

constexpr int kAllPhases = (1 << TB2_PHASE_ENCODER) | (1 << TB2_PHASE_DECODER);

// LSTM, Hidden2Normal and InputEmbedding weight gradients: one reduction over all S * rows (step, row) records per
// tensor.  dxin_phases (bit 1 << phase): those cells first compute dX_in = dgates . W_ih of all their steps (the social
// backward, and the rollout backward's decoder, compute dX_in step by step inside the time loop instead, where the grid
// MLP's backward or the position chain needs it).  A NULL field of g skips its reduction; dX_in is computed either way.
static int lstm_weight_grads(const tb2_lstm* m, const tb2_lstm_weights* w, const tb2_lstm_grads* g, const RowRecords& b,
                             int rows, int S, int S_enc, int dxin_phases, cudaStream_t st) {
    const int K = m->K_gate, E = m->E, EP = E + m->P, H = m->H, G4 = 4 * H;
    int rc;
    for (int phase = 0; phase < 2; ++phase) {
        const int s0 = phase == TB2_PHASE_ENCODER ? 0 : S_enc;
        const int ns = phase == TB2_PHASE_ENCODER ? S_enc : S - S_enc;
        if (ns <= 0) continue;
        const bool enc = phase == TB2_PHASE_ENCODER;
        const float* DG = b.DG + (size_t)s0 * rows * G4;
        const float* X = b.X + (size_t)s0 * rows * K;
        const int n = ns * rows;
        // dX_in = dgates . W_ih   (torch layout [4H, E+P] is the [K = 4H, N = E+P] operand as it stands)
        if ((dxin_phases >> phase & 1) && (rc = gemm_nn(DG, G4, enc ? w->encoder_weight_ih : w->decoder_weight_ih, EP,
                                         b.DXIN + (size_t)s0 * rows * EP, EP, n, EP, G4, nullptr, st)))
            return rc;
        if ((rc = gemm_tn(DG, G4, X, K, enc ? g->encoder_weight_ih : g->decoder_weight_ih, EP, n, G4, EP, b.scratch,
                          b.scratch_floats, st)))
            return rc;
        if ((rc = gemm_tn(DG, G4, X + EP, K, enc ? g->encoder_weight_hh : g->decoder_weight_hh, H, n, G4, H, b.scratch,
                          b.scratch_floats, st)))
            return rc;
        if ((rc = colsum(DG, G4, n, G4, enc ? g->encoder_bias_ih : g->decoder_bias_ih,
                         enc ? g->encoder_bias_hh : g->decoder_bias_hh, b.scratch, b.scratch_floats, st)))
            return rc;
    }
    if ((rc = gemm_tn(b.DN, 8, b.HS, H, g->hidden2normal_weight, H, S * rows, 5, H, b.scratch, b.scratch_floats, st)))
        return rc;
    if ((rc = colsum(b.DN, 8, S * rows, 5, g->hidden2normal_bias, nullptr, b.scratch, b.scratch_floats, st))) return rc;
    if (g->input_embedding_weight || g->input_embedding_bias) {
        bwd_embed_kernel<<<E - 2, 256, 0, st>>>(b.X, K, b.DXIN, EP, b.VEL, S * rows, g->input_embedding_weight,
                                                g->input_embedding_bias);
        TB2_LAUNCH_CHECK();
    }
    return TB2_OK;
}

// d observed of the encoder steps [0, S_enc) (g->d_observed, [obs_length, M, 2], +=): input_grad_kernel per step over
// the step's records (rows: record row -> track, row_of: track -> record row or -1).  Directional grids first rebuild
// the step's pair table (pool_prepare, the winners the gather read, plus cells and range flags).  Steps in ascending
// order: each frame's two contributions are added in a fixed order.
static int observed_grads(const tb2_lstm* m, const tb2_layout* l, const RowRecords& b, const float* G, int rows,
                          const int* row_of, const float* observed, const float* states, int S_enc, Workspace& ws,
                          float* d_observed, cudaStream_t st) {
    const int K = m->K_gate, E = m->E, EP = E + m->P, H = m->H;
    const size_t M = (size_t)l->M, CG = (size_t)m->C * (size_t)m->cells;
    const int nm1 = l->n_max > 1 ? l->n_max - 1 : 1;
    const bool pairs = m->cfg.pool_type == TB2_POOL_DIRECTIONAL;
    int rc;
    for (int s = 0; s < S_enc; ++s) {
        const float* o1 = observed + (size_t)s * M * 2;
        const float* o2 = observed + (size_t)(s + 1) * M * 2;
        const float* Xs = b.X + (size_t)s * rows * K;
        const float* DXs = b.DXIN + (size_t)s * rows * EP;
        float* d1 = d_observed + (size_t)s * M * 2;
        float* d2 = d_observed + (size_t)(s + 1) * M * 2;
        if (pairs) {
            const float* h_prev = s > 0 ? states + ((size_t)(s - 1) * 2 + 0) * M * H : nullptr;
            if ((rc = launch_pool_prepare(m, l, h_prev, o1, o2, 1, 1, 0, &ws, st))) return rc;
            KernelTimer kt("bwd_input_dir_pairs", st);
            input_grad_kernel<true><<<l->B, 256, 0, st>>>(l->scene_off, row_of, (const float2*)o1, (const float2*)o2, Xs, K,
                                                          DXs, EP, E, m->We, ws.pair_cell, ws.pair_flag, nm1,
                                                          G + (size_t)s * rows * CG, m->cells, m->Wt1, d1, d2);
        } else {
            KernelTimer kt("bwd_input_vel", st);
            input_grad_kernel<false><<<l->B, 256, 0, st>>>(l->scene_off, row_of, (const float2*)o1, (const float2*)o2, Xs,
                                                           K, DXs, EP, E, m->We, nullptr, nullptr, nm1, nullptr, 0,
                                                           nullptr, d1, d2);
        }
        TB2_LAUNCH_CHECK();
    }
    return TB2_OK;
}

// Rollout backward: the caller's d normals and d positions into the chain buffers.  At obs_length 2 the positions begin
// with observed[-1] itself (lstm.py:222-223): that frame's gradient goes straight to d observed.
static int rollout_begin(const tb2_layout* l, const RolloutBuffers& ro, const float* d_normals, const float* d_positions,
                         int obs_length, int S, float* d_observed, cudaStream_t st) {
    const size_t frame = (size_t)l->M * 2;
    const size_t seed = obs_length == 2 ? 1 : 0;
    TB2_CHECK_CUDA(cudaMemcpyAsync(ro.dn, d_normals, (size_t)S * l->M * 5 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    TB2_CHECK_CUDA(cudaMemcpyAsync(ro.dp, d_positions + seed * frame, (size_t)S * frame * sizeof(float),
                                   cudaMemcpyDeviceToDevice, st));
    if (seed) {
        add_kernel<<<(unsigned)((frame + 255) / 256), 256, 0, st>>>(d_observed + (size_t)(obs_length - 1) * frame,
                                                                    d_positions, frame);
        TB2_LAUNCH_CHECK();
    }
    return TB2_OK;
}

// Rollout backward, before step s's cell kernel: d pos[s] into d mu_s and into d obs2_s
static int rollout_fold(const tb2_layout* l, const RolloutBuffers& ro, int s, int S_enc, float* d_observed,
                        cudaStream_t st) {
    const size_t M = (size_t)l->M;
    float* up = s >= S_enc ? ro.dp + (size_t)(s - 1) * M * 2 : d_observed + (size_t)(s + 1) * M * 2;
    {
        KernelTimer kt("bwd_rollout_fold", st);
        rollout_fold_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>((const float2*)(ro.dp + (size_t)s * M * 2),
                                                                          ro.dn + (size_t)s * M * 5, (float2*)up, (int)M);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// Rollout backward, right after decoder step s's dX_in (records Xs / DXs / Gs of `rows` rows, row_of: track -> row):
// d obs2_s into d pos[s - 1] and d obs1_s into d pos[s - 2] (the first decoder step: observed[-1], primaries
// pos[s - 2]) through input_grad_kernel, which the encoder steps' d observed also uses.  Directional grids rebuild the
// step's pair table and ReLU-mask the pooled columns of DXs in place first.
static int rollout_inputs(const tb2_lstm* m, const tb2_layout* l, const RolloutBuffers& ro, const float* Xs, float* DXs,
                          const float* Gs, int rows, const int* row_of, const float* observed, int obs_length,
                          const float* positions, const float* states, int s, Workspace& ws, float* d_observed,
                          cudaStream_t st) {
    const int K = m->K_gate, E = m->E, P = m->P, EP = E + P;
    const size_t M = (size_t)l->M;
    const int nm1 = l->n_max > 1 ? l->n_max - 1 : 1;
    const int first = s == obs_length - 1;
    const float *o1, *o2;
    int phase, rc;
    if ((rc = resolve_step_inputs(l, observed, obs_length, nullptr, positions, s, &ws, &o1, &o2, &phase, st))) return rc;
    float* d2 = ro.dp + (size_t)(s - 1) * M * 2;
    float* d1 = first ? ro.d1 : ro.dp + (size_t)(s - 2) * M * 2;
    if (first) TB2_CHECK_CUDA(cudaMemsetAsync(ro.d1, 0, M * 2 * sizeof(float), st));
    if (m->cfg.pool_type == TB2_POOL_DIRECTIONAL) {
        const float* h_prev = states + ((size_t)(s - 1) * 2 + 0) * M * m->H;
        if ((rc = launch_pool_prepare(m, l, h_prev, o1, o2, 1, 1, 0, &ws, st))) return rc;
        relu_mask_kernel<<<(unsigned)(((size_t)rows * P + 255) / 256), 256, 0, st>>>(Xs, K, DXs, EP, rows, E, P);
        TB2_LAUNCH_CHECK();
        KernelTimer kt("bwd_input_dir_pairs", st);
        input_grad_kernel<true><<<l->B, 256, 0, st>>>(l->scene_off, row_of, (const float2*)o1, (const float2*)o2, Xs, K,
                                                      DXs, EP, E, m->We, ws.pair_cell, ws.pair_flag, nm1, Gs, m->cells,
                                                      m->Wt1, d1, d2);
    } else {
        KernelTimer kt("bwd_input_vel", st);
        input_grad_kernel<false><<<l->B, 256, 0, st>>>(l->scene_off, row_of, (const float2*)o1, (const float2*)o2, Xs, K,
                                                       DXs, EP, E, m->We, nullptr, nullptr, nm1, nullptr, 0, nullptr, d1,
                                                       d2);
    }
    TB2_LAUNCH_CHECK();
    if (first) {
        rollout_route_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(
            (const float2*)ro.d1, l->row_scene, l->scene_off, s >= 2 ? (float2*)(ro.dp + (size_t)(s - 2) * M * 2) : nullptr,
            (float2*)(d_observed + (size_t)(obs_length - 1) * M * 2), (int)M);
        TB2_LAUNCH_CHECK();
    }
    return TB2_OK;
}

// Buffers of tb2_lstm_step_backward (external interaction module): the records of one step over all M rows
struct StepBwdBuffers : RowRecords {
    float* pooled;     // [M, pool_out] the module's rows as the gate operand (pool_to_input)
    float* h_eff;      // [M, H] h_in + pooled (pool_to_input = 0)
    float* DH;         // [M, H] dgates . W_hh
    int* rows;         // [M] 0 .. M - 1
};

static size_t carve_step_bwd(const tb2_lstm* m, const tb2_layout* l, void* base, StepBwdBuffers* b) {
    const size_t M = (size_t)l->M, H = (size_t)m->H;
    StepBwdBuffers tmp;
    StepBwdBuffers* o = b ? b : &tmp;
    Carve c{base};
    carve_records(m, M, 1, 0, c, o);
    o->pooled = c.take(m->cfg.pool_to_input ? M * (size_t)m->pool_out : 4);
    o->h_eff = c.take(m->cfg.pool_to_input ? 4 : M * H);
    o->DH = c.take(M * H);
    o->rows = reinterpret_cast<int*>(c.take(M));
    return c.bytes();
}

template <int C>
static int social_pair_kernels(const tb2_lstm* m, const tb2_layout* l, const SocBuffers& b, const float* lat,
                               int nm1, int d1, bool dw1, cudaStream_t st) {
    const bool mma = C == 16 && d1 % 32 == 0 && !m->tc_disabled;
    if (mma && b.Wt1_hi != nullptr && dgrid_mma_smem(d1) <= 200 * 1024) {
        static DynSmemConfig configured;
        TB2_CHECK_CUDA(configured.ensure(social_dgrid_mma_kernel, dgrid_mma_smem(d1), 48 * 1024));
        KernelTimer kt("social_dgrid_mma", st);
        social_dgrid_mma_kernel<<<dim3(m->cells, kDmYs), 256, dgrid_mma_smem(d1), st>>>(
            b.sorted, b.start, b.DH1, d1, b.Wt1_hi, b.Wt1_lo, nm1, b.DGRID);
    } else {
        KernelTimer kt("social_dgrid", st);
        social_dgrid_kernel<C><<<dim3(m->cells, (l->M + kDgPairs - 1) / kDgPairs), 256, 0, st>>>(
            b.sorted, b.start, b.DH1, d1, m->Wt1, nm1, b.DGRID);
    }
    TB2_LAUNCH_CHECK();
    if (!dw1) return TB2_OK;      // no pool.embedding.0.weight gradient asked for
    if (mma) {
        KernelTimer kt("social_dw1_mma", st);
        social_dw1_mma_kernel<<<dim3(m->cells, (d1 + 255) / 256), 256, 0, st>>>(
            b.sorted, b.start, nm1, l->row_scene, l->scene_off, lat, b.DH1, d1, b.dWt1);
    } else {
        KernelTimer kt("social_dw1", st);
        social_dw1_kernel<C><<<dim3(m->cells, (d1 + 255) / 256), 256, 0, st>>>(
            b.sorted, b.start, nm1, l->row_scene, l->scene_off, lat, b.DH1, d1, b.dWt1);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// (A) this step's hidden1 (b.H1, two_layer) and pooled vector (ws.pooled) as fp32, from the training cache: hi + lo
// where the forward kept the bf16 pair, a copy where it kept fp32 (pool_formats)
static int social_step_records(const tb2_lstm* m, const tb2_layout* l, const SocBuffers& b, const Workspace& ws,
                               const TrainCache& cache, int s, cudaStream_t st) {
    const size_t M = (size_t)l->M, P = (size_t)m->P, d1 = (size_t)m->mlp_dims[1];
    const PoolFormats f = pool_formats(m);
    auto merge = [&](const char* slot, size_t step, bool pair, float* dst, size_t n, int blocks) {
        const __nv_bfloat16* hi = pair ? (const __nv_bfloat16*)slot : nullptr;
        const __nv_bfloat16* lo = pair ? (const __nv_bfloat16*)(slot + step / 2) : nullptr;
        merge_split_kernel<<<blocks, 256, 0, st>>>(hi, lo, pair ? nullptr : (const float*)slot, dst, n);
    };
    if (m->n_mlp == 2) {
        merge(cache.h1 + (size_t)s * cache.h1_step, cache.h1_step, f.h1_pair, b.H1 + (size_t)s * M * d1, M * d1, 1024);
        TB2_LAUNCH_CHECK();
    }
    merge(cache.pooled + (size_t)s * cache.pooled_step, cache.pooled_step, f.pooled_pair, ws.pooled, M * P, 512);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// BPTT through social pooling: every track of a scene receives gradient, so the backward runs on
// all M rows (see the kernel comments above for the scatter part).
static int social_backward(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w,
                           const float* observed, int obs_length, const float* truth, int n_decode,
                           const float* positions, const float* states, const float* d_normals,
                           const float* d_positions, const float* d_hidden, const tb2_lstm_grads* g, Workspace& ws,
                           void* bwd_workspace, const TrainCache& cache, cudaStream_t st) {
    const int S = obs_length - 1 + n_decode, S_enc = obs_length - 1;
    const int Mi = l->M, K = m->K_gate, E = m->E, P = m->P, EP = E + P, C = m->C, cells = m->cells;
    const int H = m->H, G4 = 4 * H;
    const int d1 = m->mlp_dims[1];
    const bool two = m->n_mlp == 2;
    const size_t M = (size_t)Mi;
    const int nm1 = l->n_max > 1 ? l->n_max - 1 : 1;
    // a NULL pool field skips its reduction, as in lstm_weight_grads; the d h / d observed chain never reads them
    const bool dw1 = g->pool_embedding_weight0 != nullptr;
    SocBuffers b;
    carve_social(m, l, (size_t)S, bwd_workspace, &b);
    TB2_CHECK_CUDA(cudaMemsetAsync(b.dc, 0, M * H * sizeof(float), st));
    if (dw1) TB2_CHECK_CUDA(cudaMemsetAsync(b.dWt1, 0, (size_t)cells * C * d1 * sizeof(float), st));
    iota_kernel<<<(Mi + 255) / 256, 256, 0, st>>>(b.rows, Mi);
    TB2_LAUNCH_CHECK();
    int rc;
    if ((rc = launch_split_bf16(m->Wt1, b.Wt1_hi, b.Wt1_lo, (size_t)cells * C * d1, st))) return rc;
    const bool rollout = d_positions != nullptr;
    if (rollout && (rc = rollout_begin(l, b.ro, d_normals, d_positions, obs_length, S, g->d_observed, st))) return rc;
    const float* dnorm = rollout ? b.ro.dn : d_normals;
    // (A) forward quantities of every step: hidden1, X = [emb | pooled | h_prev]
    for (int s = 0; s < S; ++s) {
        const float *o1, *o2;
        int phase;
        if ((rc = resolve_step_inputs(l, observed, obs_length, truth, positions, s, &ws, &o1, &o2, &phase, st))) return rc;
        const float* h_prev = s > 0 ? states + ((size_t)(s - 1) * 2 + 0) * M * H : nullptr;
        if ((rc = social_step_records(m, l, b, ws, cache, s, st))) return rc;
        {
            KernelTimer kt("bwd_gather", st);
            bwd_gather_kernel<<<Mi, 256, 0, st>>>(b.rows, Mi, (const float2*)o1, (const float2*)o2, m->We, m->be,
                                                  h_prev, nullptr, nullptr, nullptr, nullptr, nullptr, nm1, C, cells,
                                                  ws.pooled, b.X + (size_t)s * M * K, nullptr,
                                                  b.VEL + (size_t)s * M * 2, b.masked + (size_t)s * M, E, P, K, H);
        }
        TB2_LAUNCH_CHECK();
    }
    // The row GEMMs (rows = all tracks) run on the 3-pass wgmma kernel of the forward (dense_layer_tc_kernel:
    // Y = A . W^T + bias, bf16 (hi, lo) operands, fp32 accumulation) when the shapes allow it: A and the (transposed)
    // weights are split once, the outputs stay fp32.  Other shapes, and TB2_DISABLE_TC=1: cuBLAS / FFMA GEMMs.
    // H % 128: the wgmma row GEMMs of the recurrent d h then use the 128-column tiles the H = 128 build was checked with
    const bool tcg = !m->tc_disabled && H % 128 == 0 && dense_tc_supported(K, G4) && dense_tc_supported(G4, H) &&
                     dense_tc_supported(G4, EP) && (!two || dense_tc_supported(P, d1));
    if (tcg) {
        TB2_CHECK_CUDA(cudaMemsetAsync(b.zero_bias, 0, (size_t)(d1 > G4 ? d1 : G4) * sizeof(float), st));
        for (int phase = 0; phase < 2; ++phase) {
            const float* Wih_p = phase == TB2_PHASE_ENCODER ? w->encoder_weight_ih : w->decoder_weight_ih;
            const float* Whh_p = phase == TB2_PHASE_ENCODER ? w->encoder_weight_hh : w->decoder_weight_hh;
            if ((rc = split2d(Wih_p, EP, G4, EP, b.Wcat_hi[phase], b.Wcat_lo[phase], K, 0, st))) return rc;
            if ((rc = split2d(Whh_p, H, G4, H, b.Wcat_hi[phase], b.Wcat_lo[phase], K, EP, st))) return rc;
            transpose_split_kernel<<<256, 256, 0, st>>>(Whh_p, G4, H, b.WhhT_hi[phase], b.WhhT_lo[phase]);
            TB2_LAUNCH_CHECK();
            transpose_split_kernel<<<512, 256, 0, st>>>(Wih_p, G4, EP, b.WihT_hi[phase], b.WihT_lo[phase]);
            TB2_LAUNCH_CHECK();
        }
        if (two) {
            transpose_split_kernel<<<1024, 256, 0, st>>>(w->pool_embedding_weight[1], P, d1, b.W2T_hi, b.W2T_lo);
            TB2_LAUNCH_CHECK();
        }
        if ((rc = split2d(b.X, K, (size_t)S * M, K, b.X_hi, b.X_lo, K, 0, st))) return rc;
    }
    if ((rc = gate_preactivations(m, b, Mi, S, S_enc, tcg ? &b : nullptr, st))) return rc;
    // (C) reverse time: cell -> input gradient -> grid MLP -> scatter to the neighbours' hidden states
    const size_t place_smem = (size_t)l->n_max * nm1 * sizeof(short);
    TB2_REQUIRE(place_smem <= 200 * 1024 && cells < 32768, "scene too large for the social backward");
    {
        static DynSmemConfig configured;
        TB2_CHECK_CUDA(configured.ensure(pair_place_kernel, place_smem, 48 * 1024));
    }
    int cur = 0;
    for (int s = S - 1; s >= 0; --s, cur ^= 1) {
        const int phase = s < S_enc ? TB2_PHASE_ENCODER : TB2_PHASE_DECODER;
        const float* c_prev = s > 0 ? states + ((size_t)(s - 1) * 2 + 1) * M * H : nullptr;
        const bool last = s == S - 1;
        const int next_phase = (s + 1) < S_enc ? TB2_PHASE_ENCODER : TB2_PHASE_DECODER;
        const float* Whh_next = next_phase == TB2_PHASE_ENCODER ? w->encoder_weight_hh : w->decoder_weight_hh;
        const float* Wih = phase == TB2_PHASE_ENCODER ? w->encoder_weight_ih : w->decoder_weight_ih;
        float* DGs = b.DG + (size_t)s * M * G4;
        float* DXs = b.DXIN + (size_t)s * M * EP;
        const float* Xs = b.X + (size_t)s * M * K;
        // recurrent part of d h: all rows are active, so dgates(s+1) . W_hh is a GEMM (DH1 is free here)
        float* dh_rec = nullptr;
        if (!last) {
            dh_rec = b.DH1;
            if (tcg) {      // dgates(s + 1) was split at the end of the previous iteration
                if ((rc = launch_dense_tc(b.DG_hi[(s + 1) & 1], b.DG_lo[(s + 1) & 1], b.WhhT_hi[next_phase], b.WhhT_lo[next_phase],
                                          b.zero_bias, dh_rec, nullptr, nullptr, Mi, G4, H, 0, st)))
                    return rc;
            } else if ((rc = gemm_nn(b.DG + (size_t)(s + 1) * M * G4, G4, Whh_next, H, dh_rec, H, Mi, H, G4, nullptr,
                                     st)))
                return rc;
        }
        if (rollout && (rc = rollout_fold(l, b.ro, s, S_enc, g->d_observed, st))) return rc;
        {
            KernelTimer kt("bwd_cell_head", st);
            rc = launch_cell_head(H, Mi, st,
                b.rows, b.masked + (size_t)s * M, b.GP + (size_t)s * M * G4, c_prev, nullptr, Whh_next, dh_rec,
                b.pass[cur ^ 1], b.pass[cur], b.dc,
                dnorm + (size_t)s * M * 5, m->Wn, m->bn, DGs, b.HS + (size_t)s * M * H,
                b.DN + (size_t)s * M * 8, d_hidden ? d_hidden + (size_t)s * M * H : nullptr, Mi);
        }
        if (rc) return rc;
        if (tcg) {
            if ((rc = split2d(DGs, G4, M, G4, b.DG_hi[s & 1], b.DG_lo[s & 1], G4, 0, st))) return rc;
            if ((rc = launch_dense_tc(b.DG_hi[s & 1], b.DG_lo[s & 1], b.WihT_hi[phase], b.WihT_lo[phase], b.zero_bias, DXs,
                                      nullptr, nullptr, Mi, G4, EP, 0, st)))
                return rc;
        } else if ((rc = gemm_nn(DGs, G4, Wih, EP, DXs, EP, Mi, EP, G4, nullptr, st))) return rc;
        if (rollout && s >= S_enc &&
            (rc = rollout_inputs(m, l, b.ro, Xs, DXs, nullptr, Mi, b.rows, observed, obs_length, positions, states, s, ws,
                                 g->d_observed, st)))
            return rc;
        const unsigned eb = (unsigned)((M * d1 + 255) / 256);
        if (two) {
            const float* H1s = b.H1 + (size_t)s * M * d1;
            relu_mask_kernel<<<(unsigned)((M * P + 255) / 256), 256, 0, st>>>(Xs, K, DXs, EP, Mi, E, P);   // dz2
            TB2_LAUNCH_CHECK();
            // d hidden1 = dz2 . W2 (torch layout [P, d1] is the [K = P, N = d1] operand), then the ReLU mask
            if (tcg) {
                if ((rc = split2d(DXs + E, EP, M, P, b.DZ2_hi, b.DZ2_lo, P, 0, st))) return rc;
                if ((rc = launch_dense_tc(b.DZ2_hi, b.DZ2_lo, b.W2T_hi, b.W2T_lo, b.zero_bias, b.DH1, nullptr, nullptr, Mi, P, d1,
                                          0, st)))
                    return rc;
            } else if ((rc = gemm_nn(DXs + E, EP, w->pool_embedding_weight[1], d1, b.DH1, d1, Mi, d1, P, nullptr, st))) return rc;
            masked_copy_kernel<<<eb, 256, 0, st>>>(H1s, d1, b.DH1, d1, b.DH1, d1, Mi, d1);
            TB2_LAUNCH_CHECK();
            // dW2 / db2: one reduction over the rows of ALL steps after the loop (dz2 stays in DXIN, hidden1 in H1)
        } else {
            masked_copy_kernel<<<eb, 256, 0, st>>>(Xs + E, K, DXs + E, EP, b.DH1, d1, Mi, d1);
            TB2_LAUNCH_CHECK();
        }
        if ((rc = colsum(b.DH1, d1, Mi, d1, g->pool_embedding_bias0, nullptr, b.scratch, b.scratch_floats, st))) return rc;
        const int* winc = cache.win_count + (size_t)s * M;
        const uint32_t* wine = cache.win_ent + (size_t)s * M * nm1;
        const int* pcell = cache.pair_cell + (size_t)s * M * nm1;
        const uint8_t* pflag = cache.pair_flag + (size_t)s * M * nm1;
        const int* msk = b.masked + (size_t)s * M;
        const float* lat = cache.lat + (size_t)s * M * C;
        {
            KernelTimer kt("social_pair_sort", st);
            pair_count_kernel<<<l->B, 256, cells * sizeof(int), st>>>(l->scene_off, msk, pcell, pflag, nm1, cells,
                                                                       b.counts);
            pair_offsets_kernel<<<1, 1024, cells * sizeof(int), st>>>(b.counts, l->B, cells, b.base, b.start);
            pair_place_kernel<<<l->B, 256, place_smem, st>>>(
                l->scene_off, msk, pcell, pflag, winc, wine, nm1, cells, b.base, b.start, l->pad_to_max, b.sorted);
        }
        TB2_LAUNCH_CHECK();
        switch (C) {
            case 4: rc = social_pair_kernels<4>(m, l, b, lat, nm1, d1, dw1, st); break;
            case 8: rc = social_pair_kernels<8>(m, l, b, lat, nm1, d1, dw1, st); break;
            case 16: rc = social_pair_kernels<16>(m, l, b, lat, nm1, d1, dw1, st); break;
            case 32: rc = social_pair_kernels<32>(m, l, b, lat, nm1, d1, dw1, st); break;
            default: set_error("social latent_dim must be 4, 8, 16 or 32"); return TB2_ERR_UNSUPPORTED;
        }
        if (rc) return rc;
        {
            KernelTimer kt("social_scene_reduce", st);
            social_scene_reduce_kernel<<<l->B, 256, (size_t)l->n_max * C * sizeof(float), st>>>(
                l->scene_off, msk, pflag, nm1, C, b.DGRID, w->pool_encoding_weight, b.DLAT + (size_t)s * M * C,
                s > 0 ? b.pass[cur] : nullptr, H);
        }
        TB2_LAUNCH_CHECK();
    }
    if (two) {
        if ((rc = gemm_tn(b.DXIN + E, EP, b.H1, d1, g->pool_embedding_weight1, d1, S * Mi, P, d1, b.scratch, b.scratch_floats, st)))
            return rc;
        if ((rc = colsum(b.DXIN + E, EP, S * Mi, P, g->pool_embedding_bias1, nullptr, b.scratch, b.scratch_floats, st))) return rc;
    }
    // (D) parameter gradients: one reduction over all (step, row) records per tensor
    if ((rc = lstm_weight_grads(m, w, g, b, Mi, S, S_enc, 0, st))) return rc;
    if (dw1) {
        untranspose_add_kernel<<<2048, 256, 0, st>>>(b.dWt1, g->pool_embedding_weight0, cells, C, d1);
        TB2_LAUNCH_CHECK();
    }
    // lat_j = W_enc h_j + b_enc (gridbased_pooling.py:160-167): h of step s-1 is states[s-1]
    for (int s = 1; s < S; ++s) {
        const float* h_prev = states + ((size_t)(s - 1) * 2 + 0) * M * H;
        if ((rc = gemm_tn(b.DLAT + (size_t)s * M * C, C, h_prev, H, g->pool_encoding_weight, H, Mi, C, H,
                          b.scratch, b.scratch_floats, st)))
            return rc;
    }
    if ((rc = colsum(b.DLAT, C, S * Mi, C, g->pool_encoding_bias, nullptr, b.scratch, b.scratch_floats, st))) return rc;
    // d observed: every track has its record row (rows = row_of = 0 .. M - 1); the grid values are hidden states, whose
    // gradient the chain above already carried into each neighbour's own inputs
    if (g->d_observed &&
        (rc = observed_grads(m, l, b, nullptr, Mi, b.rows, observed, states, S_enc, ws, g->d_observed, st)))
        return rc;
    return TB2_OK;
}
}  // namespace tb2

extern "C" {

size_t tb2_lstm_backward_workspace_bytes(const tb2_lstm* m, const tb2_layout* l, int32_t num_active,
                                         int32_t num_steps) {
    if (!m || !l || num_active < 0 || num_steps < 0) return 0;
    if (m->cfg.pool_type == TB2_POOL_SOCIAL)
        return carve_social(m, l, (size_t)(num_steps > 0 ? num_steps : 1), nullptr, nullptr);
    return carve_bwd(m, (size_t)(num_active > 0 ? num_active : 1), (size_t)(num_steps > 0 ? num_steps : 1),
                     (size_t)l->M, nullptr, nullptr);
}

// tb2_lstm_sequence_backward (d_positions = d_hidden = NULL), tb2_lstm_sequence_backward_dh (d_positions = NULL) and
// tb2_lstm_rollout_backward (d_hidden = NULL)
static int sequence_backward(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w, const float* observed,
                             int32_t obs_length, const float* truth, int32_t n_decode, const float* positions,
                             const float* states, const float* d_normals, const float* d_positions,
                             const float* d_hidden, const int32_t* active_rows, int32_t num_active, const tb2_lstm_grads* g, void* workspace,
                             size_t workspace_bytes, void* bwd_workspace, size_t bwd_workspace_bytes, const void* cache,
                             size_t cache_bytes, void* stream) {
    TB2_REQUIRE(m && l && w && g, "null handle");
    TB2_REQUIRE(m->weights_set, "tb2_lstm_set_weights has not been called");
    TB2_REQUIRE(observed && positions && states && d_normals && active_rows, "null argument");
    TB2_REQUIRE(obs_length >= 2 && n_decode >= 0, "need obs_length >= 2 and n_decode >= 0");
    if (m->G > 0) {
        set_error("training a goal-conditioned model (goal_dim > 0) is not built");
        return TB2_ERR_UNSUPPORTED;
    }
    TB2_REQUIRE(m->cfg.pool_type != TB2_POOL_EXTERNAL, kExternalPoolMessage);
    const bool social = m->cfg.pool_type == TB2_POOL_SOCIAL;
    if (social && !social_trainable(m)) {
        set_error("social training backward supports one_layer / two_layer embeddings with constant = 0");
        return TB2_ERR_UNSUPPORTED;
    }
    if (!social && m->cfg.pool_type != TB2_POOL_NONE &&
        (m->n_mlp != 1 || !m->cfg.pool_to_input || m->cfg.constant != 0.f || m->P > 1024 || m->C > 2)) {
        set_error("training backward supports one_layer grid embeddings with constant = 0 and pool_to_input");
        return TB2_ERR_UNSUPPORTED;
    }
    const int S = obs_length - 1 + n_decode;
    TB2_REQUIRE(workspace && workspace_bytes >= carve_workspace(m, l, nullptr, nullptr), "workspace too small");
    TB2_REQUIRE(bwd_workspace && bwd_workspace_bytes >= tb2_lstm_backward_workspace_bytes(m, l, num_active, S),
                "backward workspace too small");
    TrainCache tc;
    const size_t cache_need = carve_train_cache(m, l, (size_t)S, const_cast<void*>(cache), &tc);
    TB2_REQUIRE(!social || cache, "a social model trains from the cache its tb2_lstm_forward_steps call (cache_dev) filled");
    TB2_REQUIRE(cache_bytes >= cache_need, "training cache too small (tb2_lstm_train_cache_bytes)");
    if (num_active == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    Workspace ws;
    carve_workspace(m, l, workspace, &ws);
    if (social)      // every track of a scene receives gradient: all rows, active_rows is ignored
        return social_backward(m, l, w, observed, obs_length, truth, n_decode, positions, states, d_normals, d_positions,
                               d_hidden, g, ws, bwd_workspace, tc, st);
    const int R = num_active, K = m->K_gate, E = m->E, P = m->P, EP = E + P, H = m->H, G4 = 4 * H;
    const size_t M = (size_t)l->M;
    BwdBuffers b;
    carve_bwd(m, (size_t)R, (size_t)S, M, bwd_workspace, &b);
    TB2_CHECK_CUDA(cudaMemsetAsync(b.dc, 0, (size_t)R * H * sizeof(float), st));
    const int nm1 = l->n_max > 1 ? l->n_max - 1 : 1;
    const bool pooled = m->cfg.pool_type != TB2_POOL_NONE;
    const size_t CG = (size_t)m->C * (size_t)m->cells;
    const int S_enc = obs_length - 1;
    int rc;
    // (A) inputs of every step for the active rows: winners -> X = [emb | pooled | h_prev], grid rows
    for (int s = 0; s < S; ++s) {
        const float *o1, *o2;
        int phase;
        if ((rc = resolve_step_inputs(l, observed, obs_length, truth, positions, s, &ws, &o1, &o2, &phase, st))) return rc;
        const float* h_prev = s > 0 ? states + ((size_t)(s - 1) * 2 + 0) * M * H : nullptr;
        if (pooled && (rc = launch_pool_prepare(m, l, h_prev, o1, o2, 1, 0, 0, &ws, st))) return rc;   // winners
        {
            KernelTimer kt("bwd_gather", st);
            bwd_gather_kernel<<<R, 256, 0, st>>>(active_rows, R, (const float2*)o1, (const float2*)o2, m->We, m->be,
                                                 h_prev, ws.win_count, ws.win_ent, ws.win_val, m->Wt1, m->base1,
                                                 nm1, m->C, m->cells, nullptr, b.X + (size_t)s * R * K,
                                                 pooled ? b.G + (size_t)s * R * CG : nullptr,
                                                 b.VEL + (size_t)s * R * 2, b.masked + (size_t)s * R, E, P, K, H);
        }
        TB2_LAUNCH_CHECK();
    }
    if ((rc = gate_preactivations(m, b, R, S, S_enc, nullptr, st))) return rc;
    if (g->d_observed) {     // the active rows' inputs, and through the directional pairs their neighbours'
        TB2_CHECK_CUDA(cudaMemsetAsync(b.row_of, 0xff, M * sizeof(int), st));
        row_of_kernel<<<(R + 255) / 256, 256, 0, st>>>(active_rows, R, b.row_of);
        TB2_LAUNCH_CHECK();
    }
    const bool rollout = d_positions != nullptr;
    if (rollout && (rc = rollout_begin(l, b.ro, d_normals, d_positions, obs_length, S, g->d_observed, st))) return rc;
    const float* dnorm = rollout ? b.ro.dn : d_normals;
    // (C) the sequential chain: one kernel per step (the rollout backward adds its decoder steps' input gradients)
    int cur = 0;
    for (int s = S - 1; s >= 0; --s, cur ^= 1) {
        const float* c_prev = s > 0 ? states + ((size_t)(s - 1) * 2 + 1) * M * H : nullptr;
        const bool last = s == S - 1;
        const int next_phase = (s + 1) < S_enc ? TB2_PHASE_ENCODER : TB2_PHASE_DECODER;
        const float* Whh_next = next_phase == TB2_PHASE_ENCODER ? w->encoder_weight_hh : w->decoder_weight_hh;
        if (rollout && (rc = rollout_fold(l, b.ro, s, S_enc, g->d_observed, st))) return rc;
        {
            KernelTimer kt("bwd_cell_head", st);
            rc = launch_cell_head(H, R, st,
                active_rows, b.masked + (size_t)s * R, b.GP + (size_t)s * R * G4, c_prev,
                last ? nullptr : b.DG + (size_t)(s + 1) * R * G4, Whh_next, nullptr, b.pass[cur ^ 1], b.pass[cur], b.dc,
                dnorm + (size_t)s * M * 5, m->Wn, m->bn, b.DG + (size_t)s * R * G4,
                b.HS + (size_t)s * R * H, b.DN + (size_t)s * R * 8, d_hidden ? d_hidden + (size_t)s * M * H : nullptr, R);
        }
        if (rc) return rc;
        if (rollout && s >= S_enc) {
            float* DXs = b.DXIN + (size_t)s * R * EP;
            if ((rc = gemm_nn(b.DG + (size_t)s * R * G4, G4, w->decoder_weight_ih, EP, DXs, EP, R, EP, G4, nullptr, st)))
                return rc;
            if ((rc = rollout_inputs(m, l, b.ro, b.X + (size_t)s * R * K, DXs, pooled ? b.G + (size_t)s * R * CG : nullptr,
                                     R, b.row_of, observed, obs_length, positions, states, s, ws, g->d_observed, st)))
                return rc;
        }
    }
    // (D) + (E) input gradients of all steps (the rollout's decoder steps have theirs) and the parameter gradients: one
    // reduction per tensor
    if ((rc = lstm_weight_grads(m, w, g, b, R, S, S_enc, rollout ? 1 << TB2_PHASE_ENCODER : kAllPhases, st))) return rc;
    if (pooled) {
        relu_mask_kernel<<<(unsigned)(((size_t)S * R * P + 255) / 256), 256, 0, st>>>(b.X, K, b.DXIN, EP, S * R, E, P);
        TB2_LAUNCH_CHECK();
        if ((rc = gemm_tn(b.DXIN + E, EP, b.G, (int)CG, g->pool_embedding_weight0, (int)CG, S * R, P, (int)CG,
                          b.scratch, b.scratch_floats, st)))
            return rc;
        if ((rc = colsum(b.DXIN + E, EP, S * R, P, g->pool_embedding_bias0, nullptr, b.scratch, b.scratch_floats, st)))
            return rc;
    }
    if (g->d_observed &&
        (rc = observed_grads(m, l, b, b.G, R, b.row_of, observed, states, S_enc, ws, g->d_observed, st)))
        return rc;
    return TB2_OK;
}

int tb2_lstm_sequence_backward(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w,
                               const float* observed, int32_t obs_length, const float* truth, int32_t n_decode,
                               const float* positions, const float* states, const float* d_normals,
                               const int32_t* active_rows, int32_t num_active, const tb2_lstm_grads* g,
                               void* workspace, size_t workspace_bytes, void* bwd_workspace,
                               size_t bwd_workspace_bytes, const void* cache, size_t cache_bytes, void* stream) {
    return sequence_backward(m, l, w, observed, obs_length, truth, n_decode, positions, states, d_normals, nullptr,
                             nullptr, active_rows, num_active, g, workspace, workspace_bytes, bwd_workspace,
                             bwd_workspace_bytes, cache, cache_bytes, stream);
}

int tb2_lstm_sequence_backward_dh(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w,
                                  const float* observed, int32_t obs_length, const float* truth, int32_t n_decode,
                                  const float* positions, const float* states, const float* d_normals,
                                  const float* d_hidden, const int32_t* active_rows, int32_t num_active,
                                  const tb2_lstm_grads* g, void* workspace, size_t workspace_bytes, void* bwd_workspace,
                                  size_t bwd_workspace_bytes, const void* cache, size_t cache_bytes, void* stream) {
    return sequence_backward(m, l, w, observed, obs_length, truth, n_decode, positions, states, d_normals, nullptr,
                             d_hidden, active_rows, num_active, g, workspace, workspace_bytes, bwd_workspace,
                             bwd_workspace_bytes, cache, cache_bytes, stream);
}

int tb2_lstm_rollout_backward(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w, const float* observed,
                              int32_t obs_length, int32_t n_decode, const float* positions, const float* states,
                              const float* d_normals, const float* d_positions, const int32_t* active_rows,
                              int32_t num_active, const tb2_lstm_grads* g, void* workspace, size_t workspace_bytes,
                              void* bwd_workspace, size_t bwd_workspace_bytes, const void* cache, size_t cache_bytes,
                              void* stream) {
    TB2_REQUIRE(g && g->d_observed && d_positions, "the rollout backward needs d_positions and grads->d_observed");
    return sequence_backward(m, l, w, observed, obs_length, nullptr, n_decode, positions, states, d_normals, d_positions,
                             nullptr, active_rows, num_active, g, workspace, workspace_bytes, bwd_workspace,
                             bwd_workspace_bytes, cache, cache_bytes, stream);
}

size_t tb2_lstm_step_backward_workspace_bytes(const tb2_lstm* m, const tb2_layout* l) {
    if (!m || !l) return 0;
    return carve_step_bwd(m, l, nullptr, nullptr);
}

// One step of the external-module LSTM backward, on all M rows (the module couples the tracks of a scene through their
// hidden states): the gather (bwd_gather_kernel) and gate GEMM of phases (A) / (B), the cell / head kernel of (C) with
// the incoming d h as its recurrent input, and the weight reductions of (D) / (E) over the step's M records.
int tb2_lstm_step_backward(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w, int32_t phase,
                           const float* obs1, const float* obs2, const float* pooled_pad, const float* h_in,
                           const float* c_in, const float* d_h_out, const float* d_c_out, const float* d_normal,
                           float* d_h_in, float* d_c_in, float* d_pooled_pad, const tb2_lstm_grads* g,
                           void* bwd_workspace, size_t bwd_workspace_bytes, void* stream) {
    TB2_REQUIRE(m && l && w && g, "null handle");
    TB2_REQUIRE(m->weights_set, "tb2_lstm_set_weights has not been called");
    TB2_REQUIRE(m->cfg.pool_type == TB2_POOL_EXTERNAL,
                "tb2_lstm_step_backward serves external interaction modules (TB2_POOL_EXTERNAL); the built-in models "
                "train through tb2_lstm_sequence_backward");
    if (m->G > 0) {
        set_error("training a goal-conditioned model (goal_dim > 0) is not built");
        return TB2_ERR_UNSUPPORTED;
    }
    TB2_REQUIRE(phase == TB2_PHASE_ENCODER || phase == TB2_PHASE_DECODER, "bad phase");
    TB2_REQUIRE(obs1 && obs2 && pooled_pad && h_in && c_in && d_h_out && d_c_out && d_normal && d_h_in && d_c_in &&
                    d_pooled_pad, "null argument");
    const bool enc = phase == TB2_PHASE_ENCODER;
    TB2_REQUIRE(w->input_embedding_weight && w->input_embedding_bias && w->hidden2normal_weight && w->hidden2normal_bias &&
                    (enc ? w->encoder_weight_ih && w->encoder_weight_hh : w->decoder_weight_ih && w->decoder_weight_hh),
                "weights of the input embedding, the phase's LSTMCell and hidden2normal are required");
    TB2_REQUIRE(g->input_embedding_weight && g->input_embedding_bias && g->hidden2normal_weight && g->hidden2normal_bias &&
                    (enc ? g->encoder_weight_ih && g->encoder_weight_hh && g->encoder_bias_ih && g->encoder_bias_hh
                         : g->decoder_weight_ih && g->decoder_weight_hh && g->decoder_bias_ih && g->decoder_bias_hh),
                "gradients of the input embedding, the phase's LSTMCell and hidden2normal are required");
    TB2_REQUIRE(bwd_workspace && bwd_workspace_bytes >= carve_step_bwd(m, l, nullptr, nullptr),
                "backward workspace too small (tb2_lstm_step_backward_workspace_bytes)");
    TB2_REQUIRE(((uintptr_t)bwd_workspace & 15) == 0, "backward workspace must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    const int M = l->M, K = m->K_gate, E = m->E, P = m->P, EP = E + P, H = m->H, G4 = 4 * H;
    const bool to_input = m->cfg.pool_to_input != 0;
    StepBwdBuffers b;
    carve_step_bwd(m, l, bwd_workspace, &b);
    int rc;
    iota_kernel<<<(M + 255) / 256, 256, 0, st>>>(b.rows, M);
    TB2_LAUNCH_CHECK();
    // (A) X = [emb | pooled | h_in] (pool_to_input) or [emb | h_in + pooled]: the operand the forward's gate kernel read
    if ((rc = launch_external_pooled(m, l, obs1, obs2, pooled_pad, to_input ? nullptr : h_in,
                                     to_input ? b.pooled : b.h_eff, nullptr, nullptr, st)))
        return rc;
    {
        KernelTimer kt("bwd_gather", st);
        bwd_gather_kernel<<<M, 256, 0, st>>>(b.rows, M, (const float2*)obs1, (const float2*)obs2, m->We, m->be,
                                             to_input ? h_in : b.h_eff, nullptr, nullptr, nullptr, nullptr, nullptr, 1,
                                             m->C, m->cells, to_input ? b.pooled : nullptr, b.X, nullptr, b.VEL,
                                             b.masked, E, P, K, H);
    }
    TB2_LAUNCH_CHECK();
    // (B) gate pre-activations
    if ((rc = gemm_nn(b.X, K, m->WgT[phase], G4, b.GP, G4, M, G4, K, m->bg[phase], st))) return rc;
    // (C) cell + head backward: d h_out enters as the recurrent input, d c_out is updated in place into d c_in
    TB2_CHECK_CUDA(cudaMemsetAsync(b.pass[1], 0, (size_t)M * H * sizeof(float), st));
    if (d_c_in != d_c_out)
        TB2_CHECK_CUDA(cudaMemcpyAsync(d_c_in, d_c_out, (size_t)M * H * sizeof(float), cudaMemcpyDeviceToDevice, st));
    {
        KernelTimer kt("bwd_cell_head", st);
        rc = launch_cell_head(H, M, st, b.rows, b.masked, b.GP, c_in, nullptr, nullptr, d_h_out, b.pass[1], b.pass[0],
                              d_c_in, d_normal, m->Wn, m->bn, b.DG, b.HS, b.DN, nullptr, M);
    }
    if (rc) return rc;
    // (D) + (E) dX_in = dgates . W_ih and the step's weight gradients; d h_in through W_hh
    if ((rc = lstm_weight_grads(m, w, g, b, M, 1, enc ? 1 : 0, kAllPhases, st))) return rc;
    if ((rc = gemm_nn(b.DG, G4, enc ? w->encoder_weight_hh : w->decoder_weight_hh, H, b.DH, H, M, H, G4, nullptr, st)))
        return rc;
    if (g->d_obs1 || g->d_obs2) {     // d obs1 / d obs2 through the step's velocity input
        TB2_REQUIRE(g->d_obs1 && g->d_obs2, "d_obs1 and d_obs2 are set together");
        KernelTimer kt("bwd_input_vel", st);
        input_grad_kernel<false><<<l->B, 256, 0, st>>>(l->scene_off, b.rows, (const float2*)obs1, (const float2*)obs2, b.X,
                                                       K, b.DXIN, EP, E, m->We, nullptr, nullptr, 1, nullptr, 0, nullptr,
                                                       g->d_obs1, g->d_obs2);
        TB2_LAUNCH_CHECK();
    }
    // d pooled: the pooled columns of dX_in, or d (h_in + pooled) = d h_in's recurrent part (pool_to_input = 0)
    return launch_external_step_grads(l, b.masked, to_input ? b.DXIN : b.DH, to_input ? EP : H, to_input ? E : 0,
                                      m->pool_out, b.pass[0], b.DH, H, d_pooled_pad, d_h_in, st);
}

}  // extern "C"
