// Fused recurrence step on the Hopper tensor cores: LSTMCell gate GEMM (wgmma + TMA + mbarrier)
// with the cell update, the Gaussian head and the position feedback in the epilogue.
//
// Same contract as lstm_gates_kernel (csrc/lstm_step.cu; reference LSTM.step lstm.py:118-168,
// torch.nn.LSTMCell, Hidden2Normal modules.py:56-64), specialised for E = 64, H = 64, 128, 192 or 256,
// pool_to_input: gates[M, 4H] = [emb | pooled | h][M, K] . [W_ih | W_hh]^T, K = 64 + P + H.  A goal-conditioned
// model (kGoal) has the goal embedding after emb: [emb | goal_emb | pooled | h], K = 64 + G + P + H, 64 + G a
// multiple of 64, and embed_split writes both embeddings as one [M, 64 + G] operand.
//
// All three K segments arrive as bf16 (hi, lo) pairs written by their producers (embed_split,
// the grid-embedding layer's epilogue, the previous step's epilogue) and the product is the
// 3-pass split  A_hi.W_hi + A_hi.W_lo + A_lo.W_hi  accumulated in fp32 registers.
//
// Grid: (H / 64, ceil(M / 128)) in clusters of H / 64 CTAs along x (set at launch).  The CTAs of a
// cluster share a 128-row tile and rank r owns hidden units [64 r, 64 r + 64) x 4 gates (N = 256;
// W rows are permuted at repack so a CTA's tile holds complete i/f/g/o quadruples).  The mainloop is TcRing (wgmma.cuh)
// with 32-wide k-blocks, each taken from the segment (emb, pooled or h) it falls in: warpgroup 2 is the TMA producer,
// warpgroups 0 and 1 each run wgmma.m64n256k16 on 64 rows.  In the accumulator fragment (wgmma.cuh) the four
// gates of a unit sit in the same thread (columns u, 64 + u, 128 + u, 192 + u), so the epilogue
// updates c / h (fp32 state + bf16 split for the next step) straight from registers and
// accumulates its share of the 5-wide Hidden2Normal dot products; the four threads of a row add
// theirs with shuffles, ranks 1 .. H/64 - 1 ship their partial sums to rank 0 through distributed
// shared memory and rank 0 adds them in rank order and finishes mu / sigma / rho and the fed-back
// position.
#include <cuda.h>
#include <cuda_bf16.h>
#include <math_constants.h>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "wgmma.cuh"

namespace tb2 {

constexpr int kGtBM = 128;
constexpr int kGtBN = 256;          // 64 units x 4 gates
// 32-wide k-blocks (64-byte rows, 64B swizzle): 48 KB a stage, so a 3-stage ring fits beside the epilogue's shared
// memory (the cell state it reads is staged there too) and two stages' loads can be in flight behind the one being
// multiplied
constexpr int kGtBK = 32;
using GateRing = TcRing<kGtBM, kGtBN, kGtBK, 3>;
constexpr int kGtThreads = 384;     // two MMA + epilogue warpgroups, one producer warpgroup

// Gate non-linearities on the SFU (ex2.approx, ~2 ulp) -- the epilogue was bound by the ~200
// instructions per hidden unit of the libm-accurate expf / tanhf.  Absolute error ~1e-7 per
// activation, the same order as fp32 summation-order noise; parity is re-measured in the tests.
__device__ __forceinline__ float g_sigmoid(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float g_tanh(float x) { return 1.f - __fdividef(2.f, __expf(2.f * x) + 1.f); }

struct GateTcParams {
    SplitMap emb, pool, h;      // A segments [M, 64 + G], [M, P], [M, H]
    SplitMap w;                 // [4H (rank, gate, unit), K]
    const float2* obs1;
    const float2* obs2;
    const float* h_in;          // [M, H] fp32 state before the step
    const float* c_in;
    float* h_out;
    float* c_out;
    __nv_bfloat16* hs_out_hi;   // [M, H] split of h_out for the next step
    __nv_bfloat16* hs_out_lo;
    float* normal_out;          // [M, 5]
    float2* pos_out;            // [M] or null
    const float* bg;            // [4H] b_ih + b_hh, original gate order
    const float* Wn;            // [5, H]
    const float* bn;            // [5]
    int M, P;
    int G;                      // goal embedding width (kGoal instances only)
};

// R = cluster size = H / 64 (1 to 4; a cluster of one at H = 64): the strides and the rank loop of the epilogue are compile-time constants
template <int R, bool kGoal>
__global__ void __launch_bounds__(kGtThreads, 1)
lstm_gates_tc_kernel(const __grid_constant__ GateTcParams p) {
    extern __shared__ __align__(1024) unsigned char smem_gt[];
    __shared__ GateRing tc;
    __shared__ float wn_s[5][64];          // Hidden2Normal weights of this CTA's 64 units
    __shared__ float bg_s[4][64];          // fused gate bias of this CTA's units
    constexpr int H = 64 * R;
    __shared__ float peer_part[R > 1 ? R - 1 : 1][kGtBM][5];  // rank 0: partial head sums of ranks 1, 2, ..
    // c_in of each consumer thread's 16 (row, unit pair) slots, [slot][thread], copied during the mainloop: read from
    // global memory in the epilogue, each load would wait behind the previous slot's stores (possible aliasing)
    __shared__ float2 c_s[16][256];
    __shared__ float2 obs_s[kGtBM][2];     // obs1, obs2 of the tile's rows, copied with c_s

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = blockIdx.x;           // cluster rank == n-tile: units [64 rank, 64 rank + 64)
    const int m0 = blockIdx.y * kGtBM;
    const int kb_pool = p.P / kGtBK;       // k-blocks: [emb (+ goal_emb) x kb_emb | pooled x kb_pool | h x H / 32]
    const int kb_emb = (64 + (kGoal ? p.G : 0)) / kGtBK;
    const int num_kb = kb_emb + kb_pool + H / kGtBK;
    const uint32_t ring = (smem_u32(smem_gt) + 1023u) & ~1023u;

    for (int i = threadIdx.x; i < 5 * 64; i += kGtThreads) wn_s[i / 64][i % 64] = p.Wn[(i / 64) * H + rank * 64 + (i % 64)];
    for (int i = threadIdx.x; i < 4 * 64; i += kGtThreads) bg_s[i / 64][i % 64] = p.bg[(i / 64) * H + rank * 64 + (i % 64)];

    if (threadIdx.x == 0) tc.init();
    __syncthreads();
    grid_dep_wait();          // embedding / pooled / state operands come from the previous kernels
    grid_dep_launch();
    // cluster barrier phase 1 (arrive now, wait before the first DSMEM access): a CTA may only
    // touch its peer's shared memory once the peer is known to be resident
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    bool waited_phase1 = false;

    // rows (rl, rl + 8) of the tile and their quarter-row share of the head sums (consumer threads)
    const int rl = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    if (wg < 2) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int row = m0 + rl + 8 * hr;
            if (row >= p.M) continue;
            if ((lane & 3) == 0) {
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;"
                             ::"r"(smem_u32(&obs_s[rl + 8 * hr][0])), "l"(p.obs1 + row) : "memory");
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;"
                             ::"r"(smem_u32(&obs_s[rl + 8 * hr][1])), "l"(p.obs2 + row) : "memory");
            }
#pragma unroll
            for (int n8 = 0; n8 < 8; ++n8)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;"
                             ::"r"(smem_u32(&c_s[8 * hr + n8][threadIdx.x])),
                               "l"(p.c_in + (size_t)row * H + rank * 64 + 8 * n8 + 2 * (lane & 3)) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    float part[2][5] = {{0.f, 0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f, 0.f}};

    float acc[kGtBN / 2];
    tc.run(ring, num_kb, m0, [&](int kb) {
        if (kb < kb_emb) return TcATile{&p.emb, kb * kGtBK};
        if (kb < kb_emb + kb_pool) return TcATile{&p.pool, (kb - kb_emb) * kGtBK};
        return TcATile{&p.h, (kb - kb_emb - kb_pool) * kGtBK};
    }, p.w, rank * kGtBN, acc);
    if (wg < 2) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");       // this thread's c_s slots and its rows' obs_s
        asm volatile("bar.sync 1, 256;" ::: "memory");             // obs_s rows copied by the other threads of a quad
        // gate g of unit u = 8 n8 + 2 (lane % 4) + j, row rl + 8 hr: acc[4 (8 g + n8) + 2 hr + j]
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int row = m0 + rl + 8 * hr;
            if (row >= p.M || (TB2_GEMM_ABLATE == 3 && p.M > 0)) continue;
            const float2 o1 = obs_s[rl + 8 * hr][0], o2 = obs_s[rl + 8 * hr][1];
            const bool masked = isnan(o1.x) || isnan(o2.x);                  // lstm.py:118
#pragma unroll
            for (int n8 = 0; n8 < 8; ++n8) {
                const int u = 8 * n8 + 2 * (lane & 3);
                const size_t o = (size_t)row * H + rank * 64 + u;
                float2 c = c_s[8 * hr + n8][threadIdx.x];
                float2 h;
                if (!masked) {
                    float cn[2], hn[2];
                    const float cc[2] = {c.x, c.y};
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int r = 4 * n8 + 2 * hr + j;
                        const float ig = g_sigmoid(acc[r] + bg_s[0][u + j]);
                        const float fg = g_sigmoid(acc[r + 32] + bg_s[1][u + j]);
                        const float gt = g_tanh(acc[r + 64] + bg_s[2][u + j]);
                        const float og = g_sigmoid(acc[r + 96] + bg_s[3][u + j]);
                        cn[j] = fg * cc[j] + ig * gt;
                        hn[j] = og * g_tanh(cn[j]);
#pragma unroll
                        for (int q = 0; q < 5; ++q) part[hr][q] = fmaf(hn[j], wn_s[q][u + j], part[hr][q]);
                    }
                    c = make_float2(cn[0], cn[1]);
                    h = make_float2(hn[0], hn[1]);
                } else {
                    // absent track: state copied through unchanged (lstm.py:158-166)
                    h = *reinterpret_cast<const float2*>(p.h_in + o);
                }
                *reinterpret_cast<float2*>(p.h_out + o) = h;
                *reinterpret_cast<float2*>(p.c_out + o) = c;
                split_bf16x2(h, *reinterpret_cast<uint32_t*>(p.hs_out_hi + o),
                             *reinterpret_cast<uint32_t*>(p.hs_out_lo + o));
            }
        }
        // the four threads of a row add their shares (fixed order: deterministic)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr)
#pragma unroll
            for (int q = 0; q < 5; ++q) {
                part[hr][q] += __shfl_xor_sync(0xffffffffu, part[hr][q], 1);
                part[hr][q] += __shfl_xor_sync(0xffffffffu, part[hr][q], 2);
            }
        if (rank > 0) {
            asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");     // phase 1: rank 0 is resident
            waited_phase1 = true;
            // ship this rank's head sums to rank 0 through distributed shared memory
            if ((lane & 3) == 0) {
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
                    const uint32_t local = smem_u32(&peer_part[rank - 1][rl + 8 * hr][0]);
                    uint32_t remote;
                    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(0));
#pragma unroll
                    for (int q = 0; q < 5; ++q)
                        asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(remote + 4 * q), "f"(part[hr][q]) : "memory");
                }
            }
            __syncwarp();
        }
    }
    // cluster barrier phase 2: the other ranks' partial sums are visible in rank 0's shared memory afterwards
    if (!waited_phase1) asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    if (wg < 2 && rank == 0 && (lane & 3) == 0) {
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            const int row = m0 + rl + 8 * hr;
            if (row >= p.M || (TB2_GEMM_ABLATE == 3 && p.M > 0)) continue;
            float* no = p.normal_out + (size_t)row * 5;
            const float2 o1 = obs_s[rl + 8 * hr][0], o2 = obs_s[rl + 8 * hr][1];
            if (isnan(o1.x) || isnan(o2.x)) {
#pragma unroll
                for (int q = 0; q < 5; ++q) no[q] = CUDART_NAN_F;
                if (p.pos_out) p.pos_out[row] = make_float2(CUDART_NAN_F, CUDART_NAN_F);
            } else {
                float s[5];
#pragma unroll
                for (int q = 0; q < 5; ++q) {
                    s[q] = part[hr][q];
#pragma unroll
                    for (int r = 1; r < R; ++r) s[q] += peer_part[r - 1][rl + 8 * hr][q];
                    s[q] += p.bn[q];
                }
                const float n0 = s[0], n1 = s[1];
                no[0] = n0;
                no[1] = n1;
                no[2] = 0.01f + 0.2f * g_sigmoid(s[2]);                           // modules.py:60-62
                no[3] = 0.01f + 0.2f * g_sigmoid(s[3]);
                no[4] = 0.7f * g_sigmoid(s[4]);
                if (p.pos_out) p.pos_out[row] = make_float2(o2.x + n0, o2.y + n1);   // lstm.py:232,255
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// producers of the split operands
// ------------------------------------------------------------------------------------------
// emb[M, 64] = cat(relu(W_e . (4 v) + b_e), 0, 0) as bf16 (hi, lo)   (modules.py:24-30); kGoal: [M, E + G] rows
// [emb | cat(relu(W_g . (4 d) + b_g), 0, 0)], d = (obs2 - goal) / |obs2 - goal|, 0 at norm 0 (lstm.py:131-139)
struct GoalEmbed {
    const float2* goals;
    const float* Wg;
    const float* bg;
    int G;
};

template <bool kGoal>
__global__ void embed_split_kernel(const float2* __restrict__ obs1, const float2* __restrict__ obs2,
                                   const float* __restrict__ We, const float* __restrict__ be,
                                   __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int M, int E,
                                   GoalEmbed ge) {
    grid_dep_wait();
    grid_dep_launch();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int W = kGoal ? E + ge.G : E;
    if (idx >= M * W) return;
    const int m = idx / W, k = idx - m * W;
    const float2 a = obs1[m], b = obs2[m];
    float v = 0.f;
    if (k < E - 2 && !(isnan(a.x) || isnan(b.x))) {
        const float vx = (b.x - a.x) * 4.0f, vy = (b.y - a.y) * 4.0f;
        v = fmaxf(fmaf(We[2 * k + 1], vy, fmaf(We[2 * k], vx, be[k])), 0.f);
    } else if (kGoal && k >= E && k < W - 2 && !(isnan(a.x) || isnan(b.x))) {
        const int kg = k - E;
        const float2 g = ge.goals[m];
        const float dx = b.x - g.x, dy = b.y - g.y;
        const float n = sqrtf(dx * dx + dy * dy);
        const float gx = n != 0.f ? dx / n : 0.f, gy = n != 0.f ? dy / n : 0.f;
        v = fmaxf(fmaf(ge.Wg[2 * kg + 1], gy * 4.0f, fmaf(ge.Wg[2 * kg], gx * 4.0f, ge.bg[kg])), 0.f);
    }
    split_bf16(v, hi[idx], lo[idx]);
}

// W_cat[n][k] = [W_ih | W_hh] with rows permuted to (rank, gate, unit) order, as bf16 (hi, lo)
__global__ void repack_gates_tc_kernel(const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                                       __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                       int in_dim, int H) {
    const int K = in_dim + H;
    size_t total = (size_t)4 * H * K;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (size_t)gridDim.x * blockDim.x) {
        const int k = (int)(idx % K);
        const int n = (int)(idx / K);                 // permuted row: rank * 256 + gate * 64 + ul
        const int rank = n / 256, gate = (n % 256) / 64, ul = n % 64;
        const int src = gate * H + rank * 64 + ul;    // original gate column
        const float v = k < in_dim ? w_ih[(size_t)src * in_dim + k] : w_hh[(size_t)src * H + (k - in_dim)];
        split_bf16(v, hi[idx], lo[idx]);
    }
}

// the segments are whole multiples of 64 columns (two k-blocks), the widths the kernel has always taken
bool gates_tc_supported(const tb2_lstm* m) {
    if (m->H % 64 != 0 || m->E != 64 || (m->E + m->G) % 64 != 0) return false;
    if (m->cfg.pool_type != TB2_POOL_NONE && !m->cfg.pool_to_input) return false;
    if (m->P % 64 != 0) return false;
    return true;
}

int launch_repack_gates_tc(const float* w_ih, const float* w_hh, void* hi, void* lo, int in_dim, int H,
                           cudaStream_t st) {
    repack_gates_tc_kernel<<<512, 256, 0, st>>>(w_ih, w_hh, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, in_dim, H);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int launch_embed_split(const tb2_lstm* m, int M, const float* obs1, const float* obs2, const float* goals, void* hi,
                       void* lo, cudaStream_t st) {
    const int total = M * (m->E + m->G);
    const GoalEmbed ge{(const float2*)goals, m->Wgl, m->bgl, m->G};
    {
        KernelTimer kt("embed_split", st);
        launch_pdl(m->G > 0 ? embed_split_kernel<true> : embed_split_kernel<false>, dim3((total + 255) / 256), dim3(256), 0,
                   st, (const float2*)obs1, (const float2*)obs2, (const float*)m->We, (const float*)m->be,
                   (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, M, m->E, ge);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int launch_gates_tc(const tb2_lstm* m, const tb2_layout* l, int phase, const float* obs1, const float* obs2,
                    const void* emb_hi, const void* emb_lo, const void* pool_hi, const void* pool_lo,
                    const void* hs_in_hi, const void* hs_in_lo, void* hs_out_hi, void* hs_out_lo,
                    const float* h_in, const float* c_in, float* h_out, float* c_out, float* normal_out,
                    float* pos_out, cudaStream_t st) {
    const int M = l->M;
    GateTcParams p;
    int rc;
    if ((rc = make_split_map(&p.emb, emb_hi, emb_lo, M, 64 + m->G, kGtBM, kGtBK))) return rc;
    if (m->P > 0) {
        if ((rc = make_split_map(&p.pool, pool_hi, pool_lo, M, m->P, kGtBM, kGtBK))) return rc;
    } else {
        p.pool = p.emb;
    }
    if ((rc = make_split_map(&p.h, hs_in_hi, hs_in_lo, M, m->H, kGtBM, kGtBK))) return rc;
    if ((rc = make_split_map(&p.w, m->Wg_hi[phase], m->Wg_lo[phase], 4 * m->H, m->K_gate, kGtBN, kGtBK))) return rc;
    p.obs1 = (const float2*)obs1;
    p.obs2 = (const float2*)obs2;
    p.h_in = h_in; p.c_in = c_in; p.h_out = h_out; p.c_out = c_out;
    p.hs_out_hi = (__nv_bfloat16*)hs_out_hi; p.hs_out_lo = (__nv_bfloat16*)hs_out_lo;
    p.normal_out = normal_out;
    p.pos_out = (float2*)pos_out;
    p.bg = m->bg[phase];
    p.Wn = m->Wn;
    p.bn = m->bn;
    p.M = M;
    p.P = m->P;
    p.G = m->G;
    // one instance per cluster size R = H / 64 and goal input, each configured for its shared memory on its own
    static void (*const kernels[4][2])(GateTcParams) = {
        {lstm_gates_tc_kernel<1, false>, lstm_gates_tc_kernel<1, true>},
        {lstm_gates_tc_kernel<2, false>, lstm_gates_tc_kernel<2, true>},
        {lstm_gates_tc_kernel<3, false>, lstm_gates_tc_kernel<3, true>},
        {lstm_gates_tc_kernel<4, false>, lstm_gates_tc_kernel<4, true>}};
    static DynSmemConfig configured[4][2];
    const int R = m->H / 64;
    if (m->H % 64 != 0 || R < 1 || R > 4) {
        set_error(kHiddenDimMessage);
        return TB2_ERR_UNSUPPORTED;
    }
    const int goal = p.G > 0;
    TB2_CHECK_CUDA(configured[R - 1][goal].ensure(kernels[R - 1][goal], GateRing::kSmemBytes));
    {
        KernelTimer kt("lstm_gates_tc", st);
        launch_pdl_cluster(kernels[R - 1][goal], dim3(R, (M + kGtBM - 1) / kGtBM), dim3(kGtThreads), GateRing::kSmemBytes,
                           st, (unsigned)R, p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // namespace tb2
