// HiddenStateMLPPooling on the device (--type hiddenstatemlp, the Social-GAN pooling module).
//
//   pooled_i = max over ALL tracks j of the scene (j = i included) of
//                [ relu(Ws (pos_j - pos_i) + bs) | relu(Wh h_j + bh) | relu(Wv 4 (v_j - v_i) + bv) ]
//              with -100 where an input of the embedding is NaN,
//   out_i    = Wo pooled_i + bo
//   (reference: trajnetbaselines/lstm/non_gridbased_pooling.py:49-58 embed_with_masking, :150-239)
//
// One CTA per scene: the pair terms are 2-input Linears (N^2 x 64 x 2 FMAs), the hidden embedding and the output
// projection are N x 128 x {64, out_dim} -- a few hundred kFLOP per scene, FP32 FFMA, no tensor cores.  The
// reference materialises [B, N, N, 128] tensors and three masked scatters per step.
#include <math_constants.h>

#include "common.cuh"

namespace tb2 {

constexpr int kMpThreads = 256;

struct MlpPoolParams {
    const float2* obs1;
    const float2* obs2;
    const float* hidden;      // [M, H]
    const int* scene_off;
    const float* Ws;          // [ds, 2]
    const float* bs;
    const float* Wv;          // [dv, 2]
    const float* bv;
    const float* WhT;         // [H, dh]
    const float* bh;
    const float* WoT;         // [ds + dh + dv, out_dim]
    const float* bo;
    float* out;               // [M, out_dim]
    int H, ds, dv, dh, out_dim;
};

__global__ void __launch_bounds__(kMpThreads) hidden_mlp_pool_kernel(MlpPoolParams p) {
    extern __shared__ __align__(16) float smem_mp[];
    const int scene = blockIdx.x;
    const int row0 = p.scene_off[scene];
    const int n = p.scene_off[scene + 1] - row0;
    const int D = p.ds + p.dh + p.dv;
    float2* pos = reinterpret_cast<float2*>(smem_mp);              // [n] obs2 (NaN kept)
    float2* vel = pos + n;                                         // [n] obs2 - obs1 (NaN if either is)
    float* hemb = reinterpret_cast<float*>(vel + n);               // [n][dh]
    float* hmax = hemb + (size_t)n * p.dh;                         // [dh]
    float* pooled = hmax + p.dh;                                   // [n][D]
    const int tid = threadIdx.x;
    grid_dep_wait();
    grid_dep_launch();
    for (int j = tid; j < n; j += kMpThreads) {
        const float2 a = p.obs1[row0 + j], b = p.obs2[row0 + j];
        pos[j] = b;
        vel[j] = make_float2(b.x - a.x, b.y - a.y);
    }
    // hidden embedding of every track (a row with a NaN is masked to -100)
    for (int idx = tid; idx < n * p.dh; idx += kMpThreads) {
        const int j = idx / p.dh, k = idx - j * p.dh;
        const float* h = p.hidden + (size_t)(row0 + j) * p.H;
        float acc = 0.f;
        bool bad = false;
        for (int c = 0; c < p.H; ++c) {
            const float hv = __ldg(h + c);
            bad |= isnan(hv);
            acc = fmaf(hv, __ldg(p.WhT + (size_t)c * p.dh + k), acc);
        }
        hemb[idx] = bad ? -100.f : fmaxf(acc + p.bh[k], 0.f);
    }
    __syncthreads();
    for (int k = tid; k < p.dh; k += kMpThreads) {
        float m = -CUDART_INF_F;
        for (int j = 0; j < n; ++j) m = fmaxf(m, hemb[j * p.dh + k]);
        hmax[k] = m;
    }
    __syncthreads();
    // pooled[i] = [spatial | hidden | velocity]
    for (int idx = tid; idx < n * D; idx += kMpThreads) {
        const int i = idx / D, k = idx - i * D;
        float m;
        if (k >= p.ds && k < p.ds + p.dh) {
            m = hmax[k - p.ds];
        } else {
            const bool sp = k < p.ds;
            const int kk = sp ? k : k - p.ds - p.dh;
            const float w0 = sp ? p.Ws[2 * kk] : p.Wv[2 * kk], w1 = sp ? p.Ws[2 * kk + 1] : p.Wv[2 * kk + 1];
            const float b = sp ? p.bs[kk] : p.bv[kk];
            const float2 ci = sp ? pos[i] : vel[i];
            const float scale = sp ? 1.f : 4.f;
            m = -CUDART_INF_F;
            for (int j = 0; j < n; ++j) {
                const float2 cj = sp ? pos[j] : vel[j];
                const float rx = (cj.x - ci.x) * scale, ry = (cj.y - ci.y) * scale;
                float e = -100.f;                                  // embed_with_masking fill value
                if (!(isnan(rx) || isnan(ry))) e = fmaxf(fmaf(ry, w1, fmaf(rx, w0, b)), 0.f);
                m = fmaxf(m, e);
            }
        }
        pooled[idx] = m;
    }
    __syncthreads();
    for (int idx = tid; idx < n * p.out_dim; idx += kMpThreads) {
        const int i = idx / p.out_dim, o = idx - i * p.out_dim;
        const float* pi = pooled + (size_t)i * D;
        float a0 = 0.f, a1 = 0.f;
        int k = 0;
        for (; k + 1 < D; k += 2) {
            a0 = fmaf(pi[k], __ldg(p.WoT + (size_t)k * p.out_dim + o), a0);
            a1 = fmaf(pi[k + 1], __ldg(p.WoT + (size_t)(k + 1) * p.out_dim + o), a1);
        }
        if (k < D) a0 = fmaf(pi[k], __ldg(p.WoT + (size_t)k * p.out_dim + o), a0);
        p.out[(size_t)(row0 + i) * p.out_dim + o] = (a0 + a1) + p.bo[o];
    }
}

int launch_hidden_mlp_pool(const tb2_lstm* m, const tb2_layout* l, const float* hidden, const float* obs1,
                           const float* obs2, float* out, cudaStream_t st) {
    MlpPoolParams p;
    p.obs1 = (const float2*)obs1;
    p.obs2 = (const float2*)obs2;
    p.hidden = hidden;
    p.scene_off = l->scene_off;
    p.Ws = m->mp_Ws; p.bs = m->mp_bs; p.Wv = m->mp_Wv; p.bv = m->mp_bv;
    p.WhT = m->mp_WhT; p.bh = m->mp_bh; p.WoT = m->mp_WoT; p.bo = m->mp_bo;
    p.out = out;
    p.H = m->H;
    p.ds = m->cfg.mlp_dim_spatial; p.dv = m->cfg.mlp_dim_vel; p.dh = m->cfg.mlp_dim_hidden;
    p.out_dim = m->pool_out;
    const int D = p.ds + p.dh + p.dv;
    const size_t smem = ((size_t)l->n_max * (4 + p.dh + D) + p.dh) * sizeof(float) + 16;
    TB2_REQUIRE(smem <= 200 * 1024, "scene too large for the hidden-state MLP pooling kernel");
    static DynSmemConfig configured;
    TB2_CHECK_CUDA(configured.ensure(hidden_mlp_pool_kernel, smem, 48 * 1024));
    {
        KernelTimer kt("hidden_mlp_pool", st);
        launch_pdl(hidden_mlp_pool_kernel, dim3(l->B), dim3(kMpThreads), smem, st, p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// ------------------------------------------------------------------------------------------
// AttentionMLPPooling on the device (--type attentionmlp, reference non_gridbased_pooling.py:242-351).
//
//   e_ij = [ relu(Ws (pos_j - pos_i) + bs) | relu(Wh h_j + bh) | relu(Wv 4 (v_j - v_i) + bv) ]   (NaN input -> fill / 0 / fill)
//   for track i: query from e_ii, keys / values from e_ij over EVERY slot j of the (padded) scene,
//   q = (Aq e + bq) / sqrt(E), k = Ak e + bk, v = Av e + bv with A* = in-projection . w{q,k,v} (combined at
//   tb2_lstm_set_weights), out_i = Wout (Wo (softmax_j(q_i . k_ij) v_ij) + bo) + bout.
//
// The key / value maps are linear, so the whole pair part is folded:
//   q_i . k_ij = u_i . e_ij + q_i . bk,   u_i = Ak^T q_i   (per track, not per pair; q_i . bk is the same for every j
//                                                            and cancels in the softmax, so it is dropped)
//   sum_j a_ij v_ij = Av (sum_j a_ij e_ij) + bv             (the weights a_ij sum to 1)
// which leaves ~4 E operations per pair instead of 2 x E x E.  One CTA per scene, one warp per track, online softmax.
// Shared memory holds what every warp reads -- pos, vel and the hidden embedding of every slot, (4 + dh) floats per
// slot -- and the queries / attention outputs of one chunk of 32 tracks (2 x 32 x E floats), whose projections run over
// the whole CTA; a scene of (200 KB - 32 KB) / ((4 + dh) x 4 B) slots fits: 632 at the default widths (dh = 64).
// ------------------------------------------------------------------------------------------
struct AttnPoolParams {
    const float2* obs1;
    const float2* obs2;
    const float* hidden;
    const int* scene_off;
    const float *Ws, *bs, *Wv, *bv, *WhT, *bh;      // embeddings (WhT [H][dh])
    const float *AqT, *Ak, *AvT, *bqkv;             // [E][E]: Aq, Av transposed (input-major), Ak output-major; biases [3E]
    const float *WoT, *bo;                          // attention out-projection [E][E] transposed, [E]
    const float *WoutT, *bout;                      // out_projection [E][out_dim] transposed, [out_dim]
    float* out;
    int H, ds, dv, dh, out_dim, n_max, pad_to_max;
    float fill;
};

constexpr int kAtThreads = 256, kAtWarps = kAtThreads / 32, kAtChunk = 32;

__global__ void __launch_bounds__(kAtThreads) attn_mlp_pool_kernel(AttnPoolParams p) {
    extern __shared__ __align__(16) float smem_at[];
    const int scene = blockIdx.x;
    const int row0 = p.scene_off[scene];
    const int n = p.scene_off[scene + 1] - row0;
    const int ns = p.pad_to_max ? p.n_max : n;                     // slots of the sequence (padded slots are absent tracks)
    const int E = p.ds + p.dh + p.dv, dsh = p.ds + p.dh;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float* qb = smem_at;                                           // [kAtChunk][E] scaled queries, later Wo att + bo
    float* ab = qb + (size_t)kAtChunk * E;                         // [kAtChunk][E] attention outputs
    float2* pos = reinterpret_cast<float2*>(ab + (size_t)kAtChunk * E);   // [ns] obs2 (NaN for padded slots)
    float2* vel = pos + ns;                                        // [ns] 4 x velocity is applied at use
    float* hemb = reinterpret_cast<float*>(vel + ns);              // [ns][dh]  (0 for absent rows)
    const float scale = rsqrtf((float)E);
    grid_dep_wait();
    grid_dep_launch();
    for (int j = tid; j < ns; j += kAtThreads) {
        float2 a = make_float2(CUDART_NAN_F, CUDART_NAN_F), b = a;
        if (j < n) { a = p.obs1[row0 + j]; b = p.obs2[row0 + j]; }
        pos[j] = b;
        vel[j] = make_float2(b.x - a.x, b.y - a.y);
    }
    // hidden embedding of every slot (a row with a NaN, or a padded slot, embeds to 0)
    for (int idx = tid; idx < ns * p.dh; idx += kAtThreads) {
        const int j = idx / p.dh, k = idx - j * p.dh;
        float val = 0.f;
        if (j < n) {
            const float* h = p.hidden + (size_t)(row0 + j) * p.H;
            float acc = 0.f;
            bool bad = false;
            for (int c = 0; c < p.H; ++c) {
                const float hv = __ldg(h + c);
                bad |= isnan(hv);
                acc = fmaf(hv, __ldg(p.WhT + (size_t)c * p.dh + k), acc);
            }
            val = bad ? 0.f : fmaxf(acc + p.bh[k], 0.f);
        }
        hemb[idx] = val;
    }
    __syncthreads();
    // the tracks in chunks of kAtChunk: the projections run over the whole CTA, the attention one warp per track
    for (int i0 = 0; i0 < n; i0 += kAtChunk) {
        const int nc = min(kAtChunk, n - i0);
        // q_i = (Aq e_ii + bq) / sqrt(E), e_ii = [relu(bs) | hemb_i | relu(bv)] (fill where the track itself is absent)
        for (int idx = tid; idx < nc * E; idx += kAtThreads) {
            const int t = idx / E, o = idx - t * E, i = i0 + t;
            const bool pbad = isnan(pos[i].x) || isnan(pos[i].y), vbad = isnan(vel[i].x) || isnan(vel[i].y);
            float acc = p.bqkv[o];
            for (int c = 0; c < p.ds; ++c) acc = fmaf(__ldg(p.AqT + (size_t)c * E + o), pbad ? p.fill : fmaxf(p.bs[c], 0.f), acc);
            for (int c = 0; c < p.dh; ++c) acc = fmaf(__ldg(p.AqT + (size_t)(p.ds + c) * E + o), hemb[i * p.dh + c], acc);
            for (int c = 0; c < p.dv; ++c)
                acc = fmaf(__ldg(p.AqT + (size_t)(dsh + c) * E + o), vbad ? p.fill : fmaxf(p.bv[c], 0.f), acc);
            qb[idx] = acc * scale;
        }
        __syncthreads();
        // attention of track i over the slots j: lane owns the features c = lane + 32 r (r < 4) of e_ij = [spatial | hidden | velocity]
        for (int t = warp; t < nc; t += kAtWarps) {
            const int i = i0 + t;
            const float* qi = qb + (size_t)t * E;
            float u[4] = {0.f, 0.f, 0.f, 0.f};                       // u_i[c] = sum_o q_i[o] Ak[o][c]
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int c = lane + 32 * r;
                if (c < E) {
                    float acc = 0.f;
                    for (int o = 0; o < E; ++o) acc = fmaf(qi[o], __ldg(p.Ak + (size_t)o * E + c), acc);
                    u[r] = acc;
                }
            }
            const float2 pi = pos[i], vi = vel[i];
            float m_run = -CUDART_INF_F, l_run = 0.f;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            for (int j = 0; j < ns; ++j) {
                const float rx = pos[j].x - pi.x, ry = pos[j].y - pi.y;
                const float wx = (vel[j].x - vi.x) * 4.f, wy = (vel[j].y - vi.y) * 4.f;
                const bool pbad = isnan(rx) || isnan(ry), vbad = isnan(wx) || isnan(wy);
                float f[4] = {0.f, 0.f, 0.f, 0.f};
                float part = 0.f;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int c = lane + 32 * r;
                    if (c < p.ds) f[r] = pbad ? p.fill : fmaxf(fmaf(ry, p.Ws[2 * c + 1], fmaf(rx, p.Ws[2 * c], p.bs[c])), 0.f);
                    else if (c < dsh) f[r] = hemb[(size_t)j * p.dh + (c - p.ds)];
                    else if (c < E) {
                        const int cv = c - dsh;
                        f[r] = vbad ? p.fill : fmaxf(fmaf(wy, p.Wv[2 * cv + 1], fmaf(wx, p.Wv[2 * cv], p.bv[cv])), 0.f);
                    }
                    part = fmaf(u[r], f[r], part);
                }
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) part += __shfl_xor_sync(0xffffffffu, part, off);
                const float m_new = fmaxf(m_run, part);
                const float corr = __expf(m_run - m_new), a = __expf(part - m_new);  // first slot: corr = exp(-inf) = 0
                l_run = l_run * corr + a;
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[r] = acc[r] * corr + a * f[r];
                m_run = m_new;
            }
            const float inv = 1.f / l_run;
            // att_i = Av (sum_j a_ij e_ij) + bv   (features are spread over the lanes: broadcast each one)
            float o4[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int o = lane + 32 * r;
                o4[r] = o < E ? p.bqkv[2 * E + o] : 0.f;
            }
            for (int c = 0; c < E; ++c) {
                const float fc = __shfl_sync(0xffffffffu, acc[c >> 5], c & 31) * inv;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const int o = lane + 32 * r;
                    if (o < E) o4[r] = fmaf(__ldg(p.AvT + (size_t)c * E + o), fc, o4[r]);
                }
            }
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int o = lane + 32 * r;
                if (o < E) ab[(size_t)t * E + o] = o4[r];
            }
        }
        __syncthreads();
        // attention out-projection (into the query buffer), then out_projection
        for (int idx = tid; idx < nc * E; idx += kAtThreads) {
            const int t = idx / E, o = idx - t * E;
            float acc = p.bo[o];
            for (int c = 0; c < E; ++c) acc = fmaf(ab[(size_t)t * E + c], __ldg(p.WoT + (size_t)c * E + o), acc);
            qb[idx] = acc;
        }
        __syncthreads();
        for (int idx = tid; idx < nc * p.out_dim; idx += kAtThreads) {
            const int t = idx / p.out_dim, o = idx - t * p.out_dim;
            float acc = p.bout[o];
            for (int c = 0; c < E; ++c) acc = fmaf(qb[(size_t)t * E + c], __ldg(p.WoutT + (size_t)c * p.out_dim + o), acc);
            p.out[(size_t)(row0 + i0 + t) * p.out_dim + o] = acc;
        }
        __syncthreads();                                             // qb / ab are rewritten by the next chunk
    }
}

int launch_attn_mlp_pool(const tb2_lstm* m, const tb2_layout* l, const float* hidden, const float* obs1, const float* obs2,
                         float* out, cudaStream_t st) {
    AttnPoolParams p;
    p.obs1 = (const float2*)obs1;
    p.obs2 = (const float2*)obs2;
    p.hidden = hidden;
    p.scene_off = l->scene_off;
    p.Ws = m->mp_Ws; p.bs = m->mp_bs; p.Wv = m->mp_Wv; p.bv = m->mp_bv; p.WhT = m->mp_WhT; p.bh = m->mp_bh;
    p.AqT = m->at_AqT; p.Ak = m->at_Ak; p.AvT = m->at_AvT; p.bqkv = m->at_bqkv;
    p.WoT = m->at_WoT; p.bo = m->at_bo;
    p.WoutT = m->mp_WoT; p.bout = m->mp_bo;
    p.out = out;
    p.H = m->H;
    p.ds = m->cfg.mlp_dim_spatial; p.dv = m->cfg.mlp_dim_vel; p.dh = m->cfg.mlp_dim_hidden;
    p.out_dim = m->pool_out;
    p.n_max = l->n_max;
    p.pad_to_max = l->pad_to_max;
    p.fill = m->cfg.attn_fill;
    const int E = p.ds + p.dh + p.dv;
    const size_t smem = ((size_t)kAtChunk * 2 * E + (size_t)l->n_max * (4 + p.dh)) * sizeof(float);
    TB2_REQUIRE(smem <= 200 * 1024, "scene too large for the attention pooling kernel");
    static DynSmemConfig configured;
    TB2_CHECK_CUDA(configured.ensure(attn_mlp_pool_kernel, smem, 48 * 1024));
    {
        KernelTimer kt("attn_mlp_pool", st);
        launch_pdl(attn_mlp_pool_kernel, dim3(l->B), dim3(kAtThreads), smem, st, p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// ------------------------------------------------------------------------------------------
// TrajectronPooling features (--type traj_pool, reference non_gridbased_pooling.py:509-529): a visible track embeds
// [own (pos, vel) | sum of (pos, vel) over the OTHER visible tracks]; the reference sums over the whole flattened
// batch, so with the padded (trainer) layout the other scenes' sums are included, with the per-scene layout they are not.
// Kernel 1: one warp per scene sums its visible tracks in index order.  Kernel 2: one CTA per scene; "others" = the
// other scenes' sums (fixed order) + the own scene's other tracks, then Linear(8, out_dim) + ReLU; invisible tracks: 0.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) traj_scene_sum_kernel(const float2* __restrict__ obs1, const float2* __restrict__ obs2,
                                                             const int* __restrict__ scene_off, int B, float* __restrict__ scene_sum) {
    grid_dep_wait();
    grid_dep_launch();
    const int scene = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (scene >= B) return;
    const int row0 = scene_off[scene], n = scene_off[scene + 1] - row0;
    if (lane == 0) {         // sequential over the scene's tracks: a few dozen additions, fixed order
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
        for (int j = 0; j < n; ++j) {
            const float2 a = obs1[row0 + j], b = obs2[row0 + j];
            const float vx = b.x - a.x, vy = b.y - a.y;
            if (isnan(b.x) || isnan(b.y) || isnan(vx) || isnan(vy)) continue;
            s0 += b.x; s1 += b.y; s2 += vx; s3 += vy;
        }
        scene_sum[scene * 4 + 0] = s0; scene_sum[scene * 4 + 1] = s1; scene_sum[scene * 4 + 2] = s2; scene_sum[scene * 4 + 3] = s3;
    }
}

struct TrajFeatParams {
    const float2* obs1;
    const float2* obs2;
    const int* scene_off;
    const float* scene_sum;    // [B, 4]
    const float* W;            // [D, 8]
    const float* b;            // [D]
    float* feat;               // [M, D]
    int B, D, whole_batch;
};

__global__ void __launch_bounds__(256) traj_feat_kernel(TrajFeatParams p) {
    extern __shared__ __align__(16) float smem_tj[];
    const int scene = blockIdx.x;
    const int row0 = p.scene_off[scene], n = p.scene_off[scene + 1] - row0;
    float4* st = reinterpret_cast<float4*>(smem_tj);              // [n] (pos, vel), NaN kept
    float* in8 = reinterpret_cast<float*>(st + n);                // [n][8]
    __shared__ float other_scenes[4];
    const int tid = threadIdx.x;
    grid_dep_wait();
    grid_dep_launch();
    for (int j = tid; j < n; j += blockDim.x) {
        const float2 a = p.obs1[row0 + j], b = p.obs2[row0 + j];
        st[j] = make_float4(b.x, b.y, b.x - a.x, b.y - a.y);
    }
    if (tid < 4) {
        float s = 0.f;
        if (p.whole_batch)
            for (int b = 0; b < p.B; ++b)
                if (b != scene) s += p.scene_sum[b * 4 + tid];
        other_scenes[tid] = s;
    }
    __syncthreads();
    for (int i = tid; i < n; i += blockDim.x) {
        const float4 me = st[i];
        const bool vis = !(isnan(me.x) || isnan(me.y) || isnan(me.z) || isnan(me.w));
        float s0 = other_scenes[0], s1 = other_scenes[1], s2 = other_scenes[2], s3 = other_scenes[3];
        if (vis)
            for (int j = 0; j < n; ++j) {
                if (j == i) continue;
                const float4 o = st[j];
                if (isnan(o.x) || isnan(o.y) || isnan(o.z) || isnan(o.w)) continue;
                s0 += o.x; s1 += o.y; s2 += o.z; s3 += o.w;
            }
        float* x = in8 + (size_t)i * 8;
        x[0] = vis ? me.x : CUDART_NAN_F; x[1] = me.y; x[2] = me.z; x[3] = me.w;
        x[4] = s0; x[5] = s1; x[6] = s2; x[7] = s3;
    }
    __syncthreads();
    for (int idx = tid; idx < n * p.D; idx += blockDim.x) {
        const int i = idx / p.D, o = idx - i * p.D;
        const float* x = in8 + (size_t)i * 8;
        float v = 0.f;
        if (!isnan(x[0])) {
            float acc = p.b[o];
#pragma unroll
            for (int c = 0; c < 8; ++c) acc = fmaf(x[c], __ldg(p.W + (size_t)o * 8 + c), acc);
            v = fmaxf(acc, 0.f);
        }
        p.feat[(size_t)(row0 + i) * p.D + o] = v;
    }
}

int launch_trajectron_feat(const tb2_lstm* m, const tb2_layout* l, const float* obs1, const float* obs2, float* scene_sum,
                           float* feat, cudaStream_t st) {
    {
        KernelTimer kt("traj_scene_sum", st);
        launch_pdl(traj_scene_sum_kernel, dim3((l->B + 3) / 4), dim3(128), 0, st, (const float2*)obs1, (const float2*)obs2,
                   (const int*)l->scene_off, l->B, scene_sum);
    }
    TB2_LAUNCH_CHECK();
    TrajFeatParams p;
    p.obs1 = (const float2*)obs1; p.obs2 = (const float2*)obs2; p.scene_off = l->scene_off; p.scene_sum = scene_sum;
    p.W = m->mp_Ws; p.b = m->mp_bs; p.feat = feat; p.B = l->B; p.D = m->cfg.out_dim; p.whole_batch = l->pad_to_max;
    const size_t smem = (size_t)l->n_max * 12 * sizeof(float) + 16;
    TB2_REQUIRE(smem <= 48 * 1024, "scene too large for the Trajectron pooling kernel");
    {
        KernelTimer kt("traj_feat", st);
        launch_pdl(traj_feat_kernel, dim3(l->B), dim3(256), smem, st, p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// ------------------------------------------------------------------------------------------
// Interaction-encoder LSTMCell of NearestNeighborLSTM (--type nn_lstm, reference non_gridbased_pooling.py:445-451):
//   gates = W_ih feat + b_ih + W_hh h + b_hh (order i, f, g, o); c' = sigma(f) c + sigma(i) tanh(g); h' = sigma(o) tanh(c');
//   out = hidden2pool(h').   Every track is updated every step (absent ones with zero features).
// One CTA per 16 tracks: the inputs [feat | h] of its rows sit in shared memory, thread = gate column(s), the transposed
// weights stream coalesced from L2 with 16 accumulators per column; FP32 FFMA, accurate expf / tanhf.  The CTA's shared
// memory is Rows x (D + 6 Hp) floats; where 16 rows exceed 200 KB (D + 6 Hp > 3200, e.g. Hp = 512 with D >= 128) the
// tile is 8 rows, which holds every width the constructors accept (D <= 1024, Hp <= 512: 128 KB).  A row's arithmetic
// is the same in either tile.
// ------------------------------------------------------------------------------------------

struct PoolLstmParams {
    const float* feat;     // [M, D]
    float* h;              // [M, Hp] state, updated in place
    float* c;
    const float* WihT;     // [D][4 Hp]
    const float* WhhT;     // [Hp][4 Hp]
    const float* b;        // [4 Hp]
    const float* WoT;      // [Hp][D]
    const float* bo;       // [D]
    float* out;            // [M, D]
    int M, D, Hp;
};

template <int kPlRows>
__global__ void __launch_bounds__(256) pool_lstm_cell_kernel(PoolLstmParams p) {
    extern __shared__ __align__(16) float smem_pl[];
    const int K = p.D + p.Hp, G = 4 * p.Hp;
    float* x = smem_pl;                        // [K][kPlRows]  (input-major: one k at a time is a broadcast row)
    float* gates = x + (size_t)K * kPlRows;    // [kPlRows][G]
    float* hn = gates + (size_t)kPlRows * G;   // [kPlRows][Hp]
    const int tid = threadIdx.x, r0 = blockIdx.x * kPlRows;
    const int nr = min(kPlRows, p.M - r0);
    grid_dep_wait();
    grid_dep_launch();
    for (int idx = tid; idx < kPlRows * K; idx += blockDim.x) {
        const int r = idx / K, k = idx - r * K;
        float v = 0.f;
        if (r < nr) v = k < p.D ? p.feat[(size_t)(r0 + r) * p.D + k] : p.h[(size_t)(r0 + r) * p.Hp + (k - p.D)];
        x[(size_t)k * kPlRows + r] = v;
    }
    __syncthreads();
    for (int col = tid; col < G; col += blockDim.x) {
        float acc[kPlRows];
        const float b = p.b[col];
#pragma unroll
        for (int r = 0; r < kPlRows; ++r) acc[r] = b;
        for (int k = 0; k < K; ++k) {
            const float w = k < p.D ? __ldg(p.WihT + (size_t)k * G + col) : __ldg(p.WhhT + (size_t)(k - p.D) * G + col);
            const float4* xr = reinterpret_cast<const float4*>(x + (size_t)k * kPlRows);
#pragma unroll
            for (int q = 0; q < kPlRows / 4; ++q) {
                const float4 xv = xr[q];
                acc[4 * q] = fmaf(xv.x, w, acc[4 * q]); acc[4 * q + 1] = fmaf(xv.y, w, acc[4 * q + 1]);
                acc[4 * q + 2] = fmaf(xv.z, w, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(xv.w, w, acc[4 * q + 3]);
            }
        }
#pragma unroll
        for (int r = 0; r < kPlRows; ++r) gates[(size_t)r * G + col] = acc[r];
    }
    __syncthreads();
    for (int idx = tid; idx < kPlRows * p.Hp; idx += blockDim.x) {
        const int r = idx / p.Hp, u = idx - r * p.Hp;
        float hv = 0.f;
        if (r < nr) {
            const float* g = gates + (size_t)r * G;
            const float ig = 1.f / (1.f + expf(-g[u]));
            const float fg = 1.f / (1.f + expf(-g[p.Hp + u]));
            const float gt = tanhf(g[2 * p.Hp + u]);
            const float og = 1.f / (1.f + expf(-g[3 * p.Hp + u]));
            const size_t o = (size_t)(r0 + r) * p.Hp + u;
            const float cn = fg * p.c[o] + ig * gt;
            hv = og * tanhf(cn);
            p.c[o] = cn;
            p.h[o] = hv;
        }
        hn[idx] = hv;
    }
    __syncthreads();
    for (int idx = tid; idx < nr * p.D; idx += blockDim.x) {
        const int r = idx / p.D, o = idx - r * p.D;
        float acc = p.bo[o];
        for (int k = 0; k < p.Hp; ++k) acc = fmaf(hn[(size_t)r * p.Hp + k], __ldg(p.WoT + (size_t)k * p.D + o), acc);
        p.out[(size_t)(r0 + r) * p.D + o] = acc;
    }
}

int launch_pool_lstm_cell(const tb2_lstm* m, const tb2_layout* l, const float* feat, float* h, float* c, float* out,
                          cudaStream_t st) {
    PoolLstmParams p;
    p.feat = feat; p.h = h; p.c = c;
    p.WihT = m->pl_WihT; p.WhhT = m->pl_WhhT; p.b = m->pl_b; p.WoT = m->mp_WoT; p.bo = m->mp_bo;
    p.out = out;
    p.M = l->M; p.D = m->cfg.out_dim; p.Hp = m->cfg.mlp_dim_hidden;
    const size_t row_bytes = (size_t)(p.D + 6 * p.Hp) * sizeof(float);      // [feat | h], 4 gates, h' of one row
    TB2_REQUIRE(8 * row_bytes <= 200 * 1024, "interaction-encoder LSTM too wide for the kernel");
    {
        KernelTimer kt("pool_lstm_cell", st);
        if (16 * row_bytes <= 200 * 1024) {
            static DynSmemConfig configured;
            TB2_CHECK_CUDA(configured.ensure(pool_lstm_cell_kernel<16>, 16 * row_bytes, 48 * 1024));
            launch_pdl(pool_lstm_cell_kernel<16>, dim3((l->M + 15) / 16), dim3(256), 16 * row_bytes, st, p);
        } else {
            static DynSmemConfig configured;
            TB2_CHECK_CUDA(configured.ensure(pool_lstm_cell_kernel<8>, 8 * row_bytes, 48 * 1024));
            launch_pdl(pool_lstm_cell_kernel<8>, dim3((l->M + 7) / 8), dim3(256), 8 * row_bytes, st, p);
        }
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

// ------------------------------------------------------------------------------------------
// NearestNeighborMLP on the device (--type nn, reference non_gridbased_pooling.py:64-147).
//
//   for every track i: the n nearest other tracks of its scene by ||pos_j - pos_i|| (absent tracks count as 1000 m,
//   reference :131-132), in ascending distance; per kept neighbour the features [pos_j - pos_i | v_j - v_i] (NaN -> 0,
//   :141; missing neighbours are zero rows, :134-136) go through Linear(2 or 4 -> out_dim / n) + ReLU; the n
//   embeddings are concatenated.  One warp per track: lane = candidate neighbour, n rounds of a warp arg-min.
// ------------------------------------------------------------------------------------------
struct NnPoolParams {
    const float2* obs1;
    const float2* obs2;
    const int* scene_off;
    const float* W;            // [d, 2 or 4]
    const float* b;            // [d]
    float* out;                // [M, n * d]
    int n, d, with_vel;
};

__global__ void __launch_bounds__(256) nn_mlp_pool_kernel(NnPoolParams p) {
    extern __shared__ __align__(16) float smem_nn[];
    const int scene = blockIdx.x;
    const int row0 = p.scene_off[scene];
    const int ns = p.scene_off[scene + 1] - row0;
    float2* pos = reinterpret_cast<float2*>(smem_nn);              // [ns] obs2 (NaN kept)
    float2* vel = pos + ns;                                        // [ns] obs2 - obs1
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;
    grid_dep_wait();
    grid_dep_launch();
    for (int j = tid; j < ns; j += blockDim.x) {
        const float2 a = p.obs1[row0 + j], b = p.obs2[row0 + j];
        pos[j] = b;
        vel[j] = make_float2(b.x - a.x, b.y - a.y);
    }
    __syncthreads();
    for (int i = warp; i < ns; i += nwarps) {
        const float2 pi = pos[i], vi = vel[i];
        float* out = p.out + (size_t)(row0 + i) * p.n * p.d;
        float last_d = -1.f;
        int last_j = -1;
        for (int k = 0; k < p.n; ++k) {
            // arg-min over the candidates after (last_d, last_j) in (distance, index) order: selection without marking
            float best = CUDART_INF_F;
            int best_j = 0x7fffffff;
            for (int j = lane; j < ns; j += 32) {
                if (j == i) continue;
                const float rx = pos[j].x - pi.x, ry = pos[j].y - pi.y;
                float dist = sqrtf(__fadd_rn(__fmul_rn(rx, rx), __fmul_rn(ry, ry)));
                if (isnan(dist)) dist = 1000.f;
                const bool after = dist > last_d || (dist == last_d && j > last_j);
                if (after && (dist < best || (dist == best && j < best_j))) { best = dist; best_j = j; }
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, off);
                const int oj = __shfl_xor_sync(0xffffffffu, best_j, off);
                if (ob < best || (ob == best && oj < best_j)) { best = ob; best_j = oj; }
            }
            float f[4] = {0.f, 0.f, 0.f, 0.f};                     // fewer than n other tracks: zero features
            if (best_j != 0x7fffffff) {
                last_d = best; last_j = best_j;
                const float2 pj = pos[best_j], vj = vel[best_j];
                f[0] = pj.x - pi.x; f[1] = pj.y - pi.y; f[2] = vj.x - vi.x; f[3] = vj.y - vi.y;
#pragma unroll
                for (int c = 0; c < 4; ++c) f[c] = isnan(f[c]) ? 0.f : (isinf(f[c]) ? copysignf(3.402823466e+38f, f[c]) : f[c]);
            } else {
                last_d = CUDART_INF_F;
            }
            const int in_dim = p.with_vel ? 4 : 2;
            for (int o = lane; o < p.d; o += 32) {
                float acc = p.b[o];
                for (int c = 0; c < in_dim; ++c) acc = fmaf(f[c], p.W[o * in_dim + c], acc);
                out[k * p.d + o] = fmaxf(acc, 0.f);
            }
        }
    }
}

int launch_nn_mlp_pool(const tb2_lstm* m, const tb2_layout* l, const float* obs1, const float* obs2, float* out,
                       cudaStream_t st) {
    NnPoolParams p;
    p.obs1 = (const float2*)obs1;
    p.obs2 = (const float2*)obs2;
    p.scene_off = l->scene_off;
    p.W = m->mp_Ws;
    p.b = m->mp_bs;
    p.out = out;
    p.n = m->cfg.n;
    p.d = m->cfg.mlp_dim_spatial;
    p.with_vel = m->cfg.mlp_dim_vel != 0;
    const size_t smem = (size_t)l->n_max * 4 * sizeof(float) + 16;
    TB2_REQUIRE(smem <= 48 * 1024, "scene too large for the nearest-neighbour pooling kernel");
    {
        KernelTimer kt("nn_mlp_pool", st);
        launch_pdl(nn_mlp_pool_kernel, dim3(l->B), dim3(256), smem, st, p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // namespace tb2
