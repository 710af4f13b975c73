// Social-NCE contrastive term (lstm/contrast.py, DESIGN §1 A24): InfoNCE between the primary's hidden state at the
// end of the observation (the query) and events around where the people of its scene will be.
//
// tb2_snce_forward runs one CTA per scene.  For every horizon delta it streams the scene's samples (the positive, then
// 8 negatives around each neighbour with a finite position) through the event encoder twice: once for the
// log-sum-exp (an online max / sum per thread, combined in a fixed tree), once for the gradients, a chunk of
// kThreads samples at a time, whose per-sample operands go through shared memory to the thread that owns each
// parameter entry.  No key is kept, so a scene of any size fits.  It writes each pair's term, the pair's finiteness and
// the scene's gradients of sum_delta term wrt its query row and every parameter (unscaled partials).
// tb2_snce_backward sums the partials in ascending scene order and scales them by d loss / max(number of finite
// pairs, 1), both read on the device.  Nothing uses atomics and a CTA reads only its own scene: a scene's outputs do
// not depend on the batch around it, and reruns are bit-identical.
#include <math.h>

#include "common.cuh"

namespace tb2 {
namespace {

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;

// parameter layout of the packed vector: event encoder W1 [D, 3], b1 [D], W2 [E, D], b2 [E]; projection head
// V1 [D, H], c1 [D], V2 [E, D], c2 [E] (SocialNCE.parameters() order)
struct Offsets {
    int W1, b1, W2, b2, V1, c1, V2, c2, total;
};

__host__ __device__ inline Offsets offsets(int D, int E, int H) {
    Offsets o;
    o.W1 = 0;
    o.b1 = o.W1 + 3 * D;
    o.W2 = o.b1 + D;
    o.b2 = o.W2 + E * D;
    o.V1 = o.b2 + E;
    o.c1 = o.V1 + D * H;
    o.V2 = o.c1 + D;
    o.c2 = o.V2 + E * D;
    o.total = o.c2 + E;
    return o;
}

__device__ __forceinline__ bool finite2(float2 v) { return isfinite(v.x) && isfinite(v.y); }

// (max, sum of exp(x - max)) pairs; an empty side has max = -inf
__device__ __forceinline__ void lse_combine(float& m, float& s, float m2, float s2) {
    if (m2 == -INFINITY) return;
    if (m == -INFINITY) { m = m2; s = s2; return; }
    if (m2 > m) { s = s * expf(m - m2) + s2; m = m2; }
    else s = s + s2 * expf(m2 - m);
}

template <int D, int E>
struct Smem {
    float W1[3 * D], b1[D], W2[E * D], b2[E];
    float q[E];                         // normalised query
    float acc[3 * D + D + E * D + E];   // the event encoder's parameter gradients, one owner thread per entry
    float in[kThreads][3];
    float z[kThreads][D + 1];
    float dz[kThreads][D + 1];
    float de[kThreads][E + 1];
    float red_m[kWarps], red_s[kWarps];
    float lse, lpos;
    float zq[D], dzq[D], deq[E], dq[E];
};

// the event encoder on one sample: z = relu(W1 [x, y, delta] + b1), e = W2 z + b2, key = e / max(|e|, 1e-12)
template <int D, int E>
__device__ __forceinline__ float encode(const Smem<D, E>& sm, float x, float y, float dl, float (&z)[D], float (&k)[E],
                                        float& nrm) {
#pragma unroll
    for (int c = 0; c < D; ++c)
        z[c] = fmaxf(fmaf(sm.W1[3 * c + 2], dl, fmaf(sm.W1[3 * c + 1], y, fmaf(sm.W1[3 * c], x, sm.b1[c]))), 0.f);
    float ss = 0.f;
#pragma unroll
    for (int o = 0; o < E; ++o) {
        float a = sm.b2[o];
#pragma unroll
        for (int c = 0; c < D; ++c) a = fmaf(sm.W2[o * D + c], z[c], a);
        k[o] = a;
        ss = fmaf(a, a, ss);
    }
    nrm = sqrtf(ss);
    const float den = fmaxf(nrm, 1e-12f);
    float dot = 0.f;
#pragma unroll
    for (int o = 0; o < E; ++o) {
        k[o] = k[o] / den;
        dot = fmaf(sm.q[o], k[o], dot);
    }
    return dot;
}

// backward of v = e / max(|e|, 1e-12) (F.normalize): de = (dv - v (v . dv)) / |e|, or dv / 1e-12 below the clamp
template <int E>
__device__ __forceinline__ void normalize_backward(const float (&v)[E], const float (&dv)[E], float nrm, float (&de)[E]) {
    if (nrm > 1e-12f) {
        float vd = 0.f;
#pragma unroll
        for (int o = 0; o < E; ++o) vd = fmaf(v[o], dv[o], vd);
#pragma unroll
        for (int o = 0; o < E; ++o) de[o] = (dv[o] - v[o] * vd) / nrm;
    } else {
#pragma unroll
        for (int o = 0; o < E; ++o) de[o] = dv[o] / 1e-12f;
    }
}

template <int D, int E>
__global__ void __launch_bounds__(kThreads) snce_forward_kernel(
    const float2* __restrict__ X, int T, int M, const int* __restrict__ scene_off, int n_max, int f0, int horizon,
    const float* __restrict__ hq, int H, const float* __restrict__ theta, float inv_tau, float rho, float sigma,
    const float2* __restrict__ eps, float* __restrict__ terms, float* __restrict__ valid, float* __restrict__ dq_part,
    float* __restrict__ dp_part) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem<D, E>& sm = *reinterpret_cast<Smem<D, E>*>(smem_raw);
    const Offsets off = offsets(D, E, H);
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int p = scene_off[b];
    const int n = min(scene_off[b + 1] - p, n_max);
    const int ns_max = 1 + 8 * (n_max - 1);
    const int ns = 1 + 8 * (n - 1);
    constexpr int kPhi = 3 * D + D + E * D + E;
    for (int i = tid; i < 3 * D; i += kThreads) sm.W1[i] = theta[off.W1 + i];
    for (int i = tid; i < D; i += kThreads) sm.b1[i] = theta[off.b1 + i];
    for (int i = tid; i < E * D; i += kThreads) sm.W2[i] = theta[off.W2 + i];
    for (int i = tid; i < E; i += kThreads) sm.b2[i] = theta[off.b2 + i];
    for (int i = tid; i < kPhi; i += kThreads) sm.acc[i] = 0.f;
    // the query: zq = relu(V1 h + c1) (one warp per unit, lanes over h in a fixed order), then V2 zq + c2, normalised
    const float* h = hq + (size_t)p * H;
    for (int c = warp; c < D; c += kWarps) {
        float a = 0.f;
        for (int u = lane; u < H; u += 32) a = fmaf(theta[off.V1 + c * H + u], h[u], a);
#pragma unroll
        for (int sh = 16; sh > 0; sh >>= 1) a += __shfl_xor_sync(0xffffffffu, a, sh);
        if (lane == 0) sm.zq[c] = fmaxf(a + theta[off.c1 + c], 0.f);
    }
    __syncthreads();
    float eq[E], qn[E], nq;
    {
        float ss = 0.f;
#pragma unroll
        for (int o = 0; o < E; ++o) {
            float a = theta[off.c2 + o];
            for (int c = 0; c < D; ++c) a = fmaf(theta[off.V2 + o * D + c], sm.zq[c], a);
            eq[o] = a;
            ss = fmaf(a, a, ss);
        }
        nq = sqrtf(ss);
        const float den = fmaxf(nq, 1e-12f);
#pragma unroll
        for (int o = 0; o < E; ++o) qn[o] = eq[o] / den;
    }
    if (tid < E) sm.q[tid] = qn[tid];
    __syncthreads();

    float dq_acc[E];
#pragma unroll
    for (int o = 0; o < E; ++o) dq_acc[o] = 0.f;
    const float2 x0 = X[(size_t)f0 * M + p];
    for (int d = 1; d <= horizon; ++d) {
        const int f = f0 + d;
        const float2 xp = X[(size_t)f * M + p];
        const bool ok = finite2(x0) && finite2(xp);
        if (tid == 0) {
            valid[b * horizon + d - 1] = ok ? 1.f : 0.f;
            if (!ok) terms[b * horizon + d - 1] = 0.f;
        }
        if (!ok) continue;            // uniform over the CTA
        const float2* ep = eps + ((size_t)b * horizon + (d - 1)) * ns_max;
        const float dl = (float)d;
        // sample i: 0 = the positive, 1 + 8 jj + k = neighbour p + 1 + jj shifted by rho (cos k pi/4, sin k pi/4)
        auto sample = [&](int i, float& x, float& y) -> bool {
            float2 base;
            float ox = 0.f, oy = 0.f;
            if (i == 0) {
                base = xp;
            } else {
                const int jj = (i - 1) >> 3, k = (i - 1) & 7;
                base = X[(size_t)f * M + p + 1 + jj];
                if (!finite2(base)) return false;
                // cos / sin of k pi / 4, exact where they are 0 or +-1
                const float r2 = 0.70710678118654752f;
                const float cs[8] = {1.f, r2, 0.f, -r2, -1.f, -r2, 0.f, r2};
                ox = rho * cs[k];
                oy = rho * cs[(k + 6) & 7];
            }
            const float2 e = ep[i];
            x = fmaf(sigma, e.x, (base.x - x0.x) + ox);
            y = fmaf(sigma, e.y, (base.y - x0.y) + oy);
            return true;
        };
        // two passes over the same sample loop: 0 = the log-sum-exp of the logits, 1 = d term / d logit_i =
        // softmax_i - [i = 0] through the key and the event encoder.  The logit is rounded before anything uses it
        // (__fmul_rn: no FMA contraction into l - Mx), so both passes see the same bits and a pair without negatives
        // gets exactly 0 and a zero gradient
        float m = -INFINITY, s = 0.f, Mx = 0.f, inv_S = 0.f;
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
            for (int c0 = 0; c0 < ns; c0 += kThreads) {
                const int i = c0 + tid;
                float x = 0.f, y = 0.f;
                const bool live = i < ns && sample(i, x, y);
                float z[D], k[E], nrm = 0.f, de[E], l = 0.f;
#pragma unroll
                for (int c = 0; c < D; ++c) z[c] = 0.f;
#pragma unroll
                for (int o = 0; o < E; ++o) de[o] = 0.f;
                if (live) l = __fmul_rn(encode<D, E>(sm, x, y, dl, z, k, nrm), inv_tau);
                if (pass == 0) {
                    if (live) {
                        if (i == 0) sm.lpos = l;
                        lse_combine(m, s, l, 1.f);
                    }
                    continue;
                }
                if (live) {
                    const float g = (expf(l - Mx) * inv_S - (i == 0 ? 1.f : 0.f)) * inv_tau;
                    float dk[E];
#pragma unroll
                    for (int o = 0; o < E; ++o) {
                        dq_acc[o] = fmaf(g, k[o], dq_acc[o]);
                        dk[o] = g * sm.q[o];
                    }
                    normalize_backward<E>(k, dk, nrm, de);
                }
                sm.in[tid][0] = live ? x : 0.f;
                sm.in[tid][1] = live ? y : 0.f;
                sm.in[tid][2] = live ? dl : 0.f;
#pragma unroll
                for (int c = 0; c < D; ++c) {
                    float a = 0.f;
#pragma unroll
                    for (int o = 0; o < E; ++o) a = fmaf(sm.W2[o * D + c], de[o], a);
                    sm.z[tid][c] = z[c];
                    sm.dz[tid][c] = z[c] > 0.f ? a : 0.f;
                }
#pragma unroll
                for (int o = 0; o < E; ++o) sm.de[tid][o] = de[o];
                __syncthreads();
                for (int e = tid; e < kPhi; e += kThreads) {
                    float a = 0.f;
                    if (e < 3 * D) {
                        const int c = e / 3, j = e % 3;
                        for (int t = 0; t < kThreads; ++t) a = fmaf(sm.dz[t][c], sm.in[t][j], a);
                    } else if (e < 4 * D) {
                        const int c = e - 3 * D;
                        for (int t = 0; t < kThreads; ++t) a += sm.dz[t][c];
                    } else if (e < 4 * D + E * D) {
                        const int o = (e - 4 * D) / D, c = (e - 4 * D) % D;
                        for (int t = 0; t < kThreads; ++t) a = fmaf(sm.de[t][o], sm.z[t][c], a);
                    } else {
                        const int o = e - 4 * D - E * D;
                        for (int t = 0; t < kThreads; ++t) a += sm.de[t][o];
                    }
                    sm.acc[e] += a;
                }
                __syncthreads();
            }
            if (pass == 1) break;
#pragma unroll
            for (int sh = 16; sh > 0; sh >>= 1) {
                const float m2 = __shfl_xor_sync(0xffffffffu, m, sh), s2 = __shfl_xor_sync(0xffffffffu, s, sh);
                lse_combine(m, s, m2, s2);
            }
            if (lane == 0) { sm.red_m[warp] = m; sm.red_s[warp] = s; }
            __syncthreads();
            if (tid == 0) {
                float M0 = sm.red_m[0], S0 = sm.red_s[0];
                for (int w = 1; w < kWarps; ++w) lse_combine(M0, S0, sm.red_m[w], sm.red_s[w]);
                sm.red_m[0] = M0;
                sm.red_s[0] = S0;
                // with no negatives lse = lpos + log(1): the term is exactly 0
                sm.lse = M0 + logf(S0);
                terms[b * horizon + d - 1] = sm.lse - sm.lpos;
            }
            __syncthreads();
            Mx = sm.red_m[0];
            inv_S = 1.f / sm.red_s[0];
        }
    }
    // d query: the threads' accumulators summed in a fixed tree (warp shuffles, then the warps in order)
#pragma unroll
    for (int o = 0; o < E; ++o) {
        float a = dq_acc[o];
#pragma unroll
        for (int sh = 16; sh > 0; sh >>= 1) a += __shfl_xor_sync(0xffffffffu, a, sh);
        if (lane == 0) sm.de[warp][o] = a;
    }
    __syncthreads();
    if (tid == 0) {
        float dqs[E], deqs[E];
#pragma unroll
        for (int o = 0; o < E; ++o) {
            float a = sm.de[0][o];
            for (int w = 1; w < kWarps; ++w) a += sm.de[w][o];
            dqs[o] = a;
        }
        normalize_backward<E>(qn, dqs, nq, deqs);
#pragma unroll
        for (int o = 0; o < E; ++o) sm.deq[o] = deqs[o];
    }
    __syncthreads();
    for (int c = tid; c < D; c += kThreads) {
        float a = 0.f;
        for (int o = 0; o < E; ++o) a = fmaf(theta[off.V2 + o * D + c], sm.deq[o], a);
        sm.dzq[c] = sm.zq[c] > 0.f ? a : 0.f;
    }
    __syncthreads();
    float* part = dp_part + (size_t)b * off.total;
    for (int e = tid; e < kPhi; e += kThreads) part[e] = sm.acc[e];       // W1, b1, W2, b2 are contiguous from 0
    for (int e = tid; e < D * H; e += kThreads) part[off.V1 + e] = sm.dzq[e / H] * h[e % H];
    for (int c = tid; c < D; c += kThreads) part[off.c1 + c] = sm.dzq[c];
    for (int e = tid; e < E * D; e += kThreads) part[off.V2 + e] = sm.deq[e / D] * sm.zq[e % D];
    for (int o = tid; o < E; o += kThreads) part[off.c2 + o] = sm.deq[o];
    for (int u = tid; u < H; u += kThreads) {
        float a = 0.f;
        for (int c = 0; c < D; ++c) a = fmaf(theta[off.V1 + c * H + u], sm.dzq[c], a);
        dq_part[(size_t)b * H + u] = a;
    }
}

// d params = scale * sum over ascending scenes of the partials; d h of each primary row = scale * its partial;
// scale = d loss / max(finite pairs, 1)
__global__ void snce_backward_kernel(const float* __restrict__ d_loss, const float* __restrict__ count,
                                     const int* __restrict__ scene_off, int B, int H, int NP,
                                     const float* __restrict__ dq_part, const float* __restrict__ dp_part,
                                     float* __restrict__ d_hidden, float* __restrict__ d_params) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const float scale = d_loss[0] / fmaxf(count[0], 1.f);
    if (idx < NP) {
        float a = 0.f;
        for (int b = 0; b < B; ++b) a += dp_part[(size_t)b * NP + idx];
        d_params[idx] = a * scale;
    } else if (idx - NP < B * H) {
        const int b = (idx - NP) / H, u = (idx - NP) % H;
        d_hidden[(size_t)scene_off[b] * H + u] = dq_part[(size_t)b * H + u] * scale;
    }
}

template <int D, int E>
int launch_forward(const float* X, int T, int M, const tb2_layout* l, int f0, int horizon, const float* hq, int H,
                   const float* theta, float tau, float rho, float sigma, const float* eps, float* terms, float* valid,
                   float* dq_part, float* dp_part, cudaStream_t st) {
    const size_t smem = sizeof(Smem<D, E>);
    static DynSmemConfig configured;
    TB2_CHECK_CUDA(configured.ensure(snce_forward_kernel<D, E>, smem, 48 * 1024));
    KernelTimer kt("snce_forward", st);
    snce_forward_kernel<D, E><<<l->B, kThreads, smem, st>>>(
        reinterpret_cast<const float2*>(X), T, M, l->scene_off, l->n_max, f0, horizon, hq, H, theta, 1.f / tau, rho,
        sigma, reinterpret_cast<const float2*>(eps), terms, valid, dq_part, dp_part);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // namespace
}  // namespace tb2

using namespace tb2;

extern "C" {

int32_t tb2_snce_num_params(int32_t hidden_dim, int32_t mlp_dim, int32_t head_dim) {
    return offsets(mlp_dim, head_dim, hidden_dim).total;
}

int tb2_snce_forward(const tb2_layout* l, const float* scene_dev, int32_t num_frames, int32_t obs_frame,
                     int32_t horizon, const float* hidden_dev, int32_t hidden_dim, const float* params_dev,
                     int32_t mlp_dim, int32_t head_dim, float temperature, float rho, float sigma, const float* eps_dev,
                     float* terms_out, float* valid_out, float* d_hidden_part_out, float* d_params_part_out,
                     void* stream) {
    TB2_REQUIRE(l, "null layout");
    TB2_REQUIRE(scene_dev && hidden_dev && params_dev && eps_dev && terms_out && valid_out && d_hidden_part_out &&
                    d_params_part_out, "null argument");
    TB2_REQUIRE(horizon >= 1 && obs_frame >= 0 && obs_frame + horizon < num_frames,
                "need horizon >= 1 and obs_frame + horizon < num_frames");
    TB2_REQUIRE(hidden_dim >= 1 && hidden_dim <= 1024, "hidden_dim must be in 1..1024");
    TB2_REQUIRE(temperature > 0.f && isfinite(temperature), "temperature must be > 0");
    // samples are counted in int32 per scene and pair: 1 + 8 (n_max - 1) per horizon step
    TB2_REQUIRE(l->n_max <= (1 << 24) / horizon, "scene too large for the Social-NCE sample index");
    if (l->B == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
#define TB2_SNCE_CASE(DD, EE)                                                                                      \
    if (mlp_dim == DD && head_dim == EE)                                                                           \
        return launch_forward<DD, EE>(scene_dev, num_frames, l->M, l, obs_frame, horizon, hidden_dev, hidden_dim, \
                                      params_dev, temperature, rho, sigma, eps_dev, terms_out, valid_out,          \
                                      d_hidden_part_out, d_params_part_out, st);
    TB2_SNCE_CASE(16, 4) TB2_SNCE_CASE(16, 8) TB2_SNCE_CASE(16, 16)
    TB2_SNCE_CASE(32, 4) TB2_SNCE_CASE(32, 8) TB2_SNCE_CASE(32, 16)
    TB2_SNCE_CASE(64, 4) TB2_SNCE_CASE(64, 8) TB2_SNCE_CASE(64, 16)
#undef TB2_SNCE_CASE
    set_error("Social-NCE is built for mlp_dim 16, 32 or 64 and head_dim 4, 8 or 16");
    return TB2_ERR_UNSUPPORTED;
}

int tb2_snce_backward(const tb2_layout* l, const float* d_loss_dev, const float* count_dev, int32_t hidden_dim,
                      int32_t num_params, const float* d_hidden_part_dev, const float* d_params_part_dev,
                      float* d_hidden_out, float* d_params_out, void* stream) {
    TB2_REQUIRE(l, "null layout");
    TB2_REQUIRE(d_loss_dev && count_dev && d_hidden_part_dev && d_params_part_dev && d_hidden_out && d_params_out,
                "null argument");
    TB2_REQUIRE(hidden_dim >= 1 && num_params >= 1, "need hidden_dim >= 1 and num_params >= 1");
    const size_t n = (size_t)num_params + (size_t)l->B * hidden_dim;
    TB2_REQUIRE(n < (1u << 31), "too many Social-NCE gradients");
    cudaStream_t st = (cudaStream_t)stream;
    KernelTimer kt("snce_backward", st);
    snce_backward_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_loss_dev, count_dev, l->scene_off, l->B,
                                                                     hidden_dim, num_params, d_hidden_part_dev,
                                                                     d_params_part_dev, d_hidden_out, d_params_out);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // extern "C"
