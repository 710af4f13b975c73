// Collision attack on LSTM forecasts (attack.py): the objective and the projected-gradient step, one launch each, no
// atomics (bit-identical from run to run).
//
// Objective: per scene, D = the smallest distance between the primary's and a neighbour's predicted positions at the
// points the scorer's Col-I test samples (metrics.cu `collides`): consecutive frames where both tracks are finite form a
// segment on each track, each sampled at linspace(p_prev, p_t, 3), paired between the tracks.  On the same values
// D <= 0.2 m exactly when Col-I fires for the scene: the distances are the same double operations, and this file is
// compiled with -fmad=false like metrics.cu.
#include <math.h>

#include "common.cuh"

namespace tb2 {
namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr double kColLimit = 2.0 * 0.1;

__device__ __forceinline__ bool finite2(float2 p) { return isfinite(p.x) && isfinite(p.y); }

// One warp per scene, one neighbour per lane.  The gradient of D is the subgradient at the first minimiser in
// (neighbour, frame, sample) order, spread onto the four segment endpoints with the interpolation weights (0, 1/2, 1);
// a zero distance, and a scene without a finite pair (D = +inf), get a zero gradient.
__global__ void __launch_bounds__(32) attack_objective_kernel(const float2* __restrict__ pos, const int* __restrict__ scene_off,
                                                               int F, int first, int M, double* __restrict__ D_out,
                                                               float2* __restrict__ dpos) {
    const int b = blockIdx.x, lane = threadIdx.x;
    const int r0 = scene_off[b], r1 = scene_off[b + 1];
    for (int idx = lane; idx < F * (r1 - r0); idx += 32) {
        const int f = idx / (r1 - r0), r = r0 + idx - f * (r1 - r0);
        dpos[(size_t)f * M + r] = make_float2(0.f, 0.f);
    }
    double best = INFINITY;
    int bj = 0x7fffffff, bprev = 0, bt = 0, bk = 0;
    for (int j = r0 + 1 + lane; j < r1; j += 32) {
        int prev = -1;
        for (int t = first; t < F; ++t) {
            const float2 a2 = pos[(size_t)t * M + r0], b2 = pos[(size_t)t * M + j];
            if (!finite2(a2) || !finite2(b2)) continue;
            if (prev >= 0) {
                const float2 a1 = pos[(size_t)prev * M + r0], b1 = pos[(size_t)prev * M + j];
                const double p1x = a1.x, p1y = a1.y, p2x = a2.x, p2y = a2.y;
                const double p3x = b1.x, p3y = b1.y, p4x = b2.x, p4y = b2.y;
                const double ax[3] = {p1x, p1x + (p2x - p1x) / 2.0, p2x}, ay[3] = {p1y, p1y + (p2y - p1y) / 2.0, p2y};
                const double bx[3] = {p3x, p3x + (p4x - p3x) / 2.0, p4x}, by[3] = {p3y, p3y + (p4y - p3y) / 2.0, p4y};
                for (int k = 0; k < 3; ++k) {
                    const double dx = ax[k] - bx[k], dy = ay[k] - by[k];
                    const double d = sqrt(dx * dx + dy * dy);
                    if (d < best) {
                        best = d;
                        bj = j;
                        bprev = prev;
                        bt = t;
                        bk = k;
                    }
                }
            }
            prev = t;
        }
    }
    // the smallest (D, neighbour): each lane's candidates are already first in (frame, sample) order
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(kFull, best, o);
        const int oj = __shfl_xor_sync(kFull, bj, o), op = __shfl_xor_sync(kFull, bprev, o);
        const int ot = __shfl_xor_sync(kFull, bt, o), ok = __shfl_xor_sync(kFull, bk, o);
        if (ob < best || (ob == best && oj < bj)) {
            best = ob;
            bj = oj;
            bprev = op;
            bt = ot;
            bk = ok;
        }
    }
    __syncwarp();
    if (lane != 0) return;
    D_out[b] = best;
    if (!(best > 0.0) || !isfinite(best)) return;
    const float2 a1 = pos[(size_t)bprev * M + r0], a2 = pos[(size_t)bt * M + r0];
    const float2 b1 = pos[(size_t)bprev * M + bj], b2 = pos[(size_t)bt * M + bj];
    const double w = 0.5 * bk;
    const double ax = bk == 0 ? a1.x : bk == 2 ? a2.x : (double)a1.x + ((double)a2.x - a1.x) / 2.0;
    const double ay = bk == 0 ? a1.y : bk == 2 ? a2.y : (double)a1.y + ((double)a2.y - a1.y) / 2.0;
    const double bx = bk == 0 ? b1.x : bk == 2 ? b2.x : (double)b1.x + ((double)b2.x - b1.x) / 2.0;
    const double by = bk == 0 ? b1.y : bk == 2 ? b2.y : (double)b1.y + ((double)b2.y - b1.y) / 2.0;
    const double ux = (ax - bx) / best, uy = (ay - by) / best;
    dpos[(size_t)bprev * M + r0] = make_float2((float)((1.0 - w) * ux), (float)((1.0 - w) * uy));
    dpos[(size_t)bt * M + r0] = make_float2((float)(w * ux), (float)(w * uy));
    dpos[(size_t)bprev * M + bj] = make_float2((float)(-(1.0 - w) * ux), (float)(-(1.0 - w) * uy));
    dpos[(size_t)bt * M + bj] = make_float2((float)(-w * ux), (float)(-w * uy));
}

// One CTA per scene.  Records the iterate (delta, D, its positions) when D beats the best so far (ties keep the
// earlier one), then, with `move` and unless the best D is <= 0.2 m (the scene is frozen), steps the primary's
// observed frames: delta_t <- proj_eps(delta_t - alpha g_t / |g_t|).  A frame whose gradient is 0 or not finite, or
// whose observed position is not finite, stays.  observed_adv = observed + delta on the primary rows.
__global__ void __launch_bounds__(256) attack_step_kernel(
    const float2* __restrict__ d_obs, const float2* __restrict__ obs, int obs_length, const int* __restrict__ scene_off,
    int M, int B, float2* __restrict__ delta, const double* __restrict__ D_cur, int F, const float2* __restrict__ pos,
    double* __restrict__ best_D, float2* __restrict__ best_delta, float2* __restrict__ best_pos,
    float2* __restrict__ obs_adv, double eps, double alpha, int move) {
    const int b = blockIdx.x, r0 = scene_off[b], n = scene_off[b + 1] - r0;
    const double d = D_cur[b], prev_best = best_D[b];
    const bool improved = d < prev_best;
    const double best = improved ? d : prev_best;
    if (improved) {
        for (int t = threadIdx.x; t < obs_length; t += blockDim.x) best_delta[(size_t)t * B + b] = delta[(size_t)t * B + b];
        for (int idx = threadIdx.x; idx < F * n; idx += blockDim.x) {
            const int f = idx / n, r = r0 + idx - f * n;
            best_pos[(size_t)f * M + r] = pos[(size_t)f * M + r];
        }
    }
    __syncthreads();                       // every thread has read best_D[b]
    if (threadIdx.x == 0) best_D[b] = best;
    if (!move) return;
    const bool frozen = best <= kColLimit;
    for (int t = threadIdx.x; t < obs_length; t += blockDim.x) {
        const size_t i = (size_t)t * B + b;
        const float2 o = obs[(size_t)t * M + r0];
        float2 v = delta[i];
        const float2 g = d_obs[(size_t)t * M + r0];
        const double gn = sqrt((double)g.x * g.x + (double)g.y * g.y);
        if (!frozen && finite2(o) && isfinite(gn) && gn > 0.0) {
            double vx = (double)v.x - alpha * ((double)g.x / gn), vy = (double)v.y - alpha * ((double)g.y / gn);
            const double vn = sqrt(vx * vx + vy * vy);
            if (vn > eps) {
                vx *= eps / vn;
                vy *= eps / vn;
            }
            v = make_float2((float)vx, (float)vy);
            delta[i] = v;
        }
        obs_adv[(size_t)t * M + r0] = make_float2(o.x + v.x, o.y + v.y);
    }
}

}  // namespace
}  // namespace tb2

using namespace tb2;

extern "C" {

int tb2_attack_objective(const tb2_layout* l, const float* positions, int32_t num_frames, int32_t first_frame,
                         double* D_out, float* d_positions_out, void* stream) {
    TB2_REQUIRE(l && positions && D_out && d_positions_out, "null argument");
    TB2_REQUIRE(num_frames >= 0 && first_frame >= 0 && first_frame <= num_frames, "need 0 <= first_frame <= num_frames");
    if (l->B == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("attack_objective", st);
        attack_objective_kernel<<<l->B, 32, 0, st>>>((const float2*)positions, l->scene_off, num_frames, first_frame, l->M,
                                                     D_out, (float2*)d_positions_out);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int tb2_attack_step(const tb2_layout* l, const float* d_observed, const float* observed, int32_t obs_length,
                    float* delta, const double* D, int32_t num_frames, const float* positions, double* best_D,
                    float* best_delta, float* best_positions, float* observed_adv, float eps, float alpha, int32_t move,
                    void* stream) {
    TB2_REQUIRE(l && observed && delta && D && positions && best_D && best_delta && best_positions, "null argument");
    TB2_REQUIRE(!move || (d_observed && observed_adv), "a step needs d_observed and observed_adv");
    TB2_REQUIRE(obs_length >= 0 && num_frames >= 0, "negative size");
    TB2_REQUIRE(eps >= 0.f && alpha >= 0.f, "need eps >= 0 and alpha >= 0");
    if (l->B == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("attack_step", st);
        attack_step_kernel<<<l->B, 256, 0, st>>>((const float2*)d_observed, (const float2*)observed, obs_length,
                                                 l->scene_off, l->M, l->B, (float2*)delta, D, num_frames,
                                                 (const float2*)positions, best_D, (float2*)best_delta,
                                                 (float2*)best_positions, (float2*)observed_adv, (double)eps,
                                                 (double)alpha, move);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // extern "C"
