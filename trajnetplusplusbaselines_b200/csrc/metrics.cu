// Scoring of TrajNet++ predictions on the device: per scene the ADE / FDE of every predicted mode of the primary, the
// two collision metrics (Col-II against the ground-truth neighbours, Col-I against the predicted ones) and the KDE
// negative log-likelihood of the ground truth under the predicted modes (reference: evaluator/trajnet_evaluator.py
// TrajnetEvaluator.aggregate, evaluator/eval_utils.py ade / fde / collision / topk_*, scipy.stats.gaussian_kde).
//
// One CTA per scene.  Warp w < T (with NLL) fits and evaluates the KDE of timestep w in fp64, one mode per lane and a
// log-sum-exp over the modes; the last warp does ADE / FDE (one mode per lane) and the collision tests (one neighbour per
// lane).  Every reduction has a fixed order and there are no atomics, so the records are bit-identical from run to run.
// The file is compiled with -fmad=false: the collision distances are the same additions and multiplications numpy does,
// so a distance at the 0.2 m threshold decides the same way on both sides.
#include <math.h>

#include "common.cuh"
#include "metrics.cuh"

namespace tb2 {
namespace {

constexpr unsigned kFull = 0xffffffffu;
// Warps per CTA: the task loop strides over the T NLL timesteps plus the ADE / collision task, so any count >= 1 is
// correct; 16 warps x 128 registers fill the register file of an SM.
constexpr int kScoreMaxWarps = 16;

__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

__device__ __forceinline__ double warp_max(double v) {
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(kFull, v, o));
    return v;
}

// eval_utils.collision restricted to the frames both tracks have: consecutive kept frames form a segment on each track,
// each segment is sampled at 3 equally spaced points (np.linspace(p1, p2, 3)), and the tracks collide when the smallest
// distance between paired points is <= 2 * 0.1 m.  np.min propagates NaN, so a segment with a NaN distance never collides.
__device__ bool collides(const double2* __restrict__ prim, const double2* __restrict__ nb, const uint8_t* __restrict__ mask,
                         int T) {
    const double limit = 2.0 * 0.1;
    int prev = -1;
    for (int t = 0; t < T; ++t) {
        if (!mask[t]) continue;
        if (prev >= 0) {
            const double2 p1 = prim[prev], p2 = prim[t], p3 = nb[prev], p4 = nb[t];
            const double ax[3] = {p1.x, p1.x + (p2.x - p1.x) / 2.0, p2.x}, ay[3] = {p1.y, p1.y + (p2.y - p1.y) / 2.0, p2.y};
            const double bx[3] = {p3.x, p3.x + (p4.x - p3.x) / 2.0, p4.x}, by[3] = {p3.y, p3.y + (p4.y - p3.y) / 2.0, p4.y};
            double dmin = INFINITY;
            bool nan = false;
            for (int k = 0; k < 3; ++k) {
                const double dx = ax[k] - bx[k], dy = ay[k] - by[k];
                const double d = sqrt(dx * dx + dy * dy);
                if (isnan(d)) nan = true;
                else dmin = fmin(dmin, d);
            }
            if (!nan && dmin <= limit) return true;
        }
        prev = t;
    }
    return false;
}

// log of the Gaussian KDE of the K modes (Scott factor K^(-1/6), covariance with ddof = 1) at the ground truth, clipped
// below at -20.  Returns false where the timestep is skipped: all modes identical, singular covariance (the Cholesky
// factorisation fails), a NaN, infinite or > 100 value (a NaN ground truth gives a NaN density).
__device__ bool kde_logpdf(const double2* __restrict__ modes, int K, int T, int t, double2 gt, int lane, double* out) {
    if (isnan(gt.x) || isnan(gt.y)) return false;
    const double2 m0 = modes[t];
    bool same = true;
    double sx = 0.0, sy = 0.0;
    for (int m = lane; m < K; m += 32) {
        const double2 p = modes[(size_t)m * T + t];
        same = same && p.x == m0.x && p.y == m0.y;
        sx += p.x;
        sy += p.y;
    }
    if (__all_sync(kFull, same)) return false;
    const double mx = warp_sum(sx) / K, my = warp_sum(sy) / K;
    double cxx = 0.0, cyy = 0.0, cxy = 0.0;
    for (int m = lane; m < K; m += 32) {
        const double2 p = modes[(size_t)m * T + t];
        const double dx = p.x - mx, dy = p.y - my;
        cxx += dx * dx;
        cyy += dy * dy;
        cxy += dx * dy;
    }
    cxx = warp_sum(cxx) / (K - 1);
    cyy = warp_sum(cyy) / (K - 1);
    cxy = warp_sum(cxy) / (K - 1);
    // lower Cholesky factor of the data covariance, then scaled by the bandwidth factor
    if (!(cxx > 0.0)) return false;
    const double d00 = sqrt(cxx), d10 = cxy / d00, r = cyy - d10 * d10;
    if (!(r > 0.0)) return false;
    const double f = pow((double)K, -1.0 / 6.0);
    const double l00 = d00 * f, l10 = d10 * f, l11 = sqrt(r) * f;
    // log-sum-exp over the modes of -|L^-1 (gt - mode)|^2 / 2
    double vmax = -INFINITY;
    for (int m = lane; m < K; m += 32) {
        const double2 p = modes[(size_t)m * T + t];
        const double z0 = (gt.x - p.x) / l00, z1 = ((gt.y - p.y) - l10 * z0) / l11;
        vmax = fmax(vmax, -0.5 * (z0 * z0 + z1 * z1));
    }
    vmax = warp_max(vmax);
    double lp;
    if (vmax == -INFINITY) {
        lp = -INFINITY;
    } else {
        double s = 0.0;
        for (int m = lane; m < K; m += 32) {
            const double2 p = modes[(size_t)m * T + t];
            const double z0 = (gt.x - p.x) / l00, z1 = ((gt.y - p.y) - l10 * z0) / l11;
            s += exp(-0.5 * (z0 * z0 + z1 * z1) - vmax);
        }
        s = warp_sum(s);
        const double two_pi = 6.283185307179586476925286766559;
        lp = vmax + log(s) - log((double)K) - log(two_pi) - log(l00 * l11);
    }
    if (isnan(lp)) return false;
    lp = fmax(lp, -20.0);
    if (isinf(lp) || lp > 100.0) return false;
    *out = lp;
    return true;
}

__global__ void __launch_bounds__(32 * kScoreMaxWarps, 1) score_scenes_kernel(int T, int K, const double2* __restrict__ gt_prim, const double2* __restrict__ pred_prim,
                                    const int32_t* __restrict__ num_modes, const int32_t* __restrict__ gt_off,
                                    const double2* __restrict__ gt_nb, const uint8_t* __restrict__ gt_mask,
                                    const int32_t* __restrict__ pr_off, const double2* __restrict__ pr_nb,
                                    const uint8_t* __restrict__ pr_mask, int with_nll, double* __restrict__ ade,
                                    double* __restrict__ fde, double* __restrict__ nll, int32_t* __restrict__ flags) {
    extern __shared__ double s_lp[];                           // [T] log-likelihoods, then [T] kept flags
    int* s_kept = reinterpret_cast<int*>(s_lp + T);
    const int s = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nw = blockDim.x >> 5;
    const int Ks = min(num_modes[s], K);
    const double2* gt = gt_prim + (size_t)s * T;
    const double2* modes = pred_prim + (size_t)s * K * T;
    const int nll_tasks = with_nll ? T : 0;
    int32_t flag = 0;
    for (int task = warp; task <= nll_tasks; task += nw) {
        if (task < nll_tasks) {
            double lp = 0.0;
            const bool kept = kde_logpdf(modes, Ks, T, task, gt[task], lane, &lp);
            if (lane == 0) {
                s_lp[task] = kept ? lp : 0.0;
                s_kept[task] = kept;
            }
            continue;
        }
        for (int m = lane; m < K; m += 32) {
            double a = NAN, f = NAN;
            if (m < Ks) ade_fde([&](int t) { return modes[(size_t)m * T + t]; }, gt, T, a, f);
            ade[(size_t)s * K + m] = a;
            fde[(size_t)s * K + m] = f;
        }
        const int g0 = gt_off[s], g1 = gt_off[s + 1], p0 = pr_off[s], p1 = pr_off[s + 1];
        bool hit = false;
        for (int j = g0 + lane; j < g1; j += 32) hit = hit || collides(modes, gt_nb + (size_t)j * T, gt_mask + (size_t)j * T, T);
        if (__any_sync(kFull, hit)) flag |= TB2_SCORE_COL_GT;
        hit = false;
        for (int j = p0 + lane; j < p1; j += 32) hit = hit || collides(modes, pr_nb + (size_t)j * T, pr_mask + (size_t)j * T, T);
        if (__any_sync(kFull, hit)) flag |= TB2_SCORE_COL_PRED;
        if (g1 - g0 != p1 - p0) flag |= TB2_SCORE_NEIGH_COUNT_DIFFERS;
    }
    __syncthreads();
    if (threadIdx.x == (unsigned)(32 * (nll_tasks % nw))) {           // lane 0 of the warp that ran the last task
        if (with_nll) {
            double sum = 0.0;
            int kept = 0;
            for (int t = 0; t < T; ++t) {
                if (s_kept[t]) { sum += s_lp[t]; ++kept; }
            }
            if (kept) nll[s] = -(sum / kept);
            else { nll[s] = NAN; flag |= TB2_SCORE_NLL_ALL_SKIPPED; }
        }
        flags[s] = flag;
    }
}

}  // namespace
}  // namespace tb2

using namespace tb2;

extern "C" int tb2_score_scenes(int32_t num_scenes, int32_t pred_length, int32_t max_modes, const double* gt_primary_dev,
                                const double* pred_primary_dev, const int32_t* num_modes_dev, const int32_t* gt_neigh_off_dev,
                                const double* gt_neigh_dev, const uint8_t* gt_neigh_mask_dev,
                                const int32_t* pred_neigh_off_dev, const double* pred_neigh_dev,
                                const uint8_t* pred_neigh_mask_dev, int32_t with_nll, double* ade_out_dev,
                                double* fde_out_dev, double* nll_out_dev, int32_t* flags_out_dev, void* stream) {
    TB2_REQUIRE(num_scenes >= 0, "negative scene count");
    TB2_REQUIRE(pred_length >= 1 && pred_length <= 1024 && max_modes >= 1, "pred_length in 1..1024 and max_modes >= 1");
    if (num_scenes == 0) return TB2_OK;
    TB2_REQUIRE(gt_primary_dev && pred_primary_dev && num_modes_dev && gt_neigh_off_dev && pred_neigh_off_dev && ade_out_dev &&
                    fde_out_dev && flags_out_dev && (!with_nll || nll_out_dev),
                "null argument");
    const auto aligned = [](const void* p) { return ((uintptr_t)p & 15) == 0; };   // positions are read as double2
    TB2_REQUIRE(aligned(gt_primary_dev) && aligned(pred_primary_dev) && aligned(gt_neigh_dev) && aligned(pred_neigh_dev),
                "position arrays must be 16-byte aligned");
    const int warps = with_nll ? (pred_length + 1 < kScoreMaxWarps ? pred_length + 1 : kScoreMaxWarps) : 1;
    const size_t smem = (size_t)pred_length * (sizeof(double) + sizeof(int));
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("score_scenes", st);
        score_scenes_kernel<<<num_scenes, 32 * warps, smem, st>>>(
            pred_length, max_modes, (const double2*)gt_primary_dev, (const double2*)pred_primary_dev, num_modes_dev,
            gt_neigh_off_dev, (const double2*)gt_neigh_dev, gt_neigh_mask_dev, pred_neigh_off_dev,
            (const double2*)pred_neigh_dev, pred_neigh_mask_dev, with_nll ? 1 : 0, ade_out_dev, fde_out_dev, nll_out_dev,
            flags_out_dev);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}
