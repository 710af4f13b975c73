// Shapley attribution of the primary's forecast error to its nearest neighbours (lstm/shapley.py).
//
// tb2_shapley_expand builds the counterfactual scenes: for each scene its K players (the K nearest neighbours of the
// primary at the last observed frame) and, per coalition S of them, one instance = the scene with the players outside S
// deleted, the remaining rows in their original order.  One CTA per instance, which selects the players itself (each
// thread ranks its rows against the others), so nothing per row is built on the host.
//
// tb2_shapley_values scores every instance's primary forecast (ADE / FDE, metrics.cuh: the evaluator's arithmetic)
// into a shared-memory table of the scene's 2^K values, then sums each player's weighted marginals in ascending
// coalition order.  One CTA per scene, no atomics: the results are bit-identical from run to run.  Compiled with
// -fmad=false (build.py), so the values are the evaluator's bits and the sums the float64 restatement's.
//
// The sampled estimator (any K): tb2_shapley_sample_expand selects each scene's players once (one CTA per scene), then
// writes the instances of the permutation prefixes (one CTA per instance); tb2_shapley_sample_values scores every
// instance into global memory (one thread per instance), then reduces each player's antithetic-pair marginals in
// ascending pair order (one CTA per scene, no atomics).
#include <math.h>

#include "common.cuh"
#include "metrics.cuh"

namespace tb2 {
namespace {

constexpr int kMaxPlayers = 12;
constexpr int kExpandThreads = 128;
constexpr int kValuesThreads = 256;
// The expansion keeps one float64 distance per row of a scene in shared memory (48 KB without opting in)
constexpr int kMaxSceneRows = 6144;

// The scene an instance belongs to: the last b with instance_first[b] <= i
__device__ __forceinline__ int scene_of(const int32_t* __restrict__ instance_first, int B, int i) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (instance_first[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// The scene's K players, by rank, into player[0, K): the K nearest neighbours of the primary at the last observed frame
// last [N] (primary first), squared distance in float64, +inf where not finite, ties to the lower row.  s_dist [N] is
// shared scratch; player may be shared or global.  The caller synchronises before reading player.
__device__ __forceinline__ void select_players(const float2* __restrict__ last, int N, int K, double* s_dist,
                                               int32_t* player) {
    const float2 p0 = last[0];
    for (int j = 1 + threadIdx.x; j < N; j += blockDim.x) {
        const float2 p = last[j];
        const double dx = (double)p.x - (double)p0.x, dy = (double)p.y - (double)p0.y;
        const double d = dx * dx + dy * dy;
        s_dist[j] = isfinite(d) ? d : INFINITY;
    }
    __syncthreads();
    // rank of row j among the neighbours: nearer rows first, ties to the lower row; ranks < K are the players
    for (int j = 1 + threadIdx.x; j < N; j += blockDim.x) {
        const double d = s_dist[j];
        int rank = 0;
        for (int r = 1; r < N && rank < K; ++r) rank += (s_dist[r] < d || (s_dist[r] == d && r < j)) ? 1 : 0;
        if (rank < K) player[rank] = j;
    }
}

// s_dest [N]: on entry 1 for a kept row and 0 for a deleted one; on return the kept row's position in the instance
// (its rank among the kept rows), -1 for a deleted one.  s_part [blockDim.x] is scratch.  Then every kept row of the
// scene's observation goes to its position in the instance at out0.
__device__ __forceinline__ void copy_kept_rows(const float2* __restrict__ observed, int obs_length, int num_tracks,
                                               int row0, int N, int* s_dest, int* s_part,
                                               float2* __restrict__ expanded, int out_tracks, int out0) {
    const int per = (N + blockDim.x - 1) / blockDim.x;
    const int j0 = min(N, (int)threadIdx.x * per), j1 = min(N, j0 + per);
    int kept = 0;
    for (int j = j0; j < j1; ++j) kept += s_dest[j];
    s_part[threadIdx.x] = kept;
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int t = 0; t < (int)blockDim.x; ++t) {
            const int c = s_part[t];
            s_part[t] = acc;
            acc += c;
        }
    }
    __syncthreads();
    int pos = s_part[threadIdx.x];
    for (int j = j0; j < j1; ++j) s_dest[j] = s_dest[j] ? pos++ : -1;
    __syncthreads();
    for (int idx = threadIdx.x; idx < obs_length * N; idx += blockDim.x) {
        const int t = idx / N, j = idx - t * N;
        const int d = s_dest[j];
        if (d >= 0) expanded[(size_t)t * out_tracks + out0 + d] = observed[(size_t)t * num_tracks + row0 + j];
    }
}

__global__ void __launch_bounds__(kExpandThreads) shapley_expand_kernel(
        const float2* __restrict__ observed, int obs_length, int num_tracks, const int32_t* __restrict__ scene_off,
        const int32_t* __restrict__ instance_first, const int32_t* __restrict__ instance_split, int B, int out_tracks,
        float2* __restrict__ expanded, int32_t* __restrict__ player_rows, int32_t* __restrict__ coalition) {
    extern __shared__ double s_dist[];                  // [N] squared distance to the primary, then the rows' positions
    __shared__ int s_player[kMaxPlayers];               // row of the player of each rank
    __shared__ int s_part[kExpandThreads];
    const int i = blockIdx.x;
    const int b = scene_of(instance_first, B, i);
    const int K = 31 - __clz(instance_first[b + 1] - instance_first[b]);
    const int mask = i - instance_first[b];
    const int row0 = scene_off[b], N = scene_off[b + 1] - row0;
    select_players(observed + (size_t)(obs_length - 1) * num_tracks + row0, N, K, s_dist, s_player);
    __syncthreads();
    if (mask == 0 && threadIdx.x < kMaxPlayers) player_rows[b * kMaxPlayers + threadIdx.x] = threadIdx.x < K ? s_player[threadIdx.x] : -1;
    if (threadIdx.x == 0) coalition[i] = mask;
    // the distances are done with: their storage holds the rows' flags, then positions
    int* s_dest = reinterpret_cast<int*>(s_dist);
    for (int j = threadIdx.x; j < N; j += blockDim.x) s_dest[j] = 1;
    __syncthreads();
    // a deleted player is a rank r < K with bit r of mask clear
    if (threadIdx.x < K && !((mask >> threadIdx.x) & 1)) s_dest[s_player[threadIdx.x]] = 0;
    __syncthreads();
    copy_kept_rows(observed, obs_length, num_tracks, row0, N, s_dest, s_part, expanded, out_tracks, instance_split[i]);
}

// Instances of a scene with K players under the sampled estimator: 1 for K = 0, else 2 + P (K - 1)
__device__ __forceinline__ int sampled_players(int instances, int P) {
    return instances == 1 ? 0 : (instances - 2) / P + 1;
}

// Local instance of the first k players of permutation p: 0 the empty coalition, 1 the full one, then P runs of K - 1
__device__ __forceinline__ int sampled_instance(int p, int k, int K) {
    return k == 0 ? 0 : k == K ? 1 : 2 + p * (K - 1) + k - 1;
}

__global__ void __launch_bounds__(kExpandThreads) shapley_sample_players_kernel(
        const float2* __restrict__ observed, int obs_length, int num_tracks, const int32_t* __restrict__ scene_off,
        const int32_t* __restrict__ instance_first, int P, int max_players, int32_t* __restrict__ player_rows) {
    extern __shared__ double s_dist[];                  // [N]
    const int b = blockIdx.x;
    const int K = sampled_players(instance_first[b + 1] - instance_first[b], P);
    const int row0 = scene_off[b], N = scene_off[b + 1] - row0;
    int32_t* rows = player_rows + (size_t)b * max_players;
    select_players(observed + (size_t)(obs_length - 1) * num_tracks + row0, N, K, s_dist, rows);
    for (int r = K + threadIdx.x; r < max_players; r += blockDim.x) rows[r] = -1;
}

__global__ void __launch_bounds__(kExpandThreads) shapley_sample_expand_kernel(
        const float2* __restrict__ observed, int obs_length, int num_tracks, const int32_t* __restrict__ scene_off,
        const int32_t* __restrict__ instance_first, const int32_t* __restrict__ instance_split,
        const int32_t* __restrict__ perms, int B, int pairs, int max_players, const int32_t* __restrict__ player_rows,
        int out_tracks, float2* __restrict__ expanded) {
    extern __shared__ int s_dest[];                     // [N] the rows' flags, then positions
    __shared__ int s_part[kExpandThreads];
    const int i = blockIdx.x;
    const int b = scene_of(instance_first, B, i);
    const int P = 2 * pairs;
    const int K = sampled_players(instance_first[b + 1] - instance_first[b], P);
    const int m = i - instance_first[b];
    const int row0 = scene_off[b], N = scene_off[b + 1] - row0;
    const int32_t* prow = player_rows + (size_t)b * max_players;
    for (int j = threadIdx.x; j < N; j += blockDim.x) s_dest[j] = 1;
    __syncthreads();
    if (m == 0) {
        for (int r = threadIdx.x; r < K; r += blockDim.x) s_dest[prow[r]] = 0;
    } else if (m >= 2) {
        // permutation p (pair p / 2's drawn one for even p, reversed for odd p) keeps its first k ranks
        const int p = (m - 2) / (K - 1), k = m - 2 - p * (K - 1) + 1;
        const int32_t* pi = perms + ((size_t)b * pairs + (p >> 1)) * max_players;
        for (int r = k + threadIdx.x; r < K; r += blockDim.x) s_dest[prow[(p & 1) ? pi[K - 1 - r] : pi[r]]] = 0;
    }
    __syncthreads();
    copy_kept_rows(observed, obs_length, num_tracks, row0, N, s_dest, s_part, expanded, out_tracks, instance_split[i]);
}

// The frame of scene b ([cx, cy, cos, sin] of frame [B, 4]); the identity without one
struct SceneFrame {
    double cx = 0.0, cy = 0.0, ct = 1.0, st = 0.0;
    bool on = false;
    __device__ __forceinline__ SceneFrame(const double* __restrict__ frame, int b) {
        if (frame) {
            cx = frame[b * 4 + 0];
            cy = frame[b * 4 + 1];
            ct = frame[b * 4 + 2];
            st = frame[b * 4 + 3];
            on = true;
        }
    }
};

// (ADE, FDE) of the primary at row of positions against gt [T], in the world frame as tb2_scenes_inverse computes it
// (inverse_scenes): rotate, then add the centre
__device__ __forceinline__ void score_primary(const float2* __restrict__ positions, int num_frames, int num_tracks,
                                              int T, int row, const double2* __restrict__ gt, const SceneFrame& fr,
                                              double& a, double& f) {
    const float2* p = positions + (size_t)(num_frames - T) * num_tracks + row;
    ade_fde([&](int t) {
        const float2 q = p[(size_t)t * num_tracks];
        double2 v = make_double2((double)q.x, (double)q.y);
        if (fr.on) {
            v = rotate_rn(v, fr.ct, fr.st);
            v.x = __dadd_rn(v.x, fr.cx);
            v.y = __dadd_rn(v.y, fr.cy);
        }
        return v;
    }, gt, T, a, f);
}

__global__ void __launch_bounds__(kValuesThreads) shapley_sample_score_kernel(
        const float2* __restrict__ positions, int num_frames, int num_tracks, int T,
        const int32_t* __restrict__ instance_first, const int32_t* __restrict__ instance_split,
        const double2* __restrict__ truth, const double* __restrict__ frame, int B, int I, double* __restrict__ values) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= I) return;
    const int b = scene_of(instance_first, B, i);
    double a, f;
    score_primary(positions, num_frames, num_tracks, T, instance_split[i], truth + (size_t)b * T, SceneFrame(frame, b),
                  a, f);
    values[(size_t)i * 2 + 0] = a;
    values[(size_t)i * 2 + 1] = f;
}

// Thread (metric, j) of scene b's CTA: per pair q, a_q = (m + m') * 0.5 with m, m' j's marginals v(first k + 1) -
// v(first k) in the pair's drawn permutation and in its reverse; phi = (sum over ascending q of a_q) / Q, se =
// sqrt((sum over ascending q of (a_q - phi)^2) / (Q (Q - 1))).  phi and se are accumulated in place.
__global__ void __launch_bounds__(kValuesThreads) shapley_sample_reduce_kernel(
        const double* __restrict__ values, const int32_t* __restrict__ instance_first, const int32_t* __restrict__ perms,
        int B, int pairs, int max_players, double* __restrict__ phi_ade, double* __restrict__ phi_fde,
        double* __restrict__ se_ade, double* __restrict__ se_fde, double* __restrict__ v_out) {
    extern __shared__ int s_inv[];                      // [K] the position of each rank in the pair's permutation
    const int b = blockIdx.x;
    const int first = instance_first[b];
    const int P = 2 * pairs;
    const int K = sampled_players(instance_first[b + 1] - first, P);
    const double* v = values + (size_t)first * 2;
    const double Q = (double)pairs;
    for (int pass = 0; pass < 2; ++pass) {
        for (int q = 0; q < pairs; ++q) {
            const int32_t* pi = perms + ((size_t)b * pairs + q) * max_players;
            __syncthreads();
            for (int k = threadIdx.x; k < K; k += blockDim.x) s_inv[pi[k]] = k;
            __syncthreads();
            for (int task = threadIdx.x; task < 2 * K; task += blockDim.x) {
                const int metric = task >= K, j = task - metric * K;
                const int k = s_inv[j], kr = K - 1 - k;
                const double m0 = v[sampled_instance(2 * q, k + 1, K) * 2 + metric] -
                                  v[sampled_instance(2 * q, k, K) * 2 + metric];
                const double m1 = v[sampled_instance(2 * q + 1, kr + 1, K) * 2 + metric] -
                                  v[sampled_instance(2 * q + 1, kr, K) * 2 + metric];
                const double a = (m0 + m1) * 0.5;
                double* phi = (metric ? phi_fde : phi_ade) + (size_t)b * max_players + j;
                if (pass == 0) {
                    *phi = (q ? *phi : 0.0) + a;
                } else {
                    double* se = (metric ? se_fde : se_ade) + (size_t)b * max_players + j;
                    const double d = a - *phi;
                    *se = (q ? *se : 0.0) + d * d;
                }
            }
        }
        for (int task = threadIdx.x; task < 2 * K; task += blockDim.x) {
            const int metric = task >= K, j = task - metric * K;
            const size_t o = (size_t)b * max_players + j;
            if (pass == 0) (metric ? phi_fde : phi_ade)[o] /= Q;
            else (metric ? se_fde : se_ade)[o] = sqrt((metric ? se_fde : se_ade)[o] / (Q * (Q - 1.0)));
        }
    }
    for (int j = K + threadIdx.x; j < max_players; j += blockDim.x) {
        const size_t o = (size_t)b * max_players + j;
        phi_ade[o] = phi_fde[o] = se_ade[o] = se_fde[o] = NAN;
    }
    if (threadIdx.x == 0) {
        const int full = K ? 1 : 0;
        v_out[0 * B + b] = v[full * 2 + 0];
        v_out[1 * B + b] = v[full * 2 + 1];
        v_out[2 * B + b] = v[0];
        v_out[3 * B + b] = v[1];
    }
}

__global__ void __launch_bounds__(kValuesThreads) shapley_values_kernel(
        const float2* __restrict__ positions, int num_frames, int num_tracks, int T,
        const int32_t* __restrict__ instance_first, const int32_t* __restrict__ instance_split,
        const double2* __restrict__ truth, const double* __restrict__ frame, int B, double* __restrict__ phi_ade,
        double* __restrict__ phi_fde, double* __restrict__ v_out, double* __restrict__ values_out) {
    extern __shared__ double s_v[];                     // [2^K] v_ADE, then [2^K] v_FDE
    __shared__ double s_w[kMaxPlayers];                 // |S|! (K - |S| - 1)! / K!
    const int b = blockIdx.x;
    const int first = instance_first[b], n = instance_first[b + 1] - first;
    const int K = 31 - __clz(n);
    double* v_ade = s_v;
    double* v_fde = s_v + n;
    const double2* gt = truth + (size_t)b * T;
    const SceneFrame fr(frame, b);
    for (int m = threadIdx.x; m < n; m += blockDim.x) {
        double a, f;
        score_primary(positions, num_frames, num_tracks, T, instance_split[first + m], gt, fr, a, f);  // its primary
        v_ade[m] = a;
        v_fde[m] = f;
        if (values_out) {
            values_out[(size_t)(first + m) * 2 + 0] = a;
            values_out[(size_t)(first + m) * 2 + 1] = f;
        }
    }
    if (threadIdx.x < K) {
        double num = 1.0, den = 1.0;                    // exact integers up to 12! < 2^53
        for (int q = 2; q <= threadIdx.x; ++q) num *= q;
        for (int q = 2; q <= K - (int)threadIdx.x - 1; ++q) num *= q;
        for (int q = 2; q <= K; ++q) den *= q;
        s_w[threadIdx.x] = num / den;
    }
    __syncthreads();
    // thread (metric, j): phi_j = sum over S subset of P \ {j}, ascending S, of w(|S|) (v(S u {j}) - v(S))
    for (int task = threadIdx.x; task < 2 * kMaxPlayers; task += blockDim.x) {
        const int metric = task / kMaxPlayers, j = task - metric * kMaxPlayers;
        double phi = NAN;
        if (j < K) {
            const double* v = metric ? v_fde : v_ade;
            const unsigned low = (1u << j) - 1u;
            phi = 0.0;
            for (unsigned s = 0; s < (unsigned)n >> 1; ++s) {
                const unsigned S = ((s & ~low) << 1) | (s & low);
                phi += s_w[__popc(S)] * (v[S | (1u << j)] - v[S]);
            }
        }
        (metric ? phi_fde : phi_ade)[b * kMaxPlayers + j] = phi;
    }
    if (threadIdx.x == 0) {
        v_out[0 * B + b] = v_ade[n - 1];
        v_out[1 * B + b] = v_fde[n - 1];
        v_out[2 * B + b] = v_ade[0];
        v_out[3 * B + b] = v_fde[0];
    }
}

}  // namespace
}  // namespace tb2

using namespace tb2;

extern "C" int tb2_shapley_expand(const float* observed_dev, int32_t obs_length, int32_t num_tracks,
                                  const int32_t* scene_off_dev, const int32_t* instance_first_dev,
                                  const int32_t* instance_split_dev, int32_t num_scenes, int32_t num_instances,
                                  int32_t max_scene, int32_t out_tracks, float* expanded_out_dev,
                                  int32_t* player_rows_out_dev, int32_t* coalition_out_dev, void* stream) {
    TB2_REQUIRE(num_scenes >= 0 && num_instances >= num_scenes && num_tracks >= 0 && out_tracks >= 0,
                "negative size, or fewer instances than scenes");
    TB2_REQUIRE(obs_length >= 1, "obs_length must be >= 1");
    if (num_scenes == 0) return TB2_OK;
    TB2_REQUIRE(max_scene >= 1 && max_scene <= kMaxSceneRows, "max_scene must be in 1..6144");
    TB2_REQUIRE(num_instances <= num_scenes * (1 << kMaxPlayers), "more than 2^12 instances per scene");
    TB2_REQUIRE(observed_dev && scene_off_dev && instance_first_dev && instance_split_dev && expanded_out_dev &&
                    player_rows_out_dev && coalition_out_dev,
                "null argument");
    TB2_REQUIRE(((uintptr_t)observed_dev & 7) == 0 && ((uintptr_t)expanded_out_dev & 7) == 0,
                "position arrays must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("shapley_expand", st);
        shapley_expand_kernel<<<num_instances, kExpandThreads, (size_t)max_scene * sizeof(double), st>>>(
            (const float2*)observed_dev, obs_length, num_tracks, scene_off_dev, instance_first_dev, instance_split_dev,
            num_scenes, out_tracks, (float2*)expanded_out_dev, player_rows_out_dev, coalition_out_dev);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

extern "C" int tb2_shapley_values(const float* positions_dev, int32_t num_frames, int32_t num_tracks,
                                  int32_t pred_length, const int32_t* instance_first_dev,
                                  const int32_t* instance_split_dev, int32_t num_scenes, int32_t max_players,
                                  const double* truth_dev, const double* frame_dev, double* phi_ade_out_dev,
                                  double* phi_fde_out_dev, double* v_out_dev, double* values_out_dev, void* stream) {
    TB2_REQUIRE(num_scenes >= 0 && num_tracks >= 0, "negative size");
    TB2_REQUIRE(pred_length >= 1 && pred_length <= num_frames, "pred_length must be in 1..num_frames");
    TB2_REQUIRE(max_players >= 0 && max_players <= kMaxPlayers, "max_players must be in 0..12");
    if (num_scenes == 0) return TB2_OK;
    TB2_REQUIRE(positions_dev && instance_first_dev && instance_split_dev && truth_dev && phi_ade_out_dev &&
                    phi_fde_out_dev && v_out_dev,
                "null argument");
    TB2_REQUIRE(((uintptr_t)positions_dev & 7) == 0 && ((uintptr_t)truth_dev & 15) == 0,
                "positions must be 8-byte and truth 16-byte aligned");
    const size_t smem = (size_t)2 * ((size_t)1 << max_players) * sizeof(double);
    static DynSmemConfig smem_cfg;
    TB2_CHECK_CUDA(smem_cfg.ensure(shapley_values_kernel, smem, 48 * 1024));
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("shapley_values", st);
        shapley_values_kernel<<<num_scenes, kValuesThreads, smem, st>>>(
            (const float2*)positions_dev, num_frames, num_tracks, pred_length, instance_first_dev, instance_split_dev,
            (const double2*)truth_dev, frame_dev, num_scenes, phi_ade_out_dev, phi_fde_out_dev, v_out_dev,
            values_out_dev);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

extern "C" int tb2_shapley_sample_expand(const float* observed_dev, int32_t obs_length, int32_t num_tracks,
                                         const int32_t* scene_off_dev, const int32_t* instance_first_dev,
                                         const int32_t* instance_split_dev, const int32_t* permutations_dev,
                                         int32_t num_scenes, int32_t num_instances, int32_t pairs, int32_t max_players,
                                         int32_t max_scene, int32_t out_tracks, float* expanded_out_dev,
                                         int32_t* player_rows_out_dev, void* stream) {
    TB2_REQUIRE(num_scenes >= 0 && num_instances >= num_scenes && num_tracks >= 0 && out_tracks >= 0,
                "negative size, or fewer instances than scenes");
    TB2_REQUIRE(obs_length >= 1, "obs_length must be >= 1");
    TB2_REQUIRE(pairs >= 2, "pairs must be >= 2 (at least 4 permutations)");
    TB2_REQUIRE(max_players >= 1 && max_players < kMaxSceneRows, "max_players must be in 1..6143");
    if (num_scenes == 0) return TB2_OK;
    TB2_REQUIRE(max_scene >= 1 && max_scene <= kMaxSceneRows, "max_scene must be in 1..6144");
    TB2_REQUIRE(observed_dev && scene_off_dev && instance_first_dev && instance_split_dev && permutations_dev &&
                    expanded_out_dev && player_rows_out_dev,
                "null argument");
    TB2_REQUIRE(((uintptr_t)observed_dev & 7) == 0 && ((uintptr_t)expanded_out_dev & 7) == 0,
                "position arrays must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("shapley_sample_players", st);
        shapley_sample_players_kernel<<<num_scenes, kExpandThreads, (size_t)max_scene * sizeof(double), st>>>(
            (const float2*)observed_dev, obs_length, num_tracks, scene_off_dev, instance_first_dev, 2 * pairs,
            max_players, player_rows_out_dev);
    }
    TB2_LAUNCH_CHECK();
    {
        KernelTimer kt("shapley_sample_expand", st);
        shapley_sample_expand_kernel<<<num_instances, kExpandThreads, (size_t)max_scene * sizeof(int), st>>>(
            (const float2*)observed_dev, obs_length, num_tracks, scene_off_dev, instance_first_dev, instance_split_dev,
            permutations_dev, num_scenes, pairs, max_players, player_rows_out_dev, out_tracks,
            (float2*)expanded_out_dev);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

extern "C" int tb2_shapley_sample_values(const float* positions_dev, int32_t num_frames, int32_t num_tracks,
                                         int32_t pred_length, const int32_t* instance_first_dev,
                                         const int32_t* instance_split_dev, const int32_t* permutations_dev,
                                         int32_t num_scenes, int32_t num_instances, int32_t pairs, int32_t max_players,
                                         const double* truth_dev, const double* frame_dev, double* values_out_dev,
                                         double* phi_ade_out_dev, double* phi_fde_out_dev, double* se_ade_out_dev,
                                         double* se_fde_out_dev, double* v_out_dev, void* stream) {
    TB2_REQUIRE(num_scenes >= 0 && num_instances >= num_scenes && num_tracks >= 0,
                "negative size, or fewer instances than scenes");
    TB2_REQUIRE(pred_length >= 1 && pred_length <= num_frames, "pred_length must be in 1..num_frames");
    TB2_REQUIRE(pairs >= 2, "pairs must be >= 2 (at least 4 permutations)");
    TB2_REQUIRE(max_players >= 1 && max_players < kMaxSceneRows, "max_players must be in 1..6143");
    if (num_scenes == 0) return TB2_OK;
    TB2_REQUIRE(positions_dev && instance_first_dev && instance_split_dev && permutations_dev && truth_dev &&
                    values_out_dev && phi_ade_out_dev && phi_fde_out_dev && se_ade_out_dev && se_fde_out_dev &&
                    v_out_dev,
                "null argument");
    TB2_REQUIRE(((uintptr_t)positions_dev & 7) == 0 && ((uintptr_t)truth_dev & 15) == 0,
                "positions must be 8-byte and truth 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("shapley_sample_score", st);
        shapley_sample_score_kernel<<<(num_instances + kValuesThreads - 1) / kValuesThreads, kValuesThreads, 0, st>>>(
            (const float2*)positions_dev, num_frames, num_tracks, pred_length, instance_first_dev, instance_split_dev,
            (const double2*)truth_dev, frame_dev, num_scenes, num_instances, values_out_dev);
    }
    TB2_LAUNCH_CHECK();
    {
        KernelTimer kt("shapley_sample_reduce", st);
        shapley_sample_reduce_kernel<<<num_scenes, kValuesThreads, (size_t)max_players * sizeof(int), st>>>(
            values_out_dev, instance_first_dev, permutations_dev, num_scenes, pairs, max_players, phi_ade_out_dev,
            phi_fde_out_dev, se_ade_out_dev, se_fde_out_dev, v_out_dev);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}
