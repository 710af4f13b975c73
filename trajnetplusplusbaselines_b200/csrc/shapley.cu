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

__global__ void __launch_bounds__(kExpandThreads) shapley_expand_kernel(
        const float2* __restrict__ observed, int obs_length, int num_tracks, const int32_t* __restrict__ scene_off,
        const int32_t* __restrict__ instance_first, const int32_t* __restrict__ instance_split, int B, int out_tracks,
        float2* __restrict__ expanded, int32_t* __restrict__ player_rows, int32_t* __restrict__ coalition) {
    extern __shared__ double s_dist[];                  // [N] squared distance to the primary, +inf where not finite
    __shared__ int s_player[kMaxPlayers];               // row of the player of each rank
    const int i = blockIdx.x;
    const int b = scene_of(instance_first, B, i);
    const int K = 31 - __clz(instance_first[b + 1] - instance_first[b]);
    const int mask = i - instance_first[b];
    const int row0 = scene_off[b], N = scene_off[b + 1] - row0;
    const float2* last = observed + (size_t)(obs_length - 1) * num_tracks + row0;
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
        if (rank < K) s_player[rank] = j;
    }
    __syncthreads();
    if (mask == 0 && threadIdx.x < kMaxPlayers) player_rows[b * kMaxPlayers + threadIdx.x] = threadIdx.x < K ? s_player[threadIdx.x] : -1;
    if (threadIdx.x == 0) coalition[i] = mask;
    // row j goes to j - (number of deleted players below j); a deleted player is a rank r < K with bit r of mask clear
    const int out0 = instance_split[i];
    for (int idx = threadIdx.x; idx < obs_length * N; idx += blockDim.x) {
        const int t = idx / N, j = idx - t * N;
        int shift = 0;
        bool kept = true;
        for (int r = 0; r < K; ++r) {
            if ((mask >> r) & 1) continue;
            const int pr = s_player[r];
            shift += pr < j ? 1 : 0;
            kept = kept && pr != j;
        }
        if (kept) expanded[(size_t)t * out_tracks + out0 + j - shift] = observed[(size_t)t * num_tracks + row0 + j];
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
    double cx = 0.0, cy = 0.0, ct = 1.0, st = 0.0;
    if (frame) {
        cx = frame[b * 4 + 0];
        cy = frame[b * 4 + 1];
        ct = frame[b * 4 + 2];
        st = frame[b * 4 + 3];
    }
    for (int m = threadIdx.x; m < n; m += blockDim.x) {
        const int row = instance_split[first + m];      // the instance's primary
        const float2* p = positions + (size_t)(num_frames - T) * num_tracks + row;
        double a, f;
        // the world frame as tb2_scenes_inverse computes it (inverse_scenes): rotate, then add the centre
        ade_fde([&](int t) {
            const float2 q = p[(size_t)t * num_tracks];
            double2 v = make_double2((double)q.x, (double)q.y);
            if (frame) {
                v = rotate_rn(v, ct, st);
                v.x = __dadd_rn(v.x, cx);
                v.y = __dadd_rn(v.y, cy);
            }
            return v;
        }, gt, T, a, f);
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
