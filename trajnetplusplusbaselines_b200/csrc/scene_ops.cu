// Scene preprocessing on the device (SURVEY.md 8f rank 3): the O(T * M) passes the reference runs per scene in NumPy
// before a batch reaches the model -- drop_distant (lstm/lstm.py:16-22), center_scene's shift + rotation
// (lstm/utils.py:18-51), random_rotation (lstm/utils.py:10-17) -- and inverse_scene after it (augmentation.py:65-68), for a
// whole ragged batch per launch; and the whole training epoch of the native trainer (lstm/trainer.py of this package) in
// one launch: tb2_scenes_gather_epoch assembles every batch from a device-resident scene store, add_noise included.
//
// Arithmetic contract: the reference works in float64 and casts to float32 only when it builds the torch.Tensor
// (lstm/trainer.py:124, lstm/lstm.py:296), so these kernels read / compute float64 with the reference's operation order and
// explicitly unfused multiplies and adds (__dmul_rn / __dadd_rn; NumPy's einsum('ptc,ci->pti') is mul, mul, add) and round
// to float32 once at the end: the float32 batch is bit-identical to the host path.  The O(B) scalars per scene (centre,
// cos / sin of the rotation) are computed by the caller with the reference's libm calls and passed in `frame`.
#include <math_constants.h>

#include "common.cuh"

namespace tb2 {

// One CTA per scene.  keep[row] = nanmin_t |xy[t, row] - xy[t, primary]|^2 < r^2  (all-NaN -> false, like NaN < r^2).
__global__ void __launch_bounds__(128) scenes_drop_distant_kernel(const double2* __restrict__ xy, const int* __restrict__ scene_off,
                                                                  int T, int M, double r2, unsigned char* __restrict__ keep,
                                                                  int* __restrict__ kept_count) {
    const int scene = blockIdx.x;
    const int row0 = scene_off[scene], n = scene_off[scene + 1] - row0;
    int total = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        const int j = base + threadIdx.x;
        int k = 0;
        if (j < n) {
            double best = CUDART_INF;
            for (int t = 0; t < T; ++t) {
                const double2 p = xy[(size_t)t * M + row0];          // the scene's primary (ped 0)
                const double2 q = xy[(size_t)t * M + row0 + j];
                const double dx = __dsub_rn(q.x, p.x), dy = __dsub_rn(q.y, p.y);
                const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
                if (d2 < best) best = d2;                            // NaN compares false: skipped like nanmin
            }
            k = best < r2 ? 1 : 0;
            keep[row0 + j] = (unsigned char)k;
        }
        total += __syncthreads_count(k);
    }
    if (threadIdx.x == 0) kept_count[scene] = total;
}

struct SceneTransformParams {
    const double2* xy;            // [T, M]
    const int* scene_off;         // [B + 1] input rows
    const unsigned char* keep;    // [M] or null (keep all)
    const int* out_off;           // [B + 1] output rows (== scene_off when keep is null)
    const double* frame;          // [B, 4] cx, cy, cos(rotation), sin(rotation) or null
    const double* aug;            // [B, 2] cos(theta), sin(theta) of random_rotation or null
    float2* out;                  // [T, M_out]
    int T, M, M_out;
};

// rotate like einsum('ptc,ci->pti', xy, [[ct, st], [-st, ct]]): out0 = x ct + y (-st), out1 = x st + y ct
__device__ __forceinline__ double2 rotate_rn(double2 v, double ct, double st) {
    double2 o;
    o.x = __dadd_rn(__dmul_rn(v.x, ct), __dmul_rn(v.y, -st));
    o.y = __dadd_rn(__dmul_rn(v.x, st), __dmul_rn(v.y, ct));
    return o;
}

// The same rotation with einsum's accumulation: its sum of products starts from +0.0, so an exact -0.0 (both products
// -0.0, e.g. the centred primary at the last observation) comes out as +0.0; every other value is rotate_rn's.
__device__ __forceinline__ double2 einsum_rotate_rn(double2 v, double ct, double st) {
    double2 o;
    o.x = __dadd_rn(__dadd_rn(0.0, __dmul_rn(v.x, ct)), __dmul_rn(v.y, -st));
    o.y = __dadd_rn(__dadd_rn(0.0, __dmul_rn(v.x, st)), __dmul_rn(v.y, ct));
    return o;
}

// One CTA per scene: ordered compaction of the kept tracks (block scan per chunk of 128), then shift / rotate / cast.
__global__ void __launch_bounds__(128) scenes_transform_kernel(SceneTransformParams p) {
    __shared__ int warp_sum[4];
    const int scene = blockIdx.x;
    const int row0 = p.scene_off[scene], n = p.scene_off[scene + 1] - row0;
    const int out0 = p.out_off[scene];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double cx = 0.0, cy = 0.0, ct = 1.0, st = 0.0, ct2 = 1.0, st2 = 0.0;
    if (p.frame) { cx = p.frame[scene * 4 + 0]; cy = p.frame[scene * 4 + 1]; ct = p.frame[scene * 4 + 2]; st = p.frame[scene * 4 + 3]; }
    if (p.aug) { ct2 = p.aug[scene * 2 + 0]; st2 = p.aug[scene * 2 + 1]; }
    int running = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        const int j = base + threadIdx.x;
        const int k = (j < n) && (!p.keep || p.keep[row0 + j]);
        const unsigned ballot = __ballot_sync(0xffffffffu, k);
        if (lane == 0) warp_sum[warp] = __popc(ballot);
        __syncthreads();
        int before = running + __popc(ballot & ((1u << lane) - 1u));
        int chunk_total = 0;
        for (int w = 0; w < 4; ++w) {
            if (w < warp) before += warp_sum[w];
            chunk_total += warp_sum[w];
        }
        __syncthreads();
        running += chunk_total;
        if (!k) continue;
        const int dst = out0 + before;
        for (int t = 0; t < p.T; ++t) {
            double2 v = p.xy[(size_t)t * p.M + row0 + j];
            if (p.frame) {
                v.x = __dsub_rn(v.x, cx);
                v.y = __dsub_rn(v.y, cy);
                v = rotate_rn(v, ct, st);
            }
            if (p.aug) v = rotate_rn(v, ct2, st2);
            p.out[(size_t)t * p.M_out + dst] = make_float2((float)v.x, (float)v.y);      // cvt.rn, like torch.Tensor(ndarray)
        }
    }
}

struct GatherEpochParams {
    const double2* xy;                 // store [T, M]
    const int* scene_off;              // [n_store + 1] store rows
    const unsigned char* keep;         // [M] or null (keep all)
    const int* kept_count;             // [n_store] kept tracks per store scene
    const int* perm;                   // [n] epoch position -> store scene
    const long long* batch_base;       // [n_batches] first float2 of batch k's [T, M_k] block in `out`
    const int* batch_tracks;           // [n_batches] M_k
    const double* frame;               // [n_store, 4] by store scene, or null
    const double* aug;                 // [n, 2] by epoch position, or null
    const double* noise;               // float64 values, or null
    const long long* noise_off;        // [n] by epoch position: the scene's [noise_frames, kept - 1, 2] block in `noise`
    float2* out;
    int T, M, batch_size, noise_frames;
};

// One CTA per epoch position p (scene perm[p] of batch p / batch_size): its column offset inside the batch is the kept-track
// count of the batch's earlier scenes, then the same ordered compaction / shift / rotation(s) as scenes_transform_kernel
// (the rotations in einsum's accumulation order, so that even the sign of a zero is the reference's), then add_noise's `+=`
// on frames [0, noise_frames) of every non-primary column, then one cvt.rn to float32.
__global__ void __launch_bounds__(128) scenes_gather_epoch_kernel(GatherEpochParams p) {
    __shared__ int warp_sum[4];
    __shared__ int col_base;
    const int pos = blockIdx.x;
    const int scene = p.perm[pos];
    const int batch = pos / p.batch_size;
    const int row0 = p.scene_off[scene], n = p.scene_off[scene + 1] - row0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) col_base = 0;
    __syncthreads();
    int part = 0;
    for (int q = batch * p.batch_size + threadIdx.x; q < pos; q += blockDim.x) part += p.kept_count[p.perm[q]];
    if (part) atomicAdd(&col_base, part);              // integer sum: order-independent
    __syncthreads();
    const int out0 = col_base;
    const int M_b = p.batch_tracks[batch];
    float2* out = p.out + p.batch_base[batch];
    const int kept = p.kept_count[scene];
    const double* noise = p.noise ? p.noise + p.noise_off[pos] : nullptr;
    double cx = 0.0, cy = 0.0, ct = 1.0, st = 0.0, ct2 = 1.0, st2 = 0.0;
    if (p.frame) { cx = p.frame[scene * 4 + 0]; cy = p.frame[scene * 4 + 1]; ct = p.frame[scene * 4 + 2]; st = p.frame[scene * 4 + 3]; }
    if (p.aug) { ct2 = p.aug[pos * 2 + 0]; st2 = p.aug[pos * 2 + 1]; }
    int running = 0;
    for (int base = 0; base < n; base += blockDim.x) {
        const int j = base + threadIdx.x;
        const int k = (j < n) && (!p.keep || p.keep[row0 + j]);
        const unsigned ballot = __ballot_sync(0xffffffffu, k);
        if (lane == 0) warp_sum[warp] = __popc(ballot);
        __syncthreads();
        int before = running + __popc(ballot & ((1u << lane) - 1u));
        int chunk_total = 0;
        for (int w = 0; w < 4; ++w) {
            if (w < warp) before += warp_sum[w];
            chunk_total += warp_sum[w];
        }
        __syncthreads();
        running += chunk_total;
        if (!k) continue;
        const int dst = out0 + before;
        for (int t = 0; t < p.T; ++t) {
            double2 v = p.xy[(size_t)t * p.M + row0 + j];
            if (p.frame) {
                v.x = __dsub_rn(v.x, cx);
                v.y = __dsub_rn(v.y, cy);
                v = einsum_rotate_rn(v, ct, st);
            }
            if (p.aug) v = einsum_rotate_rn(v, ct2, st2);
            if (noise && before > 0 && t < p.noise_frames) {
                const double* e = noise + ((size_t)t * (kept - 1) + (before - 1)) * 2;
                v.x = __dadd_rn(v.x, e[0]);
                v.y = __dadd_rn(v.y, e[1]);
            }
            out[(size_t)t * M_b + dst] = make_float2((float)v.x, (float)v.y);
        }
    }
}

// inverse_scene (augmentation.py:65-68) of float32 predictions: float64 rotation by -rotation, then + centre.
__global__ void __launch_bounds__(128) scenes_inverse_kernel(const float2* __restrict__ xy, const int* __restrict__ scene_off, int S,
                                                             int M, const double* __restrict__ frame, double2* __restrict__ out) {
    const int scene = blockIdx.x;
    const int row0 = scene_off[scene], n = scene_off[scene + 1] - row0;
    const double cx = frame[scene * 4 + 0], cy = frame[scene * 4 + 1], ct = frame[scene * 4 + 2], st = frame[scene * 4 + 3];
    for (int idx = threadIdx.x; idx < S * n; idx += blockDim.x) {
        const int t = idx / n, j = idx - t * n;
        const float2 f = xy[(size_t)t * M + row0 + j];
        double2 v = rotate_rn(make_double2((double)f.x, (double)f.y), ct, st);
        v.x = __dadd_rn(v.x, cx);
        v.y = __dadd_rn(v.y, cy);
        out[(size_t)t * M + row0 + j] = v;
    }
}

}  // namespace tb2

using namespace tb2;

extern "C" {

int tb2_scenes_drop_distant(const double* xy, const int32_t* scene_off, int32_t T, int32_t M, int32_t B, double r_squared,
                            uint8_t* keep_out, int32_t* kept_count_out, void* stream) {
    TB2_REQUIRE(T >= 0 && M >= 0 && B >= 0, "negative size");
    if (B == 0) return TB2_OK;
    TB2_REQUIRE(xy && scene_off && keep_out && kept_count_out, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("scenes_drop_distant", st);
        scenes_drop_distant_kernel<<<B, 128, 0, st>>>((const double2*)xy, scene_off, T, M, r_squared, keep_out, kept_count_out);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int tb2_scenes_transform(const double* xy, const int32_t* scene_off, const uint8_t* keep, const int32_t* out_off, int32_t T,
                         int32_t M, int32_t M_out, int32_t B, const double* frame, const double* aug, float* xy_out,
                         void* stream) {
    TB2_REQUIRE(T >= 0 && M >= 0 && M_out >= 0 && B >= 0, "negative size");
    if (B == 0 || T == 0 || M_out == 0) return TB2_OK;
    TB2_REQUIRE(xy && scene_off && out_off && xy_out, "null argument");
    TB2_REQUIRE(keep || M_out == M, "without a keep mask the output holds every input track");
    SceneTransformParams p;
    p.xy = (const double2*)xy; p.scene_off = scene_off; p.keep = keep; p.out_off = out_off; p.frame = frame; p.aug = aug;
    p.out = (float2*)xy_out; p.T = T; p.M = M; p.M_out = M_out;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("scenes_transform", st);
        scenes_transform_kernel<<<B, 128, 0, st>>>(p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int tb2_scenes_gather_epoch(const double* xy, const int32_t* scene_off, const uint8_t* keep, const int32_t* kept_count,
                            int32_t T, int32_t M, const int32_t* perm, int32_t n, int32_t batch_size,
                            const int64_t* batch_base, const int32_t* batch_tracks, const double* frame, const double* aug,
                            const double* noise, const int64_t* noise_off, int32_t noise_frames, float* xy_out,
                            void* stream) {
    TB2_REQUIRE(T >= 0 && M >= 0 && n >= 0, "negative size");
    TB2_REQUIRE(batch_size >= 1, "batch_size must be >= 1");
    TB2_REQUIRE(noise_frames >= 0 && noise_frames <= T, "noise_frames must lie in [0, T]");
    if (n == 0 || T == 0) return TB2_OK;
    TB2_REQUIRE(xy && scene_off && kept_count && perm && batch_base && batch_tracks && xy_out, "null argument");
    TB2_REQUIRE(!noise || noise_off, "noise needs noise_off");
    GatherEpochParams p;
    p.xy = (const double2*)xy; p.scene_off = scene_off; p.keep = keep; p.kept_count = kept_count; p.perm = perm;
    p.batch_base = (const long long*)batch_base; p.batch_tracks = batch_tracks; p.frame = frame; p.aug = aug;
    p.noise = noise; p.noise_off = (const long long*)noise_off; p.out = (float2*)xy_out;
    p.T = T; p.M = M; p.batch_size = batch_size; p.noise_frames = noise_frames;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("scenes_gather_epoch", st);
        scenes_gather_epoch_kernel<<<n, 128, 0, st>>>(p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int tb2_scenes_inverse(const float* xy, const int32_t* scene_off, int32_t S, int32_t M, int32_t B, const double* frame,
                       double* xy_out, void* stream) {
    TB2_REQUIRE(S >= 0 && M >= 0 && B >= 0, "negative size");
    if (B == 0 || S == 0 || M == 0) return TB2_OK;
    TB2_REQUIRE(xy && scene_off && frame && xy_out, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("scenes_inverse", st);
        scenes_inverse_kernel<<<B, 128, 0, st>>>((const float2*)xy, scene_off, S, M, frame, (double2*)xy_out);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // extern "C"
