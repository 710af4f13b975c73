// External interaction modules (TB2_POOL_EXTERNAL): any torch.nn.Module that follows the reference's pool plug,
// run by the caller between the step's kernels (reference: LSTM.step, lstm/lstm.py:141-151, with any `pool`).
//
//   pool_inputs_padded_kernel     generate_pooling_inputs (lstm.py:25-42): the ragged obs1 / obs2 / h rows of a step
//                                 as [B, n_pad, .] with NaN in the padding slots, n_pad = the batch's largest scene.
//                                 Every track's hidden state goes in, absent tracks included.
//   pool_inputs_padded_bwd_kernel its backward: d h[m] += d h_padded[slot of m]
//   external_pooled_kernel        pool_sample[track_mask_positions] (lstm.py:148): the module's row of every present
//                                 track as the gate operand (fp32 or the bf16 (hi, lo) pair); zero for absent tracks
//   external_step_grads_kernel    the last phase of tb2_lstm_step_backward: d h_in and the padded d pooled
#include <algorithm>

#include <cuda_bf16.h>
#include <math_constants.h>

#include "common.cuh"

namespace tb2 {

// one CTA per slot (b, j) of [B, n_pad]: track scene_off[b] + j when j is inside scene b, NaN padding otherwise
__global__ void __launch_bounds__(128) pool_inputs_padded_kernel(const int* __restrict__ scene_off, int n_pad,
                                                                 const float2* __restrict__ obs1,
                                                                 const float2* __restrict__ obs2,
                                                                 const float* __restrict__ h, int H,
                                                                 float2* __restrict__ obs1_pad,
                                                                 float2* __restrict__ obs2_pad,
                                                                 float* __restrict__ h_pad) {
    const int slot = blockIdx.x, b = slot / n_pad, j = slot - b * n_pad;
    const int first = scene_off[b];
    const bool real = j < scene_off[b + 1] - first;
    const size_t m = (size_t)first + j;
    const float2 nan2 = make_float2(CUDART_NAN_F, CUDART_NAN_F);
    if (threadIdx.x == 0) {
        obs1_pad[slot] = real ? obs1[m] : nan2;
        obs2_pad[slot] = real ? obs2[m] : nan2;
    }
    float* dst = h_pad + (size_t)slot * H;
    for (int u = threadIdx.x; u < H; u += blockDim.x) dst[u] = real ? h[m * H + u] : CUDART_NAN_F;
}

__global__ void pool_inputs_padded_bwd_kernel(const int* __restrict__ scene_off, const int* __restrict__ row_scene,
                                              int n_pad, const float* __restrict__ d_h_pad, int H,
                                              float* __restrict__ d_h, int M) {
    const size_t total = (size_t)M * H;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int m = (int)(idx / H), u = (int)(idx - (size_t)m * H);
        const int b = row_scene[m], j = m - scene_off[b];
        d_h[idx] += d_h_pad[((size_t)b * n_pad + j) * H + u];
    }
}

// out[m] = (base[m] +) the module's row of track m when it is present at the step (obs1 and obs2 not NaN, lstm.py:118),
// 0 (+ base) otherwise; written as fp32 (out) and / or the bf16 (hi, lo) split of the tensor-core gate operand
__global__ void external_pooled_kernel(const int* __restrict__ scene_off, const int* __restrict__ row_scene, int n_pad,
                                       const float2* __restrict__ obs1, const float2* __restrict__ obs2,
                                       const float* __restrict__ pooled_pad, int P, const float* __restrict__ base,
                                       float* __restrict__ out, __nv_bfloat16* __restrict__ hi,
                                       __nv_bfloat16* __restrict__ lo, int M) {
    const size_t total = (size_t)M * P;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int m = (int)(idx / P), k = (int)(idx - (size_t)m * P);
        const bool present = !(isnan(obs1[m].x) || isnan(obs2[m].x));
        float v = 0.f;
        if (present) {
            const int b = row_scene[m], j = m - scene_off[b];
            v = pooled_pad[((size_t)b * n_pad + j) * P + k];
        }
        if (base) v += base[idx];
        if (out) out[idx] = v;
        if (hi) split_bf16(v, hi[idx], lo[idx]);
    }
}

// one CTA per slot (b, j): d pooled_pad[slot] = d of the pooled operand of a present track (src[m, col .. col + P)),
// 0 for absent tracks and padding; d h_in[m] = pass[m] + dh_rec[m] for the track of a real slot
__global__ void __launch_bounds__(128) external_step_grads_kernel(const int* __restrict__ scene_off, int n_pad,
                                                                  const int* __restrict__ masked,
                                                                  const float* __restrict__ src, int ld_src, int col,
                                                                  int P, const float* __restrict__ pass,
                                                                  const float* __restrict__ dh_rec, int H,
                                                                  float* __restrict__ d_pooled_pad,
                                                                  float* __restrict__ d_h_in) {
    const int slot = blockIdx.x, b = slot / n_pad, j = slot - b * n_pad;
    const int first = scene_off[b];
    const bool real = j < scene_off[b + 1] - first;
    const size_t m = (size_t)first + j;
    const bool present = real && !masked[m];
    float* dp = d_pooled_pad + (size_t)slot * P;
    for (int k = threadIdx.x; k < P; k += blockDim.x) dp[k] = present ? src[m * ld_src + col + k] : 0.f;
    if (!real) return;
    for (int u = threadIdx.x; u < H; u += blockDim.x) d_h_in[m * H + u] = pass[m * H + u] + dh_rec[m * H + u];
}

static unsigned grid_stride_blocks(size_t n) { return (unsigned)std::min<size_t>((n + 255) / 256, 1184); }

int launch_external_pooled(const tb2_lstm* m, const tb2_layout* l, const float* obs1, const float* obs2,
                           const float* pooled_pad, const float* base, float* out, void* hi, void* lo, cudaStream_t st) {
    const int P = m->pool_out;
    if ((size_t)l->M * P == 0) return TB2_OK;
    {
        KernelTimer kt("external_pooled", st);
        external_pooled_kernel<<<grid_stride_blocks((size_t)l->M * P), 256, 0, st>>>(
            l->scene_off, l->row_scene, l->n_max, (const float2*)obs1, (const float2*)obs2, pooled_pad, P, base, out,
            (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, l->M);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int launch_external_step_grads(const tb2_layout* l, const int* masked, const float* src, int ld_src, int col, int P,
                               const float* pass, const float* dh_rec, int H, float* d_pooled_pad, float* d_h_in,
                               cudaStream_t st) {
    {
        KernelTimer kt("external_step_grads", st);
        external_step_grads_kernel<<<l->B * l->n_max, 128, 0, st>>>(l->scene_off, l->n_max, masked, src, ld_src, col, P,
                                                                     pass, dh_rec, H, d_pooled_pad, d_h_in);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // namespace tb2

using namespace tb2;

extern "C" {

int tb2_pool_inputs_padded(const tb2_layout* l, const float* obs1, const float* obs2, const float* h, int32_t H,
                           float* obs1_pad_out, float* obs2_pad_out, float* h_pad_out, void* stream) {
    TB2_REQUIRE(l && obs1 && obs2 && h && obs1_pad_out && obs2_pad_out && h_pad_out, "null argument");
    TB2_REQUIRE(H >= 1, "hidden width");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("pool_inputs_padded", st);
        pool_inputs_padded_kernel<<<l->B * l->n_max, 128, 0, st>>>(l->scene_off, l->n_max, (const float2*)obs1,
                                                                    (const float2*)obs2, h, H, (float2*)obs1_pad_out,
                                                                    (float2*)obs2_pad_out, h_pad_out);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int tb2_pool_inputs_padded_backward(const tb2_layout* l, const float* d_h_pad, int32_t H, float* d_h, void* stream) {
    TB2_REQUIRE(l && d_h_pad && d_h, "null argument");
    TB2_REQUIRE(H >= 1, "hidden width");
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("pool_inputs_padded_bwd", st);
        pool_inputs_padded_bwd_kernel<<<grid_stride_blocks((size_t)l->M * H), 256, 0, st>>>(
            l->scene_off, l->row_scene, l->n_max, d_h_pad, H, d_h, l->M);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // extern "C"
