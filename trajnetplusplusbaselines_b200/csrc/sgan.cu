// S-GAN generator glue between encoder and decoder -- reference: LSTMGenerator.adding_noise
// (trajnetbaselines/sgan/sgan.py:200-221): h <- cat(ReLU(Linear(H -> H - noise_dim)(h)), z) for
// every track (z is one noise vector shared by all tracks of the call), c unchanged.  The VAE's
// counterpart (h <- h * ReLU(fc z)) and the batched forms that build the decoder state of k modes
// in one pass over the encoder state live here too.
#include "common.cuh"

namespace tb2 {

// ReLU(W[u] . row + b[u]) of one decoder-context unit u < H - nd: the arithmetic every S-GAN context path shares, so that
// the batched decoder context is bit-identical to sgan_add_noise_kernel on a clone of the state.
__device__ __forceinline__ float sgan_context_unit(const float* __restrict__ W, const float* __restrict__ b,
                                                   const float* row_s, int u, int H) {
    const float* w = W + (size_t)u * H;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = 0;
    for (; k + 3 < H; k += 4) {
        a0 = fmaf(w[k], row_s[k], a0);
        a1 = fmaf(w[k + 1], row_s[k + 1], a1);
        a2 = fmaf(w[k + 2], row_s[k + 2], a2);
        a3 = fmaf(w[k + 3], row_s[k + 3], a3);
    }
    for (; k < H; ++k) a0 = fmaf(w[k], row_s[k], a0);
    return fmaxf(((a0 + a1) + (a2 + a3)) + b[u], 0.f);
}

__global__ void __launch_bounds__(128) sgan_add_noise_kernel(const float* __restrict__ W,
                                                             const float* __restrict__ b,
                                                             const float* __restrict__ noise,
                                                             float* __restrict__ h, int M, int H, int nd) {
    extern __shared__ float row_s[];          // [H] the track's hidden state
    const int m = blockIdx.x;
    if (m >= M) return;
    float* hr = h + (size_t)m * H;
    for (int k = threadIdx.x; k < H; k += blockDim.x) row_s[k] = hr[k];
    __syncthreads();
    const int keep = H - nd;
    for (int u = threadIdx.x; u < H; u += blockDim.x) hr[u] = u < keep ? sgan_context_unit(W, b, row_s, u, H) : noise[u - keep];
}

// Decoder starting state of k modes at once, mode-major: output row q * M + m is track m in mode q.
// ReLU(W . h_enc[m] + b) does not depend on the mode, so one CTA per track computes it once and writes it into all k
// replicas, each followed by the noise vector of its (mode, scene): noise[q * G + group_of_row[m]], G scenes per mode.
// The cell state is copied unchanged.
__global__ void __launch_bounds__(128) sgan_decoder_context_kernel(const float* __restrict__ W,
                                                                   const float* __restrict__ b,
                                                                   const float* __restrict__ noise,
                                                                   const int* __restrict__ group_of_row, int G,
                                                                   const float* __restrict__ h_enc,
                                                                   const float* __restrict__ c_enc, int M, int H,
                                                                   int nd, int k, float* __restrict__ h_out,
                                                                   float* __restrict__ c_out) {
    extern __shared__ float row_s[];          // [H] the track's encoder hidden state
    const int m = blockIdx.x;
    if (m >= M) return;
    const float* hr = h_enc + (size_t)m * H;
    const float* cr = c_enc + (size_t)m * H;
    for (int j = threadIdx.x; j < H; j += blockDim.x) row_s[j] = hr[j];
    __syncthreads();
    const int keep = H - nd;
    const size_t g = (size_t)group_of_row[m];
    for (int u = threadIdx.x; u < H; u += blockDim.x) {
        const float cu = cr[u];
        if (u < keep) {
            const float v = sgan_context_unit(W, b, row_s, u, H);
            for (int q = 0; q < k; ++q) {
                const size_t row = (size_t)q * M + m;
                h_out[row * H + u] = v;
                c_out[row * H + u] = cu;
            }
        } else {
            for (int q = 0; q < k; ++q) {
                const size_t row = (size_t)q * M + m;
                h_out[row * H + u] = noise[((size_t)q * G + g) * nd + (u - keep)];
                c_out[row * H + u] = cu;
            }
        }
    }
}

// VAE.add_noise at test time (vae/vae.py:87-106): h[m] <- h[m] * ReLU(fc . z[m] + bias), one latent
// sample z[m] per track; c unchanged.
// ReLU(W[u] . z + b[u]) of one hidden unit: the gate every VAE context path shares (bit-identical results).
__device__ __forceinline__ float vae_gate_unit(const float* __restrict__ W, const float* __restrict__ b,
                                               const float* z_s, int u, int L) {
    const float* w = W + (size_t)u * L;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = 0;
    for (; k + 3 < L; k += 4) {
        a0 = fmaf(w[k], z_s[k], a0);
        a1 = fmaf(w[k + 1], z_s[k + 1], a1);
        a2 = fmaf(w[k + 2], z_s[k + 2], a2);
        a3 = fmaf(w[k + 3], z_s[k + 3], a3);
    }
    for (; k < L; ++k) a0 = fmaf(w[k], z_s[k], a0);
    return fmaxf(((a0 + a1) + (a2 + a3)) + b[u], 0.f);
}

__global__ void __launch_bounds__(128) vae_scale_hidden_kernel(const float* __restrict__ W,
                                                               const float* __restrict__ b,
                                                               const float* __restrict__ z,
                                                               float* __restrict__ h, int M, int H, int L) {
    extern __shared__ float z_s[];            // [L] the track's latent sample
    const int m = blockIdx.x;
    if (m >= M) return;
    for (int k = threadIdx.x; k < L; k += blockDim.x) z_s[k] = z[(size_t)m * L + k];
    __syncthreads();
    for (int u = threadIdx.x; u < H; u += blockDim.x) h[(size_t)m * H + u] *= vae_gate_unit(W, b, z_s, u, L);
}

// Decoder starting state of k modes at once, mode-major: output row r = q * M + m is track m in mode q,
// h_out[r] = h_enc[m] * ReLU(W . z[r] + b) with one latent sample per (mode, track); c_out[r] = c_enc[m].
__global__ void __launch_bounds__(128) vae_decoder_context_kernel(const float* __restrict__ W,
                                                                  const float* __restrict__ b,
                                                                  const float* __restrict__ z,
                                                                  const float* __restrict__ h_enc,
                                                                  const float* __restrict__ c_enc, int M, int H,
                                                                  int L, int k, float* __restrict__ h_out,
                                                                  float* __restrict__ c_out) {
    extern __shared__ float z_s[];            // [L] the row's latent sample
    const size_t r = blockIdx.x;
    if (r >= (size_t)k * M) return;
    const size_t m = r % (size_t)M;
    for (int j = threadIdx.x; j < L; j += blockDim.x) z_s[j] = z[r * L + j];
    __syncthreads();
    for (int u = threadIdx.x; u < H; u += blockDim.x) {
        h_out[r * H + u] = h_enc[m * H + u] * vae_gate_unit(W, b, z_s, u, L);
        c_out[r * H + u] = c_enc[m * H + u];
    }
}

// Sampled LSTM positions (no reference counterpart: the reference feeds back the mean, lstm/lstm.py:232,255): row r of
// one step moves from obs2 + mu to a draw of the step's bivariate normal,
//   pos[r] += (sx e1, sy (rho e1 + sqrt(1 - rho^2) e2)),   (sx, sy, rho) = normals[r, 2:5], (e1, e2) = eps[r],
// the Cholesky factor of [[sx^2, rho sx sy], [rho sx sy, sy^2]] applied to a standard normal pair.  A pair of exactly
// (0, 0) leaves the row's bits untouched (the mean mode keeps its signed zeros); a NaN normal leaves a NaN position.
// Launched inside the PDL step chain: the step's gate kernel wrote normals / pos, the next step's kernels read pos.
__global__ void __launch_bounds__(256) sample_positions_kernel(const float* __restrict__ normals,
                                                               float* __restrict__ pos,
                                                               const float* __restrict__ eps, int rows) {
    grid_dep_wait();          // normals / positions come from the step's gate kernel
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < rows) {
        const float e1 = eps[2 * (size_t)r], e2 = eps[2 * (size_t)r + 1];
        if (e1 != 0.f || e2 != 0.f) {
            const float* n = normals + (size_t)r * 5;
            const float sx = n[2], sy = n[3], rho = n[4];
            const float a = sqrtf(1.f - rho * rho);
            pos[2 * (size_t)r] += sx * e1;
            pos[2 * (size_t)r + 1] += sy * (rho * e1 + a * e2);
        }
    }
    grid_dep_launch();        // after the writes: the next step reads the sampled positions
}

int launch_sample_positions(const float* normals, float* pos, const float* eps, int rows, cudaStream_t st) {
    if (rows <= 0) return TB2_OK;
    {
        KernelTimer kt("sample_positions", st);
        launch_pdl(sample_positions_kernel, dim3((rows + 255) / 256), dim3(256), 0, st, normals, pos, eps, rows);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

}  // namespace tb2

using namespace tb2;

extern "C" int tb2_lstm_sample_positions(const float* normals, float* positions, const float* eps, int32_t rows,
                                         void* stream) {
    TB2_REQUIRE(normals && positions && eps, "null argument (normals, positions and eps are required)");
    TB2_REQUIRE(rows >= 0, "bad sizes");
    return launch_sample_positions(normals, positions, eps, rows, (cudaStream_t)stream);
}

extern "C" int tb2_vae_scale_hidden(const float* weight, const float* bias, const float* z, float* h, int32_t M,
                                    int32_t H, int32_t latent_dim, void* stream) {
    TB2_REQUIRE(weight && bias && z && h, "null argument");
    TB2_REQUIRE(M >= 0 && H > 0 && latent_dim > 0, "bad sizes");
    if (M == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("vae_scale_hidden", st);
        vae_scale_hidden_kernel<<<M, 128, (size_t)latent_dim * sizeof(float), st>>>(weight, bias, z, h, M, H,
                                                                                   latent_dim);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

extern "C" int tb2_sgan_add_noise(const float* weight, const float* bias, const float* noise, float* h,
                                  int32_t M, int32_t H, int32_t noise_dim, void* stream) {
    TB2_REQUIRE(weight && bias && h && (noise || noise_dim == 0), "null argument");
    TB2_REQUIRE(M >= 0 && H > 0 && noise_dim >= 0 && noise_dim < H, "bad sizes");
    if (M == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("sgan_add_noise", st);
        sgan_add_noise_kernel<<<M, 128, (size_t)H * sizeof(float), st>>>(weight, bias, noise, h, M, H, noise_dim);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

extern "C" int tb2_sgan_decoder_context(const float* weight, const float* bias, const float* noise,
                                        const int32_t* group_of_row, int32_t num_groups, const float* h_enc,
                                        const float* c_enc, int32_t M, int32_t H, int32_t noise_dim, int32_t k,
                                        float* h_out, float* c_out, void* stream) {
    TB2_REQUIRE(weight && bias && group_of_row && h_enc && c_enc && h_out && c_out && (noise || noise_dim == 0),
                "null argument");
    TB2_REQUIRE(M >= 0 && H > 0 && noise_dim >= 0 && noise_dim < H && k >= 1 && num_groups >= 1, "bad sizes");
    TB2_REQUIRE((int64_t)k * M <= INT32_MAX, "k * M rows do not fit in 32 bits");
    if (M == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("sgan_decoder_context", st);
        sgan_decoder_context_kernel<<<M, 128, (size_t)H * sizeof(float), st>>>(weight, bias, noise, group_of_row,
                                                                               num_groups, h_enc, c_enc, M, H,
                                                                               noise_dim, k, h_out, c_out);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

extern "C" int tb2_vae_decoder_context(const float* weight, const float* bias, const float* z, const float* h_enc,
                                       const float* c_enc, int32_t M, int32_t H, int32_t latent_dim, int32_t k,
                                       float* h_out, float* c_out, void* stream) {
    TB2_REQUIRE(weight && bias && z && h_enc && c_enc && h_out && c_out, "null argument");
    TB2_REQUIRE(M >= 0 && H > 0 && latent_dim > 0 && k >= 1, "bad sizes");
    TB2_REQUIRE((int64_t)k * M <= INT32_MAX, "k * M rows do not fit in 32 bits");
    if (M == 0) return TB2_OK;
    cudaStream_t st = (cudaStream_t)stream;
    {
        KernelTimer kt("vae_decoder_context", st);
        vae_decoder_context_kernel<<<(unsigned)((int64_t)k * M), 128, (size_t)latent_dim * sizeof(float), st>>>(
            weight, bias, z, h_enc, c_enc, M, H, latent_dim, k, h_out, c_out);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}
