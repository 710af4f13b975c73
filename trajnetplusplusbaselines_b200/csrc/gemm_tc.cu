// Dense layers of the grid embedding on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
//   Y[M, N] = relu(A[M, K] . W[N, K]^T + b)          (reference: the Linear + ReLU pairs of
//   GridBasedPooling.two_layer / three_layer, trajnetbaselines/lstm/gridbased_pooling.py:316-335)
//
// The ADE/FDE gate (1e-4 m) rules out single-pass bf16/tf32 inputs, so the fp32 operands are
// split into bf16 (hi, lo) pairs and the product is accumulated in fp32 registers from three
// tensor-core passes:  A.W ~= A_hi.W_hi + A_hi.W_lo + A_lo.W_hi   (dropped terms ~ 2^-17 rel.).
// A_hi / A_lo are written by the producing kernel (sparse_layer1), W_hi / W_lo at weight repack.
//
// Kernel shape (one 128 x BN output tile per CTA, 384 threads), mainloop TcRing (wgmma.cuh) with 64-wide k-blocks:
//   warpgroup 2   TMA producer (one thread): A_hi, A_lo 128x64, W_hi, W_lo BNx64 per stage (128B-swizzled)
//   warpgroups 0, 1  rows [64 wg, 64 wg + 64) of the tile: 12 wgmma.m64nBNk16 per stage into fp32 register
//                 accumulators, then bias + ReLU (+ bf16 split) through shared memory and whole-row stores
#include <cuda.h>
#include <cuda_bf16.h>
#include <algorithm>

#include "common.cuh"
#include "wgmma.cuh"

namespace tb2 {

constexpr int kTcBM = 128;
constexpr int kTcBK = 64;          // 64 bf16 = 128 bytes = one swizzle atom
constexpr int kTcThreads = 384;
// BN = 128: 64 KB / stage, 3 stages;  BN = 64: 48 KB / stage, 4 stages (narrow layers)
template <int BN> using DenseRing = TcRing<kTcBM, BN, kTcBK, BN == 128 ? 3 : 4>;

struct TcParams {
    SplitMap a;                // A [M, K]
    SplitMap w;                // W [N, K]
    const float* bias;
    float* Y;                  // fp32 output, or null
    __nv_bfloat16* Y_hi;       // bf16 (hi, lo) split output for a tensor-core consumer, or null
    __nv_bfloat16* Y_lo;
    int M, N, K, relu;
};

template <int kTcBN>
__global__ void __launch_bounds__(kTcThreads, 1) dense_layer_tc_kernel(const __grid_constant__ TcParams p) {
    extern __shared__ __align__(1024) unsigned char smem_tc[];
    __shared__ DenseRing<kTcBN> tc;
    __shared__ float bias_s[kTcBN];

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * kTcBM, n0 = blockIdx.x * kTcBN;
    // 1024-byte aligned tile ring (dynamic smem base alignment is only guaranteed to 16 B)
    const uint32_t ring = (smem_u32(smem_tc) + 1023u) & ~1023u;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a.hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.a.lo) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.w.hi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&p.w.lo) : "memory");
        tc.init();
    }
    __syncthreads();
    grid_dep_wait();          // the A operand is the previous kernel's output
    grid_dep_launch();
    // the bias tile in shared memory: a global load in the epilogue waits its latency (it was issued after stores the
    // compiler cannot rule out that it aliases)
    if (threadIdx.x < kTcBN) bias_s[threadIdx.x] = p.bias[n0 + threadIdx.x];
    float acc[kTcBN / 2];
    tc.run(ring, p.K / kTcBK, m0, [&](int kb) { return TcATile{&p.a, kb * kTcBK}; }, p.w, n0, acc);
    if (wg == 2) return;
    asm volatile("bar.sync 1, 256;" ::: "memory");     // bias_s written, and every consumer is done with the ring
    // epilogue: bias + ReLU (+ bf16 split) from the accumulator fragment (per register pair, one row and two adjacent
    // columns) into row-major tiles in the ring, then whole rows out in 16-byte stores.  Stored from the fragment
    // directly, a warp's store covers 16 or 32 bytes of each of 8 rows.  Row strides are padded by 32 bytes so that
    // the 8 rows of a fragment store fall in different banks.
    constexpr int kYStride = kTcBN + 8;                 // floats
    constexpr int kHStride = kTcBN + 16;                // bf16
    static_assert(kTcBM * (kYStride * 4 + 2 * kHStride * 2) <= DenseRing<kTcBN>::kRingBytes, "output tiles fit the ring");
    float* y_s = reinterpret_cast<float*>(smem_tc + (ring - smem_u32(smem_tc)));
    uint32_t* hi_s = reinterpret_cast<uint32_t*>(y_s + kTcBM * kYStride);
    uint32_t* lo_s = hi_s + kTcBM * kHStride / 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < kTcBN / 2; i += 2) {
        const int r = r0 + 8 * ((i >> 1) & 1);
        const int c = c0 + 8 * (i >> 2);
        float v0 = acc[i] + bias_s[c], v1 = acc[i + 1] + bias_s[c + 1];
        if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        *reinterpret_cast<float2*>(y_s + r * kYStride + c) = make_float2(v0, v1);
        split_bf16x2(make_float2(v0, v1), hi_s[(r * kHStride + c) / 2], lo_s[(r * kHStride + c) / 2]);
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (TB2_GEMM_ABLATE == 3 && p.M > 0) return;
    if (p.Y) {
        constexpr int kChunks = kTcBN / 4;              // 16-byte chunks of a fp32 row
        for (int q = threadIdx.x; q < kTcBM * kChunks; q += 256) {
            const int r = q / kChunks, c = 4 * (q % kChunks);
            if (m0 + r < p.M)
                *reinterpret_cast<float4*>(p.Y + (size_t)(m0 + r) * p.N + n0 + c) =
                    *reinterpret_cast<const float4*>(y_s + r * kYStride + c);
        }
    }
    if (p.Y_hi) {
        constexpr int kChunks = kTcBN / 8;              // 16-byte chunks of a bf16 row
        for (int q = threadIdx.x; q < kTcBM * kChunks; q += 256) {
            const int r = q / kChunks, c = 8 * (q % kChunks);
            if (m0 + r < p.M) {
                const size_t o = (size_t)(m0 + r) * p.N + n0 + c;
                *reinterpret_cast<uint4*>(p.Y_hi + o) = *reinterpret_cast<const uint4*>(hi_s + (r * kHStride + c) / 2);
                *reinterpret_cast<uint4*>(p.Y_lo + o) = *reinterpret_cast<const uint4*>(lo_s + (r * kHStride + c) / 2);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// host side: tensor maps (cuTensorMapEncodeTiled through the runtime's driver entry point, so the
// library does not link libcuda directly)
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// bf16 row-major [rows, cols] matrix, box = [box_rows, box_cols], box_cols = 64 (128B swizzle) or 32 (64B swizzle)
// A descriptor depends on (address, shape, box) only, and the step kernels are launched with the same few operand
// buffers over and over: a small per-thread direct-mapped cache keeps the driver's encode call (a few microseconds,
// 12 per recurrence step) off the launch path.
static int make_bf16_tile_map(CUtensorMap* map, const void* base, int rows, int cols, int box_rows, int box_cols) {
    struct Entry { const void* base; int rows, cols, box_rows, box_cols; bool valid; CUtensorMap map; };
    static thread_local Entry cache[256] = {};
    const uintptr_t key = reinterpret_cast<uintptr_t>(base);
    Entry& e = cache[((key >> 8) ^ (key >> 17) ^ (uintptr_t)(rows * 131 + cols * 7 + box_rows + box_cols)) & 255];
    if (e.valid && e.base == base && e.rows == rows && e.cols == cols && e.box_rows == box_rows &&
        e.box_cols == box_cols) {
        *map = e.map;
        return TB2_OK;
    }
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled unavailable"); return TB2_ERR_CUDA; }
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, box_cols == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")"); return TB2_ERR_CUDA; }
    e.base = base; e.rows = rows; e.cols = cols; e.box_rows = box_rows; e.box_cols = box_cols; e.map = *map;
    e.valid = true;
    return TB2_OK;
}

int make_split_map(SplitMap* map, const void* hi, const void* lo, int rows, int cols, int box_rows, int box_cols) {
    const int rc = make_bf16_tile_map(&map->hi, hi, rows, cols, box_rows, box_cols);
    return rc ? rc : make_bf16_tile_map(&map->lo, lo, rows, cols, box_rows, box_cols);
}

bool dense_tc_supported(int K, int N) { return K >= kTcBK && K % kTcBK == 0 && N % 64 == 0; }

template <int BN>
static int launch_dense_tc_t(const TcParams& p, cudaStream_t st) {
    const size_t smem = DenseRing<BN>::kSmemBytes;
    static DynSmemConfig configured;
    TB2_CHECK_CUDA(configured.ensure(dense_layer_tc_kernel<BN>, smem));
    dim3 grid(p.N / BN, (p.M + kTcBM - 1) / kTcBM);
    {
        KernelTimer kt("dense_layer_tc", st);
        launch_pdl(dense_layer_tc_kernel<BN>, grid, dim3(kTcThreads), smem, st, p);
    }
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int launch_dense_tc(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                    float* Y, void* Y_hi, void* Y_lo, int M, int K, int N, int relu, cudaStream_t st) {
    TB2_REQUIRE(dense_tc_supported(K, N), "tensor-core dense layer needs K % 64 == 0 and N % 64 == 0");
    TcParams p;
    int rc;
    if ((rc = make_split_map(&p.a, a_hi, a_lo, M, K, kTcBM, kTcBK))) return rc;
    const int bn = (N % 128 == 0) ? 128 : 64;
    if ((rc = make_split_map(&p.w, w_hi, w_lo, N, K, bn, kTcBK))) return rc;
    p.bias = bias;
    p.Y = Y;
    p.Y_hi = (__nv_bfloat16*)Y_hi;
    p.Y_lo = (__nv_bfloat16*)Y_lo;
    p.M = M;
    p.N = N;
    p.K = K;
    p.relu = relu;
    return bn == 128 ? launch_dense_tc_t<128>(p, st) : launch_dense_tc_t<64>(p, st);
}

// fp32 [rows, cols] (leading dimension ld_src) -> bf16 (hi, lo) of leading dimension ld_dst; a flat array is one row
__global__ void split_bf16_kernel(const float* __restrict__ src, size_t ld_src, size_t rows, size_t cols,
                                  __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, size_t ld_dst) {
    const size_t total = rows * cols;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = rows == 1 ? 0 : i / cols;         // no 64-bit division for a flat array
        const size_t c = i - r * cols;
        split_bf16(src[r * ld_src + c], hi[r * ld_dst + c], lo[r * ld_dst + c]);
    }
}

int launch_split_bf16_rows(const float* src, size_t ld_src, size_t rows, size_t cols, void* hi, void* lo, size_t ld_dst,
                           unsigned max_blocks, cudaStream_t st) {
    if (rows * cols == 0) return TB2_OK;
    const unsigned blocks = (unsigned)std::min<size_t>((rows * cols + 255) / 256, max_blocks);
    split_bf16_kernel<<<blocks, 256, 0, st>>>(src, ld_src, rows, cols, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ld_dst);
    TB2_LAUNCH_CHECK();
    return TB2_OK;
}

int launch_split_bf16(const float* src, void* hi, void* lo, size_t n, cudaStream_t st) {
    // at most 1184 CTAs of 256 threads (about 9 per SM of a 132-SM H100: one resident wave)
    return launch_split_bf16_rows(src, n, 1, n, hi, lo, n, 1184, st);
}

}  // namespace tb2
