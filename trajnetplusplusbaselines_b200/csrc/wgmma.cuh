// Hopper (sm_90a) building blocks of the tensor-core kernels: mbarrier, TMA tile loads,
// warpgroup MMA (wgmma) on bf16 operands in 128-byte-swizzled, K-major shared-memory tiles, and
// TcRing, the 3-pass mainloop dense_layer_tc and lstm_gates_tc share.
//
// Tile layout (written by TMA with CU_TENSOR_MAP_SWIZZLE_128B): rows of 64 bf16 (128 bytes),
// 8-row atoms of 1024 bytes, so a tile must start on a 1024-byte boundary (SWIZZLE_64B: rows of 32
// bf16, 512-byte atoms).  One wgmma consumes K = 16 (32 bytes of a row); the next K step advances
// the descriptor's start address by 32 bytes.
//
// Accumulator fragment of wgmma.m64nNk16 (f32), thread t of the warpgroup, register i < N / 2:
//   row = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),   col = 8 * (i / 4) + 2 * (t % 4) + i % 2
#pragma once
#include <cuda.h>
#include <stdint.h>

#include "common.cuh"

// TB2_GEMM_ABLATE (scripts/step_gemm_ablate.py, timing only, results wrong) takes one part out of dense_layer_tc and
// lstm_gates_tc: 1 = no wgmma (loads and barriers only), 2 = one stage loaded, every k-block reads it (wgmma issue
// without the L2 operand stream), 3 = no epilogue stores (nor the arithmetic that feeds them), 4 = one wgmma group in
// flight: wait_group 1 after committing k-block kb, then kb - 1's stage released.  1, 2 and 4 act in TcRing, 3 in the
// kernels' epilogues.  Unset in the library, which waits for each k-block's group before releasing its stage: the
// variant was no faster (DESIGN §8).
#ifndef TB2_GEMM_ABLATE
#define TB2_GEMM_ABLATE 0
#endif

namespace tb2 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}

// wgmma shared-memory matrix descriptor: K-major rows of kRowBytes (128: SWIZZLE_128B, 64 bf16 a row; 64:
// SWIZZLE_64B, 32 bf16 a row), stride byte offset 8 rows between 8-row atoms (the leading byte offset is unused for
// swizzled K-major tiles)
template <int kRowBytes = 128>
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr) {
    static_assert(kRowBytes == 128 || kRowBytes == 64, "128- or 64-byte swizzled rows");
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);          // start address, bits [0,14)
    d |= (uint64_t)1 << 16;                               // leading byte offset (unused)
    d |= (uint64_t)(8 * kRowBytes >> 4) << 32;            // stride byte offset, bits [32,46)
    d |= (uint64_t)(kRowBytes == 128 ? 1 : 2) << 62;      // layout type SWIZZLE_128B / SWIZZLE_64B
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64, N] (+)= A[64, 16] . B[N, 16]^T, both operands bf16 K-major in shared memory, fp32 accumulate;
// accumulate == 0 overwrites D.  Overloaded on N through the accumulator array (N / 2 registers).
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(accumulate));
}

// k-block kb's A operand in TcRing: the tiles at (col, m0) of `map`
struct TcATile {
    const SplitMap* map;
    int col;
};

// The 3-pass mainloop of dense_layer_tc and lstm_gates_tc, 384 threads.  Thread 256 (warpgroup 2) streams k-block kb's
// tiles, A_hi / A_lo [BM, BK] and W_hi / W_lo [BN, BK] (bf16, K-major, 2 BK-byte swizzled rows), into a ring of kStages
// stages, each guarded by a tx-counted full barrier and an empty barrier that every consumer warp arrives on.
// Warpgroups 0 and 1 multiply rows [64 wg, 64 wg + 64) into acc: per k16 step A_hi.W_hi (overwriting acc at the first),
// A_hi.W_lo, A_lo.W_hi, one commit per k-block, waited for before the stage is released.
template <int BM, int BN, int BK, int kStages>
struct TcRing {
    static_assert(BM == 128, "two consumer warpgroups of 64 rows");
    static constexpr uint32_t kABytes = BM * BK * 2;
    static constexpr uint32_t kBBytes = BN * BK * 2;
    static constexpr uint32_t kStageBytes = 2 * kABytes + 2 * kBBytes;
    static constexpr uint32_t kRingBytes = kStages * kStageBytes;
    static constexpr size_t kSmemBytes = kRingBytes + 1024;       // dynamic shared memory: + slack to align the ring

    uint64_t full_bar[kStages];
    uint64_t empty_bar[kStages];

    // thread 0, before the __syncthreads that precedes run()
    __device__ __forceinline__ void init() {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(smem_u32(&full_bar[s]), 1);
            mbar_init(smem_u32(&empty_bar[s]), 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }

    // every thread: a_tile(kb) is k-block kb's TcATile, W's tiles are at (kb * BK, n0).  Returns with the warps
    // converged and, in warpgroups 0 and 1, the product in acc.
    template <class ATileOf>
    __device__ __forceinline__ void run(uint32_t ring, int num_kb, int m0, ATileOf a_tile, const SplitMap& w, int n0,
                                        float (&acc)[BN / 2]) {
        const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
        if (wg == 2) {
            if (threadIdx.x == 256) {
                for (int kb = 0; kb < (TB2_GEMM_ABLATE == 2 ? 1 : num_kb); ++kb) {
                    const int s = kb % kStages;
                    const uint32_t phase = (kb / kStages) & 1;
                    mbar_wait(smem_u32(&empty_bar[s]), phase ^ 1);
                    const uint32_t bar = smem_u32(&full_bar[s]);
                    const uint32_t base = ring + s * kStageBytes;
                    mbar_expect_tx(bar, kStageBytes);
                    const TcATile a = a_tile(kb);
                    tma_load_2d(base, &a.map->hi, bar, a.col, m0);
                    tma_load_2d(base + kABytes, &a.map->lo, bar, a.col, m0);
                    tma_load_2d(base + 2 * kABytes, &w.hi, bar, kb * BK, n0);
                    tma_load_2d(base + 2 * kABytes + kBBytes, &w.lo, bar, kb * BK, n0);
                }
            }
            __syncwarp();
            return;
        }
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        const uint32_t a_off = (uint32_t)wg * 64 * 2 * BK;        // this warpgroup's 64 rows of the A tiles
        for (int kb = 0; kb < num_kb; ++kb) {
            const int s = TB2_GEMM_ABLATE == 2 ? 0 : kb % kStages;
            const uint32_t phase = TB2_GEMM_ABLATE == 2 ? 0 : (kb / kStages) & 1;
            mbar_wait(smem_u32(&full_bar[s]), phase);
            const uint32_t base = ring + s * kStageBytes;
            const uint64_t a_hi = wgmma_desc<2 * BK>(base + a_off);
            const uint64_t a_lo = wgmma_desc<2 * BK>(base + kABytes + a_off);
            const uint64_t b_hi = wgmma_desc<2 * BK>(base + 2 * kABytes);
            const uint64_t b_lo = wgmma_desc<2 * BK>(base + 2 * kABytes + kBBytes);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < (TB2_GEMM_ABLATE == 1 ? 0 : BK / 16); ++k) {
                const uint64_t adv = (uint64_t)((k * 16 * 2) >> 4);      // 32 bytes per K step
                wgmma_bf16(acc, a_hi + adv, b_hi + adv, (kb | k) != 0);
                wgmma_bf16(acc, a_hi + adv, b_lo + adv, 1u);
                wgmma_bf16(acc, a_lo + adv, b_hi + adv, 1u);
            }
            wgmma_commit();
#if TB2_GEMM_ABLATE == 4
            wgmma_wait<1>();
            if (kb > 0 && lane == 0) mbar_arrive(smem_u32(&empty_bar[(kb - 1) % kStages]));
#else
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s]));        // this warp no longer reads the stage
#endif
        }
        wgmma_wait<0>();
    }
};

}  // namespace tb2
