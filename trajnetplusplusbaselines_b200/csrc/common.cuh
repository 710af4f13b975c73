// Shared host/device declarations of libtrajnet_b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include <string>
#include <vector>

#include "trajnet_b200.h"

namespace tb2 {

void set_error(const std::string& msg);
extern std::atomic<uint64_t> g_launch_count;

#define TB2_CHECK_CUDA(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            ::tb2::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));         \
            return TB2_ERR_CUDA;                                                          \
        }                                                                                 \
    } while (0)

#define TB2_REQUIRE(cond, msg)                                                            \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            ::tb2::set_error(std::string("invalid argument: ") + (msg));                  \
            return TB2_ERR_INVALID;                                                       \
        }                                                                                 \
    } while (0)

#define TB2_LAUNCH_CHECK()                                                                \
    do {                                                                                  \
        ::tb2::g_launch_count.fetch_add(1, std::memory_order_relaxed);                    \
        TB2_CHECK_CUDA(cudaGetLastError());                                               \
    } while (0)

// Programmatic dependent launch: the kernels of a recurrence step are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so the next kernel's CTAs become resident
// and run their prologue (barrier init, tensor-map prefetch) while the previous
// kernel drains.  Every thread executes grid_dep_wait() before its first access to global memory
// (it returns once the preceding grid has completed and its writes are visible), then
// grid_dep_launch() lets the following kernel start its own prologue.
#ifdef __CUDACC__
__device__ __forceinline__ void grid_dep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_dep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// The operand format of every 3-pass bf16 tensor-core product: an fp32 v is stored as hi = rn(v), lo = rn(v - hi),
// and A.W ~= A_hi.W_hi + A_hi.W_lo + A_lo.W_hi (the dropped terms ~ 2^-17 relative)
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi = h;
    lo = __float2bfloat16_rn(v - __bfloat162float(h));
}
// two adjacent values as packed bf16x2 words (v.x in the low half)
__device__ __forceinline__ void split_bf16x2(float2 v, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(v.x, v.y);
    const __nv_bfloat162 l = __floats2bfloat162_rn(v.x - __low2float(h), v.y - __high2float(h));
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = *reinterpret_cast<const uint32_t*>(&l);
}

// Warp-level D += A . B, m16n8k16, bf16 inputs, fp32 accumulation (the 3-pass split kernels of pool.cu and train.cu)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// launch_pdl with clusters of cluster_x CTAs along x, chosen at launch (the kernel carries no __cluster_dims__)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                      unsigned cluster_x, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = cluster_x;
    attr[1].val.clusterDim.y = 1;
    attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 2;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) applies to the CURRENT device: the size a launch
// site has configured is remembered per device, so a second model on another GPU of the same
// process configures its own copy of the kernel.
struct DynSmemConfig {
    size_t bytes[64];      // zero-initialised (function-local static)
    template <typename K>
    cudaError_t ensure(K kernel, size_t smem, size_t preset = 0) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        size_t& have = bytes[dev & 63];
        if (have < preset) have = preset;          // e.g. the 48 KB every kernel may use without opting in
        if (smem <= have) return cudaSuccess;
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) have = smem;
        return e;
    }
};

// Optional per-kernel timing (tb2_profile_begin / tb2_profile_end): CUDA events recorded on the
// launching stream around every kernel of the library.  Off by default (zero overhead).
struct KernelTimer {
    KernelTimer(const char* name, cudaStream_t st);
    ~KernelTimer();
    int slot;
    cudaStream_t st;
};

constexpr int kMaxMlpLayers = 3;
// LSTM widths the gate and backward kernels are built for: 32, 64, ..., 256
constexpr int kMaxHidden = 256;
inline bool hidden_dim_supported(int H) { return H >= 32 && H <= kMaxHidden && H % 32 == 0; }
constexpr const char* kHiddenDimMessage = "hidden_dim must be a multiple of 32 from 32 to 256 (32, 64, 96, ..., 256)";
constexpr int kGateBK = 16;        // K-chunk of the gate GEMM; weight rows are padded to it
// Zero columns after the last cell of sparse_layer1_mma's weight image: the kernel loads whole 256-column chunks
// without bounds checks, and the columns past d1 (never written out) of the last cell fall into this tail.
constexpr int kLayer1MmaTailCols = 256;
// Refusal of the fused calls for a model whose interaction module the caller runs (TB2_POOL_EXTERNAL)
constexpr const char* kExternalPoolMessage =
    "an external interaction module (TB2_POOL_EXTERNAL) runs step by step: tb2_pool_inputs_padded, the module, "
    "tb2_lstm_step_forward with pooled_padded_dev, and tb2_lstm_step_backward for training";

}  // namespace tb2

// Opaque handle bodies ---------------------------------------------------------------------
struct tb2_lstm {
    tb2_lstm_config cfg = {};
    int H = 0, E = 0, C = 0, cells = 0, n_mlp = 0;
    int G = 0;             // goal embedding width (cfg.goal_dim; 0: no goal input)
    int P = 0;             // pooled width fed to the LSTM input (0 if none / pool_to_input == 0)
    int pool_out = 0;      // width of the pool output (grid width when n_mlp == 0)
    int mlp_dims[tb2::kMaxMlpLayers + 1] = {};  // [grid_dim, d1, ..]
    int K_gate = 0, K_gate_pad = 0;
    bool weights_set = false;
    bool tc_disabled = false;   // TB2_DISABLE_TC=1 at creation: every kernel choice takes the fp32 FFMA version
    // device buffers (owned)
    float* We = nullptr;        // [E-2, 2]
    float* be = nullptr;        // [E-2]
    float* Wgl = nullptr;       // [G-2, 2] goal embedding (G > 0)
    float* bgl = nullptr;       // [G-2]
    float* WgT[2] = {};         // [K_gate_pad, 4H]  rows: emb | goal | pooled | h
    float* bg[2] = {};          // [4H] = b_ih + b_hh
    float* Wn = nullptr;        // [5, H]
    float* bn = nullptr;        // [5]
    float* WencT = nullptr;     // [H, C]
    float* benc = nullptr;      // [C]
    float* Wt1 = nullptr;       // [cells, C, d1]  cell-major slabs of pool.embedding.0.weight
    float* base1 = nullptr;     // [d1] = b1 + constant * rowsum(W1)
    void* Wt1_hi = nullptr;     // social, C == 16: bf16 [cells, d1, 16] (hi, lo) slabs for sparse_layer1_mma
    void* Wt1_lo = nullptr;
    float* WT[tb2::kMaxMlpLayers] = {};   // layers >= 2: [K, N] transposed
    float* bl[tb2::kMaxMlpLayers] = {};   // biases of layers >= 2
    void* W_hi[tb2::kMaxMlpLayers] = {};  // [1] only (second Linear): bf16 [N, K] (hi, lo) split for the wgmma path (null: FFMA path)
    void* W_lo[tb2::kMaxMlpLayers] = {};
    // tb2_lstm_forward_steps with host outputs: one event per recurrence step, created on first use (hence mutable:
    // the call takes a const model)
    mutable std::vector<cudaEvent_t> step_events;
    // HiddenStateMLPPooling (TB2_POOL_HIDDEN_MLP)
    float *mp_Ws = nullptr, *mp_bs = nullptr, *mp_Wv = nullptr, *mp_bv = nullptr, *mp_WhT = nullptr, *mp_bh = nullptr,
          *mp_WoT = nullptr, *mp_bo = nullptr;
    // AttentionMLPPooling (TB2_POOL_ATTN_MLP): in-projection . wq / wk / wv combined, q and v transposed [E in][E out],
    // k [E out][E in]; biases, out-projection transposed
    float *at_AqT = nullptr, *at_Ak = nullptr, *at_AvT = nullptr, *at_bqkv = nullptr, *at_WoT = nullptr, *at_bo = nullptr;
    // NearestNeighborLSTM (TB2_POOL_NN_LSTM): interaction-encoder LSTMCell, weights transposed [in][4 Hp], fused bias
    float *pl_WihT = nullptr, *pl_WhhT = nullptr, *pl_b = nullptr;
    void* Wg_hi[2] = {};        // gate weights [4H (rank, gate, unit), K_gate] bf16 split (null: FFMA gates)
    void* Wg_lo[2] = {};
    std::vector<void*> owned;
};

struct tb2_layout {
    int B, M, n_max;
    int pad_to_max = 1;    // 1: scenes padded to the batch maximum like the reference's batched call (padded
                           // slots clobber grid cell 0); 0: every scene as if it were called on its own
    std::vector<int> scene_off_host;
    int* scene_off;        // [B+1] device
    int* row_scene;        // [M]   device
    // scene groups for the sparse grid-MLP kernel: consecutive scenes, <= cap rows each
    int group_cap[2];
    int num_groups[2];
    int* group_off[2];     // [G+1] scene indices, device
    std::vector<void*> owned;
};

namespace tb2 {

struct Workspace {
    float* obs1;           // [M,2] resolved step inputs
    float* obs2;           // [M,2]
    float* lat;            // [M,C]
    int* win_count;        // [M]
    uint32_t* win_ent;     // [M, nm1]  cell << 16 | scene-local j
    float* win_val;        // [M, nm1, 2]
    int* pair_cell;        // [M, nm1]
    uint8_t* pair_flag;    // [M, nm1]
    float* act[2];         // ping-pong MLP activations [M, max width]
    float* act2;           // third scratch (three_layer with a tensor-core second layer)
    float* pooled;         // [M, pool_out]
    void* emb_hi;          // [M, 64 + G] bf16 split operands of the tensor-core gate kernel ([emb | goal_emb]; E == 64 there)
    void* emb_lo;
    void* pool_hi;         // [M, P]
    void* pool_lo;
    void* hs_hi[2];        // [M, H] ping-pong split of the hidden state
    void* hs_lo[2];
    size_t bytes;
    int write_pairs;       // pool_prepare also exports the pair tables (training forward with a cache)
    float* pool_feat;      // [M, out_dim] neighbour features of NearestNeighborLSTM (null otherwise)
    float* pool_h;         // [M, Hp] state of its interaction-encoder LSTM, kept over the steps of a sequence
    float* pool_c;
    float* scene_sum;      // [B, 4] TrajectronPooling: sum of (pos, vel) over the visible tracks of every scene
};

// How a forward step hands on hidden1 (the grid embedding's first Linear output, read by the second Linear) and the
// pooled vector (read by the gate kernel): as a bf16 (hi, lo) pair only where the producing kernel writes the pair
// itself, as fp32 wherever an fp32 tensor is made (also when that fp32 tensor is split afterwards).  hidden1 is a pair
// for the wgmma second Linear; the pooled vector is a pair when the tensor-core gates read it from a last layer that
// writes the split (the first Linear, or the wgmma second Linear).  The training cache keeps both in this format.
struct PoolFormats {
    bool h1_pair;
    bool pooled_pair;
};
inline PoolFormats pool_formats(const tb2_lstm* m) {
    const bool tc2 = m->n_mlp >= 2 && m->W_hi[1] != nullptr;
    return {tc2, m->Wg_hi[0] != nullptr && (m->n_mlp == 1 || (m->n_mlp == 2 && tc2))};
}

// The social models the training backward supports; exactly these keep a training cache
inline bool social_trainable(const tb2_lstm* m) {
    return m->cfg.pool_type == TB2_POOL_SOCIAL && m->n_mlp >= 1 && m->n_mlp <= 2 && m->cfg.pool_to_input &&
           m->cfg.constant == 0.f && m->G == 0;
}

// Per-step forward quantities the training forward (tb2_lstm_forward_steps with cache_dev) keeps for the social backward,
// which reads its grid-embedding records from here only.  Step s of hidden1 / the pooled vector is a slot of
// h1_step / pooled_step bytes at h1 / pooled + s * step: fp32 [M][n], or bf16 hi [M][n] followed by lo [M][n] at
// step / 2 (pool_formats).  Every slot and half is 256-byte aligned, like the workspace buffers it stands in for.
struct TrainCache {
    float* lat;            // [S][M][C]
    int* win_count;        // [S][M]
    uint32_t* win_ent;     // [S][M][nm1]
    int* pair_cell;        // [S][M][nm1]
    uint8_t* pair_flag;    // [S][M * nm1]
    char* h1;              // two_layer: [S] slots of [M][d1]; null otherwise
    char* pooled;          // [S] slots of [M][P]
    size_t h1_step, pooled_step;
};
// 0 for models without a cache (all but social_trainable ones)
size_t carve_train_cache(const tb2_lstm* m, const tb2_layout* l, size_t S, void* base, TrainCache* out);
size_t carve_workspace(const tb2_lstm* m, const tb2_layout* l, void* base, Workspace* ws);

// kernel launchers (all asynchronous on `st`)
int launch_resolve_obs(const tb2_layout* l, const float* base, const float* pred, float* out,
                       cudaStream_t st);
int launch_pool_prepare(const tb2_lstm* m, const tb2_layout* l, const float* hidden,
                        const float* obs1, const float* obs2, int skip_masked, int write_pairs,
                        int write_emb, Workspace* ws, cudaStream_t st, const float* goals = nullptr);
// pooled_out fp32 and/or (pool_hi, pool_lo) bf16 split (either may be null, not both)
int launch_pool_mlp(const tb2_lstm* m, const tb2_layout* l, Workspace* ws, float* pooled_out,
                    void* pool_hi, void* pool_lo, cudaStream_t st);
// goals [M, 2]: null unless m->G > 0
int launch_gates(const tb2_lstm* m, const tb2_layout* l, int phase, const float* obs1,
                 const float* obs2, const float* goals, const float* pooled, const float* h_in, const float* c_in,
                 float* h_out, float* c_out, float* normal_out, float* pos_out, cudaStream_t st);
int launch_repack(tb2_lstm* m, const tb2_lstm_weights* w, cudaStream_t st);
int launch_repack_layer1_mma(const float* W1, void* hi, void* lo, int OUT, int cells, cudaStream_t st);
int launch_hidden_mlp_pool(const tb2_lstm* m, const tb2_layout* l, const float* hidden, const float* obs1,
                           const float* obs2, float* out, cudaStream_t st);
int launch_attn_mlp_pool(const tb2_lstm* m, const tb2_layout* l, const float* hidden, const float* obs1, const float* obs2,
                         float* out, cudaStream_t st);
int launch_trajectron_feat(const tb2_lstm* m, const tb2_layout* l, const float* obs1, const float* obs2, float* scene_sum,
                           float* feat, cudaStream_t st);
int launch_pool_lstm_cell(const tb2_lstm* m, const tb2_layout* l, const float* feat, float* h, float* c, float* out,
                          cudaStream_t st);
int launch_nn_mlp_pool(const tb2_lstm* m, const tb2_layout* l, const float* obs1, const float* obs2, float* out,
                       cudaStream_t st);
// C = act(A . B + bias), B [K, N] row-major, on the fp32 FFMA kernel (never cuBLAS); act = ReLU when relu != 0
int launch_gemm_ffma(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K,
                     const float* bias, int relu, const char* name, cudaStream_t st);
bool dense_tc_supported(int K, int N);
int launch_dense_tc(const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo, const float* bias,
                    float* Y, void* Y_hi, void* Y_lo, int M, int K, int N, int relu, cudaStream_t st);
bool gates_tc_supported(const tb2_lstm* m);
int launch_repack_gates_tc(const float* w_ih, const float* w_hh, void* hi, void* lo, int in_dim, int H, cudaStream_t st);
int launch_embed_split(const tb2_lstm* m, int M, const float* obs1, const float* obs2, const float* goals, void* hi, void* lo,
                       cudaStream_t st);
int launch_gates_tc(const tb2_lstm* m, const tb2_layout* l, int phase, const float* obs1, const float* obs2,
                    const void* emb_hi, const void* emb_lo, const void* pool_hi, const void* pool_lo,
                    const void* hs_in_hi, const void* hs_in_lo, void* hs_out_hi, void* hs_out_lo,
                    const float* h_in, const float* c_in, float* h_out, float* c_out, float* normal_out,
                    float* pos_out, cudaStream_t st);
// TMA maps of a bf16 (hi, lo) split operand, row-major [rows, cols], box [box_rows, box_cols]; box_cols = 64 (128-byte
// swizzle) or 32 (64-byte swizzle)
struct SplitMap {
    CUtensorMap hi, lo;
};
int make_split_map(SplitMap* map, const void* hi, const void* lo, int rows, int cols, int box_rows, int box_cols);
// fp32 [rows, cols] (leading dimension ld_src) -> bf16 (hi, lo) of leading dimension ld_dst, on at most max_blocks CTAs
int launch_split_bf16_rows(const float* src, size_t ld_src, size_t rows, size_t cols, void* hi, void* lo, size_t ld_dst,
                           unsigned max_blocks, cudaStream_t st);
// flat array of n floats
int launch_split_bf16(const float* src, void* hi, void* lo, size_t n, cudaStream_t st);
// pos [rows, 2] += the offset of the bivariate normal normals [rows, 5] at the standard normal pairs eps [rows, 2]
int launch_sample_positions(const float* normals, float* pos, const float* eps, int rows, cudaStream_t st);
// TB2_POOL_EXTERNAL: the caller's pooled_pad [B * n_max, pool_out] row of every present track (0 for absent ones,
// + base when given) as fp32 `out` and / or the bf16 (hi, lo) split
int launch_external_pooled(const tb2_lstm* m, const tb2_layout* l, const float* obs1, const float* obs2,
                           const float* pooled_pad, const float* base, float* out, void* hi, void* lo, cudaStream_t st);
// d pooled_pad [B * n_max, P] from src[m, col .. col + P) of the present tracks; d_h_in = pass + dh_rec on the M rows
int launch_external_step_grads(const tb2_layout* l, const int* masked, const float* src, int ld_src, int col, int P,
                               const float* pass, const float* dh_rec, int H, float* d_pooled_pad, float* d_h_in,
                               cudaStream_t st);
int launch_grid_indices_copy(const tb2_layout* l, const Workspace* ws, int32_t* cell_out,
                             uint8_t* flag_out, cudaStream_t st);

}  // namespace tb2
