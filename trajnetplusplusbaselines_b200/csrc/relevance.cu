// Layer-wise relevance propagation (LRP) of a free-running LSTM forecast (tb2_lstm_relevance): how much each
// prediction of a scene's primary relies on the primary's own motion and on each neighbour, step by step.
//
// Explained quantity, per scene b and prediction t (row r = t * B + b of the pass): y = |mu| of the primary's mean
// velocity at step s_t = obs_length - 2 + t, written y = d . mu with d = mu / |mu| held fixed (y = 0 when mu is 0 or
// not finite, or the primary is absent there).  Rules (z' = z + eps sign(z), sign(0) = +1):
//   head     R_h[u] = h_u (d . Wn[0:2, u]) / y' * y
//   cell     signal-take-all (Arras et al. 2017): R_c = R_h (+ R_c_prev of the later step), R_c_prev = f c_prev / c' R_c,
//            R_g = i g / c' R_c; the gates i, f, o get nothing
//   operand  eps-rule through the g block: R_X[k] = X_k sum_u W_g[u, k] R_g[u] / z_g[u]'; the h_prev part and R_c_prev
//            continue at step s - 1
//   own      the emb part through ReLU(Linear(2 -> E - 2)) of 4 vel (one eps-rule): the sum over both components
//   grid     the pooled part through the grid embedding's ReLU(Linear) layers (one eps-rule each) to each cell value;
//            a cell's relevance (summed over its channels) goes to the neighbour that won the cell at that step
//   absent   a step where the primary is absent carries its state unchanged: relevance passes through untouched
// A ReLU unit's relevance is a_o Q_o (Q: the transposed product of the layer above), so the eps-rule below it divides
// by z' = a_o + eps where a_o > 0 and sends nothing where a_o = 0: only post-activation records are needed.
//
// Records: the training backward's, on the B primaries' rows (train.cu phases (A) and (B)): resolve_step_inputs, the
// forward's winners (pool_prepare), X = [emb | pooled | h_prev] and the grid rows (bwd_gather_kernel), the gate
// pre-activations (gate_preactivations).  Social grids rebuild the winners' latents and the embedding here.  Every
// product is the fp32 FFMA kernel (launch_gemm_ffma: one fmaf chain per output), never cuBLAS, so a row's bits do not
// depend on how many rows a call has; no atomics anywhere: reruns and per-scene calls give identical bits.
#include "common.cuh"

namespace tb2 {

int resolve_step_inputs(const tb2_layout* l, const float* observed, int obs_length, const float* truth,
                        const float* positions, int s, Workspace* ws, const float** o1, const float** o2,
                        int* phase, cudaStream_t st);

__device__ __forceinline__ float rel_sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float stab(float z, float eps) { return z + (z >= 0.f ? eps : -eps); }

// Head rule at each row's explained step: Rinit [R][H], explained [R] (= [T][B]).  One CTA of H threads per row.
__global__ void rel_head_kernel(const int* __restrict__ scene_off, const int* __restrict__ masked,
                                const float* __restrict__ states, const float* __restrict__ Wn,
                                const float* __restrict__ bn, int B, int M, int H, int obs_length, float eps,
                                float* __restrict__ Rinit, float* __restrict__ explained) {
    __shared__ float red[2][kMaxHidden];
    const int r = blockIdx.x, t = r / B, b = r - t * B, u = threadIdx.x;
    const int s = obs_length - 2 + t, m = scene_off[b];
    const float h = states[(size_t)s * 2 * M * H + (size_t)m * H + u];
    red[0][u] = Wn[u] * h;
    red[1][u] = Wn[H + u] * h;
    __syncthreads();
    for (int k = kMaxHidden / 2; k > 0; k >>= 1) {
        if (u < k && u + k < H) {
            red[0][u] += red[0][u + k];
            red[1][u] += red[1][u + k];
        }
        __syncthreads();
    }
    const float mx = red[0][0] + bn[0], my = red[1][0] + bn[1];
    const float y = sqrtf(mx * mx + my * my);
    const bool ok = !masked[(size_t)s * B + b] && y > 0.f && isfinite(y);
    float R = 0.f;
    if (ok) R = h * (mx / y * Wn[u] + my / y * Wn[H + u]) / (y + eps) * y;
    Rinit[(size_t)r * H + u] = R;
    if (u == 0) explained[r] = ok ? y : 0.f;
}

// Cell rule of step s for rows r0 + blockIdx.x (H threads).  In: RH = R_h from step s + 1 (+ Rinit at s = s_t), RC =
// R_c_prev from step s + 1.  Out: RC = R_c_prev of this step, V = R_g / z_g' (the gate-operand GEMM's input), RH = the
// total R_h (an absent primary passes it on unchanged, rel_operand_kernel).
__global__ void rel_cell_kernel(int r0, int B, int s, int obs_length, const int* __restrict__ scene_off,
                                const int* __restrict__ masked, const float* __restrict__ GP,
                                const float* __restrict__ c_prev, const float* __restrict__ Rinit, float* __restrict__ RH,
                                float* __restrict__ RC, float* __restrict__ V, int H, float eps) {
    const int r = r0 + blockIdx.x, t = r / B, b = r - t * B, u = threadIdx.x;
    const size_t i = (size_t)r * H + u;
    float rh = RH[i];
    if (s == obs_length - 2 + t) rh += Rinit[i];
    RH[i] = rh;
    if (masked[b]) {
        V[i] = 0.f;
        return;       // RC stays as it is
    }
    const float* gp = GP + (size_t)b * 4 * H;
    const float ig = rel_sigm(gp[u]), fg = rel_sigm(gp[H + u]), gg = tanhf(gp[2 * H + u]);
    const float cp = c_prev ? c_prev[(size_t)scene_off[b] * H + u] : 0.f;
    const float cs = stab(fg * cp + ig * gg, eps);
    const float rc = rh + RC[i];
    RC[i] = fg * cp / cs * rc;
    V[i] = ig * gg / cs * rc / stab(gp[2 * H + u], eps);
}

// Gate-operand rule of step s (Qin = V . W_ih_g, Qh = V . W_hh_g): RH = h_prev (.) Qh for step s - 1 (an absent primary
// keeps the total), and the own column rel[t][s][primary] = sum_c 4 vel_c sum_k We[k, c] R_emb[k] / (emb_k + eps).
__global__ void __launch_bounds__(128) rel_operand_kernel(
    int r0, int B, int s, int S, int M, const int* __restrict__ scene_off, const int* __restrict__ masked,
    const float* __restrict__ X, int K, const float* __restrict__ VEL, const float* __restrict__ Qin, int EP,
    const float* __restrict__ Qh, const float* __restrict__ We, int E, int H, float eps, float* __restrict__ RH,
    float* __restrict__ rel) {
    __shared__ float red[2][128];
    const int r = r0 + blockIdx.x, t = r / B, b = r - t * B, tid = threadIdx.x;
    if (masked[b]) return;        // the own column stays 0
    const float* x = X + (size_t)b * K;
    for (int u = tid; u < H; u += 128) RH[(size_t)r * H + u] = x[K - H + u] * Qh[(size_t)r * H + u];
    float sx = 0.f, sy = 0.f;
    for (int k = tid; k < E - 2; k += 128) {
        const float a = x[k];
        if (a > 0.f) {
            const float v = a * Qin[(size_t)r * EP + k] / (a + eps);
            sx = fmaf(We[2 * k], v, sx);
            sy = fmaf(We[2 * k + 1], v, sy);
        }
    }
    red[0][tid] = sx;
    red[1][tid] = sy;
    __syncthreads();
    for (int k = 64; k > 0; k >>= 1) {
        if (tid < k) {
            red[0][tid] += red[0][tid + k];
            red[1][tid] += red[1][tid + k];
        }
        __syncthreads();
    }
    if (tid == 0)
        rel[((size_t)t * S + s) * M + scene_off[b]] = VEL[2 * b] * red[0][0] + VEL[2 * b + 1] * red[1][0];
}

// eps-rule below a ReLU layer whose output a (record row b of each pass row r) has relevance a (.) Q:
// V = a > 0 ? a Q / (a + eps) : 0, the input of the next transposed product
__global__ void rel_relu_scale_kernel(int r0, int B, int rows, const float* __restrict__ a, int lda,
                                      const float* __restrict__ Q, int ldq, float* __restrict__ V, int ldv, int cols,
                                      float eps) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)rows * cols) return;
    const int r = r0 + (int)(idx / cols), o = (int)(idx % cols), b = r % B;
    const float av = a[(size_t)b * lda + o];
    V[(size_t)r * ldv + o] = av > 0.f ? av * Q[(size_t)r * ldq + o] / (av + eps) : 0.f;
}

// owner[b][cell] = scene-local index of the neighbour that won the cell in the primary's grid at this step (the
// forward's last-writer-wins winners, pool_prepare), -1 for an empty cell
__global__ void rel_owner_kernel(const int* __restrict__ scene_off, const int* __restrict__ win_count,
                                 const uint32_t* __restrict__ win_ent, int nm1, int cells, int* __restrict__ owner) {
    const int b = blockIdx.x, m = scene_off[b];
    int* o = owner + (size_t)b * cells;
    for (int c = threadIdx.x; c < cells; c += blockDim.x) o[c] = -1;
    __syncthreads();
    const int cnt = win_count[m];
    for (int e = threadIdx.x; e < cnt; e += blockDim.x) {      // one winner per cell: plain stores
        const uint32_t ent = win_ent[(size_t)m * nm1 + e];
        const int j = (int)(ent & 0xffff);
        o[ent >> 16] = j == 0xffff ? -1 : j;
    }
}

// Social grid of the primary of scene b at this step: G [C * cells] (channel-major, as bwd_gather_kernel writes the
// other grids) holds each winner's latent lat_j = W_enc h_j + b_enc (pool_prepare's ws.lat), and
// out = relu(b1 + W1 G), the first Linear on the winners only (Wt1: cell-major slabs of W1, d1 <= 1024).
__global__ void __launch_bounds__(256) rel_social_grid_kernel(
    const int* __restrict__ scene_off, const int* __restrict__ win_count, const uint32_t* __restrict__ win_ent,
    const float* __restrict__ lat, int nm1, int C, int cells, const float* __restrict__ Wt1,
    const float* __restrict__ base1, int d1, float* __restrict__ G, float* __restrict__ out, int ld_out) {
    __shared__ uint32_t ent_s[64];
    const int b = blockIdx.x, m = scene_off[b];
    float* g = G + (size_t)b * C * cells;
    for (int k = threadIdx.x; k < C * cells; k += blockDim.x) g[k] = 0.f;
    float acc[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int o = threadIdx.x + q * 256;
        acc[q] = o < d1 ? base1[o] : 0.f;
    }
    const int cnt = win_count[m];
    for (int e0 = 0; e0 < cnt; e0 += 64) {
        const int n = min(64, cnt - e0);
        __syncthreads();
        if (threadIdx.x < n) ent_s[threadIdx.x] = win_ent[(size_t)m * nm1 + e0 + threadIdx.x];
        __syncthreads();
        for (int idx = threadIdx.x; idx < n * C; idx += blockDim.x) {
            const uint32_t ent = ent_s[idx / C];
            const int ch = idx % C, j = (int)(ent & 0xffff);
            if (j != 0xffff) g[ch * cells + (ent >> 16)] = lat[(size_t)(m + j) * C + ch];
        }
        for (int e = 0; e < n; ++e) {
            const int cell = ent_s[e] >> 16, j = (int)(ent_s[e] & 0xffff);
            if (j == 0xffff) continue;
            for (int ch = 0; ch < C; ++ch) {
                const float v = lat[(size_t)(m + j) * C + ch];
                const float* wrow = Wt1 + ((size_t)cell * C + ch) * d1;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int o = threadIdx.x + q * 256;
                    if (o < d1) acc[q] = fmaf(wrow[o], v, acc[q]);
                }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int o = threadIdx.x + q * 256;
        if (o < d1) out[(size_t)b * ld_out + o] = fmaxf(acc[q], 0.f);
    }
}

// Cell -> winner reduction of step s: one warp per row.  R_cell = sum_ch G[ch, cell] Q1[ch, cell] (the grid rule's
// last eps-rule), then each neighbour j (one lane each) adds the cells it won in ascending order:
// rel[t][s][row0 + j].  No atomics.
__global__ void __launch_bounds__(32) rel_neighbour_kernel(int r0, int B, int s, int S, int M,
                                                           const int* __restrict__ scene_off,
                                                           const float* __restrict__ G, const float* __restrict__ Q1,
                                                           const int* __restrict__ owner, int C, int cells,
                                                           float* __restrict__ rel) {
    extern __shared__ float cell_s[];          // [cells] relevance, then [cells] owner
    int* own_s = reinterpret_cast<int*>(cell_s + cells);
    const int r = r0 + blockIdx.x, t = r / B, b = r - t * B, lane = threadIdx.x;
    const int row0 = scene_off[b], n_s = scene_off[b + 1] - row0;
    const size_t CG = (size_t)C * cells;
    const float* g = G + (size_t)b * CG;
    const float* q = Q1 + (size_t)r * CG;
    for (int cell = lane; cell < cells; cell += 32) {
        float sum = 0.f;
        for (int ch = 0; ch < C; ++ch) sum += g[(size_t)ch * cells + cell] * q[(size_t)ch * cells + cell];
        cell_s[cell] = sum;
        own_s[cell] = owner[(size_t)b * cells + cell];
    }
    __syncwarp();
    float* out = rel + ((size_t)t * S + s) * M + row0;
    for (int j = 1 + lane; j < n_s; j += 32) {
        float acc = 0.f;
        for (int cell = 0; cell < cells; ++cell)
            if (own_s[cell] == j) acc += cell_s[cell];
        out[j] = acc;
    }
}

// Workspace of tb2_lstm_relevance: the forward's Workspace (pool_prepare, resolve_step_inputs), then the records of the
// B primaries over S steps and the pass's per-row buffers (R = T * B rows); a null base only counts the bytes.
struct RelBuffers {
    Workspace ws;
    float *X, *GP, *G, *VEL, *H1, *PZ, *ZH;        // records [S][B][..]; PZ [M, P], ZH [M, H] zeros (social)
    int *masked, *owner;                           // [S][B], [S][B][cells]
    float *Rinit, *RH, *RC, *V, *Qin, *Qh, *VT, *Q2, *V1, *Q1;
};

static size_t carve_relevance(const tb2_lstm* m, const tb2_layout* l, int T, int obs_length, void* base,
                              RelBuffers* o) {
    const size_t B = (size_t)l->B, M = (size_t)l->M, S = (size_t)(obs_length - 2 + T), R = (size_t)T * B;
    const size_t K = (size_t)m->K_gate, H = (size_t)m->H, P = (size_t)m->P, EP = (size_t)(m->E + m->P);
    const bool pooled = m->cfg.pool_type != TB2_POOL_NONE, social = m->cfg.pool_type == TB2_POOL_SOCIAL;
    const size_t CG = pooled ? (size_t)m->C * m->cells : 0, cells = pooled ? (size_t)m->cells : 0;
    const size_t d1 = social && m->n_mlp == 2 ? (size_t)m->mlp_dims[1] : 0;
    RelBuffers tmp;
    RelBuffers* b = o ? o : &tmp;
    size_t off = (carve_workspace(m, l, base, &b->ws) + 255) & ~(size_t)255;
    auto take = [&](size_t n) {
        float* p = base ? reinterpret_cast<float*>(static_cast<char*>(base) + off) : nullptr;
        off += ((n > 0 ? n : 1) * sizeof(float) + 255) & ~(size_t)255;
        return p;
    };
    b->X = take(S * B * K);
    b->GP = take(S * B * 4 * H);
    b->G = take(S * B * CG);
    b->VEL = take(S * B * 2);
    b->H1 = take(S * B * d1);
    b->PZ = take(social ? M * P : 0);
    b->ZH = take(social ? M * H : 0);
    b->masked = reinterpret_cast<int*>(take(S * B));
    b->owner = reinterpret_cast<int*>(take(S * B * cells));
    b->Rinit = take(R * H);
    b->RH = take(R * H);
    b->RC = take(R * H);
    b->V = take(R * H);
    b->Qin = take(R * EP);
    b->Qh = take(R * H);
    b->VT = take(R * P);
    b->Q2 = take(R * d1);
    b->V1 = take(R * d1);
    b->Q1 = take(R * CG);
    return off;
}

// The configurations the pass is built for: refusal message, or null
static const char* relevance_unsupported(const tb2_lstm* m) {
    if (m->G > 0) return "relevance of a goal-conditioned model (goal_dim > 0) is not built";
    switch (m->cfg.pool_type) {
        case TB2_POOL_NONE: return nullptr;
        case TB2_POOL_SOCIAL:
            if (!social_trainable(m)) return "social relevance supports one_layer / two_layer embeddings with constant = 0 and pool_to_input";
            if (m->mlp_dims[1] > 1024) return "social relevance supports grid embedding widths up to 1024";
            return nullptr;
        case TB2_POOL_OCCUPANCY:
        case TB2_POOL_DIRECTIONAL:
            if (m->n_mlp != 1 || !m->cfg.pool_to_input || m->cfg.constant != 0.f || m->P > 1024 || m->C > 2)
                return "grid relevance supports one_layer embeddings up to 1024 wide with constant = 0 and pool_to_input";
            return nullptr;
        default: return "relevance of a non-grid or external interaction module is not built";
    }
}

static int relevance(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w, const float* observed,
                     int obs_length, int n_decode, const float* positions, const float* states, float eps,
                     float* rel, float* explained, void* workspace, cudaStream_t st) {
    const int T = n_decode + 1, S_enc = obs_length - 1, S = S_enc + n_decode;
    const int B = l->B, Mi = l->M, R = T * B, K = m->K_gate, E = m->E, P = m->P, EP = E + P, H = m->H;
    const size_t M = (size_t)Mi;
    const bool pooled = m->cfg.pool_type != TB2_POOL_NONE, social = m->cfg.pool_type == TB2_POOL_SOCIAL;
    const bool two = social && m->n_mlp == 2;
    const int C = m->C, cells = m->cells, CG = pooled ? C * cells : 0, d1 = m->mlp_dims[1];
    const int nm1 = l->n_max > 1 ? l->n_max - 1 : 1;
    RelBuffers b;
    carve_relevance(m, l, T, obs_length, workspace, &b);
    int rc;
    if (social) {
        TB2_CHECK_CUDA(cudaMemsetAsync(b.PZ, 0, M * P * sizeof(float), st));
        TB2_CHECK_CUDA(cudaMemsetAsync(b.ZH, 0, M * H * sizeof(float), st));
    }
    // (A) records of the primaries (rows = scene_off[0 .. B)): winners, X = [emb | pooled | h_prev], grid rows
    for (int s = 0; s < S; ++s) {
        const float *o1, *o2;
        int phase;
        if ((rc = resolve_step_inputs(l, observed, obs_length, nullptr, positions, s, &b.ws, &o1, &o2, &phase, st)))
            return rc;
        const float* h_prev = s > 0 ? states + (size_t)(s - 1) * 2 * M * H : (social ? b.ZH : nullptr);
        if (pooled) {
            if ((rc = launch_pool_prepare(m, l, h_prev, o1, o2, 1, 0, 0, &b.ws, st))) return rc;
            {
                KernelTimer kt("rel_owner", st);
                rel_owner_kernel<<<B, 256, 0, st>>>(l->scene_off, b.ws.win_count, b.ws.win_ent, nm1, cells,
                                                    b.owner + (size_t)s * B * cells);
            }
            TB2_LAUNCH_CHECK();
        }
        float* Xs = b.X + (size_t)s * B * K;
        // social: the gather copies zeros into the pooled columns; the winners' latents give them below
        if ((rc = launch_bwd_gather(m, l->scene_off, B, o1, o2, h_prev, pooled && !social ? &b.ws : nullptr,
                                    social ? b.PZ : nullptr, nm1, Xs, pooled && !social ? b.G + (size_t)s * B * CG : nullptr,
                                    b.VEL + (size_t)s * B * 2, b.masked + (size_t)s * B, st)))
            return rc;
        if (social) {
            KernelTimer kt("rel_social_grid", st);
            rel_social_grid_kernel<<<B, 256, 0, st>>>(l->scene_off, b.ws.win_count, b.ws.win_ent, b.ws.lat, nm1, C, cells,
                                                      m->Wt1, m->base1, d1, b.G + (size_t)s * B * CG,
                                                      two ? b.H1 + (size_t)s * B * d1 : Xs + E, two ? d1 : K);
            TB2_LAUNCH_CHECK();
        }
    }
    // two_layer: pooled = relu(W2 hidden1 + b2) of every (step, primary) record, into X's pooled columns
    if (two && (rc = launch_gemm_ffma(b.H1, d1, m->WT[1], P, b.X + E, K, S * B, P, d1, m->bl[1], 1, "rel_gemm", st)))
        return rc;
    if ((rc = launch_gate_preactivations(m, b.X, b.GP, B, S, S_enc, st))) return rc;
    {
        KernelTimer kt("rel_head", st);
        rel_head_kernel<<<R, H, 0, st>>>(l->scene_off, b.masked, states, m->Wn, m->bn, B, Mi, H, obs_length, eps, b.Rinit,
                                         explained);
    }
    TB2_LAUNCH_CHECK();
    TB2_CHECK_CUDA(cudaMemsetAsync(b.RH, 0, (size_t)R * H * sizeof(float), st));
    TB2_CHECK_CUDA(cudaMemsetAsync(b.RC, 0, (size_t)R * H * sizeof(float), st));
    TB2_CHECK_CUDA(cudaMemsetAsync(rel, 0, (size_t)T * S * M * sizeof(float), st));
    // (C) one chain per row from its explained step down to step 0; rows with s_t >= s (t >= s - obs_length + 2) are the
    // suffix [r0, R) of the row order
    for (int s = S - 1; s >= 0; --s) {
        const int t0 = s - (obs_length - 2);
        const int r0 = (t0 > 0 ? t0 : 0) * B, nr = R - r0;
        const bool enc = s < S_enc;
        const float* Wih = enc ? w->encoder_weight_ih : w->decoder_weight_ih;
        const float* Whh = enc ? w->encoder_weight_hh : w->decoder_weight_hh;
        const float* c_prev = s > 0 ? states + ((size_t)(s - 1) * 2 + 1) * M * H : nullptr;
        const int* msk = b.masked + (size_t)s * B;
        const float* Xs = b.X + (size_t)s * B * K;
        {
            KernelTimer kt("rel_cell", st);
            rel_cell_kernel<<<nr, H, 0, st>>>(r0, B, s, obs_length, l->scene_off, msk, b.GP + (size_t)s * B * 4 * H,
                                              c_prev, b.Rinit, b.RH, b.RC, b.V, H, eps);
        }
        TB2_LAUNCH_CHECK();
        // the g block of W_ih / W_hh (rows 2H .. 3H of the torch layout) is the [K = H, N] operand as it stands
        if ((rc = launch_gemm_ffma(b.V + (size_t)r0 * H, H, Wih + (size_t)2 * H * EP, EP, b.Qin + (size_t)r0 * EP, EP, nr,
                                   EP, H, nullptr, 0, "rel_gemm", st)))
            return rc;
        if ((rc = launch_gemm_ffma(b.V + (size_t)r0 * H, H, Whh + (size_t)2 * H * H, H, b.Qh + (size_t)r0 * H, H, nr, H, H,
                                   nullptr, 0, "rel_gemm", st)))
            return rc;
        {
            KernelTimer kt("rel_operand", st);
            rel_operand_kernel<<<nr, 128, 0, st>>>(r0, B, s, S, Mi, l->scene_off, msk, Xs, K, b.VEL + (size_t)s * B * 2,
                                                   b.Qin, EP, b.Qh, m->We, E, H, eps, b.RH, rel);
        }
        TB2_LAUNCH_CHECK();
        if (!pooled) continue;
        auto relu_scale = [&](const float* a, int lda, const float* Q, int ldq, float* V, int cols) {
            KernelTimer kt("rel_relu_scale", st);
            rel_relu_scale_kernel<<<(unsigned)(((size_t)nr * cols + 255) / 256), 256, 0, st>>>(r0, B, nr, a, lda, Q, ldq,
                                                                                             V, cols, cols, eps);
        };
        relu_scale(Xs + E, K, b.Qin + E, EP, b.VT, P);      // the pooled vector (last ReLU layer of the embedding)
        TB2_LAUNCH_CHECK();
        const float* V1 = b.VT;
        int width = P;
        if (two) {
            if ((rc = launch_gemm_ffma(b.VT + (size_t)r0 * P, P, w->pool_embedding_weight[1], d1, b.Q2 + (size_t)r0 * d1, d1,
                                       nr, d1, P, nullptr, 0, "rel_gemm", st)))
                return rc;
            relu_scale(b.H1 + (size_t)s * B * d1, d1, b.Q2, d1, b.V1, d1);
            TB2_LAUNCH_CHECK();
            V1 = b.V1;
            width = d1;
        }
        if ((rc = launch_gemm_ffma(V1 + (size_t)r0 * width, width, w->pool_embedding_weight[0], CG, b.Q1 + (size_t)r0 * CG,
                                   CG, nr, CG, width, nullptr, 0, "rel_gemm", st)))
            return rc;
        {
            KernelTimer kt("rel_neighbours", st);
            rel_neighbour_kernel<<<nr, 32, (size_t)cells * 2 * sizeof(float), st>>>(
                r0, B, s, S, Mi, l->scene_off, b.G + (size_t)s * B * CG, b.Q1, b.owner + (size_t)s * B * cells, C, cells,
                rel);
        }
        TB2_LAUNCH_CHECK();
    }
    return TB2_OK;
}

}  // namespace tb2

using namespace tb2;

extern "C" {

size_t tb2_lstm_relevance_workspace_bytes(const tb2_lstm* m, const tb2_layout* l, int32_t n_predict,
                                          int32_t obs_length) {
    if (!m || !l || n_predict < 1 || obs_length < 2 || relevance_unsupported(m)) return 0;
    return carve_relevance(m, l, n_predict, obs_length, nullptr, nullptr);
}

int tb2_lstm_relevance(const tb2_lstm* m, const tb2_layout* l, const tb2_lstm_weights* w, const float* observed,
                       int32_t obs_length, int32_t n_decode, const float* positions, const float* states, float eps,
                       float* relevance_out, float* explained_out, void* workspace, size_t workspace_bytes,
                       void* stream) {
    TB2_REQUIRE(m && l && w, "null handle");
    TB2_REQUIRE(m->weights_set, "tb2_lstm_set_weights has not been called");
    TB2_REQUIRE(observed && positions && states && relevance_out && explained_out, "null argument");
    TB2_REQUIRE(obs_length >= 2 && n_decode >= 0, "need obs_length >= 2 and n_decode >= 0");
    TB2_REQUIRE(eps >= 0.f && isfinite(eps), "eps must be finite and >= 0");
    if (const char* why = relevance_unsupported(m)) {
        set_error(why);
        return TB2_ERR_UNSUPPORTED;
    }
    TB2_REQUIRE(hidden_dim_supported(m->H), kHiddenDimMessage);
    TB2_REQUIRE(m->cfg.pool_type == TB2_POOL_NONE || (size_t)m->cells * 2 * sizeof(float) <= 48 * 1024,
                "grid too large for the relevance reduction");
    TB2_REQUIRE(workspace && workspace_bytes >= carve_relevance(m, l, n_decode + 1, obs_length, nullptr, nullptr),
                "workspace too small (tb2_lstm_relevance_workspace_bytes)");
    TB2_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    if (l->B == 0) return TB2_OK;
    return relevance(m, l, w, observed, obs_length, n_decode, positions, states, eps, relevance_out, explained_out,
                     workspace, (cudaStream_t)stream);
}

}  // extern "C"
