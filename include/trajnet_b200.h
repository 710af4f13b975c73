/*
 * trajnet_b200.h -- C ABI of the H100-native TrajNet++ hot path (libtrajnet_b200.so).
 *
 * The reference (vita-epfl/trajnetplusplusbaselines) is pure Python and has no FFI; this
 * header is the boundary a maintainer binds with ctypes (see INTEGRATION.md).  Every entry
 * point names the reference interface it replaces (paths relative to
 * /root/reference/trajnetbaselines/).
 *
 * Conventions
 *   - plain C: pointers + sizes, no C++/torch types.  Return 0 on success, < 0 on error;
 *     tb2_last_error() returns a thread-local message.  No exceptions cross the ABI.
 *   - Buffers named *_dev are CALLER-OWNED device pointers (fp32 unless noted), borrowed for
 *     the call.  The library allocates device memory only inside the opaque handles
 *     (repacked weights, scene layout) created/destroyed explicitly.
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it (no hidden
 *     synchronisation) unless documented otherwise.
 *   - There is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef TRAJNET_B200_H
#define TRAJNET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB2_OK 0
#define TB2_ERR_INVALID (-1)      /* bad argument / unsupported configuration */
#define TB2_ERR_CUDA (-2)         /* CUDA runtime error (message holds cudaGetErrorString) */
#define TB2_ERR_UNSUPPORTED (-3)  /* valid in the reference, not built here (fails loudly) */

#define TB2_POOL_NONE 0           /* --type vanilla */
#define TB2_POOL_OCCUPANCY 1      /* GridBasedPooling(type_='occupancy')   gridbased_pooling.py:112-116 */
#define TB2_POOL_DIRECTIONAL 2    /* GridBasedPooling(type_='directional') gridbased_pooling.py:118-143 */
#define TB2_POOL_SOCIAL 3         /* GridBasedPooling(type_='social')      gridbased_pooling.py:145-170 */
#define TB2_POOL_HIDDEN_MLP 4     /* HiddenStateMLPPooling (--type hiddenstatemlp) non_gridbased_pooling.py:150-239 */
#define TB2_POOL_NN_MLP 5         /* NearestNeighborMLP (--type nn) non_gridbased_pooling.py:64-147: `n` = neighbours kept,
                                   * mlp_dim_spatial = width of one neighbour's embedding (out_dim / n), mlp_dim_vel != 0 <=>
                                   * no_vel == False (inputs [rel pos | rel vel]); weights pool_spatial_weight
                                   * [out_dim / n, 2 or 4] / pool_spatial_bias = pool.embedding.0.{weight, bias} */

#define TB2_POOL_ATTN_MLP 6       /* AttentionMLPPooling (--type attentionmlp) non_gridbased_pooling.py:242-351: the
                                   * embeddings of TB2_POOL_HIDDEN_MLP (fill value attn_fill instead of -100, 0 for the
                                   * hidden part), wq / wk / wv, a one-head torch.nn.MultiheadAttention, out_projection */

#define TB2_POOL_NN_LSTM 7        /* NearestNeighborLSTM (--type nn_lstm) non_gridbased_pooling.py:354-451: the features of
                                   * TB2_POOL_NN_MLP (always with velocities) drive a per-track LSTMCell (mlp_dim_hidden =
                                   * its hidden_dim) whose state lives in the caller's workspace over the steps of a
                                   * sequence; interaction vector = hidden2pool(h') */

#define TB2_POOL_TRAJECTRON 8     /* TrajectronPooling (--type traj_pool) non_gridbased_pooling.py:454-537: every visible track
                                   * embeds [own (pos, vel) | sum over the other visible tracks] with pool_spatial_weight
                                   * [out_dim, 8]; the sum runs over the whole batch in the padded (trainer) layout and over
                                   * the scene in the per-scene layout; then the LSTMCell / hidden2pool of TB2_POOL_NN_LSTM */

#define TB2_POOL_EXTERNAL 16      /* any other interaction module (a torch.nn.Module with the reference's pool plug,
                                   * lstm.py:25-42,141-151): the caller runs it between the step's kernels.  out_dim = its
                                   * width; the library keeps no pool weights; pool_to_input 0 (out_dim == hidden_dim) or 1.
                                   * Only the step calls below serve it: tb2_pool_inputs_padded, the module,
                                   * tb2_lstm_step_forward with pooled_padded_dev (tb2_lstm_step_backward for training).
                                   * tb2_pool_forward, tb2_lstm_forward_steps and tb2_lstm_sequence_backward return
                                   * TB2_ERR_INVALID; goals are not built with it */

#define TB2_PHASE_ENCODER 0
#define TB2_PHASE_DECODER 1

const char* tb2_last_error(void);
/* 106: one step call (tb2_lstm_step_forward) and one step-range call (tb2_lstm_forward_steps) take the goal, external
 * module, sampling, training-cache and host-output arguments that separate entry points took before.
 * 107: tb2_lstm_rollout_backward, tb2_attack_objective and tb2_attack_step.
 * 108: tb2_lstm_sequence_backward and tb2_lstm_rollout_backward skip the reduction of every NULL tb2_lstm_grads
 *      parameter field (the social backward no longer requires its pool fields).
 * 109: tb2_lstm_relevance_workspace_bytes and tb2_lstm_relevance.
 * 110: tb2_shapley_expand and tb2_shapley_values. */
int tb2_version(void);
/* Number of library kernel launches issued by this process so far (bench "gpu_launches"). */
uint64_t tb2_launch_count(void);

/* Per-kernel timing for bench.py's roofline: between begin and end every library kernel is
 * bracketed by CUDA events on its launching stream.  tb2_profile_end synchronises the device and
 * writes {"kernel": {"launches": n, "total_ms": t}, ...} into json_out. */
int tb2_profile_begin(void);
int tb2_profile_end(char* json_out, size_t capacity);

/* ---------------------------------------------------------------------------------------
 * Model configuration = constructor arguments of LSTM (lstm/lstm.py:46) and
 * GridBasedPooling (lstm/gridbased_pooling.py:16-19).
 * ------------------------------------------------------------------------------------- */
typedef struct tb2_lstm_config {
    int32_t hidden_dim;      /* LSTM hidden_dim: 32, 64, 96, ..., 256 (default 128); any other width
                              * fails tb2_lstm_create with TB2_ERR_UNSUPPORTED     */
    int32_t embedding_dim;   /* LSTM embedding_dim (64); Linear(2, E-2)+2 zero tags */
    int32_t pool_type;       /* TB2_POOL_*                                         */
    int32_t pool_to_input;   /* 1: concat pooled to LSTM input, 0: h += pooled     */
    int32_t n;               /* grid cells per side                                */
    float cell_side;         /* metres                                             */
    int32_t pool_size;       /* must be 1 (CLI never sets it, trainer.py:483-487)  */
    int32_t blur_size;       /* must be 1                                          */
    int32_t front;           /* GridBasedPooling(front=...)                        */
    float constant;          /* background value of the grid                       */
    int32_t latent_dim;      /* social: hidden_dim_encoding out features (16)      */
    int32_t num_layers;      /* grid-embedding MLP: 0 ('None'), 1, 2 or 3 layers   */
    int32_t layer_dims[2];   /* hidden widths of the two/three_layer MLP           */
    int32_t out_dim;         /* pool.out_dim                                       */
    /* TB2_POOL_HIDDEN_MLP only (0 otherwise): widths of the three per-neighbour embeddings whose
     * concatenation (mlp_dim = their sum) is max-pooled over the scene and projected to out_dim */
    int32_t mlp_dim_spatial; /* Linear(2, .) on pos_j - pos_i                      */
    int32_t mlp_dim_vel;     /* Linear(2, .) on 4 (v_j - v_i); may be 0            */
    int32_t mlp_dim_hidden;  /* Linear(H, .) on h_j; may be 0                      */
    float attn_fill;         /* TB2_POOL_ATTN_MLP: fill_value of embed_with_masking (-10) */
    int32_t goal_dim;        /* LSTM(goal_flag=True): goal_dim, the width of the goal embedding appended to the
                              * input embedding (lstm.py:72-85,131-139); 0 = no goal input.  Inference only:
                              * the training forward (cache_dev) and the backward return TB2_ERR_UNSUPPORTED */
} tb2_lstm_config;

/* Device pointers to the parameters in the reference's state_dict layout (row-major
 * [out_features, in_features], SURVEY.md 8b/B2).  Unused entries may be NULL. */
typedef struct tb2_lstm_weights {
    const float* input_embedding_weight;  /* input_embedding.input_embeddings.0.weight [E-2, 2] */
    const float* input_embedding_bias;    /* [E-2] */
    const float* encoder_weight_ih;       /* [4H, E (+out_dim)] */
    const float* encoder_weight_hh;       /* [4H, H] */
    const float* encoder_bias_ih;         /* [4H] */
    const float* encoder_bias_hh;         /* [4H] */
    const float* decoder_weight_ih;
    const float* decoder_weight_hh;
    const float* decoder_bias_ih;
    const float* decoder_bias_hh;
    const float* hidden2normal_weight;    /* hidden2normal.linear.weight [5, H] */
    const float* hidden2normal_bias;      /* [5] */
    const float* pool_encoding_weight;    /* pool.hidden_dim_encoding.weight [latent, H] (social) */
    const float* pool_encoding_bias;      /* [latent] */
    const float* pool_embedding_weight[3];/* pool.embedding.{0,2,4}.weight */
    const float* pool_embedding_bias[3];  /* pool.embedding.{0,2,4}.bias   */
    /* TB2_POOL_HIDDEN_MLP (NULL otherwise) */
    const float* pool_spatial_weight;     /* pool.spatial_embedding.0.weight [mlp_dim_spatial, 2]; TB2_POOL_NN_MLP / _NN_LSTM:
                                           * pool.embedding.0.weight [out_dim / n, 2 or 4]; TB2_POOL_TRAJECTRON: [out_dim, 8] */
    const float* pool_spatial_bias;
    const float* pool_vel_weight;         /* pool.vel_embedding.0.weight [mlp_dim_vel, 2] */
    const float* pool_vel_bias;
    const float* pool_hidden_weight;      /* pool.hidden_embedding.0.weight [mlp_dim_hidden, H] */
    const float* pool_hidden_bias;
    const float* pool_out_weight;         /* pool.out_projection.weight [out_dim, mlp_dim] */
    const float* pool_out_bias;
    /* TB2_POOL_ATTN_MLP (NULL otherwise), E = mlp_dim */
    const float* pool_attn_wq;            /* pool.wq.weight [E, E] (no bias) */
    const float* pool_attn_wk;            /* pool.wk.weight */
    const float* pool_attn_wv;            /* pool.wv.weight */
    const float* pool_attn_in_proj_weight;  /* pool.multihead_attn.in_proj_weight [3E, E] */
    const float* pool_attn_in_proj_bias;    /* pool.multihead_attn.in_proj_bias [3E] */
    const float* pool_attn_out_proj_weight; /* pool.multihead_attn.out_proj.weight [E, E] */
    const float* pool_attn_out_proj_bias;   /* pool.multihead_attn.out_proj.bias [E] */
    /* TB2_POOL_NN_LSTM / TB2_POOL_TRAJECTRON (NULL otherwise), Hp = mlp_dim_hidden; hidden2pool = pool_out_weight / pool_out_bias */
    const float* pool_lstm_weight_ih;     /* pool.pool_lstm.weight_ih [4 Hp, out_dim] */
    const float* pool_lstm_weight_hh;     /* pool.pool_lstm.weight_hh [4 Hp, Hp] */
    const float* pool_lstm_bias_ih;       /* [4 Hp] */
    const float* pool_lstm_bias_hh;       /* [4 Hp] */
    /* goal_dim > 0 (NULL otherwise); encoder / decoder weight_ih columns are then [emb | goal | pooled] */
    const float* goal_embedding_weight;   /* goal_embedding.input_embeddings.0.weight [goal_dim-2, 2] */
    const float* goal_embedding_bias;     /* [goal_dim-2] */
} tb2_lstm_weights;

typedef struct tb2_lstm tb2_lstm;          /* opaque: config + repacked weights on the device */
typedef struct tb2_layout tb2_layout;      /* opaque: scene partition (batch_split) on the device */

/* Replaces LSTM.__init__ + GridBasedPooling.__init__ weight ownership (lstm.py:46-89,
 * gridbased_pooling.py:16-92).  Allocates the repacked weight buffers; tb2_lstm_set_weights
 * must be called before any compute (and again whenever the parameters change). */
int tb2_lstm_create(const tb2_lstm_config* cfg, tb2_lstm** out);
int tb2_lstm_destroy(tb2_lstm* model);
/* Asynchronous device-side repack (transposes / cell-major slabs / fused biases). */
int tb2_lstm_set_weights(tb2_lstm* model, const tb2_lstm_weights* w, void* stream);

/* Replaces the `batch_split` argument of LSTM.forward (lstm.py:170,179-181): scene b owns
 * tracks [scene_offsets[b], scene_offsets[b+1]); its first row is the primary.
 * scene_offsets_host is a HOST pointer (int64, like the reference's LongTensor); the call
 * copies it to the device (synchronous, tiny). */
int tb2_layout_create(const int64_t* scene_offsets_host, int32_t num_scenes, tb2_layout** out);
int tb2_layout_destroy(tb2_layout* layout);
int32_t tb2_layout_num_tracks(const tb2_layout* layout);
int32_t tb2_layout_max_scene(const tb2_layout* layout);
/* 1 (default): scenes behave as in ONE batched call of the reference, i.e. padded to the largest scene
 * of the batch; the NaN-padded slots count as out-of-range neighbours and clobber grid cell 0
 * (gridbased_pooling.py:248-249,281-293) -- what the trainer sees.  0: every scene behaves as if the
 * reference had been called on it alone (what the evaluator does, lstm/trajnet_evaluator.py:15-19), so a
 * batch of scenes reproduces per-scene calls exactly. */
int tb2_layout_set_padding(tb2_layout* layout, int32_t pad_to_batch_max);

/* Bytes of caller-provided scratch needed by the step / sequence / pool calls below. */
size_t tb2_lstm_workspace_bytes(const tb2_lstm* model, const tb2_layout* layout);

/* Debug export for the bit-exactness gate.  Replaces the index arithmetic of
 * GridBasedPooling.occupancy (gridbased_pooling.py:248-249,257-263,273-287).
 *   obs_dev      [M, 2]  positions (NaN = absent)
 *   cell_out_dev [M, n_max-1] int32: flattened cell index oi of neighbour slot jj
 *                (j = jj + (jj >= i) inside the scene padded to n_max); 0 when out of range
 *   in_range_out_dev [M, n_max-1] uint8
 * n_max = tb2_layout_max_scene(layout) (the reference pads every scene to the batch max). */
int tb2_grid_indices(const tb2_lstm* model, const tb2_layout* layout, const float* obs_dev,
                     int32_t* cell_out_dev, uint8_t* in_range_out_dev, void* stream);

/* The pool plug: replaces GridBasedPooling.forward (gridbased_pooling.py:94-110) on the ragged
 * layout.  hidden_dev [M, H], obs1_dev/obs2_dev [M, 2] -> pooled_out_dev [M, out_dim].
 * Rows absent at obs2 still get a (discarded-by-the-caller) row, like the reference. */
int tb2_pool_forward(const tb2_lstm* model, const tb2_layout* layout, const float* hidden_dev,
                     const float* obs1_dev, const float* obs2_dev, float* pooled_out_dev,
                     void* workspace_dev, size_t workspace_bytes, void* stream);

/* One recurrence step: replaces LSTM.step (lstm.py:91-168).
 *   phase            TB2_PHASE_ENCODER / TB2_PHASE_DECODER (which LSTMCell)
 *   obs1_dev/obs2_dev [M, 2]
 *   goals_dev        [M, 2] every track's goal (LSTM(goal_flag=True), lstm.py:131-139): each step feeds the LSTM
 *                    [emb(velocity) | goal_emb | pooled] with goal_emb = cat(ReLU(W_g . 4 d + b_g), 0, 0),
 *                    d = (obs2 - goal) / |obs2 - goal| (0 where that norm is 0).  Required when goal_dim > 0 (NULL:
 *                    TB2_ERR_INVALID, the reference never substitutes zero goals), ignored otherwise.
 *   pooled_padded_dev [B * n_pad, out_dim] the output of the caller's interaction module (TB2_POOL_EXTERNAL, see the
 *                    external-module section below): required by such a model, NULL for any other (TB2_ERR_INVALID).
 *                    The row of every present track (pool_sample[track_mask_positions], lstm.py:148) is concatenated to
 *                    the LSTM input (pool_to_input) or added to its hidden state (lstm.py:151).
 *   h_in/c_in -> h_out/c_out [M, H] (may alias); absent tracks keep their state
 *   normal_out_dev   [M, 5]  (mu_x, mu_y, sigma_x, sigma_y, rho), NaN rows for absent tracks
 *   pos_out_dev      [M, 2]  obs2 + mu (lstm.py:232,255), may be NULL
 * An external model with goal_dim > 0 returns TB2_ERR_UNSUPPORTED. */
int tb2_lstm_step_forward(const tb2_lstm* model, const tb2_layout* layout, int32_t phase,
                          const float* obs1_dev, const float* obs2_dev, const float* goals_dev,
                          const float* pooled_padded_dev,
                          const float* h_in_dev, const float* c_in_dev, float* h_out_dev, float* c_out_dev,
                          float* normal_out_dev, float* pos_out_dev,
                          void* workspace_dev, size_t workspace_bytes, void* stream);

/* Steps [first_step, last_step) of the time loop of LSTM.forward (lstm.py:170-264), including the decoder input rule
 * (lstm.py:240-250); S = obs_length - 1 + n_decode steps in all, [0, S) is the whole forward.
 *   observed_dev  [obs_length, M, 2]
 *   truth_dev     [n_decode, M, 2] teacher-forcing positions (prediction_truth) or NULL for a
 *                 free-running rollout (n_predict = n_decode + 1)
 *   goals_dev     [M, 2] as in tb2_lstm_step_forward: required when goal_dim > 0, ignored otherwise
 *   normals_out_dev   [S, M, 5],  positions_out_dev [S, M, 2]
 *   h_dev, c_dev  [M, H] state buffers.  first_step = 0 zeroes them; otherwise they hold the state after step
 *                 first_step - 1 -- possibly edited by the caller in between, which is how the S-GAN generator injects
 *                 noise between encoder and decoder (sgan/sgan.py:200-221,373) -- and positions_out_dev holds the
 *                 positions of the earlier steps.  They hold the final state on return.
 *   states_out_dev optional [S, 2, M, H] (h, c after every step; training) or NULL.
 * Options, each NULL when not used:
 *   eps_dev       sampled forward (no reference counterpart: the reference feeds back the mean of every step's bivariate
 *                 normal, lstm/lstm.py:232,255).  After every step s >= obs_length - 2 of the range (the last encoder
 *                 step's output and every decoder step: the n_decode + 1 predicted positions) the step's position is
 *                 replaced by a draw of its normal before anything reads it, so the draw is what the following steps
 *                 are fed back:
 *                   pos[s, m] += (sx e1, sy (rho e1 + sqrt(1 - rho^2) e2)),   (sx, sy, rho) = normals[s, m, 2:5],
 *                   (e1, e2) = eps_dev[s - (obs_length - 2), m]
 *                 eps_dev [n_decode + 1, M, 2] holds standard normal pairs aligned with the last n_decode + 1 steps.  A
 *                 pair of exactly (0, 0) leaves the position bit-unchanged (all zeros: the bits of eps_dev = NULL);
 *                 rows with NaN normals stay NaN.  A goal-conditioned model returns TB2_ERR_UNSUPPORTED.
 *   cache_dev     training forward: keeps, per step, the grid-embedding records the social backward reads (winners,
 *                 latent vectors, hidden1 and the pooled vector; reference: everything autograd saves inside
 *                 GridBasedPooling.forward, lstm/gridbased_pooling.py:94-170,308-335).  Needs states_out_dev, the whole
 *                 range [0, S) and cache_bytes >= tb2_lstm_train_cache_bytes(S) > 0 (TB2_ERR_INVALID otherwise); the
 *                 buffer must stay untouched until tb2_lstm_sequence_backward has run.  A goal-conditioned model
 *                 returns TB2_ERR_UNSUPPORTED.
 *   normals_host, positions_host, copy_stream  (set together) host outputs, for callers whose results live in HOST
 *                 memory (the reference's predictor / evaluator boundary hands numpy arrays back): after every step of
 *                 the range the step's slices of normals / positions are copied to these page-locked buffers
 *                 [S, M, 5] / [S, M, 2] on `copy_stream`, ordered behind the step by an event, while the later steps
 *                 compute -- the device-to-host traffic (M x 28 bytes per step) hides under the forward instead of
 *                 following it.  The call does not synchronise: results are complete once `copy_stream` is.  The
 *                 device outputs are written as well.
 * A TB2_POOL_EXTERNAL model returns TB2_ERR_INVALID: it runs step by step (tb2_lstm_step_forward). */
int tb2_lstm_forward_steps(const tb2_lstm* model, const tb2_layout* layout,
                           const float* observed_dev, int32_t obs_length, const float* truth_dev, int32_t n_decode,
                           const float* goals_dev, const float* eps_dev, int32_t first_step, int32_t last_step,
                           float* normals_out_dev, float* positions_out_dev, float* h_dev, float* c_dev,
                           float* states_out_dev, void* cache_dev, size_t cache_bytes,
                           float* normals_host, float* positions_host, void* copy_stream,
                           void* workspace_dev, size_t workspace_bytes, void* stream);

/* Bytes of the training cache (cache_dev of tb2_lstm_forward_steps) for num_steps steps: > 0 for every social model
 * the backward supports and 0 for the other models, which keep no cache (pass NULL / 0). */
size_t tb2_lstm_train_cache_bytes(const tb2_lstm* model, const tb2_layout* layout, int32_t num_steps);

/* The sampling of tb2_lstm_forward_steps (eps_dev) on one step's rows: positions [rows, 2] += the offset above from
 * normals [rows, 5] and eps [rows, 2], in place.  The batched multi-mode decode applies it to the replicated output of
 * the last encoder step before the decoder steps run. */
int tb2_lstm_sample_positions(const float* normals_dev, float* positions_dev, const float* eps_dev, int32_t rows,
                              void* stream);

/* LSTMGenerator.adding_noise (sgan/sgan.py:200-221), in place on the hidden state of all tracks:
 *   h[m] <- cat(ReLU(weight . h[m] + bias), noise)   weight [H - noise_dim, H] (mlp_decoder_context.0),
 * noise [noise_dim] is one vector shared by all tracks.  Called between the encoder steps and the
 * decoder steps of tb2_lstm_forward_steps. */
int tb2_sgan_add_noise(const float* weight_dev, const float* bias_dev, const float* noise_dev, float* h_dev,
                       int32_t M, int32_t H, int32_t noise_dim, void* stream);

/* VAE.add_noise at test time (vae/vae.py:87-106), in place: h[m] <- h[m] * ReLU(weight . z[m] + bias),
 * weight [H, latent_dim] (vae_decoder.fc), z [M, latent_dim] one latent sample per track. */
int tb2_vae_scale_hidden(const float* weight_dev, const float* bias_dev, const float* z_dev, float* h_dev,
                         int32_t M, int32_t H, int32_t latent_dim, void* stream);

/* Decoder starting state of k modes in one pass over the encoder state (M tracks), mode-major:
 * output row q * M + m is track m in mode q, for q < k.
 *   h_out[q*M + m] = cat(ReLU(weight . h_enc[m] + bias), noise[q * num_groups + group_of_row[m]])
 *   c_out[q*M + m] = c_enc[m]
 * weight [H - noise_dim, H]; noise [k * num_groups, noise_dim] holds one vector per (mode, scene);
 * group_of_row [M] is the scene of every track.  ReLU(weight . h + bias) is computed once per track; every
 * replica row is bit-identical to tb2_sgan_add_noise on a copy of h_enc with that row's noise vector.
 * h_out / c_out [k * M, H] must not overlap the inputs. */
int tb2_sgan_decoder_context(const float* weight_dev, const float* bias_dev, const float* noise_dev,
                             const int32_t* group_of_row_dev, int32_t num_groups, const float* h_enc_dev,
                             const float* c_enc_dev, int32_t M, int32_t H, int32_t noise_dim, int32_t k,
                             float* h_out_dev, float* c_out_dev, void* stream);

/* The VAE's counterpart, mode-major like tb2_sgan_decoder_context, with one latent sample per (mode, track):
 *   h_out[q*M + m] = h_enc[m] * ReLU(weight . z[q*M + m] + bias),   c_out[q*M + m] = c_enc[m]
 * weight [H, latent_dim], z [k * M, latent_dim]; bit-identical to tb2_vae_scale_hidden on a copy of h_enc. */
int tb2_vae_decoder_context(const float* weight_dev, const float* bias_dev, const float* z_dev,
                            const float* h_enc_dev, const float* c_enc_dev, int32_t M, int32_t H,
                            int32_t latent_dim, int32_t k, float* h_out_dev, float* c_out_dev, void* stream);

/* ---------------------------------------------------------------------------------------
 * External interaction modules (TB2_POOL_EXTERNAL): one recurrence step with the module run by the caller.
 * n_pad = tb2_layout_max_scene(layout); slot (b, j) of the padded layout [B, n_pad] is track scene_offsets[b] + j
 * when j < the size of scene b, padding otherwise.
 * ------------------------------------------------------------------------------------- */
/* generate_pooling_inputs (lstm.py:25-42): obs1 / obs2 [M, 2] and h [M, H] of the ragged layout ->
 * obs1_pad / obs2_pad [B, n_pad, 2] and h_pad [B, n_pad, H], NaN in the padding slots.  Every track's hidden state goes
 * in, absent tracks included.  The module is then called as pool(h_pad, obs1_pad, obs2_pad) -> [B * n_pad, out_dim]. */
int tb2_pool_inputs_padded(const tb2_layout* layout, const float* obs1_dev, const float* obs2_dev, const float* h_dev,
                           int32_t H, float* obs1_pad_out_dev, float* obs2_pad_out_dev, float* h_pad_out_dev,
                           void* stream);
/* Its backward: d_h_dev [M, H] += the rows of d_h_pad_dev [B, n_pad, H] at every track's slot (padding is dropped). */
int tb2_pool_inputs_padded_backward(const tb2_layout* layout, const float* d_h_pad_dev, int32_t H, float* d_h_dev,
                                    void* stream);
/* ---------------------------------------------------------------------------------------
 * Training: backward of the whole time loop (what autograd does for Trainer.train_batch,
 * lstm/trainer.py:229-269, through LSTM.forward).  Gradient accumulators are fp32 device
 * buffers in the reference's parameter layout (+=, caller zeroes them).  Zero the whole struct
 * before filling it (memset / `= {0}`): a NULL field is a gradient the call does not compute, and
 * fields appended by later versions then stay NULL.  tb2_lstm_sequence_backward and tb2_lstm_rollout_backward skip the
 * reduction of each NULL parameter field (version 108); any of them may be NULL.  d_observed does not depend on which
 * parameter fields are set (bit for bit), and a field that is set gets the bits of the call with every field set.
 * ------------------------------------------------------------------------------------- */
typedef struct tb2_lstm_grads {
    float* input_embedding_weight;   /* [E-2, 2] */
    float* input_embedding_bias;     /* [E-2]    */
    float* encoder_weight_ih;        /* [4H, E (+out_dim)] */
    float* encoder_weight_hh;        /* [4H, H] */
    float* encoder_bias_ih;          /* [4H] */
    float* encoder_bias_hh;          /* [4H] */
    float* decoder_weight_ih;
    float* decoder_weight_hh;
    float* decoder_bias_ih;
    float* decoder_bias_hh;
    float* hidden2normal_weight;     /* [5, H] */
    float* hidden2normal_bias;       /* [5] */
    float* pool_embedding_weight0;   /* pool.embedding.0.weight grad [d1, C*n*n] or NULL */
    float* pool_embedding_bias0;     /* [d1] or NULL */
    float* pool_embedding_weight1;   /* pool.embedding.2.weight grad [out_dim, d1] (two_layer, social) or NULL */
    float* pool_embedding_bias1;     /* [out_dim] or NULL */
    float* pool_encoding_weight;     /* pool.hidden_dim_encoding.weight grad [latent, H] (social) or NULL */
    float* pool_encoding_bias;       /* [latent] or NULL */
    /* Gradient wrt the observed positions (version 105), NULL = not computed.  It flows through the encoder steps'
     * velocity inputs (vel = obs2 - obs1), the directional grid's relative velocities and, with social pooling, the
     * hidden states the grid reads.  Decoder inputs are detached: fed-back positions, teacher-forced truth and the
     * copy of observed[-1] (lstm.py:235-250).  The head term pred = obs2 + mu is the caller's: the call cannot tell
     * d pred from d mu in d_normals. */
    float* d_observed;               /* [obs_length, M, 2] (+=), tb2_lstm_sequence_backward */
    float* d_obs1;                   /* [M, 2] (+=), tb2_lstm_step_backward; set both or neither */
    float* d_obs2;                   /* [M, 2] (+=), tb2_lstm_step_backward */
} tb2_lstm_grads;

/* scratch for tb2_lstm_sequence_backward: per (step, active row) records + per-step buffers */
size_t tb2_lstm_backward_workspace_bytes(const tb2_lstm* model, const tb2_layout* layout, int32_t num_active,
                                         int32_t num_steps);

/* BPTT over the rows that receive gradient.
 *   weights          the same fp32 parameter pointers given to tb2_lstm_set_weights
 *   observed/truth   inputs of the forward call (truth: teacher forcing or NULL)
 *   positions_dev    [S, M, 2] and states_dev [S, 2, M, H]: outputs of tb2_lstm_forward_steps
 *   d_normals_dev    [S, M, 5] upstream gradient wrt rel_pred_scene (d pred_scene already added to
 *                    its first two columns by the caller: pred = obs2 + mu, lstm.py:232,255)
 *   active_rows_dev  int32 [num_active]: tracks with a non-zero upstream gradient (PredictionLoss
 *                    touches the scene primaries only, lstm/loss.py:57,67)
 * Supported: vanilla, occupancy / directional pooling with a one_layer embedding (the D-LSTM
 * training config), and social pooling with a one_layer / two_layer embedding (constant = 0).
 * Social pooling couples all tracks of a scene through the hidden-state scatter (the reference
 * does not detach hidden_states_to_pool, lstm.py:26): the backward then runs on all M rows and
 * active_rows is ignored.
 *   cache_dev        the training cache tb2_lstm_forward_steps filled (social pooling; without it
 *                    the call returns TB2_ERR_INVALID).  Other models have none: NULL / 0. */
int tb2_lstm_sequence_backward(const tb2_lstm* model, const tb2_layout* layout, const tb2_lstm_weights* weights,
                               const float* observed_dev, int32_t obs_length, const float* truth_dev,
                               int32_t n_decode, const float* positions_dev, const float* states_dev,
                               const float* d_normals_dev, const int32_t* active_rows_dev, int32_t num_active,
                               const tb2_lstm_grads* grads, void* workspace_dev, size_t workspace_bytes,
                               void* bwd_workspace_dev, size_t bwd_workspace_bytes, const void* cache_dev,
                               size_t cache_bytes, void* stream);

/* Backward of a free-running forward (tb2_lstm_forward_steps with truth = NULL and a training cache for social pooling)
 * on the graph where nothing is detached (version 107): the decoder's fed-back positions carry gradient.  Decoder step
 * S_enc reads obs1 = observed[-1] (the scene primaries: positions[S_enc - 2], lstm.py:240-241) and
 * obs2 = positions[S_enc - 1]; step S_enc + k (k >= 1) reads positions[S_enc + k - 2] and positions[S_enc + k - 1];
 * every step outputs positions[s] = obs2 + mu.  A decoder input gets gradient through the same paths an encoder input
 * does: the velocity input, the directional grid's relative velocities and pos = obs2 + mu (cell binning is piecewise
 * constant: no gradient).  Same arguments as tb2_lstm_sequence_backward without truth, and:
 *   d_normals_dev    [S, M, 5] gradient wrt rel_pred_scene alone (nothing added by the caller)
 *   d_positions_dev  [S + (obs_length == 2), M, 2] gradient wrt LSTM.forward's pred_scene (at obs_length 2 it begins
 *                    with observed[-1] itself)
 *   grads->d_observed  required; the parameter gradients include the fed-back terms.  With every parameter field NULL
 *                    this is the inputs-only call (the collision attack's backward): no parameter reduction runs.
 * active_rows: tracks with a non-zero d_normals or d_positions row; directional pooling couples the tracks of a scene
 * through the relative velocities, so there every track must be listed (social pooling runs on all rows anyway).
 * Workspace: tb2_lstm_backward_workspace_bytes.  Goal models: TB2_ERR_UNSUPPORTED. */
int tb2_lstm_rollout_backward(const tb2_lstm* model, const tb2_layout* layout, const tb2_lstm_weights* weights,
                              const float* observed_dev, int32_t obs_length, int32_t n_decode,
                              const float* positions_dev, const float* states_dev, const float* d_normals_dev,
                              const float* d_positions_dev, const int32_t* active_rows_dev, int32_t num_active,
                              const tb2_lstm_grads* grads, void* workspace_dev, size_t workspace_bytes,
                              void* bwd_workspace_dev, size_t bwd_workspace_bytes, const void* cache_dev,
                              size_t cache_bytes, void* stream);

/* Layer-wise relevance (LRP) of a free-running forecast: for every scene b and prediction t (0 .. n_decode), how much
 * the primary's predicted mean velocity at step s_t = obs_length - 2 + t relies on the primary's own velocity input and
 * on each neighbour, at every step.  The explained scalar is y = |mu| of that step (0 when mu is 0 or not finite, or the
 * primary is absent there).  Rules, with z' = z + eps sign(z): the eps-rule for hidden2normal (d = mu / |mu| fixed), the
 * gate operand's g block and the embeddings' Linear layers; signal-take-all for the LSTM cell (the i, f, o gates get
 * nothing); a grid cell's relevance goes to the neighbour that won it (last writer), a social cell's stops at the
 * winner's latent.  Only the primaries are explained; y - sum(relevance) is what the biases and eps absorbed.
 *   observed_dev, positions_dev, states_dev  as for tb2_lstm_rollout_backward: the forward of
 *                    tb2_lstm_forward_steps over the S = obs_length - 1 + n_decode steps, no teacher forcing
 *   relevance_out_dev [n_decode + 1, S, M]  the own column at each scene's primary, neighbour columns elsewhere
 *   explained_out_dev [n_decode + 1, B]     y
 * Vanilla, occupancy / directional (one_layer, constant 0, pool_to_input, widths <= 1024) and social (one_layer /
 * two_layer, constant 0, pool_to_input, widths <= 1024) models; TB2_ERR_UNSUPPORTED names any other configuration
 * (goal models, the non-grid and external modules, other grid embeddings).  Workspace:
 * tb2_lstm_relevance_workspace_bytes (0 for an unsupported model), 256-byte aligned.  No host synchronisation; the
 * result is bit-identical from run to run, and with per-scene padding (tb2_layout_set_padding 0) to per-scene calls. */
size_t tb2_lstm_relevance_workspace_bytes(const tb2_lstm* model, const tb2_layout* layout, int32_t n_predict,
                                          int32_t obs_length);
int tb2_lstm_relevance(const tb2_lstm* model, const tb2_layout* layout, const tb2_lstm_weights* weights,
                       const float* observed_dev, int32_t obs_length, int32_t n_decode, const float* positions_dev,
                       const float* states_dev, float eps, float* relevance_out_dev, float* explained_out_dev,
                       void* workspace_dev, size_t workspace_bytes, void* stream);

/* Shapley attribution of the primary's forecast error to its nearest neighbours (lstm/shapley.py), one launch each per
 * chunk of scenes, no atomics.  A scene b of N_b rows (primary first) has K_b <= 12 players, the K_b nearest neighbours
 * of the primary at the last observed frame (squared distance in float64 of the float32 positions, a non-finite one
 * counts as +inf, ties go to the lower row), and 2^K_b instances, one per coalition mask (bit r = the player of rank r):
 * the scene with the players outside the coalition deleted, the other rows in their original order.  instance_first
 * [B + 1] gives each scene's first instance (instance_first[b + 1] - instance_first[b] = 2^K_b), instance_split [I + 1]
 * the instances' rows, as the caller's batch_split of the instance batch (rows of instance i: N_b - K_b + popcount(mask)).
 * tb2_shapley_expand -- expanded_out [obs_length, out_tracks, 2] = every instance's rows of observed [obs_length,
 *   num_tracks, 2] (scene_off [B + 1]: the scenes' rows there); player_rows_out [B, 12] = each scene's player rows, by
 *   rank, relative to the scene's first row (-1 past K_b); coalition_out [I] = each instance's mask.  max_scene >= every
 *   N_b, at most 6144.
 * tb2_shapley_values -- from positions [num_frames, num_tracks, 2] (the instance batch's forecast; its last pred_length
 *   frames are scored) and truth [B, pred_length, 2] (double, the primaries' ground truth): per instance v = (ADE, FDE)
 *   of its primary, tb2_score_scenes' arithmetic; with frame [B, 4] (cx, cy, cos, sin; NULL: none) the prediction is
 *   first taken to the world frame as tb2_scenes_inverse does.  phi_{ade,fde}_out [B, 12] (double, NaN past K_b):
 *   phi_j = sum over S subset of the players without j, in ascending mask order, of |S|! (K - |S| - 1)! / K! (v(S + j) -
 *   v(S)); v_out [4, B] = v_ADE(all), v_FDE(all), v_ADE(none), v_FDE(none); values_out [I, 2] (optional) = v.
 *   max_players >= every K_b (it sizes the shared-memory value table). */
int tb2_shapley_expand(const float* observed_dev, int32_t obs_length, int32_t num_tracks, const int32_t* scene_off_dev,
                       const int32_t* instance_first_dev, const int32_t* instance_split_dev, int32_t num_scenes,
                       int32_t num_instances, int32_t max_scene, int32_t out_tracks, float* expanded_out_dev,
                       int32_t* player_rows_out_dev, int32_t* coalition_out_dev, void* stream);
int tb2_shapley_values(const float* positions_dev, int32_t num_frames, int32_t num_tracks, int32_t pred_length,
                       const int32_t* instance_first_dev, const int32_t* instance_split_dev, int32_t num_scenes,
                       int32_t max_players, const double* truth_dev, const double* frame_dev, double* phi_ade_out_dev,
                       double* phi_fde_out_dev, double* v_out_dev, double* values_out_dev, void* stream);

/* Backward of one tb2_lstm_step_forward step of a TB2_POOL_EXTERNAL model, from the step's inputs: the gate
 * pre-activations are recomputed (one GEMM), then
 *   d_h_in_dev, d_c_in_dev  [M, H]                gradient wrt h_in / c_in (absent tracks: d_h_out / d_c_out unchanged)
 *   d_pooled_padded_dev     [B * n_pad, out_dim]  gradient wrt pooled_padded (0 for absent tracks and padding slots)
 * and the step's gradients are ADDED to `grads`: input embedding, the phase's LSTMCell and hidden2normal (those fields
 * must be set; the other phase's may be NULL).  d_normal_dev [M, 5] is the upstream gradient wrt the step's normals
 * with that wrt pos already added to its first two columns (pos = obs2 + mu); NaN entries count as 0.  d_c_in may alias
 * d_c_out.  grads->d_obs1 / d_obs2 (optional) receive the gradient through the step's velocity input; the term of
 * pos = obs2 + mu is the caller's. */
size_t tb2_lstm_step_backward_workspace_bytes(const tb2_lstm* model, const tb2_layout* layout);
int tb2_lstm_step_backward(const tb2_lstm* model, const tb2_layout* layout, const tb2_lstm_weights* weights,
                           int32_t phase, const float* obs1_dev, const float* obs2_dev, const float* pooled_padded_dev,
                           const float* h_in_dev, const float* c_in_dev, const float* d_h_out_dev,
                           const float* d_c_out_dev, const float* d_normal_dev, float* d_h_in_dev, float* d_c_in_dev,
                           float* d_pooled_padded_dev, const tb2_lstm_grads* grads, void* bwd_workspace_dev,
                           size_t bwd_workspace_bytes, void* stream);

/* TB2_POOL_NN_LSTM / TB2_POOL_TRAJECTRON: zero the interaction-encoder LSTM state kept in `workspace`
 * (NearestNeighborLSTM.reset, non_gridbased_pooling.py:385-389; TrajectronPooling.reset, :481-485).  tb2_lstm_forward_steps(first_step = 0) does this itself; the
 * stand-alone plug (tb2_pool_forward) advances the state on every call and needs it after a reset().  No-op for the
 * other pool types. */
int tb2_pool_state_reset(const tb2_lstm* model, const tb2_layout* layout, void* workspace_dev, size_t workspace_bytes,
                         void* stream);

/* PredictionLoss on the device (lstm/loss.py:52-91, gaussian_2d :24-50): per (frame, scene)
 *   values_out  [T, B]    = -log(0.01 + bg N(x|mu,3,3,0) + (0.99-bg) N(x|mu,s1,s2,rho)) of the primary
 *   dinputs_out [T, B, 5] = d value / d (mu1, mu2, s1, s2, rho) (optional, NULL to skip)
 * inputs [T, M, 5], targets [T, M, 2] device fp32; primary_rows int32 [B] = batch_split[:-1].
 * The mean / keep_batch_dim reductions of the reference stay with the caller. */
int tb2_prediction_loss(const float* inputs_dev, const float* targets_dev, const int32_t* primary_rows_dev,
                        int32_t T, int32_t M, int32_t B, float background_rate, float* values_out_dev,
                        float* dinputs_out_dev, void* stream);

/* L2Loss (lstm/loss.py:93-135): per (frame, scene) 0.5 * |mu - target|^2 of the primary (= the mean over
 * the two coordinates); dinputs_out [T, B, 5] = (dx, dy, 0, 0, 0) (optional).  The x100 multiplier and the
 * mean reductions stay with the caller.  Same argument layout as tb2_prediction_loss. */
int tb2_l2_loss(const float* inputs_dev, const float* targets_dev, const int32_t* primary_rows_dev, int32_t T,
                int32_t M, int32_t B, float* values_out_dev, float* dinputs_out_dev, void* stream);

/* CollisionLoss (lstm/loss.py:138-162): per (frame, scene) col_wt * sum over neighbours closer
 * than col_distance to the primary of (1 - dist / col_distance); NaN coordinates read as -1000;
 * neighbours are constants.  positions [T, M, 2]; loss_out [T, B]; dprimary_out [T, B, 2]
 * (gradient wrt the primary's position, optional). */
int tb2_collision_loss(const tb2_layout* layout, const float* positions_dev, int32_t T, float col_wt,
                       float col_distance, float* loss_out_dev, float* dprimary_out_dev, void* stream);

/* Collision attack on free-running forecasts (attack.py), one launch each, no atomics.
 * tb2_attack_objective -- per scene D_out [B] (double) = the smallest distance between the primary's and any neighbour's
 *   positions at the points the scorer's Col-I test samples (tb2_score_scenes): frames [first_frame, num_frames) of
 *   positions [num_frames, M, 2] where both tracks are finite, each segment between consecutive such frames sampled at
 *   linspace(p_prev, p_t, 3) on both tracks.  D <= 0.2 m exactly when Col-I fires on the same values.  A scene without a
 *   finite pair gets +inf.  d_positions_out [num_frames, M, 2] = the subgradient of D at the first minimiser in
 *   (neighbour, frame, sample) order on the four segment endpoints (0 elsewhere, and for D = +inf or D = 0).
 * tb2_attack_step -- per scene: when D [B] < best_D [B] (in/out; start at +inf) the iterate is recorded: best_D, the
 *   primary's delta [obs_length, B, 2] into best_delta and the scene's rows of positions [num_frames, M, 2] into
 *   best_positions.  Then with move != 0, unless best_D <= 0.2 m, every observed frame t of the primary whose position
 *   and gradient g_t = d_observed[t, primary] are finite and g_t != 0 steps:
 *   delta_t <- proj_eps(delta_t - alpha g_t / |g_t|) (L2 ball of radius eps per frame), and observed_adv
 *   [obs_length, M, 2] gets observed + delta on the primary rows (its other rows are the caller's). */
int tb2_attack_objective(const tb2_layout* layout, const float* positions_dev, int32_t num_frames, int32_t first_frame,
                         double* D_out_dev, float* d_positions_out_dev, void* stream);
int tb2_attack_step(const tb2_layout* layout, const float* d_observed_dev, const float* observed_dev, int32_t obs_length,
                    float* delta_dev, const double* D_dev, int32_t num_frames, const float* positions_dev,
                    double* best_D_dev, float* best_delta_dev, float* best_positions_dev, float* observed_adv_dev,
                    float eps, float alpha, int32_t move, void* stream);

/* ---------------------------------------------------------------------------------------
 * Scene preprocessing on the device (SURVEY.md 8f rank 3): the O(T * M) NumPy passes the reference runs scene by scene
 * before a batch reaches the model, for a whole ragged batch per launch.  xy is float64 [T, M, 2] (the dtype
 * Reader.paths_to_xy produces), scene_off int32 [B + 1] row offsets ON THE DEVICE; the primary of a scene is its first
 * row.  All arithmetic is float64 in the reference's operation order with unfused multiplies / adds; the float32 batch is
 * rounded once at the end (torch.Tensor(ndarray), lstm/trainer.py:124), so it equals the host path bit for bit.
 *
 * tb2_scenes_drop_distant -- drop_distant (lstm/lstm.py:16-22): keep_out [M] = 1 where the track comes within r of its
 *   scene's primary in some frame (nanmin over frames of the squared distance < r_squared; the caller passes r ** 2),
 *   kept_count_out [B] = kept tracks per scene (the caller's cumulative sum is the new batch_split).
 * tb2_scenes_transform -- compaction by `keep` (NULL: keep all, then M_out == M and out_off == scene_off) into out_off
 *   [B + 1], then center_scene (lstm/utils.py:32-51; frame [B, 4] = centre x, centre y, cos(rotation), sin(rotation); NULL: skip)
 *   = shift by the centre and einsum('ptc,ci->pti', xy, [[ct, st], [-st, ct]]), then random_rotation (lstm/utils.py:10-17;
 *   aug [B, 2] = cos(theta), sin(theta); NULL: skip); xy_out float32 [T, M_out, 2].  The O(B) scalars of `frame` / `aug` come
 *   from the caller (the reference's own libm calls on the primary's last two observed positions).
 * tb2_scenes_inverse -- inverse_scene (augmentation.py:65-68) of float32 predictions [S, M, 2]: rotation by
 *   frame [B, 4] = centre x, centre y, cos(-rotation), sin(-rotation), then + centre; xy_out float64 [S, M, 2].
 * tb2_scenes_gather_epoch -- every batch of a training epoch (lstm/trainer.py:96-133) in one launch, from a scene store
 *   xy [T, M] with scene_off [n_store + 1], the drop_distant mask `keep` [M] (NULL: keep all) and kept_count [n_store].
 *   Epoch position p holds store scene perm[p] (p < n) and belongs to batch p / batch_size.  Batch k is written as ONE
 *   contiguous float32 block [T, batch_tracks[k], 2] starting at float2 element batch_base[k] of xy_out; inside it the
 *   scenes' kept tracks follow in position order (np.concatenate(axis=1)).  Per scene, in the reference's order: ordered
 *   compaction by `keep`, center_scene (frame [n_store, 4] indexed by STORE scene; NULL: skip), random_rotation
 *   (aug [n, 2] = cos, sin of theta indexed by epoch POSITION; NULL: skip), add_noise(ped='neigh') = `+=` of the float64
 *   values noise[noise_off[p] + (t * (kept - 1) + j - 1) * 2 + c] on frames t < noise_frames of kept columns j >= 1
 *   (NULL: skip; the reference's window is 9 frames whatever obs_length is), then one rounding to float32. */
int tb2_scenes_drop_distant(const double* xy_dev, const int32_t* scene_off_dev, int32_t T, int32_t M, int32_t B,
                            double r_squared, uint8_t* keep_out_dev, int32_t* kept_count_out_dev, void* stream);
int tb2_scenes_transform(const double* xy_dev, const int32_t* scene_off_dev, const uint8_t* keep_dev,
                         const int32_t* out_off_dev, int32_t T, int32_t M, int32_t M_out, int32_t B,
                         const double* frame_dev, const double* aug_dev, float* xy_out_dev, void* stream);
int tb2_scenes_inverse(const float* xy_dev, const int32_t* scene_off_dev, int32_t S, int32_t M, int32_t B,
                       const double* frame_dev, double* xy_out_dev, void* stream);
int tb2_scenes_gather_epoch(const double* xy_dev, const int32_t* scene_off_dev, const uint8_t* keep_dev,
                            const int32_t* kept_count_dev, int32_t T, int32_t M, const int32_t* perm_dev, int32_t n,
                            int32_t batch_size, const int64_t* batch_base_dev, const int32_t* batch_tracks_dev,
                            const double* frame_dev, const double* aug_dev, const double* noise_dev,
                            const int64_t* noise_off_dev, int32_t noise_frames, float* xy_out_dev, void* stream);

/* ---------------------------------------------------------------------------------------
 * Host-side ndjson codec of the batched evaluator path (SURVEY.md 8f rank 1; no CUDA).  The TrajNet++ on-disk format as the
 * reference reads / writes it through trajnetplusplustools (evaluator/write_utils.py:42-81, DATA_BLOCK files): one JSON
 * object per line, {"track": {"f", "p", "x", "y"[, "prediction_number", "scene_id"]}} or {"scene": {"id", "p", "s", "e", "fps", "tag"}}.
 *
 * tb2_ndjson_parse -- text -> column arrays (caller-allocated, max_rows = number of lines): track rows in file order and
 *   scene rows in file order.  Numbers are read as json.loads reads them (integer literals for f / p / id / s / e, float(str)
 *   = correctly rounded strtod for x / y, NaN / Infinity accepted).  A line the parser is not certain about (string
 *   escapes, a missing or non-integer field, an unknown record type) stops it: refused_line_out = its 0-based index
 *   (else -1) and the caller takes its json.loads path for the whole file.
 * tb2_ndjson_format -- prediction records -> text: per scene one scene line then rows_per_scene[i] track lines, in the
 *   caller's row order, byte-identical to json.dumps of the reference writer's dictionaries with coordinates round(v, 2).
 *   Returns the byte count needed (whole lines are written while they fit into `capacity`, nothing past it;
 *   <= 160 bytes per line), or a negative error
 *   (TB2_ERR_UNSUPPORTED for finite |coordinate| >= 1e15, where repr() would need an exponent). */
int tb2_ndjson_parse(const char* text, size_t len, int64_t max_rows, int64_t* track_frame, int64_t* track_ped,
                     double* track_x, double* track_y, int64_t* num_tracks_out, int64_t* scene_id, int64_t* scene_ped,
                     int64_t* scene_start, int64_t* scene_end, int64_t* num_scenes_out, int64_t* refused_line_out);
int64_t tb2_ndjson_format(int64_t num_scenes, const int64_t* scene_id, const int64_t* scene_ped, const int64_t* scene_start,
                          const int64_t* scene_end, const int64_t* rows_per_scene, const int64_t* row_frame,
                          const int64_t* row_ped, const double* row_x, const double* row_y, const int64_t* row_mode,
                          char* out, int64_t capacity);

/* tb2_ndjson_parse_meta -- tb2_ndjson_parse plus the metadata the scorer reads: per track row prediction_number and
 *   scene_id (-1 where the key is absent), per scene row the tag as main type (-1 where absent) and sub-types as a
 *   bitmask (bit k = sub-type k).  A tag is an integer or [main, [sub, ...]] with sub-types 0..62; prediction_number and
 *   scene_id are non-negative integers.  Anything else in those keys refuses the line, as above. */
int tb2_ndjson_parse_meta(const char* text, size_t len, int64_t max_rows, int64_t* track_frame, int64_t* track_ped,
                          double* track_x, double* track_y, int64_t* track_prediction_number, int64_t* track_scene_id,
                          int64_t* num_tracks_out, int64_t* scene_id, int64_t* scene_ped, int64_t* scene_start,
                          int64_t* scene_end, int64_t* scene_tag, int64_t* scene_sub_tags, int64_t* num_scenes_out,
                          int64_t* refused_line_out);

/* ---------------------------------------------------------------------------------------
 * Scoring of predictions (evaluator/trajnet_evaluator.py TrajnetEvaluator.aggregate, evaluator/eval_utils.py): one launch
 * per file, one record per scene, no atomics (bit-identical from run to run).  S scenes, T = pred_length frames, K modes.
 * All positions are float64 (x, y) pairs on the ground truth's last T frames of the primary, read as double2 (the four
 * position arrays must be 16-byte aligned; TB2_ERR_INVALID otherwise); pred_length 1..1024:
 *   gt_primary_dev      [S, T, 2]      ground-truth primary
 *   pred_primary_dev    [S, K, T, 2]   predicted primary per mode (modes >= num_modes_dev[s] are not read)
 *   num_modes_dev       [S] int32      modes of scene s (>= 1)
 *   gt_neigh_off_dev    [S + 1] int32  scene s owns ground-truth neighbours gt_neigh_off[s] .. gt_neigh_off[s + 1] - 1
 *   gt_neigh_dev        [G, T, 2], gt_neigh_mask_dev [G, T] uint8 (1 = the neighbour has a row at that frame)
 *   pred_neigh_*        the same for the predicted neighbours (mode 0)
 * Outputs: ade_out / fde_out [S, K] per mode (NaN for absent modes); flags_out [S] (TB2_SCORE_* bits; the collisions use
 * mode 0); with_nll != 0: nll_out [S] = -(mean over the kept timesteps of the clipped KDE log-density), NaN and
 * TB2_SCORE_NLL_ALL_SKIPPED when no timestep is kept. */
#define TB2_SCORE_COL_GT 1
#define TB2_SCORE_COL_PRED 2
#define TB2_SCORE_NEIGH_COUNT_DIFFERS 4
#define TB2_SCORE_NLL_ALL_SKIPPED 8
int tb2_score_scenes(int32_t num_scenes, int32_t pred_length, int32_t max_modes, const double* gt_primary_dev,
                     const double* pred_primary_dev, const int32_t* num_modes_dev, const int32_t* gt_neigh_off_dev,
                     const double* gt_neigh_dev, const uint8_t* gt_neigh_mask_dev, const int32_t* pred_neigh_off_dev,
                     const double* pred_neigh_dev, const uint8_t* pred_neigh_mask_dev, int32_t with_nll,
                     double* ade_out_dev, double* fde_out_dev, double* nll_out_dev, int32_t* flags_out_dev, void* stream);

/* ---------------------------------------------------------------------------------------
 * Classical crowd simulators (classical/socialforce.py, classical/orca.py).  One simulator
 * per scene, all scenes stepped in lockstep by one persistent kernel; no collective.
 * State is SoA-free AoS fp32: scenes are contiguous ranges of agents (layout handle).
 * ------------------------------------------------------------------------------------- */
typedef struct tb2_sf_params {
    double delta_t;     /* 1/fps = 0.05            socialforce.py:80,91 (float64 like upstream) */
    double tau;         /* sf_params[0] = 0.5      socialforce.py:92    */
    double v0;          /* sf_params[1] = 2.1      socialforce.py:89    */
    double sigma;       /* sf_params[2] = 0.3      socialforce.py:89    */
    int32_t n_steps;    /* pred_length * sampling_rate = 96   socialforce.py:93 */
    int32_t sample_every; /* sampling_rate = 8; sample kept when step_index % 8 == 0 (:95) */
} tb2_sf_params;

/* Replaces socialforce.Simulator(...).step() x n_steps (socialforce.py:91-95).  float64 like
 * the upstream numpy package.
 *   state_dev  [A, 6] double (x, y, vx, vy, dx, dy) initial state, socialforce.py:15-55
 *   out_dev    [n_samples, A, 2] double sampled positions, n_samples = ceil(n_steps / sample_every) */
int tb2_sf_simulate(const tb2_layout* layout, const tb2_sf_params* p, const double* state_dev,
                    double* out_dev, void* stream);

typedef struct tb2_orca_params {
    float time_step;       /* 1/fps                         orca.py:90 */
    float neighbor_dist;   /* orca_params[0] = 1.5                     */
    int32_t max_neighbors; /* 10                                       */
    float time_horizon;    /* orca_params[1] = 1.5                     */
    float radius;          /* orca_params[2] = 0.4                     */
    double end_range;      /* 0.05 (orca.py:97), compared in double like the reference */
    int32_t n_steps;       /* sampling_rate * pred_length + 1 = 97 (orca.py:99) */
    int32_t sample_every;  /* 8: sample when step_count % 8 == 0 (orca.py:107) */
} tb2_orca_params;

/* Replaces rvo2.PyRVOSimulator + the doStep/setAgentPrefVelocity loop (orca.py:90-119).
 *   pos_dev [A,2] float, vel_dev [A,2] float (RVO2 is float), goal_dev [A,2] double,
 *   speed_dev [A] double (initial speed; maxSpeed = 1.3 x, pref-velocity clip; orca.py:36,116)
 *   out_dev [n_samples, A, 2] float, n_samples = n_steps / sample_every */
int tb2_orca_simulate(const tb2_layout* layout, const tb2_orca_params* p, const float* pos_dev,
                      const float* vel_dev, const double* goal_dev, const double* speed_dev,
                      float* out_dev, void* stream);

/* Parameter sweeps: every scene under every setting in one call, only the primary's ADE / FDE written
 * (socialforce_eval.py's per-setting re-runs, :236-258, and Evaluator.aggregate's scoring, :25-84).  Work item = (scene,
 * setting); one CTA per scene runs all its settings, scenes of <= 32 pedestrians packed several settings per warp.  The
 * rollout is exactly the one of tb2_sf_simulate / tb2_orca_simulate with that setting (same step code).  Scene b's
 * pedestrian 0 is its primary:
 *   ade_out[s * B + b] = (sum over samples j, in order, of |truth_j - position_j|) / n_samples   (float64)
 *   fde_out[s * B + b] = |truth_last - position_last|
 * truth_dev [B, truth_len, 2] double: the primary's true positions; its last n_samples rows are compared.  NaN propagates
 * (a social-force primary standing on its destination has a NaN desired direction: its ADE is NaN).  No atomics: reruns
 * are bit-identical.  Synchronous on `stream` up to the launch: the P x 3 parameters are read back to be checked.
 * TB2_ERR_INVALID for P < 1, P x B >= 2^31, a non-finite parameter, truth_len < n_samples, and the non-positive values
 * named below.
 *   tb2_sf_sweep    params_dev [P, 3] double = tau (> 0), v0, sigma (> 0); the other fields from `p`
 *   tb2_orca_sweep  params_dev [P, 3] float = neighbor_dist, time_horizon (> 0), radius (> 0); the other fields from
 *                   `p`; positions widened to double before the difference (orca.py's astype(np.float64)) */
int tb2_sf_sweep(const tb2_layout* layout, const tb2_sf_params* p, const double* params_dev, int32_t P,
                 const double* state_dev, const double* truth_dev, int32_t truth_len, double* ade_out_dev,
                 double* fde_out_dev, void* stream);
int tb2_orca_sweep(const tb2_layout* layout, const tb2_orca_params* p, const float* params_dev, int32_t P,
                   const float* pos_dev, const float* vel_dev, const double* goal_dev, const double* speed_dev,
                   const double* truth_dev, int32_t truth_len, double* ade_out_dev, double* fde_out_dev, void* stream);

/* tb2_sf_sweep with the derivatives of every item's ADE / FDE with respect to its setting (forward mode: each quantity
 * of the rollout carries its partials d/d(tau, v0, sigma) as float64 duals).  Same arguments as tb2_sf_sweep, plus
 *   dade_out_dev [P, B, 3], dfde_out_dev [P, B, 3] double: d/d(tau, v0, sigma) of ade_out[s * B + b] / fde_out[s * B + b]
 * ade_out / fde_out equal tb2_sf_sweep's bit for bit (the values are the same operations in the same order).  The
 * field-of-view weight and the speed clip are piecewise: their tangent is that of the branch the value takes.  A
 * non-finite ADE has non-finite derivatives.  No atomics: reruns are bit-identical.  TB2_ERR_INVALID as tb2_sf_sweep,
 * and for a scene of more than 256 pedestrians (the tangent rollout's register budget), before any launch. */
int tb2_sf_sweep_grad(const tb2_layout* layout, const tb2_sf_params* p, const double* params_dev, int32_t P,
                      const double* state_dev, const double* truth_dev, int32_t truth_len, double* ade_out_dev,
                      double* fde_out_dev, double* dade_out_dev, double* dfde_out_dev, void* stream);

/* Kalman predictor, HOST code (BASELINE configs[0] is CPU-only), float64.  Replaces
 * pykalman.KalmanFilter(...).em / .smooth / expected .sample rollout (classical/kalman.py:40-60).
 *   obs_host            [total_obs, 2] observed positions of all tracks, concatenated
 *   track_offsets_host  [n_tracks + 1]
 *   pred_out_host       [n_tracks, n_predict, 2] expectation C A^k x_last, k = 1..n_predict
 *   q_out_host [n_tracks,4,4], r_out_host [n_tracks,2,2], last_state_out_host [n_tracks,4]:
 *   fitted noise covariances / last smoothed state (optional, NULL to skip) so the caller can
 *   add the reference's mean-of-5 sampled noise (kalman.py:53-60). */
int tb2_kalman_predict(const double* obs_host, const int64_t* track_offsets_host, int32_t n_tracks,
                       int32_t n_predict, int32_t em_iterations, double* pred_out_host,
                       double* q_out_host, double* r_out_host, double* last_state_out_host);

/* The same predictor on the device: one thread per track runs the EM / smoother code of tb2_kalman_predict (shared
 * source, no FMA contraction on either side), so pred (without noise), q, r and last state equal the host's bit for bit.
 *   obs_dev [total_obs, 2], track_offsets_dev [n_tracks + 1]; track_offsets_host: the same offsets on the host, checked
 *   before the launch (TB2_ERR_INVALID for a track of fewer than 2 observations, like the host; nothing is launched).
 *   eps_dev [n_tracks, n_predict, 6] standard normals (4 transition + 2 observation per step) or NULL.  With eps_dev and
 *   n_samples >= 1, pred gets the noise of the mean of n_samples sampled rollouts (kalman.py:53-60), i.e. one rollout
 *   driven by Q / n_samples and R / n_samples (Cholesky factors with a zero-pivot guard; z_0 dropped like the
 *   reference's [1:]); eps_dev = NULL or n_samples = 0: the expectation.
 *   pred_out_dev [n_tracks, n_predict, 2]; q_out_dev [n_tracks,4,4], r_out_dev [n_tracks,2,2],
 *   last_state_out_dev [n_tracks,4] optional (NULL to skip).  A track whose predicted covariance is singular (the
 *   host's error) gets NaN in every output.
 *   workspace_dev: caller-owned, >= tb2_kalman_workspace_bytes(track_offsets_host, n_tracks) bytes
 *   (T_max x 76 doubles per track: the smoother's per-step arrays, interleaved over the tracks).
 * Asynchronous on `stream`; n_tracks = 0 launches nothing. */
size_t tb2_kalman_workspace_bytes(const int64_t* track_offsets_host, int32_t n_tracks);
int tb2_kalman_predict_device(const double* obs_dev, const int64_t* track_offsets_host,
                              const int64_t* track_offsets_dev, int32_t n_tracks, int32_t n_predict,
                              int32_t em_iterations, int32_t n_samples, const double* eps_dev,
                              double* pred_out_dev, double* q_out_dev, double* r_out_dev,
                              double* last_state_out_dev, void* workspace_dev, size_t workspace_bytes,
                              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TRAJNET_B200_H */
