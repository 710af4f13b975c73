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

#define TB2_PHASE_ENCODER 0
#define TB2_PHASE_DECODER 1

const char* tb2_last_error(void);
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
    int32_t hidden_dim;      /* LSTM hidden_dim (128)                              */
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
 *   h_in/c_in -> h_out/c_out [M, H] (may alias); absent tracks keep their state
 *   normal_out_dev   [M, 5]  (mu_x, mu_y, sigma_x, sigma_y, rho), NaN rows for absent tracks
 *   pos_out_dev      [M, 2]  obs2 + mu (lstm.py:232,255), may be NULL */
int tb2_lstm_step_forward(const tb2_lstm* model, const tb2_layout* layout, int32_t phase,
                          const float* obs1_dev, const float* obs2_dev,
                          const float* h_in_dev, const float* c_in_dev,
                          float* h_out_dev, float* c_out_dev,
                          float* normal_out_dev, float* pos_out_dev,
                          void* workspace_dev, size_t workspace_bytes, void* stream);

/* Whole time loop: replaces LSTM.forward (lstm.py:170-264) including the decoder input rule
 * (lstm.py:240-250).
 *   observed_dev  [obs_length, M, 2]
 *   truth_dev     [n_decode, M, 2] teacher-forcing positions (prediction_truth) or NULL for a
 *                 free-running rollout (n_predict = n_decode + 1)
 *   normals_out_dev   [S, M, 5],  S = obs_length - 1 + n_decode
 *   positions_out_dev [S, M, 2]
 *   h_dev, c_dev  [M, H] state buffers: zeroed by the call, hold the final state on return.
 *   states_out_dev optional [S, 2, M, H] (h, c after every step; training) or NULL. */
int tb2_lstm_forward_sequence(const tb2_lstm* model, const tb2_layout* layout,
                              const float* observed_dev, int32_t obs_length,
                              const float* truth_dev, int32_t n_decode,
                              float* normals_out_dev, float* positions_out_dev,
                              float* h_dev, float* c_dev, float* states_out_dev,
                              void* workspace_dev, size_t workspace_bytes, void* stream);

/* The same time loop for callers whose results live in HOST memory (the reference's predictor / evaluator
 * boundary hands numpy arrays back): after every recurrence step the step's slices of normals / positions are
 * copied to the pinned host buffers on `copy_stream`, ordered behind the step by an event, while the later
 * steps compute -- the device-to-host traffic (S x M x 28 bytes) hides under the forward instead of following
 * it.  The call does not synchronise: results are complete once `copy_stream` is.  normals_host / positions_host
 * [S, M, 5] / [S, M, 2] must be page-locked; the device outputs are written as well. */
int tb2_lstm_forward_sequence_host(tb2_lstm* model, const tb2_layout* layout,
                                   const float* observed_dev, int32_t obs_length,
                                   const float* truth_dev, int32_t n_decode,
                                   float* normals_out_dev, float* positions_out_dev,
                                   float* h_dev, float* c_dev,
                                   void* workspace_dev, size_t workspace_bytes,
                                   float* normals_host, float* positions_host,
                                   void* stream, void* copy_stream);

/* Steps [first_step, last_step) of the same time loop (S = obs_length - 1 + n_decode steps in all).
 * first_step = 0 starts from the zero state; otherwise h_dev / c_dev hold the state after step
 * first_step - 1 -- possibly edited by the caller in between, which is how the S-GAN generator
 * injects noise between encoder and decoder (sgan/sgan.py:200-221,373) -- and positions_out_dev
 * holds the positions of the earlier steps.  tb2_lstm_forward_sequence == steps [0, S). */
int tb2_lstm_forward_steps(const tb2_lstm* model, const tb2_layout* layout,
                           const float* observed_dev, int32_t obs_length,
                           const float* truth_dev, int32_t n_decode, int32_t first_step, int32_t last_step,
                           float* normals_out_dev, float* positions_out_dev,
                           float* h_dev, float* c_dev, float* states_out_dev,
                           void* workspace_dev, size_t workspace_bytes, void* stream);

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

/* ---------------------------------------------------------------------------------------
 * Training: backward of the whole time loop (what autograd does for Trainer.train_batch,
 * lstm/trainer.py:229-269, through LSTM.forward).  Gradient accumulators are fp32 device
 * buffers in the reference's parameter layout (+=, caller zeroes them).
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
} tb2_lstm_grads;

/* scratch for tb2_lstm_sequence_backward: per (step, active row) records + per-step buffers */
size_t tb2_lstm_backward_workspace_bytes(const tb2_lstm* model, const tb2_layout* layout, int32_t num_active,
                                         int32_t num_steps);

/* BPTT over the rows that receive gradient.
 *   weights          the same fp32 parameter pointers given to tb2_lstm_set_weights
 *   observed/truth   inputs of the forward call (truth: teacher forcing or NULL)
 *   positions_dev    [S, M, 2] and states_dev [S, 2, M, H]: outputs of tb2_lstm_forward_sequence
 *   d_normals_dev    [S, M, 5] upstream gradient wrt rel_pred_scene (d pred_scene already added to
 *                    its first two columns by the caller: pred = obs2 + mu, lstm.py:232,255)
 *   active_rows_dev  int32 [num_active]: tracks with a non-zero upstream gradient (PredictionLoss
 *                    touches the scene primaries only, lstm/loss.py:57,67)
 * Supported: vanilla, occupancy / directional pooling with a one_layer embedding (the D-LSTM
 * training config), and social pooling with a one_layer / two_layer embedding (constant = 0).
 * Social pooling couples all tracks of a scene through the hidden-state scatter (the reference
 * does not detach hidden_states_to_pool, lstm.py:26): the backward then runs on all M rows and
 * active_rows is ignored. */
int tb2_lstm_sequence_backward(const tb2_lstm* model, const tb2_layout* layout, const tb2_lstm_weights* weights,
                               const float* observed_dev, int32_t obs_length, const float* truth_dev,
                               int32_t n_decode, const float* positions_dev, const float* states_dev,
                               const float* d_normals_dev, const int32_t* active_rows_dev, int32_t num_active,
                               const tb2_lstm_grads* grads, void* workspace_dev, size_t workspace_bytes,
                               void* bwd_workspace_dev, size_t bwd_workspace_bytes, void* stream);

/* TB2_POOL_NN_LSTM / TB2_POOL_TRAJECTRON: zero the interaction-encoder LSTM state kept in `workspace`
 * (NearestNeighborLSTM.reset, non_gridbased_pooling.py:385-389; TrajectronPooling.reset, :481-485).  tb2_lstm_forward_sequence / _steps(first_step = 0) do this themselves; the
 * stand-alone plug (tb2_pool_forward) advances the state on every call and needs it after a reset().  No-op for the
 * other pool types. */
int tb2_pool_state_reset(const tb2_lstm* model, const tb2_layout* layout, void* workspace_dev, size_t workspace_bytes,
                         void* stream);

/* Training forward that keeps, per step, what the social backward would otherwise recompute (winners, latent vectors,
 * hidden1 and the pooled vector of the grid embedding; reference: everything autograd saves inside
 * GridBasedPooling.forward, lstm/gridbased_pooling.py:94-170,308-335).  tb2_lstm_train_cache_bytes returns 0 for
 * configurations without a cache (then use tb2_lstm_forward_sequence / tb2_lstm_sequence_backward); `cache` is a
 * caller-owned device buffer that must stay untouched until tb2_lstm_sequence_backward_cached has run. */
size_t tb2_lstm_train_cache_bytes(const tb2_lstm* model, const tb2_layout* layout, int32_t num_steps);
int tb2_lstm_forward_sequence_train(const tb2_lstm* model, const tb2_layout* layout, const float* observed_dev,
                                    int32_t obs_length, const float* truth_dev, int32_t n_decode, float* normals_out_dev,
                                    float* positions_out_dev, float* h_dev, float* c_dev, float* states_out_dev,
                                    void* cache_dev, size_t cache_bytes, void* workspace_dev, size_t workspace_bytes,
                                    void* stream);
int tb2_lstm_sequence_backward_cached(const tb2_lstm* model, const tb2_layout* layout, const tb2_lstm_weights* weights,
                                      const float* observed_dev, int32_t obs_length, const float* truth_dev,
                                      int32_t n_decode, const float* positions_dev, const float* states_dev,
                                      const float* d_normals_dev, const int32_t* active_rows_dev, int32_t num_active,
                                      const tb2_lstm_grads* grads, void* workspace_dev, size_t workspace_bytes,
                                      void* bwd_workspace_dev, size_t bwd_workspace_bytes, const void* cache_dev,
                                      size_t cache_bytes, void* stream);

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
 *   frame [B, 4] = centre x, centre y, cos(-rotation), sin(-rotation), then + centre; xy_out float64 [S, M, 2]. */
int tb2_scenes_drop_distant(const double* xy_dev, const int32_t* scene_off_dev, int32_t T, int32_t M, int32_t B,
                            double r_squared, uint8_t* keep_out_dev, int32_t* kept_count_out_dev, void* stream);
int tb2_scenes_transform(const double* xy_dev, const int32_t* scene_off_dev, const uint8_t* keep_dev,
                         const int32_t* out_off_dev, int32_t T, int32_t M, int32_t M_out, int32_t B,
                         const double* frame_dev, const double* aug_dev, float* xy_out_dev, void* stream);
int tb2_scenes_inverse(const float* xy_dev, const int32_t* scene_off_dev, int32_t S, int32_t M, int32_t B,
                       const double* frame_dev, double* xy_out_dev, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* TRAJNET_B200_H */
