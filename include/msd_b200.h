/* msd_b200.h -- C ABI of libmsd_b200.so: the H100 (sm_90a) implementation of the DDPM
 * sampling hot path of magenta/music-spectrogram-diffusion.
 *
 * The reference has no FFI/plugin layer (it is pure Python on JAX/XLA); the drop-in boundary
 * is the Python protocol of `inference.InferenceModel` (music_spectrogram_diffusion/
 * inference.py:68-203).  These entry points are what a binding for that protocol binds; each
 * one names the reference code it replaces.  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions: every function returns 0 on success, a negative code on failure
 * (-1 bad argument / unsupported configuration, -2 CUDA error, -3 missing weight);
 * `msd_last_error()` returns a thread-local message.  Pointers documented "device" are CUDA
 * device pointers owned by the caller; "host" are ordinary host pointers.  A context is bound
 * to one GPU and one stream at a time and is not thread-safe.  `stream` is a cudaStream_t
 * passed as void* (NULL = legacy default stream).
 */
#ifndef MSD_B200_H_
#define MSD_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MSD_B200_ABI_VERSION 6

typedef struct msd_ctx msd_ctx;

/* Static model + sampler description.
 * Mirrors network.T5Config (models/diffusion/network.py:54-72), the task feature lengths
 * (gin/tasks/mt3/context_mega.gin:5), diffusion_utils.DiffusionConfig/SamplerConfig
 * (models/diffusion/diffusion_utils.py:25-59) and the MelGAN codec constants
 * (audio_codecs.py:204-213). */
typedef struct msd_config {
  int32_t vocab_size;            /* T5Config.vocab_size (1536 for the mt3 vocabulary) */
  int32_t emb_dim;               /* multiple of 128, <= 1024 */
  int32_t num_heads;
  int32_t head_dim;              /* must be 64 */
  int32_t num_encoder_layers;
  int32_t num_decoder_layers;
  int32_t mlp_dim;               /* gated ('gelu','linear') MLP; multiple of 64 */
  int32_t inputs_length;         /* token positions, multiple of 128 */
  int32_t targets_length;        /* mel frames per segment, multiple of 128 */
  int32_t context_length;        /* context frames, multiple of 128 */
  int32_t n_dims;                /* mel bins, must be 128 */
  int32_t num_steps;             /* sampler schedule num_steps */
  int32_t max_batch;             /* segments per call (B) */
  int32_t sampler;               /* 0 = ddpm, 1 = ddim */
  int32_t logvar_type;           /* 0 = large, 1 = small, 2 = 'medium:<logvar_frac>' (ddpm only) */
  int32_t clip_x0;               /* SamplerConfig.clip_x0 */
  int32_t context_positions;     /* 0 = regular, 1 = terminal_relative */
  float max_decoder_noise_time;  /* T5Config.max_decoder_noise_time (2e4) */
  float eval_condition_weight;   /* classifier-free guidance weight; 1 disables the 2nd pass */
  float feature_min;             /* codec min_value (log 1e-5) */
  float feature_max;             /* codec max_value (4.0) */
  /* ABI 2: sampler variants of diffusion_utils.py (all 0 = the shipped gin defaults) */
  int32_t model_output;          /* DiffusionConfig.model_output: 0 eps, 1 x0, 2 v (288-321) */
  int32_t sampler_schedule;      /* sampler.schedule.name: 0 cosine, 1 linear (166-202) */
  int32_t train_schedule;        /* train_schedule.name: 0 cosine, 1 linear */
  int32_t train_num_steps;       /* train_schedule.num_steps (linear only) */
  float logvar_frac;             /* frac of 'medium:<frac>' (141-156) */
  float sampler_beta_start;      /* linear sampler schedule: beta range */
  float sampler_beta_stop;
  float train_beta_start;        /* linear train schedule: beta range */
  float train_beta_stop;
  int32_t cross_attend_style;    /* T5Config.decoder_cross_attend_style: 0 concat_encodings,
                                    1 sum_cross_attends (network.py:199-216) */
  int32_t rng_kind;              /* noise when msd_sample gets no init_z / noise: 0 = Philox4x32-10
                                    (library stream), 1 = jax.random threefry2x32 stream of
                                    PRNGKey(seed) / fold_in(key, i) (inference.py:203,
                                    diffusion_utils.py:389-390, 462) */
  /* ABI 3 */
  int32_t precision;             /* T5Config.dtype as executed: 0 = bf16 tensor-core operands with
                                    fp32 accumulation / residual / softmax (the fast path);
                                    1 = fp32-accurate: every dense layer as a 3 x bf16 split-
                                    precision tensor-core product (~2^-16 per product), fp32
                                    attention, exact tanh -- what the shipped gins ask for
                                    (gin/models/diffusion/context/t5_base.gin:72 dtype float32) */
} msd_config;

/* A named fp32 parameter in the reference's own layout (flax tree path joined by '/',
 * kernels [in, out]); see SURVEY.md App. B. */
typedef struct msd_tensor {
  const char* name;
  const float* data; /* host pointer */
  int32_t ndim;
  int64_t shape[4];
} msd_tensor;

const char* msd_last_error(void);
int msd_abi_version(void);

/* Replaces InferenceModel.__init__'s model construction (inference.py:71-111). */
int msd_create(const msd_config* cfg, int device, msd_ctx** out);
void msd_destroy(msd_ctx* ctx);

/* Replaces InferenceModel._restore_from_checkpoint (inference.py:159-176): takes the fp32
 * parameter tree, repacks it into the kernel layouts (bf16 [out, in], fused QKV / gated-MLP /
 * split-precision projections) and tabulates the timestep conditioning for all num_steps
 * (network.py:377-394 + layers.py:652-666: FiLM scale|bias for every (step, layer)). */
int msd_load_weights(msd_ctx* ctx, const msd_tensor* tensors, int32_t n);

/* Replaces ContextDiffusionModel.predict_batch_with_aux's scale_features + module.encode
 * (models/diffusion/models.py:361-371; network.py:537-559) and additionally projects the
 * concatenated encodings to every decoder layer's cross-attention K/V once (network.py:217-230
 * is loop-invariant).  tokens [B, inputs_length] int32, ctx_features [B, context_length,
 * n_dims] f32 in codec feature units, ctx_mask [B, context_length] int32: device pointers. */
int msd_encode(msd_ctx* ctx, const int32_t* tokens, const float* ctx_features,
               const int32_t* ctx_mask, int32_t batch, void* stream);

/* Replaces diffusion_utils.eval_scan + scale_to_features (diffusion_utils.py:456-476;
 * models.py:393-395) for the batch passed to the preceding msd_encode.
 * init_z  [B, targets_length, n_dims] f32 device, or NULL -> Philox N(0,1) from `seed`.
 * noise   [num_steps, B, targets_length, n_dims] f32 device (noise[i] is used at step i),
 *         or NULL -> Philox from `seed`.
 * mel_out [B, targets_length, n_dims] f32 device, codec feature units. */
int msd_sample(msd_ctx* ctx, const float* init_z, const float* noise, uint64_t seed,
               float* mel_out, void* stream);

/* As msd_sample with generated noise, but row b of the batch of the preceding msd_encode draws
 * init_z and every step's noise from seeds[b] alone (host array of cur_batch entries): exactly
 * the draws msd_sample(seeds[b]) makes at batch 1.  This lets several songs share one batch
 * (one song per row, beam/evaluation.py:156-223 runs each song on its own with predict(batch),
 * inference.py:203) without a song's audio depending on which other songs share its batch or
 * which row it sits in.  The same captured step graph serves msd_sample; rng_kind selects the
 * stream as there.  Refused (-1) without a preceding msd_encode or with a peer attached
 * (msd_p2p_attach). */
int msd_sample_rows(msd_ctx* ctx, const uint64_t* seeds, float* mel_out, void* stream);

/* ---- one song on two GPUs: classifier-free guidance split (BASELINE config 5, SURVEY 8e-iii) ----
 * The two decoder passes of a reverse step (diffusion_utils.py:415, 428-429) are independent until
 * the guidance combine (430-433).  With a peer attached, a context runs ONE of them (role 1: the
 * conditional pass incl. cross-attention, role 2: the unconditional one) and its sampler kernel
 * exchanges the 128 KB of predicted noise with the peer by direct NVLink stores plus a flag word
 * (no NCCL call, no host involvement inside the loop); both GPUs then apply the identical update,
 * so both hold the same z and the same final mel.  Protocol: each process calls msd_p2p_export,
 * the 64-byte handles are swapped by any host channel (torch.distributed in distributed.py), each
 * calls msd_p2p_attach with the OTHER rank's handle, and then both make the same msd_encode /
 * msd_sample calls.  The processes must live on one node with peer access between the GPUs. */
int msd_p2p_export(msd_ctx* ctx, void* handle_out /* 64 bytes */);
int msd_p2p_attach(msd_ctx* ctx, const void* peer_handle /* 64 bytes */, int32_t role);
int msd_p2p_detach(msd_ctx* ctx);

/* Test hook == module.decode (network.py:561-573) at diffusion step `step_i`
 * (time = (step_i + 1) / num_steps): z [B, targets_length, n_dims] f32 device ->
 * eps_out [B, ...] f32 device.  conditioned = 0 multiplies encodings and masks by 0
 * (models.py:376-377). */
int msd_decode_eps(msd_ctx* ctx, const float* z, int32_t step_i, int32_t conditioned,
                   float* eps_out, void* stream);

/* Test hook: copies the encoder outputs of the last msd_encode as bf16-rounded f32:
 * enc_out [B, inputs_length + context_length, emb_dim] device f32. */
int msd_get_encodings(msd_ctx* ctx, float* enc_out, void* stream);

/* Host copy of the per-step sampler scalars [num_steps][16]:
 * 0 x0_scale, 1 eps_scale (predict_x0_from_eps at the sampler's logsnr_t), 2 c_z, 3 c_x0,
 * 4 sigma (ddpm: mean = c_z z + c_x0 x0, std sigma; ddim: 2 = stdv_s, 3 = alpha_s),
 * 5 is_last, 6 logsnr_t, 7 logsnr_s, 8 p0, 9 p1 (eps = p0 z + p1 model_output, train schedule),
 * 10 q0, 11 q1 (x0 = q0 z + q1 model_output, train schedule), 12 e1, 13 e2
 * (predict_eps_from_x0 at logsnr_t: eps = e1 (z - x0 e2)), 14 logsnr_train, 15 reserved. */
int msd_get_step_table(msd_ctx* ctx, float* table_host);

/* The same table for a configuration, without a context or a GPU: validates cfg as msd_create does
 * (-1 when it would refuse it), then writes table_host [cfg->num_steps][16] (host). */
int msd_step_table(const msd_config* cfg, float* table_host);

/* Profiling hook: runs diffusion step `step_i` (1 <= step_i < num_steps) of the batch of the
 * last msd_encode `reps` times WITHOUT graph capture, bracketing every kernel launch with CUDA
 * events on the launching stream.  out[5][4] (doubles), one row per kernel class
 * {0 gemm, 1 attention, 2 rmsnorm/FiLM, 3 sampler, 4 other}:
 * {milliseconds per step, launches per step, algorithmic FLOPs per step, algorithmic bytes per
 * step}.  Leaves the sampler state (z) modified; call msd_sample afterwards as usual. */
int msd_profile_step(msd_ctx* ctx, int32_t step_i, int32_t reps, double* out);

/* Kernel launches issued so far by this library in this process (graph replays count their
 * kernel nodes). */
uint64_t msd_launch_count(void);

/* ---- operator-level entry points (unit parity against msd/layers.py) ------------------- */

/* DenseGeneral (layers.py:397-442): out[M,N] f32 = A[M,K] * W, with A given as bf16-rounded
 * f32 [M,K] device and W as f32 [K,N] host-layout device pointer (packed internally). */
int msd_op_dense(const float* a, const float* w, int32_t M, int32_t N, int32_t K, float* out,
                 void* stream);

/* Same, selecting the tile-width choice: variant 0 = widest tile that fills the SMs (default),
 * 1 = power-of-two widths only; block_n 0 = auto or one of 64/128/192/256 (192 only with variant 0). */
int msd_op_dense_variant(const float* a, const float* w, int32_t M, int32_t N, int32_t K,
                         float* out, int32_t variant, int32_t block_n, void* stream);

/* Micro-benchmark hook: average milliseconds of `iters` back-to-back launches of the bf16 GEMM
 * [M,K] x [N,K]^T with the given epilogue (0 bf16, 1 f32, 2 f32 + residual, 3 gated-GELU) on
 * zero-filled scratch buffers. */
int msd_bench_gemm(int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t variant,
                   int32_t block_n, int32_t iters, float* ms_out);

/* Micro-benchmark hook: average milliseconds of `iters` back-to-back launches of the bf16
 * attention kernel (+ its combine kernel when the keys are split) on scratch
 * buffers filled with small pseudo-random values; kv_static as in the decoder's cross-attention.
 * The instance / split is chosen as in production (or forced by MSD_ATTN_BKV / _SPLITS). */
int msd_bench_attention(int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, int32_t iters,
                        float* ms_out);

/* dot_product_attention (layers.py:109-181) for head_dim 64 with a key-padding mask:
 * q [nb, Lq, heads*64], k/v [nb, Lk, heads*64] f32 device, key_mask [nb, Lk] int32 or NULL,
 * out [nb, Lq, heads*64] f32 device. */
int msd_op_attention(const float* q, const float* k, const float* v, const int32_t* key_mask,
                     int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, float* out, void* stream);

/* DenseGeneral with each fused epilogue of the hot path (kernels.h GemmEpilogue), for unit parity:
 *   0 bf16 out                      out [M, N]            = bf16(a w)
 *   2 f32 + residual                out [M, N]            = a w + resid [M, N]
 *   3 gated GELU (layers.py:483-509) out [M, N]           = bf16(gelu_tanh(a w) * (a w1)), w / w1 [K, N]
 *   4 f32 + position rows           out [M (+ dup), N]    = a w + pos[(r % pos_rows - shift[r /
 *                                    pos_rows]) mod pos_rows] (network.py:327-334, 420-427), rows
 *                                    also stored at r + dup_rows when dup_rows > 0
 *   5 gated GELU, fp32-accurate     out [M, N]            = hi + lo of the [hi | lo | hi] output,
 *                                    computed from 3 x bf16 split operands (a, w, w1 used in full
 *                                    fp32 precision)
 * a [M, K], w [K, N] f32 device (bf16-rounded by the caller for epilogues 0-4); block_n 0 = auto.
 * Unused pointers may be NULL.  out is f32 device. */
int msd_op_dense_epilogue(const float* a, const float* w, const float* w1, int32_t M, int32_t N,
                          int32_t K, int32_t epilogue, int32_t block_n, const float* resid,
                          const float* pos, int32_t pos_rows, const int32_t* pos_shift,
                          int32_t dup_rows, float* out, void* stream);

/* The deferred-normalisation pair of the bf16 hot path (DESIGN section 5): a residual projection
 * whose epilogue also prepares the next pre-norm, and the projection that consumes it.
 *   stage 1   x_out [M, d] = x + a w_out;  operand = bf16(x_out * g(row)), g = g_lo for rows <
 *             split_row, else g_hi;  row sums of squares of x_out kept per column tile
 *   stage 2   y [M, N2] = bf16(rsqrt(mean(x_out^2) + 1e-6)[row] * (operand w2) + bias)     (w2b NULL)
 *             y = bf16(gelu_tanh(u) * u1), u | u1 the same through w2 | w2b                (gated)
 * i.e. y == bf16((rmsnorm(x_out) * g) w2 + bias) up to operand rounding (layers.py:632-666 with
 * g = scale * (1 + film_scale), bias = film_bias w2).  a [M, K], w_out [K, d], x [M, d], g_* [d],
 * w2 / w2b [d, N2], bias [N2] (gated: [2 * N2] in accumulator column order: 32 of w2, 32 of w2b,
 * ...) or NULL; all f32 device, a / w_out / w2 / w2b bf16-rounded by the callee.  block_n1 /
 * block_n2: tile widths of the two GEMMs (0 = auto).  Outputs f32 device. */
int msd_op_dense_deferred_norm(const float* a, const float* w_out, const float* x, int32_t M, int32_t d,
                               int32_t K, const float* g_lo, const float* g_hi, int32_t split_row,
                               const float* w2, const float* w2b, int32_t N2, const float* bias,
                               int32_t block_n1, int32_t block_n2, float* x_out, float* y_out,
                               void* stream);

/* dot_product_attention of the fp32-accurate mode: as msd_op_attention, but q / k / v are used in
 * full fp32 and the result is returned as hi + lo of the kernel's [hi | lo | hi] output. */
int msd_op_attention_f32(const float* q, const float* k, const float* v, const int32_t* key_mask,
                         int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, float* out,
                         void* stream);

/* The attention kernel on caller-owned device buffers, launched the way the engine launches it
 * (views into fused / cached buffers).  precision 0: bf16 q / k / v and the tensor-core kernel;
 * 1: fp32 q / k / v and the fp32 kernel.
 *   q / k / v   element offset + leading dimension (elements); head h reads columns h*64 .. +64 of
 *               the view.  Q rows [nb * Lq]; K / V row of batch b, key j: b * kv_batch_rows +
 *               kv_row0 + j (kv_batch_rows 0 = Lk).  k and v may be the same buffer.
 *   key_mask    int32 [nb, mask_len] (> 0 = attend) or NULL; packed to mask_len / 32 words per row,
 *               the attention reads words [mask_word0, mask_word0 + Lk / 32) of each row.
 *   kv_static   bf16 mode: K / V and the mask are read ahead of the programmatic-dependency wait.
 *               The hook completes all prior work on the stream, then rewrites the Q view (same
 *               values) with a kernel of its own and launches the attention right behind it.
 *   out         bf16; head h of row r written at out[o_col + r * o_ld + h*64 ..] (precision 0), or
 *               as [hi | lo | hi] at out[o_col + r * 3 * o_ld + {0, o_ld, 2 o_ld} + h*64 ..]
 *               (precision 1: o_ld is the width of one third).  Nothing else is written.
 *   part_o / part_ml  split-KV workspace for up to 12 splits: f32 [nb * Lq * heads * 12 * 64] and
 *               [nb * Lq * heads * 12 * 2].
 *   splits      0 = automatic, else forced (<= 12); tail (bf16 only): > 0 moves the last `tail`
 *               key blocks of an unsplit 128-key launch to a second CTA, 0 = none.
 * The key-block size follows MSD_ATTN_BKV as in the engine.  Synchronises the stream. */
int msd_op_attention_view(int32_t precision, void* q, int64_t q_off, int32_t ldq, const void* k,
                          int64_t k_off, int32_t ldk, const void* v, int64_t v_off, int32_t ldv,
                          int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, int32_t kv_batch_rows,
                          int32_t kv_row0, const int32_t* key_mask, int32_t mask_len,
                          int32_t mask_word0, int32_t kv_static, void* out, int64_t o_col,
                          int32_t o_ld, float* part_o, float* part_ml, int32_t splits, int32_t tail,
                          void* stream);

/* The GEMM on caller-owned device buffers, launched with every argument the engine's decoder sets
 * (views into fused buffers, step-indexed tables, deferred normalisation):
 *   a, b        bf16 operands as element offset + leading dimension: out = A[M, K] B[N, K]^T.
 *   epilogue    0 bf16, 1 f32, 2 f32 + resid, 3 gated GELU (bf16 [M, N / 2]), 4 f32 + position rows,
 *               5 gated GELU split [hi | lo | hi] (bf16 [M, 3 N / 2]), 6 deferred-normalisation
 *               producer (out == resid, f32 in place; see msd_op_dense_deferred_norm).
 *   block_n     0 = automatic, else 64 / 96 / 128 / 192 / 256; variant as in msd_op_dense_variant.
 *   out         f32 (epilogues 1, 2, 4, 6) or bf16 (0, 3, 5) at element offset out_off, row stride ldo;
 *               resid f32 at resid_off with the same ldo, or NULL.
 *   pos / pos_rows / pos_shift / dup_rows   epilogue 4, as in msd_op_dense_epilogue.
 *   step        device int32 diffusion step index the *_step_stride arguments multiply, or NULL.
 *   prep_*      epilogue 6: column gains g_lo (rows < prep_split_row) / g_hi at base + step * stride,
 *               bf16 operand written to prep_a [M, prep_lda], row sums of squares of each column tile
 *               t written to prep_ss[t * prep_ss_stride + row].
 *   rs_*        epilogues 0 / 3 (rs_ss_lo != NULL): row r's accumulator is scaled by
 *               rsqrt(inv_d * sum_{t < parts} ss[t * rs_ss_stride + r] + 1e-6), ss / parts = the _lo
 *               pair for r < rs_split_row, else the _hi pair; then rs_col_bias + step * stride is added.
 * *block_n_out (host, may be NULL) receives the tile width that ran: epilogue 6 writes N / width
 * partial sums per row.  The launch waits for all earlier work on the stream; synchronises it. */
int msd_op_gemm_view(const void* a, int64_t a_off, int32_t lda, const void* b, int64_t b_off, int32_t ldb,
                     int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t block_n, int32_t variant,
                     void* out, int64_t out_off, int32_t ldo, const float* resid, int64_t resid_off,
                     const float* pos, int32_t pos_rows, const int32_t* pos_shift, int32_t dup_rows,
                     const int32_t* step, const float* prep_g_lo, int64_t prep_g_lo_step_stride,
                     const float* prep_g_hi, int64_t prep_g_hi_step_stride, int32_t prep_split_row,
                     void* prep_a, int32_t prep_lda, float* prep_ss, int32_t prep_ss_stride,
                     const float* rs_ss_lo, int32_t rs_parts_lo, const float* rs_ss_hi, int32_t rs_parts_hi,
                     int32_t rs_split_row, int32_t rs_ss_stride, float rs_inv_d, const float* rs_col_bias,
                     int64_t rs_bias_step_stride, int32_t* block_n_out, void* stream);

/* The first decoder layer's deferred-normalisation prep (no GEMM produced its stream): a_out bf16
 * [rows, lda] = bf16(x * g), g at g + (*step) * g_step_stride; ss_out[row] = sum of x^2 over the
 * row.  x f32 [rows, d], d = k * 128 <= 1024; step device int32.  Synchronises the stream. */
int msd_op_prep_rows(const float* x, const float* g, int64_t g_step_stride, const int32_t* step, int32_t rows,
                     int32_t d, void* a_out, int32_t lda, float* ss_out, void* stream);

/* Host copies of the load-time conditioning tables (NULL skips one):
 *   film      [num_steps][2 L][2 d]   FiLM scale | bias of each layer's two FiLM layers (j = 2l self,
 *                                     2l + 1 mlp): the time MLP and FiLM dense of every step
 *   gain      [num_steps][2 L][d]     gamma (1 + scale) of the same pre-norms
 *   bias_qkv  [num_steps][L][3 hh]    FiLM bias of the self-attention pre-norm times the packed
 *                                     bf16 QKV weights
 *   bias_wi   [num_steps][L][2 F]     ... of the MLP pre-norm times the packed gated wi weights
 *                                     (columns interleaved 32 of wi_0, 32 of wi_1)
 * The last three exist with deferred normalisation only (bf16 mode); asking for them otherwise
 * is refused (-1). */
int msd_get_conditioning_tables(msd_ctx* ctx, float* film, float* gain, float* bias_qkv, float* bias_wi);

/* The sampler kernel (one reverse step: guidance combine, x0, clip, DDPM / DDIM update, noise) on
 * caller-owned device buffers, with the fields the engine sets (no guidance split, no prefetch):
 *   eps       f32 [passes * n]: the model output of the conditional pass, then the unconditional one
 *   z         f32 [n], updated in place; z_split bf16 [n / n_dims, 3 n_dims] = [hi | lo | hi] of new z
 *   mel_out   f32 [n] or NULL: scale_to_features(z) written at step 0 only
 *   noise     f32 [num_steps, n] (row i read at step i) or NULL: generated from seed (rng_kind 0,
 *             Philox stream i + 1) or rng_keys [num_steps + 1][2] (rng_kind 1, row i + 1)
 *   coef      f32 [num_steps, 16] (msd_get_step_table layout)
 *   per_row   generated noise of row b = idx / n_row from row_seeds[b] (uint64, rng_kind 0) or
 *             row_keys + b * row_key_stride (rng_kind 1): n_row % 8 == 0, n < 2^32
 * step != NULL: the step index is read from that device int32 (one launch, per_row 0).
 * step == NULL: the graph's path.  A device RunArgs {noise, mel_out, seed, step = run_step, per_row}
 * is built, the kernel runs `launches` times behind each other (each launch advances the step), and
 * run_out[0] / run_out[1] (host) receive the RunArgs step and done counter found afterwards.
 * Refused (-1): null z / z_split / eps / coef, n not a positive multiple of n_dims (both multiples of
 * 4), passes other than 1 or 2, the jax stream without keys or with n % 8 != 0 or n >= 2^32, per-row
 * streams without their table or with n_row % 8 != 0 or n >= 2^32, and steps outside the table.
 * Synchronises the stream. */
int msd_op_sampler_step(const float* eps, float* z, void* z_split, float* mel_out, const float* noise,
                        const float* coef, int32_t num_steps, const int32_t* step, int64_t n, int32_t n_dims,
                        int32_t passes, float cond_weight, int32_t clip_x0, int32_t ddim, float feat_min,
                        float feat_max, uint64_t seed, int32_t rng_kind, const uint32_t* rng_keys,
                        int64_t n_row, const uint32_t* row_keys, int64_t row_key_stride,
                        const uint64_t* row_seeds, int32_t run_step, int32_t per_row, int32_t launches,
                        int32_t* run_out, void* stream);

/* The sampler's initial state: z f32 [n] = init_z (device copy) or, with init_z NULL, the draw of
 * Philox stream 0 of seed (rng_kind 0) or of key rng_keys[0..1] (rng_kind 1); n_row > 0: row b's own
 * draw from row_seeds[b] / rng_keys + b * row_key_stride.  z_split as in msd_op_sampler_step.
 * Synchronises the stream. */
int msd_op_init_z(const float* init_z, float* z, void* z_split, int64_t n, int32_t n_dims, uint64_t seed,
                  int32_t rng_kind, const uint32_t* rng_keys, int64_t n_row, int64_t row_key_stride,
                  const uint64_t* row_seeds, void* stream);

/* The encoder's context-feature front end (scale_features(clip=True), audio_codecs.py:166-174):
 * feat f32 [rows, n_dims] -> out_split bf16 [rows, 3 n_dims] = [hi | lo | hi] of
 * 2 (clip(f, feat_min, feat_max) - feat_min) / (feat_max - feat_min) - 1.  Synchronises the stream. */
int msd_op_scale_split(const float* feat, void* out_split, int64_t rows, int32_t n_dims, float feat_min,
                       float feat_max, void* stream);

/* LayerNorm (layers.py:632-649) followed by optional FiLM (layers.py:652-666) with explicit
 * scale|bias vector film [2*d] (NULL = none): out f32 (bf16-rounded) [rows, d]. */
int msd_op_rmsnorm_film(const float* x, const float* gamma, const float* film, int32_t rows,
                        int32_t d, float* out, void* stream);

/* jax.random.normal of the sampler's stream: step < 0 -> normal(PRNGKey(seed), [n]) (init_z,
 * diffusion_utils.py:462), else normal(fold_in(PRNGKey(seed), step), [n]) (389-390).
 * out: device f32 [n], n a multiple of 8.  Test hook for the rng_kind = 1 generator. */
int msd_op_jax_normal(uint64_t seed, int32_t step, int64_t n, float* out, void* stream);

/* The raw threefry2x32 words those normals are made from (jax.random.bits of the same key):
 * out device uint32 [n].  Integer work: the test compares bit-exactly. */
int msd_op_jax_bits(uint64_t seed, int32_t step, int64_t n, uint32_t* out, void* stream);

/* MelGAN.encode (audio_codecs.py:43-143, 204-247): audio [rows, n_samples] f32 device ->
 * mel_out [rows, F, 128] f32 device in codec feature units, F = ceil(n_samples / 320).  Frame k
 * of a row is samples [320 k, 320 k + 640) (zero past the end), times window [640] f32 device
 * (periodic Hann), zero-padded to 1024; out = log(clip(|rfft| @ mel_weights, 1e-5, 1e8)) with
 * mel_weights [513, 128] f32 device (linear_to_mel_weight_matrix(128, 513, 16000, 0, 8000)).
 * Computed in fp32; a frame's output depends on its own 640 samples and the two tables only, so
 * a song encoded whole and sliced equals the song encoded in pieces.  Refused (-1): a null
 * pointer, a negative size, or more than 2^31 - 1 output frames; rows = 0 or n_samples = 0
 * launches nothing.  Asynchronous on `stream`; needs no context. */
int msd_op_audio_mel(const float* audio, int32_t rows, int64_t n_samples, const float* window,
                     const float* mel_weights, float* mel_out, void* stream);

/* Resampling of recordings to the codec's rate as the reference does it (preprocessors.py:150-155,
 * 332-333, 518-521: librosa.resample(y, sr, 16000) and librosa.load(sr=16000), i.e. librosa 0.9
 * res_type='kaiser_best' = resampy 0.2.2 `resample_f`): x [rows, n_in] f32 device -> y [rows,
 * n_out] f32 device, n_out = int(n_in * ((double)target_sr / orig_sr)) (resampy's length; the
 * caller zero-pads to librosa's ceil).  half_window [window_len] f64 device is the unscaled filter
 * half (kaiser_best: 32769 entries), scaled by the ratio when downsampling as resampy does.
 * precision is log2 of the window's entries per zero crossing: 9 for kaiser_best, whose
 * get_filter returns num_table = 2^9 = 512 (resampy passes that to resample_f).  time_segments [n_segments, 3] f64 device
 * (t_s, r_s, d), t_s ascending from 0, describe resampy's running float64 time register: for
 * t_s <= t < t_{s+1}, r_t = r_s + (t - t_s) d exactly (audio_codecs.time_register_segments).
 * Every tap is a float64 multiply and add rounded to float32, in resampy's order: the result is
 * bit for bit the sequential loop's.  Refused (-1): a null pointer, a negative size, a rate <= 0,
 * an n_out other than the length above, more than 65535 rows or 2^31 - 1 samples in or out, a
 * precision outside 0..24, window_len < 2, n_segments < 1, or a ratio below one window entry per
 * input sample.  rows = 0 or n_out = 0 launches nothing.  Asynchronous on `stream`; needs no
 * context. */
int msd_op_audio_resample(const float* x, int32_t rows, int64_t n_in, int32_t orig_sr,
                          int32_t target_sr, const double* half_window, int32_t window_len,
                          int32_t precision, const double* time_segments, int32_t n_segments,
                          float* y, int64_t n_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MSD_B200_H_ */
