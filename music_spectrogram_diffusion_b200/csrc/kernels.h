// Host-side launcher prototypes for the sm_90a kernels (internal to libmsd_b200.so).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

namespace msd {

typedef __nv_bfloat16 bf16;

// Global count of kernel launches issued through the launchers below (a graph
// replay adds its node count).  Reported as bench.py's "gpu_launches".
extern std::atomic<unsigned long long> g_launch_count;

// ---------------------------------------------------------------------------
// Optional per-launch profiling (msd_profile_step): when a recorder is armed every launcher
// brackets its kernel with CUDA events on the launching stream and notes its algorithmic work.
// ---------------------------------------------------------------------------
enum KernelClass : int { KC_GEMM = 0, KC_ATTENTION = 1, KC_NORM = 2, KC_SAMPLER = 3, KC_OTHER = 4,
                         KC_COUNT = 5 };
struct ProfRecorder;
extern ProfRecorder* g_prof;
void prof_begin(int cls, double flops, double bytes, cudaStream_t st);
void prof_end(cudaStream_t st);
struct ProfScope {
  cudaStream_t st;
  bool on;
  ProfScope(int cls, double flops, double bytes, cudaStream_t s) : st(s), on(g_prof != nullptr) {
    if (on) prof_begin(cls, flops, bytes, st);
  }
  ~ProfScope() {
    if (on) prof_end(st);
  }
};

// ---------------------------------------------------------------------------
// Launch helper: cudaLaunchKernelEx with the programmatic-stream-serialization attribute when
// PDL is enabled (default; MSD_PDL=0 disables).  Works under stream capture (programmatic edges).
// ---------------------------------------------------------------------------
extern bool g_use_pdl;
extern thread_local bool g_pdl_skip_next;  // next launch (of this host thread) waits for its predecessor to complete: plain launch
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                 cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (g_use_pdl && !g_pdl_skip_next) ? 1 : 0;
  g_pdl_skip_next = false;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// SMs of the current device (132 on H100 SXM), kept per host thread until it switches devices:
// every tile, split and grid policy sizes its launches from it.  132 when the device cannot be
// queried; the launch that follows then reports the CUDA error.
int device_sm_count();

// ---------------------------------------------------------------------------
// TMA tensor maps (driver entry point fetched at run time; no libcuda link).
// ---------------------------------------------------------------------------
// 2D row-major bf16 matrix [rows, cols] with leading dimension ld (elements);
// box = [box_rows, 64 cols] (128-byte inner extent), SWIZZLE_128B; with inner_bytes = 64,
// box = [box_rows, 32 cols], SWIZZLE_64B.
int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows, int inner_bytes = 128);

// ---------------------------------------------------------------------------
// GEMM: D[M,N] = A[M,K] * B[N,K]^T, bf16 operands (both K-major), fp32 accumulate
// in registers (wgmma.mma_async), TMA-fed smem ring, warp-specialised.
// ---------------------------------------------------------------------------
enum GemmEpilogue : int {
  EPI_BF16 = 0,        // out bf16 [M, ldo] = acc
  EPI_F32 = 1,         // out f32  [M, ldo] = acc
  EPI_RESID_F32 = 2,   // out f32  [M, ldo] = acc + resid[M, ldo]      (in place allowed)
  EPI_GATED_GELU = 3,  // out bf16 [M, N/2]: per 64 acc columns, gelu(acc[0:32]) * acc[32:64]
  EPI_POS_F32 = 4,     // out f32 = acc + pos[(r % pos_rows - shift[r / pos_rows]) mod pos_rows]
                       //   optionally duplicated to out[r + dup_rows]
  EPI_GATED_GELU_SPLIT3 = 5,  // fp32-accurate mode: g = gelu(acc[0:32]) * acc[32:64] with the exact
                              //   tanh, written as bf16 [M, 3 * N/2] = [hi(g) | lo(g) | hi(g)]
                              //   (the A operand of a 3 x bf16 split-precision GEMM)
  EPI_RESID_PREP = 6,  // deferred normalisation, producer side (out == resid):
                       //   x = acc + resid (f32, in place); prep.a[r, :] = bf16(x[r, :] * g(r)[:])
                       //   with g = prep.g_lo for r < prep.split_row else prep.g_hi; and
                       //   prep.ss[tile_n, r] = sum over the tile's columns of x^2
};

// Deferred normalisation (bf16 mode; DESIGN section 5): instead of a stand-alone rmsnorm (+FiLM)
// kernel between a residual projection and the next projection,
//   y = (rmsnorm(x) * gamma * (1 + fs) + fb) W   ==   inv_r[r] * ((x * g') W) + (fb W)
// with g' = gamma (1 + fs) per column and inv_r = rsqrt(mean(x^2) + eps) per row.  The residual
// GEMM that produces x also writes the column-scaled bf16 operand and the row sums of squares
// (GemmPrep); the consuming GEMM scales its accumulator rows and adds the bias row (GemmRowScale).
// Vectors that depend on the diffusion step are addressed as base + (*step) * step_stride.
struct GemmPrep {
  const float* g_lo;        // [N] column scale for rows < split_row
  const float* g_hi;        // [N] column scale for rows >= split_row (may equal g_lo)
  long long g_lo_step_stride, g_hi_step_stride;
  int split_row;
  bf16* a;                  // [M, lda] scaled operand of the next GEMM
  int lda;
  float* ss;                // [N / block_n, ss_stride] partial row sums of squares
  int ss_stride;
};
struct GemmRowScale {
  const float* ss_lo;       // partial sums for rows < split_row: ss_lo[t * ss_stride + r], t < parts_lo
  const float* ss_hi;       // same for rows >= split_row
  int parts_lo, parts_hi, split_row, ss_stride;
  float inv_d;              // 1 / (normalised width)
  const float* col_bias;    // [N] added after the row scale, or null
  long long bias_step_stride;
};

struct GemmArgs {
  const bf16* A;  // [M, lda]
  const bf16* B;  // [N, ldb]   (weights packed [out, in])
  int M, N, K;
  int lda, ldb;
  int epilogue;
  void* out;
  int ldo;
  const float* resid;    // EPI_RESID_F32
  const float* pos;      // EPI_POS_F32: [pos_rows, N]
  int pos_rows;
  const int* pos_shift;  // EPI_POS_F32: per (r / pos_rows) roll amount or nullptr
  int dup_rows;          // EPI_POS_F32: also store to row r + dup_rows when > 0
  int block_n;           // 0 = auto
  long long* trace;      // debugging: per-tile stamps (8 int64 per tile, first 512 tiles), or null
  // deferred normalisation: prep.a != null with EPI_RESID_PREP; rs.ss_lo != null
  // with EPI_BF16 / EPI_GATED_GELU; `step` is the device step index the strides multiply
  GemmPrep prep;
  GemmRowScale rs;
  const int* step;
};
int launch_gemm(const GemmArgs& a, cudaStream_t stream);
int gemm_configure();  // opt in to the kernels' dynamic shared memory sizes (idempotent)
// The tile width launch_gemm(a) runs with: a.block_n when given, else the one that takes the
// fewest tile times on this device's SMs; 0 when that width is not allowed (64 / 128 / 192 / 256,
// and 96 for the fp32-output epilogues) or does not divide N.  Whoever sizes per-tile outputs
// (EPI_RESID_PREP's partial row sums: N / width of them) must take the width from here.
int gemm_resolve_block_n(const GemmArgs& a);

// ---------------------------------------------------------------------------
// Attention: O = softmax(Q K^T + keymask) V, no 1/sqrt(d), head_dim 64.
// Q rows [nbatch*Lq, ldq], K/V rows [nbatch*Lk, ldk/ldv]; head h uses columns
// [h*64, h*64+64).  mask_bits: [nbatch, mask_stride_words] uint32 bit per key
// (1 = attend) or nullptr.  Rows with no attendable key produce 0.
// ---------------------------------------------------------------------------
struct AttnArgs {
  const bf16* Q; int ldq;
  const bf16* K; int ldk;
  const bf16* V; int ldv;
  bf16* O; int ldo;
  int nbatch, heads, Lq, Lk;
  const uint32_t* mask_bits; int mask_stride_words;
  // split-KV workspace (optional): part_o [attention_workspace_floats(..)] f32, part_ml
  // [rows*heads*max_splits*2] f32; splits 0 = choose automatically (attention_pick_splits),
  // capped by max_splits.
  float* part_o; float* part_ml; int splits; int max_splits;
  // tail split of an otherwise unsplit launch of the 128-key instance (needs the workspace):
  // tail > 0 = the last `tail` key blocks go to a second (short) CTA per tile, merged by the
  // combine kernel; <= 0 = none.
  int tail;
  // K, V and mask_bits were written well before the preceding kernel (safe to read ahead of the
  // programmatic-dependency wait): true for the cross-attention over the per-segment K/V cache.
  int kv_static;
  // K/V rows of batch b, key block j start at b * kv_batch_rows + kv_row0 + j * 128
  // (kv_batch_rows 0 = Lk): lets one source of a concatenated [tokens | context] cache be attended.
  int kv_batch_rows, kv_row0;
};
// workspace sizing for part_o (floats) of a launch with up to max_splits splits
size_t attention_workspace_floats(int nbatch, int heads, int Lq, int max_splits);
int attention_pick_splits(int nbatch, int heads, int Lq, int Lk);
int launch_attention(const AttnArgs& a, cudaStream_t stream);
int attention_configure();

// ---------------------------------------------------------------------------
// Row-wise and element-wise kernels
// ---------------------------------------------------------------------------
// y = rmsnorm(x; g) [ * (1 + s) + b ], written as bf16.  s|b = film[(*step) * film_stride +
// film_offset + {0, d}] when film != nullptr.  split3: write [hi | lo | hi] (3*d wide).
int elementwise_configure();
int launch_rmsnorm(const float* x, const float* gamma, int rows, int d, bf16* out, int ldo,
                   const float* film, const int* step, long long film_step_stride,
                   long long film_offset, int split3, cudaStream_t stream);

constexpr int MSD_STEP_COLS = 16;  // floats per diffusion step in the sampler table
// Per-call arguments of msd_sample that live in DEVICE memory, so that the captured step graph does
// not depend on them (a new noise tensor / output buffer / seed does not force a re-capture).
struct RunArgs {
  const float* noise;        // [num_steps, B*N*n_dims] or nullptr -> generator(seed)
  float* mel_out;            // written at step 0
  unsigned long long seed;   // Philox stream (rng_kind 0)
  int step;                  // current reverse-step index i (decremented by the sampler kernel)
  unsigned int done;         // sampler blocks that have finished reading `step` (kept at 0)
  // guidance split across two GPUs: sequence number of the NEXT exchange (identical on both
  // ranks; advanced by the sampler kernel) and the counter of blocks that have sent their share
  unsigned int xseq;
  unsigned int xsent;
  // generated noise drawn per batch row (msd_sample_rows) from SamplerArgs::row_keys / row_seeds
  // instead of one draw over the whole batch (msd_sample sets 0)
  int per_row;
};
struct SamplerArgs {
  const float* eps;       // [(passes*B)*N, n_dims] rows: cond block then uncond block
  float* z;               // [B*N*n_dims] state, updated in place
  bf16* z_split;          // [B*N, 3*n_dims] = [hi | lo | hi] of the new z
  const float* noise;     // [num_steps, B*N*n_dims] or nullptr -> philox(seed)
  const float* coef;      // [num_steps, MSD_STEP_COLS], columns documented at msd_get_step_table
  const int* step;        // device step index i
  float* mel_out;         // written when i == 0: scale_to_features(z)
  long long n;            // B*N*n_dims
  int n_dims;
  int passes;             // 2 with classifier-free guidance, 1 without
  float cond_weight;
  int clip_x0;
  int ddim;               // 1 = ddim_step, 0 = ddpm_step
  float feat_min, feat_max;
  unsigned long long seed;
  // rng_kind 1: jax.random threefry stream; keys [num_steps + 1][2] (row 0 PRNGKey(seed), row
  // i + 1 fold_in(key, i)), device memory
  int rng_kind;
  const uint32_t* rng_keys;
  // per-row streams (run->per_row): element idx of row b = idx / n_row is element idx - b * n_row
  // of an n_row-element draw from row b's own key table row_keys + b * row_key_stride (same layout
  // as rng_keys; rng_kind 1) or Philox seed row_seeds[b] (rng_kind 0): the draws that row would
  // get alone at batch 1.  n_row is a multiple of 8, so a float4 never straddles two rows.
  long long n_row;
  const uint32_t* row_keys;
  long long row_key_stride;
  const unsigned long long* row_seeds;
  // when non-null: noise / mel_out / seed / step are read from here (device memory) instead of the
  // fields above, and the last block to finish decrements run->step (the step advance)
  RunArgs* run;
  // per-step tables [num_steps][pf_step_floats[t]] the decoder layers read (the FiLM table, or the
  // deferred normalisation's column gains and two bias-row tables), unused entries null: the rows
  // of the NEXT step are prefetched into L2 here, so that the next step's kernels do not each wait
  // for HBM (the FiLM table is 147 MB for base, every row is read once per call)
  const float* pf[3]; long long pf_step_floats[3];
  // Classifier-free guidance split over two GPUs (BASELINE config 5, SURVEY 8e-iii): this GPU ran
  // ONE of the two decoder passes (xrole 1: the conditional one, 2: the unconditional one) and
  // `eps` holds its n values.  The kernel stores them into the peer GPU's exchange buffer with
  // plain st.global over NVLink (peer mapping of the other process's allocation), raises the
  // peer's flag, waits for the peer's values in its own buffer and then does the update both
  // GPUs need -- a fused compute + exchange kernel, no NCCL call in the loop.  Exchange buffer
  // layout (floats): [2 parities][n] values, then 2 flag words at xflags_off.
  int xrole;
  float* xlocal;        // this GPU's buffer (the peer writes into it)
  float* xpeer;         // the peer's buffer, mapped into this process
  long long xparity_floats, xflags_off;
};
int launch_sampler_step(const SamplerArgs& a, cudaStream_t stream);

// z0 = init (copy or philox normal), plus its [hi | lo | hi] split.
// rng_kind / rng_keys as in SamplerArgs (keys row 0 is used).  n_row > 0: per-row streams as in
// SamplerArgs, rng_keys then being the per-row table (row_key_stride words per row) and row_seeds
// the per-row Philox seeds.
int launch_init_z(const float* init_z, float* z, bf16* z_split, long long n, int n_dims,
                  unsigned long long seed, cudaStream_t stream, int rng_kind = 0,
                  const uint32_t* rng_keys = nullptr, long long n_row = 0,
                  long long row_key_stride = 0, const unsigned long long* row_seeds = nullptr);

// x[b,t,:] = E[tok[b,t]] + P[t]
int launch_embed_tokens(const int* tokens, const float* emb, const float* pos, float* x, int B,
                        int T, int d, int vocab, cudaStream_t stream);
// ctx features -> clip, scale to [-1,1], [hi | lo | hi] split for the input projection
int launch_scale_split(const float* feat, bf16* out_split, long long rows, int n_dims, float fmin,
                       float fmax, cudaStream_t stream);
// fp32 rows [rows, cols] -> bf16 [rows, 3 * cols] = [hi | lo | hi]
int launch_split3_rows(const float* src, bf16* out_split, long long rows, int cols,
                       cudaStream_t stream);
// key-mask bit words + terminal-relative roll amounts
int launch_build_masks(const int* tokens, const int* ctx_mask, int B, int T, int C,
                       uint32_t* bits /*[B,(T+C)/32]*/, int* ctx_seq_len /*[B]*/,
                       int terminal_relative, cudaStream_t stream);
// fp32 rows -> bf16 rows (encodings), with row remap b*src_len+t -> b*dst_len+dst_off+t
int launch_rmsnorm_rows_remap(const float* x, const float* gamma, int B, int src_len, int d,
                              bf16* out, int dst_len, int dst_off, cudaStream_t stream,
                              int split3 = 0);

// ---------------------------------------------------------------------------
// fp32 attention (the fp32-accurate mode of BASELINE config 2): same contract as AttnArgs'
// kernel, but Q / K / V are fp32, every product and the softmax are fp32 (exact expf), and the
// output is written as bf16 [rows, 3 * ldo_third] = [hi | lo | hi] of the fp32 result, i.e. the A
// operand of the split-precision output projection.  SIMT (CUDA-core) kernel: accuracy mode.
// ---------------------------------------------------------------------------
struct AttnF32Args {
  const float* Q; int ldq;
  const float* K; int ldk;
  const float* V; int ldv;
  bf16* O; int o_third;      // O row stride = 3 * o_third; head h -> columns h*64 of each third
  int nbatch, heads, Lq, Lk;
  const uint32_t* mask_bits; int mask_stride_words;
  int kv_batch_rows, kv_row0;  // as in AttnArgs
  // optional split-KV workspace as in AttnArgs (part_o [rows*heads*max_splits*64] f32, part_ml
  // [..*2]); splits 0 = automatic (small grids only)
  float* part_o; float* part_ml; int splits; int max_splits;
};
int launch_attention_f32(const AttnF32Args& a, cudaStream_t stream);

// ---------------------------------------------------------------------------
// Load-time kernels
// ---------------------------------------------------------------------------
// dst[n_off + n, k_off + k] = cvt(W[k, n]) for W fp32 [K, N] row-major; dst bf16 [*, ldd].
// part: 0 = bf16(w), 1 = bf16(w - bf16(w)) (low half of the split).
int launch_pack_weight(const float* W, int K, int N, bf16* dst, int ldd, int n_off, int k_off,
                       int part, cudaStream_t stream);
// Gated-MLP pack: dst rows interleave 32 columns of W0 then 32 of W1; columns [k_off, k_off + K)
// receive part 0 (bf16(w)) or part 1 (bf16(w - bf16(w))).
int launch_pack_gated(const float* W0, const float* W1, int K, int F, bf16* dst, int ldd,
                      cudaStream_t stream, int k_off = 0, int part = 0);
// Deferred normalisation (GemmPrep / GemmRowScale): the operand + row sums of a residual stream
// that no GEMM epilogue produced (first layer): a_out = bf16(x * g), ss_out[row] = sum x^2
int launch_prep_rows(const float* x, const float* g, long long g_step_stride, const int* step, int rows,
                     int d, bf16* a_out, int lda, float* ss_out, cudaStream_t stream);
// load-time tables: out[s, :] = gamma * (1 + film[s, :]);  out[s, n] = sum_k fb[s, k] * W[n, k]
int launch_film_gain(const float* film, long long film_stride, const float* gamma, float* out,
                     long long out_stride, int steps, int d, cudaStream_t stream);
int launch_film_bias(const float* fb, long long fb_stride, const bf16* W, int ldw, float* out,
                     long long out_stride, int steps, int N, int K, cudaStream_t stream);
// C[M,N] = act(A[M,K] * B[K,N]) fp32 SIMT (act: 0 none, 1 swish)
int launch_sgemm_f32(const float* A, const float* B, float* C, int ldc, int M, int N, int K,
                     int act, cudaStream_t stream);
// fp32 <-> bf16 row copies and int mask -> bit words (operator-level hooks)
int launch_f32_to_bf16(const float* src, bf16* dst, long long n, cudaStream_t stream);
int launch_bf16_to_f32(const bf16* src, float* dst, long long n, cudaStream_t stream);
int launch_mask_bits(const int* mask, int nb, int L, uint32_t* bits, cudaStream_t stream);
// dst[r * ld_dst + c] = src[r * ld_src + c] for `rows` rows of row_bytes bytes (strides in bytes,
// everything 16-byte aligned); a PDL launch that lets its dependents start at once
int launch_copy_rows(const void* src, long long ld_src, void* dst, long long ld_dst, long long rows,
                     int row_bytes, cudaStream_t stream);
// dst [rows, cols] f32 = src[r * ld + c] (+ src[r * ld + lo_off + c] when lo_off > 0)
int launch_bf16_rows_to_f32(const bf16* src, int ld, int lo_off, float* dst, long long rows, int cols,
                            cudaStream_t stream);
// out[0..n) = jax.random.normal(key, [n]) for key = (k0, k1); n a multiple of 8 (test hook)
int launch_jax_normal(uint32_t k0, uint32_t k1, long long n, float* out, cudaStream_t stream);
// the raw uint32 words the normals above are made from (same in-kernel code path)
int launch_jax_bits(uint32_t k0, uint32_t k1, long long n, uint32_t* out, cudaStream_t stream);
// audio [rows, n_samples] f32 -> MelGAN log-mel out [rows, audio_mel_frames(n_samples), 128] f32
// (audio_mel.cu); window [640], weights [513, 128] f32 device
long long audio_mel_frames(long long n_samples);
int launch_audio_mel(const float* audio, int rows, long long n_samples, const float* window,
                     const float* weights, float* out, cudaStream_t stream);
// x [rows, n_in] f32 -> y [rows, n_out] f32 resampled by ratio = target / orig as resampy's
// resample_f (audio_resample.cu); window [window_len] f64 unscaled half window with num_table
// entries per zero crossing, segments [n_segments, 3] f64 (t_s, r_s, d) of the time register
int launch_audio_resample(const float* x, int rows, int n_in, double ratio, const double* window,
                          int window_len, int num_table, const double* segments, int n_segments,
                          float* y, int n_out, cudaStream_t stream);
// Griffin-Lim decoding of MelGAN features (audio_griffin_lim.cu), per frame of `total` = rows x F:
// features [total, 128] f32 -> magnitude mag [total, 513] f32 by n_iter FISTA steps of NNLS
// against weights [513, 128] from max(0, exp(features) pinv), pinv [128, 513], beta [n_iter]
int launch_gl_nnls(const float* features, long long total, const float* weights, const float* pinv,
                   float inv_l, const float* beta, int n_iter, float* mag, cudaStream_t stream);
// angles [rows, F, 513] complex f32 = e^{2 pi i u}, u from Philox4x32-10 keyed by seed
int launch_gl_phase_init(int rows, long long frames, unsigned long long seed, float2* angles,
                         cudaStream_t stream);
// n_iter fast Griffin-Lim iterations on angles and tprev [rows, F, 513] complex f32, in place;
// work is scratch of the same size; window [640] f32
int launch_gl_iterate(const float* mag, int rows, long long frames, const float* window,
                      float2* angles, float2* tprev, float2* work, float momentum, int n_iter,
                      cudaStream_t stream);
// audio [rows, 320 F] f32 = ISTFT(mag angles)
int launch_gl_istft(const float* mag, const float2* angles, int rows, long long frames,
                    const float* window, float* audio, cudaStream_t stream);

}  // namespace msd
