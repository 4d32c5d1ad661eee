// Entry points of the C ABI (include/msd_b200.h) that take no msd_ctx: the operator-level hooks
// that run one kernel as the engine launches it (tests/ compares them with the oracle), the GEMM
// and attention benchmarks (tools/), and the audio operators.  Every hook except the audio ones
// returns once its results are complete on the caller's stream.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/msd_b200.h"
#include "common.cuh"
#include "host.h"
#include "kernels.h"

namespace msd {

// The fields AttnArgs and AttnF32Args share, with Q / K / V as elements of type T
template <typename Args, typename T> static Args attn_args(const AttnView& v) {
  Args a;
  memset(&a, 0, sizeof(a));
  a.Q = static_cast<const T*>(v.Q) + v.q_off; a.ldq = v.ldq;
  a.K = static_cast<const T*>(v.K) + v.k_off; a.ldk = v.ldk;
  a.V = static_cast<const T*>(v.V) + v.v_off; a.ldv = v.ldv;
  a.O = v.O;
  a.nbatch = v.nbatch; a.heads = v.heads; a.Lq = v.Lq; a.Lk = v.Lk;
  a.mask_bits = v.mask_bits; a.mask_stride_words = v.mask_stride_words;
  a.kv_batch_rows = v.kv_batch_rows; a.kv_row0 = v.kv_row0;
  a.part_o = v.part_o; a.part_ml = v.part_ml; a.splits = v.splits; a.max_splits = v.max_splits;
  return a;
}

int launch_attention_view(const AttnView& v, cudaStream_t st) {
  if (v.f32) {
    AttnF32Args a = attn_args<AttnF32Args, float>(v);
    a.o_third = v.ldo;
    return launch_attention_f32(a, st);
  }
  AttnArgs a = attn_args<AttnArgs, bf16>(v);
  a.ldo = v.ldo; a.tail = v.tail; a.kv_static = v.kv_static;
  return launch_attention(a, st);
}

// out [M, N] f32 = the GEMM of a [M, K] f32 with w [K, N] f32 (gated epilogues: w and w1, each
// [K, N]), run with g's epilogue, its operands and its tile width.  a is converted and the
// weights packed as the engine packs them (EPI_GATED_GELU_SPLIT3: both in split precision); a bf16
// output is converted back.
static int dense_f32(const float* a, const float* w, const float* w1, int M, int N, int K, GemmArgs g,
                     float* out, cudaStream_t st) {
  const bool gated = g.epilogue == EPI_GATED_GELU || g.epilogue == EPI_GATED_GELU_SPLIT3;
  const bool split = g.epilogue == EPI_GATED_GELU_SPLIT3;
  const int ks = split ? 3 : 1;
  const int Ng = gated ? 2 * N : N;   // GEMM width
  TempBufs tb;
  bf16 *ab = nullptr, *wb = nullptr, *ob = nullptr;
  MSD_TRY(tb.get(&ab, static_cast<size_t>(M) * K * ks));
  MSD_TRY(tb.get(&wb, static_cast<size_t>(Ng) * K * ks));
  if (split) {
    // A = [hi | lo | hi]: the rmsnorm kernel's split writer with unit gamma would renormalise, so
    // build it from the scale/split kernel's cousin: plain split of the fp32 values
    MSD_TRY(launch_split3_rows(a, ab, static_cast<long long>(M), K, st));
    MSD_TRY(launch_pack_gated(w, w1, K, N, wb, 3 * K, st, 0, 0));
    MSD_TRY(launch_pack_gated(w, w1, K, N, wb, 3 * K, st, K, 0));
    MSD_TRY(launch_pack_gated(w, w1, K, N, wb, 3 * K, st, 2 * K, 1));
  } else {
    MSD_TRY(launch_f32_to_bf16(a, ab, static_cast<long long>(M) * K, st));
    if (gated) MSD_TRY(launch_pack_gated(w, w1, K, N, wb, K, st));
    else MSD_TRY(launch_pack_weight(w, K, N, wb, K, 0, 0, 0, st));
  }
  g.A = ab; g.B = wb; g.M = M; g.N = Ng; g.K = K * ks; g.lda = K * ks; g.ldb = K * ks;
  const bool bf16_out = g.epilogue == EPI_BF16 || gated;
  if (bf16_out) {
    MSD_TRY(tb.get(&ob, static_cast<size_t>(M) * N * ks));
    g.out = ob; g.ldo = N * ks;
  } else {
    g.out = out; g.ldo = N;
  }
  MSD_TRY(launch_gemm(g, st));
  if (bf16_out)
    MSD_TRY(launch_bf16_rows_to_f32(ob, N * ks, split ? N : 0, out, M, N, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

// A benchmark's stream and timing events, destroyed with it.  time(): *ms_out = milliseconds per
// launch() over `iters` launches that follow 3 untimed ones.
struct BenchStream {
  cudaStream_t st = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  ~BenchStream() {
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (st) cudaStreamDestroy(st);
  }
  int create() {
    MSD_CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    MSD_CUDA_CHECK(cudaEventCreate(&e0));
    MSD_CUDA_CHECK(cudaEventCreate(&e1));
    return 0;
  }
  template <typename F> int time(int iters, F launch, float* ms_out) {
    for (int i = 0; i < 3; ++i) MSD_TRY(launch());
    MSD_CUDA_CHECK(cudaEventRecord(e0, st));
    for (int i = 0; i < iters; ++i) MSD_TRY(launch());
    MSD_CUDA_CHECK(cudaEventRecord(e1, st));
    MSD_CUDA_CHECK(cudaStreamSynchronize(st));
    float ms = 0.f;
    MSD_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    *ms_out = ms / iters;
    return 0;
  }
};

// The sizes every Griffin-Lim hook (named `fn`) checks: rows, frames (and *n_iter when given) >= 0,
// and at most 2^31 - 1 frames in all
static int check_gl_frames(const char* fn, int32_t rows, int64_t frames, const int32_t* n_iter = nullptr) {
  if (n_iter)
    MSD_REQUIRE(rows >= 0 && frames >= 0 && *n_iter >= 0, "%s: rows=%d, frames=%lld, n_iter=%d must be >= 0",
                fn, rows, static_cast<long long>(frames), *n_iter);
  else
    MSD_REQUIRE(rows >= 0 && frames >= 0, "%s: rows=%d, frames=%lld must be >= 0", fn, rows,
                static_cast<long long>(frames));
  MSD_REQUIRE(rows == 0 || frames <= INT32_MAX / rows, "%s: %d rows x %lld frames exceed 2^31 - 1 frames", fn,
              rows, static_cast<long long>(frames));
  return 0;
}

}  // namespace msd

using namespace msd;

extern "C" {

int msd_bench_gemm(int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t block_n, int32_t iters,
                   float* ms_out) {
  MSD_REQUIRE(ms_out && iters > 0, "msd_bench_gemm: bad argument");
  TempBufs tb;
  bf16 *a = nullptr, *b = nullptr;
  float* o = nullptr;
  MSD_TRY(tb.get(&a, static_cast<size_t>(M) * K));
  MSD_TRY(tb.get(&b, static_cast<size_t>(N) * K));
  MSD_TRY(tb.get(&o, static_cast<size_t>(M) * N));
  MSD_CUDA_CHECK(cudaMemset(a, 0, static_cast<size_t>(M) * K * 2));
  MSD_CUDA_CHECK(cudaMemset(b, 0, static_cast<size_t>(N) * K * 2));
  MSD_CUDA_CHECK(cudaMemset(o, 0, static_cast<size_t>(M) * N * 4));
  GemmArgs ga;
  memset(&ga, 0, sizeof(ga));
  ga.A = a; ga.B = b; ga.M = M; ga.N = N; ga.K = K; ga.lda = K; ga.ldb = K;
  ga.epilogue = epilogue; ga.out = o; ga.ldo = (epilogue == EPI_GATED_GELU) ? N / 2 : N;
  ga.resid = o;  // in place, like the engine
  ga.block_n = block_n;
  const bool trace = getenv("MSD_GEMM_TRACE") != nullptr;
  if (trace && (epilogue == EPI_BF16 || epilogue == EPI_GATED_GELU)) {
    // traced like the decoder's QKV / cross-q / wi launches: a row scale from one partial sum per
    // row and a bias row (zero-filled tables)
    float *ss = nullptr, *bias = nullptr;
    MSD_TRY(tb.get(&ss, static_cast<size_t>(M)));
    MSD_TRY(tb.get(&bias, static_cast<size_t>(N)));
    MSD_CUDA_CHECK(cudaMemset(ss, 0, static_cast<size_t>(M) * 4));
    MSD_CUDA_CHECK(cudaMemset(bias, 0, static_cast<size_t>(N) * 4));
    ga.rs.ss_lo = ss; ga.rs.ss_hi = ss; ga.rs.parts_lo = 1; ga.rs.parts_hi = 1;
    ga.rs.split_row = M; ga.rs.ss_stride = M; ga.rs.inv_d = 1.0f / static_cast<float>(K);
    ga.rs.col_bias = bias;
  }
  BenchStream bs;
  MSD_TRY(bs.create());
  const cudaStream_t st = bs.st;
  MSD_TRY(bs.time(iters, [&] { return launch_gemm(ga, st); }, ms_out));
  if (!trace) return 0;
  // one more launch with per-tile stamps (after a warm one right before it, like in the loop)
  long long* tr = nullptr;
  MSD_TRY(tb.get(&tr, 8 * 512));
  MSD_CUDA_CHECK(cudaMemsetAsync(tr, 0, 8 * 512 * sizeof(long long), st));
  MSD_TRY(launch_gemm(ga, st));
  ga.trace = tr;
  // without the programmatic dependency the traced launch starts after the warm one has
  // finished, so its main loop does not include waiting for that launch's tail
  g_pdl_skip_next = true;
  MSD_TRY(launch_gemm(ga, st));
  ga.trace = nullptr;
  std::vector<long long> h(8 * 512);
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  MSD_CUDA_CHECK(cudaMemcpy(h.data(), tr, h.size() * sizeof(long long), cudaMemcpyDeviceToHost));
  long long t0 = 0, t1 = 0;
  int n = 0;
  double sum[4] = {0, 0, 0, 0};
  for (int b = 0; b < 512; ++b) {
    const long long* r = &h[b * 8];
    if (r[1] == 0) continue;
    if (n == 0 || r[1] < t0) t0 = r[1];
    if (n == 0 || r[2] > t1) t1 = r[2];
    // r[3] = cycles in the tile; r[4..7] clock64 offsets from its start
    sum[0] += static_cast<double>(r[3]);
    sum[1] += static_cast<double>(r[4]);
    sum[2] += static_cast<double>(r[6] - r[5]);
    sum[3] += static_cast<double>(r[7] - r[6]);
    ++n;
  }
  const double inv_n = n ? 1.0 / n : 0.0;
  GemmArgs automatic = ga;
  automatic.block_n = 0;
  fprintf(stderr, "[gemm trace] M=%d N=%d K=%d epi=%d block_n=%d (automatic %d): %d tiles, first start -> "
          "last end %.2f us, mean cycles per tile %.0f: set-up %.0f, main loop %.0f (%.0f per k-block), "
          "epilogue %.0f\n", M, N, K, epilogue, gemm_resolve_block_n(ga), gemm_resolve_block_n(automatic), n,
          (t1 - t0) * 1e-3, sum[0] * inv_n, sum[1] * inv_n, sum[2] * inv_n, sum[2] * inv_n / (K / 64),
          sum[3] * inv_n);
  for (int b = 0; b < 4 && b < 512; ++b) {
    const long long* r = &h[b * 8];
    if (r[1] == 0) continue;
    fprintf(stderr, "[gemm trace]   tile %d sm %lld: start +%.2f us, end +%.2f us; cycles: total %lld, "
            "setup->wait %lld, wait->acc %lld, acc->stored %lld\n", b, r[0], (r[1] - t0) * 1e-3,
            (r[2] - t0) * 1e-3, r[3], r[5] - r[4], r[6] - r[5], r[7] - r[6]);
  }
  // the tiles of CTA 0 in order: main loop, drain (bf16 outputs: until the last sub-tile is
  // handed to TMA, whose global writes then run under the next tile's main loop)
  const int grid = std::min(n, device_sm_count());
  for (int b = 0, i = 0; grid > 0 && b < 512; b += grid, ++i) {
    const long long* r = &h[b * 8];
    if (r[1] == 0) break;
    fprintf(stderr, "[gemm trace]   CTA 0 tile %d (#%d): start +%.2f us; cycles: main loop %lld, drain %lld\n",
            i, b, (r[1] - t0) * 1e-3, r[6] - r[5], r[7] - r[6]);
  }
  return 0;
}

int msd_bench_attention(int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, int32_t iters,
                        float* ms_out) {
  MSD_REQUIRE(ms_out && iters > 0, "msd_bench_attention: bad argument");
  const int w = heads * 64;
  TempBufs tb;
  bf16 *qb, *kb, *vb, *ob;
  float *tmp, *po, *pml;
  const size_t nq = static_cast<size_t>(nb) * Lq * w, nk = static_cast<size_t>(nb) * Lk * w;
  MSD_TRY(tb.get(&qb, nq)); MSD_TRY(tb.get(&kb, nk)); MSD_TRY(tb.get(&vb, nk)); MSD_TRY(tb.get(&ob, nq));
  MSD_TRY(tb.get(&tmp, nk));
  MSD_TRY(tb.get(&po, attention_workspace_floats(nb, heads, Lq, 12)));
  MSD_TRY(tb.get(&pml, static_cast<size_t>(nb) * Lq * heads * 12 * 2));
  BenchStream bs;
  MSD_TRY(bs.create());
  const cudaStream_t st = bs.st;
  // N(0,1) * 0.3-ish values through the jax generator (any bounded values would do)
  MSD_TRY(launch_jax_normal(1u, 2u, static_cast<long long>(nk), tmp, st));
  MSD_TRY(launch_f32_to_bf16(tmp, kb, static_cast<long long>(nk), st));
  MSD_TRY(launch_f32_to_bf16(tmp, vb, static_cast<long long>(nk), st));
  MSD_TRY(launch_f32_to_bf16(tmp, qb, static_cast<long long>(nq), st));
  const AttnSwitches sw = attn_switches();
  AttnView view = {};
  view.Q = qb; view.ldq = w; view.K = kb; view.ldk = w; view.V = vb; view.ldv = w; view.O = ob; view.ldo = w;
  view.nbatch = nb; view.heads = heads; view.Lq = Lq; view.Lk = Lk;
  view.part_o = po; view.part_ml = pml; view.max_splits = 12; view.kv_static = 1;
  view.splits = sw.splits; view.tail = sw.tail;
  return bs.time(iters, [&] { return launch_attention_view(view, st); }, ms_out);
}

int msd_op_attention(const float* q, const float* k, const float* v, const int32_t* key_mask,
                     int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, float* out, void* stream) {
  MSD_REQUIRE(q && k && v && out, "msd_op_attention: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int w = heads * 64;
  TempBufs tb;
  bf16 *qb, *kb, *vb, *ob;
  float *po, *pml;
  uint32_t* bits = nullptr;
  MSD_TRY(tb.get(&qb, static_cast<size_t>(nb) * Lq * w));
  MSD_TRY(tb.get(&kb, static_cast<size_t>(nb) * Lk * w));
  MSD_TRY(tb.get(&vb, static_cast<size_t>(nb) * Lk * w));
  MSD_TRY(tb.get(&ob, static_cast<size_t>(nb) * Lq * w));
  MSD_TRY(tb.get(&po, attention_workspace_floats(nb, heads, Lq, 12)));
  MSD_TRY(tb.get(&pml, static_cast<size_t>(nb) * Lq * heads * 12 * 2));
  MSD_TRY(launch_f32_to_bf16(q, qb, static_cast<long long>(nb) * Lq * w, st));
  MSD_TRY(launch_f32_to_bf16(k, kb, static_cast<long long>(nb) * Lk * w, st));
  MSD_TRY(launch_f32_to_bf16(v, vb, static_cast<long long>(nb) * Lk * w, st));
  if (key_mask) {
    MSD_TRY(tb.get(&bits, static_cast<size_t>(nb) * (Lk / 32)));
    MSD_TRY(launch_mask_bits(key_mask, nb, Lk, bits, st));
  }
  const AttnSwitches sw = attn_switches();
  AttnView view = {};
  view.Q = qb; view.ldq = w; view.K = kb; view.ldk = w; view.V = vb; view.ldv = w; view.O = ob; view.ldo = w;
  view.nbatch = nb; view.heads = heads; view.Lq = Lq; view.Lk = Lk;
  view.mask_bits = bits; view.mask_stride_words = Lk / 32;
  view.part_o = po; view.part_ml = pml; view.max_splits = 12;
  view.splits = sw.splits; view.tail = sw.tail;
  MSD_TRY(launch_attention_view(view, st));
  MSD_TRY(launch_bf16_to_f32(ob, out, static_cast<long long>(nb) * Lq * w, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_jax_normal(uint64_t seed, int32_t step, int64_t n, float* out, void* stream) {
  MSD_REQUIRE(out != nullptr, "msd_op_jax_normal: null argument");
  uint32_t key[2];
  if (step >= 0) fold_in(seed, static_cast<uint32_t>(step), key);
  else prng_key(seed, key);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(launch_jax_normal(key[0], key[1], n, out, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_jax_bits(uint64_t seed, int32_t step, int64_t n, uint32_t* out, void* stream) {
  MSD_REQUIRE(out != nullptr, "msd_op_jax_bits: null argument");
  uint32_t key[2];
  if (step >= 0) fold_in(seed, static_cast<uint32_t>(step), key);
  else prng_key(seed, key);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(launch_jax_bits(key[0], key[1], n, out, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_audio_mel(const float* audio, int32_t rows, int64_t n_samples, const float* window,
                     const float* mel_weights, float* mel_out, void* stream) {
  MSD_REQUIRE(audio && window && mel_weights && mel_out, "msd_op_audio_mel: null argument");
  MSD_REQUIRE(rows >= 0 && n_samples >= 0, "msd_op_audio_mel: rows=%d, n_samples=%lld must be >= 0",
              rows, static_cast<long long>(n_samples));
  const long long frames = audio_mel_frames(n_samples);
  MSD_REQUIRE(rows == 0 || frames <= INT32_MAX / rows,
              "msd_op_audio_mel: %d rows x %lld frames exceed 2^31 - 1 output frames", rows, frames);
  MSD_TRY(launch_audio_mel(audio, rows, n_samples, window, mel_weights, mel_out,
                           reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int msd_op_audio_resample(const float* x, int32_t rows, int64_t n_in, int32_t orig_sr,
                          int32_t target_sr, const double* half_window, int32_t window_len,
                          int32_t precision, const double* time_segments, int32_t n_segments,
                          float* y, int64_t n_out, void* stream) {
  MSD_REQUIRE(x && half_window && time_segments && y, "msd_op_audio_resample: null argument");
  MSD_REQUIRE(rows >= 0 && n_in >= 0 && n_out >= 0,
              "msd_op_audio_resample: rows=%d, n_in=%lld, n_out=%lld must be >= 0", rows,
              static_cast<long long>(n_in), static_cast<long long>(n_out));
  MSD_REQUIRE(orig_sr > 0 && target_sr > 0, "msd_op_audio_resample: rates %d -> %d must be > 0",
              orig_sr, target_sr);
  const double ratio = static_cast<double>(target_sr) / orig_sr;
  const long long want = static_cast<long long>(static_cast<double>(n_in) * ratio);
  MSD_REQUIRE(n_out == want, "msd_op_audio_resample: n_out=%lld, int(n_in * ratio) is %lld",
              static_cast<long long>(n_out), want);
  MSD_REQUIRE(n_in <= INT32_MAX && n_out <= INT32_MAX && rows <= 65535,
              "msd_op_audio_resample: %d rows x %lld -> %lld samples: at most 65535 rows of "
              "2^31 - 1 samples", rows, static_cast<long long>(n_in), static_cast<long long>(n_out));
  MSD_REQUIRE(precision >= 0 && precision <= 24 && window_len >= 2 && n_segments >= 1,
              "msd_op_audio_resample: precision=%d (0..24), window_len=%d (>= 2), "
              "n_segments=%d (>= 1)", precision, window_len, n_segments);
  const int num_table = 1 << precision;
  MSD_REQUIRE(static_cast<int>((ratio < 1.0 ? ratio : 1.0) * num_table) >= 1,
              "msd_op_audio_resample: %d -> %d Hz is below one window entry per input sample",
              orig_sr, target_sr);
  MSD_TRY(launch_audio_resample(x, rows, static_cast<int>(n_in), ratio, half_window, window_len,
                                num_table, time_segments, n_segments, y, static_cast<int>(n_out),
                                reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int msd_op_griffin_lim_magnitude(const float* features, int32_t rows, int64_t frames,
                                 const float* mel_weights, const float* pinv, float inv_lipschitz,
                                 const float* beta, int32_t n_iter, float* mag_out, void* stream) {
  MSD_REQUIRE(features && mel_weights && pinv && beta && mag_out,
              "msd_op_griffin_lim_magnitude: null argument");
  MSD_TRY(check_gl_frames("msd_op_griffin_lim_magnitude", rows, frames, &n_iter));
  MSD_TRY(launch_gl_nnls(features, static_cast<long long>(rows) * frames, mel_weights, pinv,
                         inv_lipschitz, beta, n_iter, mag_out, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int msd_op_griffin_lim_init(int32_t rows, int64_t frames, uint64_t seed, float* angles, void* stream) {
  MSD_REQUIRE(angles, "msd_op_griffin_lim_init: null argument");
  MSD_TRY(check_gl_frames("msd_op_griffin_lim_init", rows, frames));
  MSD_TRY(launch_gl_phase_init(rows, frames, seed, reinterpret_cast<float2*>(angles),
                               reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int msd_op_griffin_lim_iterate(const float* mag, int32_t rows, int64_t frames, const float* window,
                               float* angles, float* tprev, float* work, float momentum,
                               int32_t n_iter, void* stream) {
  MSD_REQUIRE(mag && window && angles && tprev && work, "msd_op_griffin_lim_iterate: null argument");
  MSD_TRY(check_gl_frames("msd_op_griffin_lim_iterate", rows, frames, &n_iter));
  MSD_REQUIRE(momentum >= 0.f, "msd_op_griffin_lim_iterate: momentum=%g must be >= 0",
              static_cast<double>(momentum));
  MSD_TRY(launch_gl_iterate(mag, rows, frames, window, reinterpret_cast<float2*>(angles),
                            reinterpret_cast<float2*>(tprev), reinterpret_cast<float2*>(work),
                            momentum, n_iter, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int msd_op_griffin_lim_istft(const float* mag, const float* angles, int32_t rows, int64_t frames,
                             const float* window, float* audio_out, void* stream) {
  MSD_REQUIRE(mag && angles && window && audio_out, "msd_op_griffin_lim_istft: null argument");
  MSD_TRY(check_gl_frames("msd_op_griffin_lim_istft", rows, frames));
  MSD_TRY(launch_gl_istft(mag, reinterpret_cast<const float2*>(angles), rows, frames, window,
                          audio_out, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int msd_op_dense_epilogue(const float* a, const float* w, const float* w1, int32_t M, int32_t N,
                          int32_t K, int32_t epilogue, int32_t block_n, const float* resid,
                          const float* pos, int32_t pos_rows, const int32_t* pos_shift,
                          int32_t dup_rows, float* out, void* stream) {
  MSD_REQUIRE(a && w && out, "msd_op_dense_epilogue: null argument");
  const bool gated = epilogue == EPI_GATED_GELU || epilogue == EPI_GATED_GELU_SPLIT3;
  MSD_REQUIRE(epilogue == EPI_BF16 || epilogue == EPI_F32 || epilogue == EPI_RESID_F32 || epilogue == EPI_POS_F32 ||
                  gated,
              "msd_op_dense_epilogue: unknown epilogue %d", epilogue);
  MSD_REQUIRE(!gated || w1 != nullptr, "msd_op_dense_epilogue: the gated epilogues need w1");
  MSD_REQUIRE(epilogue != EPI_RESID_F32 || resid != nullptr, "msd_op_dense_epilogue: resid is null");
  MSD_REQUIRE(epilogue != EPI_POS_F32 || (pos != nullptr && pos_rows > 0),
              "msd_op_dense_epilogue: pos / pos_rows missing");
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.epilogue = epilogue; g.block_n = block_n;
  g.resid = resid; g.pos = pos; g.pos_rows = pos_rows; g.pos_shift = pos_shift; g.dup_rows = dup_rows;
  return dense_f32(a, w, w1, M, N, K, g, out, reinterpret_cast<cudaStream_t>(stream));
}

int msd_op_dense_deferred_norm(const float* a, const float* w_out, const float* x, int32_t M, int32_t d,
                               int32_t K, const float* g_lo, const float* g_hi, int32_t split_row,
                               const float* w2, const float* w2b, int32_t N2, const float* bias,
                               int32_t block_n1, int32_t block_n2, float* x_out, float* y_out,
                               void* stream) {
  MSD_REQUIRE(a && w_out && x && g_lo && g_hi && w2 && x_out && y_out,
              "msd_op_dense_deferred_norm: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool gated = w2b != nullptr;
  const int Ng = gated ? 2 * N2 : N2;
  TempBufs tb;
  bf16 *ab = nullptr, *wo = nullptr, *opnd = nullptr, *w2p = nullptr, *yb = nullptr;
  float* ss = nullptr;
  int* step0 = nullptr;
  GemmArgs g1;
  memset(&g1, 0, sizeof(g1));
  g1.M = M; g1.N = d; g1.K = K; g1.epilogue = EPI_RESID_PREP; g1.block_n = block_n1;
  const int bn1 = gemm_resolve_block_n(g1);
  MSD_REQUIRE(bn1 > 0, "msd_op_dense_deferred_norm: no valid tile width for d=%d (block_n1 %d)", d,
              block_n1);
  const int parts = d / bn1;
  MSD_TRY(tb.get(&ab, static_cast<size_t>(M) * K));
  MSD_TRY(tb.get(&wo, static_cast<size_t>(d) * K));
  MSD_TRY(tb.get(&opnd, static_cast<size_t>(M) * d));
  MSD_TRY(tb.get(&w2p, static_cast<size_t>(Ng) * d));
  MSD_TRY(tb.get(&yb, static_cast<size_t>(M) * N2));
  MSD_TRY(tb.get(&ss, static_cast<size_t>(parts) * M));
  MSD_TRY(tb.get(&step0, 1));
  MSD_CUDA_CHECK(cudaMemsetAsync(step0, 0, sizeof(int), st));
  MSD_TRY(launch_f32_to_bf16(a, ab, static_cast<long long>(M) * K, st));
  MSD_TRY(launch_pack_weight(w_out, K, d, wo, K, 0, 0, 0, st));
  if (gated) MSD_TRY(launch_pack_gated(w2, w2b, d, N2, w2p, d, st));
  else MSD_TRY(launch_pack_weight(w2, d, N2, w2p, d, 0, 0, 0, st));
  MSD_CUDA_CHECK(cudaMemcpyAsync(x_out, x, static_cast<size_t>(M) * d * sizeof(float),
                                 cudaMemcpyDeviceToDevice, st));
  g1.A = ab; g1.B = wo; g1.lda = K; g1.ldb = K;
  g1.out = x_out; g1.ldo = d; g1.resid = x_out; g1.block_n = bn1;
  g1.step = step0;
  g1.prep.g_lo = g_lo; g1.prep.g_hi = g_hi; g1.prep.split_row = split_row;
  g1.prep.a = opnd; g1.prep.lda = d; g1.prep.ss = ss; g1.prep.ss_stride = M;
  MSD_TRY(launch_gemm(g1, st));
  GemmArgs g2;
  memset(&g2, 0, sizeof(g2));
  g2.A = opnd; g2.B = w2p; g2.M = M; g2.N = Ng; g2.K = d; g2.lda = d; g2.ldb = d;
  g2.epilogue = gated ? EPI_GATED_GELU : EPI_BF16; g2.out = yb; g2.ldo = N2; g2.block_n = block_n2;
  g2.step = step0;
  g2.rs.ss_lo = ss; g2.rs.ss_hi = ss; g2.rs.parts_lo = parts; g2.rs.parts_hi = parts;
  g2.rs.split_row = M; g2.rs.ss_stride = M; g2.rs.inv_d = 1.0f / static_cast<float>(d);
  g2.rs.col_bias = bias;
  MSD_TRY(launch_gemm(g2, st));
  MSD_TRY(launch_bf16_rows_to_f32(yb, N2, 0, y_out, M, N2, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_attention_f32(const float* q, const float* k, const float* v, const int32_t* key_mask,
                         int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, float* out,
                         void* stream) {
  MSD_REQUIRE(q && k && v && out, "msd_op_attention_f32: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int w = heads * 64;
  TempBufs tb;
  bf16* ob = nullptr;
  float *po = nullptr, *pml = nullptr;
  uint32_t* bits = nullptr;
  MSD_TRY(tb.get(&ob, static_cast<size_t>(nb) * Lq * w * 3));
  if (key_mask) {
    MSD_REQUIRE(Lk % 128 == 0, "msd_op_attention_f32: masked Lk must be a multiple of 128");
    MSD_TRY(tb.get(&bits, static_cast<size_t>(nb) * (Lk / 32)));
    MSD_TRY(launch_mask_bits(key_mask, nb, Lk, bits, st));
  }
  MSD_TRY(tb.get(&po, attention_workspace_floats(nb, heads, Lq, 8)));
  MSD_TRY(tb.get(&pml, static_cast<size_t>(nb) * Lq * heads * 8 * 2));
  AttnView view = {};
  view.f32 = true;
  view.Q = q; view.ldq = w; view.K = k; view.ldk = w; view.V = v; view.ldv = w; view.O = ob; view.ldo = w;
  view.nbatch = nb; view.heads = heads; view.Lq = Lq; view.Lk = Lk;
  view.mask_bits = bits; view.mask_stride_words = Lk / 32;
  view.part_o = po; view.part_ml = pml; view.max_splits = 8;
  view.splits = attn_switches().splits;
  MSD_TRY(launch_attention_view(view, st));
  MSD_TRY(launch_bf16_rows_to_f32(ob, 3 * w, w, out, static_cast<long long>(nb) * Lq, w, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_attention_view(const msd_attention_view_args* args, void* stream) {
  MSD_REQUIRE(args && args->q && args->k && args->v && args->out && args->part_o && args->part_ml,
              "msd_op_attention_view: null argument");
  const msd_attention_view_args& a = *args;
  MSD_REQUIRE(a.precision == 0 || a.precision == 1, "msd_op_attention_view: precision must be 0 or 1");
  MSD_REQUIRE(a.nb > 0 && a.heads > 0 && a.Lq > 0 && a.Lk > 0 && a.q_off >= 0 && a.k_off >= 0 && a.v_off >= 0 &&
                  a.o_col >= 0 && a.kv_row0 >= 0 && a.kv_batch_rows >= 0,
              "msd_op_attention_view: bad sizes or offsets");
  MSD_REQUIRE(a.splits >= 0 && a.splits <= 12 && a.tail >= 0 && (a.precision == 0 || a.tail == 0),
              "msd_op_attention_view: splits must be in [0, 12], tail >= 0 (bf16 mode only)");
  MSD_REQUIRE(!a.key_mask || (a.mask_len % 128 == 0 && a.mask_word0 >= 0 && a.mask_word0 % 4 == 0 &&
                              a.mask_word0 + a.Lk / 32 <= a.mask_len / 32),
              "msd_op_attention_view: mask words [%d, %d) outside rows of %d keys", a.mask_word0,
              a.mask_word0 + a.Lk / 32, a.mask_len);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t es = a.precision ? 4 : 2;
  const int width = a.heads * 64;
  const long long rows_q = static_cast<long long>(a.nb) * a.Lq;
  char* qv = static_cast<char*>(a.q) + a.q_off * es;
  TempBufs tb;
  uint32_t* bits = nullptr;
  if (a.key_mask) {
    MSD_TRY(tb.get(&bits, static_cast<size_t>(a.nb) * (a.mask_len / 32)));
    MSD_TRY(launch_mask_bits(a.key_mask, a.nb, a.mask_len, bits, st));
  }
  // K, V and the mask must be complete before the attention starts (kv_static reads them ahead of
  // its dependency wait, as after the plain first launch of a diffusion step).  Q is then written
  // back from a staging copy by a kernel of its own, so that the attention is a PDL launch behind a
  // live predecessor, as in the step graph.
  char* stage = nullptr;
  MSD_TRY(tb.get(&stage, static_cast<size_t>(rows_q) * width * es));
  MSD_CUDA_CHECK(cudaMemcpy2DAsync(stage, width * es, qv, a.ldq * es, width * es, rows_q,
                                   cudaMemcpyDeviceToDevice, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  MSD_TRY(launch_copy_rows(stage, static_cast<long long>(width * es), qv, static_cast<long long>(a.ldq) * es,
                           rows_q, static_cast<int>(width * es), st));
  AttnView view = {};
  view.f32 = a.precision == 1;
  view.Q = qv; view.ldq = a.ldq;
  view.K = a.k; view.k_off = a.k_off; view.ldk = a.ldk;
  view.V = a.v; view.v_off = a.v_off; view.ldv = a.ldv;
  view.O = static_cast<bf16*>(a.out) + a.o_col; view.ldo = a.o_ld;
  view.nbatch = a.nb; view.heads = a.heads; view.Lq = a.Lq; view.Lk = a.Lk;
  view.mask_bits = bits ? bits + a.mask_word0 : nullptr; view.mask_stride_words = a.mask_len / 32;
  view.part_o = a.part_o; view.part_ml = a.part_ml; view.max_splits = 12;
  view.splits = a.splits; view.tail = a.tail;
  view.kv_static = a.kv_static; view.kv_batch_rows = a.kv_batch_rows; view.kv_row0 = a.kv_row0;
  MSD_TRY(launch_attention_view(view, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_gemm_view(const msd_gemm_view_args* args, int32_t* block_n_out, void* stream) {
  MSD_REQUIRE(args && args->a && args->b && args->out, "msd_op_gemm_view: null argument");
  const msd_gemm_view_args& v = *args;
  MSD_REQUIRE(v.epilogue >= EPI_BF16 && v.epilogue <= EPI_RESID_PREP, "msd_op_gemm_view: unknown epilogue %d",
              v.epilogue);
  MSD_REQUIRE(v.a_off >= 0 && v.b_off >= 0 && v.out_off >= 0 && v.resid_off >= 0,
              "msd_op_gemm_view: negative offset");
  const bool f32_out = v.epilogue == EPI_F32 || v.epilogue == EPI_RESID_F32 || v.epilogue == EPI_POS_F32 ||
                       v.epilogue == EPI_RESID_PREP;
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.A = static_cast<const bf16*>(v.a) + v.a_off; g.lda = v.lda;
  g.B = static_cast<const bf16*>(v.b) + v.b_off; g.ldb = v.ldb;
  g.M = v.M; g.N = v.N; g.K = v.K; g.epilogue = v.epilogue; g.block_n = v.block_n;
  g.out = f32_out ? static_cast<void*>(static_cast<float*>(v.out) + v.out_off)
                  : static_cast<void*>(static_cast<bf16*>(v.out) + v.out_off);
  g.ldo = v.ldo;
  g.resid = v.resid ? v.resid + v.resid_off : nullptr;
  g.pos = v.pos; g.pos_rows = v.pos_rows; g.pos_shift = v.pos_shift; g.dup_rows = v.dup_rows;
  g.step = v.step;
  g.prep.g_lo = v.prep.g_lo; g.prep.g_lo_step_stride = v.prep.g_lo_step_stride;
  g.prep.g_hi = v.prep.g_hi; g.prep.g_hi_step_stride = v.prep.g_hi_step_stride;
  g.prep.split_row = v.prep.split_row;
  g.prep.a = static_cast<bf16*>(v.prep.a); g.prep.lda = v.prep.lda;
  g.prep.ss = v.prep.ss; g.prep.ss_stride = v.prep.ss_stride;
  g.rs.ss_lo = v.rs.ss_lo; g.rs.parts_lo = v.rs.parts_lo; g.rs.ss_hi = v.rs.ss_hi; g.rs.parts_hi = v.rs.parts_hi;
  g.rs.split_row = v.rs.split_row; g.rs.ss_stride = v.rs.ss_stride; g.rs.inv_d = v.rs.inv_d;
  g.rs.col_bias = v.rs.col_bias; g.rs.bias_step_stride = v.rs.bias_step_stride;
  MSD_REQUIRE(v.epilogue != EPI_RESID_PREP || g.prep.a != nullptr,
              "msd_op_gemm_view: EPI_RESID_PREP needs prep_a");
  MSD_REQUIRE(v.epilogue != EPI_POS_F32 || (v.pos != nullptr && v.pos_rows > 0),
              "msd_op_gemm_view: EPI_POS_F32 needs pos / pos_rows");
  const int bn = gemm_resolve_block_n(g);
  MSD_REQUIRE(bn > 0, "msd_op_gemm_view: N=%d has no tile width (block_n %d)", v.N, v.block_n);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  g_pdl_skip_next = true;   // the operands were just written by the caller's own kernels
  MSD_TRY(launch_gemm(g, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  if (block_n_out) *block_n_out = bn;
  return 0;
}

int msd_op_prep_rows(const float* x, const float* g, int64_t g_step_stride, const int32_t* step, int32_t rows,
                     int32_t d, void* a_out, int32_t lda, float* ss_out, void* stream) {
  MSD_REQUIRE(x && g && step && a_out && ss_out, "msd_op_prep_rows: null argument");
  MSD_REQUIRE(rows > 0 && lda >= d && lda % 8 == 0, "msd_op_prep_rows: rows %d / lda %d (d %d)", rows, lda, d);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  g_pdl_skip_next = true;
  MSD_TRY(launch_prep_rows(x, g, g_step_stride, step, rows, d, static_cast<bf16*>(a_out), lda, ss_out, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_sampler_step(const msd_sampler_step_args* args, int32_t* run_out, void* stream) {
  MSD_REQUIRE(args && args->eps && args->z && args->z_split && args->coef, "msd_op_sampler_step: null argument");
  const msd_sampler_step_args& s = *args;
  const msd_noise_streams& ns = s.streams;
  MSD_REQUIRE(s.n > 0 && s.n_dims > 0 && s.n % 4 == 0 && s.n_dims % 4 == 0 && s.n % s.n_dims == 0 && s.num_steps > 0,
              "msd_op_sampler_step: n=%lld must be a positive multiple of n_dims=%d, both multiples of 4",
              static_cast<long long>(s.n), s.n_dims);
  MSD_REQUIRE(s.passes == 1 || s.passes == 2, "msd_op_sampler_step: passes must be 1 or 2 (got %d)", s.passes);
  MSD_REQUIRE(ns.rng_kind == 0 || ns.rng_kind == 1, "msd_op_sampler_step: rng_kind must be 0 or 1");
  MSD_REQUIRE(ns.rng_kind == 0 || s.per_row || (ns.rng_keys != nullptr && s.n % 8 == 0 && s.n < (1ll << 32)),
              "msd_op_sampler_step: the jax stream needs its key table and a draw of k*8 < 2^32 elements");
  MSD_REQUIRE(!s.per_row || (ns.n_row > 0 && ns.n_row % 8 == 0 && s.n % ns.n_row == 0 && s.n < (1ll << 32) &&
                             (ns.rng_kind == 0 ? ns.row_seeds != nullptr : ns.row_keys != nullptr)),
              "msd_op_sampler_step: per-row streams need rows of k*8 elements, n < 2^32 and the row table");
  MSD_REQUIRE(s.step == nullptr || (!s.per_row && s.launches == 1),
              "msd_op_sampler_step: per-row streams and several launches need the RunArgs path (step NULL)");
  MSD_REQUIRE(s.step != nullptr || run_out != nullptr, "msd_op_sampler_step: the RunArgs path needs run_out");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int first = s.run_step;
  if (s.step != nullptr) MSD_CUDA_CHECK(cudaMemcpy(&first, s.step, sizeof(int), cudaMemcpyDeviceToHost));
  MSD_REQUIRE(s.launches >= 1 && first < s.num_steps && first - s.launches + 1 >= 0,
              "msd_op_sampler_step: %d launch(es) from step %d leave the table of %d steps", s.launches, first,
              s.num_steps);
  SamplerArgs a;
  memset(&a, 0, sizeof(a));
  a.eps = s.eps; a.z = s.z; a.z_split = static_cast<bf16*>(s.z_split); a.coef = s.coef;
  a.n = s.n; a.n_dims = s.n_dims; a.passes = s.passes; a.cond_weight = s.cond_weight;
  a.clip_x0 = s.clip_x0; a.ddim = s.ddim; a.feat_min = s.feat_min; a.feat_max = s.feat_max;
  a.rng_kind = ns.rng_kind; a.rng_keys = ns.rng_keys;
  a.n_row = ns.n_row; a.row_keys = ns.row_keys; a.row_key_stride = ns.row_key_stride;
  a.row_seeds = reinterpret_cast<const unsigned long long*>(ns.row_seeds);
  TempBufs tb;
  if (s.step != nullptr) {
    a.step = s.step; a.noise = s.noise; a.mel_out = s.mel_out; a.seed = ns.seed;
    g_pdl_skip_next = true;   // the inputs were just written by the caller's own kernels
    MSD_TRY(launch_sampler_step(a, st));
    MSD_CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
  }
  RunArgs ra;
  memset(&ra, 0, sizeof(ra));
  ra.noise = s.noise; ra.mel_out = s.mel_out; ra.seed = ns.seed; ra.step = s.run_step; ra.per_row = s.per_row;
  MSD_TRY(tb.get(&a.run, 1));
  MSD_CUDA_CHECK(cudaMemcpyAsync(a.run, &ra, sizeof(ra), cudaMemcpyHostToDevice, st));
  // the first launch follows the upload; the next ones are PDL launches behind the previous step's
  // sampler kernel, which is what the step graph's first kernel sees
  g_pdl_skip_next = true;
  for (int i = 0; i < s.launches; ++i) MSD_TRY(launch_sampler_step(a, st));
  MSD_CUDA_CHECK(cudaMemcpyAsync(&ra, a.run, sizeof(ra), cudaMemcpyDeviceToHost, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  run_out[0] = ra.step;
  run_out[1] = static_cast<int32_t>(ra.done);
  return 0;
}

int msd_op_init_z(const msd_init_z_args* args, void* stream) {
  MSD_REQUIRE(args && args->z && args->z_split, "msd_op_init_z: null argument");
  const msd_init_z_args& a = *args;
  const msd_noise_streams& ns = a.streams;
  MSD_REQUIRE(a.n > 0 && a.n_dims > 0 && a.n % 4 == 0 && a.n_dims % 4 == 0 && a.n % a.n_dims == 0,
              "msd_op_init_z: n=%lld must be a positive multiple of n_dims=%d, both multiples of 4",
              static_cast<long long>(a.n), a.n_dims);
  MSD_REQUIRE(ns.rng_kind == 0 || ns.rng_kind == 1, "msd_op_init_z: rng_kind must be 0 or 1");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // launch_init_z reads the per-row key tables from its rng_keys argument
  MSD_TRY(launch_init_z(a.init_z, a.z, static_cast<bf16*>(a.z_split), a.n, a.n_dims, ns.seed, st, ns.rng_kind,
                        ns.n_row > 0 ? ns.row_keys : ns.rng_keys, ns.n_row, ns.row_key_stride,
                        reinterpret_cast<const unsigned long long*>(ns.row_seeds)));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_scale_split(const float* feat, void* out_split, int64_t rows, int32_t n_dims, float feat_min,
                       float feat_max, void* stream) {
  MSD_REQUIRE(feat && out_split, "msd_op_scale_split: null argument");
  MSD_REQUIRE(rows > 0 && n_dims > 0 && n_dims % 4 == 0, "msd_op_scale_split: rows %lld / n_dims %d",
              static_cast<long long>(rows), n_dims);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(launch_scale_split(feat, static_cast<bf16*>(out_split), rows, n_dims, feat_min, feat_max, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_rmsnorm_view(const msd_rmsnorm_view_args* args, void* stream) {
  MSD_REQUIRE(args && args->x && args->gamma && args->out, "msd_op_rmsnorm_view: null argument");
  const msd_rmsnorm_view_args& a = *args;
  MSD_REQUIRE(a.rows > 0 && a.d > 0 && a.d % 128 == 0 && a.d <= 1024,
              "msd_op_rmsnorm_view: rows=%d must be > 0 and d=%d k*128 <= 1024", a.rows, a.d);
  MSD_REQUIRE(a.split3 == 0 || a.split3 == 1, "msd_op_rmsnorm_view: split3 must be 0 or 1");
  MSD_REQUIRE(a.out_off >= 0 && a.film_offset >= 0 && a.film_step_stride >= 0 && a.src_len >= 0 &&
                  a.dst_len >= 0 && a.dst_off >= 0,
              "msd_op_rmsnorm_view: negative offset, stride or length");
  // the kernel moves 4 values at a time: 16-byte loads of x / gamma / FiLM, 8-byte stores of bf16
  MSD_REQUIRE(a.out_off % 4 == 0 && a.ldo % 4 == 0 && a.film_offset % 4 == 0 && a.film_step_stride % 4 == 0,
              "msd_op_rmsnorm_view: out_off, ldo, film_offset and film_step_stride must be multiples of 4");
  MSD_REQUIRE(((reinterpret_cast<uintptr_t>(a.x) | reinterpret_cast<uintptr_t>(a.gamma) |
                reinterpret_cast<uintptr_t>(a.film) | reinterpret_cast<uintptr_t>(a.out)) & 15) == 0,
              "msd_op_rmsnorm_view: x, gamma, film and out must be 16-byte aligned");
  const int width = a.split3 ? 3 * a.d : a.d;
  MSD_REQUIRE(a.ldo >= width, "msd_op_rmsnorm_view: ldo=%d below the %d values of a row", a.ldo, width);
  MSD_REQUIRE(!a.film || a.step, "msd_op_rmsnorm_view: FiLM rows need the device step");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  bf16* out = static_cast<bf16*>(a.out) + a.out_off;
  g_pdl_skip_next = true;   // the inputs were just written by the caller's own kernels
  if (a.src_len > 0) {
    MSD_REQUIRE(!a.film, "msd_op_rmsnorm_view: a remapped launch takes no FiLM");
    MSD_REQUIRE(a.rows % a.src_len == 0 && a.dst_off + a.src_len <= a.dst_len && a.ldo == width,
                "msd_op_rmsnorm_view: remap of rows=%d in sequences of %d to [%d, +%d) of %d with ldo=%d "
                "(must be %d)", a.rows, a.src_len, a.dst_off, a.src_len, a.dst_len, a.ldo, width);
    MSD_TRY(launch_rmsnorm_rows_remap(a.x, a.gamma, a.rows / a.src_len, a.src_len, a.d, out, a.dst_len,
                                      a.dst_off, st, a.split3));
  } else {
    MSD_TRY(launch_rmsnorm(a.x, a.gamma, a.rows, a.d, out, a.ldo, a.film, a.film ? a.step : nullptr,
                           a.film_step_stride, a.film_offset, a.split3, st));
  }
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_encoder_inputs(const msd_encoder_inputs_args* args, void* stream) {
  MSD_REQUIRE(args && args->tokens && args->embedding && args->pos && args->bits && args->ctx_seq_len &&
                  args->x && (args->C == 0 || args->ctx_mask),
              "msd_op_encoder_inputs: null argument");
  const msd_encoder_inputs_args& a = *args;
  MSD_REQUIRE(a.B >= 1 && a.T > 0 && a.T % 128 == 0 && a.C >= 0 && a.C % 128 == 0,
              "msd_op_encoder_inputs: B=%d must be >= 1, T=%d > 0 and C=%d >= 0 multiples of 128", a.B, a.T,
              a.C);
  MSD_REQUIRE(a.d > 0 && a.d % 4 == 0 && a.vocab >= 1, "msd_op_encoder_inputs: d=%d (multiple of 4), vocab=%d",
              a.d, a.vocab);
  MSD_REQUIRE(a.terminal_relative == 0 || (a.terminal_relative == 1 && a.C > 0),
              "msd_op_encoder_inputs: terminal_relative must be 0 or 1, and 0 without a context");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(launch_build_masks(a.tokens, a.C > 0 ? a.ctx_mask : nullptr, a.B, a.T, a.C, a.bits, a.ctx_seq_len,
                             a.terminal_relative, st));
  MSD_TRY(launch_embed_tokens(a.tokens, a.embedding, a.pos, a.x, a.B, a.T, a.d, a.vocab, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
