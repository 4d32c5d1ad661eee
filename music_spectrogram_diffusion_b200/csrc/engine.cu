// Engine behind the C ABI (include/msd_b200.h): weight repacking, the two encoders, the
// FiLM-conditioned decoder, the per-step CUDA graph and the 1000-step DDPM loop.
//
// Reference call stack replaced (SURVEY §3.1):
//   ContextDiffusionModel.predict_batch_with_aux   msd/models/diffusion/models.py:340-400
//   ContinuousContextTransformer.encode / .decode  msd/models/diffusion/network.py:537-573
//   eval_scan / eval_step / ddpm_step              msd/models/diffusion/diffusion_utils.py:382-476
//
// Exact algebraic shortcuts relative to the graph as written (each proven equal to the oracle
// in tests/):
//   * cross-attention K/V of every decoder layer are projected once per msd_encode (they do not
//     depend on the diffusion step; network.py:217-230 recomputes them every call);
//   * the unconditional pass skips cross-attention: with encodings and masks multiplied by 0
//     (models.py:376-377) zero_activations_if_masked makes the branch exactly 0;
//   * time_emb_dense0/1 + every FiLM Dense depend only on the step index -> tabulated at load.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/msd_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace msd {

// ---------------------------------------------------------------------------
// error string
// ---------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---------------------------------------------------------------------------
// per-launch profiling recorder
// ---------------------------------------------------------------------------
struct ProfRecorder {
  struct Rec { int cls; double flops, bytes; cudaEvent_t e0, e1; };
  std::vector<Rec> recs;
};
ProfRecorder* g_prof = nullptr;
thread_local bool g_pdl_skip_next = false;
bool g_use_pdl = [] {
  const char* v = getenv("MSD_PDL");
  return !(v && v[0] == '0');
}();
void prof_begin(int cls, double flops, double bytes, cudaStream_t st) {
  ProfRecorder::Rec r;
  r.cls = cls; r.flops = flops; r.bytes = bytes;
  cudaEventCreate(&r.e0);
  cudaEventCreate(&r.e1);
  cudaEventRecord(r.e0, st);
  g_prof->recs.push_back(r);
}
void prof_end(cudaStream_t st) { cudaEventRecord(g_prof->recs.back().e1, st); }

// ---------------------------------------------------------------------------
// TMA tensor map encoder (driver entry point resolved through the runtime)
// ---------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;

static int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                        uint64_t ld, uint32_t box_rows, int elem_bytes, int inner_bytes = 128);

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t ld, uint32_t box_rows) {
  return make_tmap_2d(out, base, rows, cols, ld, box_rows, 2);
}

static int make_tmap_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                        uint64_t ld, uint32_t box_rows, int elem_bytes, int inner_bytes) {
  if (g_encode == nullptr) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    MSD_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    MSD_REQUIRE(fn != nullptr && qres == cudaDriverEntryPointSuccess,
                "cuTensorMapEncodeTiled not available from this driver");
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  MSD_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (ld * elem_bytes) % 16 == 0,
              "tensor map: base/stride must be 16-byte aligned (ld=%llu)", (unsigned long long)ld);
  MSD_REQUIRE(box_rows >= 1 && box_rows <= 256, "tensor map: box rows %u out of range", box_rows);
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * elem_bytes};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(inner_bytes / elem_bytes), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                             : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                        2, const_cast<void*>(base), gdim,
                        gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        inner_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MSD_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with %d (rows=%llu cols=%llu ld=%llu)",
              (int)r, (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld);
  return 0;
}

// ---------------------------------------------------------------------------
// device memory helper
// ---------------------------------------------------------------------------
struct Arena {
  std::vector<void*> ptrs;
  size_t total = 0;
  template <typename T>
  int alloc(T** out, size_t count) {
    void* p = nullptr;
    size_t bytes = count * sizeof(T);
    if (bytes == 0) bytes = 16;
    MSD_CUDA_CHECK(cudaMalloc(&p, bytes));
    ptrs.push_back(p);
    total += bytes;
    *out = reinterpret_cast<T*>(p);
    return 0;
  }
  void release() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
  }
};

struct AttnWeights {
  bf16* qkv = nullptr;  // [3*hh, d]   (query | key | value rows)
  bf16* out = nullptr;  // [d, hh]
};
struct MlpWeights {
  bf16* wi = nullptr;  // [2F, d] rows interleaved 32 x wi_0 | 32 x wi_1
  bf16* wo = nullptr;  // [d, F]
};
struct EncLayer {
  float* ln_attn = nullptr;
  float* ln_mlp = nullptr;
  AttnWeights attn;
  MlpWeights mlp;
};
struct DecLayer {
  float* ln_self = nullptr;
  float* ln_cross = nullptr;
  float* ln_mlp = nullptr;
  AttnWeights self_attn;
  // concat_encodings: one attention over [tokens | context]; sum_cross_attends: one per source
  // with q stacked along N ([2*hh, d]) and out stacked along K ([d, 2*hh]) so that both sources
  // still cost one projection GEMM each way.
  bf16* cross_q = nullptr;    // [hh, d] | [2*hh, d]
  bf16* cross_kv = nullptr;   // [2*hh, d]  (key | value rows), source 0 (tokens) or both
  bf16* cross_kv1 = nullptr;  // [2*hh, d]  source 1 (context), sum_cross_attends only
  bf16* cross_out = nullptr;  // [d, hh] | [d, 2*hh]
  MlpWeights mlp;
};
struct Encoder {
  std::vector<EncLayer> layers;
  float* final_norm = nullptr;
  float* pos = nullptr;  // [len, d]
};

}  // namespace msd

using namespace msd;

// most column tiles a residual projection can have (narrowest tile: 64 columns of d <= 1024)
static constexpr size_t kSsParts = 16;

struct msd_ctx {
  msd_config cfg;
  int device = 0;
  // derived sizes
  int d = 0, H = 0, hh = 0, F = 0, T = 0, N = 0, C = 0, Mkv = 0, nd = 0, Bmax = 0, passes = 2;
  // fp32-accurate mode (cfg.precision == 1): every GEMM runs as a 3 x bf16 split-precision product
  // (A = [hi | lo | hi], W = [hi | hi | lo], K tripled: ks == 3), q/k/v and the cross K/V cache
  // are fp32, attention is the fp32 kernel and its output / the gated-GELU output are split again.
  bool acc = false;
  int ks = 1;
  bool weights_loaded = false;
  Arena arena;
  cudaStream_t work = nullptr, work2 = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr, ev_fork = nullptr, ev_join = nullptr;
  bool two_streams = false;

  // ---- parameters
  float* tok_emb = nullptr;  // [vocab, d] f32
  Encoder tok_enc, ctx_enc;
  bf16* ctx_in_proj = nullptr;  // [d, 3*nd] split [hi|hi|lo]
  bf16* dec_in_proj = nullptr;  // [d, 3*nd]
  float* dec_pos = nullptr;     // [N, d]
  std::vector<DecLayer> dec;
  float* dec_norm = nullptr;
  bf16* spec_out = nullptr;   // [nd, 3*d] split [hi|hi|lo]
  float* film = nullptr;      // [steps, 2*L, 2*d]
  float* coef = nullptr;      // [steps, MSD_STEP_COLS] device
  uint32_t* rng_keys = nullptr;  // [steps + 1, 2] jax.random keys of the current seed (rng_kind 1)
  unsigned long long rng_keys_seed = ~0ull;
  // per-row noise streams (msd_sample_rows): jax keys [Bmax][steps + 1][2] and Philox seeds [Bmax]
  // of each batch row's own seed, device; host copies of the seeds they were built from
  uint32_t* row_keys = nullptr;
  unsigned long long* row_seeds = nullptr;
  std::vector<unsigned long long> row_seeds_host;
  std::vector<char> row_keys_valid;
  std::vector<float> coef_host;

  // ---- activations (decoder, rows = passes*B*N)
  float* x = nullptr;      // residual stream f32 [R, d]
  bf16* xn = nullptr;      // normalised input [R, 3*d]
  // (acc: the q/k/v buffers and the K/V cache hold fp32, the GEMM-input buffers are ks x wider)
  bf16* qkv = nullptr;     // [R, 3*hh]      acc: f32 [R, 3*hh]
  bf16* attn = nullptr;    // [R, ks*hh]
  bf16* hmid = nullptr;    // [R, ks*F]
  bf16* qc = nullptr;      // [B*N, hh] (sum_cross_attends: [B*N, 2*hh])      acc: f32
  bf16* attn2 = nullptr;   // [B*N, ks*2*hh] outputs of the two cross-attentions (sum_cross_attends)
  float* attn_part_o = nullptr;   // split-KV partials of the cross-attention [B*N*H*8, 64]
  float* attn_part_ml = nullptr;  // [B*N*H*8, 2]
  float* attn_part_o2 = nullptr;  // second scratch set: sum_cross_attends launches two cross-
  float* attn_part_ml2 = nullptr; //   attentions back to back (PDL lets them overlap)
  // deferred normalisation (bf16 mode; kernels.h GemmPrep / GemmRowScale): no stand-alone rmsnorm
  // kernels inside the decoder layers
  bool fused_norm = false;
  float* gtab = nullptr;      // [steps, 2*Ld, d]  gamma * (1 + FiLM scale): j = 2l self, 2l+1 mlp
  float* btab_qkv = nullptr;  // [steps, Ld, 3*hh] FiLM bias row through the QKV weights
  float* btab_wi = nullptr;   // [steps, Ld, 2*F]  FiLM bias row through the packed wi weights
  float* ss_x = nullptr;      // partial row sums of squares [kSsParts, R]: stream entering a layer
  float* ss_so = nullptr;     //   ... after the self-attention projection
  float* ss_co = nullptr;     //   ... after the cross-attention projection
  float* eps = nullptr;    // [R, nd]
  float* z = nullptr;      // [B*N*nd]
  bf16* z_split = nullptr; // [B*N, 3*nd]
  bf16* kv_cache = nullptr;  // [L][B*Mkv, 2*hh]      acc: f32
  bf16* enc = nullptr;       // [B*Mkv, ks*d]
  // ---- activations (encoders, rows = B*T)
  float* ex = nullptr;
  bf16* exn = nullptr;
  bf16* eqkv = nullptr;
  bf16* eattn = nullptr;
  bf16* eh = nullptr;
  bf16* ctx_split = nullptr;  // [B*C, 3*nd]
  uint32_t* mask_bits = nullptr;  // [B, Mkv/32]
  int* ctx_seq_len = nullptr;     // [B]
  RunArgs* run = nullptr;         // per-call arguments + step index, device memory
  int* d_step = nullptr;          // == &run->step

  // ---- classifier-free guidance split over two GPUs (msd_p2p_*): exchange buffer of this GPU
  // ([2 parities][Bmax*N*nd] eps values + flag words; the peer writes into it) and the peer's,
  // mapped through CUDA IPC
  float* xchg = nullptr;
  float* xchg_peer = nullptr;
  int xrole = 0;                    // 0 off, 1 this GPU runs the conditional pass, 2 the unconditional
  unsigned long long xcalls = 0;    // msd_sample calls since the attach (same on both ranks)

  int cur_batch = 0;
  // per-step graph: depends on the batch size only (noise / output / seed / step live in `run`)
  cudaGraphExec_t graph_exec = nullptr;
  int graph_batch = -1;
  unsigned long long graph_nodes = 0;
};

namespace msd {

// ---------------------------------------------------------------------------
// host-side scalar tables
// ---------------------------------------------------------------------------
// Cosine log-SNR, diffusion_utils.py:181-187, evaluated in float like the reference's fp32 jnp.
static float logsnr_cosine(float t) {
  const double b = atan(exp(-0.5 * 20.0));
  const double a = atan(exp(-0.5 * -20.0)) - b;
  const float arg = static_cast<float>(a) * t + static_cast<float>(b);
  return -2.0f * logf(tanf(arg));
}

// Linear-beta log-SNR, diffusion_utils.py:189-199: float64 table of
// log(alphas_cumprod) - log1p(-alphas_cumprod) clipped to [-20, 20], then jnp.interp over
// linspace(0, 1, num_steps) in float32.
struct LinearSchedule {
  std::vector<float> xp, fp;
  void build(double start, double stop, int n) {
    xp.resize(n); fp.resize(n);
    double cum = 1.0;
    for (int i = 0; i < n; ++i) {
      const double beta = n > 1 ? start + (stop - start) * static_cast<double>(i) / (n - 1) : start;
      cum *= 1.0 - beta;
      double l = log(cum) - log1p(-cum);
      l = l < -20.0 ? -20.0 : (l > 20.0 ? 20.0 : l);
      fp[i] = static_cast<float>(l);
      xp[i] = static_cast<float>(n > 1 ? static_cast<double>(i) / (n - 1) : 0.0);
    }
    if (n > 1) xp[n - 1] = 1.0f;
  }
  float at(float t) const {
    const int n = static_cast<int>(xp.size());
    if (n == 1) return fp[0];
    if (t < xp[0]) return fp[0];
    if (t > xp[n - 1]) return fp[n - 1];
    int i = static_cast<int>(std::upper_bound(xp.begin(), xp.end(), t) - xp.begin());  // side='right'
    i = i < 1 ? 1 : (i > n - 1 ? n - 1 : i);
    const float df = fp[i] - fp[i - 1], dx = xp[i] - xp[i - 1], delta = t - xp[i - 1];
    return dx == 0.f ? fp[i] : fp[i - 1] + (delta / dx) * df;
  }
};

// Threefry-2x32, 20 rounds (host twin of the device function in elementwise.cu)
static void threefry2x32_host(uint32_t k0, uint32_t k1, uint32_t x0, uint32_t x1, uint32_t* out) {
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  static const int rot[2][4] = {{13, 15, 26, 6}, {17, 29, 16, 24}};
  x0 += ks[0];
  x1 += ks[1];
  for (int g = 0; g < 5; ++g) {
    for (int j = 0; j < 4; ++j) {
      x0 += x1;
      x1 = ((x1 << rot[g & 1][j]) | (x1 >> (32 - rot[g & 1][j]))) ^ x0;
    }
    x0 += ks[(g + 1) % 3];
    x1 += ks[(g + 2) % 3] + static_cast<uint32_t>(g + 1);
  }
  out[0] = x0;
  out[1] = x1;
}

static void build_step_table(const msd_config& c, std::vector<float>& tab) {
  const int n = c.num_steps;
  tab.assign(static_cast<size_t>(n) * MSD_STEP_COLS, 0.f);
  LinearSchedule lin_s, lin_t;
  if (c.sampler_schedule == 1) lin_s.build(c.sampler_beta_start, c.sampler_beta_stop, n);
  if (c.train_schedule == 1) lin_t.build(c.train_beta_start, c.train_beta_stop, c.train_num_steps);
  auto logsnr_sampler = [&](float t) { return c.sampler_schedule == 1 ? lin_s.at(t) : logsnr_cosine(t); };
  auto logsnr_train = [&](float t) { return c.train_schedule == 1 ? lin_t.at(t) : logsnr_cosine(t); };
  auto sigmoidf = [](float v) { return 1.0f / (1.0f + expf(-v)); };
  auto log_sigmoidf = [](float v) { return v < 0.f ? v - log1pf(expf(v)) : -log1pf(expf(-v)); };
  for (int i = 0; i < n; ++i) {
    const float t = (static_cast<float>(i) + 1.0f) / static_cast<float>(n);
    const float s = static_cast<float>(i) / static_cast<float>(n);
    const float lt = logsnr_sampler(t), ls = logsnr_sampler(s), ltr = logsnr_train(t);
    float* r = &tab[static_cast<size_t>(i) * MSD_STEP_COLS];
    // predict_x0_from_eps (215-222): x0 = sqrt(1+e^-lt) * (z - eps * rsqrt(1+e^lt))
    r[0] = sqrtf(1.0f + expf(-lt));
    r[1] = 1.0f / sqrtf(1.0f + expf(lt));
    if (c.sampler == 0) {
      // diffusion_reverse (120-163)
      const float alpha_st = sqrtf((1.0f + expf(-lt)) / (1.0f + expf(-ls)));
      const float alpha_s = sqrtf(sigmoidf(ls));
      const float rr = expf(lt - ls);
      const float omr = -expm1f(lt - ls);
      float var;
      if (c.logvar_type == 0) {
        var = omr * sigmoidf(-lt);
      } else if (c.logvar_type == 1) {
        var = omr * sigmoidf(-ls);
      } else {
        // log1mexp (100-106) of x = ls - lt > 0, then the log-space interpolation (148-156)
        const float x = ls - lt;
        const float l1mr = x > logf(2.0f) ? log1pf(-expf(-x)) : logf(-expm1f(-x));
        const float min_logvar = l1mr + log_sigmoidf(-ls), max_logvar = l1mr + log_sigmoidf(-lt);
        var = expf(c.logvar_frac * max_logvar + (1.0f - c.logvar_frac) * min_logvar);
      }
      r[2] = rr * alpha_st;
      r[3] = omr * alpha_s;
      r[4] = sqrtf(var);
    } else {
      // ddim_step (369-379): z_s = alpha_s x0 + stdv_s eps
      r[2] = sqrtf(sigmoidf(-ls));
      r[3] = sqrtf(sigmoidf(ls));
      r[4] = 0.0f;
    }
    r[5] = (i == 0) ? 1.0f : 0.0f;
    r[6] = lt;
    r[7] = ls;
    // _get_x0_and_eps_from_model_output (288-321) at the TRAIN schedule's logsnr(time):
    // eps = p0 z + p1 out, x0 = q0 z + q1 out
    const float A = sqrtf(1.0f + expf(-ltr)), Bc = 1.0f / sqrtf(1.0f + expf(ltr));   // x0 from eps
    const float C = sqrtf(1.0f + expf(ltr)), D = 1.0f / sqrtf(1.0f + expf(-ltr));   // eps from x0
    if (c.model_output == 0) {
      r[8] = 0.f; r[9] = 1.f; r[10] = A; r[11] = -A * Bc;
    } else if (c.model_output == 1) {
      r[8] = C; r[9] = -C * D; r[10] = 0.f; r[11] = 1.f;
    } else {
      const float al = sqrtf(sigmoidf(ltr)), sg = sqrtf(sigmoidf(-ltr));  // x0 = al z - sg v (225-233)
      r[10] = al; r[11] = -sg;
      r[8] = C * (1.0f - D * al); r[9] = C * D * sg;
    }
    // predict_eps_from_x0 (205-212) at the sampler's logsnr_t
    r[12] = sqrtf(1.0f + expf(lt));
    r[13] = 1.0f / sqrtf(1.0f + expf(-lt));
    r[14] = ltr;
  }
}

// get_timing_signal_1d (diffusion_utils.py:69-97) for every step's time, host float math.
static void build_timing_table(const msd_config& c, std::vector<float>& tab) {
  const int n = c.num_steps, d = c.emb_dim, half = d / 2;
  tab.assign(static_cast<size_t>(n) * d, 0.f);
  const double inc = log(static_cast<double>(c.max_decoder_noise_time) / 1.0) / (half - 1.0);
  const float incf = static_cast<float>(-inc);
  for (int i = 0; i < n; ++i) {
    const float t = (static_cast<float>(i) + 1.0f) / static_cast<float>(n);
    const float pos = t * c.max_decoder_noise_time;
    for (int k = 0; k < half; ++k) {
      const float inv = expf(static_cast<float>(k) * incf);
      const float st = pos * inv;
      tab[static_cast<size_t>(i) * d + k] = sinf(st);
      tab[static_cast<size_t>(i) * d + half + k] = cosf(st);
    }
  }
}

// ---------------------------------------------------------------------------
// weight loading
// ---------------------------------------------------------------------------
struct Loader {
  int ks = 1;  // 3 in the fp32-accurate mode: every weight is packed [hi | hi | lo] along K
  std::unordered_map<std::string, const msd_tensor*> map;
  float* stage = nullptr;  // device staging buffers
  float* stage2 = nullptr;
  size_t stage_elems = 0;
  cudaStream_t st = nullptr;

  const msd_tensor* find(const std::string& name, int64_t s0, int64_t s1) {
    auto it = map.find(name);
    if (it == map.end()) {
      set_error("missing parameter '%s'", name.c_str());
      return nullptr;
    }
    const msd_tensor* t = it->second;
    const int64_t g0 = t->shape[0], g1 = t->ndim > 1 ? t->shape[1] : 1;
    if (g0 != s0 || g1 != s1 || t->ndim > 2) {
      set_error("parameter '%s' has shape [%lld,%lld], expected [%lld,%lld]", name.c_str(),
                (long long)g0, (long long)g1, (long long)s0, (long long)s1);
      return nullptr;
    }
    return t;
  }
  // upload to staging buffer `which` and return the device pointer
  int upload(const msd_tensor* t, int which, const float** dev) {
    size_t n = 1;
    for (int i = 0; i < t->ndim; ++i) n *= static_cast<size_t>(t->shape[i]);
    MSD_REQUIRE(n <= stage_elems, "staging buffer too small for '%s'", t->name);
    float* dst = which ? stage2 : stage;
    MSD_CUDA_CHECK(cudaMemcpyAsync(dst, t->data, n * sizeof(float), cudaMemcpyHostToDevice, st));
    *dev = dst;
    return 0;
  }
};

#define MSD_TRY(expr)        \
  do {                       \
    int _rc = (expr);        \
    if (_rc != 0) return _rc; \
  } while (0)

static int load_f32(Loader& L, Arena& A, const std::string& name, int64_t s0, int64_t s1,
                    float** out) {
  const msd_tensor* t = L.find(name, s0, s1);
  if (!t) return -3;
  MSD_TRY(A.alloc(out, static_cast<size_t>(s0 * s1)));
  MSD_CUDA_CHECK(cudaMemcpyAsync(*out, t->data, static_cast<size_t>(s0 * s1) * sizeof(float),
                                 cudaMemcpyHostToDevice, L.st));
  return 0;
}

// W [K, N] f32 (reference layout) -> dst rows [n_off, n_off+N) x cols [k_off, k_off+K) bf16 of
// a matrix with `ldd` logical columns; in the fp32-accurate mode the matrix is 3*ldd wide and
// holds [hi | hi | lo] of the whole logical matrix.
static int pack_into(Loader& L, const std::string& name, int K, int N, bf16* dst, int ldd,
                     int n_off, int k_off) {
  const msd_tensor* t = L.find(name, K, N);
  if (!t) return -3;
  const float* dev = nullptr;
  MSD_TRY(L.upload(t, 0, &dev));
  if (L.ks == 1) {
    MSD_TRY(launch_pack_weight(dev, K, N, dst, ldd, n_off, k_off, 0, L.st));
  } else {
    MSD_TRY(launch_pack_weight(dev, K, N, dst, 3 * ldd, n_off, k_off, 0, L.st));
    MSD_TRY(launch_pack_weight(dev, K, N, dst, 3 * ldd, n_off, ldd + k_off, 0, L.st));
    MSD_TRY(launch_pack_weight(dev, K, N, dst, 3 * ldd, n_off, 2 * ldd + k_off, 1, L.st));
  }
  MSD_CUDA_CHECK(cudaStreamSynchronize(L.st));  // staging buffer is reused
  return 0;
}

static int load_attn(Loader& L, Arena& A, const std::string& prefix, int d, int hh, AttnWeights* w) {
  MSD_TRY(A.alloc(&w->qkv, static_cast<size_t>(3) * hh * d * L.ks));
  MSD_TRY(A.alloc(&w->out, static_cast<size_t>(d) * hh * L.ks));
  MSD_TRY(pack_into(L, prefix + "/query/kernel", d, hh, w->qkv, d, 0, 0));
  MSD_TRY(pack_into(L, prefix + "/key/kernel", d, hh, w->qkv, d, hh, 0));
  MSD_TRY(pack_into(L, prefix + "/value/kernel", d, hh, w->qkv, d, 2 * hh, 0));
  MSD_TRY(pack_into(L, prefix + "/out/kernel", hh, d, w->out, hh, 0, 0));
  return 0;
}

static int load_mlp(Loader& L, Arena& A, const std::string& prefix, int d, int F, MlpWeights* w) {
  MSD_TRY(A.alloc(&w->wi, static_cast<size_t>(2) * F * d * L.ks));
  MSD_TRY(A.alloc(&w->wo, static_cast<size_t>(d) * F * L.ks));
  const msd_tensor* t0 = L.find(prefix + "/wi_0/kernel", d, F);
  const msd_tensor* t1 = L.find(prefix + "/wi_1/kernel", d, F);
  if (!t0 || !t1) return -3;
  const float *d0 = nullptr, *d1 = nullptr;
  MSD_TRY(L.upload(t0, 0, &d0));
  MSD_TRY(L.upload(t1, 1, &d1));
  if (L.ks == 1) {
    MSD_TRY(launch_pack_gated(d0, d1, d, F, w->wi, d, L.st));
  } else {
    MSD_TRY(launch_pack_gated(d0, d1, d, F, w->wi, 3 * d, L.st, 0, 0));
    MSD_TRY(launch_pack_gated(d0, d1, d, F, w->wi, 3 * d, L.st, d, 0));
    MSD_TRY(launch_pack_gated(d0, d1, d, F, w->wi, 3 * d, L.st, 2 * d, 1));
  }
  MSD_CUDA_CHECK(cudaStreamSynchronize(L.st));
  MSD_TRY(pack_into(L, prefix + "/wo/kernel", F, d, w->wo, F, 0, 0));
  return 0;
}

// split-precision pack: dst [N, 3K] = [hi | hi | lo] of W^T
static int pack_split3(Loader& L, const std::string& name, int K, int N, bf16* dst) {
  const msd_tensor* t = L.find(name, K, N);
  if (!t) return -3;
  const float* dev = nullptr;
  MSD_TRY(L.upload(t, 0, &dev));
  MSD_TRY(launch_pack_weight(dev, K, N, dst, 3 * K, 0, 0, 0, L.st));
  MSD_TRY(launch_pack_weight(dev, K, N, dst, 3 * K, 0, K, 0, L.st));
  MSD_TRY(launch_pack_weight(dev, K, N, dst, 3 * K, 0, 2 * K, 1, L.st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(L.st));
  return 0;
}

static int load_encoder(Loader& L, Arena& A, const std::string& name, int layers, int len, int d,
                        int hh, int F, Encoder* e) {
  e->layers.resize(layers);
  MSD_TRY(load_f32(L, A, name + "/Embed_0/embedding", len, d, &e->pos));
  for (int l = 0; l < layers; ++l) {
    const std::string p = name + "/layers_" + std::to_string(l);
    EncLayer& el = e->layers[l];
    MSD_TRY(load_f32(L, A, p + "/pre_attention_layer_norm/scale", d, 1, &el.ln_attn));
    MSD_TRY(load_attn(L, A, p + "/attention", d, hh, &el.attn));
    MSD_TRY(load_f32(L, A, p + "/pre_mlp_layer_norm/scale", d, 1, &el.ln_mlp));
    MSD_TRY(load_mlp(L, A, p + "/mlp", d, F, &el.mlp));
  }
  MSD_TRY(load_f32(L, A, name + "/encoder_norm/scale", d, 1, &e->final_norm));
  return 0;
}

static int load_all(msd_ctx* c, Loader& L) {
  Arena& A = c->arena;
  const msd_config& g = c->cfg;
  const int d = c->d, hh = c->hh, F = c->F, nd = c->nd;
  MSD_TRY(load_f32(L, A, "token_encoder/token_embedder/embedding", g.vocab_size, d, &c->tok_emb));
  MSD_TRY(load_encoder(L, A, "token_encoder", g.num_encoder_layers, c->T, d, hh, F, &c->tok_enc));
  MSD_TRY(load_encoder(L, A, "continuous_encoder", g.num_encoder_layers, c->C, d, hh, F,
                       &c->ctx_enc));
  MSD_TRY(A.alloc(&c->ctx_in_proj, static_cast<size_t>(d) * 3 * nd));
  MSD_TRY(pack_split3(L, "continuous_encoder/input_proj/kernel", nd, d, c->ctx_in_proj));
  MSD_TRY(A.alloc(&c->dec_in_proj, static_cast<size_t>(d) * 3 * nd));
  MSD_TRY(pack_split3(L, "decoder/continuous_inputs_projection/kernel", nd, d, c->dec_in_proj));
  MSD_TRY(load_f32(L, A, "decoder/Embed_0/embedding", c->N, d, &c->dec_pos));
  c->dec.resize(g.num_decoder_layers);
  for (int l = 0; l < g.num_decoder_layers; ++l) {
    const std::string p = "decoder/layers_" + std::to_string(l);
    DecLayer& dl = c->dec[l];
    MSD_TRY(load_f32(L, A, p + "/pre_self_attention_layer_norm/scale", d, 1, &dl.ln_self));
    MSD_TRY(load_attn(L, A, p + "/self_attention", d, hh, &dl.self_attn));
    MSD_TRY(load_f32(L, A, p + "/pre_cross_attention_layer_norm/scale", d, 1, &dl.ln_cross));
    const int nsrc = g.cross_attend_style == 1 ? 2 : 1;
    MSD_TRY(A.alloc(&dl.cross_q, static_cast<size_t>(nsrc) * hh * d * L.ks));
    MSD_TRY(A.alloc(&dl.cross_kv, static_cast<size_t>(2) * hh * d * L.ks));
    if (nsrc == 2) MSD_TRY(A.alloc(&dl.cross_kv1, static_cast<size_t>(2) * hh * d * L.ks));
    MSD_TRY(A.alloc(&dl.cross_out, static_cast<size_t>(d) * nsrc * hh * L.ks));
    for (int sidx = 0; sidx < nsrc; ++sidx) {
      const std::string x = p + "/MultiHeadDotProductAttention_" + std::to_string(sidx);
      bf16* kvw = sidx == 0 ? dl.cross_kv : dl.cross_kv1;
      MSD_TRY(pack_into(L, x + "/query/kernel", d, hh, dl.cross_q, d, sidx * hh, 0));
      MSD_TRY(pack_into(L, x + "/key/kernel", d, hh, kvw, d, 0, 0));
      MSD_TRY(pack_into(L, x + "/value/kernel", d, hh, kvw, d, hh, 0));
      MSD_TRY(pack_into(L, x + "/out/kernel", hh, d, dl.cross_out, nsrc * hh, 0, sidx * hh));
    }
    MSD_TRY(load_f32(L, A, p + "/pre_mlp_layer_norm/scale", d, 1, &dl.ln_mlp));
    MSD_TRY(load_mlp(L, A, p + "/mlp", d, F, &dl.mlp));
  }
  MSD_TRY(load_f32(L, A, "decoder/decoder_norm/scale", d, 1, &c->dec_norm));
  MSD_TRY(A.alloc(&c->spec_out, static_cast<size_t>(nd) * 3 * d));
  MSD_TRY(pack_split3(L, "decoder/spec_out_dense/kernel", d, nd, c->spec_out));

  // ---- timestep conditioning tables (network.py:377-394; layers.py:652-666), all fp32
  const int steps = g.num_steps, Ld = g.num_decoder_layers;
  std::vector<float> timing;
  build_timing_table(g, timing);
  float *d_timing = nullptr, *c1 = nullptr, *c2 = nullptr;
  MSD_CUDA_CHECK(cudaMalloc(&d_timing, timing.size() * sizeof(float)));
  MSD_CUDA_CHECK(cudaMalloc(&c1, static_cast<size_t>(steps) * 4 * d * sizeof(float)));
  MSD_CUDA_CHECK(cudaMalloc(&c2, static_cast<size_t>(steps) * 4 * d * sizeof(float)));
  int rc = 0;
  do {
    if (cudaMemcpyAsync(d_timing, timing.data(), timing.size() * sizeof(float),
                        cudaMemcpyHostToDevice, L.st) != cudaSuccess) { rc = -2; break; }
    const msd_tensor* t0 = L.find("decoder/time_emb_dense0/kernel", d, 4 * d);
    const msd_tensor* t1 = L.find("decoder/time_emb_dense1/kernel", 4 * d, 4 * d);
    if (!t0 || !t1) { rc = -3; break; }
    const float* dev = nullptr;
    if ((rc = L.upload(t0, 0, &dev))) break;
    if ((rc = launch_sgemm_f32(d_timing, dev, c1, 4 * d, steps, 4 * d, d, 1, L.st))) break;
    if (cudaStreamSynchronize(L.st) != cudaSuccess) { rc = -2; break; }
    if ((rc = L.upload(t1, 0, &dev))) break;
    if ((rc = launch_sgemm_f32(c1, dev, c2, 4 * d, steps, 4 * d, 4 * d, 1, L.st))) break;
    if (cudaStreamSynchronize(L.st) != cudaSuccess) { rc = -2; break; }
    if ((rc = A.alloc(&c->film, static_cast<size_t>(steps) * 2 * Ld * 2 * d))) break;
    for (int l = 0; l < Ld && rc == 0; ++l) {
      for (int f = 0; f < 2 && rc == 0; ++f) {
        const std::string nm = "decoder/layers_" + std::to_string(l) + "/FiLMLayer_" +
                               std::to_string(f) + "/DenseGeneral_0/kernel";
        const msd_tensor* tf = L.find(nm, 4 * d, 2 * d);
        if (!tf) { rc = -3; break; }
        if ((rc = L.upload(tf, 0, &dev))) break;
        float* dst = c->film + static_cast<size_t>(2 * l + f) * 2 * d;
        if ((rc = launch_sgemm_f32(c2, dev, dst, 2 * Ld * 2 * d, steps, 2 * d, 4 * d, 0, L.st))) break;
        if (cudaStreamSynchronize(L.st) != cudaSuccess) { rc = -2; break; }
      }
    }
    if (rc != 0 || !c->fused_norm) break;
    // deferred normalisation: per step and layer, the column gains and the FiLM bias rows pushed
    // through the QKV / wi weights (as the GEMM reads them: packed bf16)
    const int hh = c->hh, F = c->F;
    const long long fstride = static_cast<long long>(2) * Ld * 2 * d;
    if ((rc = A.alloc(&c->gtab, static_cast<size_t>(steps) * 2 * Ld * d))) break;
    if ((rc = A.alloc(&c->btab_qkv, static_cast<size_t>(steps) * Ld * 3 * hh))) break;
    if ((rc = A.alloc(&c->btab_wi, static_cast<size_t>(steps) * Ld * 2 * F))) break;
    for (int l = 0; l < Ld && rc == 0; ++l) {
      const DecLayer& w = c->dec[l];
      for (int f = 0; f < 2 && rc == 0; ++f) {
        const float* film = c->film + static_cast<size_t>(2 * l + f) * 2 * d;
        rc = launch_film_gain(film, fstride, f == 0 ? w.ln_self : w.ln_mlp,
                              c->gtab + static_cast<size_t>(2 * l + f) * d,
                              static_cast<long long>(2) * Ld * d, steps, d, L.st);
      }
      if (rc == 0)
        rc = launch_film_bias(c->film + static_cast<size_t>(2 * l) * 2 * d + d, fstride, w.self_attn.qkv,
                              d, c->btab_qkv + static_cast<size_t>(l) * 3 * hh,
                              static_cast<long long>(Ld) * 3 * hh, steps, 3 * hh, d, L.st);
      if (rc == 0)
        rc = launch_film_bias(c->film + static_cast<size_t>(2 * l + 1) * 2 * d + d, fstride, w.mlp.wi, d,
                              c->btab_wi + static_cast<size_t>(l) * 2 * F,
                              static_cast<long long>(Ld) * 2 * F, steps, 2 * F, d, L.st);
    }
    if (rc == 0 && cudaStreamSynchronize(L.st) != cudaSuccess) rc = -2;
  } while (0);
  cudaFree(d_timing);
  cudaFree(c1);
  cudaFree(c2);
  if (rc == -2) set_error("CUDA error while building conditioning tables: %s",
                          cudaGetErrorString(cudaGetLastError()));
  return rc;
}

// ---------------------------------------------------------------------------
// network building blocks
// ---------------------------------------------------------------------------
static int gemm(const bf16* A, int lda, const bf16* B, int ldb, int M, int N, int K, int epi,
                void* out, int ldo, const float* resid, cudaStream_t st) {
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.A = A; a.B = B; a.M = M; a.N = N; a.K = K; a.lda = lda; a.ldb = ldb;
  a.epilogue = epi; a.out = out; a.ldo = ldo; a.resid = resid;
  return launch_gemm(a, st);
}

// Dense layer over a GEMM-input buffer of logical width K: in the fp32-accurate mode the buffer
// holds [hi | lo | hi] (3K wide) and the packed weight [hi | hi | lo], so one bf16 GEMM with 3K
// computes hi*hi + lo*hi + hi*lo (relative error ~2^-16 per product instead of 2^-8).
static int dense(const msd_ctx* c, const bf16* A, const bf16* W, int M, int N, int K, int epi,
                 void* out, int ldo, const float* resid, cudaStream_t st) {
  return gemm(A, K * c->ks, W, K * c->ks, M, N, K * c->ks, epi, out, ldo, resid, st);
}
// epilogue of a projection whose output feeds the attention (q / k / v): bf16, or fp32 in acc mode
static int epi_qkv(const msd_ctx* c) { return c->acc ? EPI_F32 : EPI_BF16; }
static int epi_gated(const msd_ctx* c) { return c->acc ? EPI_GATED_GELU_SPLIT3 : EPI_GATED_GELU; }
// byte size of an element of the q / k / v / cache buffers
static size_t qkv_elem(const msd_ctx* c) { return c->acc ? 4 : 2; }
static const void* at(const msd_ctx* c, const void* base, size_t elems) {
  return static_cast<const char*>(base) + elems * qkv_elem(c);
}
static void* at(const msd_ctx* c, void* base, size_t elems) {
  return static_cast<char*>(base) + elems * qkv_elem(c);
}

static int gemm_pos(const bf16* A, int lda, const bf16* B, int ldb, int M, int N, int K,
                    float* out, const float* pos, int pos_rows, const int* shift, int dup_rows,
                    cudaStream_t st) {
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.A = A; a.B = B; a.M = M; a.N = N; a.K = K; a.lda = lda; a.ldb = ldb;
  a.epilogue = EPI_POS_F32; a.out = out; a.ldo = N; a.pos = pos; a.pos_rows = pos_rows;
  a.pos_shift = shift; a.dup_rows = dup_rows;
  return launch_gemm(a, st);
}

// Attention over q / k / v views given as (buffer, element offset, leading dimension); the
// element type follows the mode.  O: the output-projection's input buffer of logical width
// `o_width` (bf16 [rows, o_width], acc: [rows, 3 * o_width] = [hi | lo | hi]); head h goes to
// columns o_col + h*64.
struct AttnExtra {
  float* part_o = nullptr; float* part_ml = nullptr;
  int kv_static = 0, kv_batch_rows = 0, kv_row0 = 0;
};
static int attention(const msd_ctx* c, const void* Q, size_t qoff, int ldq, const void* K,
                     size_t koff, int ldk, const void* V, size_t voff, int ldv, bf16* O, int o_width,
                     int o_col, int nb, int H, int Lq, int Lk, const uint32_t* bits,
                     int stride_words, cudaStream_t st, const AttnExtra& x = AttnExtra()) {
  if (c->acc) {
    AttnF32Args a;
    memset(&a, 0, sizeof(a));
    a.Q = static_cast<const float*>(at(c, Q, qoff)); a.ldq = ldq;
    a.K = static_cast<const float*>(at(c, K, koff)); a.ldk = ldk;
    a.V = static_cast<const float*>(at(c, V, voff)); a.ldv = ldv;
    a.O = O + o_col; a.o_third = o_width;
    a.nbatch = nb; a.heads = H; a.Lq = Lq; a.Lk = Lk; a.mask_bits = bits;
    a.mask_stride_words = stride_words; a.kv_batch_rows = x.kv_batch_rows; a.kv_row0 = x.kv_row0;
    a.part_o = x.part_o; a.part_ml = x.part_ml; a.max_splits = 12;
    return launch_attention_f32(a, st);
  }
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.kv_static = x.kv_static; a.kv_batch_rows = x.kv_batch_rows; a.kv_row0 = x.kv_row0;
  a.part_o = x.part_o; a.part_ml = x.part_ml; a.max_splits = 12;
  {
    // tuning / test hook: n > 0 forces a tail of n key blocks on every attention of the step that
    // has more than n blocks of 128 keys (the cross-attentions; the self-attention has 2)
    const char* f = getenv("MSD_ATTN_TAIL");
    const int t = f ? atoi(f) : 0;
    a.tail = (t > 0 && t < Lk / 128) ? t : 0;
  }
  a.Q = static_cast<const bf16*>(at(c, Q, qoff)); a.ldq = ldq;
  a.K = static_cast<const bf16*>(at(c, K, koff)); a.ldk = ldk;
  a.V = static_cast<const bf16*>(at(c, V, voff)); a.ldv = ldv;
  a.O = O + o_col; a.ldo = o_width;
  a.nbatch = nb; a.heads = H; a.Lq = Lq; a.Lk = Lk; a.mask_bits = bits;
  a.mask_stride_words = stride_words;
  return launch_attention(a, st);
}

// rmsnorm (+FiLM) into a GEMM-input buffer of logical width d
static int norm_into(const msd_ctx* c, const float* x, const float* gamma, int rows, bf16* out,
                     const float* film, long long film_offset, cudaStream_t st) {
  const long long fstride = static_cast<long long>(2) * c->cfg.num_decoder_layers * 2 * c->d;
  return launch_rmsnorm(x, gamma, rows, c->d, out, c->d * c->ks, film, film ? c->d_step : nullptr,
                        film ? fstride : 0, film_offset, c->acc ? 1 : 0, st);
}

// EncoderLayer stack (network.py:109-158) + final norm written into the concatenated
// encodings buffer at key offset `dst_off`.
static int run_encoder(msd_ctx* c, const Encoder& e, int B, int len, const uint32_t* bits,
                       int dst_off, cudaStream_t st) {
  const int d = c->d, hh = c->hh, F = c->F, rows = B * len;
  const int stride_words = c->Mkv / 32;
  for (const EncLayer& l : e.layers) {
    MSD_TRY(norm_into(c, c->ex, l.ln_attn, rows, c->exn, nullptr, 0, st));
    MSD_TRY(dense(c, c->exn, l.attn.qkv, rows, 3 * hh, d, epi_qkv(c), c->eqkv, 3 * hh, nullptr, st));
    MSD_TRY(attention(c, c->eqkv, 0, 3 * hh, c->eqkv, hh, 3 * hh, c->eqkv, 2 * hh, 3 * hh, c->eattn,
                      hh, 0, B, c->H, len, len, bits, stride_words, st));
    MSD_TRY(dense(c, c->eattn, l.attn.out, rows, d, hh, EPI_RESID_F32, c->ex, d, c->ex, st));
    MSD_TRY(norm_into(c, c->ex, l.ln_mlp, rows, c->exn, nullptr, 0, st));
    MSD_TRY(dense(c, c->exn, l.mlp.wi, rows, 2 * F, d, epi_gated(c), c->eh, F * c->ks, nullptr, st));
    MSD_TRY(dense(c, c->eh, l.mlp.wo, rows, d, F, EPI_RESID_F32, c->ex, d, c->ex, st));
  }
  MSD_TRY(launch_rmsnorm_rows_remap(c->ex, e.final_norm, B, len, d, c->enc, c->Mkv, dst_off, st,
                                    c->acc ? 1 : 0));
  return 0;
}

// Cross-attention block of a DecoderLayer (network.py:196-235) over `nseg` conditioned segments:
// rows x / xn (scratch) / attn (scratch).  concat_encodings attends the concatenated
// [tokens | context] cache once; sum_cross_attends runs one attention per source (each zeroed
// where its source is fully masked) and sums them inside the stacked output projection.
static int cross_attention_block(msd_ctx* c, const DecLayer& w, int l, float* x, bf16* xn, bf16* attn,
                                 int nseg, cudaStream_t st) {
  const int d = c->d, hh = c->hh, N = c->N, R = nseg * N;
  MSD_TRY(norm_into(c, x, w.ln_cross, R, xn, nullptr, 0, st));
  const size_t kv_off = static_cast<size_t>(l) * c->Bmax * c->Mkv * 2 * hh;  // elements
  AttnExtra ex;
  ex.part_o = c->attn_part_o; ex.part_ml = c->attn_part_ml;
  ex.kv_static = 1;
  if (c->cfg.cross_attend_style == 0) {
    MSD_TRY(dense(c, xn, w.cross_q, R, hh, d, epi_qkv(c), c->qc, hh, nullptr, st));
    MSD_TRY(attention(c, c->qc, 0, hh, c->kv_cache, kv_off, 2 * hh, c->kv_cache, kv_off + hh, 2 * hh,
                      attn, hh, 0, nseg, c->H, N, c->Mkv, c->mask_bits, c->Mkv / 32, st, ex));
    MSD_TRY(dense(c, attn, w.cross_out, R, d, hh, EPI_RESID_F32, x, d, x, st));
    return 0;
  }
  MSD_TRY(dense(c, xn, w.cross_q, R, 2 * hh, d, epi_qkv(c), c->qc, 2 * hh, nullptr, st));
  ex.kv_batch_rows = c->Mkv;
  ex.kv_row0 = 0;
  MSD_TRY(attention(c, c->qc, 0, 2 * hh, c->kv_cache, kv_off, 2 * hh, c->kv_cache, kv_off + hh, 2 * hh,
                    c->attn2, 2 * hh, 0, nseg, c->H, N, c->T, c->mask_bits, c->Mkv / 32, st, ex));
  ex.kv_row0 = c->T;
  ex.part_o = c->attn_part_o2; ex.part_ml = c->attn_part_ml2;
  MSD_TRY(attention(c, c->qc, hh, 2 * hh, c->kv_cache, kv_off, 2 * hh, c->kv_cache, kv_off + hh, 2 * hh,
                    c->attn2, 2 * hh, hh, nseg, c->H, N, c->C, c->mask_bits + c->T / 32, c->Mkv / 32,
                    st, ex));
  MSD_TRY(dense(c, c->attn2, w.cross_out, R, d, 2 * hh, EPI_RESID_F32, x, d, x, st));
  return 0;
}

// The 12 DecoderLayers (network.py:161-258) over segments [seg0, seg0 + nseg) of the row buffers.
// The first `ncross` of these segments cross-attend to the cached encodings (conditional pass;
// the unconditional rows skip the block: with encodings and masks multiplied by 0 it is exactly
// 0); every other kernel batches all rows.
static int decoder_layers(msd_ctx* c, int seg0, int nseg, int ncross, cudaStream_t st) {
  const int d = c->d, hh = c->hh, F = c->F, N = c->N, ks = c->ks;
  const int R = nseg * N;
  const size_t r0 = static_cast<size_t>(seg0) * N;
  const int Ld = c->cfg.num_decoder_layers;
  float* x = c->x + r0 * d;
  bf16* xn = c->xn + r0 * d * ks;  // [rows, ks*d] view of the scratch buffer (disjoint per range)
  const size_t qkv_off = r0 * 3 * hh;
  bf16* attn = c->attn + r0 * hh * ks;
  bf16* hmid = c->hmid + r0 * F * ks;
  for (int l = 0; l < Ld; ++l) {
    const DecLayer& w = c->dec[l];
    // self-attention block (174-193)
    MSD_TRY(norm_into(c, x, w.ln_self, R, xn, c->film, static_cast<long long>(2 * l) * 2 * d, st));
    MSD_TRY(dense(c, xn, w.self_attn.qkv, R, 3 * hh, d, epi_qkv(c), at(c, c->qkv, qkv_off), 3 * hh,
                  nullptr, st));
    MSD_TRY(attention(c, c->qkv, qkv_off, 3 * hh, c->qkv, qkv_off + hh, 3 * hh, c->qkv,
                      qkv_off + 2 * hh, 3 * hh, attn, hh, 0, nseg, c->H, N, N, nullptr, 0, st));
    MSD_TRY(dense(c, attn, w.self_attn.out, R, d, hh, EPI_RESID_F32, x, d, x, st));
    // cross-attention block (196-235), conditioned rows only (the first ncross segments)
    if (ncross > 0) MSD_TRY(cross_attention_block(c, w, l, x, xn, attn, ncross, st));
    // MLP block (241-256)
    MSD_TRY(norm_into(c, x, w.ln_mlp, R, xn, c->film, static_cast<long long>(2 * l + 1) * 2 * d, st));
    MSD_TRY(dense(c, xn, w.mlp.wi, R, 2 * F, d, epi_gated(c), hmid, F * ks, nullptr, st));
    MSD_TRY(dense(c, hmid, w.mlp.wo, R, d, F, EPI_RESID_F32, x, d, x, st));
  }
  return 0;
}

// The same 12 DecoderLayers with DEFERRED NORMALISATION (bf16 mode, one chain; kernels.h GemmPrep /
// GemmRowScale): every pre-norm (+FiLM) of layers.py:632-666 is split into a column gain applied
// where the residual stream is produced and a row scale + bias row applied where the next
// projection's accumulator is drained,
//     (rmsnorm(x) gamma (1 + fs) + fb) W  ==  rsqrt(mean(x^2) + eps) * ((x gamma (1 + fs)) W) + fb W,
// so no stand-alone rmsnorm kernel runs inside the layers (35 fewer kernels per step).
//   xn      bf16 operand of the next projection: x * g' (unnormalised)
//   ss_x    row sums of squares of x entering a layer (prep kernel, then each wo projection)
//   ss_so   ... after the self-attention output projection; ss_co after the cross-attention one
// Rows of the unconditional pass (>= ncross * N) skip the cross-attention block: their operand for
// the MLP is written by the self-attention projection already (g_hi), their row sums stay in ss_so.
static int decoder_layers_fused(msd_ctx* c, int nseg, int ncross, cudaStream_t st) {
  const int d = c->d, hh = c->hh, F = c->F, N = c->N;
  const int R = nseg * N, Rc = ncross * N;
  const int Ld = c->cfg.num_decoder_layers;
  const int nsrc = c->cfg.cross_attend_style == 1 ? 2 : 1;
  const long long gstride = static_cast<long long>(2) * Ld * d;
  const int ss_stride = c->passes * c->Bmax * N;
  float* x = c->x;
  bf16* xn = c->xn;
  auto base_args = [&](const bf16* A, int lda, const bf16* W, int M, int Nn, int K, int epi, void* out,
                       int ldo) {
    GemmArgs a;
    memset(&a, 0, sizeof(a));
    a.A = A; a.B = W; a.M = M; a.N = Nn; a.K = K; a.lda = lda; a.ldb = K;
    a.epilogue = epi; a.out = out; a.ldo = ldo; a.step = c->d_step;
    return a;
  };
  // residual projection + operand / row sums for what follows
  auto resid_prep = [&](const bf16* A, const bf16* W, int M, int K, const float* g_lo, long long s_lo,
                        const float* g_hi, long long s_hi, int split_row, float* ss, int* parts) {
    GemmArgs a = base_args(A, K, W, M, d, K, EPI_RESID_PREP, x, d);
    a.resid = x;
    a.prep.g_lo = g_lo; a.prep.g_lo_step_stride = s_lo;
    a.prep.g_hi = g_hi; a.prep.g_hi_step_stride = s_hi;
    a.prep.split_row = split_row;
    a.prep.a = xn; a.prep.lda = d;
    a.prep.ss = ss; a.prep.ss_stride = ss_stride;
    const int bn = gemm_resolve_block_n(a);   // the partial row sums are per column tile that runs
    MSD_REQUIRE(bn > 0, "resid_prep: no tile width for M=%d d=%d", M, d);
    *parts = d / bn;
    return launch_gemm(a, st);
  };
  auto row_scale = [&](GemmArgs& a, const float* lo, int parts_lo, const float* hi, int parts_hi,
                       int split_row, const float* bias, long long bias_stride) {
    a.rs.ss_lo = lo; a.rs.parts_lo = parts_lo; a.rs.ss_hi = hi; a.rs.parts_hi = parts_hi;
    a.rs.split_row = split_row; a.rs.ss_stride = ss_stride; a.rs.inv_d = 1.0f / static_cast<float>(d);
    a.rs.col_bias = bias; a.rs.bias_step_stride = bias_stride;
  };
  // layer 0: the stream comes from the input projection, not from a residual epilogue
  MSD_TRY(launch_prep_rows(x, c->gtab, gstride, c->d_step, R, d, xn, d, c->ss_x, st));
  int parts_x = 1, parts_so = 1, parts_co = 1;
  for (int l = 0; l < Ld; ++l) {
    const DecLayer& w = c->dec[l];
    const float* g_mlp = c->gtab + static_cast<size_t>(2 * l + 1) * d;
    // self-attention block (174-193)
    {
      GemmArgs a = base_args(xn, d, w.self_attn.qkv, R, 3 * hh, d, EPI_BF16, c->qkv, 3 * hh);
      row_scale(a, c->ss_x, parts_x, c->ss_x, parts_x, R, c->btab_qkv + static_cast<size_t>(l) * 3 * hh,
                static_cast<long long>(Ld) * 3 * hh);
      MSD_TRY(launch_gemm(a, st));
    }
    MSD_TRY(attention(c, c->qkv, 0, 3 * hh, c->qkv, hh, 3 * hh, c->qkv, 2 * hh, 3 * hh, c->attn, hh, 0,
                      nseg, c->H, N, N, nullptr, 0, st));
    // x += attn W_out; rows that cross-attend get the cross pre-norm's gain, the others the MLP's
    MSD_TRY(resid_prep(c->attn, w.self_attn.out, R, hh, Rc > 0 ? w.ln_cross : g_mlp, Rc > 0 ? 0 : gstride,
                       g_mlp, gstride, Rc, c->ss_so, &parts_so));
    // cross-attention block (196-235), conditioned rows only
    if (Rc > 0) {
      GemmArgs a = base_args(xn, d, w.cross_q, Rc, nsrc * hh, d, EPI_BF16, c->qc, nsrc * hh);
      row_scale(a, c->ss_so, parts_so, c->ss_so, parts_so, Rc, nullptr, 0);
      MSD_TRY(launch_gemm(a, st));
      const size_t kv_off = static_cast<size_t>(l) * c->Bmax * c->Mkv * 2 * hh;
      AttnExtra ex;
      ex.part_o = c->attn_part_o; ex.part_ml = c->attn_part_ml;
      ex.kv_static = 1;
      if (nsrc == 1) {
        MSD_TRY(attention(c, c->qc, 0, hh, c->kv_cache, kv_off, 2 * hh, c->kv_cache, kv_off + hh, 2 * hh,
                          c->attn, hh, 0, ncross, c->H, N, c->Mkv, c->mask_bits, c->Mkv / 32, st, ex));
        MSD_TRY(resid_prep(c->attn, w.cross_out, Rc, hh, g_mlp, gstride, g_mlp, gstride, Rc, c->ss_co,
                           &parts_co));
      } else {
        ex.kv_batch_rows = c->Mkv;
        ex.kv_row0 = 0;
        MSD_TRY(attention(c, c->qc, 0, 2 * hh, c->kv_cache, kv_off, 2 * hh, c->kv_cache, kv_off + hh,
                          2 * hh, c->attn2, 2 * hh, 0, ncross, c->H, N, c->T, c->mask_bits, c->Mkv / 32,
                          st, ex));
        ex.kv_row0 = c->T;
        ex.part_o = c->attn_part_o2; ex.part_ml = c->attn_part_ml2;
        MSD_TRY(attention(c, c->qc, hh, 2 * hh, c->kv_cache, kv_off, 2 * hh, c->kv_cache, kv_off + hh,
                          2 * hh, c->attn2, 2 * hh, hh, ncross, c->H, N, c->C, c->mask_bits + c->T / 32,
                          c->Mkv / 32, st, ex));
        MSD_TRY(resid_prep(c->attn2, w.cross_out, Rc, 2 * hh, g_mlp, gstride, g_mlp, gstride, Rc,
                           c->ss_co, &parts_co));
      }
    }
    // MLP block (241-256)
    {
      GemmArgs a = base_args(xn, d, w.mlp.wi, R, 2 * F, d, EPI_GATED_GELU, c->hmid, F);
      if (Rc > 0) row_scale(a, c->ss_co, parts_co, c->ss_so, parts_so, Rc,
                            c->btab_wi + static_cast<size_t>(l) * 2 * F, static_cast<long long>(Ld) * 2 * F);
      else row_scale(a, c->ss_so, parts_so, c->ss_so, parts_so, R,
                     c->btab_wi + static_cast<size_t>(l) * 2 * F, static_cast<long long>(Ld) * 2 * F);
      MSD_TRY(launch_gemm(a, st));
    }
    if (l + 1 < Ld) {
      const float* g_next = c->gtab + static_cast<size_t>(2 * (l + 1)) * d;
      MSD_TRY(resid_prep(c->hmid, w.mlp.wo, R, F, g_next, gstride, g_next, gstride, R, c->ss_x, &parts_x));
    } else {
      // the decoder_norm that follows is a stand-alone (split-precision) kernel reading x itself
      MSD_TRY(dense(c, c->hmid, w.mlp.wo, R, d, F, EPI_RESID_F32, x, d, x, st));
    }
  }
  return 0;
}

// Decoder.__call__ (network.py:360-457) over `total` segments of which the first `ncond`
// cross-attend to the cached encodings.  Input: c->z_split; output: c->eps [total*N, nd].
// With `two_streams` the conditional and unconditional passes -- independent until the guidance
// combine -- run as two concurrent kernel chains (fork/join on c->work2); a measured-slower
// experiment (MSD_TWO_STREAMS=1), see msd_create.
static int run_decoder(msd_ctx* c, int B, int ncond, int total, cudaStream_t st,
                       bool two_streams = false) {
  const int d = c->d, N = c->N, nd = c->nd;
  const int R = total * N;
  // continuous_inputs_projection + position encodings (420-427); both passes start equal.
  // The first kernel of a step is a plain (fully dependent) launch: kernels further down read
  // per-segment constants (cross K/V cache, key mask, step index) ahead of their programmatic
  // dependency wait, which is only sound if everything before this step has completed.
  g_pdl_skip_next = true;
  MSD_TRY(gemm_pos(c->z_split, 3 * nd, c->dec_in_proj, 3 * nd, B * N, d, 3 * nd, c->x, c->dec_pos,
                   N, nullptr, total > B ? B * N : 0, st));
  const int nuncond = total - ncond;
  if (two_streams && ncond > 0 && nuncond > 0) {
    MSD_CUDA_CHECK(cudaEventRecord(c->ev_fork, st));
    MSD_CUDA_CHECK(cudaStreamWaitEvent(c->work2, c->ev_fork, 0));
    g_pdl_skip_next = true;  // first kernel of the side chain depends on another stream
    MSD_TRY(decoder_layers(c, ncond, nuncond, 0, c->work2));
    MSD_TRY(decoder_layers(c, 0, ncond, ncond, st));
    MSD_CUDA_CHECK(cudaEventRecord(c->ev_join, c->work2));
    MSD_CUDA_CHECK(cudaStreamWaitEvent(st, c->ev_join, 0));
    g_pdl_skip_next = true;  // the join kernel has two predecessors
  } else {
    // one chain, both passes batched per kernel except the cross-attention block
    if (c->fused_norm) MSD_TRY(decoder_layers_fused(c, total, ncond, st));
    else MSD_TRY(decoder_layers(c, 0, total, ncond, st));
  }
  // decoder_norm + spec_out_dense in split precision (445-456: fp32 "for stability")
  MSD_TRY(launch_rmsnorm(c->x, c->dec_norm, R, d, c->xn, 3 * d, nullptr, nullptr, 0, 0, 1, st));
  MSD_TRY(gemm(c->xn, 3 * d, c->spec_out, 3 * d, R, nd, 3 * d, EPI_F32, c->eps, nd, nullptr, st));
  return 0;
}

// One reverse-diffusion update.  With `use_run` the per-call arguments and the step index are
// read from c->run (device memory) and the kernel also advances the step (the graph path).
static int sampler_step(msd_ctx* c, int B, const float* noise, unsigned long long seed,
                        float* mel_out, cudaStream_t st, bool use_run) {
  SamplerArgs a;
  memset(&a, 0, sizeof(a));
  a.eps = c->eps; a.z = c->z; a.z_split = c->z_split; a.noise = noise; a.coef = c->coef;
  a.step = c->d_step; a.mel_out = mel_out;
  a.n = static_cast<long long>(B) * c->N * c->nd;
  a.n_dims = c->nd; a.passes = c->passes; a.cond_weight = c->cfg.eval_condition_weight;
  a.clip_x0 = c->cfg.clip_x0; a.ddim = c->cfg.sampler == 1; a.feat_min = c->cfg.feature_min; a.feat_max = c->cfg.feature_max;
  a.seed = seed; a.rng_kind = c->cfg.rng_kind; a.rng_keys = c->rng_keys;
  a.n_row = static_cast<long long>(c->N) * c->nd;
  a.row_keys = c->row_keys; a.row_key_stride = 2 * (static_cast<long long>(c->cfg.num_steps) + 1);
  a.row_seeds = c->row_seeds;
  a.run = use_run ? c->run : nullptr;
  a.film = c->film;
  a.film_step_floats = static_cast<long long>(2) * c->cfg.num_decoder_layers * 2 * c->d;
  if (c->fused_norm) {
    // the layers read the derived tables instead of the FiLM rows
    const long long Ld = c->cfg.num_decoder_layers;
    a.film = nullptr;
    a.pf[0] = c->gtab; a.pf_step_floats[0] = 2 * Ld * c->d;
    a.pf[1] = c->btab_qkv; a.pf_step_floats[1] = Ld * 3 * c->hh;
    a.pf[2] = c->btab_wi; a.pf_step_floats[2] = Ld * 2 * c->F;
  }
  if (use_run && c->xrole != 0) {
    a.passes = 2;   // both passes exist, one of them on the peer GPU
    a.xrole = c->xrole; a.xlocal = c->xchg; a.xpeer = c->xchg_peer;
    a.xparity_floats = static_cast<long long>(c->Bmax) * c->N * c->nd;
    a.xflags_off = 2 * a.xparity_floats;
  }
  return launch_sampler_step(a, st);
}


static int validate(const msd_config* g) {
  MSD_REQUIRE(g->head_dim == 64, "head_dim must be 64 (got %d)", g->head_dim);
  MSD_REQUIRE(g->n_dims == 128, "n_dims must be 128 (got %d)", g->n_dims);
  MSD_REQUIRE(g->emb_dim % 128 == 0 && g->emb_dim <= 1024, "emb_dim must be k*128 <= 1024");
  MSD_REQUIRE(g->mlp_dim % 64 == 0, "mlp_dim must be a multiple of 64");
  MSD_REQUIRE((g->num_heads * 64) % 64 == 0 && g->num_heads > 0, "bad num_heads");
  MSD_REQUIRE(g->inputs_length % 128 == 0 && g->targets_length % 128 == 0 &&
                  g->context_length % 128 == 0,
              "sequence lengths must be multiples of 128");
  MSD_REQUIRE(g->num_steps > 0 && g->max_batch > 0, "num_steps and max_batch must be positive");
  MSD_REQUIRE(g->sampler == 0 || g->sampler == 1, "sampler must be 0 (ddpm) or 1 (ddim)");
  MSD_REQUIRE(g->logvar_type >= 0 && g->logvar_type <= 2, "logvar_type must be 0, 1 or 2");
  MSD_REQUIRE(g->logvar_type != 2 || (g->logvar_frac >= 0.f && g->logvar_frac <= 1.f),
              "logvar_frac must be in [0, 1]");
  MSD_REQUIRE(g->model_output >= 0 && g->model_output <= 2, "model_output must be 0 (eps), 1 (x0) or 2 (v)");
  MSD_REQUIRE((g->sampler_schedule == 0 || g->sampler_schedule == 1) &&
                  (g->train_schedule == 0 || g->train_schedule == 1),
              "schedules must be 0 (cosine) or 1 (linear)");
  MSD_REQUIRE(g->rng_kind == 0 || g->rng_kind == 1, "rng_kind must be 0 (philox) or 1 (jax threefry)");
  MSD_REQUIRE(g->cross_attend_style == 0 || g->cross_attend_style == 1,
              "cross_attend_style must be 0 (concat_encodings) or 1 (sum_cross_attends)");
  MSD_REQUIRE(g->train_schedule == 0 || g->train_num_steps > 0,
              "linear train schedule needs train_num_steps > 0");
  MSD_REQUIRE(g->vocab_size > 0 && g->num_encoder_layers > 0 && g->num_decoder_layers > 0,
              "bad layer/vocab sizes");
  MSD_REQUIRE(g->precision == 0 || g->precision == 1,
              "precision must be 0 (bf16 operands) or 1 (fp32-accurate)");
  return 0;
}

static void drop_graph(msd_ctx* c) {
  if (c->graph_exec) cudaGraphExecDestroy(c->graph_exec);
  c->graph_exec = nullptr;
  c->graph_batch = -1;
}

struct TempBufs {
  std::vector<void*> p;
  ~TempBufs() { for (void* q : p) cudaFree(q); }
  template <typename T> int get(T** out, size_t n) {
    void* q = nullptr;
    MSD_CUDA_CHECK(cudaMalloc(&q, (n ? n : 1) * sizeof(T)));
    p.push_back(q);
    *out = reinterpret_cast<T*>(q);
    return 0;
  }
};

}  // namespace msd

// ===========================================================================
// C ABI
// ===========================================================================
extern "C" {

const char* msd_last_error(void) { return g_err; }
int msd_abi_version(void) { return MSD_B200_ABI_VERSION; }
uint64_t msd_launch_count(void) { return g_launch_count; }

int msd_create(const msd_config* cfg, int device, msd_ctx** out) {
  MSD_REQUIRE(cfg != nullptr && out != nullptr, "msd_create: null argument");
  MSD_TRY(validate(cfg));
  int ndev = 0;
  MSD_CUDA_CHECK(cudaGetDeviceCount(&ndev));
  MSD_REQUIRE(device >= 0 && device < ndev, "msd_create: device %d not present (%d GPUs)", device, ndev);
  MSD_CUDA_CHECK(cudaSetDevice(device));
  cudaDeviceProp prop;
  MSD_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  MSD_REQUIRE(prop.major == 9, "msd_create: device %d is sm_%d%d; this library is sm_90a only",
              device, prop.major, prop.minor);
  MSD_TRY(gemm_configure());
  MSD_TRY(attention_configure());
  MSD_TRY(elementwise_configure());
  msd_ctx* c = new msd_ctx();
  c->cfg = *cfg;
  c->device = device;
  c->d = cfg->emb_dim; c->H = cfg->num_heads; c->hh = cfg->num_heads * 64; c->F = cfg->mlp_dim;
  c->T = cfg->inputs_length; c->N = cfg->targets_length; c->C = cfg->context_length;
  c->Mkv = c->T + c->C; c->nd = cfg->n_dims; c->Bmax = cfg->max_batch;
  c->passes = (cfg->eval_condition_weight != 1.0f) ? 2 : 1;
  c->acc = cfg->precision == 1;
  c->ks = c->acc ? 3 : 1;
  const size_t ks = static_cast<size_t>(c->ks);
  const size_t qe = c->acc ? 2 : 1;  // q / k / v buffers: fp32 = two bf16 slots per element
  Arena& A = c->arena;
  const size_t R = static_cast<size_t>(c->passes) * c->Bmax * c->N;
  const size_t BN = static_cast<size_t>(c->Bmax) * c->N;
  const size_t ER = static_cast<size_t>(c->Bmax) * (c->T > c->C ? c->T : c->C);
  int rc = 0;
  do {
    {
      // Opt-in experiment (MSD_TWO_STREAMS=1): conditional / unconditional passes as two concurrent
      // kernel chains.  Every GEMM / attention CTA owns a whole SM's shared memory, so the chains
      // mostly time-share SMs, and the half-height GEMMs are less efficient -> off by default.
      const char* ts = getenv("MSD_TWO_STREAMS");
      c->two_streams = (ts && ts[0] == '1') && !c->acc;
    }
    if (cudaStreamCreateWithFlags(&c->work, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->work2, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_out, cudaEventDisableTiming) != cudaSuccess) {
      set_error("msd_create: stream/event creation failed");
      rc = -2;
      break;
    }
    if ((rc = A.alloc(&c->x, R * c->d))) break;
    if ((rc = A.alloc(&c->xn, R * 3 * c->d))) break;
    if ((rc = A.alloc(&c->qkv, R * 3 * c->hh * qe))) break;
    if ((rc = A.alloc(&c->attn, R * c->hh * ks))) break;
    if ((rc = A.alloc(&c->hmid, R * c->F * ks))) break;
    if ((rc = A.alloc(&c->qc, BN * c->hh * (cfg->cross_attend_style == 1 ? 2 : 1) * qe))) break;
    if (cfg->cross_attend_style == 1 && (rc = A.alloc(&c->attn2, BN * 2 * c->hh * ks))) break;
    constexpr int kMaxSplits = 12;
    const size_t npart = attention_workspace_floats(c->Bmax, c->H, c->N, kMaxSplits);
    if ((rc = A.alloc(&c->attn_part_o, npart))) break;
    if ((rc = A.alloc(&c->attn_part_ml, BN * c->H * kMaxSplits * 2))) break;
    c->attn_part_o2 = c->attn_part_o; c->attn_part_ml2 = c->attn_part_ml;
    if (cfg->cross_attend_style == 1) {
      if ((rc = A.alloc(&c->attn_part_o2, npart))) break;
      if ((rc = A.alloc(&c->attn_part_ml2, BN * c->H * kMaxSplits * 2))) break;
    }
    {
      // MSD_FUSED_NORM=0: tuning / test hook, keeps the stand-alone rmsnorm kernels
      const char* fn = getenv("MSD_FUSED_NORM");
      c->fused_norm = !c->acc && !c->two_streams && !(fn && fn[0] == '0');
      if (c->fused_norm) {
        if ((rc = A.alloc(&c->ss_x, kSsParts * R))) break;
        if ((rc = A.alloc(&c->ss_so, kSsParts * R))) break;
        if ((rc = A.alloc(&c->ss_co, kSsParts * R))) break;
      }
    }
    if ((rc = A.alloc(&c->eps, R * c->nd))) break;
    if ((rc = A.alloc(&c->z, BN * c->nd))) break;
    if ((rc = A.alloc(&c->z_split, BN * 3 * c->nd))) break;
    if ((rc = A.alloc(&c->kv_cache, static_cast<size_t>(cfg->num_decoder_layers) * c->Bmax *
                                        c->Mkv * 2 * c->hh * qe))) break;
    if ((rc = A.alloc(&c->enc, static_cast<size_t>(c->Bmax) * c->Mkv * c->d * ks))) break;
    if ((rc = A.alloc(&c->ex, ER * c->d))) break;
    if ((rc = A.alloc(&c->exn, ER * c->d * ks))) break;
    if ((rc = A.alloc(&c->eqkv, ER * 3 * c->hh * qe))) break;
    if ((rc = A.alloc(&c->eattn, ER * c->hh * ks))) break;
    if ((rc = A.alloc(&c->eh, ER * c->F * ks))) break;
    if ((rc = A.alloc(&c->ctx_split, static_cast<size_t>(c->Bmax) * c->C * 3 * c->nd))) break;
    if ((rc = A.alloc(&c->mask_bits, static_cast<size_t>(c->Bmax) * (c->Mkv / 32)))) break;
    if ((rc = A.alloc(&c->ctx_seq_len, static_cast<size_t>(c->Bmax)))) break;
    if ((rc = A.alloc(&c->run, 1))) break;
    if (cudaMemset(c->run, 0, sizeof(RunArgs)) != cudaSuccess) {
      set_error("msd_create: cudaMemset failed");
      rc = -2;
      break;
    }
    c->d_step = &c->run->step;
    {
      const size_t xf = 2 * BN * c->nd + 64;
      if ((rc = A.alloc(&c->xchg, xf))) break;
      if (cudaMemset(c->xchg, 0, xf * sizeof(float)) != cudaSuccess) {
        set_error("msd_create: cudaMemset failed");
        rc = -2;
        break;
      }
    }
    if ((rc = A.alloc(&c->coef, static_cast<size_t>(cfg->num_steps) * MSD_STEP_COLS))) break;
    if ((rc = A.alloc(&c->rng_keys, (static_cast<size_t>(cfg->num_steps) + 1) * 2))) break;
    if (cudaMemset(c->rng_keys, 0, (static_cast<size_t>(cfg->num_steps) + 1) * 2 * sizeof(uint32_t)) !=
        cudaSuccess) {
      set_error("msd_create: cudaMemset failed");
      rc = -2;
      break;
    }
    if ((rc = A.alloc(&c->row_keys, static_cast<size_t>(c->Bmax) * (cfg->num_steps + 1) * 2))) break;
    if ((rc = A.alloc(&c->row_seeds, static_cast<size_t>(c->Bmax)))) break;
    c->row_seeds_host.assign(c->Bmax, 0ull);
    c->row_keys_valid.assign(c->Bmax, 0);
    build_step_table(*cfg, c->coef_host);
    if (cudaMemcpy(c->coef, c->coef_host.data(), c->coef_host.size() * sizeof(float),
                   cudaMemcpyHostToDevice) != cudaSuccess) {
      set_error("msd_create: coefficient upload failed");
      rc = -2;
    }
  } while (0);
  if (rc != 0) {
    msd_destroy(c);
    return rc;
  }
  *out = c;
  return 0;
}

void msd_destroy(msd_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  drop_graph(c);
  if (c->xchg_peer) cudaIpcCloseMemHandle(c->xchg_peer);
  c->arena.release();
  if (c->ev_in) cudaEventDestroy(c->ev_in);
  if (c->ev_out) cudaEventDestroy(c->ev_out);
  if (c->ev_fork) cudaEventDestroy(c->ev_fork);
  if (c->ev_join) cudaEventDestroy(c->ev_join);
  if (c->work2) cudaStreamDestroy(c->work2);
  if (c->work) cudaStreamDestroy(c->work);
  delete c;
}

int msd_load_weights(msd_ctx* c, const msd_tensor* tensors, int32_t n) {
  MSD_REQUIRE(c != nullptr && tensors != nullptr && n > 0, "msd_load_weights: null argument");
  MSD_REQUIRE(!c->weights_loaded, "msd_load_weights: weights already loaded for this context");
  MSD_CUDA_CHECK(cudaSetDevice(c->device));
  Loader L;
  size_t biggest = 0;
  for (int i = 0; i < n; ++i) {
    MSD_REQUIRE(tensors[i].name && tensors[i].data && tensors[i].ndim >= 1 && tensors[i].ndim <= 4,
                "msd_load_weights: malformed tensor %d", i);
    L.map[tensors[i].name] = &tensors[i];
    size_t e = 1;
    for (int k = 0; k < tensors[i].ndim; ++k) e *= static_cast<size_t>(tensors[i].shape[k]);
    if (e > biggest) biggest = e;
  }
  L.stage_elems = biggest;
  L.st = c->work;
  L.ks = c->ks;
  MSD_CUDA_CHECK(cudaMalloc(&L.stage, biggest * sizeof(float)));
  if (cudaMalloc(&L.stage2, biggest * sizeof(float)) != cudaSuccess) {
    cudaFree(L.stage);
    set_error("msd_load_weights: staging allocation failed");
    return -2;
  }
  int rc = load_all(c, L);
  cudaError_t e = cudaStreamSynchronize(c->work);
  cudaFree(L.stage);
  cudaFree(L.stage2);
  if (rc == 0 && e != cudaSuccess) {
    set_error("msd_load_weights: %s", cudaGetErrorString(e));
    rc = -2;
  }
  if (rc == 0) c->weights_loaded = true;
  return rc;
}

static int begin_on(msd_ctx* c, cudaStream_t caller) {
  MSD_CUDA_CHECK(cudaSetDevice(c->device));
  MSD_CUDA_CHECK(cudaEventRecord(c->ev_in, caller));
  MSD_CUDA_CHECK(cudaStreamWaitEvent(c->work, c->ev_in, 0));
  return 0;
}
static int end_on(msd_ctx* c, cudaStream_t caller) {
  MSD_CUDA_CHECK(cudaEventRecord(c->ev_out, c->work));
  MSD_CUDA_CHECK(cudaStreamWaitEvent(caller, c->ev_out, 0));
  return 0;
}

int msd_encode(msd_ctx* c, const int32_t* tokens, const float* ctx_features,
               const int32_t* ctx_mask, int32_t batch, void* stream) {
  MSD_REQUIRE(c && tokens && ctx_features && ctx_mask, "msd_encode: null argument");
  MSD_REQUIRE(c->weights_loaded, "msd_encode: call msd_load_weights first");
  MSD_REQUIRE(batch >= 1 && batch <= c->Bmax, "msd_encode: batch %d outside [1, %d]", batch, c->Bmax);
  cudaStream_t caller = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(begin_on(c, caller));
  cudaStream_t st = c->work;
  const int B = batch, d = c->d, hh = c->hh, nd = c->nd;
  MSD_TRY(launch_build_masks(tokens, ctx_mask, B, c->T, c->C, c->mask_bits, c->ctx_seq_len,
                             c->cfg.context_positions, st));
  // token encoder (network.py:261-303)
  MSD_TRY(launch_embed_tokens(tokens, c->tok_emb, c->tok_enc.pos, c->ex, B, c->T, d,
                              c->cfg.vocab_size, st));
  MSD_TRY(run_encoder(c, c->tok_enc, B, c->T, c->mask_bits, 0, st));
  // continuous encoder (models.py:361-363 scale_features; network.py:306-357)
  MSD_TRY(launch_scale_split(ctx_features, c->ctx_split, static_cast<long long>(B) * c->C, nd,
                             c->cfg.feature_min, c->cfg.feature_max, st));
  MSD_TRY(gemm_pos(c->ctx_split, 3 * nd, c->ctx_in_proj, 3 * nd, B * c->C, d, 3 * nd, c->ex,
                   c->ctx_enc.pos, c->C, c->ctx_seq_len, 0, st));
  MSD_TRY(run_encoder(c, c->ctx_enc, B, c->C, c->mask_bits + c->T / 32, c->T, st));
  // cross-attention K/V of every decoder layer, once per segment batch
  const size_t dk = static_cast<size_t>(d) * c->ks;  // row length of the encodings buffer
  for (int l = 0; l < c->cfg.num_decoder_layers; ++l) {
    const size_t kv_off = static_cast<size_t>(l) * c->Bmax * c->Mkv * 2 * hh;  // elements
    if (c->cfg.cross_attend_style == 0) {
      MSD_TRY(dense(c, c->enc, c->dec[l].cross_kv, B * c->Mkv, 2 * hh, d, epi_qkv(c),
                    at(c, c->kv_cache, kv_off), 2 * hh, nullptr, st));
      continue;
    }
    // sum_cross_attends: each source has its own key / value kernels; same cache layout
    for (int b = 0; b < B; ++b) {
      const size_t r0 = static_cast<size_t>(b) * c->Mkv;
      MSD_TRY(dense(c, c->enc + r0 * dk, c->dec[l].cross_kv, c->T, 2 * hh, d, epi_qkv(c),
                    at(c, c->kv_cache, kv_off + r0 * 2 * hh), 2 * hh, nullptr, st));
      MSD_TRY(dense(c, c->enc + (r0 + c->T) * dk, c->dec[l].cross_kv1, c->C, 2 * hh, d, epi_qkv(c),
                    at(c, c->kv_cache, kv_off + (r0 + c->T) * 2 * hh), 2 * hh, nullptr, st));
    }
  }
  c->cur_batch = B;
  MSD_TRY(end_on(c, caller));
  return 0;
}

int msd_get_encodings(msd_ctx* c, float* enc_out, void* stream) {
  MSD_REQUIRE(c && enc_out && c->cur_batch > 0, "msd_get_encodings: nothing encoded");
  cudaStream_t caller = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(begin_on(c, caller));
  MSD_TRY(launch_bf16_rows_to_f32(c->enc, c->d * c->ks, c->acc ? c->d : 0, enc_out,
                                  static_cast<long long>(c->cur_batch) * c->Mkv, c->d, c->work));
  MSD_TRY(end_on(c, caller));
  return 0;
}

int msd_get_step_table(msd_ctx* c, float* table_host) {
  MSD_REQUIRE(c && table_host, "msd_get_step_table: null argument");
  memcpy(table_host, c->coef_host.data(), c->coef_host.size() * sizeof(float));
  return 0;
}

int msd_step_table(const msd_config* cfg, float* table_host) {
  MSD_REQUIRE(cfg && table_host, "msd_step_table: null argument");
  MSD_TRY(validate(cfg));
  std::vector<float> tab;
  build_step_table(*cfg, tab);
  memcpy(table_host, tab.data(), tab.size() * sizeof(float));
  return 0;
}

int msd_decode_eps(msd_ctx* c, const float* z, int32_t step_i, int32_t conditioned, float* eps_out,
                   void* stream) {
  MSD_REQUIRE(c && z && eps_out, "msd_decode_eps: null argument");
  MSD_REQUIRE(c->cur_batch > 0, "msd_decode_eps: call msd_encode first");
  MSD_REQUIRE(step_i >= 0 && step_i < c->cfg.num_steps, "msd_decode_eps: step %d out of range", step_i);
  cudaStream_t caller = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(begin_on(c, caller));
  cudaStream_t st = c->work;
  const int B = c->cur_batch;
  const long long n = static_cast<long long>(B) * c->N * c->nd;
  MSD_CUDA_CHECK(cudaMemcpyAsync(c->d_step, &step_i, sizeof(int), cudaMemcpyHostToDevice, st));
  MSD_TRY(launch_init_z(z, c->z, c->z_split, n, c->nd, 0, st));
  MSD_TRY(run_decoder(c, B, conditioned ? B : 0, B, st));
  MSD_CUDA_CHECK(cudaMemcpyAsync(eps_out, c->eps, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  MSD_TRY(end_on(c, caller));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));  // step_i lives on the caller's stack
  return 0;
}

// The reverse steps of msd_sample / msd_sample_rows after init_z: per-call arguments to c->run,
// then num_steps launches of the step graph (captured on first use for this batch size).
static int run_steps(msd_ctx* c, const float* noise, unsigned long long seed, int per_row,
                     float* mel_out, cudaStream_t st) {
  const int B = c->cur_batch, steps = c->cfg.num_steps;
  // Per-call arguments + the step index go to device memory: the captured graph reads them from
  // there, so neither a new noise tensor / output buffer / seed / noise mode nor the step forces a
  // re-capture.
  RunArgs ra;
  ra.noise = noise; ra.mel_out = mel_out; ra.seed = seed; ra.step = steps - 1; ra.done = 0u;
  ra.per_row = per_row;
  // guidance split: exchange sequence numbers 1, 2, ... identical on both ranks (they make the same
  // calls), parity = buffer half
  ra.xseq = static_cast<unsigned int>(c->xcalls * static_cast<unsigned long long>(steps) + 1ull);
  ra.xsent = 0u;
  if (c->xrole != 0) ++c->xcalls;
  MSD_CUDA_CHECK(cudaMemcpyAsync(c->run, &ra, sizeof(ra), cudaMemcpyHostToDevice, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));  // `ra` is a stack variable
  // One diffusion step == one graph launch; the same executable graph serves all num_steps
  // iterations of every call with this batch size.
  if (c->graph_exec == nullptr || c->graph_batch != B) {
    drop_graph(c);
    const unsigned long long before = g_launch_count;
    cudaGraph_t graph = nullptr;
    MSD_CUDA_CHECK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    int rc = c->xrole == 0 ? run_decoder(c, B, B, c->passes * B, st, c->two_streams)
                           : run_decoder(c, B, c->xrole == 1 ? B : 0, B, st, false);
    if (rc == 0) rc = sampler_step(c, B, nullptr, 0, nullptr, st, true);
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc != 0) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    MSD_CUDA_CHECK(ce);
    c->graph_nodes = g_launch_count - before;
    g_launch_count = before;  // capture does not execute
    cudaError_t ie = cudaGraphInstantiate(&c->graph_exec, graph, 0);
    cudaGraphDestroy(graph);
    MSD_CUDA_CHECK(ie);
    c->graph_batch = B;
  }
  for (int i = 0; i < steps; ++i) {
    MSD_CUDA_CHECK(cudaGraphLaunch(c->graph_exec, st));
    g_launch_count += c->graph_nodes;
  }
  return 0;
}

int msd_sample(msd_ctx* c, const float* init_z, const float* noise, uint64_t seed, float* mel_out,
               void* stream) {
  MSD_REQUIRE(c && mel_out, "msd_sample: null argument");
  MSD_REQUIRE(c->cur_batch > 0, "msd_sample: call msd_encode first");
  cudaStream_t caller = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(begin_on(c, caller));
  cudaStream_t st = c->work;
  const int B = c->cur_batch, steps = c->cfg.num_steps;
  const long long n = static_cast<long long>(B) * c->N * c->nd;
  if (c->cfg.rng_kind == 1 && c->rng_keys_seed != seed) {
    // PRNGKey(seed) and fold_in(key, i) for every scan index (host threefry, 8 KB upload); the
    // captured step graph reads the table, so a new seed does not force a re-capture
    std::vector<uint32_t> keys(2 * (static_cast<size_t>(steps) + 1));
    keys[0] = static_cast<uint32_t>(seed >> 32);
    keys[1] = static_cast<uint32_t>(seed);
    for (int i = 0; i < steps; ++i)
      threefry2x32_host(keys[0], keys[1], 0u, static_cast<uint32_t>(i), &keys[2 * (i + 1)]);
    MSD_CUDA_CHECK(cudaMemcpyAsync(c->rng_keys, keys.data(), keys.size() * sizeof(uint32_t),
                                   cudaMemcpyHostToDevice, st));
    MSD_CUDA_CHECK(cudaStreamSynchronize(st));
    c->rng_keys_seed = seed;
  }
  MSD_TRY(launch_init_z(init_z, c->z, c->z_split, n, c->nd, seed, st, c->cfg.rng_kind, c->rng_keys));
  MSD_TRY(run_steps(c, noise, seed, 0, mel_out, st));
  MSD_TRY(end_on(c, caller));
  return 0;
}

int msd_sample_rows(msd_ctx* c, const uint64_t* seeds, float* mel_out, void* stream) {
  MSD_REQUIRE(c && seeds && mel_out, "msd_sample_rows: null argument");
  MSD_REQUIRE(c->cur_batch > 0, "msd_sample_rows: call msd_encode first");
  MSD_REQUIRE(c->xrole == 0,
              "msd_sample_rows: a peer is attached (msd_p2p_attach); the guidance split samples one "
              "song through msd_sample");
  const int B = c->cur_batch, steps = c->cfg.num_steps;
  const long long n_row = static_cast<long long>(c->N) * c->nd;
  const long long n = B * n_row;
  const size_t stride = 2 * (static_cast<size_t>(steps) + 1);
  MSD_REQUIRE(n < (1ll << 32), "msd_sample_rows: %lld elements per call, per-row streams need < 2^32", n);
  cudaStream_t caller = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(begin_on(c, caller));
  cudaStream_t st = c->work;
  // Row b's tables: Philox seed seeds[b], and (jax) PRNGKey(seeds[b]) / fold_in(key, i) exactly as
  // msd_sample builds them for one seed.  Rows whose seed is unchanged keep their keys.
  bool dirty = false;
  std::vector<uint32_t> keys(c->cfg.rng_kind == 1 ? B * stride : 0);
  for (int b = 0; b < B; ++b) {
    if (c->row_keys_valid[b] && c->row_seeds_host[b] == seeds[b]) continue;
    dirty = true;
    c->row_seeds_host[b] = seeds[b];
    c->row_keys_valid[b] = 0;  // until the upload below has completed
    if (c->cfg.rng_kind != 1) continue;
    uint32_t* k = keys.data() + b * stride;
    k[0] = static_cast<uint32_t>(seeds[b] >> 32);
    k[1] = static_cast<uint32_t>(seeds[b]);
    for (int i = 0; i < steps; ++i)
      threefry2x32_host(k[0], k[1], 0u, static_cast<uint32_t>(i), &k[2 * (i + 1)]);
    MSD_CUDA_CHECK(cudaMemcpyAsync(c->row_keys + b * stride, k, stride * sizeof(uint32_t),
                                   cudaMemcpyHostToDevice, st));
  }
  if (dirty) {
    MSD_CUDA_CHECK(cudaMemcpyAsync(c->row_seeds, c->row_seeds_host.data(),
                                   static_cast<size_t>(B) * sizeof(unsigned long long),
                                   cudaMemcpyHostToDevice, st));
    MSD_CUDA_CHECK(cudaStreamSynchronize(st));  // `keys` is a local
    for (int b = 0; b < B; ++b) c->row_keys_valid[b] = 1;
  }
  MSD_TRY(launch_init_z(nullptr, c->z, c->z_split, n, c->nd, 0, st, c->cfg.rng_kind, c->row_keys,
                        n_row, static_cast<long long>(stride), c->row_seeds));
  MSD_TRY(run_steps(c, nullptr, 0, 1, mel_out, st));
  MSD_TRY(end_on(c, caller));
  return 0;
}

int msd_p2p_export(msd_ctx* c, void* handle_out) {
  MSD_REQUIRE(c && handle_out, "msd_p2p_export: null argument");
  MSD_CUDA_CHECK(cudaSetDevice(c->device));
  cudaIpcMemHandle_t h;
  MSD_CUDA_CHECK(cudaIpcGetMemHandle(&h, c->xchg));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &h, sizeof(h));
  return 0;
}

int msd_p2p_attach(msd_ctx* c, const void* peer_handle, int32_t role) {
  MSD_REQUIRE(c && peer_handle, "msd_p2p_attach: null argument");
  MSD_REQUIRE(role == 1 || role == 2, "msd_p2p_attach: role must be 1 (conditional pass) or 2 (unconditional)");
  MSD_REQUIRE(c->passes == 2, "msd_p2p_attach: guidance is off (eval_condition_weight == 1): nothing to split");
  MSD_REQUIRE(c->xchg_peer == nullptr, "msd_p2p_attach: already attached; call msd_p2p_detach first");
  MSD_CUDA_CHECK(cudaSetDevice(c->device));
  cudaIpcMemHandle_t h;
  memcpy(&h, peer_handle, sizeof(h));
  void* peer = nullptr;
  MSD_CUDA_CHECK(cudaIpcOpenMemHandle(&peer, h, cudaIpcMemLazyEnablePeerAccess));
  MSD_CUDA_CHECK(cudaStreamSynchronize(c->work));
  // both ranks start from a clean slate: flags and sequence numbers restart at this point
  const size_t xf = 2 * static_cast<size_t>(c->Bmax) * c->N * c->nd + 64;
  MSD_CUDA_CHECK(cudaMemset(c->xchg, 0, xf * sizeof(float)));
  c->xchg_peer = static_cast<float*>(peer);
  c->xrole = role;
  c->xcalls = 0;
  drop_graph(c);
  return 0;
}

int msd_p2p_detach(msd_ctx* c) {
  MSD_REQUIRE(c != nullptr, "msd_p2p_detach: null argument");
  MSD_CUDA_CHECK(cudaSetDevice(c->device));
  MSD_CUDA_CHECK(cudaStreamSynchronize(c->work));
  if (c->xchg_peer) MSD_CUDA_CHECK(cudaIpcCloseMemHandle(c->xchg_peer));
  c->xchg_peer = nullptr;
  c->xrole = 0;
  drop_graph(c);
  return 0;
}

int msd_profile_step(msd_ctx* c, int32_t step_i, int32_t reps, double* out) {
  MSD_REQUIRE(c && out && reps >= 1, "msd_profile_step: bad argument");
  MSD_REQUIRE(c->cur_batch > 0, "msd_profile_step: call msd_encode first");
  MSD_REQUIRE(step_i >= 1 && step_i < c->cfg.num_steps, "msd_profile_step: step out of range");
  MSD_CUDA_CHECK(cudaSetDevice(c->device));
  cudaStream_t st = c->work;
  const int B = c->cur_batch;
  ProfRecorder rec;
  for (int i = 0; i < 4 * KC_COUNT; ++i) out[i] = 0.0;
  const unsigned long long before = g_launch_count;
  int rc = 0;
  MSD_CUDA_CHECK(cudaMemcpyAsync(c->d_step, &step_i, sizeof(int), cudaMemcpyHostToDevice, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int r = 0; r < reps + 1 && rc == 0; ++r) {
    // repetition 0 is an untimed warm-up; z just keeps evolving, the work per step is identical
    // (the same kernels as the captured step graph; the step index is simply not advanced)
    if (r == 1) g_prof = &rec;
    rc = run_decoder(c, B, B, c->passes * B, st);
    if (rc == 0) rc = sampler_step(c, B, nullptr, 1234, nullptr, st, false);
  }
  g_prof = nullptr;
  g_launch_count = before;
  cudaError_t e = cudaStreamSynchronize(st);
  for (auto& r : rec.recs) {
    float ms = 0.f;
    if (e == cudaSuccess && rc == 0 && cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) {
      out[r.cls * 4 + 0] += ms / reps;
      out[r.cls * 4 + 1] += 1.0 / reps;
      out[r.cls * 4 + 2] += r.flops / reps;
      out[r.cls * 4 + 3] += r.bytes / reps;
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  if (rc != 0) return rc;
  MSD_CUDA_CHECK(e);
  return 0;
}

// ---------------------------------------------------------------------------
// operator-level entry points
// ---------------------------------------------------------------------------
int msd_op_dense(const float* a, const float* w, int32_t M, int32_t N, int32_t K, float* out,
                 void* stream) {
  return msd_op_dense_variant(a, w, M, N, K, out, 0, 0, stream);
}

int msd_op_dense_variant(const float* a, const float* w, int32_t M, int32_t N, int32_t K,
                         float* out, int32_t variant, int32_t block_n, void* stream) {
  MSD_REQUIRE(a && w && out, "msd_op_dense: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TempBufs tb;
  bf16 *ab = nullptr, *wb = nullptr;
  MSD_TRY(tb.get(&ab, static_cast<size_t>(M) * K));
  MSD_TRY(tb.get(&wb, static_cast<size_t>(N) * K));
  MSD_TRY(launch_f32_to_bf16(a, ab, static_cast<long long>(M) * K, st));
  MSD_TRY(launch_pack_weight(w, K, N, wb, K, 0, 0, 0, st));
  GemmArgs ga;
  memset(&ga, 0, sizeof(ga));
  ga.A = ab; ga.B = wb; ga.M = M; ga.N = N; ga.K = K; ga.lda = K; ga.ldb = K;
  ga.epilogue = EPI_F32; ga.out = out; ga.ldo = N; ga.variant = variant; ga.block_n = block_n;
  MSD_TRY(launch_gemm(ga, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_bench_gemm(int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t variant,
                   int32_t block_n, int32_t iters, float* ms_out) {
  MSD_REQUIRE(ms_out && iters > 0, "msd_bench_gemm: bad argument");
  TempBufs tb;
  bf16 *a = nullptr, *b = nullptr;
  float *o = nullptr, *r = nullptr;
  MSD_TRY(tb.get(&a, static_cast<size_t>(M) * K));
  MSD_TRY(tb.get(&b, static_cast<size_t>(N) * K));
  MSD_TRY(tb.get(&o, static_cast<size_t>(M) * N));
  MSD_TRY(tb.get(&r, static_cast<size_t>(M) * N));
  MSD_CUDA_CHECK(cudaMemset(a, 0, static_cast<size_t>(M) * K * 2));
  MSD_CUDA_CHECK(cudaMemset(b, 0, static_cast<size_t>(N) * K * 2));
  MSD_CUDA_CHECK(cudaMemset(r, 0, static_cast<size_t>(M) * N * 4));
  GemmArgs ga;
  memset(&ga, 0, sizeof(ga));
  ga.A = a; ga.B = b; ga.M = M; ga.N = N; ga.K = K; ga.lda = K; ga.ldb = K;
  ga.epilogue = epilogue; ga.out = o; ga.ldo = (epilogue == EPI_GATED_GELU) ? N / 2 : N;
  ga.resid = (variant == 1) ? r : o;  // default variant: in place, like the engine
  ga.variant = variant; ga.block_n = block_n;
  cudaStream_t st = nullptr;
  MSD_CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  int rc = 0;
  for (int i = 0; i < 3 && rc == 0; ++i) rc = launch_gemm(ga, st);
  cudaEventRecord(e0, st);
  for (int i = 0; i < iters && rc == 0; ++i) rc = launch_gemm(ga, st);
  cudaEventRecord(e1, st);
  cudaError_t e = cudaStreamSynchronize(st);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  *ms_out = ms / iters;
  if (getenv("MSD_GEMM_TRACE") && variant != 1 && rc == 0 && e == cudaSuccess) {
    // one more launch with per-CTA stamps (after a warm one right before it, like in the loop)
    long long* tr = nullptr;
    if (tb.get(&tr, 8 * 512) == 0) {
      cudaMemsetAsync(tr, 0, 8 * 512 * sizeof(long long), st);
      launch_gemm(ga, st);
      ga.trace = tr;
      launch_gemm(ga, st);
      ga.trace = nullptr;
      std::vector<long long> h(8 * 512);
      cudaStreamSynchronize(st);
      cudaMemcpy(h.data(), tr, h.size() * sizeof(long long), cudaMemcpyDeviceToHost);
      long long t0 = 0, t1 = 0;
      int n = 0;
      double sum[5] = {0, 0, 0, 0, 0};
      for (int b = 0; b < 512; ++b) {
        const long long* r = &h[b * 8];
        if (r[1] == 0) continue;
        if (n == 0 || r[1] < t0) t0 = r[1];
        if (n == 0 || r[2] > t1) t1 = r[2];
        // r[3] = total cycles; r[4..7] absolute clock64 stamps; entry clock = exit - total
        sum[0] += static_cast<double>(r[3]);
        ++n;
      }
      fprintf(stderr, "[gemm trace] M=%d N=%d K=%d epi=%d: %d CTAs, first entry -> last exit %.2f us, mean "
              "cycles in CTA %.0f\n", M, N, K, epilogue, n, (t1 - t0) * 1e-3, n ? sum[0] / n : 0.0);
      for (int b = 0; b < 4 && b < 512; ++b) {
        const long long* r = &h[b * 8];
        if (r[1] == 0) continue;
        fprintf(stderr, "[gemm trace]   CTA %d sm %lld: entry +%.2f us, exit +%.2f us; cycles: total %lld, "
                "setup->wait %lld, wait->acc %lld, acc->stored %lld\n", b, r[0], (r[1] - t0) * 1e-3,
                (r[2] - t0) * 1e-3, r[3], r[5] - r[4], r[6] - r[5], r[7] - r[6]);
      }
    }
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaStreamDestroy(st);
  if (rc != 0) return rc;
  MSD_CUDA_CHECK(e);
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
  cudaStream_t st = nullptr;
  MSD_CUDA_CHECK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  // N(0,1) * 0.3-ish values through the jax generator (any bounded values would do)
  MSD_TRY(launch_jax_normal(1u, 2u, static_cast<long long>(nk), tmp, st));
  MSD_TRY(launch_f32_to_bf16(tmp, kb, static_cast<long long>(nk), st));
  MSD_TRY(launch_f32_to_bf16(tmp, vb, static_cast<long long>(nk), st));
  MSD_TRY(launch_f32_to_bf16(tmp, qb, static_cast<long long>(nq), st));
  AttnArgs aa;
  memset(&aa, 0, sizeof(aa));
  aa.Q = qb; aa.ldq = w; aa.K = kb; aa.ldk = w; aa.V = vb; aa.ldv = w; aa.O = ob; aa.ldo = w;
  aa.nbatch = nb; aa.heads = heads; aa.Lq = Lq; aa.Lk = Lk;
  aa.part_o = po; aa.part_ml = pml; aa.max_splits = 12; aa.kv_static = 1;
  {
    const char* f = getenv("MSD_ATTN_SPLITS");
    aa.splits = f ? atoi(f) : 0;
    const char* t = getenv("MSD_ATTN_TAIL");
    aa.tail = t ? atoi(t) : 0;
  }
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  int rc = 0;
  for (int i = 0; i < 3 && rc == 0; ++i) rc = launch_attention(aa, st);
  cudaEventRecord(e0, st);
  for (int i = 0; i < iters && rc == 0; ++i) rc = launch_attention(aa, st);
  cudaEventRecord(e1, st);
  cudaError_t e = cudaStreamSynchronize(st);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  *ms_out = ms / iters;
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaStreamDestroy(st);
  if (rc != 0) return rc;
  MSD_CUDA_CHECK(e);
  return 0;
}

int msd_op_attention(const float* q, const float* k, const float* v, const int32_t* key_mask,
                     int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, float* out, void* stream) {
  MSD_REQUIRE(q && k && v && out, "msd_op_attention: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int w = heads * 64;
  TempBufs tb;
  bf16 *qb, *kb, *vb, *ob;
  uint32_t* bits = nullptr;
  MSD_TRY(tb.get(&qb, static_cast<size_t>(nb) * Lq * w));
  MSD_TRY(tb.get(&kb, static_cast<size_t>(nb) * Lk * w));
  MSD_TRY(tb.get(&vb, static_cast<size_t>(nb) * Lk * w));
  MSD_TRY(tb.get(&ob, static_cast<size_t>(nb) * Lq * w));
  MSD_TRY(launch_f32_to_bf16(q, qb, static_cast<long long>(nb) * Lq * w, st));
  MSD_TRY(launch_f32_to_bf16(k, kb, static_cast<long long>(nb) * Lk * w, st));
  MSD_TRY(launch_f32_to_bf16(v, vb, static_cast<long long>(nb) * Lk * w, st));
  if (key_mask) {
    MSD_TRY(tb.get(&bits, static_cast<size_t>(nb) * (Lk / 32)));
    MSD_TRY(launch_mask_bits(key_mask, nb, Lk, bits, st));
  }
  {
    AttnArgs aa;
    memset(&aa, 0, sizeof(aa));
    aa.Q = qb; aa.ldq = w; aa.K = kb; aa.ldk = w; aa.V = vb; aa.ldv = w; aa.O = ob; aa.ldo = w;
    aa.nbatch = nb; aa.heads = heads; aa.Lq = Lq; aa.Lk = Lk; aa.mask_bits = bits;
    aa.mask_stride_words = Lk / 32;
    float *po = nullptr, *pml = nullptr;
    MSD_TRY(tb.get(&po, attention_workspace_floats(nb, heads, Lq, 12)));
    MSD_TRY(tb.get(&pml, static_cast<size_t>(nb) * Lq * heads * 12 * 2));
    aa.part_o = po; aa.part_ml = pml; aa.max_splits = 12;
    {
      const char* f = getenv("MSD_ATTN_SPLITS");  // test hook: force a split count
      aa.splits = f ? atoi(f) : 0;
      const char* t = getenv("MSD_ATTN_TAIL");    // test hook: force a tail length
      aa.tail = t ? atoi(t) : 0;
    }
    MSD_TRY(launch_attention(aa, st));
  }
  MSD_TRY(launch_bf16_to_f32(ob, out, static_cast<long long>(nb) * Lq * w, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_jax_normal(uint64_t seed, int32_t step, int64_t n, float* out, void* stream) {
  MSD_REQUIRE(out != nullptr, "msd_op_jax_normal: null argument");
  uint32_t key[2] = {static_cast<uint32_t>(seed >> 32), static_cast<uint32_t>(seed)};
  if (step >= 0) {
    uint32_t folded[2];
    threefry2x32_host(key[0], key[1], 0u, static_cast<uint32_t>(step), folded);
    key[0] = folded[0];
    key[1] = folded[1];
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(launch_jax_normal(key[0], key[1], n, out, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_jax_bits(uint64_t seed, int32_t step, int64_t n, uint32_t* out, void* stream) {
  MSD_REQUIRE(out != nullptr, "msd_op_jax_bits: null argument");
  uint32_t key[2] = {static_cast<uint32_t>(seed >> 32), static_cast<uint32_t>(seed)};
  if (step >= 0) {
    uint32_t folded[2];
    threefry2x32_host(key[0], key[1], 0u, static_cast<uint32_t>(step), folded);
    key[0] = folded[0];
    key[1] = folded[1];
  }
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

int msd_op_dense_epilogue(const float* a, const float* w, const float* w1, int32_t M, int32_t N,
                          int32_t K, int32_t epilogue, int32_t block_n, const float* resid,
                          const float* pos, int32_t pos_rows, const int32_t* pos_shift,
                          int32_t dup_rows, float* out, void* stream) {
  MSD_REQUIRE(a && w && out, "msd_op_dense_epilogue: null argument");
  const bool gated = epilogue == EPI_GATED_GELU || epilogue == EPI_GATED_GELU_SPLIT3;
  MSD_REQUIRE(epilogue == EPI_BF16 || epilogue == EPI_RESID_F32 || epilogue == EPI_POS_F32 || gated,
              "msd_op_dense_epilogue: unknown epilogue %d", epilogue);
  MSD_REQUIRE(!gated || w1 != nullptr, "msd_op_dense_epilogue: the gated epilogues need w1");
  MSD_REQUIRE(epilogue != EPI_RESID_F32 || resid != nullptr, "msd_op_dense_epilogue: resid is null");
  MSD_REQUIRE(epilogue != EPI_POS_F32 || (pos != nullptr && pos_rows > 0),
              "msd_op_dense_epilogue: pos / pos_rows missing");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool split = epilogue == EPI_GATED_GELU_SPLIT3;
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
  GemmArgs ga;
  memset(&ga, 0, sizeof(ga));
  ga.A = ab; ga.B = wb; ga.M = M; ga.N = Ng; ga.K = K * ks; ga.lda = K * ks; ga.ldb = K * ks;
  ga.epilogue = epilogue; ga.block_n = block_n;
  ga.resid = resid; ga.pos = pos; ga.pos_rows = pos_rows; ga.pos_shift = pos_shift;
  ga.dup_rows = dup_rows;
  const bool bf16_out = epilogue == EPI_BF16 || gated;
  if (bf16_out) {
    MSD_TRY(tb.get(&ob, static_cast<size_t>(M) * N * ks));
    ga.out = ob; ga.ldo = N * ks;
  } else {
    ga.out = out; ga.ldo = N;
  }
  MSD_TRY(launch_gemm(ga, st));
  if (bf16_out)
    MSD_TRY(launch_bf16_rows_to_f32(ob, N * ks, split ? N : 0, out, M, N, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
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
  uint32_t* bits = nullptr;
  MSD_TRY(tb.get(&ob, static_cast<size_t>(nb) * Lq * w * 3));
  if (key_mask) {
    MSD_REQUIRE(Lk % 128 == 0, "msd_op_attention_f32: masked Lk must be a multiple of 128");
    MSD_TRY(tb.get(&bits, static_cast<size_t>(nb) * (Lk / 32)));
    MSD_TRY(launch_mask_bits(key_mask, nb, Lk, bits, st));
  }
  AttnF32Args aa;
  memset(&aa, 0, sizeof(aa));
  aa.Q = q; aa.ldq = w; aa.K = k; aa.ldk = w; aa.V = v; aa.ldv = w; aa.O = ob; aa.o_third = w;
  aa.nbatch = nb; aa.heads = heads; aa.Lq = Lq; aa.Lk = Lk; aa.mask_bits = bits;
  aa.mask_stride_words = Lk / 32;
  float *po = nullptr, *pml = nullptr;
  MSD_TRY(tb.get(&po, static_cast<size_t>(nb) * Lq * heads * 8 * 64));
  MSD_TRY(tb.get(&pml, static_cast<size_t>(nb) * Lq * heads * 8 * 2));
  aa.part_o = po; aa.part_ml = pml; aa.max_splits = 8;
  {
    const char* f = getenv("MSD_ATTN_SPLITS");  // test hook: force a split count
    aa.splits = f ? atoi(f) : 0;
  }
  MSD_TRY(launch_attention_f32(aa, st));
  MSD_TRY(launch_bf16_rows_to_f32(ob, 3 * w, w, out, static_cast<long long>(nb) * Lq, w, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_attention_view(int32_t precision, void* q, int64_t q_off, int32_t ldq, const void* k,
                          int64_t k_off, int32_t ldk, const void* v, int64_t v_off, int32_t ldv,
                          int32_t nb, int32_t heads, int32_t Lq, int32_t Lk, int32_t kv_batch_rows,
                          int32_t kv_row0, const int32_t* key_mask, int32_t mask_len,
                          int32_t mask_word0, int32_t kv_static, void* out, int64_t o_col,
                          int32_t o_ld, float* part_o, float* part_ml, int32_t splits, int32_t tail,
                          void* stream) {
  MSD_REQUIRE(q && k && v && out && part_o && part_ml, "msd_op_attention_view: null argument");
  MSD_REQUIRE(precision == 0 || precision == 1, "msd_op_attention_view: precision must be 0 or 1");
  MSD_REQUIRE(nb > 0 && heads > 0 && Lq > 0 && Lk > 0 && q_off >= 0 && k_off >= 0 && v_off >= 0 &&
                  o_col >= 0 && kv_row0 >= 0 && kv_batch_rows >= 0,
              "msd_op_attention_view: bad sizes or offsets");
  MSD_REQUIRE(splits >= 0 && splits <= 12 && tail >= 0 && (precision == 0 || tail == 0),
              "msd_op_attention_view: splits must be in [0, 12], tail >= 0 (bf16 mode only)");
  MSD_REQUIRE(!key_mask || (mask_len % 128 == 0 && mask_word0 >= 0 && mask_word0 % 4 == 0 &&
                            mask_word0 + Lk / 32 <= mask_len / 32),
              "msd_op_attention_view: mask words [%d, %d) outside rows of %d keys", mask_word0,
              mask_word0 + Lk / 32, mask_len);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t es = precision ? 4 : 2;
  const int width = heads * 64;
  const long long rows_q = static_cast<long long>(nb) * Lq;
  char* qv = static_cast<char*>(q) + q_off * es;
  TempBufs tb;
  uint32_t* bits = nullptr;
  if (key_mask) {
    MSD_TRY(tb.get(&bits, static_cast<size_t>(nb) * (mask_len / 32)));
    MSD_TRY(launch_mask_bits(key_mask, nb, mask_len, bits, st));
  }
  // K, V and the mask must be complete before the attention starts (kv_static reads them ahead of
  // its dependency wait, as after the plain first launch of a diffusion step).  Q is then written
  // back from a staging copy by a kernel of its own, so that the attention is a PDL launch behind a
  // live predecessor, as in the step graph.
  char* stage = nullptr;
  MSD_TRY(tb.get(&stage, static_cast<size_t>(rows_q) * width * es));
  MSD_CUDA_CHECK(cudaMemcpy2DAsync(stage, width * es, qv, ldq * es, width * es, rows_q,
                                   cudaMemcpyDeviceToDevice, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  MSD_TRY(launch_copy_rows(stage, static_cast<long long>(width * es), qv, static_cast<long long>(ldq) * es,
                           rows_q, static_cast<int>(width * es), st));
  const uint32_t* mbits = bits ? bits + mask_word0 : nullptr;
  if (precision == 0) {
    AttnArgs a;
    memset(&a, 0, sizeof(a));
    a.Q = reinterpret_cast<const bf16*>(qv); a.ldq = ldq;
    a.K = static_cast<const bf16*>(k) + k_off; a.ldk = ldk;
    a.V = static_cast<const bf16*>(v) + v_off; a.ldv = ldv;
    a.O = static_cast<bf16*>(out) + o_col; a.ldo = o_ld;
    a.nbatch = nb; a.heads = heads; a.Lq = Lq; a.Lk = Lk;
    a.mask_bits = mbits; a.mask_stride_words = mask_len / 32;
    a.part_o = part_o; a.part_ml = part_ml; a.splits = splits; a.max_splits = 12; a.tail = tail;
    a.kv_static = kv_static; a.kv_batch_rows = kv_batch_rows; a.kv_row0 = kv_row0;
    MSD_TRY(launch_attention(a, st));
  } else {
    AttnF32Args a;
    memset(&a, 0, sizeof(a));
    a.Q = reinterpret_cast<const float*>(qv); a.ldq = ldq;
    a.K = static_cast<const float*>(k) + k_off; a.ldk = ldk;
    a.V = static_cast<const float*>(v) + v_off; a.ldv = ldv;
    a.O = static_cast<bf16*>(out) + o_col; a.o_third = o_ld;
    a.nbatch = nb; a.heads = heads; a.Lq = Lq; a.Lk = Lk;
    a.mask_bits = mbits; a.mask_stride_words = mask_len / 32;
    a.kv_batch_rows = kv_batch_rows; a.kv_row0 = kv_row0;
    a.part_o = part_o; a.part_ml = part_ml; a.splits = splits; a.max_splits = 12;
    MSD_TRY(launch_attention_f32(a, st));
  }
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

int msd_op_gemm_view(const void* a, int64_t a_off, int32_t lda, const void* b, int64_t b_off, int32_t ldb,
                     int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t block_n, int32_t variant,
                     void* out, int64_t out_off, int32_t ldo, const float* resid, int64_t resid_off,
                     const float* pos, int32_t pos_rows, const int32_t* pos_shift, int32_t dup_rows,
                     const int32_t* step, const float* prep_g_lo, int64_t prep_g_lo_step_stride,
                     const float* prep_g_hi, int64_t prep_g_hi_step_stride, int32_t prep_split_row,
                     void* prep_a, int32_t prep_lda, float* prep_ss, int32_t prep_ss_stride,
                     const float* rs_ss_lo, int32_t rs_parts_lo, const float* rs_ss_hi, int32_t rs_parts_hi,
                     int32_t rs_split_row, int32_t rs_ss_stride, float rs_inv_d, const float* rs_col_bias,
                     int64_t rs_bias_step_stride, int32_t* block_n_out, void* stream) {
  MSD_REQUIRE(a && b && out, "msd_op_gemm_view: null argument");
  MSD_REQUIRE(epilogue >= EPI_BF16 && epilogue <= EPI_RESID_PREP, "msd_op_gemm_view: unknown epilogue %d",
              epilogue);
  MSD_REQUIRE(a_off >= 0 && b_off >= 0 && out_off >= 0 && resid_off >= 0,
              "msd_op_gemm_view: negative offset");
  const bool f32_out = epilogue == EPI_F32 || epilogue == EPI_RESID_F32 || epilogue == EPI_POS_F32 ||
                       epilogue == EPI_RESID_PREP;
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.A = static_cast<const bf16*>(a) + a_off; g.lda = lda;
  g.B = static_cast<const bf16*>(b) + b_off; g.ldb = ldb;
  g.M = M; g.N = N; g.K = K; g.epilogue = epilogue; g.block_n = block_n; g.variant = variant;
  g.out = f32_out ? static_cast<void*>(static_cast<float*>(out) + out_off)
                  : static_cast<void*>(static_cast<bf16*>(out) + out_off);
  g.ldo = ldo;
  g.resid = resid ? resid + resid_off : nullptr;
  g.pos = pos; g.pos_rows = pos_rows; g.pos_shift = pos_shift; g.dup_rows = dup_rows;
  g.step = step;
  g.prep.g_lo = prep_g_lo; g.prep.g_lo_step_stride = prep_g_lo_step_stride;
  g.prep.g_hi = prep_g_hi; g.prep.g_hi_step_stride = prep_g_hi_step_stride;
  g.prep.split_row = prep_split_row;
  g.prep.a = static_cast<bf16*>(prep_a); g.prep.lda = prep_lda;
  g.prep.ss = prep_ss; g.prep.ss_stride = prep_ss_stride;
  g.rs.ss_lo = rs_ss_lo; g.rs.parts_lo = rs_parts_lo; g.rs.ss_hi = rs_ss_hi; g.rs.parts_hi = rs_parts_hi;
  g.rs.split_row = rs_split_row; g.rs.ss_stride = rs_ss_stride; g.rs.inv_d = rs_inv_d;
  g.rs.col_bias = rs_col_bias; g.rs.bias_step_stride = rs_bias_step_stride;
  MSD_REQUIRE(epilogue != EPI_RESID_PREP || g.prep.a != nullptr,
              "msd_op_gemm_view: EPI_RESID_PREP needs prep_a");
  MSD_REQUIRE(epilogue != EPI_POS_F32 || (pos != nullptr && pos_rows > 0),
              "msd_op_gemm_view: EPI_POS_F32 needs pos / pos_rows");
  const int bn = gemm_resolve_block_n(g);
  MSD_REQUIRE(bn > 0, "msd_op_gemm_view: N=%d has no tile width (block_n %d, variant %d)", N, block_n, variant);
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

int msd_op_sampler_step(const float* eps, float* z, void* z_split, float* mel_out, const float* noise,
                        const float* coef, int32_t num_steps, const int32_t* step, int64_t n, int32_t n_dims,
                        int32_t passes, float cond_weight, int32_t clip_x0, int32_t ddim, float feat_min,
                        float feat_max, uint64_t seed, int32_t rng_kind, const uint32_t* rng_keys,
                        int64_t n_row, const uint32_t* row_keys, int64_t row_key_stride,
                        const uint64_t* row_seeds, int32_t run_step, int32_t per_row, int32_t launches,
                        int32_t* run_out, void* stream) {
  MSD_REQUIRE(eps && z && z_split && coef, "msd_op_sampler_step: null argument");
  MSD_REQUIRE(n > 0 && n_dims > 0 && n % 4 == 0 && n_dims % 4 == 0 && n % n_dims == 0 && num_steps > 0,
              "msd_op_sampler_step: n=%lld must be a positive multiple of n_dims=%d, both multiples of 4",
              static_cast<long long>(n), n_dims);
  MSD_REQUIRE(passes == 1 || passes == 2, "msd_op_sampler_step: passes must be 1 or 2 (got %d)", passes);
  MSD_REQUIRE(rng_kind == 0 || rng_kind == 1, "msd_op_sampler_step: rng_kind must be 0 or 1");
  MSD_REQUIRE(rng_kind == 0 || per_row || (rng_keys != nullptr && n % 8 == 0 && n < (1ll << 32)),
              "msd_op_sampler_step: the jax stream needs its key table and a draw of k*8 < 2^32 elements");
  MSD_REQUIRE(!per_row || (n_row > 0 && n_row % 8 == 0 && n % n_row == 0 && n < (1ll << 32) &&
                           (rng_kind == 0 ? row_seeds != nullptr : row_keys != nullptr)),
              "msd_op_sampler_step: per-row streams need rows of k*8 elements, n < 2^32 and the row table");
  MSD_REQUIRE(step == nullptr || (!per_row && launches == 1),
              "msd_op_sampler_step: per-row streams and several launches need the RunArgs path (step NULL)");
  MSD_REQUIRE(step != nullptr || run_out != nullptr, "msd_op_sampler_step: the RunArgs path needs run_out");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int first = run_step;
  if (step != nullptr) MSD_CUDA_CHECK(cudaMemcpy(&first, step, sizeof(int), cudaMemcpyDeviceToHost));
  MSD_REQUIRE(launches >= 1 && first < num_steps && first - launches + 1 >= 0,
              "msd_op_sampler_step: %d launch(es) from step %d leave the table of %d steps", launches, first,
              num_steps);
  SamplerArgs a;
  memset(&a, 0, sizeof(a));
  a.eps = eps; a.z = z; a.z_split = static_cast<bf16*>(z_split); a.coef = coef;
  a.n = n; a.n_dims = n_dims; a.passes = passes; a.cond_weight = cond_weight;
  a.clip_x0 = clip_x0; a.ddim = ddim; a.feat_min = feat_min; a.feat_max = feat_max;
  a.rng_kind = rng_kind; a.rng_keys = rng_keys;
  a.n_row = n_row; a.row_keys = row_keys; a.row_key_stride = row_key_stride;
  a.row_seeds = reinterpret_cast<const unsigned long long*>(row_seeds);
  TempBufs tb;
  if (step != nullptr) {
    a.step = step; a.noise = noise; a.mel_out = mel_out; a.seed = seed;
    g_pdl_skip_next = true;   // the inputs were just written by the caller's own kernels
    MSD_TRY(launch_sampler_step(a, st));
    MSD_CUDA_CHECK(cudaStreamSynchronize(st));
    return 0;
  }
  RunArgs ra;
  memset(&ra, 0, sizeof(ra));
  ra.noise = noise; ra.mel_out = mel_out; ra.seed = seed; ra.step = run_step; ra.per_row = per_row;
  MSD_TRY(tb.get(&a.run, 1));
  MSD_CUDA_CHECK(cudaMemcpyAsync(a.run, &ra, sizeof(ra), cudaMemcpyHostToDevice, st));
  // the first launch follows the upload; the next ones are PDL launches behind the previous step's
  // sampler kernel, which is what the step graph's first kernel sees
  g_pdl_skip_next = true;
  for (int i = 0; i < launches; ++i) MSD_TRY(launch_sampler_step(a, st));
  MSD_CUDA_CHECK(cudaMemcpyAsync(&ra, a.run, sizeof(ra), cudaMemcpyDeviceToHost, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  run_out[0] = ra.step;
  run_out[1] = static_cast<int32_t>(ra.done);
  return 0;
}

int msd_op_init_z(const float* init_z, float* z, void* z_split, int64_t n, int32_t n_dims, uint64_t seed,
                  int32_t rng_kind, const uint32_t* rng_keys, int64_t n_row, int64_t row_key_stride,
                  const uint64_t* row_seeds, void* stream) {
  MSD_REQUIRE(z && z_split, "msd_op_init_z: null argument");
  MSD_REQUIRE(n > 0 && n_dims > 0 && n % 4 == 0 && n_dims % 4 == 0 && n % n_dims == 0,
              "msd_op_init_z: n=%lld must be a positive multiple of n_dims=%d, both multiples of 4",
              static_cast<long long>(n), n_dims);
  MSD_REQUIRE(rng_kind == 0 || rng_kind == 1, "msd_op_init_z: rng_kind must be 0 or 1");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  MSD_TRY(launch_init_z(init_z, z, static_cast<bf16*>(z_split), n, n_dims, seed, st, rng_kind, rng_keys, n_row,
                        row_key_stride, reinterpret_cast<const unsigned long long*>(row_seeds)));
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

int msd_get_conditioning_tables(msd_ctx* c, float* film, float* gain, float* bias_qkv, float* bias_wi) {
  MSD_REQUIRE(c != nullptr, "msd_get_conditioning_tables: null context");
  MSD_REQUIRE(c->weights_loaded, "msd_get_conditioning_tables: call msd_load_weights first");
  MSD_REQUIRE(c->fused_norm || (!gain && !bias_qkv && !bias_wi),
              "msd_get_conditioning_tables: deferred normalisation is off, there are no gain / bias tables");
  const size_t steps = static_cast<size_t>(c->cfg.num_steps), Ld = static_cast<size_t>(c->cfg.num_decoder_layers);
  const struct { float* dst; const float* src; size_t n; } tabs[4] = {
      {film, c->film, steps * 2 * Ld * 2 * c->d},
      {gain, c->gtab, steps * 2 * Ld * c->d},
      {bias_qkv, c->btab_qkv, steps * Ld * 3 * c->hh},
      {bias_wi, c->btab_wi, steps * Ld * 2 * c->F}};
  for (const auto& t : tabs)
    if (t.dst) MSD_CUDA_CHECK(cudaMemcpy(t.dst, t.src, t.n * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

int msd_op_rmsnorm_film(const float* x, const float* gamma, const float* film, int32_t rows,
                        int32_t d, float* out, void* stream) {
  MSD_REQUIRE(x && gamma && out, "msd_op_rmsnorm_film: null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TempBufs tb;
  bf16* ob = nullptr;
  int* zero = nullptr;
  MSD_TRY(tb.get(&ob, static_cast<size_t>(rows) * d));
  MSD_TRY(tb.get(&zero, 1));
  MSD_CUDA_CHECK(cudaMemsetAsync(zero, 0, sizeof(int), st));
  MSD_TRY(launch_rmsnorm(x, gamma, rows, d, ob, d, film, zero, 0, 0, 0, st));
  MSD_TRY(launch_bf16_to_f32(ob, out, static_cast<long long>(rows) * d, st));
  MSD_CUDA_CHECK(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
