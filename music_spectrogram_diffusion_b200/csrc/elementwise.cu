// Row-wise / element-wise kernels of the DDPM hot path (HBM-bound; vectorised, coalesced):
//   rmsnorm(+FiLM)   msd/layers.py:632-649 (T5 RMS norm), 652-666 (FiLM x*(1+s)+b)
//   sampler step     msd/models/diffusion/diffusion_utils.py:398-453, 382-395, 120-163, 215-222
//   token embedding  msd/layers.py:556-559 + network.py:278-287
//   feature scaling  msd/audio_codecs.py:166-183
//   masks            msd/models/diffusion/network.py:28-51, 546; msd/layers.py:341-348
#include "common.cuh"
#include "kernels.h"

#define MSD_TRY_RC(expr)      \
  do {                       \
    int _rc = (expr);        \
    if (_rc != 0) return _rc; \
  } while (0)

namespace msd {

std::atomic<unsigned long long> g_launch_count{0};

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void split_bf16(float x, bf16& hi, bf16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// ---------------------------------------------------------------------------
// RMSNorm (+FiLM) : one warp per row, row kept in registers, bf16 output
// ---------------------------------------------------------------------------
struct NormDev {
  const float* x;
  const float* gamma;
  bf16* out;
  const float* film;
  const int* step;
  long long film_step_stride, film_offset;
  int rows, d, ldo, split3;
  int src_len, dst_len, dst_off;  // row remap when src_len > 0
  // deferred normalisation (launch_prep_rows): out = bf16(x * gamma) with gamma taken at
  // gamma + (*step) * gamma_step_stride, NOT normalised; ss_out[row] = sum of squares
  float* ss_out;
  long long gamma_step_stride;
};

constexpr int NORM_MAX_ITERS = 8;  // d <= 1024

// ITERS = d / 128 (float4 per lane), a template parameter so that the per-row constants (gamma
// and the FiLM scale | bias rows) can be requested together with the row itself: their L2 round
// trip then overlaps the row's instead of following the warp reduction (the kernel is a pure
// latency chain: ~5 us for 19 MB of traffic).
template <int ITERS>
__global__ void __launch_bounds__(256) rmsnorm_film_kernel(const NormDev p) {
  griddep_launch_dependents();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= p.rows) return;
  constexpr int D = ITERS * 128;
  // per-segment constants: safe to read ahead of the dependency wait (written at load time)
  float4 g[ITERS];
  // (the step index only changes in the last kernel of a step: stable from here on)
  const float* gamma = p.ss_out ? p.gamma + static_cast<long long>(*p.step) * p.gamma_step_stride : p.gamma;
#pragma unroll
  for (int i = 0; i < ITERS; ++i)
    g[i] = __ldg(reinterpret_cast<const float4*>(gamma + (i * 32 + lane) * 4));
  griddep_wait();
  const float4* xr = reinterpret_cast<const float4*>(p.x + static_cast<size_t>(warp) * D);
  float4 v[ITERS];
#pragma unroll
  for (int i = 0; i < ITERS; ++i) v[i] = xr[i * 32 + lane];
  float4 fsv[ITERS], fbv[ITERS];
  const bool has_film = p.film != nullptr;
  if (has_film) {
    const long long base = static_cast<long long>(*p.step) * p.film_step_stride + p.film_offset;
    const float* fs = p.film + base;
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
      const int c = (i * 32 + lane) * 4;
      fsv[i] = __ldg(reinterpret_cast<const float4*>(fs + c));
      fbv[i] = __ldg(reinterpret_cast<const float4*>(fs + D + c));
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < ITERS; ++i)
    ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
  ss = warp_sum(ss);
  const float inv = p.ss_out ? 1.0f : rsqrtf(ss / static_cast<float>(D) + 1e-6f);
  if (p.ss_out && lane == 0) p.ss_out[warp] = ss;
  int orow = warp;
  if (p.src_len > 0) {
    const int b = warp / p.src_len;
    orow = b * p.dst_len + p.dst_off + (warp - b * p.src_len);
  }
  bf16* o = p.out + static_cast<size_t>(orow) * p.ldo;
#pragma unroll
  for (int i = 0; i < ITERS; ++i) {
    const int c = (i * 32 + lane) * 4;
    float y0 = v[i].x * inv * g[i].x, y1 = v[i].y * inv * g[i].y;
    float y2 = v[i].z * inv * g[i].z, y3 = v[i].w * inv * g[i].w;
    if (has_film) {
      y0 = y0 * (fsv[i].x + 1.0f) + fbv[i].x; y1 = y1 * (fsv[i].y + 1.0f) + fbv[i].y;
      y2 = y2 * (fsv[i].z + 1.0f) + fbv[i].z; y3 = y3 * (fsv[i].w + 1.0f) + fbv[i].w;
    }
    if (!p.split3) {
      uint2 u;
      u.x = pack_bf16(y0, y1);
      u.y = pack_bf16(y2, y3);
      *reinterpret_cast<uint2*>(o + c) = u;
    } else {
      bf16 h0, h1, h2, h3, l0, l1, l2, l3;
      split_bf16(y0, h0, l0); split_bf16(y1, h1, l1);
      split_bf16(y2, h2, l2); split_bf16(y3, h3, l3);
      __nv_bfloat162 a = __halves2bfloat162(h0, h1), b2 = __halves2bfloat162(h2, h3);
      __nv_bfloat162 c0 = __halves2bfloat162(l0, l1), c1 = __halves2bfloat162(l2, l3);
      uint2 uh, ul;
      uh.x = *reinterpret_cast<uint32_t*>(&a); uh.y = *reinterpret_cast<uint32_t*>(&b2);
      ul.x = *reinterpret_cast<uint32_t*>(&c0); ul.y = *reinterpret_cast<uint32_t*>(&c1);
      *reinterpret_cast<uint2*>(o + c) = uh;            // hi
      *reinterpret_cast<uint2*>(o + D + c) = ul;        // lo
      *reinterpret_cast<uint2*>(o + 2 * D + c) = uh;    // hi
    }
  }
}

template <int ITERS>
int launch_norm_iters(const NormDev& p, cudaStream_t stream) {
  static const int configured = [] {
    return cudaFuncSetAttribute(rmsnorm_film_kernel<ITERS>, cudaFuncAttributePreferredSharedMemoryCarveout,
                                100) == cudaSuccess ? 0 : -2;
  }();
  MSD_REQUIRE(configured == 0, "rmsnorm: cudaFuncSetAttribute failed");
  MSD_CUDA_CHECK(launch_kernel(rmsnorm_film_kernel<ITERS>, dim3((p.rows + 7) / 8), dim3(256), 0, stream, p));
  return 0;
}
int launch_norm(const NormDev& p, cudaStream_t stream) {
  switch (p.d >> 7) {
    case 1: return launch_norm_iters<1>(p, stream);
    case 2: return launch_norm_iters<2>(p, stream);
    case 3: return launch_norm_iters<3>(p, stream);
    case 4: return launch_norm_iters<4>(p, stream);
    case 5: return launch_norm_iters<5>(p, stream);
    case 6: return launch_norm_iters<6>(p, stream);
    case 7: return launch_norm_iters<7>(p, stream);
    default: return launch_norm_iters<8>(p, stream);
  }
}

// ---------------------------------------------------------------------------
// Philox4x32-10 + Box-Muller (perf-mode noise; parity runs inject noise instead)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                              uint32_t k0, uint32_t k1, uint32_t (&out)[4]) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ float4 philox_normal4(unsigned long long seed, uint32_t stream,
                                                 unsigned long long idx4) {
  uint32_t r[4];
  philox4x32_10(static_cast<uint32_t>(idx4), static_cast<uint32_t>(idx4 >> 32), stream, 0x6d7364u,
                static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), r);
  const float s = 2.3283064365386963e-10f;  // 2^-32
  const float u0 = (static_cast<float>(r[0]) + 0.5f) * s, u1 = (static_cast<float>(r[1]) + 0.5f) * s;
  const float u2 = (static_cast<float>(r[2]) + 0.5f) * s, u3 = (static_cast<float>(r[3]) + 0.5f) * s;
  const float ra = sqrtf(-2.0f * logf(fminf(fmaxf(u0, 1e-12f), 1.0f)));
  const float rb = sqrtf(-2.0f * logf(fminf(fmaxf(u2, 1e-12f), 1.0f)));
  float sa, ca, sb, cb;
  sincospif(2.0f * u1, &sa, &ca);
  sincospif(2.0f * u3, &sb, &cb);
  return make_float4(ra * ca, ra * sa, rb * cb, rb * sb);
}

// clip(v, lo, hi) as jnp.clip and torch.clamp compute it: a NaN stays NaN (fminf / fmaxf alone
// return the non-NaN operand, which would turn a NaN into a plausible bound)
__device__ __forceinline__ float clip_nan(float v, float lo, float hi) {
  return v != v ? v : fminf(fmaxf(v, lo), hi);
}

__device__ __forceinline__ void store_split4(bf16* zs, long long idx, int n_dims, float4 v) {
  const long long row = idx / n_dims;
  const int col = static_cast<int>(idx - row * n_dims);
  bf16* o = zs + row * (3LL * n_dims) + col;
  bf16 h0, h1, h2, h3, l0, l1, l2, l3;
  split_bf16(v.x, h0, l0); split_bf16(v.y, h1, l1);
  split_bf16(v.z, h2, l2); split_bf16(v.w, h3, l3);
  __nv_bfloat162 a = __halves2bfloat162(h0, h1), b = __halves2bfloat162(h2, h3);
  __nv_bfloat162 c = __halves2bfloat162(l0, l1), d = __halves2bfloat162(l2, l3);
  uint2 uh, ul;
  uh.x = *reinterpret_cast<uint32_t*>(&a); uh.y = *reinterpret_cast<uint32_t*>(&b);
  ul.x = *reinterpret_cast<uint32_t*>(&c); ul.y = *reinterpret_cast<uint32_t*>(&d);
  *reinterpret_cast<uint2*>(o) = uh;
  *reinterpret_cast<uint2*>(o + n_dims) = ul;
  *reinterpret_cast<uint2*>(o + 2 * n_dims) = uh;
}

// ---------------------------------------------------------------------------
// jax.random (threefry2x32) noise, restated from the published algorithm (jax 0.3.16 defaults;
// CPU twin and derivation: music_spectrogram_diffusion_b200/jax_rng.py).  Element e of an
// n-element draw is word e of threefry_2x32(key, arange(n)): the counters are split into halves,
// so e < n/2 is the first output word of the pair (e, e + n/2) and e >= n/2 the second word of
// (e - n/2, e).
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint2 threefry2x32(uint32_t k0, uint32_t k1, uint32_t x0, uint32_t x1) {
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  x0 += ks[0];
  x1 += ks[1];
#pragma unroll
  for (int g = 0; g < 5; ++g) {
    const int r0 = (g & 1) ? 17 : 13, r1 = (g & 1) ? 29 : 15, r2 = (g & 1) ? 16 : 26, r3 = (g & 1) ? 24 : 6;
    x0 += x1; x1 = __funnelshift_l(x1, x1, r0) ^ x0;
    x0 += x1; x1 = __funnelshift_l(x1, x1, r1) ^ x0;
    x0 += x1; x1 = __funnelshift_l(x1, x1, r2) ^ x0;
    x0 += x1; x1 = __funnelshift_l(x1, x1, r3) ^ x0;
    x0 += ks[(g + 1) % 3];
    x1 += ks[(g + 2) % 3] + static_cast<uint32_t>(g + 1);
  }
  return make_uint2(x0, x1);
}

// XLA's float32 erfinv (Giles' two single-precision polynomials in w = -log1p(-x^2))
__device__ __forceinline__ float erfinv_xla(float x) {
  const float w = -log1pf(-x * x);
  float p;
  if (w < 5.0f) {
    const float v = w - 2.5f;
    p = 2.81022636e-08f;
    p = 3.43273939e-07f + p * v; p = -3.5233877e-06f + p * v; p = -4.39150654e-06f + p * v;
    p = 0.00021858087f + p * v; p = -0.00125372503f + p * v; p = -0.00417768164f + p * v;
    p = 0.246640727f + p * v; p = 1.50140941f + p * v;
  } else {
    const float v = sqrtf(w) - 3.0f;
    p = -0.000200214257f;
    p = 0.000100950558f + p * v; p = 0.00134934322f + p * v; p = -0.00367342844f + p * v;
    p = 0.00573950773f + p * v; p = -0.0076224613f + p * v; p = 0.00943887047f + p * v;
    p = 1.00167406f + p * v; p = 2.83297682f + p * v;
  }
  return p * x;
}

__device__ __forceinline__ float jax_normal_from_bits(uint32_t bits) {
  const float f = __uint_as_float((bits >> 9) | 0x3F800000u) - 1.0f;
  const float lo = -0.99999994f;                       // nextafter(-1, 0); (1 - lo) rounds to 2
  const float u = fmaxf(lo, __fadd_rn(__fmul_rn(f, 2.0f), lo));
  return 1.41421354f * erfinv_xla(u);
}

// random words for elements [4*i4, 4*i4 + 4) of an n-element draw (n a multiple of 8)
__device__ __forceinline__ uint4 jax_bits4(const uint32_t* key, long long n, long long i4) {
  const uint32_t k0 = key[0], k1 = key[1];
  const long long half = n >> 1, e = i4 * 4;
  uint32_t r[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long ej = e + j;
    const bool second = ej >= half;
    const uint32_t c0 = static_cast<uint32_t>(second ? ej - half : ej);
    const uint2 o = threefry2x32(k0, k1, c0, static_cast<uint32_t>(c0 + half));
    r[j] = second ? o.y : o.x;
  }
  return make_uint4(r[0], r[1], r[2], r[3]);
}
// normals for the same elements
__device__ __forceinline__ float4 jax_normal4(const uint32_t* key, long long n, long long i4) {
  const uint4 b = jax_bits4(key, n, i4);
  return make_float4(jax_normal_from_bits(b.x), jax_normal_from_bits(b.y),
                     jax_normal_from_bits(b.z), jax_normal_from_bits(b.w));
}

// ---------------------------------------------------------------------------
// One reverse-diffusion update (CFG combine + x0 + clip + DDPM/DDIM mean + noise)
// ---------------------------------------------------------------------------
__device__ __forceinline__ void sampler_step_body(const SamplerArgs& a, int step,
                                                  const float* noise_base, float* mel_base,
                                                  unsigned long long seed, long long i4,
                                                  bool per_row,
                                                  const float* eps_cond = nullptr,
                                                  const float* eps_uncond = nullptr) {
  const long long idx = i4 * 4;
  if (eps_cond == nullptr) {
    eps_cond = a.eps;
    eps_uncond = a.eps + a.n;
  }
  const float* cf = a.coef + static_cast<size_t>(step) * MSD_STEP_COLS;
  const float x0_scale = cf[0], eps_scale = cf[1], c_z = cf[2], c_x0 = cf[3], sigma = cf[4];
  const bool last = cf[5] != 0.f;
  const float p0 = cf[8], p1 = cf[9], q0 = cf[10], q1 = cf[11], e1 = cf[12], e2 = cf[13];
  const float4 z = *reinterpret_cast<const float4*>(a.z + idx);
  const float4 mo = *reinterpret_cast<const float4*>(eps_cond + idx);
  // _get_x0_and_eps_from_model_output (diffusion_utils.py:288-321): eps = p0 z + p1 out and
  // x0 = q0 z + q1 out (for model_output == 'eps': p0 = 0, p1 = 1, i.e. eps = out exactly)
  float4 e, x0;
  e.x = fmaf(p1, mo.x, p0 * z.x); e.y = fmaf(p1, mo.y, p0 * z.y);
  e.z = fmaf(p1, mo.z, p0 * z.z); e.w = fmaf(p1, mo.w, p0 * z.w);
  if (p0 == 0.f && p1 == 1.f) e = mo;
  if (a.passes == 2) {
    // classifier-free guidance on eps, then x0 from the combined eps at logsnr_t (424-433)
    const float4 mu = *reinterpret_cast<const float4*>(eps_uncond + idx);
    float4 eu;
    eu.x = fmaf(p1, mu.x, p0 * z.x); eu.y = fmaf(p1, mu.y, p0 * z.y);
    eu.z = fmaf(p1, mu.z, p0 * z.z); eu.w = fmaf(p1, mu.w, p0 * z.w);
    if (p0 == 0.f && p1 == 1.f) eu = mu;
    const float w = a.cond_weight, wu = 1.0f - a.cond_weight;
    e.x = w * e.x + wu * eu.x; e.y = w * e.y + wu * eu.y;
    e.z = w * e.z + wu * eu.z; e.w = w * e.w + wu * eu.w;
    x0.x = x0_scale * (z.x - e.x * eps_scale); x0.y = x0_scale * (z.y - e.y * eps_scale);
    x0.z = x0_scale * (z.z - e.z * eps_scale); x0.w = x0_scale * (z.w - e.w * eps_scale);
  } else if (q0 == 0.f && q1 == 1.f) {
    x0 = mo;
  } else if (p0 == 0.f && p1 == 1.f) {
    // predict_x0_from_eps at the train schedule's logsnr: q0 = A, q1 = -A * B
    const float A = q0, Bc = -q1 / q0;
    x0.x = A * (z.x - mo.x * Bc); x0.y = A * (z.y - mo.y * Bc);
    x0.z = A * (z.z - mo.z * Bc); x0.w = A * (z.w - mo.w * Bc);
  } else {
    x0.x = fmaf(q1, mo.x, q0 * z.x); x0.y = fmaf(q1, mo.y, q0 * z.y);
    x0.z = fmaf(q1, mo.z, q0 * z.z); x0.w = fmaf(q1, mo.w, q0 * z.w);
  }
  if (a.clip_x0) {
    x0.x = clip_nan(x0.x, -1.f, 1.f); x0.y = clip_nan(x0.y, -1.f, 1.f);
    x0.z = clip_nan(x0.z, -1.f, 1.f); x0.w = clip_nan(x0.w, -1.f, 1.f);
    if (a.ddim) {  // pred_eps = predict_eps_from_x0(z, clipped x0, logsnr_t) (437-439)
      e.x = e1 * (z.x - x0.x * e2); e.y = e1 * (z.y - x0.y * e2);
      e.z = e1 * (z.z - x0.z * e2); e.w = e1 * (z.w - x0.w * e2);
    }
  }
  float4 zn;
  if (last) {
    zn = x0;
  } else if (a.ddim) {
    // ddim_step (369-379): z_s = alpha_s x0 + stdv_s eps; table columns 3 / 2
    zn.x = c_x0 * x0.x + c_z * e.x; zn.y = c_x0 * x0.y + c_z * e.y;
    zn.z = c_x0 * x0.z + c_z * e.z; zn.w = c_x0 * x0.w + c_z * e.w;
  } else {
    float4 nz = make_float4(0.f, 0.f, 0.f, 0.f);
    if (sigma != 0.f) {
      if (noise_base != nullptr) {
        nz = *reinterpret_cast<const float4*>(noise_base + static_cast<size_t>(step) * a.n + idx);
      } else {
        long long n = a.n, j4 = i4;
        const uint32_t* keys = a.rng_keys;
        if (per_row) {  // row b's own draw of n_row elements (i4 < 2^30: n < 2^32 is required)
          const unsigned int b = static_cast<unsigned int>(i4) / static_cast<unsigned int>(a.n_row >> 2);
          n = a.n_row;
          j4 = i4 - static_cast<long long>(b) * (a.n_row >> 2);
          keys = a.row_keys + b * a.row_key_stride;
          if (a.rng_kind == 0) seed = a.row_seeds[b];
        }
        nz = a.rng_kind == 1
                 ? jax_normal4(keys + 2 * (step + 1), n, j4)
                 : philox_normal4(seed, static_cast<uint32_t>(step) + 1u,
                                  static_cast<unsigned long long>(j4));
      }
    }
    zn.x = c_z * z.x + c_x0 * x0.x + sigma * nz.x; zn.y = c_z * z.y + c_x0 * x0.y + sigma * nz.y;
    zn.z = c_z * z.z + c_x0 * x0.z + sigma * nz.z; zn.w = c_z * z.w + c_x0 * x0.w + sigma * nz.w;
  }
  *reinterpret_cast<float4*>(a.z + idx) = zn;
  store_split4(a.z_split, idx, a.n_dims, zn);
  if (last && mel_base != nullptr) {
    // scale_to_features, msd/audio_codecs.py:176-183 with input_range (-1, 1)
    const float span = a.feat_max - a.feat_min;
    float4 f;
    f.x = (zn.x + 1.f) * 0.5f * span + a.feat_min; f.y = (zn.y + 1.f) * 0.5f * span + a.feat_min;
    f.z = (zn.z + 1.f) * 0.5f * span + a.feat_min; f.w = (zn.w + 1.f) * 0.5f * span + a.feat_min;
    *reinterpret_cast<float4*>(mel_base + idx) = f;
  }
}

__device__ __forceinline__ void prefetch_next_film(const SamplerArgs& a, int step, long long gid) {
  if (step < 1) return;
  const long long off = gid * 32;  // one 128-byte line per thread and table
  if (a.film != nullptr && off < a.film_step_floats) {
    const float* ptr = a.film + static_cast<long long>(step - 1) * a.film_step_floats + off;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
  }
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    if (a.pf[t] != nullptr && off < a.pf_step_floats[t]) {
      const float* ptr = a.pf[t] + static_cast<long long>(step - 1) * a.pf_step_floats[t] + off;
      asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr));
    }
  }
}

__global__ void __launch_bounds__(256) sampler_step_kernel(const SamplerArgs a) {
  griddep_launch_dependents();
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  griddep_wait();
  if (a.run == nullptr) {
    const int step = *a.step;
    prefetch_next_film(a, step, i4);
    if (i4 * 4 < a.n) sampler_step_body(a, step, a.noise, a.mel_out, a.seed, i4, false);
    return;
  }
  // Per-call arguments and the step index live in device memory (RunArgs).  The step advance is
  // folded in: every block counts itself done once all its threads hold `step` in a register, and
  // the last one to arrive decrements it for the next graph launch.
  __shared__ int s_step;
  if (threadIdx.x == 0) {
    // thread 0 alone reads the step index (its store to shared memory needs the loaded value, so
    // the load has completed before the atomic below is issued) and hands it to the block
    const int st = *reinterpret_cast<volatile int*>(&a.run->step);
    s_step = st;
    __threadfence();
    const unsigned int prev = atomicAdd(&a.run->done, 1u);
    if (prev == gridDim.x - 1) {
      a.run->done = 0u;
      a.run->step = st - 1;
    }
  }
  __syncthreads();
  const int step = s_step;
  prefetch_next_film(a, step, i4);
  const float* noise_base = a.run->noise;
  float* mel_base = a.run->mel_out;
  const unsigned long long seed = a.run->seed;
  const bool per_row = a.run->per_row != 0;
  if (a.xrole != 0) {
    // ---- guidance split: send my pass's eps to the peer, receive the peer's
    __shared__ unsigned int s_seq;
    if (threadIdx.x == 0) s_seq = *reinterpret_cast<volatile unsigned int*>(&a.run->xseq);
    __syncthreads();
    const unsigned int seq = s_seq;
    const long long par = static_cast<long long>(seq & 1u) * a.xparity_floats;
    if (i4 * 4 < a.n)
      *reinterpret_cast<float4*>(a.xpeer + par + i4 * 4) = *reinterpret_cast<const float4*>(a.eps + i4 * 4);
    __threadfence_system();   // my stores are visible to the peer before the flag is
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned int prev = atomicAdd(&a.run->xsent, 1u);
      if (prev == gridDim.x - 1) {   // every block's share is on its way: raise the peer's flag
        a.run->xsent = 0u;
        a.run->xseq = seq + 1u;
        unsigned int* pflag = reinterpret_cast<unsigned int*>(a.xpeer + a.xflags_off) + (seq & 1u);
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(pflag), "r"(seq) : "memory");
      }
      // wait for the peer's values of this step
      const unsigned int* lflag = reinterpret_cast<const unsigned int*>(a.xlocal + a.xflags_off) + (seq & 1u);
      unsigned int v;
      unsigned long long spins = 0;
      do {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(lflag) : "memory");
        if (v != seq) {
          __nanosleep(200);
          if (++spins > (1ull << 26)) __trap();   // ~15 s: the peer is gone, fail loudly
        }
      } while (v != seq);
    }
    __syncthreads();
    const float* other = a.xlocal + par;
    const float* ec = a.xrole == 1 ? a.eps : other;
    const float* eu = a.xrole == 1 ? other : a.eps;
    if (i4 * 4 < a.n) sampler_step_body(a, step, noise_base, mel_base, seed, i4, per_row, ec, eu);
    return;
  }
  if (i4 * 4 < a.n) sampler_step_body(a, step, noise_base, mel_base, seed, i4, per_row);
}

__global__ void __launch_bounds__(256)
init_z_kernel(const float* init_z, float* z, bf16* zs, long long n, int n_dims,
              unsigned long long seed, int rng_kind, const uint32_t* rng_keys, long long n_row,
              long long row_key_stride, const unsigned long long* row_seeds) {
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long idx = i4 * 4;
  if (idx >= n) return;
  float4 v;
  if (init_z != nullptr) {
    v = *reinterpret_cast<const float4*>(init_z + idx);
  } else {
    long long m = n, j4 = i4;
    if (n_row > 0) {  // per-row streams, as in sampler_step_body
      const unsigned int b = static_cast<unsigned int>(i4) / static_cast<unsigned int>(n_row >> 2);
      m = n_row;
      j4 = i4 - static_cast<long long>(b) * (n_row >> 2);
      rng_keys += b * row_key_stride;
      if (rng_kind == 0) seed = row_seeds[b];
    }
    v = rng_kind == 1 ? jax_normal4(rng_keys, m, j4)
                      : philox_normal4(seed, 0u, static_cast<unsigned long long>(j4));
  }
  *reinterpret_cast<float4*>(z + idx) = v;
  store_split4(zs, idx, n_dims, v);
}

// ---------------------------------------------------------------------------
// Encoder front ends
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_tokens_kernel(const int* tokens, const float* emb, const float* pos, float* x, int rows,
                    int T, int d, int vocab) {
  const int d4 = d >> 2;
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long long>(rows) * d4) return;
  const int row = static_cast<int>(gid / d4), c = static_cast<int>(gid - static_cast<long long>(row) * d4);
  int tok = tokens[row];
  tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
  const int t = row % T;
  const float4 e = __ldg(reinterpret_cast<const float4*>(emb + static_cast<size_t>(tok) * d) + c);
  const float4 pp = __ldg(reinterpret_cast<const float4*>(pos + static_cast<size_t>(t) * d) + c);
  reinterpret_cast<float4*>(x + static_cast<size_t>(row) * d)[c] =
      make_float4(e.x + pp.x, e.y + pp.y, e.z + pp.z, e.w + pp.w);
}

__global__ void __launch_bounds__(256)
scale_split_kernel(const float* feat, bf16* out, long long n, int n_dims, float fmin, float fmax) {
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long idx = i4 * 4;
  if (idx >= n) return;
  float4 f = *reinterpret_cast<const float4*>(feat + idx);
  // scale_features(clip=True), msd/audio_codecs.py:166-174 with output_range (-1, 1)
  const float inv = 1.0f / (fmax - fmin);
  f.x = (clip_nan(f.x, fmin, fmax) - fmin) * inv * 2.0f - 1.0f;
  f.y = (clip_nan(f.y, fmin, fmax) - fmin) * inv * 2.0f - 1.0f;
  f.z = (clip_nan(f.z, fmin, fmax) - fmin) * inv * 2.0f - 1.0f;
  f.w = (clip_nan(f.w, fmin, fmax) - fmin) * inv * 2.0f - 1.0f;
  store_split4(out, idx, n_dims, f);
}

// rows of fp32 -> [hi | lo | hi] bf16 rows (A operand of a split-precision GEMM)
__global__ void __launch_bounds__(256)
split3_rows_kernel(const float* src, bf16* out, long long n, int cols) {
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long idx = i4 * 4;
  if (idx >= n) return;
  store_split4(out, idx, cols, *reinterpret_cast<const float4*>(src + idx));
}

// One block per batch row: key-mask bit words for [tokens | context] and the
// terminal-relative roll amount (= get_sequence_length of the context mask).
__global__ void __launch_bounds__(256)
build_masks_kernel(const int* tokens, const int* ctx_mask, int T, int C, uint32_t* bits,
                   int* ctx_seq_len, int terminal_relative) {
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int words_t = T >> 5, words_c = C >> 5;
  uint32_t* brow = bits + static_cast<size_t>(b) * (words_t + words_c);
  __shared__ int first_zero;
  if (threadIdx.x == 0) first_zero = C;
  __syncthreads();
  for (int w = warp; w < words_t; w += nw) {
    const uint32_t m = __ballot_sync(0xffffffffu, tokens[static_cast<size_t>(b) * T + w * 32 + lane] > 0);
    if (lane == 0) brow[w] = m;
  }
  for (int w = warp; w < words_c; w += nw) {
    const int v = ctx_mask[static_cast<size_t>(b) * C + w * 32 + lane];
    const uint32_t m = __ballot_sync(0xffffffffu, v > 0);
    const uint32_t z = __ballot_sync(0xffffffffu, v == 0);
    if (lane == 0) {
      brow[words_t + w] = m;
      if (z) atomicMin(&first_zero, w * 32 + __ffs(z) - 1);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // network.py:28-39: first zero index, or the full length when there is no zero.
    int len = first_zero;  // == C when no zero was found
    ctx_seq_len[b] = terminal_relative ? (len % C) : 0;  // roll by C == roll by 0
  }
}

// ---------------------------------------------------------------------------
// Load-time: weight packing and fp32 SIMT GEMM
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
pack_weight_kernel(const float* W, int K, int N, bf16* dst, int ldd, int n_off, int k_off,
                   int part) {
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= static_cast<long long>(K) * N) return;
  const int n = static_cast<int>(gid / K), k = static_cast<int>(gid - static_cast<long long>(n) * K);
  const float w = W[static_cast<size_t>(k) * N + n];
  bf16 hi, lo;
  split_bf16(w, hi, lo);
  dst[static_cast<size_t>(n_off + n) * ldd + k_off + k] = part ? lo : hi;
}

__global__ void __launch_bounds__(256)
pack_gated_kernel(const float* W0, const float* W1, int K, int F, bf16* dst, int ldd, int k_off,
                  int part) {
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (gid >= 2LL * F * K) return;
  const int r = static_cast<int>(gid / K), k = static_cast<int>(gid - static_cast<long long>(r) * K);
  const int g = r >> 6, j = r & 63;
  const float* W = (j < 32) ? W0 : W1;
  const int col = g * 32 + (j & 31);
  bf16 hi, lo;
  split_bf16(W[static_cast<size_t>(k) * F + col], hi, lo);
  dst[static_cast<size_t>(r) * ldd + k_off + k] = part ? lo : hi;
}

constexpr int SG_T = 64, SG_K = 16;
__global__ void __launch_bounds__(256)
sgemm_f32_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C,
                 int ldc, int M, int N, int K, int act) {
  __shared__ float sA[SG_K][SG_T + 1];
  __shared__ float sB[SG_K][SG_T + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * SG_T, n0 = blockIdx.x * SG_T;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += SG_K) {
    for (int e = threadIdx.x; e < SG_T * SG_K; e += 256) {
      const int am = e / SG_K, ak = e % SG_K;
      const int gm = m0 + am, gk = k0 + ak;
      sA[ak][am] = (gm < M && gk < K) ? A[static_cast<size_t>(gm) * K + gk] : 0.f;
      const int bk = e / SG_T, bn = e % SG_T;
      const int gn = n0 + bn, gk2 = k0 + bk;
      sB[bk][bn] = (gn < N && gk2 < K) ? B[static_cast<size_t>(gk2) * N + gn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SG_K; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sA[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = sB[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gm = m0 + ty * 4 + i, gn = n0 + tx * 4 + j;
      if (gm < M && gn < N) {
        float v = acc[i][j];
        if (act == 1) v = v / (1.0f + expf(-v));  // swish = x * sigmoid(x)
        C[static_cast<size_t>(gm) * ldc + gn] = v;
      }
    }
}

__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* s, bf16* d, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) d[i] = __float2bfloat16_rn(s[i]);
}
__global__ void __launch_bounds__(256) bf16_to_f32_kernel(const bf16* s, float* d, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) d[i] = __bfloat162float(s[i]);
}
// dst[r][c] = src[r * ld + c] (+ src[r * ld + lo_off + c] when lo_off > 0: hi + lo of a split row)
__global__ void __launch_bounds__(256)
bf16_rows_to_f32_kernel(const bf16* s, int ld, int lo_off, float* d, long long rows, int cols) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const long long r = i / cols;
  const int c = static_cast<int>(i - r * cols);
  float v = __bfloat162float(s[r * ld + c]);
  if (lo_off > 0) v += __bfloat162float(s[r * ld + lo_off + c]);
  d[i] = v;
}
// dst rows [rows, units] of 16-byte units with row strides in units; triggers its dependents at
// entry, so a kernel launched behind it with PDL overlaps it up to its own dependency wait
__global__ void __launch_bounds__(256)
copy_rows_kernel(const uint4* s, long long lds, uint4* d, long long ldd, long long rows, int units) {
  griddep_launch_dependents();
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  griddep_wait();
  if (i >= rows * units) return;
  const long long r = i / units;
  const int c = static_cast<int>(i - r * units);
  d[r * ldd + c] = s[r * lds + c];
}
__global__ void __launch_bounds__(256)
mask_bits_kernel(const int* mask, long long words, uint32_t* bits) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= words) return;
  const uint32_t m = __ballot_sync(0xffffffffu, mask[w * 32 + lane] > 0);
  if (lane == 0) bits[w] = m;
}

inline int blocks_for(long long n, int per_block) {
  return static_cast<int>((n + per_block - 1) / per_block);
}

}  // namespace

// Every kernel of the per-step graph asks for the maximum shared-memory carve-out, including the
// ones that use no shared memory: alternating carve-outs between consecutive kernels forces an SM
// reconfiguration (the SM must drain first), which also defeats programmatic dependent launch.
int elementwise_configure() {
  MSD_CUDA_CHECK(cudaFuncSetAttribute(sampler_step_kernel,
                                      cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  MSD_CUDA_CHECK(cudaFuncSetAttribute(init_z_kernel,
                                      cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  return 0;
}

int launch_rmsnorm(const float* x, const float* gamma, int rows, int d, bf16* out, int ldo,
                   const float* film, const int* step, long long film_step_stride,
                   long long film_offset, int split3, cudaStream_t stream) {
  MSD_REQUIRE(d % 128 == 0 && d <= 128 * NORM_MAX_ITERS, "rmsnorm: d=%d must be k*128 <= 1024", d);
  NormDev p;
  p.x = x; p.gamma = gamma; p.out = out; p.film = film; p.step = step;
  p.film_step_stride = film_step_stride; p.film_offset = film_offset;
  p.rows = rows; p.d = d; p.ldo = ldo; p.split3 = split3;
  p.src_len = 0; p.dst_len = 0; p.dst_off = 0;
  p.ss_out = nullptr; p.gamma_step_stride = 0;
  ProfScope prof(KC_NORM, 0.0, static_cast<double>(rows) * d * (4.0 + (split3 ? 6.0 : 2.0)), stream);
  MSD_TRY_RC(launch_norm(p, stream));
  ++g_launch_count;
  return 0;
}

int launch_prep_rows(const float* x, const float* g, long long g_step_stride, const int* step, int rows,
                     int d, bf16* a_out, int lda, float* ss_out, cudaStream_t stream) {
  MSD_REQUIRE(d % 128 == 0 && d <= 128 * NORM_MAX_ITERS, "prep_rows: d=%d must be k*128 <= 1024", d);
  MSD_REQUIRE(x && g && step && a_out && ss_out, "prep_rows: null argument");
  NormDev p;
  p.x = x; p.gamma = g; p.out = a_out; p.film = nullptr; p.step = step;
  p.film_step_stride = 0; p.film_offset = 0;
  p.rows = rows; p.d = d; p.ldo = lda; p.split3 = 0;
  p.src_len = 0; p.dst_len = 0; p.dst_off = 0;
  p.ss_out = ss_out; p.gamma_step_stride = g_step_stride;
  ProfScope prof(KC_NORM, 0.0, static_cast<double>(rows) * d * 6.0, stream);
  MSD_TRY_RC(launch_norm(p, stream));
  ++g_launch_count;
  return 0;
}

int launch_rmsnorm_rows_remap(const float* x, const float* gamma, int B, int src_len, int d,
                              bf16* out, int dst_len, int dst_off, cudaStream_t stream,
                              int split3) {
  MSD_REQUIRE(d % 128 == 0 && d <= 128 * NORM_MAX_ITERS, "rmsnorm: d=%d must be k*128 <= 1024", d);
  NormDev p;
  p.x = x; p.gamma = gamma; p.out = out; p.film = nullptr; p.step = nullptr;
  p.film_step_stride = 0; p.film_offset = 0;
  p.rows = B * src_len; p.d = d; p.ldo = split3 ? 3 * d : d; p.split3 = split3;
  p.src_len = src_len; p.dst_len = dst_len; p.dst_off = dst_off;
  p.ss_out = nullptr; p.gamma_step_stride = 0;
  MSD_TRY_RC(launch_norm(p, stream));
  ++g_launch_count;
  return 0;
}

int launch_sampler_step(const SamplerArgs& a, cudaStream_t stream) {
  MSD_REQUIRE(a.n % 4 == 0 && a.n_dims % 4 == 0, "sampler: sizes must be multiples of 4");
  ProfScope prof(KC_SAMPLER, 0.0, static_cast<double>(a.n) * (4.0 * (a.passes + 3) + 6.0), stream);
  MSD_CUDA_CHECK(launch_kernel(sampler_step_kernel, dim3(blocks_for(a.n / 4, 256)), dim3(256), 0, stream, a));
  ++g_launch_count;
  return 0;
}

__global__ void __launch_bounds__(256)
jax_normal_kernel(uint32_t k0, uint32_t k1, long long n, float* out) {
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i4 * 4 >= n) return;
  const uint32_t key[2] = {k0, k1};
  *reinterpret_cast<float4*>(out + i4 * 4) = jax_normal4(key, n, i4);
}

__global__ void __launch_bounds__(256)
jax_bits_kernel(uint32_t k0, uint32_t k1, long long n, uint32_t* out) {
  const long long i4 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i4 * 4 >= n) return;
  const uint32_t key[2] = {k0, k1};
  *reinterpret_cast<uint4*>(out + i4 * 4) = jax_bits4(key, n, i4);
}

int launch_jax_bits(uint32_t k0, uint32_t k1, long long n, uint32_t* out, cudaStream_t stream) {
  MSD_REQUIRE(n > 0 && n % 8 == 0 && n < (1ll << 32), "jax_bits: n must be k*8 < 2^32");
  jax_bits_kernel<<<blocks_for(n / 4, 256), 256, 0, stream>>>(k0, k1, n, out);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_jax_normal(uint32_t k0, uint32_t k1, long long n, float* out, cudaStream_t stream) {
  MSD_REQUIRE(n > 0 && n % 8 == 0 && n < (1ll << 32), "jax_normal: n must be k*8 < 2^32");
  jax_normal_kernel<<<blocks_for(n / 4, 256), 256, 0, stream>>>(k0, k1, n, out);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_init_z(const float* init_z, float* z, bf16* z_split, long long n, int n_dims,
                  unsigned long long seed, cudaStream_t stream, int rng_kind,
                  const uint32_t* rng_keys, long long n_row, long long row_key_stride,
                  const unsigned long long* row_seeds) {
  MSD_REQUIRE(rng_kind == 0 || (rng_keys != nullptr && n % 8 == 0 && n < (1ll << 32)),
              "init_z: the jax stream needs its key table and a draw of k*8 < 2^32 elements");
  MSD_REQUIRE(n_row == 0 || (n_row > 0 && n_row % 8 == 0 && n % n_row == 0 && n < (1ll << 32) &&
                             rng_keys != nullptr && row_seeds != nullptr),
              "init_z: per-row streams need rows of k*8 elements, n < 2^32 and both row tables");
  init_z_kernel<<<blocks_for(n / 4, 256), 256, 0, stream>>>(init_z, z, z_split, n, n_dims, seed,
                                                            rng_kind, rng_keys, n_row,
                                                            row_key_stride, row_seeds);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

int launch_embed_tokens(const int* tokens, const float* emb, const float* pos, float* x, int B,
                        int T, int d, int vocab, cudaStream_t stream) {
  const long long n = static_cast<long long>(B) * T * (d / 4);
  embed_tokens_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(tokens, emb, pos, x, B * T, T, d,
                                                              vocab);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

int launch_scale_split(const float* feat, bf16* out_split, long long rows, int n_dims, float fmin,
                       float fmax, cudaStream_t stream) {
  const long long n = rows * n_dims;
  scale_split_kernel<<<blocks_for(n / 4, 256), 256, 0, stream>>>(feat, out_split, n, n_dims, fmin,
                                                                 fmax);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

int launch_split3_rows(const float* src, bf16* out_split, long long rows, int cols,
                       cudaStream_t stream) {
  MSD_REQUIRE(cols % 4 == 0, "split3_rows: cols must be a multiple of 4");
  const long long n = rows * cols;
  split3_rows_kernel<<<blocks_for(n / 4, 256), 256, 0, stream>>>(src, out_split, n, cols);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_build_masks(const int* tokens, const int* ctx_mask, int B, int T, int C, uint32_t* bits,
                       int* ctx_seq_len, int terminal_relative, cudaStream_t stream) {
  MSD_REQUIRE(T % 128 == 0 && C % 128 == 0, "masks: lengths must be multiples of 128");
  build_masks_kernel<<<B, 256, 0, stream>>>(tokens, ctx_mask, T, C, bits, ctx_seq_len,
                                            terminal_relative);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

int launch_pack_weight(const float* W, int K, int N, bf16* dst, int ldd, int n_off, int k_off,
                       int part, cudaStream_t stream) {
  pack_weight_kernel<<<blocks_for(static_cast<long long>(K) * N, 256), 256, 0, stream>>>(
      W, K, N, dst, ldd, n_off, k_off, part);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_pack_gated(const float* W0, const float* W1, int K, int F, bf16* dst, int ldd,
                      cudaStream_t stream, int k_off, int part) {
  MSD_REQUIRE(F % 32 == 0, "pack_gated: F must be a multiple of 32");
  pack_gated_kernel<<<blocks_for(2LL * F * K, 256), 256, 0, stream>>>(W0, W1, K, F, dst, ldd, k_off,
                                                                      part);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_f32_to_bf16(const float* src, bf16* dst, long long n, cudaStream_t stream) {
  f32_to_bf16_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(src, dst, n);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}
int launch_bf16_to_f32(const bf16* src, float* dst, long long n, cudaStream_t stream) {
  bf16_to_f32_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(src, dst, n);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}
int launch_bf16_rows_to_f32(const bf16* src, int ld, int lo_off, float* dst, long long rows, int cols,
                            cudaStream_t stream) {
  bf16_rows_to_f32_kernel<<<blocks_for(rows * cols, 256), 256, 0, stream>>>(src, ld, lo_off, dst,
                                                                            rows, cols);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}
int launch_mask_bits(const int* mask, int nb, int L, uint32_t* bits, cudaStream_t stream) {
  MSD_REQUIRE(L % 128 == 0, "mask_bits: L must be a multiple of 128");
  const long long words = static_cast<long long>(nb) * (L / 32);
  mask_bits_kernel<<<blocks_for(words * 32, 256), 256, 0, stream>>>(mask, words, bits);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}
int launch_copy_rows(const void* src, long long ld_src, void* dst, long long ld_dst, long long rows,
                     int row_bytes, cudaStream_t stream) {
  MSD_REQUIRE(row_bytes % 16 == 0 && ld_src % 16 == 0 && ld_dst % 16 == 0 &&
                  (reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
              "copy_rows: rows, strides and pointers must be 16-byte aligned");
  const int units = row_bytes / 16;
  MSD_CUDA_CHECK(launch_kernel(copy_rows_kernel, dim3(blocks_for(rows * units, 256)), dim3(256), 0, stream,
                               static_cast<const uint4*>(src), ld_src / 16, static_cast<uint4*>(dst),
                               ld_dst / 16, rows, units));
  ++g_launch_count;
  return 0;
}

// Deferred-normalisation tables (load time).  gain[s, :] = gamma * (1 + film_scale[s, :]);
// bias[s, n] = sum_k film_bias[s, k] * W[n, k] (W: packed bf16 weight rows, as the GEMM reads them).
__global__ void film_gain_kernel(const float* __restrict__ film, long long film_stride,
                                 const float* __restrict__ gamma, float* __restrict__ out,
                                 long long out_stride, int steps, int d) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(steps) * d) return;
  const int s = static_cast<int>(i / d), k = static_cast<int>(i - static_cast<long long>(s) * d);
  out[s * out_stride + k] = gamma[k] * (1.0f + film[s * film_stride + k]);
}
constexpr int FB_STEPS = 8;
__global__ void __launch_bounds__(128)
film_bias_kernel(const float* __restrict__ fb, long long fb_stride, const bf16* __restrict__ W,
                 int ldw, float* __restrict__ out, long long out_stride, int steps, int N, int K) {
  extern __shared__ float s_fb[];  // [FB_STEPS][K]
  const int s0 = blockIdx.y * FB_STEPS;
  for (int i = threadIdx.x; i < FB_STEPS * K; i += blockDim.x) {
    const int s = i / K, k = i - s * K;
    s_fb[i] = (s0 + s < steps) ? fb[(s0 + s) * fb_stride + k] : 0.f;
  }
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float acc[FB_STEPS];
#pragma unroll
  for (int s = 0; s < FB_STEPS; ++s) acc[s] = 0.f;
  const uint4* wr = reinterpret_cast<const uint4*>(W + static_cast<size_t>(n) * ldw);
  for (int k8 = 0; k8 < K / 8; ++k8) {
    const uint4 u = wr[k8];
    const uint32_t uu[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float w0 = __uint_as_float(uu[j] << 16), w1 = __uint_as_float(uu[j] & 0xffff0000u);
#pragma unroll
      for (int s = 0; s < FB_STEPS; ++s) {
        acc[s] = fmaf(s_fb[s * K + k8 * 8 + 2 * j], w0, acc[s]);
        acc[s] = fmaf(s_fb[s * K + k8 * 8 + 2 * j + 1], w1, acc[s]);
      }
    }
  }
#pragma unroll
  for (int s = 0; s < FB_STEPS; ++s)
    if (s0 + s < steps) out[(s0 + s) * out_stride + n] = acc[s];
}
int launch_film_gain(const float* film, long long film_stride, const float* gamma, float* out,
                     long long out_stride, int steps, int d, cudaStream_t stream) {
  film_gain_kernel<<<blocks_for(static_cast<long long>(steps) * d, 256), 256, 0, stream>>>(
      film, film_stride, gamma, out, out_stride, steps, d);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}
int launch_film_bias(const float* fb, long long fb_stride, const bf16* W, int ldw, float* out,
                     long long out_stride, int steps, int N, int K, cudaStream_t stream) {
  MSD_REQUIRE(K % 8 == 0 && ldw % 8 == 0 && FB_STEPS * K * 4 <= 48 * 1024,
              "film_bias: K=%d must be a multiple of 8 and <= 1536", K);
  dim3 grid((N + 127) / 128, (steps + FB_STEPS - 1) / FB_STEPS);
  film_bias_kernel<<<grid, 128, FB_STEPS * K * sizeof(float), stream>>>(fb, fb_stride, W, ldw, out,
                                                                       out_stride, steps, N, K);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int launch_sgemm_f32(const float* A, const float* B, float* C, int ldc, int M, int N, int K,
                     int act, cudaStream_t stream) {
  dim3 grid((N + SG_T - 1) / SG_T, (M + SG_T - 1) / SG_T);
  sgemm_f32_kernel<<<grid, 256, 0, stream>>>(A, B, C, ldc, M, N, K, act);
  MSD_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace msd
