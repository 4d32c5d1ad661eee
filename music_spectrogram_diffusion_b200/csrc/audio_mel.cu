// Audio -> MelGAN log-mel features (msd/audio_codecs.py:43-143, 204-247: Audio2Mel with MelGAN's
// constants), one fused fp32 kernel:
//   frame k = samples [320k, 320k + 640) of its row, zero past the end (tf.signal.frame, pad_end)
//   * periodic Hann window -> zero-padded to 1024 -> real FFT -> |X| (513 bins)
//   -> |X| @ W (W [513, 128], each column's non-zero band only) -> log(clip(., 1e-5, 1e8)).
// The FFT is a 512-point complex Stockham FFT (three radix-8 passes) of the even/odd-packed
// samples z[m] = x[2m] + i x[2m+1], followed by the real-split pass; twiddles are rounded from
// double.  It runs on the fp32 CUDA cores: tensor cores (and 3 x bf16 splits) cannot keep the
// ~2^-24 relative error the features are held to (DESIGN section 4).
//
// One warp computes one frame at a time, start to finish, through the same instructions whatever
// the frame's index, row or the size of the launch: a frame's output bits depend on its 640
// samples (and the two tables) only.
#include "common.cuh"
#include "kernels.h"

namespace msd {
namespace {

constexpr int kWin = 640;      // window (frame) length, samples
constexpr int kHop = 320;      // frame step, samples
constexpr int kHalf = 512;     // complex FFT length (1024-point real FFT)
constexpr int kBins = 513;     // rfft bins
constexpr int kMels = 128;
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kBandCap = 2048;  // packed band weights held in shared memory (MelGAN's: 1012)

struct MelSmem {
  float2 tw[kHalf];            // e^{-2 pi i k / 1024}
  float win[kWin];
  int band_lo[kMels];          // column j's weights: rows [lo, lo + len) of W ...
  int band_len[kMels];
  int band_off[kMels];         // ... packed at band_w[off ..]
  int band_total;
  float band_w[kBandCap];
  float2 buf[kWarps][kHalf];   // per warp: the FFT in place, then the 513 magnitudes
};

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 mul_neg_i(float2 a) { return make_float2(a.y, -a.x); }

// e^{-2 pi i e / 512}, 0 <= e < 512
__device__ __forceinline__ float2 w512(const float2* tw, int e) {
  if (e < kHalf / 2) return tw[2 * e];
  const float2 t = tw[2 * e - kHalf];
  return make_float2(-t.x, -t.y);
}

__device__ __forceinline__ void dft4(float2& a0, float2& a1, float2& a2, float2& a3) {
  const float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = mul_neg_i(csub(a1, a3));
  a0 = cadd(t0, t2);
  a1 = cadd(t1, t3);
  a2 = csub(t0, t2);
  a3 = csub(t1, t3);
}

// V[s] = sum_r v[r] e^{-2 pi i r s / 8}, in place
__device__ __forceinline__ void dft8(float2 (&v)[8]) {
  constexpr float h = 0.70710678118654752f;
  dft4(v[0], v[2], v[4], v[6]);  // even half E[0..3] in v[0], v[2], v[4], v[6]
  dft4(v[1], v[3], v[5], v[7]);  // odd half  O[0..3] in v[1], v[3], v[5], v[7]
  const float2 o0 = v[1];
  const float2 o1 = make_float2(h * (v[3].x + v[3].y), h * (v[3].y - v[3].x));
  const float2 o2 = mul_neg_i(v[5]);
  const float2 o3 = make_float2(h * (v[7].y - v[7].x), -h * (v[7].x + v[7].y));
  const float2 e0 = v[0], e1 = v[2], e2 = v[4], e3 = v[6];
  v[0] = cadd(e0, o0);
  v[1] = cadd(e1, o1);
  v[2] = cadd(e2, o2);
  v[3] = cadd(e3, o3);
  v[4] = csub(e0, o0);
  v[5] = csub(e1, o1);
  v[6] = csub(e2, o2);
  v[7] = csub(e3, o3);
}

__global__ void __launch_bounds__(kThreads)
audio_mel_kernel(const float* __restrict__ audio, long long n, int frames, long long total,
                 const float* __restrict__ window, const float* __restrict__ weights,
                 float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MelSmem& s = *reinterpret_cast<MelSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- tables: twiddles, window, and each mel column's band of non-zero weights
  for (int k = tid; k < kHalf; k += kThreads) {
    double sn, cs;
    sincospi(static_cast<double>(k) / kHalf, &sn, &cs);
    s.tw[k] = make_float2(static_cast<float>(cs), static_cast<float>(-sn));
  }
  for (int i = tid; i < kWin; i += kThreads) s.win[i] = window[i];
  {
    // threads j and j + 128 scan rows [0, 257) and [257, 513) of column j
    const int j = tid & (kMels - 1);
    const int k0 = tid < kMels ? 0 : 257, k1 = tid < kMels ? 257 : kBins;
    int lo = -1, hi = -1;
#pragma unroll 8
    for (int k = k0; k < k1; ++k) {
      if (weights[k * kMels + j] != 0.f) {
        if (lo < 0) lo = k;
        hi = k;
      }
    }
    if (tid >= kMels) {
      s.band_lo[j] = lo;
      s.band_len[j] = hi;
    }
    __syncthreads();
    if (tid < kMels) {
      const int lo2 = s.band_lo[j], hi2 = s.band_len[j];
      const int first = lo >= 0 ? lo : lo2, last = hi2 >= 0 ? hi2 : hi;
      s.band_lo[j] = first < 0 ? 0 : first;
      s.band_len[j] = first < 0 ? 0 : last - first + 1;
    }
    __syncthreads();
    if (tid == 0) {
      int off = 0;
      for (int c = 0; c < kMels; ++c) {
        s.band_off[c] = off;
        off += s.band_len[c];
      }
      s.band_total = off;
    }
    __syncthreads();
    if (s.band_total <= kBandCap && tid < kMels) {
      for (int t = 0; t < s.band_len[j]; ++t)
        s.band_w[s.band_off[j] + t] = weights[(s.band_lo[j] + t) * kMels + j];
    }
    __syncthreads();
  }
  // a table whose bands do not fit is read from global memory instead (same arithmetic)
  const bool packed = s.band_total <= kBandCap;

  float2* buf = s.buf[warp];
  float* mag = reinterpret_cast<float*>(buf);
  const long long stride = static_cast<long long>(gridDim.x) * kWarps;
  for (long long g = static_cast<long long>(blockIdx.x) * kWarps + warp; g < total; g += stride) {
    const long long row = g / frames;
    const long long start = (g - row * frames) * kHop;
    const float* x = audio + row * n + start;
    const long long avail = n - start;  // samples of this frame inside the row (> 0)

    // pass 1 (span 1) straight from global memory: butterfly j takes z[j + 64 r], and
    // z[m] = 0 for m >= 320 (the window is 640 samples, the FFT 1024), i.e. for r >= 5
    float2 v[2][8];
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int j = lane + 32 * b;
#pragma unroll
      for (int r = 0; r < 5; ++r) {
        const int i0 = 2 * (j + 64 * r);
        const float a0 = i0 < avail ? __ldg(x + i0) : 0.f;
        const float a1 = i0 + 1 < avail ? __ldg(x + i0 + 1) : 0.f;
        v[b][r] = make_float2(s.win[i0] * a0, s.win[i0 + 1] * a1);
      }
#pragma unroll
      for (int r = 5; r < 8; ++r) v[b][r] = make_float2(0.f, 0.f);
      dft8(v[b]);
    }
    __syncwarp();  // the previous frame's projection has read mag
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int j = lane + 32 * b;
#pragma unroll
      for (int q = 0; q < 8; ++q) buf[8 * j + q] = v[b][q];
    }
    __syncwarp();

    // passes 2 and 3 (span 8, 64): Stockham, in place through registers
#pragma unroll
    for (int ns = 8; ns < kHalf; ns *= 8) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int j = lane + 32 * b, m = j % ns;
        v[b][0] = buf[j];
#pragma unroll
        for (int r = 1; r < 8; ++r) v[b][r] = cmul(buf[j + 64 * r], w512(s.tw, r * m * (64 / ns)));
        dft8(v[b]);
      }
      __syncwarp();
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int j = lane + 32 * b, m = j % ns;
        const int d = (j / ns) * ns * 8 + m;
#pragma unroll
        for (int q = 0; q < 8; ++q) buf[d + q * ns] = v[b][q];
      }
      __syncwarp();
    }

    // real split: X[k] = (Z[k] + conj Z[512-k]) / 2 - i/2 e^{-2 pi i k / 1024} (Z[k] - conj Z[512-k])
    float mk[17];
#pragma unroll
    for (int i = 0; i < 17; ++i) {
      const int k = lane + 32 * i;
      mk[i] = 0.f;
      if (k <= kHalf) {
        const float2 a = buf[k & (kHalf - 1)];
        const float2 c = buf[(kHalf - k) & (kHalf - 1)];
        const float2 sum = make_float2(a.x + c.x, a.y - c.y);   // Z[k] + conj Z[512-k]
        const float2 dif = make_float2(a.x - c.x, a.y + c.y);   // Z[k] - conj Z[512-k]
        const float2 t = cmul(k < kHalf ? s.tw[k] : make_float2(-1.f, 0.f), dif);
        const float re = 0.5f * sum.x + 0.5f * t.y;
        const float im = 0.5f * sum.y - 0.5f * t.x;
        mk[i] = sqrtf(fmaf(re, re, im * im));
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 17; ++i) {
      const int k = lane + 32 * i;
      if (k <= kHalf) mag[k] = mk[i];
    }
    __syncwarp();

    // mel projection over each column's band, clip, log
    float* o = out + g * kMels;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = lane + 32 * q;
      const int lo = s.band_lo[c], len = s.band_len[c];
      float acc = 0.f;
      if (packed) {
        const float* w = s.band_w + s.band_off[c];
        for (int t = 0; t < len; ++t) acc = fmaf(w[t], mag[lo + t], acc);
      } else {
        for (int t = 0; t < len; ++t) acc = fmaf(__ldg(weights + (lo + t) * kMels + c), mag[lo + t], acc);
      }
      // tf.clip_by_value: NaN stays NaN
      const float m = acc < 1e-5f ? 1e-5f : (acc > 1e8f ? 1e8f : acc);
      o[c] = logf(m);
    }
  }
}

}  // namespace

long long audio_mel_frames(long long n_samples) {
  return n_samples / kHop + (n_samples % kHop != 0);
}

int launch_audio_mel(const float* audio, int rows, long long n_samples, const float* window,
                     const float* weights, float* out, cudaStream_t stream) {
  const long long frames = audio_mel_frames(n_samples);
  const long long total = rows * frames;
  if (total == 0) return 0;
  const int smem = static_cast<int>(sizeof(MelSmem));
  MSD_CUDA_CHECK(cudaFuncSetAttribute(audio_mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem));
  int dev = 0, sms = 0, per_sm = 0;
  MSD_CUDA_CHECK(cudaGetDevice(&dev));
  MSD_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  MSD_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, audio_mel_kernel, kThreads,
                                                               smem));
  MSD_REQUIRE(per_sm > 0, "audio_mel: the kernel does not fit on an SM");
  // one wave of CTAs, each walking frames with a stride: the table set-up is paid once per CTA
  const long long want = (total + kWarps - 1) / kWarps;
  const int grid = static_cast<int>(want < static_cast<long long>(sms) * per_sm ? want
                                                                                : sms * per_sm);
  audio_mel_kernel<<<grid, kThreads, smem, stream>>>(audio, n_samples, static_cast<int>(frames),
                                                     total, window, weights, out);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

}  // namespace msd
