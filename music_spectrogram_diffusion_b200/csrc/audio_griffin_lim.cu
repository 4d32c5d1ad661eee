// MelGAN log-mel features -> audio without the vocoder: the codec's own transform (audio_mel.cu)
// inverted by band-sparse NNLS and fast Griffin-Lim (Perraudin, Balazs and Sondergaard 2013, as
// librosa.griffinlim orders it).  Four kernels, all fp32:
//   gl_nnls_kernel         M = exp(features) -> S = argmin_{S >= 0} |S W - M|^2 by a fixed number of
//                          FISTA steps from max(0, M P), P = pinv(W); one warp per frame, every
//                          step in shared memory
//   gl_phase_init_kernel   angles = e^{2 pi i u}, u uniform from Philox4x32-10 (librosa's
//                          init='random')
//   gl_tile_kernel<false>  one fast Griffin-Lim iteration: rebuilt = STFT(ISTFT(S angles)),
//                          a = rebuilt - momentum / (1 + momentum) tprev, tprev = rebuilt,
//                          angles = a / (|a| + 1e-16)
//   gl_tile_kernel<true>   audio = ISTFT(S angles)
// The transform: frame k is samples [320 k, 320 k + 640) of a signal of 320 F samples (zero past
// the end), times the periodic Hann window, zero-padded to 1024, rfft.  Its least-squares inverse
// is y[n] = sum_k w[n - 320 k] irfft(X_k)[n - 320 k] / sum_k w^2[n - 320 k], summed frame k - 1
// then frame k, with the unnormalised sum (0) where sum_k w^2 <= 1e-10 (sample 0 only).
//
// The iteration and ISTFT kernels give each CTA a tile of kTile consecutive frames of one row: it
// inverse-transforms them with one halo frame on each side, overlap-adds the tile's samples in
// shared memory and (iteration) forward-transforms its frames.  Every frame is transformed by one
// warp through the same instructions wherever it sits, so a frame's result depends on its own and
// its neighbours' inputs only, never on the tiling, the grid or the number of rows.
#include "audio_fft.cuh"
#include "common.cuh"
#include "kernels.h"
#include "philox.cuh"

namespace msd {
namespace {

constexpr int kWin = 640;       // window (frame) length, samples
constexpr int kHop = 320;       // frame step, samples
constexpr int kMels = 128;
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kBandCap = 2048;  // packed band weights held in shared memory (MelGAN's: 1012)
constexpr int kTile = 16;       // frames per CTA of the iteration and ISTFT kernels
constexpr uint32_t kPhaseTag = 0x676c70u;  // Philox counter word 3 of the phase stream ("glp")

__device__ __forceinline__ float relu_nan(float v) { return v < 0.f ? 0.f : v; }  // NaN stays NaN

// ---------------------------------------------------------------------------------------------
// NNLS: Z_0 = Y_0 = max(0, M P); Z_{j+1} = max(0, Y_j - (Y_j W - M) W^T / L);
//       Y_{j+1} = Z_{j+1} + beta_j (Z_{j+1} - Z_j); S = Z_n.
// ---------------------------------------------------------------------------------------------
struct NnlsSmem {
  int band_lo[kMels];           // column c's weights: rows [lo, lo + len) of W ...
  int band_len[kMels];
  int band_off[kMels];          // ... packed at band_w[off ..]
  int band_total;
  float band_w[kBandCap];
  int bin_off[kFftBins + 1];    // bin k's covering columns: entries [bin_off[k], bin_off[k + 1]) ...
  int bin_col[kBandCap];        // ... column index and weight, ascending in column
  float bin_w[kBandCap];
  float y[kWarps][kFftBins + 3];  // per warp: Y_j
  float m[kWarps][kMels];         // M
  float r[kWarps][kMels];         // Y_j W - M
};

__global__ void __launch_bounds__(kThreads)
gl_nnls_kernel(const float* __restrict__ feat, long long total, const float* __restrict__ weights,
               const float* __restrict__ pinv, float inv_l, const float* __restrict__ beta,
               int n_iter, float* __restrict__ mag) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NnlsSmem& s = *reinterpret_cast<NnlsSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  pack_mel_bands(weights, s.band_lo, s.band_len, s.band_off, &s.band_total, s.band_w, kBandCap, tid);
  // a filterbank whose bands do not fit gives NaN (documented in msd_b200.h)
  const bool packed = s.band_total <= kBandCap;
  if (packed) {
    // the transpose: bin k is covered by the columns whose band holds it
    for (int k = tid; k < kFftBins; k += kThreads) {
      int cnt = 0;
      for (int c = 0; c < kMels; ++c) cnt += k >= s.band_lo[c] && k < s.band_lo[c] + s.band_len[c];
      s.bin_off[k + 1] = cnt;
    }
    __syncthreads();
    if (tid == 0) {
      s.bin_off[0] = 0;
      for (int k = 0; k < kFftBins; ++k) s.bin_off[k + 1] += s.bin_off[k];
    }
    __syncthreads();
    for (int k = tid; k < kFftBins; k += kThreads) {
      int e = s.bin_off[k];
      for (int c = 0; c < kMels; ++c) {
        const int t = k - s.band_lo[c];
        if (t >= 0 && t < s.band_len[c]) {
          s.bin_col[e] = c;
          s.bin_w[e] = s.band_w[s.band_off[c] + t];
          ++e;
        }
      }
    }
    __syncthreads();
  }

  float* y = s.y[warp];
  float* m = s.m[warp];
  float* r = s.r[warp];
  const long long stride = static_cast<long long>(gridDim.x) * kWarps;
  for (long long g = static_cast<long long>(blockIdx.x) * kWarps + warp; g < total; g += stride) {
    float* out = mag + g * kFftBins;
    if (!packed) {
      for (int k = lane; k < kFftBins; k += 32) out[k] = __int_as_float(0x7fc00000);
      continue;
    }
    const float* f = feat + g * kMels;
    __syncwarp();  // the previous frame is done with m and y
#pragma unroll
    for (int q = 0; q < 4; ++q) m[lane + 32 * q] = expf(f[lane + 32 * q]);
    __syncwarp();

    // Z_0 = Y_0 = max(0, M P): lane owns bins lane + 32 i
    float z[17];
#pragma unroll
    for (int i = 0; i < 17; ++i) z[i] = 0.f;
    for (int j = 0; j < kMels; ++j) {
      const float mj = m[j];
      const float* p = pinv + j * kFftBins;
#pragma unroll
      for (int i = 0; i < 17; ++i) {
        const int k = lane + 32 * i;
        if (k < kFftBins) z[i] = fmaf(mj, __ldg(p + k), z[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 17; ++i) {
      const int k = lane + 32 * i;
      z[i] = relu_nan(z[i]);
      if (k < kFftBins) y[k] = z[i];
    }
    __syncwarp();

    for (int it = 0; it < n_iter; ++it) {
      // R = Y W - M over each column's band
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = lane + 32 * q;
        const float* w = s.band_w + s.band_off[c];
        const float* yb = y + s.band_lo[c];
        const int len = s.band_len[c];
        float acc = 0.f;
        for (int t = 0; t < len; ++t) acc = fmaf(w[t], yb[t], acc);
        r[c] = acc - m[c];
      }
      __syncwarp();
      // G = R W^T over the columns covering each bin; the projected step and the momentum
      const float b = __ldg(beta + it);
#pragma unroll
      for (int i = 0; i < 17; ++i) {
        const int k = lane + 32 * i;
        if (k < kFftBins) {
          float gk = 0.f;
          for (int e = s.bin_off[k]; e < s.bin_off[k + 1]; ++e) gk = fmaf(s.bin_w[e], r[s.bin_col[e]], gk);
          const float zn = relu_nan(fmaf(-gk, inv_l, y[k]));
          y[k] = fmaf(b, zn - z[i], zn);
          z[i] = zn;
        }
      }
      __syncwarp();
    }
#pragma unroll
    for (int i = 0; i < 17; ++i) {
      const int k = lane + 32 * i;
      if (k < kFftBins) out[k] = z[i];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Phase initialisation: element e = frame * 513 + bin of a row takes word e % 4 of
// Philox4x32-10(counter (e / 4 low, e / 4 high, 0, kPhaseTag), key seed); u = (r + 0.5) 2^-32,
// angles[e] = (cos 2 pi u, sin 2 pi u).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
gl_phase_init_kernel(long long per_row, long long quads_per_row, long long total_quads,
                     unsigned long long seed, float2* __restrict__ angles) {
  const long long stride = static_cast<long long>(gridDim.x) * kThreads;
  for (long long q = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x; q < total_quads;
       q += stride) {
    const long long row = q / quads_per_row;
    const long long e4 = q - row * quads_per_row;
    uint32_t r[4];
    philox4x32_10(static_cast<uint32_t>(e4), static_cast<uint32_t>(e4 >> 32), 0u, kPhaseTag,
                  static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), r);
    float2* a = angles + row * per_row;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long e = 4 * e4 + j;
      if (e < per_row) {
        const float u = (static_cast<float>(r[j]) + 0.5f) * 2.3283064365386963e-10f;  // 2^-32
        float sn, cs;
        sincospif(2.0f * u, &sn, &cs);
        a[e] = make_float2(cs, sn);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// ISTFT (and, for the iteration, STFT and the momentum update) over a tile of frames
// ---------------------------------------------------------------------------------------------
struct GlSmem {
  float2 tw[kFftHalf];
  float win[kWin];
  float seg[kTile + 2][kWin];      // windowed irfft of frames k0 - 1 .. k0 + kTile
  float y[(kTile + 1) * kHop];     // the signal over samples [320 k0, 320 (k0 + kTile + 1))
  float2 buf[kWarps][kFftHalf];    // per warp: the FFT in place
};

// kFinal: write audio = ISTFT(S angles) for the tile's kTile hops.  Otherwise one iteration:
// angles_out, tprev (in place) for the tile's frames from angles_in and tprev.
template <bool kFinal>
__global__ void __launch_bounds__(kThreads)
gl_tile_kernel(const float* __restrict__ mag, const float2* __restrict__ angles_in, int frames,
               long long tiles_per_row, const float* __restrict__ window, float coef,
               float2* __restrict__ angles_out, float2* __restrict__ tprev,
               float* __restrict__ audio) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  GlSmem& s = *reinterpret_cast<GlSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long tile = blockIdx.x;
  const long long row = tile / tiles_per_row;
  const long long k0 = (tile - row * tiles_per_row) * kTile;
  const long long row_frame = row * frames;

  fft_twiddles(s.tw, tid, kThreads);
  for (int i = tid; i < kWin; i += kThreads) s.win[i] = window[i];
  __syncthreads();

  // 1. frames k0 - 1 + lf: X = S angles -> irfft -> first 640 samples times the window
  float2* buf = s.buf[warp];
  const int nseg = kFinal ? kTile + 1 : kTile + 2;
  for (int lf = warp; lf < nseg; lf += kWarps) {
    const long long k = k0 - 1 + lf;
    if (k < 0 || k >= frames) continue;
    const float* sk = mag + (row_frame + k) * kFftBins;
    const float2* ak = angles_in + (row_frame + k) * kFftBins;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int kb = lane + 32 * i;  // bins kb and 512 - kb, kb <= 256
      if (kb <= kFftHalf / 2) {
        const float sa = sk[kb], sb = sk[kFftHalf - kb];
        const float2 ua = ak[kb], ub = ak[kFftHalf - kb];
        float2 a = make_float2(sa * ua.x, sa * ua.y), b = make_float2(sb * ub.x, sb * ub.y);
        if (kb == 0) a.y = b.y = 0.f;  // irfft ignores the imaginary parts of DC and Nyquist
        buf[kb] = irfft_pack(a, b, s.tw[kb]);
        if (kb != 0 && kb != kFftHalf / 2) buf[kFftHalf - kb] = irfft_pack(b, a, s.tw[kFftHalf - kb]);
      }
    }
    __syncwarp();
    fft512_passes<1>(buf, s.tw, lane);
    // irfft(X)[2m] = F[m].x / 1024, irfft(X)[2m + 1] = -F[m].y / 1024, F = FFT(conj 2Z)
    float* sg = s.seg[lf];
    for (int mm = lane; mm < kWin / 2; mm += 32) {
      const float2 v = buf[mm];
      sg[2 * mm] = s.win[2 * mm] * (v.x * (1.f / 1024.f));
      sg[2 * mm + 1] = s.win[2 * mm + 1] * (-v.y * (1.f / 1024.f));
    }
    __syncwarp();  // the next frame overwrites buf
  }
  __syncthreads();

  // 2. overlap-add: hop h = k0 + lh is frame h - 1's second half, then frame h's first half,
  // normalised by the same sum of squared window values
  const int nhop = kFinal ? kTile : kTile + 1;
  for (int i = tid; i < nhop * kHop; i += kThreads) {
    const int lh = i / kHop, a = i - lh * kHop;
    const long long h = k0 + lh;
    if (h >= frames) {
      if (!kFinal) s.y[i] = 0.f;
      continue;
    }
    float num = 0.f, den = 0.f;
    if (h >= 1) {
      const float w = s.win[kHop + a];
      num = s.seg[lh][kHop + a];
      den = w * w;
    }
    const float w = s.win[a];
    num += s.seg[lh + 1][a];
    den = fmaf(w, w, den);
    const float v = den > 1e-10f ? num / den : num;
    if (kFinal) {
      audio[row_frame * kHop + h * kHop + a] = v;
    } else {
      s.y[i] = v;
    }
  }
  if (kFinal) return;
  __syncthreads();

  // 3. STFT of the tile's frames and the fast Griffin-Lim update
  for (int lf = warp; lf < kTile; lf += kWarps) {
    const long long k = k0 + lf;
    if (k >= frames) break;
    const float* yk = s.y + lf * kHop;
    for (int mm = lane; mm < kFftHalf; mm += 32) {
      buf[mm] = mm < kWin / 2 ? make_float2(s.win[2 * mm] * yk[2 * mm], s.win[2 * mm + 1] * yk[2 * mm + 1])
                              : make_float2(0.f, 0.f);
    }
    __syncwarp();
    fft512_passes<1>(buf, s.tw, lane);
    const long long base = (row_frame + k) * kFftBins;
#pragma unroll
    for (int i = 0; i < 17; ++i) {
      const int kb = lane + 32 * i;
      if (kb < kFftBins) {
        const float2 rebuilt = rfft_bin(buf, s.tw, kb);
        const float2 tp = tprev[base + kb];
        const float2 a = make_float2(rebuilt.x - coef * tp.x, rebuilt.y - coef * tp.y);
        const float d = sqrtf(fmaf(a.x, a.x, a.y * a.y)) + 1e-16f;
        angles_out[base + kb] = make_float2(a.x / d, a.y / d);
        tprev[base + kb] = rebuilt;
      }
    }
    __syncwarp();  // the next frame overwrites buf
  }
}

template <typename Kernel>
int launch_tiles(Kernel kernel, long long grid, const float* mag, const float2* angles_in,
                 long long frames, const float* window, float coef, float2* angles_out,
                 float2* tprev, float* audio, cudaStream_t stream) {
  const int smem = static_cast<int>(sizeof(GlSmem));
  MSD_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long tiles = (frames + kTile - 1) / kTile;
  kernel<<<static_cast<unsigned>(grid), kThreads, smem, stream>>>(
      mag, angles_in, static_cast<int>(frames), tiles, window, coef, angles_out, tprev, audio);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

}  // namespace

int launch_gl_nnls(const float* features, long long total, const float* weights, const float* pinv,
                   float inv_l, const float* beta, int n_iter, float* mag, cudaStream_t stream) {
  if (total == 0) return 0;
  const int smem = static_cast<int>(sizeof(NnlsSmem));
  MSD_CUDA_CHECK(cudaFuncSetAttribute(gl_nnls_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      smem));
  int per_sm = 0;
  MSD_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gl_nnls_kernel, kThreads,
                                                               smem));
  MSD_REQUIRE(per_sm > 0, "griffin_lim nnls: the kernel does not fit on an SM");
  // one wave of CTAs, each walking frames with a stride: the table set-up is paid once per CTA
  const long long want = (total + kWarps - 1) / kWarps;
  const long long cap = static_cast<long long>(device_sm_count()) * per_sm;
  gl_nnls_kernel<<<static_cast<unsigned>(want < cap ? want : cap), kThreads, smem, stream>>>(
      features, total, weights, pinv, inv_l, beta, n_iter, mag);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

int launch_gl_phase_init(int rows, long long frames, unsigned long long seed, float2* angles,
                         cudaStream_t stream) {
  const long long per_row = frames * kFftBins;
  const long long quads = (per_row + 3) / 4;
  const long long total = rows * quads;
  if (total == 0) return 0;
  const long long want = (total + kThreads - 1) / kThreads;
  const long long cap = static_cast<long long>(device_sm_count()) * 16;
  gl_phase_init_kernel<<<static_cast<unsigned>(want < cap ? want : cap), kThreads, 0, stream>>>(
      per_row, quads, total, seed, angles);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

int launch_gl_iterate(const float* mag, int rows, long long frames, const float* window,
                      float2* angles, float2* tprev, float2* work, float momentum, int n_iter,
                      cudaStream_t stream) {
  const long long grid = rows * ((frames + kTile - 1) / kTile);
  if (grid == 0 || n_iter == 0) return 0;
  // librosa: rebuilt - (momentum / (1 + momentum)) * tprev, the coefficient rounded to f32 once
  const float coef = static_cast<float>(static_cast<double>(momentum) / (1.0 + momentum));
  // a CTA reads its neighbours' angles: each iteration writes the other buffer
  float2* src = angles;
  float2* dst = work;
  for (int it = 0; it < n_iter; ++it) {
    if (int rc = launch_tiles(gl_tile_kernel<false>, grid, mag, src, frames, window, coef, dst,
                              tprev, nullptr, stream))
      return rc;
    float2* t = src;
    src = dst;
    dst = t;
  }
  if (src != angles) {
    MSD_CUDA_CHECK(cudaMemcpyAsync(angles, src, static_cast<size_t>(rows * frames) * kFftBins *
                                                    sizeof(float2),
                                   cudaMemcpyDeviceToDevice, stream));
  }
  return 0;
}

int launch_gl_istft(const float* mag, const float2* angles, int rows, long long frames,
                    const float* window, float* audio, cudaStream_t stream) {
  const long long grid = rows * ((frames + kTile - 1) / kTile);
  if (grid == 0) return 0;
  return launch_tiles(gl_tile_kernel<true>, grid, mag, angles, frames, window, 0.f, nullptr,
                      nullptr, audio, stream);
}

}  // namespace msd
