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
#include "audio_fft.cuh"
#include "common.cuh"
#include "kernels.h"

namespace msd {
namespace {

constexpr int kWin = 640;      // window (frame) length, samples
constexpr int kHop = 320;      // frame step, samples
constexpr int kHalf = 512;     // complex FFT length (1024-point real FFT)
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

__global__ void __launch_bounds__(kThreads)
audio_mel_kernel(const float* __restrict__ audio, long long n, int frames, long long total,
                 const float* __restrict__ window, const float* __restrict__ weights,
                 float* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  MelSmem& s = *reinterpret_cast<MelSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- tables: twiddles, window, and each mel column's band of non-zero weights
  fft_twiddles(s.tw, tid, kThreads);
  for (int i = tid; i < kWin; i += kThreads) s.win[i] = window[i];
  pack_mel_bands(weights, s.band_lo, s.band_len, s.band_off, &s.band_total, s.band_w, kBandCap, tid);
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
    fft512_passes<8>(buf, s.tw, lane);

    // real split (rfft_bin) and magnitudes
    float mk[17];
#pragma unroll
    for (int i = 0; i < 17; ++i) {
      const int k = lane + 32 * i;
      mk[i] = 0.f;
      if (k <= kHalf) {
        const float2 x = rfft_bin(buf, s.tw, k);
        mk[i] = sqrtf(fmaf(x.x, x.x, x.y * x.y));
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
  const int sms = device_sm_count();
  int per_sm = 0;
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
