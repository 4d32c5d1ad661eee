// The codec's 1024-point real FFT, shared by the encoder (audio_mel.cu) and the Griffin-Lim
// decoder (audio_griffin_lim.cu).  The core is a 512-point complex Stockham FFT in three radix-8
// passes over the even/odd-packed samples z[m] = x[2m] + i x[2m+1], run by one warp on a buffer
// in shared memory; the real-split pass turns it into the 513 rfft bins.  The inverse
// (complex-to-real) transform packs the bins into the 512-point spectrum of z and runs it through
// the same forward core by conjugation.  Twiddles are tw[k] = e^{-2 pi i k / 1024}, rounded from
// double (fft_twiddles).
#pragma once

namespace msd {
namespace {

constexpr int kFftHalf = 512;  // complex FFT length (1024-point real FFT)
constexpr int kFftBins = 513;  // rfft bins

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 mul_neg_i(float2 a) { return make_float2(a.y, -a.x); }

// e^{-2 pi i e / 512}, 0 <= e < 512
__device__ __forceinline__ float2 w512(const float2* tw, int e) {
  if (e < kFftHalf / 2) return tw[2 * e];
  const float2 t = tw[2 * e - kFftHalf];
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

// tw[k] = e^{-2 pi i k / 1024}, k < 512, written by the CTA's threads
__device__ __forceinline__ void fft_twiddles(float2* tw, int tid, int nthreads) {
  for (int k = tid; k < kFftHalf; k += nthreads) {
    double sn, cs;
    sincospi(static_cast<double>(k) / kFftHalf, &sn, &cs);
    tw[k] = make_float2(static_cast<float>(cs), static_cast<float>(-sn));
  }
}

// Stockham passes of span ns0, 8 ns0, .. < 512 over buf [512] in place, one warp: with ns0 = 1 the
// whole forward 512-point FFT; with ns0 = 8 the two passes after a first pass done elsewhere.
// Every lane's earlier writes to buf must be visible (__syncwarp) before the call, and are after.
template <int ns0>
__device__ __forceinline__ void fft512_passes(float2* buf, const float2* tw, int lane) {
  float2 v[2][8];
#pragma unroll
  for (int ns = ns0; ns < kFftHalf; ns *= 8) {
#pragma unroll
    for (int b = 0; b < 2; ++b) {
      const int j = lane + 32 * b, m = j % ns;
      v[b][0] = buf[j];
#pragma unroll
      for (int r = 1; r < 8; ++r) v[b][r] = cmul(buf[j + 64 * r], w512(tw, r * m * (64 / ns)));
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
}

// rfft bin k (0 <= k <= 512) of the real signal whose packed 512-point spectrum Z is in buf:
// X[k] = (Z[k] + conj Z[512-k]) / 2 - i/2 e^{-2 pi i k / 1024} (Z[k] - conj Z[512-k])
__device__ __forceinline__ float2 rfft_bin(const float2* buf, const float2* tw, int k) {
  const float2 a = buf[k & (kFftHalf - 1)];
  const float2 c = buf[(kFftHalf - k) & (kFftHalf - 1)];
  const float2 sum = make_float2(a.x + c.x, a.y - c.y);   // Z[k] + conj Z[512-k]
  const float2 dif = make_float2(a.x - c.x, a.y + c.y);   // Z[k] - conj Z[512-k]
  const float2 t = cmul(k < kFftHalf ? tw[k] : make_float2(-1.f, 0.f), dif);
  return make_float2(0.5f * sum.x + 0.5f * t.y, 0.5f * sum.y - 0.5f * t.x);
}

// conj of 2 Z[k], the packed spectrum of irfft(X) times 1024, from the bins a = X[k], b = X[512-k]
// and twk = tw[k] (0 <= k < 512): 2 Z[k] = (a + conj b) + i e^{+2 pi i k / 1024} (a - conj b).
// The imaginary parts of X[0] and X[512] must be zeroed by the caller (irfft ignores them).
__device__ __forceinline__ float2 irfft_pack(float2 a, float2 b, float2 twk) {
  const float2 s = make_float2(a.x + b.x, a.y - b.y);
  const float2 t = cmul(make_float2(a.x - b.x, a.y + b.y), make_float2(twk.x, -twk.y));
  return make_float2(s.x - t.y, -(s.y + t.x));
}

// The mel filterbank W [513, 128] as bands: column j's weights are rows [lo_j, lo_j + len_j) of W
// (first to last non-zero), packed at band_w[off_j ..] when all bands fit in `cap` weights (the
// caller checks *band_total <= cap).  Run by all of a CTA of exactly 256 threads: threads j and
// j + 128 scan rows [0, 257) and [257, 513) of column j.  Ends with the CTA synchronised.
__device__ __forceinline__ void pack_mel_bands(const float* weights, int* band_lo, int* band_len,
                                               int* band_off, int* band_total, float* band_w,
                                               int cap, int tid) {
  constexpr int kMels = 128;
  const int j = tid & (kMels - 1);
  const int k0 = tid < kMels ? 0 : 257, k1 = tid < kMels ? 257 : kFftBins;
  int lo = -1, hi = -1;
#pragma unroll 8
  for (int k = k0; k < k1; ++k) {
    if (weights[k * kMels + j] != 0.f) {
      if (lo < 0) lo = k;
      hi = k;
    }
  }
  if (tid >= kMels) {
    band_lo[j] = lo;
    band_len[j] = hi;
  }
  __syncthreads();
  if (tid < kMels) {
    const int lo2 = band_lo[j], hi2 = band_len[j];
    const int first = lo >= 0 ? lo : lo2, last = hi2 >= 0 ? hi2 : hi;
    band_lo[j] = first < 0 ? 0 : first;
    band_len[j] = first < 0 ? 0 : last - first + 1;
  }
  __syncthreads();
  if (tid == 0) {
    int off = 0;
    for (int c = 0; c < kMels; ++c) {
      band_off[c] = off;
      off += band_len[c];
    }
    *band_total = off;
  }
  __syncthreads();
  if (*band_total <= cap && tid < kMels) {
    for (int t = 0; t < band_len[j]; ++t)
      band_w[band_off[j] + t] = weights[(band_lo[j] + t) * kMels + j];
  }
  __syncthreads();
}

}  // namespace
}  // namespace msd
