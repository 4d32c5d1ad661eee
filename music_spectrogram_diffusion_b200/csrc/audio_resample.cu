// Band-limited sinc resampling of fp32 audio, as librosa.resample(res_type='kaiser_best') computes
// it (preprocessors.py:150-155, 332-333, 518-521 through librosa 0.9 -> resampy 0.2.2
// `resample_f`): for output t at time register r_t (input samples),
//   n = int(r_t), frac = scale (r_t - n), scale = min(1, ratio)
//   left wing  i < min(n + 1, (nwin - offset) / step):        y += w(offset + i step) x[n - i]
//   right wing k < min(n_in - n - 1, (nwin - offset') / step): y += w(offset' + k step) x[n + k + 1]
// with offset = int(frac * 2^precision), eta its fractional part, step = int(scale * 2^precision)
// and w(j) = win[j] + eta (win[j + 1] - win[j]) (win scaled by ratio when downsampling; the
// difference is 0 at the last entry).  y is float32 and every tap is a float64 multiply and add
// rounded back to float32, in the order above: the kernel spells each operation out
// (__dmul_rn / __dadd_rn / __double2float_rn) so nvcc cannot contract or reorder them, and the
// output is bit for bit the sequential loop's.
//
// The time register is resampy's running float64 sum r_{t+1} = fl(r_t + 1 / ratio), not t / ratio.
// The host describes it as segments (t_s, r_s, d) over which every step adds exactly d
// (`audio_codecs.time_register_segments`), so r_t = r_s + (t - t_s) d exactly and each thread
// finds its own register without a serial pass.
//
// One thread per output sample, consecutive outputs across a warp, one row per grid.y.  Input
// samples and the f64 half window (256 KB for kaiser_best, more than shared memory holds) are
// read through the read-only cache.
#include "common.cuh"
#include "kernels.h"

namespace msd {
namespace {

constexpr int kThreads = 256;

// w(j) = win_s[j] + eta * (win_s[j + 1] - win_s[j]), win_s = win * ratio when downsampling
__device__ __forceinline__ double tap_weight(const double* __restrict__ win, int nwin, int j,
                                             bool scaled, double ratio, double eta) {
  double w0 = __ldg(win + j);
  double delta = 0.0;
  if (scaled) w0 = __dmul_rn(w0, ratio);
  if (j + 1 < nwin) {
    double w1 = __ldg(win + j + 1);
    if (scaled) w1 = __dmul_rn(w1, ratio);
    delta = __dsub_rn(w1, w0);
  }
  return __dadd_rn(w0, __dmul_rn(eta, delta));
}

// y (float32) += weight * x, in float64, rounded back to float32
__device__ __forceinline__ float tap(float acc, double weight, float x) {
  return __double2float_rn(__dadd_rn(static_cast<double>(acc), __dmul_rn(weight, static_cast<double>(x))));
}

__global__ void __launch_bounds__(kThreads)
audio_resample_kernel(const float* __restrict__ x, int n_in, float* __restrict__ y, int n_out,
                      const double* __restrict__ win, int nwin, int num_table, double ratio,
                      const double* __restrict__ seg, int nseg) {
  const long long tt = static_cast<long long>(blockIdx.x) * kThreads + threadIdx.x;
  if (tt >= n_out) return;
  const int t = static_cast<int>(tt);
  const float* xr = x + static_cast<long long>(blockIdx.y) * n_in;

  // time register: the last segment with t_s <= t (t_s of segment 0 is 0)
  int lo = 0, hi = nseg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(seg + 3 * mid) <= static_cast<double>(t)) lo = mid; else hi = mid - 1;
  }
  const double ts = __ldg(seg + 3 * lo), rs = __ldg(seg + 3 * lo + 1), d = __ldg(seg + 3 * lo + 2);
  const double r = __dadd_rn(rs, __dmul_rn(static_cast<double>(t) - ts, d));

  const bool scaled = ratio < 1.0;
  const double scale = scaled ? ratio : 1.0;
  const double table = static_cast<double>(num_table);
  const int step = static_cast<int>(__dmul_rn(scale, table));
  const int n = static_cast<int>(r);
  if (n >= n_in) {  // the register ran past the input (a table the wrapper refuses): never read there
    y[static_cast<long long>(blockIdx.y) * n_out + t] = __int_as_float(0x7fc00000);
    return;
  }
  double frac = __dmul_rn(scale, __dsub_rn(r, static_cast<double>(n)));
  float acc = 0.f;

  {  // left wing: x[n], x[n - 1], ...
    const double index_frac = __dmul_rn(frac, table);
    const int offset = static_cast<int>(index_frac);
    const double eta = __dsub_rn(index_frac, static_cast<double>(offset));
    const int i_max = min(n + 1, (nwin - offset) / step);
    for (int i = 0; i < i_max; ++i)
      acc = tap(acc, tap_weight(win, nwin, offset + i * step, scaled, ratio, eta), __ldg(xr + n - i));
  }
  frac = __dsub_rn(scale, frac);
  {  // right wing: x[n + 1], x[n + 2], ...
    const double index_frac = __dmul_rn(frac, table);
    const int offset = static_cast<int>(index_frac);
    const double eta = __dsub_rn(index_frac, static_cast<double>(offset));
    const int k_max = min(n_in - n - 1, (nwin - offset) / step);
    for (int k = 0; k < k_max; ++k)
      acc = tap(acc, tap_weight(win, nwin, offset + k * step, scaled, ratio, eta),
                __ldg(xr + n + k + 1));
  }
  y[static_cast<long long>(blockIdx.y) * n_out + t] = acc;
}

}  // namespace

int launch_audio_resample(const float* x, int rows, int n_in, double ratio, const double* window,
                          int window_len, int num_table, const double* segments, int n_segments,
                          float* y, int n_out, cudaStream_t stream) {
  if (rows == 0 || n_out == 0) return 0;
  const dim3 grid(static_cast<unsigned>((static_cast<long long>(n_out) + kThreads - 1) / kThreads),
                  static_cast<unsigned>(rows));
  audio_resample_kernel<<<grid, kThreads, 0, stream>>>(x, n_in, y, n_out, window, window_len,
                                                       num_table, ratio, segments, n_segments);
  MSD_CUDA_CHECK(cudaGetLastError());
  ++g_launch_count;
  return 0;
}

}  // namespace msd
