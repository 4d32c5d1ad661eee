"""Times audio_codecs.griffin_lim (mel -> audio by NNLS and fast Griffin-Lim, the
msd_op_griffin_lim_* kernels) on many songs at once.

Workload: --songs songs of --seconds each (default 32 x 180 s: 288,000 frames, one row per song),
features from seeded noise, NNLS at audio_codecs.NNLS_ITERS steps, --iters Griffin-Lim iterations.
Reports, as one JSON line:
  nnls_ms, init_ms, iter_ms, istft_ms   CUDA-event time per op (--reps calls each; iter_ms is per
                                        iteration, from one call of --iters iterations)
  iter_hbm_bound_ms, iter_share_of_hbm  the least time one iteration's traffic allows at the
                                        H100 SXM data-sheet 3.35 TB/s, and that over iter_ms
  iter_fft_bound_ms                     the same for its FFT flops at 67 TFLOP/s fp32
  call_ms                               the whole griffin_lim call from a host numpy array: copy in,
                                        every kernel, copy out (host clock around a call that ends
                                        in a synchronise)
  gpu, power_limit                      read in the same run (nvidia-smi)
Traffic of one iteration per frame: S read (513 f32), angles and tprev read and written
(513 complex f32 each): 18,468 bytes.  FFT work per frame: two 1024-point real FFTs at
2.5 N log2 N flops each.  Halo frames (2 per 16-frame tile) are not counted: they are the
kernel's overhead.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_FP32 = 67e12      # H100 SXM data sheet, fp32 (non-tensor), 700 W
PEAK_HBM = 3.35e12     # H100 SXM data sheet, HBM3 bytes/s


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader', '-i', '0'], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power, clock = [s.strip() for s in out.split(',')]
    return name, power, clock
  except Exception as e:  # pylint: disable=broad-except
    return f'unknown ({e})', 'unknown', 'unknown'


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--songs', type=int, default=32)
  ap.add_argument('--seconds', type=float, default=180.0)
  ap.add_argument('--iters', type=int, default=32)
  ap.add_argument('--reps', type=int, default=3)
  args = ap.parse_args()
  import torch
  from music_spectrogram_diffusion_b200 import audio_codecs, engine
  if not torch.cuda.is_available():
    raise SystemExit('griffin_lim_bench: no CUDA device (the kernels are only timed on the GPU)')
  dev = torch.device('cuda', 0)
  frames = int(args.seconds * 50)
  rng = np.random.default_rng(0)
  host = rng.uniform(np.log(1e-5), 2.0, (args.songs, frames, 128)).astype(np.float32)
  feats = torch.from_numpy(host).to(dev)
  window, weights = audio_codecs.mel_tables(dev)
  pinv, inv_l, beta = audio_codecs.griffin_lim_tables(dev)
  n_nnls = audio_codecs.NNLS_ITERS

  def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
      fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / reps

  mag = engine.op_griffin_lim_magnitude(feats, weights, pinv, inv_l, beta, n_nnls)
  nnls_ms = timed(lambda: engine.op_griffin_lim_magnitude(feats, weights, pinv, inv_l, beta, n_nnls),
                  args.reps)
  init_ms = timed(lambda: engine.op_griffin_lim_init(args.songs, frames, 0, dev), args.reps)
  angles = engine.op_griffin_lim_init(args.songs, frames, 0, dev)
  tprev = torch.zeros_like(angles)
  work = torch.empty_like(angles)
  iter_ms = timed(lambda: engine.op_griffin_lim_iterate(mag, window, angles, tprev, 0.99, args.iters,
                                                        work), 1) / args.iters
  istft_ms = timed(lambda: engine.op_griffin_lim_istft(mag, window, angles), args.reps)
  del work, tprev

  audio_codecs.griffin_lim(host[:1, :10])
  calls = []
  for _ in range(2):
    tick = time.perf_counter()
    audio_codecs.griffin_lim(host, n_iter=args.iters)
    calls.append(time.perf_counter() - tick)

  total = args.songs * frames
  iter_bytes = total * (513 * 4 + 4 * 513 * 8)
  iter_flops = total * 2 * 2.5 * 1024 * 10
  name, power, clock = card()
  print(json.dumps({
      'workload': f'{args.songs} songs x {args.seconds:g} s ({total} frames), NNLS {n_nnls} steps, '
                  f'{args.iters} iterations',
      'nnls_ms': nnls_ms, 'init_ms': init_ms, 'iter_ms': iter_ms, 'istft_ms': istft_ms,
      'iter_hbm_bound_ms': iter_bytes / PEAK_HBM * 1e3,
      'iter_fft_bound_ms': iter_flops / PEAK_FP32 * 1e3,
      'iter_share_of_hbm': iter_bytes / PEAK_HBM * 1e3 / iter_ms,
      'iter_tb_per_s': iter_bytes / (iter_ms / 1e3) / 1e12,
      'kernels_ms': nnls_ms + init_ms + args.iters * iter_ms + istft_ms,
      'call_ms': min(calls) * 1e3,
      'audio_seconds_per_call_second': args.songs * args.seconds / min(calls),
      'gpu': name, 'power_limit': power, 'max_sm_clock': clock,
  }))


if __name__ == '__main__':
  main()
