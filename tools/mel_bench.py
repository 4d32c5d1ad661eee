"""Times MelGAN.encode (the audio -> log-mel kernel, msd_op_audio_mel) on many songs at once.

Workload: --songs recordings of --seconds each (default 32 x 180 s of seeded noise, one row per
song, one launch).  Reports, as one JSON line:
  frames_per_s         mel frames per second of kernel time (CUDA events, --reps launches)
  kernel_ms            kernel time per launch
  tflops, tb_per_s     achieved rates from the algorithmic work below over kernel time
  share_of_bound       least time allowed by the binding data-sheet bound (H100 SXM: 67 TFLOP/s
                       fp32, 3.35 TB/s HBM3) over kernel time, and which bound that is
  call_ms              the whole MelGAN.encode call from a host numpy array: copy in, kernel,
                       copy out (host clock around a call that ends in a synchronise)
  gpu, power_limit     read in the same run (nvidia-smi)
Algorithmic work per frame: the windowing (640 multiplies), a 1024-point real FFT counted as
2.5 N log2 N, the magnitudes (3 per bin), and 2 per non-zero filterbank weight.  Bytes: the audio
read once, the features written once, and the two tables.
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
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=3)
  args = ap.parse_args()
  import torch
  from music_spectrogram_diffusion_b200 import audio_codecs, engine
  if not torch.cuda.is_available():
    raise SystemExit('mel_bench: no CUDA device (the kernel is only timed on the GPU)')
  dev = torch.device('cuda', 0)
  n = int(args.seconds * 16000)
  rng = np.random.default_rng(0)
  host = (rng.standard_normal((args.songs, n), dtype=np.float32) * 0.1)
  audio = torch.from_numpy(host).to(dev)
  window, weights = audio_codecs.mel_tables(dev)
  frames = args.songs * (-(-n // 320))
  nnz = int((weights != 0).sum().item())
  for _ in range(args.warmup):
    engine.op_audio_mel(audio, window, weights)
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(args.reps):
    engine.op_audio_mel(audio, window, weights)
  stop.record()
  torch.cuda.synchronize()
  kernel_s = start.elapsed_time(stop) / 1e3 / args.reps

  codec = audio_codecs.MelGAN()
  codec.encode(host[:1])
  calls = []
  for _ in range(3):
    tick = time.perf_counter()
    codec.encode(host)
    calls.append(time.perf_counter() - tick)

  flops = frames * (640 + 2.5 * 1024 * 10 + 3 * 513 + 2 * nnz)
  nbytes = audio.numel() * 4 + frames * 128 * 4 + (640 + 513 * 128) * 4
  t_flop, t_byte = flops / PEAK_FP32, nbytes / PEAK_HBM
  name, power, clock = card()
  print(json.dumps({
      'workload': f'{args.songs} songs x {args.seconds:g} s (one launch, {frames} frames)',
      'frames_per_s': frames / kernel_s,
      'kernel_ms': kernel_s * 1e3,
      'tflops': flops / kernel_s / 1e12,
      'tb_per_s': nbytes / kernel_s / 1e12,
      'binding_bound': 'fp32' if t_flop >= t_byte else 'hbm',
      'share_of_bound': max(t_flop, t_byte) / kernel_s,
      'call_ms': min(calls) * 1e3,
      'audio_seconds_per_call_second': args.songs * args.seconds / min(calls),
      'gpu': name, 'power_limit': power, 'max_sm_clock': clock,
  }))


if __name__ == '__main__':
  main()
