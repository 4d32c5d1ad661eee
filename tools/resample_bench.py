"""Times resampling to 16 kHz (the kaiser_best kernel, msd_op_audio_resample) on many recordings.

Workload: --songs recordings of --seconds each at every rate in --rates (default 32 x 180 s at
44.1 kHz and at 48 kHz, seeded noise, one row per recording, one launch).  Reports, as one JSON
line per rate and one for the loader:
  outputs_per_s        output samples per second of kernel time (CUDA events, --reps launches)
  kernel_ms            kernel time per launch
  fp64_gop_per_s, tb_per_s   achieved rates from the algorithmic work below over kernel time
  executed_fp64_gop_per_s    the fp64 operations this kernel issues over kernel time (it also
                       scales the window and forms its difference per tap, see below)
  share_of_bound       least time the algorithmic work allows at the binding data-sheet bound
                       (H100 SXM: 34 TFLOP/s fp64 non-tensor, 3.35 TB/s HBM3) over kernel time,
                       and which bound that is
  load_audio_ms        song.load_audio(resample=True) of a --wav-seconds 44.1 kHz stereo 16-bit
                       WAV from bytes: parse, mixdown, copies and kernel (host clock around a
                       call that ends in a copy back to the host)
  gpu, power_limit     read in the same run (nvidia-smi)
Algorithmic work: resampy's loop, counted from the tap counts it takes (both wings): per tap the
interpolated weight (a multiply and an add) and the multiply-add into the float32 accumulator,
4 fp64 operations, over tables resampy builds once per call.  The kernel reads the unscaled
window instead and per tap also scales two entries by the ratio when downsampling and subtracts
them: 7 executed operations per tap (5 when upsampling).  Bytes: the input read once, the
output written once, the window once.
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time
import wave

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_FP64 = 34e12      # H100 SXM data sheet, fp64 (non-tensor), 700 W
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


def taps_per_row(orig_sr, target_sr, n_in, n_out, nwin=32769, num_table=512):
  """Total taps of resampy's loop over one row (both wings), from the time register t / ratio."""
  ratio = float(target_sr) / orig_sr
  scale = min(1.0, ratio)
  step = int(scale * num_table)
  r = np.arange(n_out) / ratio
  n = r.astype(np.int64)
  frac = scale * (r - n)
  left = np.minimum(n + 1, (nwin - (frac * num_table).astype(np.int64)) // step)
  right = np.minimum(n_in - n - 1, (nwin - ((scale - frac) * num_table).astype(np.int64)) // step)
  return int(np.maximum(left, 0).sum() + np.maximum(right, 0).sum())


def stereo_wav(n, rate=44100):
  """A 16-bit stereo PCM WAV of n frames of seeded noise, as bytes."""
  x_int = np.clip(np.random.default_rng(n).normal(0, 0.1, (n, 2)) * 32767, -32768, 32767)
  buf = io.BytesIO()
  with wave.open(buf, 'wb') as w:
    w.setnchannels(2)
    w.setsampwidth(2)
    w.setframerate(rate)
    w.writeframes(x_int.astype('<i2').tobytes())
  return buf.getvalue()


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--songs', type=int, default=32)
  ap.add_argument('--seconds', type=float, default=180.0)
  ap.add_argument('--rates', type=int, nargs='+', default=[44100, 48000])
  ap.add_argument('--reps', type=int, default=10)
  ap.add_argument('--warmup', type=int, default=2)
  ap.add_argument('--wav-seconds', type=float, default=180.0)
  args = ap.parse_args()
  import torch
  from music_spectrogram_diffusion_b200 import audio_codecs, engine, song
  if not torch.cuda.is_available():
    raise SystemExit('resample_bench: no CUDA device (the kernel is only timed on the GPU)')
  dev = torch.device('cuda', 0)
  name, power, clock = card()
  window = audio_codecs.resample_window(dev)
  for rate in args.rates:
    n = int(args.seconds * rate)
    rng = np.random.default_rng(rate)
    audio = torch.from_numpy(rng.standard_normal((args.songs, n), dtype=np.float32) * 0.1).to(dev)
    n_out = audio_codecs.resampy_length(n, rate, 16000)
    segs = torch.from_numpy(audio_codecs.time_register_segments(rate, 16000, n_out)).to(dev)
    run = lambda: engine.op_audio_resample(audio, rate, 16000, window,
                                           audio_codecs.KAISER_BEST_PRECISION, segs)
    for _ in range(args.warmup):
      run()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.reps):
      run()
    stop.record()
    torch.cuda.synchronize()
    kernel_s = start.elapsed_time(stop) / 1e3 / args.reps
    taps = args.songs * taps_per_row(rate, 16000, n, n_out)
    ops = taps * 4
    executed = taps * (7 if rate > 16000 else 5)
    nbytes = audio.numel() * 4 + args.songs * n_out * 4 + window.numel() * 8
    t_op, t_byte = ops / PEAK_FP64, nbytes / PEAK_HBM
    print(json.dumps({
        'workload': f'{args.songs} recordings x {args.seconds:g} s at {rate} Hz -> 16000 Hz '
                    f'(one launch, {args.songs * n_out} outputs)',
        'outputs_per_s': args.songs * n_out / kernel_s,
        'kernel_ms': kernel_s * 1e3,
        'taps_per_output': taps / (args.songs * n_out),
        'fp64_gop_per_s': ops / kernel_s / 1e9,
        'executed_fp64_gop_per_s': executed / kernel_s / 1e9,
        'tb_per_s': nbytes / kernel_s / 1e12,
        'binding_bound': 'fp64' if t_op >= t_byte else 'hbm',
        'share_of_bound': max(t_op, t_byte) / kernel_s,
        'gpu': name, 'power_limit': power, 'max_sm_clock': clock,
    }), flush=True)
    del audio

  data = stereo_wav(int(args.wav_seconds * 44100))
  song.load_audio(stereo_wav(44100), resample=True)
  calls = []
  for _ in range(3):
    tick = time.perf_counter()
    song.load_audio(data, resample=True)
    calls.append(time.perf_counter() - tick)
  print(json.dumps({
      'workload': f'song.load_audio(resample=True): {args.wav_seconds:g} s 44.1 kHz stereo 16-bit WAV',
      'load_audio_ms': min(calls) * 1e3,
      'gpu': name, 'power_limit': power, 'max_sm_clock': clock,
  }), flush=True)


if __name__ == '__main__':
  main()
