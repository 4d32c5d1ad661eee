"""Dumps REFERENCE resampling: librosa 0.9's `resample` / `load(sr=16000)` over resampy 0.2.2.

This is the route from "parity unpinned" to pinned for the resampling kernel.  The reference calls
`librosa.resample(samples, sample_rate, 16000)` and `librosa.load(..., sr=16000)` (through
note_seq) with librosa's default res_type 'kaiser_best', which is resampy's band-limited sinc.  On
a machine with librosa 0.9.x and resampy 0.2.2 (the oldest resampy librosa 0.9 accepts), run

    python tests/golden/make_resampy_golden.py

It asserts those versions and writes `tests/golden/resampy_kaiser_best.npz`;
`tests/test_resampy_golden.py` consumes the file whenever it is present and skips otherwise.
librosa and resampy are not installable in the build image (no network), so the file is NOT
committed yet; the script is written against their published 0.9 / 0.2.2 sources, not executed.

What is dumped:
  half_window                resampy's own kaiser_best table (data/kaiser_best.npz), f64 [32769]
  num_table                  the table entries per zero crossing, as resampy's get_filter returns
                             it (sinc_window's num_bits = 2**precision: 512 for kaiser_best, the
                             value resample passes to resample_f as num_table)
  x_<rate>_<name>            seeded float32 inputs at each rate in RATES
  y_<rate>_<name>            librosa.resample(x, rate, 16000) of each (float32)
  wav_<rate>                 a generated 16-bit stereo PCM WAV at each rate (bytes, uint8)
  load_<rate>                librosa.load(that file, sr=16000, mono=True)[0]
"""
import io
import os
import tempfile
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'resampy_kaiser_best.npz')
RATES = (44100, 48000, 22050, 32000, 11025, 8000, 96000)


def inputs(rate):
  """Seeded float32 inputs: noise, a tone sweep, an impulse, and lengths around the filter's
  reach (a short input is shorter than the 64 zero crossings on either side)."""
  rng = np.random.default_rng(rate)
  n = rate + 77
  t = np.arange(n) / rate
  sig = {
      'noise': 0.5 * rng.uniform(-1, 1, n),
      'chirp': 0.8 * np.sin(2 * np.pi * (100 * t + 0.45 * rate * t * t / 2)),
      'short': rng.uniform(-1, 1, 101),
  }
  imp = np.zeros(n)
  imp[n // 3] = 1.0
  sig['impulse'] = imp
  return {k: v.astype(np.float32) for k, v in sig.items()}


def wav(rate, seconds=1.5):
  rng = np.random.default_rng(rate + 1)
  n = int(rate * seconds)
  t = np.arange(n) / rate
  x = np.stack([0.4 * np.sin(2 * np.pi * 330 * t), 0.3 * np.sin(2 * np.pi * 523 * t)], 1)
  x = x + rng.normal(0, 0.05, x.shape)
  x_int = np.clip(np.round(x * 32767), -32768, 32767).astype('<i2')
  buf = io.BytesIO()
  with wave.open(buf, 'wb') as w:
    w.setnchannels(2)
    w.setsampwidth(2)
    w.setframerate(rate)
    w.writeframes(x_int.tobytes())
  return buf.getvalue()


def build(resample, load, half_window, num_table):
  """The arrays written to OUT.  resample(x, rate) -> librosa.resample(x, rate, 16000);
  load(path) -> librosa.load(path, sr=16000, mono=True)[0]; half_window and num_table as
  resampy's get_filter('kaiser_best') returns them.  main() passes librosa's own functions;
  tests/test_resampy_golden.py passes the oracle's to check the file's layout and conventions."""
  num_table = int(num_table)
  assert num_table > 0 and num_table & (num_table - 1) == 0, num_table
  out = {'half_window': np.asarray(half_window, np.float64), 'num_table': np.int64(num_table)}
  for rate in RATES:
    for name, x in inputs(rate).items():
      out[f'x_{rate}_{name}'] = x
      out[f'y_{rate}_{name}'] = np.asarray(resample(x, rate), np.float32)
    data = wav(rate)
    out[f'wav_{rate}'] = np.frombuffer(data, np.uint8)
    with tempfile.TemporaryDirectory() as tmp:
      path = os.path.join(tmp, f'{rate}.wav')
      with open(path, 'wb') as f:
        f.write(data)
      out[f'load_{rate}'] = np.asarray(load(path), np.float32)
  return out


def main():
  import librosa  # pylint: disable=import-outside-toplevel
  import resampy  # pylint: disable=import-outside-toplevel
  assert librosa.__version__.startswith('0.9.'), librosa.__version__
  assert resampy.__version__ == '0.2.2', resampy.__version__
  half_window, num_table, _ = resampy.filters.get_filter('kaiser_best')
  out = build(lambda x, rate: librosa.resample(x, orig_sr=rate, target_sr=16000,
                                               res_type='kaiser_best'),
              lambda path: librosa.load(path, sr=16000, mono=True)[0], half_window, num_table)
  np.savez(OUT, **out)
  print(f'wrote {OUT}: {len(out)} arrays')


if __name__ == '__main__':
  main()
