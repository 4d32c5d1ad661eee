"""numpy restatement of librosa 0.9 `resample(y, orig_sr, target_sr)` with res_type='kaiser_best',
i.e. resampy 0.2.2's `resample` / `resample_f` (preprocessors.py:150-155, 332-333, 518-521 call it
through librosa.resample and librosa.load(sr=16000)).  Test infrastructure only.

Two forms of resampy's loop, which must agree bit for bit:
  resample_loop  a literal scalar transcription (slow: short inputs only);
  resample_at    the same arithmetic vectorised over outputs, for the whole signal or any chosen
                 subset of output indices, so long recordings can be checked at chosen points.
Both take the half window as data (the library's `audio_codecs.kaiser_best_window()` or resampy's
own table), and keep resampy's rounding: y is float32, and every tap is a float64 multiply and add
rounded back to float32, in the loop's order.  The time register is the sequential float64 sum
`time_register`, computed with np.add.accumulate.
"""

from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

PRECISION = 9     # kaiser_best: log2 of resampy's num_table (2^9 = 512 window entries per zero crossing)


def ratio_of(orig_sr: int, target_sr: int) -> float:
  return float(target_sr) / orig_sr


def resampy_length(n: int, orig_sr: int, target_sr: int) -> int:
  return int(n * ratio_of(orig_sr, target_sr))


def librosa_length(n: int, orig_sr: int, target_sr: int) -> int:
  return int(np.ceil(n * ratio_of(orig_sr, target_sr)))


def time_register(orig_sr: int, target_sr: int, n_out: int) -> np.ndarray:
  """resampy's time register for outputs 0 .. n_out - 1: r_0 = 0, r_{t+1} = fl(r_t + 1 / ratio),
  a sequential float64 sum (np.add.accumulate adds left to right)."""
  inc = 1.0 / ratio_of(orig_sr, target_sr)
  steps = np.full(n_out, inc, np.float64)
  steps[:1] = 0.0
  return np.add.accumulate(steps)


def filter_tables(window: np.ndarray, ratio: float) -> Tuple[np.ndarray, np.ndarray]:
  """(interp_win, interp_delta) as resampy builds them: the window times the ratio when
  downsampling, and its np.diff with 0 at the last entry."""
  win = np.array(window, np.float64)
  if ratio < 1:
    win *= ratio
  delta = np.zeros_like(win)
  delta[:-1] = np.diff(win)
  return win, delta


def _check_length(n: int, orig_sr: int, target_sr: int) -> int:
  if orig_sr <= 0 or target_sr <= 0:
    raise ValueError(f'rates must be > 0, got {orig_sr} -> {target_sr}')
  n_out = resampy_length(n, orig_sr, target_sr)
  if n_out < 1:
    raise ValueError(f'input of {n} samples is too short to resample to {target_sr} Hz')
  return n_out


def resample_loop(x: np.ndarray, orig_sr: int, target_sr: int, window: np.ndarray,
                  precision: int = PRECISION) -> np.ndarray:
  """resampy.resample(x, orig_sr, target_sr) of a 1-D float32 signal, line by line as resample_f."""
  x = np.asarray(x, np.float32)
  n_out = _check_length(x.shape[0], orig_sr, target_sr)
  sample_ratio = ratio_of(orig_sr, target_sr)
  interp_win, interp_delta = filter_tables(window, sample_ratio)
  num_table = 2 ** precision
  y = np.zeros(n_out, np.float32)
  scale = min(1.0, sample_ratio)
  time_increment = 1. / sample_ratio
  index_step = int(scale * num_table)
  time_register_ = 0.0
  nwin = interp_win.shape[0]
  n_orig = x.shape[0]
  for t in range(n_out):
    n = int(time_register_)
    frac = scale * (time_register_ - n)
    index_frac = frac * num_table
    offset = int(index_frac)
    eta = index_frac - offset
    i_max = min(n + 1, (nwin - offset) // index_step)
    for i in range(i_max):
      weight = float(interp_win[offset + i * index_step]) + eta * float(
          interp_delta[offset + i * index_step])
      y[t] = np.float32(float(y[t]) + weight * float(x[n - i]))
    frac = scale - frac
    index_frac = frac * num_table
    offset = int(index_frac)
    eta = index_frac - offset
    k_max = min(n_orig - n - 1, (nwin - offset) // index_step)
    for k in range(k_max):
      weight = float(interp_win[offset + k * index_step]) + eta * float(
          interp_delta[offset + k * index_step])
      y[t] = np.float32(float(y[t]) + weight * float(x[n + k + 1]))
    time_register_ += time_increment
  return y


def resample_at(x: np.ndarray, orig_sr: int, target_sr: int, window: np.ndarray,
                outputs: Optional[np.ndarray] = None, precision: int = PRECISION) -> np.ndarray:
  """resampy.resample(x, orig_sr, target_sr)[outputs] of a 1-D float32 signal (all outputs when
  `outputs` is None), vectorised over outputs with resample_f's arithmetic and tap order."""
  x = np.asarray(x, np.float32)
  n_out = _check_length(x.shape[0], orig_sr, target_sr)
  outputs = np.arange(n_out) if outputs is None else np.asarray(outputs, np.int64)
  if outputs.size and (outputs.min() < 0 or outputs.max() >= n_out):
    raise ValueError(f'outputs must lie in [0, {n_out})')
  ratio = ratio_of(orig_sr, target_sr)
  win, delta = filter_tables(window, ratio)
  num_table = 2 ** precision
  scale = min(1.0, ratio)
  step = int(scale * num_table)
  nwin = win.shape[0]
  r = time_register(orig_sr, target_sr, int(outputs.max()) + 1 if outputs.size else 0)[outputs]
  n = r.astype(np.int64)
  frac = scale * (r - n)
  y = np.zeros(outputs.shape, np.float32)
  for side in ('left', 'right'):
    if side == 'right':
      frac = scale - frac
    index_frac = frac * num_table
    offset = index_frac.astype(np.int64)
    eta = index_frac - offset
    if side == 'left':
      count = np.minimum(n + 1, (nwin - offset) // step)
    else:
      count = np.minimum(x.shape[0] - n - 1, (nwin - offset) // step)
    for i in range(int(count.max()) if count.size else 0):
      m = i < count
      j = offset[m] + i * step
      weight = win[j] + eta[m] * delta[j]
      xi = x[n[m] - i] if side == 'left' else x[n[m] + i + 1]
      y[m] = (y[m].astype(np.float64) + weight * xi.astype(np.float64)).astype(np.float32)
  return y


def librosa_resample(x: np.ndarray, orig_sr: int, target_sr: int, window: np.ndarray,
                     precision: int = PRECISION) -> np.ndarray:
  """librosa 0.9 resample(x, orig_sr, target_sr) (res_type='kaiser_best', fix=True, scale=False)
  of [n] or [rows, n] float32: x itself at equal rates, else resampy's output zero-padded at the
  end to ceil(n * ratio).  `precision` is log2 of the window's entries per zero crossing
  (resampy's num_table = 2^precision)."""
  x = np.asarray(x, np.float32)
  if orig_sr == target_sr:
    return x
  rows = x if x.ndim == 2 else x[None]
  n_fix = librosa_length(rows.shape[1], orig_sr, target_sr)
  out = np.zeros((rows.shape[0], n_fix), np.float32)
  for i, row in enumerate(rows):
    y = resample_at(row, orig_sr, target_sr, window, precision=precision)
    out[i, :y.shape[0]] = y
  return out if x.ndim == 2 else out[0]
