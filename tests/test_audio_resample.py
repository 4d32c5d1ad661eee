"""CPU: the kaiser_best window, resampled lengths, the numpy oracle of resampy's loop (vectorised
against the literal loop), the time-register segments the kernel uses, and the loader at 16 kHz."""
import io
import wave

import numpy as np
import pytest

from music_spectrogram_diffusion_b200 import audio_codecs as A
from music_spectrogram_diffusion_b200 import song
from oracle import resample_oracle as R

RATES = [44100, 48000, 22050, 32000, 11025, 8000, 96000]
WIN = A.kaiser_best_window()


def test_window_shape_peak_and_taper():
  assert WIN.shape == (64 * 512 + 1,) and WIN.dtype == np.float64
  assert not WIN.flags.writeable
  assert WIN[0] == A.KAISER_BEST_ROLLOFF
  assert A.kaiser_best_window() is WIN
  # sinc zeros at multiples of 1 / rolloff zero crossings; the Kaiser taper shrinks each lobe
  lobes = np.abs(WIN).reshape(-1)[:64 * 512].reshape(64, 512).max(axis=1)
  assert (np.diff(lobes) < 0).all()
  assert abs(WIN[-1]) < 1e-7 and lobes[-1] < 1e-6
  # the same window from an independent Kaiser implementation, to fp64 rounding
  signal = pytest.importorskip('scipy.signal')
  n = 64 * 512
  ref = (signal.windows.kaiser(2 * n + 1, A.KAISER_BEST_BETA)[n:] * A.KAISER_BEST_ROLLOFF *
         np.sinc(A.KAISER_BEST_ROLLOFF * np.linspace(0, 64, n + 1)))
  np.testing.assert_allclose(WIN, ref, rtol=0, atol=1e-14)


@pytest.mark.parametrize('sr', RATES)
def test_lengths(sr):
  for n in (1, 2, 3, 100, 4410, 44100, 44101, 1234567):
    ratio = 16000.0 / sr
    assert A.resampy_length(n, sr, 16000) == R.resampy_length(n, sr, 16000) == int(n * ratio)
    assert A.librosa_length(n, sr, 16000) == R.librosa_length(n, sr, 16000) == int(np.ceil(n * ratio))
  assert A.resampy_length(44100, 44100, 16000) == A.librosa_length(44100, 44100, 16000) == 16000
  assert A.resampy_length(100, 44100, 16000) == 36 and A.librosa_length(100, 44100, 16000) == 37


def test_too_short_and_bad_rates_raise_before_any_launch():
  for n in (0, 1, 2):
    with pytest.raises(ValueError, match='short'):
      R.resample_at(np.zeros(n, np.float32), 44100, 16000, WIN)
  with pytest.raises(ValueError, match='no output'):
    A.resample(np.zeros(2, np.float32), 44100)
  for orig, target in ((0, 16000), (-44100, 16000), (44100, 0), (44100.5, 16000)):
    with pytest.raises(ValueError, match='rates'):
      A.resample(np.zeros(100, np.float32), orig, target)
  with pytest.raises(ValueError, match=r'\[n\]'):
    A.resample(np.zeros((2, 2, 100), np.float32), 44100)
  # librosa keeps float64 in float64: rounding it to float32 first would not be librosa's result
  for dtype in (np.float64, np.int16, np.float16):
    with pytest.raises(ValueError, match='float32'):
      A.resample(np.zeros(1000, dtype), 44100)


def test_equal_rates_return_the_input():
  x = np.random.default_rng(0).uniform(-1, 1, 1000).astype(np.float32)
  assert A.resample(x, 16000) is x
  assert R.librosa_resample(x, 16000, 16000, WIN) is x


@pytest.mark.parametrize('sr', RATES)
def test_vectorised_oracle_equals_the_literal_loop_bitwise(sr):
  rng = np.random.default_rng(sr)
  for n in (3, 100, 1501):   # 100 at 44.1 kHz: every output is shorter than the filter's reach
    if R.resampy_length(n, sr, 16000) < 1:
      continue
    x = rng.uniform(-1, 1, n).astype(np.float32)
    want = R.resample_loop(x, sr, 16000, WIN)
    got = R.resample_at(x, sr, 16000, WIN)
    assert got.dtype == np.float32 and got.shape == (R.resampy_length(n, sr, 16000),)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (sr, n)
    sub = np.array([0, len(want) // 3, len(want) - 1])
    assert np.array_equal(R.resample_at(x, sr, 16000, WIN, outputs=sub).view(np.uint32),
                          want[sub].view(np.uint32))


def test_librosa_resample_pads_rows_to_ceil():
  x = np.random.default_rng(1).uniform(-1, 1, (2, 1001)).astype(np.float32)
  y = R.librosa_resample(x, 44100, 16000, WIN)
  n_out, n_fix = R.resampy_length(1001, 44100, 16000), R.librosa_length(1001, 44100, 16000)
  assert y.shape == (2, n_fix) and n_fix == n_out + 1
  assert (y[:, n_out:] == 0).all()
  for r in range(2):
    assert np.array_equal(y[r, :n_out], R.resample_at(x[r], 44100, 16000, WIN))


@pytest.mark.parametrize('sr', RATES + [44056, 12345, 37800, 16000])
def test_time_register_segments_equal_the_running_sum_bitwise(sr):
  """Ten minutes of output: r_s + (t - t_s) d of the segments is resampy's sequential sum."""
  n_out = 16000 * 600
  segs = A.time_register_segments(sr, 16000, n_out)
  assert segs.dtype == np.float64 and segs.shape[1] == 3 and len(segs) < 100
  assert segs[0, 0] == 0 and (np.diff(segs[:, 0]) > 0).all()
  ends = np.append(segs[1:, 0], n_out).astype(np.int64)
  full = np.concatenate([r + np.arange(e - int(t)) * d for (t, r, d), e in zip(segs, ends)])
  want = R.time_register(sr, 16000, n_out)
  assert np.array_equal(full.view(np.int64), want.view(np.int64)), sr


def test_time_register_drift_is_what_the_segments_must_reproduce():
  """The running sum is not t / ratio: at 44.1 kHz 35,805 of 9.6 M outputs land on another input
  sample; dyadic increments (48 kHz) do not drift."""
  n_out = 16000 * 600
  t = np.arange(n_out)
  for sr, differ in ((44100, 35805), (48000, 0)):
    r = R.time_register(sr, 16000, n_out)
    assert int((r.astype(np.int64) != (t * (sr / 16000.0)).astype(np.int64)).sum()) == differ


def _level_db(f, sr=44100):
  t = np.arange(sr // 2) / sr
  x = (0.5 * np.sin(2 * np.pi * f * t)).astype(np.float32)
  y = R.resample_at(x, sr, 16000, WIN).astype(np.float64)[1000:-1000]
  return 20 * np.log10(np.sqrt(np.mean(y * y)) / (0.5 / np.sqrt(2)))


def test_passband_and_stopband_of_the_filter():
  for f in (1000, 7000):
    assert abs(_level_db(f)) < 0.05, f
  for f in (8400, 9000):
    assert _level_db(f) < -58, f


def _wav(samples, rate, channels=1):
  buf = io.BytesIO()
  with wave.open(buf, 'wb') as w:
    w.setnchannels(channels)
    w.setsampwidth(2)
    w.setframerate(rate)
    w.writeframes(np.asarray(samples, '<i2').tobytes())
  return buf.getvalue()


def test_load_audio_at_16k_is_unchanged_with_resample():
  x = np.random.default_rng(2).integers(-32768, 32768, 2 * 777).astype(np.int64)
  data = _wav(x, 16000, channels=2)
  plain = song.load_audio(data)
  got = song.load_audio(data, resample=True)
  assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), plain.view(np.uint32))
  with pytest.raises(ValueError, match='resample=True'):
    song.load_audio(_wav(x, 44100))
