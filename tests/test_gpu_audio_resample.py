"""-m gpu: resampling on the CUDA kernel (msd_op_audio_resample) bit for bit against the numpy
oracle of resampy's loop, its argument checks, and recordings at 44.1 kHz through the loader, the
mel encoder and a primed song."""
import ctypes
import io
import wave

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import _native, audio_codecs as A, engine, song
from oracle import resample_oracle as R
from tests.test_gpu_song_batch import _model, _notes, tiny  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

WIN = A.kaiser_best_window()


def _bits(a):
  return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _assert_bitwise(got, want, what):
  got, want = _bits(got), _bits(want)
  assert got.shape == want.shape, what
  bad = np.flatnonzero(got != want)
  assert bad.size == 0, f'{what}: {bad.size} outputs differ, first at {bad[:5]}'


@pytest.mark.parametrize('sr', [44100, 48000, 22050, 32000, 11025, 8000, 96000])
def test_kernel_equals_oracle_bitwise(cuda_device, sr):
  rng = np.random.default_rng(sr)
  for n in (sr + 77, 1001, 100, 7):
    if R.resampy_length(n, sr, 16000) < 1:
      continue
    x = (0.7 * rng.uniform(-1, 1, n)).astype(np.float32)
    got = A.resample(x, sr)
    assert isinstance(got, np.ndarray) and got.dtype == np.float32
    assert got.shape == (R.librosa_length(n, sr, 16000),)
    _assert_bitwise(got, R.librosa_resample(x, sr, 16000, WIN), (sr, n))
  rows = (0.5 * rng.standard_normal((3, 2 * sr + 1))).astype(np.float32)
  got = A.resample(torch.from_numpy(rows).to(cuda_device), sr)
  assert got.is_cuda and got.shape == (3, R.librosa_length(rows.shape[1], sr, 16000))
  _assert_bitwise(got.cpu().numpy(), R.librosa_resample(rows, sr, 16000, WIN), (sr, 'rows'))


def test_upsampling_to_other_targets(cuda_device):
  x = np.random.default_rng(3).uniform(-1, 1, 2001).astype(np.float32)
  for orig, target in ((16000, 44100), (8000, 22050), (44100, 48000), (48000, 44100)):
    _assert_bitwise(A.resample(x, orig, target), R.librosa_resample(x, orig, target, WIN),
                    (orig, target))


def test_ten_minutes_at_44k1_pins_the_time_register(cuda_device):
  """Every output where the running float64 sum and t / ratio land on different input samples,
  plus random windows and both ends, against the oracle."""
  sr, n = 44100, 44100 * 600 + 123
  rng = np.random.default_rng(600)
  envelope = 10.0 ** rng.uniform(-4, 0, n // sr + 1).repeat(sr)[:n]
  x = (envelope * rng.uniform(-1, 1, n)).astype(np.float32)
  got = A.resample(torch.from_numpy(x).to(cuda_device), sr).cpu().numpy()
  n_out = R.resampy_length(n, sr, 16000)
  assert got.shape == (R.librosa_length(n, sr, 16000),)
  assert (got[n_out:] == 0).all()
  r = R.time_register(sr, 16000, n_out)
  t = np.arange(n_out)
  drift = np.flatnonzero(r.astype(np.int64) != (t * (sr / 16000.0)).astype(np.int64))
  assert drift.size > 30000
  starts = rng.integers(0, n_out - 2000, 6)
  pick = np.unique(np.concatenate([drift, *[np.arange(s, s + 2000) for s in starts],
                                   np.arange(2000), np.arange(n_out - 2000, n_out)]))
  _assert_bitwise(got[pick], R.resample_at(x, sr, 16000, WIN, outputs=pick), 'ten minutes')


def test_equal_rates_are_the_identity(cuda_device):
  x = np.random.default_rng(4).uniform(-1, 1, 999).astype(np.float32)
  assert A.resample(x, 16000) is x
  t = torch.from_numpy(x).to(cuda_device)
  assert A.resample(t, 16000) is t


def test_rows_are_independent_and_runs_repeat(cuda_device):
  sr = 44100
  rows = np.random.default_rng(5).normal(0, 0.3, (4, sr + 3)).astype(np.float32)
  dev = torch.from_numpy(rows).to(cuda_device)
  a = A.resample(dev, sr)
  b = A.resample(dev, sr)
  assert torch.equal(a.view(torch.int32), b.view(torch.int32))
  for i in range(4):
    assert torch.equal(a[i].view(torch.int32), A.resample(dev[i], sr).view(torch.int32)), i
  # one row changed: only its output changes
  other = dev.clone()
  other[2] = -other[2]
  c = A.resample(other, sr)
  assert torch.equal(c[[0, 1, 3]], a[[0, 1, 3]]) and not torch.equal(c[2], a[2])


def test_output_past_the_written_samples_is_untouched(cuda_device):
  sr, rows, n = 22050, 3, 5001
  x = torch.randn(rows, n, device=cuda_device)
  win = A.resample_window(cuda_device)
  n_out = R.resampy_length(n, sr, 16000)
  segs = torch.from_numpy(A.time_register_segments(sr, 16000, n_out)).to(cuda_device)
  want = engine.op_audio_resample(x, sr, 16000, win, 9, segs)
  out = torch.full((rows * n_out + 4096,), -12345.0, device=cuda_device)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  assert _native.load().msd_op_audio_resample(p(x), rows, n, sr, 16000, p(win), win.numel(), 9,
                                              p(segs), segs.shape[0], p(out), n_out, None) == 0
  torch.cuda.synchronize()
  assert torch.equal(out[:rows * n_out].view(rows, n_out), want)
  assert (out[rows * n_out:] == -12345.0).all()


def test_wrapper_and_entry_point_refuse_bad_arguments(cuda_device):
  sr, n = 44100, 1000
  win = A.resample_window(cuda_device)
  n_out = R.resampy_length(n, sr, 16000)
  segs = torch.from_numpy(A.time_register_segments(sr, 16000, n_out)).to(cuda_device)
  good = torch.zeros(2, n, device=cuda_device)
  for bad in (good.double(), good[:, ::2], good.cpu(), good[0]):
    with pytest.raises(ValueError):
      engine.op_audio_resample(bad, sr, 16000, win, 9, segs)
  for bad_win in (win.float(), win.cpu(), win[::2], win[None]):
    with pytest.raises(ValueError):
      engine.op_audio_resample(good, sr, 16000, bad_win, 9, segs)
  for bad_segs in (segs.float(), segs.cpu(), segs[:, :2].contiguous(), segs.reshape(-1), segs[:0]):
    with pytest.raises(ValueError):
      engine.op_audio_resample(good, sr, 16000, win, 9, bad_segs)
  for orig, target in ((0, 16000), (sr, -1), (44100.5, 16000)):
    with pytest.raises(ValueError):
      engine.op_audio_resample(good, orig, target, win, 9, segs)
  with pytest.raises(ValueError):
    A.resample(torch.zeros(1000), sr)
  for dtype in (torch.float64, torch.float16, torch.int16):
    with pytest.raises(ValueError, match='float32'):
      A.resample(torch.zeros(1000, dtype=dtype, device=cuda_device), sr)

  lib = _native.load()
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  out = torch.empty(2, n_out, device=cuda_device)

  def call(x=p(good), rows=2, n_in=n, orig=sr, target=16000, w=p(win), wlen=win.numel(),
           precision=9, s=p(segs), nseg=segs.shape[0], y=p(out), ny=n_out):
    return lib.msd_op_audio_resample(x, rows, n_in, orig, target, w, wlen, precision, s, nseg, y,
                                     ny, None)

  assert call() == 0
  torch.cuda.synchronize()
  for kw in (dict(x=None), dict(w=None), dict(s=None), dict(y=None),
             dict(rows=-1), dict(n_in=-5), dict(ny=-1),
             dict(orig=0), dict(target=0), dict(orig=-44100),
             dict(ny=n_out + 1), dict(ny=n_out - 1), dict(orig=48000),
             dict(rows=65536), dict(n_in=1 << 31, ny=R.resampy_length(1 << 31, sr, 16000)),
             dict(precision=-1), dict(precision=25), dict(wlen=1), dict(nseg=0),
             dict(orig=1 << 30, target=1, n_in=1 << 30, ny=1)):
    assert call(**kw) == -1, kw
    assert lib.msd_last_error()
  # nothing to do: no launch, success
  assert call(rows=0) == 0
  assert call(n_in=2, ny=0) == 0
  torch.cuda.synchronize()


def _wav_bytes(x_int, rate, channels):
  buf = io.BytesIO()
  with wave.open(buf, 'wb') as w:
    w.setnchannels(channels)
    w.setsampwidth(2)
    w.setframerate(rate)
    w.writeframes(np.asarray(x_int, '<i2').tobytes())
  return buf.getvalue()


def _stereo_44k1(seconds, seed):
  sr = 44100
  n = int(seconds * sr)
  t = np.arange(n) / sr
  rng = np.random.default_rng(seed)
  left = 0.4 * np.sin(2 * np.pi * 330 * t) + rng.normal(0, 0.05, n)
  right = 0.3 * np.sin(2 * np.pi * 523 * t + 0.5) + rng.normal(0, 0.05, n)
  x_int = np.clip(np.round(np.stack([left, right], 1) * 32767), -32768, 32767).astype(np.int64)
  mono = (x_int / 32768.0).astype(np.float32).mean(axis=1, dtype=np.float32)
  return _wav_bytes(x_int.reshape(-1), sr, 2), mono


def test_load_audio_resamples_a_44k1_stereo_wav(cuda_device):
  data, mono = _stereo_44k1(2.5, 7)
  got = song.load_audio(data, resample=True)
  assert got.dtype == np.float32 and got.shape == (R.librosa_length(len(mono), 44100, 16000),)
  _assert_bitwise(got, R.librosa_resample(mono, 44100, 16000, WIN), 'load_audio')


def test_resampled_recording_encodes_and_primes_a_song(cuda_device, tiny):
  data, mono = _stereo_44k1(6.0, 8)
  audio = song.load_audio(data, resample=True)
  want = R.librosa_resample(mono, 44100, 16000, WIN)
  model = type('M', (), {'audio_codec': A.MelGAN(), 'sequence_length': {'targets': 256}})()
  got = song.encode_song_audio(model, audio)
  ref = song.encode_song_audio(model, want)
  assert got['num_frames'] == ref['num_frames']
  _assert_bitwise(got['full_gt_encoded'], ref['full_gt_encoded'], 'encode_song_audio')
  t5, params = tiny
  m = _model(t5, params, 1)
  notes = _notes(4.0, 60)
  primed = song.synthesize_song(m, notes, seed=3, context_audio=audio)
  assert np.isfinite(primed['full_pred_encoded']).all()
  again = song.synthesize_song(m, notes, seed=3, context_audio=want)
  _assert_bitwise(primed['full_pred_encoded'], again['full_pred_encoded'], 'primed song')
