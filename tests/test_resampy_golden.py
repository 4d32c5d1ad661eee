"""Consumes tests/golden/resampy_kaiser_best.npz -- librosa 0.9 / resampy 0.2.2 resampling dumped by
tests/golden/make_resampy_golden.py.  Until that file is generated the tests of it skip with that
reason, and parity with librosa stays unpinned (the kernel is checked bit for bit against the
numpy oracle of resampy's loop in tests/test_gpu_audio_resample.py).

The same checks also run on a stand-in written by the generator's own `build()` with the oracle in
place of librosa, so the file's layout and conventions (resampy's `num_table` = 2^precision table
entries per zero crossing) are exercised before the real file exists."""
import importlib.util
import os
import wave

import numpy as np
import pytest

from music_spectrogram_diffusion_b200 import audio_codecs as A
from oracle import resample_oracle as R

HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(HERE, 'golden', 'resampy_kaiser_best.npz')


def _generator():
  spec = importlib.util.spec_from_file_location(
      'make_resampy_golden', os.path.join(HERE, 'golden', 'make_resampy_golden.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def precision_of(golden) -> int:
  """log2 of resampy's num_table: the `precision` the library and the C entry point take."""
  num_table = int(golden['num_table'])
  precision = num_table.bit_length() - 1
  assert num_table == 1 << precision, num_table
  return precision


def _cases(golden):
  for key in sorted(k for k in golden if k.startswith('x_')):
    _, rate, _ = key.split('_', 2)
    yield key, int(rate), golden[key], golden['y_' + key[2:]]


def check_window(golden):
  """The numpy-built window against resampy's shipped table (they may differ in the last bits)."""
  assert precision_of(golden) == A.KAISER_BEST_PRECISION
  assert golden['half_window'].shape == A.kaiser_best_window().shape
  np.testing.assert_allclose(A.kaiser_best_window(), golden['half_window'], rtol=0, atol=1e-15)


def check_oracle(golden):
  """The oracle, given resampy's own table, against librosa bit for bit."""
  precision = precision_of(golden)
  for key, rate, x, want in _cases(golden):
    got = R.librosa_resample(x, rate, 16000, golden['half_window'], precision=precision)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), key


def check_kernel(golden, device):
  """Bit for bit when the library's window equals resampy's table; otherwise within the rounding
  of the window difference, and bit for bit with resampy's table passed to the kernel."""
  import torch
  from music_spectrogram_diffusion_b200 import engine, song
  precision = precision_of(golden)
  same_window = np.array_equal(A.kaiser_best_window(), golden['half_window'])
  win = torch.from_numpy(np.array(golden['half_window'], np.float64)).to(device)
  for key, rate, x, want in _cases(golden):
    got = A.resample(x, rate)
    if same_window:
      assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), key
    else:
      np.testing.assert_allclose(got, want, rtol=0, atol=1e-6, err_msg=key)
    n_out = R.resampy_length(len(x), rate, 16000)
    segs = torch.from_numpy(A.time_register_segments(rate, 16000, n_out)).to(device)
    exact = engine.op_audio_resample(torch.from_numpy(x)[None].to(device), rate, 16000, win,
                                     precision, segs)[0].cpu().numpy()
    assert np.array_equal(exact.view(np.uint32), want[:n_out].view(np.uint32)), key
  for rate in sorted(int(k[4:]) for k in golden if k.startswith('wav_')):
    got = song.load_audio(golden[f'wav_{rate}'].tobytes(), resample=True)
    want = golden[f'load_{rate}']
    assert got.shape == want.shape, rate
    if same_window:
      assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), rate
    else:
      np.testing.assert_allclose(got, want, rtol=0, atol=1e-6, err_msg=str(rate))


@pytest.fixture(scope='module')
def golden():
  if not os.path.exists(PATH):
    pytest.skip('tests/golden/resampy_kaiser_best.npz not generated (needs librosa 0.9 and '
                'resampy 0.2.2: python tests/golden/make_resampy_golden.py)')
  return dict(np.load(PATH))


def _load_16k(path):
  """librosa.load(path, sr=16000, mono=True) restated: 16-bit PCM to float32, channel mean, resample."""
  with wave.open(path, 'rb') as w:
    rate, channels = w.getframerate(), w.getnchannels()
    raw = w.readframes(w.getnframes())
  x = (np.frombuffer(raw, '<i2').astype(np.float32) / 32768.0).reshape(-1, channels)
  return R.librosa_resample(x.mean(axis=1, dtype=np.float32), rate, 16000, A.kaiser_best_window())


@pytest.fixture(scope='module')
def stand_in():
  """The generator's build() with the oracle in place of librosa, and resampy's num_table (512)."""
  win = A.kaiser_best_window()
  return _generator().build(lambda x, rate: R.librosa_resample(x, rate, 16000, win), _load_16k, win,
                            1 << A.KAISER_BEST_PRECISION)


def test_window_matches_resampy(golden):
  check_window(golden)


def test_oracle_with_resampys_window_matches_librosa_bitwise(golden):
  check_oracle(golden)


@pytest.mark.gpu
def test_kernel_matches_librosa(golden, cuda_device):
  check_kernel(golden, cuda_device)


def test_stand_in_file_passes_the_cpu_checks(stand_in, tmp_path):
  assert int(stand_in['num_table']) == 512
  path = tmp_path / 'stand_in.npz'
  np.savez(path, **stand_in)
  loaded = dict(np.load(path))
  check_window(loaded)
  check_oracle(loaded)


@pytest.mark.gpu
def test_stand_in_file_passes_the_kernel_check(stand_in, cuda_device):
  check_kernel(stand_in, cuda_device)
