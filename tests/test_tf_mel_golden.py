"""Consumes tests/golden/tf_melgan_encode.npz -- MelGAN features produced by running the
reference's TensorFlow `MelGAN.encode` (tests/golden/make_tf_mel_golden.py).  Until that file is
generated every test here skips with that reason, and parity with TF stays unpinned (the kernel is
checked against the fp64 oracle in tests/test_gpu_audio_mel.py)."""
import os

import numpy as np
import pytest

from music_spectrogram_diffusion_b200 import audio_codecs
from oracle import mel_oracle as MO

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'tf_melgan_encode.npz')


@pytest.fixture(scope='module')
def golden():
  if not os.path.exists(PATH):
    pytest.skip('tests/golden/tf_melgan_encode.npz not generated (needs TensorFlow and the '
                'reference: python tests/golden/make_tf_mel_golden.py --reference ...)')
  return dict(np.load(PATH))


def test_tables_match_tf(golden):
  np.testing.assert_allclose(audio_codecs.hann_window(), golden['tf_window'], rtol=0, atol=2e-7)
  np.testing.assert_allclose(audio_codecs.linear_to_mel_weight_matrix(), golden['tf_weights'],
                             rtol=0, atol=2e-6)


@pytest.mark.gpu
def test_encode_matches_tf(golden, cuda_device):
  """Kernel and TF are each within the fp32 error bound of the fp64 oracle, so within twice it of
  each other (linear domain; elements both clip to the floor compare as equal)."""
  codec = audio_codecs.MelGAN()
  win, weights = audio_codecs.hann_window(), audio_codecs.linear_to_mel_weight_matrix()
  for key in sorted(k for k in golden if k.startswith('audio_')):
    x, want = golden[key], golden['mel_' + key[len('audio_'):]]
    got = codec.encode(x)
    assert got.shape == want.shape, key
    if not len(x):
      continue
    bound = MO.error_bound(x, win, weights)
    err = np.abs(np.exp(got.astype(np.float64)) - np.exp(want.astype(np.float64)))
    both_floor = (got <= np.log(np.float32(1e-5)) + 1e-6) & (want <= np.log(np.float32(1e-5)) + 1e-6)
    assert (err[~both_floor] <= 2 * bound[~both_floor]).all(), key
