import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: needs a real H100 (run with -m gpu)')


@pytest.fixture(scope='session')
def native_lib():
  """Build (if stale) and load the C-ABI library; never falls back to CPU."""
  from music_spectrogram_diffusion_b200 import _native
  _native.build()
  return _native.load()


@pytest.fixture(scope='session')
def cuda_device(native_lib):
  import torch
  if not torch.cuda.is_available():
    pytest.fail('test marked gpu but no CUDA device is visible')
  return torch.device('cuda', 0)
