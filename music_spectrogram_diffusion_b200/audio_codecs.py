"""Codec constants, feature scaling, and audio -> mel encoding.

Mirrors `AudioCodec.scale_features / scale_to_features` (msd/audio_codecs.py:166-183) and the
MelGAN constants (204-218).  `MelGAN.encode` is the reference's Audio2Mel (43-143) with MelGAN's
settings (226-247), computed by the library's CUDA kernel (`engine.op_audio_mel`) from the float32
tables built here (`hann_window`, `linear_to_mel_weight_matrix`, in TF's order of operations).
The vocoder (`decode`, a TF-Hub SavedModel, 249-264) is out of scope: it raises.
"""

from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

MEL_WIN_LENGTH = 640    # MelGAN._frame_length
MEL_FFT_SIZE = 1024     # MelGAN._fft_size


def hann_window(length: int = MEL_WIN_LENGTH) -> np.ndarray:
  """tf.signal.hann_window(length, periodic=True) in float32: 0.5 - 0.5 cos(2 pi i / length),
  with TF's float32 operation order."""
  n = np.float32(length + (1 - length % 2) - 1)
  count = np.arange(length, dtype=np.float32)
  cos_arg = np.float32(2 * np.pi) * count / n
  return (np.float32(0.5) - np.float32(0.5) * np.cos(cos_arg)).astype(np.float32)


def _linspace_f32(start, stop, num: int) -> np.ndarray:
  """tf.linspace in float32: start + i * delta, the last element exactly stop."""
  start, stop = np.float32(start), np.float32(stop)
  delta = (stop - start) / np.float32(num - 1)
  mid = start + np.arange(1, num - 1, dtype=np.float32) * delta
  return np.concatenate([[start], mid, [stop]]).astype(np.float32)


def _hertz_to_mel_f32(hz):
  return np.float32(1127.0) * np.log(np.float32(1.0) + np.asarray(hz, np.float32) / np.float32(700.0))


def linear_to_mel_weight_matrix(num_mel_bins: int = 128, num_spectrogram_bins: int = 513,
                                sample_rate: int = 16000, lower_edge_hertz: float = 0.0,
                                upper_edge_hertz: float = 8000.0) -> np.ndarray:
  """tf.signal.linear_to_mel_weight_matrix in float32 (HTK mel scale, DC row zero):
  f32 [num_spectrogram_bins, num_mel_bins]."""
  nyquist = np.float32(sample_rate) / np.float32(2.0)
  freqs = _linspace_f32(0.0, nyquist, num_spectrogram_bins)[1:]
  bins_mel = _hertz_to_mel_f32(freqs)[:, None]
  edges = _linspace_f32(_hertz_to_mel_f32(lower_edge_hertz), _hertz_to_mel_f32(upper_edge_hertz),
                        num_mel_bins + 2)
  lower, center, upper = edges[None, :-2], edges[None, 1:-1], edges[None, 2:]
  lower_slopes = (bins_mel - lower) / (center - lower)
  upper_slopes = (upper - bins_mel) / (upper - center)
  w = np.maximum(np.float32(0.0), np.minimum(lower_slopes, upper_slopes))
  return np.pad(w, [[1, 0], [0, 0]]).astype(np.float32)


_DEVICE_TABLES: Dict[object, Tuple[object, object]] = {}


def mel_tables(device):
  """(window f32 [640], weights f32 [513, 128]) of MelGAN on `device`, built once per device."""
  if device not in _DEVICE_TABLES:
    import torch
    _DEVICE_TABLES[device] = (
        torch.from_numpy(hann_window()).to(device),
        torch.from_numpy(linear_to_mel_weight_matrix(
            MelGAN.n_dims, MEL_FFT_SIZE // 2 + 1, MelGAN.sample_rate, 0.0,
            float(MelGAN.sample_rate // 2))).to(device))
  return _DEVICE_TABLES[device]


class AudioCodec:
  name: str
  n_dims: int
  sample_rate: int
  hop_size: int
  min_value: float
  max_value: float
  pad_value: float
  additional_frames_for_encoding: int = 0

  @property
  def abbrev_str(self):
    return self.name

  @property
  def frame_rate(self):
    return int(self.sample_rate // self.hop_size)

  def scale_features(self, features, output_range=(-1.0, 1.0), clip=False):
    min_out, max_out = output_range
    if clip:
      features = np.clip(features, self.min_value, self.max_value)
    zero_one = (features - self.min_value) / (self.max_value - self.min_value)
    return zero_one * (max_out - min_out) + min_out

  def scale_to_features(self, outputs, input_range=(-1.0, 1.0), clip=False):
    min_out, max_out = input_range
    outputs = np.clip(outputs, min_out, max_out) if clip else outputs
    zero_one = (outputs - min_out) / (max_out - min_out)
    return zero_one * (self.max_value - self.min_value) + self.min_value

  def encode(self, audio):
    raise NotImplementedError('audio -> mel is outside the DDPM hot path (SURVEY §2)')

  def decode(self, features):
    raise NotImplementedError('mel -> audio vocoder is outside the DDPM hot path (SURVEY §2)')

  @property
  def context_codec(self):
    return self


class MelGAN(AudioCodec):
  """128-bin log-mel at 16 kHz, hop 320 -> 50 frames/s (msd/audio_codecs.py:204-218)."""
  name = 'melgan'
  n_dims = 128
  sample_rate = 16000
  hop_size = 320
  min_value = float(np.log(1e-5))
  max_value = 4.0
  pad_value = float(np.log(1e-5))
  additional_frames_for_encoding = 16

  def __init__(self, decode_dither_amount: float = 0.0):
    self._decode_dither_amount = decode_dither_amount

  def encode(self, audio):
    """audio [n] or [rows, n] at 16 kHz -> log-mel features [(rows,) ceil(n / 320), 128] f32:
    frame k is samples [320 k, 320 k + 640), zero-padded at the end.  A numpy array is encoded on
    the current CUDA device and comes back as numpy; a CUDA tensor stays on its device."""
    import torch
    from music_spectrogram_diffusion_b200 import engine
    as_numpy = not torch.is_tensor(audio)
    if as_numpy:
      audio = torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32)).to(
          torch.device('cuda', torch.cuda.current_device()))
    elif not audio.is_cuda:
      raise ValueError('MelGAN.encode: a tensor must be on a CUDA device (or pass numpy)')
    if audio.dim() not in (1, 2):
      raise ValueError(f'MelGAN.encode: audio must be [n] or [rows, n], got {tuple(audio.shape)}')
    rows = (audio if audio.dim() == 2 else audio[None]).to(torch.float32).contiguous()
    if rows.numel() == 0:
      frames = 0 if rows.shape[1] == 0 else -(-rows.shape[1] // self.hop_size)
      mel = torch.zeros(rows.shape[0], frames, self.n_dims, dtype=torch.float32, device=rows.device)
    else:
      window, weights = mel_tables(rows.device)
      mel = engine.op_audio_mel(rows, window, weights)
    if audio.dim() == 1:
      mel = mel[0]
    return mel.cpu().numpy() if as_numpy else mel
