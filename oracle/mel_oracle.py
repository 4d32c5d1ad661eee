"""fp64 numpy restatement of MelGAN.encode (msd/audio_codecs.py:43-143, 204-247) and of the
full-song segmentation of its features (preprocessors.py:60-81, 631-696, 863-921).  Test
infrastructure only.

`mel_linear64` takes the float32 window and filterbank the library uses as data, so a difference
between the GPU and this oracle is the kernel's arithmetic alone; `hann_window64` and
`linear_to_mel_weight_matrix64` build the same tables in fp64 to check the float32 builders.
"""

from __future__ import annotations

from typing import Callable, Tuple

import numpy as np

HOP = 320
WIN = 640
N_FFT = 1024
N_MELS = 128
CLIP = (1e-5, 1e8)
ADDITIONAL_FRAMES = 16     # MelGAN.additional_frames_for_encoding


def num_frames(n: int) -> int:
  """tf.signal.frame(.., 640, 320, pad_end=True): ceil(n / 320) frames."""
  return -(-n // HOP)


def hann_window64(length: int = WIN) -> np.ndarray:
  return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(length) / length)


def linear_to_mel_weight_matrix64(num_mel_bins: int = N_MELS, num_spectrogram_bins: int = 513,
                                  sample_rate: float = 16000.0, lower_edge_hertz: float = 0.0,
                                  upper_edge_hertz: float = 8000.0) -> np.ndarray:
  mel = lambda f: 1127.0 * np.log(1.0 + np.asarray(f, np.float64) / 700.0)
  bins_mel = mel(np.linspace(0.0, sample_rate / 2.0, num_spectrogram_bins)[1:])[:, None]
  edges = np.linspace(mel(lower_edge_hertz), mel(upper_edge_hertz), num_mel_bins + 2)
  lo, c, up = edges[None, :-2], edges[None, 1:-1], edges[None, 2:]
  w = np.maximum(0.0, np.minimum((bins_mel - lo) / (c - lo), (up - bins_mel) / (up - c)))
  return np.pad(w, [[1, 0], [0, 0]])


def frames64(audio: np.ndarray) -> np.ndarray:
  """[n] -> [ceil(n / 320), 640] fp64: frame k = samples [320 k, 320 k + 640), zero past the end."""
  x = np.asarray(audio, np.float64)
  f = num_frames(len(x))
  padded = np.zeros(f * HOP + WIN)
  padded[:len(x)] = x
  idx = np.arange(f)[:, None] * HOP + np.arange(WIN)[None, :]
  return padded[idx]


def mel_linear64(audio: np.ndarray, window: np.ndarray, weights: np.ndarray) -> np.ndarray:
  """|rfft(frame * window, 1024)| @ weights in fp64, before clip and log: [F, 128]."""
  spec = np.abs(np.fft.rfft(frames64(audio) * np.asarray(window, np.float64), N_FFT, axis=1))
  return spec @ np.asarray(weights, np.float64)


def encode64(audio: np.ndarray, window: np.ndarray, weights: np.ndarray) -> np.ndarray:
  return np.log(np.clip(mel_linear64(audio, window, weights), *CLIP))


def error_bound(audio: np.ndarray, window: np.ndarray, weights: np.ndarray) -> np.ndarray:
  """Per frame and mel bin j, the bound on |exp(out) - clip(m64_j)| an fp32 FFT of the windowed
  frame can be held to: 2^-24 (log2(1024) sqrt(1024) ||w x||_2 sum_k W[k, j] + 4 clip(m64_j))."""
  wx = frames64(audio) * np.asarray(window, np.float64)
  energy = np.sqrt((wx * wx).sum(axis=1))[:, None]
  col = np.asarray(weights, np.float64).sum(axis=0)[None, :]
  m = np.clip(mel_linear64(audio, window, weights), *CLIP)
  return 2.0 ** -24 * (np.log2(N_FFT) * np.sqrt(N_FFT) * energy * col + 4.0 * m)


def pad_song(samples: np.ndarray) -> np.ndarray:
  """_audio_to_frames (preprocessors.py:60-81): pad by 320 - n % 320 (a whole hop when n % 320 == 0)."""
  x = np.asarray(samples)
  return np.pad(x, [0, HOP - len(x) % HOP])


def segment_spans(total: int, per_segment: int = 256) -> list:
  """split_full_song (preprocessors.py:863-921): segment s is hop-frames [start, end) with
  start = s * per_segment and end = (its last frame) + 16, cut at the song's end."""
  spans = []
  for start in range(0, total, per_segment):
    last = min(start + per_segment, total) - 1
    spans.append((start, min(last + ADDITIONAL_FRAMES, total)))
  return spans


def encode_song_by_segments(samples: np.ndarray, encode: Callable[[np.ndarray], np.ndarray],
                            per_segment: int = 256) -> Tuple[np.ndarray, int]:
  """The reference's per-segment route: each segment's samples (with its extra frames) encoded on
  their own, cut to per_segment frames and the last padded with 0.0 (encode_audio,
  preprocessors.py:631-696, and the feature converter).  Returns ([segments * per_segment, 128],
  num_frames)."""
  x = pad_song(samples)
  total = len(x) // HOP
  out = []
  for start, end in segment_spans(total, per_segment):
    enc = np.asarray(encode(x[start * HOP:end * HOP]))[:per_segment]
    seg = np.zeros((per_segment, N_MELS), enc.dtype)
    seg[:len(enc)] = enc
    out.append(seg)
  return np.concatenate(out), total
