"""Codec constants, feature scaling, and audio -> mel encoding.

Mirrors `AudioCodec.scale_features / scale_to_features` (msd/audio_codecs.py:166-183) and the
MelGAN constants (204-218).  `MelGAN.encode` is the reference's Audio2Mel (43-143) with MelGAN's
settings (226-247), computed by the library's CUDA kernel (`engine.op_audio_mel`) from the float32
tables built here (`hann_window`, `linear_to_mel_weight_matrix`, in TF's order of operations).
The vocoder (`decode`, a TF-Hub SavedModel, 249-264) is out of scope: it raises.  `griffin_lim`
stands in for it: a weight-free inversion of the encoder's own transform (band-sparse NNLS for the
linear magnitudes, then fast Griffin-Lim for the phase), computed by the library's CUDA kernels
(`engine.op_griffin_lim_*`) from the tables built here (`griffin_lim_tables`).  Its audio is not
the reference's MelGAN audio; it is an audible, deterministic rendering of the features.

Recordings at other rates are brought to 16 kHz by `resample`, librosa 0.9's
`resample(res_type='kaiser_best')` as the reference calls it (preprocessors.py:150-155, 332-333,
518-521), computed by the library's CUDA kernel (`engine.op_audio_resample`) bit for bit as
resampy 0.2.2's loop, from the filter built here (`kaiser_best_window`) and the time register
described by `time_register_segments`.
"""

from __future__ import annotations

import math
from typing import Dict, Tuple

import numpy as np

MEL_WIN_LENGTH = 640    # MelGAN._frame_length
MEL_FFT_SIZE = 1024     # MelGAN._fft_size

# resampy's 'kaiser_best' filter: sinc_window(num_zeros=64, precision=9,
# window=kaiser(beta=14.769656459379492), rolloff=0.9475937167399596)
KAISER_BEST_NUM_ZEROS = 64
KAISER_BEST_PRECISION = 9
KAISER_BEST_BETA = 14.769656459379492
KAISER_BEST_ROLLOFF = 0.9475937167399596


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


# FISTA steps of the mel -> linear-magnitude NNLS: the mean |log(S W) - log M| over bins above 1e-3
# is below 1e-3 at this count on a synthetic song (tests/test_griffin_lim.py)
NNLS_ITERS = 200

_GL_HOST: list = []
_DEVICE_GL_TABLES: Dict[object, Tuple[object, float, object]] = {}


def fista_betas(n: int) -> np.ndarray:
  """FISTA's momentum weights beta_j = (t_j - 1) / t_{j+1}, t_0 = 1,
  t_{j+1} = (1 + sqrt(1 + 4 t_j^2)) / 2, in fp64: [n]."""
  t, out = 1.0, np.empty(n, np.float64)
  for j in range(n):
    t1 = (1.0 + math.sqrt(1.0 + 4.0 * t * t)) / 2.0
    out[j] = (t - 1.0) / t1
    t = t1
  return out


def griffin_lim_host_tables() -> Tuple[np.ndarray, float, np.ndarray]:
  """(pinv f32 [128, 513], 1 / L as an f32 value, beta f32 [NNLS_ITERS]) of MelGAN's filterbank
  W (`linear_to_mel_weight_matrix`): pinv(W) and L = |W|_2^2 computed in fp64 from the float32 W,
  the FISTA weights in fp64; each rounded to float32 once (read-only)."""
  if not _GL_HOST:
    w64 = linear_to_mel_weight_matrix(MelGAN.n_dims, MEL_FFT_SIZE // 2 + 1, MelGAN.sample_rate, 0.0,
                                      float(MelGAN.sample_rate // 2)).astype(np.float64)
    pinv = np.linalg.pinv(w64).astype(np.float32)
    inv_l = float(np.float32(1.0 / np.linalg.norm(w64, 2) ** 2))
    beta = fista_betas(NNLS_ITERS).astype(np.float32)
    pinv.setflags(write=False)
    beta.setflags(write=False)
    _GL_HOST.append((pinv, inv_l, beta))
  return _GL_HOST[0]


def griffin_lim_tables(device):
  """(pinv f32 [128, 513] tensor, 1 / L float, beta f32 [NNLS_ITERS] tensor) on `device`, built
  once per device (`griffin_lim_host_tables`)."""
  if device not in _DEVICE_GL_TABLES:
    import torch
    pinv, inv_l, beta = griffin_lim_host_tables()
    _DEVICE_GL_TABLES[device] = (torch.from_numpy(pinv.copy()).to(device), inv_l,
                                 torch.from_numpy(beta.copy()).to(device))
  return _DEVICE_GL_TABLES[device]


def griffin_lim(features, n_iter: int = 32, momentum: float = 0.99, seed: int = 0):
  """MelGAN features [F, 128] or [rows, F, 128] (codec units, as `MelGAN.encode` and
  `full_pred_encoded` hold them) -> audio f32 [320 F] or [rows, 320 F] at 16 kHz, without the
  vocoder:
    1. the linear magnitudes S [F, 513] >= 0, the least-squares fit of exp(features) by S W after
       NNLS_ITERS FISTA steps from max(0, exp(features) pinv(W));
    2. random phases from the Philox stream of `seed` (librosa's init='random'; every row draws
       the same stream, so a row does not depend on its place in the batch);
    3. n_iter fast Griffin-Lim iterations with `momentum` (librosa.griffinlim's update; 0 is plain
       Griffin-Lim) through the encoder's own STFT and its least-squares inverse;
    4. the inverse STFT of S with the final phases.
  Re-encoding the audio gives F frames again.  The result is deterministic: the same call gives
  the same bits.  It is not the reference's MelGAN vocoder output.

  Songs of different lengths go in one call padded at the end with `MelGAN.pad_value` to a common
  F; cut each row to its own num_frames * 320 samples afterwards.  A padded row's last real frame
  then sees near-silence after it, so it is close to, not bit-identical with, decoding that row
  alone; equal-length rows are bit-identical.

  A numpy array is decoded on the current CUDA device and comes back as numpy; a CUDA tensor
  stays on its device.  Raises ValueError for a shape other than [F, 128] or [rows, F, 128],
  momentum < 0 or n_iter < 0, before any device is used."""
  import torch
  from music_spectrogram_diffusion_b200 import engine
  as_numpy = not torch.is_tensor(features)
  if as_numpy:
    features = np.asarray(features)
  elif not features.is_cuda:
    raise ValueError('griffin_lim: a tensor must be on a CUDA device (or pass numpy)')
  if features.ndim not in (2, 3) or features.shape[-1] != MelGAN.n_dims:
    raise ValueError(f'griffin_lim: features must be [F, {MelGAN.n_dims}] or [rows, F, '
                     f'{MelGAN.n_dims}], got {tuple(features.shape)}')
  if not momentum >= 0:
    raise ValueError(f'griffin_lim: momentum={momentum} must be >= 0')
  if int(n_iter) != n_iter or n_iter < 0:
    raise ValueError(f'griffin_lim: n_iter={n_iter} must be an integer >= 0')
  if as_numpy:
    dev = torch.device('cuda', torch.cuda.current_device())
    x = torch.from_numpy(np.ascontiguousarray(features, dtype=np.float32)).to(dev)
  else:
    dev = features.device
    x = features.to(torch.float32).contiguous()
  rows = x if x.dim() == 3 else x[None]
  window, weights = mel_tables(dev)
  pinv, inv_l, beta = griffin_lim_tables(dev)
  mag = engine.op_griffin_lim_magnitude(rows, weights, pinv, inv_l, beta, NNLS_ITERS)
  angles = engine.op_griffin_lim_init(rows.shape[0], rows.shape[1], seed, dev)
  tprev = torch.zeros_like(angles)
  engine.op_griffin_lim_iterate(mag, window, angles, tprev, momentum, int(n_iter))
  y = engine.op_griffin_lim_istft(mag, window, angles)
  if x.dim() == 2:
    y = y[0]
  return y.cpu().numpy() if as_numpy else y


_KAISER_BEST = []
_DEVICE_WINDOWS: Dict[object, object] = {}


def kaiser_best_window() -> np.ndarray:
  """resampy's 'kaiser_best' half window, f64 [64 * 2^9 + 1] (read-only):
  rolloff * sinc(rolloff * linspace(0, 64, 32769)) * kaiser(65537, beta)[32768:], with numpy's
  sinc and kaiser.  resampy ships the same table precomputed (data/kaiser_best.npz); the two may
  differ in their last bits (DESIGN section 4)."""
  if not _KAISER_BEST:
    n = (1 << KAISER_BEST_PRECISION) * KAISER_BEST_NUM_ZEROS
    sinc = KAISER_BEST_ROLLOFF * np.sinc(
        KAISER_BEST_ROLLOFF * np.linspace(0, KAISER_BEST_NUM_ZEROS, num=n + 1, endpoint=True))
    win = np.kaiser(2 * n + 1, KAISER_BEST_BETA)[n:] * sinc
    win.setflags(write=False)
    _KAISER_BEST.append(win)
  return _KAISER_BEST[0]


def resample_window(device):
  """`kaiser_best_window()` as a float64 tensor on `device`, built once per device."""
  if device not in _DEVICE_WINDOWS:
    import torch
    _DEVICE_WINDOWS[device] = torch.from_numpy(kaiser_best_window().copy()).to(device)
  return _DEVICE_WINDOWS[device]


def resampy_length(n: int, orig_sr: int, target_sr: int) -> int:
  """resampy's output length, int(n * target / orig) in float64."""
  return int(n * (float(target_sr) / orig_sr))


def librosa_length(n: int, orig_sr: int, target_sr: int) -> int:
  """librosa.resample's output length, ceil(n * target / orig) in float64 (fix=True pads the
  resampy output with zeros to it)."""
  return int(np.ceil(n * (float(target_sr) / orig_sr)))


def time_register_segments(orig_sr: int, target_sr: int, n_out: int) -> np.ndarray:
  """resampy's time register r_0 = 0, r_{t+1} = fl(r_t + 1 / ratio) for t < n_out, as f64 [S, 3]
  rows (t_s, r_s, d): for t_s <= t < t_{s+1} (t_{S} = n_out), r_t = r_s + (t - t_s) d exactly.

  While r stays inside one binade [2^e, 2^(e+1)) every r is a multiple of that binade's ulp u,
  so fl(r + inc) = r + d with d = inc rounded to a multiple of u -- the same d for every step,
  unless inc is an exact tie on that grid (round-half-even then depends on r).  A segment is
  such a run of steps, ended short of the binade's top; steps near the top, ties and r = 0 get
  segments of one output.  That gives about three segments per binade of the output's span."""
  inc = 1.0 / (float(target_sr) / orig_sr)
  segs = []
  t, r = 0, 0.0
  while t < n_out:
    d = (r + inc) - r
    length = 1
    if r > 0.0:
      e = math.frexp(r)[1]                  # r in [2^(e-1), 2^e)
      top, u = math.ldexp(1.0, e), math.ldexp(1.0, e - 53)
      if math.fmod(inc, u) != u / 2:
        # steps j < length - 1 keep r + j d + inc below top: fl adds exactly d
        length = max(1, int((top - r) / d) - 1)
    length = min(length, n_out - t)
    segs.append((t, r, d))
    t += length
    r = (r + (length - 1) * d) + inc
  return np.array(segs, np.float64).reshape(-1, 3)


def resample(audio, orig_sr: int, target_sr: int = 16000):
  """librosa 0.9 `resample(audio, orig_sr, target_sr)` with its default res_type='kaiser_best':
  float32 audio [n] or [rows, n] -> [(rows,) ceil(n * target_sr / orig_sr)] float32, each row
  resampled by resampy's band-limited sinc interpolation and zero-padded at the end to librosa's
  length.  Equal rates return `audio` unchanged, as librosa does.  Computed on the GPU with
  float64 taps into a float32 result, bit for bit resampy's loop on float32 samples (what
  librosa.load reads; `engine.op_audio_resample`).  Other dtypes are refused rather than rounded:
  librosa keeps float64 samples in float64, which this is not.  A numpy array is resampled on the
  current CUDA device and comes back as numpy; a CUDA tensor stays on its device.  Raises
  ValueError for rates <= 0, a dtype other than float32 and, as resampy does, when
  int(n * ratio) < 1."""
  import torch
  from music_spectrogram_diffusion_b200 import engine
  if int(orig_sr) != orig_sr or int(target_sr) != target_sr or orig_sr <= 0 or target_sr <= 0:
    raise ValueError(f'resample: rates must be positive integers, got {orig_sr} -> {target_sr}')
  orig_sr, target_sr = int(orig_sr), int(target_sr)
  as_numpy = not torch.is_tensor(audio)
  if as_numpy:
    audio = np.asarray(audio)
  elif not audio.is_cuda:
    raise ValueError('resample: a tensor must be on a CUDA device (or pass numpy)')
  if audio.ndim not in (1, 2):
    raise ValueError(f'resample: audio must be [n] or [rows, n], got {tuple(audio.shape)}')
  if audio.dtype not in (np.float32, torch.float32):
    raise ValueError(f'resample: audio must be float32 (librosa.load reads float32; cast first), '
                     f'got {audio.dtype}')
  if orig_sr == target_sr:
    return audio
  n = audio.shape[-1]
  n_out = resampy_length(n, orig_sr, target_sr)
  if n_out < 1:
    raise ValueError(f'resample: {n} samples at {orig_sr} Hz give no output at {target_sr} Hz')
  segs = time_register_segments(orig_sr, target_sr, n_out)
  t_s, r_s, d = segs[-1]
  if int(r_s + (n_out - 1 - t_s) * d) >= n:
    raise ValueError(f'resample: {n} samples are too long for the float64 time register '
                     f'at {orig_sr} -> {target_sr} Hz: it runs past the input')
  if as_numpy:
    dev = torch.device('cuda', torch.cuda.current_device())
    x = torch.from_numpy(np.ascontiguousarray(audio)).to(dev)
  else:
    dev = audio.device
    x = audio
  rows = (x if x.dim() == 2 else x[None]).contiguous()
  y = engine.op_audio_resample(rows, orig_sr, target_sr, resample_window(dev),
                               KAISER_BEST_PRECISION, torch.from_numpy(segs).to(dev))
  y = torch.nn.functional.pad(y, (0, librosa_length(n, orig_sr, target_sr) - n_out))
  if audio.ndim == 1:
    y = y[0]
  return y.cpu().numpy() if as_numpy else y


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
    raise NotImplementedError('mel -> audio vocoder is outside the DDPM hot path (SURVEY §2); '
                              'audio_codecs.griffin_lim renders features to audio without it')

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
