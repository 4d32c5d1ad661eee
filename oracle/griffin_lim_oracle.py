"""fp64 numpy restatement of the library's Griffin-Lim decoding of MelGAN features
(`audio_codecs.griffin_lim`, csrc/audio_griffin_lim.cu).  Test infrastructure only.

The transform is the encoder's (`mel_oracle.frames64`): frame k is samples [320 k, 320 k + 640)
of a signal of 320 F samples, times the window, zero-padded to 1024, rfft.  `istft64` is its
least-squares inverse.  The tables (window, filterbank, pinv, 1 / L, beta) are taken as data, the
float32 values the library uses, so a difference between the GPU and this oracle is the kernels'
arithmetic alone.  Each `*_bound` function gives the error an fp32 evaluation of the same step,
from the same inputs, can be held to (2^-24 units, in the style of `mel_oracle.error_bound`).
"""

from __future__ import annotations

import numpy as np

from oracle import mel_oracle as MO
from oracle.philox import philox4x32_10

HOP = MO.HOP
WIN = MO.WIN
N_FFT = MO.N_FFT
BINS = N_FFT // 2 + 1
PHASE_TAG = 0x676c70     # Philox counter word 3 of the phase stream (the sampler's is 0x6d7364)
EPS = 1e-16              # angles = a / (|a| + EPS)
DEN_FLOOR = 1e-10        # ISTFT: below this sum of squared windows, the unnormalised sum
U = 2.0 ** -24


def fista_betas(n: int) -> np.ndarray:
  """beta_j = (t_j - 1) / t_{j+1}, t_0 = 1, t_{j+1} = (1 + sqrt(1 + 4 t_j^2)) / 2: fp64 [n]."""
  t, out = 1.0, []
  for _ in range(n):
    t1 = (1.0 + np.sqrt(1.0 + 4.0 * t * t)) / 2.0
    out.append((t - 1.0) / t1)
    t = t1
  return np.array(out, np.float64)


def uniform(seed: int, n: int, tag: int = PHASE_TAG) -> np.ndarray:
  """n float32 uniforms (r + 0.5) 2^-32, element e from word e % 4 of Philox4x32-10 at counter
  (e / 4 low, e / 4 high, 0, tag) keyed by seed: the phase stream of one row."""
  idx4 = np.arange(-(-n // 4), dtype=np.uint64)
  c0 = (idx4 & np.uint64(0xFFFFFFFF)).astype(np.uint32)
  c1 = (idx4 >> np.uint64(32)).astype(np.uint32)
  r = philox4x32_10(c0, c1, np.zeros_like(c0), np.full_like(c0, np.uint32(tag)),
                    seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
  words = np.stack(r, axis=1).reshape(-1)[:n]
  return (words.astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -32)


def phase_init64(seed: int, frames: int) -> np.ndarray:
  """librosa's init='random': e^{2 pi i u} in fp64 of the float32 u, complex [F, 513]."""
  u = uniform(seed, frames * BINS).astype(np.float64)
  return np.exp(2j * np.pi * u).reshape(frames, BINS)


def stft64(y: np.ndarray, window: np.ndarray) -> np.ndarray:
  """[320 F] -> complex [F, 513]: the encoder's frames, windowed, rfft of 1024."""
  return np.fft.rfft(MO.frames64(y) * np.asarray(window, np.float64), N_FFT, axis=1)


def _ola(parts: np.ndarray, frames: int) -> np.ndarray:
  """Overlap-add [F, 640] at hop 320, frame k - 1 before frame k: [320 F]."""
  out = np.zeros((frames + 1) * HOP)
  for k in range(frames):
    out[k * HOP:k * HOP + WIN] += parts[k]
  return out[:frames * HOP]


def istft64(X: np.ndarray, window: np.ndarray) -> np.ndarray:
  """complex [F, 513] -> [320 F]: sum_k w irfft(X_k)[:640] / sum_k w^2, unnormalised where
  sum_k w^2 <= 1e-10."""
  w = np.asarray(window, np.float64)
  F = X.shape[0]
  num = _ola(np.fft.irfft(X, N_FFT, axis=1)[:, :WIN] * w, F)
  den = _ola(np.broadcast_to(w * w, (F, WIN)), F)
  return np.where(den > DEN_FLOOR, num / np.where(den > DEN_FLOOR, den, 1.0), num)


def nnls64(features: np.ndarray, weights: np.ndarray, pinv: np.ndarray, inv_l: float,
           betas: np.ndarray, n_iter: int) -> np.ndarray:
  """[F, 128] codec features -> S [F, 513] >= 0 after n_iter FISTA steps of
  min |S W - exp(features)|^2 from Z_0 = Y_0 = max(0, M P)."""
  W = np.asarray(weights, np.float64)
  M = np.exp(np.asarray(features, np.float64))
  Z = np.maximum(0.0, M @ np.asarray(pinv, np.float64))
  Y = Z
  for j in range(n_iter):
    Zn = np.maximum(0.0, Y - ((Y @ W - M) @ W.T) * float(inv_l))
    Y = Zn + float(betas[j]) * (Zn - Z)
    Z = Zn
  return Z


def momentum_coef(momentum: float) -> float:
  """momentum / (1 + momentum) as the kernel uses it: from the float32 momentum, rounded to f32."""
  m = float(np.float32(momentum))
  return float(np.float32(m / (1.0 + m)))


def gl_iteration64(S: np.ndarray, angles: np.ndarray, tprev: np.ndarray, window: np.ndarray,
                   momentum: float):
  """One fast Griffin-Lim iteration: (angles, tprev, rebuilt, a)."""
  rebuilt = stft64(istft64(S * angles, window), window)
  a = rebuilt - momentum_coef(momentum) * tprev
  return a / (np.abs(a) + EPS), rebuilt, rebuilt, a


def decode64(features: np.ndarray, window: np.ndarray, weights: np.ndarray, pinv: np.ndarray,
             inv_l: float, betas: np.ndarray, nnls_iters: int, n_iter: int = 32,
             momentum: float = 0.99, seed: int = 0):
  """The whole decode of one row: (audio [320 F], S [F, 513])."""
  S = nnls64(features, weights, pinv, inv_l, betas, nnls_iters)
  angles = phase_init64(seed, S.shape[0])
  tprev = np.zeros_like(angles)
  for _ in range(n_iter):
    angles, tprev, _, _ = gl_iteration64(S, angles, tprev, window, momentum)
  return istft64(S * angles, window), S


def spectral_convergence(y: np.ndarray, S: np.ndarray, window: np.ndarray) -> float:
  """|(|STFT(y)| - S)|_F / |S|_F."""
  return float(np.linalg.norm(np.abs(stft64(y, window)) - S) / np.linalg.norm(S))


def inconsistency(X: np.ndarray, window: np.ndarray) -> float:
  """|STFT(ISTFT(X)) - X|_F."""
  return float(np.linalg.norm(stft64(istft64(X, window), window) - X))


# ---- error bounds of the fp32 kernels, from the same float32 inputs ----------------------------

def nnls_bound(features: np.ndarray, weights: np.ndarray, pinv: np.ndarray, inv_l: float,
               S64: np.ndarray, n_iter: int) -> np.ndarray:
  """Per frame, the bound on max_k |S_k - S64_k| of the fp32 kernel from the same tables.

  The start max(0, M P) is a 128-term dot product per bin after expf (2 ulp):
  b0 = 2^-24 (128 + 4) max_k sum_j |m_j| |P_jk|.  W has full column rank, so the NNLS problem is
  underdetermined and the iteration does not contract that error; the projected gradient step is
  non-expansive and a constant error cancels in the momentum term, so it is carried with a factor
  2.  Each step rounds a band sum of at most max_len terms (the widest band of W, 21 for MelGAN),
  the residual, and the projected update with its 1 / L-scaled transpose: at most
  2^-24 (max_len + 4) max(colsum / L, 1) s, s the frame's largest |Z| and colsum the largest
  column sum of W.  FISTA's momentum can grow a step's error by up to a factor j + 1 by step j
  (the transient of the linearised iteration, whose momentum weight tends to 1), so n steps add
  at most (n + 1)^2 / 2 of them: b = 2 b0 + (n + 1)^2 / 2 * step.  For n = 0 the bound is b0."""
  W = np.asarray(weights, np.float64)
  M = np.exp(np.asarray(features, np.float64))
  P = np.asarray(pinv, np.float64)
  b0 = U * 132.0 * (M @ np.abs(P)).max(axis=1)
  if n_iter == 0:
    return b0
  nz = W != 0
  first = np.where(nz.any(axis=0), nz.argmax(axis=0), 0)
  last = np.where(nz.any(axis=0), W.shape[0] - 1 - nz[::-1].argmax(axis=0), -1)
  max_len = int((last - first + 1).max())
  colsum = W.sum(axis=0).max()
  s = np.maximum(np.abs(S64).max(axis=1), np.maximum(0.0, M @ P).max(axis=1))
  step = U * (max_len + 4) * max(colsum * float(inv_l), 1.0) * s
  return 2.0 * b0 + 0.5 * (n_iter + 1) ** 2 * step


def log_fit(S: np.ndarray, features: np.ndarray, weights: np.ndarray, floor: float = 1e-3) -> float:
  """Mean |log(S W) - log M| over the bins where M = exp(features) exceeds `floor`."""
  M = np.exp(np.asarray(features, np.float64))
  rec = np.asarray(S, np.float64) @ np.asarray(weights, np.float64)
  above = M > floor
  return float(np.abs(np.log(np.maximum(rec[above], 1e-300)) - np.log(M[above])).mean())


def _frame_irfft_norms(X: np.ndarray) -> np.ndarray:
  """|irfft(X_k)|_2 over the 1024 samples, per frame [F]."""
  return np.sqrt((np.fft.irfft(X, N_FFT, axis=1) ** 2).sum(axis=1))


def istft_bound(S: np.ndarray, angles: np.ndarray, window: np.ndarray) -> np.ndarray:
  """Per sample [320 F], the bound on |y - istft64(S angles)| of an fp32 ISTFT from the f32 S and
  angles: each frame's irfft (S angles rounded, the packing, 3 radix-8 passes) is within
  e_k = 2^-24 (log2(1024) + 6) |irfft(X_k)|_2 of exact per sample; the windowing, the two-term sum
  and the f32 sum of squared windows add 2^-24 6 (|w_a x_{k-1}| + |w_b x_k|); the division by
  den spreads both."""
  w = np.asarray(window, np.float64)
  X = S * angles
  F = X.shape[0]
  x = np.fft.irfft(X, N_FFT, axis=1)[:, :WIN]
  e = U * (np.log2(N_FFT) + 6.0) * _frame_irfft_norms(X)
  parts = w[None, :] * e[:, None] + U * 6.0 * np.abs(w[None, :] * x)
  num = _ola(parts, F)
  den = _ola(np.broadcast_to(w * w, (F, WIN)), F)
  return np.where(den > DEN_FLOOR, num / np.where(den > DEN_FLOOR, den, 1.0), num)


def stft_bound(y: np.ndarray, y_bound: np.ndarray, window: np.ndarray) -> np.ndarray:
  """Per frame and bin [F, 513], the bound on |STFT_fp32(y') - stft64(y)| for any y' within
  y_bound of y: sum_n w_n y_bound_n over the frame, plus the fp32 FFT's own
  2^-24 (log2(1024) sqrt(1024) |w y|_2 + 4 |Y_k|)."""
  w = np.asarray(window, np.float64)
  spread = (MO.frames64(y_bound) * w).sum(axis=1)
  wy = MO.frames64(y) * w
  energy = np.sqrt((wy * wy).sum(axis=1))
  Y = np.abs(np.fft.rfft(wy, N_FFT, axis=1))
  return spread[:, None] + U * (np.log2(N_FFT) * np.sqrt(N_FFT) * energy[:, None] + 4.0 * Y)


def iteration_bounds(S: np.ndarray, angles: np.ndarray, tprev: np.ndarray, window: np.ndarray,
                     momentum: float):
  """(tprev bound [F, 513], a bound [F, 513], |a| [F, 513], angles bound [F, 513]) of one fp32
  iteration from the same inputs.  tprev = rebuilt: `stft_bound` of the ISTFT's bound.  a adds
  2^-24 2 (|rebuilt| + c |tprev|).  angles = a / (|a| + 1e-16) is held where |a| > its bound
  B_a: 2 B_a / (|a| - B_a) + 2^-24 6."""
  y = istft64(S * angles, window)
  tb = stft_bound(y, istft_bound(S, angles, window), window)
  rebuilt = stft64(y, window)
  c = momentum_coef(momentum)
  a = rebuilt - c * tprev
  ab = tb + U * 2.0 * (np.abs(rebuilt) + c * np.abs(tprev))
  mag = np.abs(a)
  with np.errstate(divide='ignore', invalid='ignore'):
    angb = np.where(mag > ab, 2.0 * ab / (mag - ab) + U * 6.0, np.inf)
  return tb, ab, mag, angb
