"""CPU: the fp64 Griffin-Lim oracle (oracle/griffin_lim_oracle.py), the host tables, the phase
stream's Philox helper, the WAV writer, griffin_lim's argument checks, and that moving the FFT and
Philox code into shared headers left the encoder's and the sampler's machine code unchanged."""
import io
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from music_spectrogram_diffusion_b200 import _native, audio_codecs, song
from oracle import griffin_lim_oracle as G
from oracle import mel_oracle as MO
from oracle import philox

SR = 16000
WIN = audio_codecs.hann_window()
WEIGHTS = audio_codecs.linear_to_mel_weight_matrix()
PINV, INV_L, BETA = audio_codecs.griffin_lim_host_tables()


def song_signal(seconds=6.0, seed=0):
  """12 random harmonic notes with attack and decay envelopes, padded to whole hops."""
  rng = np.random.default_rng(seed)
  n = int(seconds * SR)
  t = np.arange(n) / SR
  x = np.zeros(n)
  for _ in range(12):
    f0, start, decay = rng.uniform(80, 1000), rng.uniform(0, seconds - 1), rng.uniform(1, 4)
    dt = np.maximum(t - start, 0.0)
    env = np.where(t >= start, np.exp(-dt * decay) * (1 - np.exp(-dt * 200)), 0.0)
    for h in range(1, 6):
      x += 0.05 / h * env * np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 2 * np.pi))
  return np.pad(x, [0, MO.num_frames(n) * 320 - n])


def decode_features():
  """[F, 128] f32 of a 3 s song with a silent stretch and a loud full-band burst: the features the
  GPU tests decode."""
  x = song_signal(3.0, seed=3)
  x[16000:20000] = 0.0
  x[30000:32000] += np.random.default_rng(4).uniform(-0.8, 0.8, 2000)
  return MO.encode64(x, WIN, WEIGHTS).astype(np.float32)


NNLS_TOL = 5e-3   # at NNLS_ITERS, per frame: max |S - S64| <= NNLS_TOL * max |S64|


def nnls_failures(got, ref, features, n_iter):
  """The checks the kernel's NNLS magnitudes `got` [F, 513] are held to against the oracle's
  `ref` after n_iter steps, as a list of the ones that fail:
    - per frame, max |got - ref| within `G.nnls_bound`;
    - at NNLS_ITERS, per frame, max |got - ref| <= NNLS_TOL max |ref| (the model bound grows as
      (n + 1)^2 and is loose there: this catches a lost momentum or a short step count);
    - the mean |log(S W) - log M| over bins above 1e-3 within half the oracle's, plus 1e-6."""
  got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
  err = np.abs(got - ref).max(axis=1)
  failed = []
  bound = G.nnls_bound(features, WEIGHTS, PINV, INV_L, ref, n_iter)
  if not (err <= bound).all():
    failed.append(f'bound: err/bound {float((err / bound).max()):.3g}')
  if n_iter == audio_codecs.NNLS_ITERS:
    rel = err / np.abs(ref).max(axis=1)
    if not (rel <= NNLS_TOL).all():
      failed.append(f'tolerance: max err / max|S| {float(rel.max()):.3g}')
  fit, fit_ref = G.log_fit(got, features, WEIGHTS), G.log_fit(ref, features, WEIGHTS)
  if abs(fit - fit_ref) > 0.5 * fit_ref + 1e-6:
    failed.append(f'log fit {fit:.3g} vs {fit_ref:.3g}')
  return failed


@pytest.fixture(scope='module')
def features():
  return MO.encode64(song_signal(), WIN, WEIGHTS).astype(np.float32)


@pytest.fixture(scope='module')
def magnitude(features):
  return G.nnls64(features, WEIGHTS, PINV, INV_L, BETA, audio_codecs.NNLS_ITERS)


def test_istft_inverts_stft():
  rng = np.random.default_rng(1)
  x = rng.uniform(-1, 1, 320 * 23)
  y = G.istft64(G.stft64(x, WIN), WIN)
  assert y.shape == x.shape
  # sample 0: the window is 0 there and only frame 0 covers it
  assert y[0] == 0.0
  err = np.abs(y - x)
  assert err[16:].max() <= 1e-12
  # the first samples are divided by w[n]^2 ~ (pi n / 640)^4 alone: rounding grows by 1 / w[n]
  w = WIN.astype(np.float64)
  assert (err[1:16] * w[1:16] <= 1e-14).all(), err[1:16]


def test_nnls_reaches_the_mel_at_the_default_count(features, magnitude):
  m = np.exp(features.astype(np.float64))
  rec = magnitude @ WEIGHTS.astype(np.float64)
  above = m > 1e-3
  err = np.abs(np.log(np.maximum(rec[above], 1e-300)) - np.log(m[above])).mean()
  assert err <= 1e-3, err
  assert (magnitude >= 0).all()
  # the clamped pseudo-inverse alone, the start, is far off
  start = G.nnls64(features, WEIGHTS, PINV, INV_L, BETA, 0) @ WEIGHTS.astype(np.float64)
  assert np.abs(np.log(np.maximum(start[above], 1e-300)) - np.log(m[above])).mean() > 10 * err


def test_plain_griffin_lim_inconsistency_never_increases(magnitude):
  S = magnitude[:100]
  angles = G.phase_init64(0, S.shape[0])
  tprev = np.zeros_like(angles)
  seen = [G.inconsistency(S * angles, WIN)]
  for _ in range(40):
    angles, tprev, _, _ = G.gl_iteration64(S, angles, tprev, WIN, 0.0)
    seen.append(G.inconsistency(S * angles, WIN))
  assert all(b <= a * (1 + 1e-12) for a, b in zip(seen, seen[1:])), seen
  assert seen[-1] < 0.5 * seen[0]


def test_fast_griffin_lim_converges_further_than_plain(features, magnitude):
  sc = {}
  for momentum in (0.0, 0.99):
    y, S = G.decode64(features, WIN, WEIGHTS, PINV, INV_L, BETA, audio_codecs.NNLS_ITERS, 32,
                      momentum, seed=0)
    assert y.shape == (features.shape[0] * 320,)
    sc[momentum] = G.spectral_convergence(y, S, WIN)
  assert sc[0.99] < sc[0.0], sc


def test_nnls_checks_see_the_momentum_and_the_step_count():
  """The checks the GPU's NNLS is held to fail for a kernel without FISTA's momentum or one that
  stops early, and the bound stays far below the magnitudes while the momentum acts."""
  feats = decode_features()
  nomo = np.zeros_like(BETA)
  for n in (3, 10, audio_codecs.NNLS_ITERS):
    ref = G.nnls64(feats, WEIGHTS, PINV, INV_L, BETA, n)
    assert nnls_failures(ref, ref, feats, n) == []
    assert nnls_failures(G.nnls64(feats, WEIGHTS, PINV, INV_L, nomo, n), ref, feats, n), n
    bound = G.nnls_bound(feats, WEIGHTS, PINV, INV_L, ref, n)
    if n <= 10:
      assert (bound <= 1e-3 * np.abs(ref).max(axis=1)).all(), n
  ref = G.nnls64(feats, WEIGHTS, PINV, INV_L, BETA, audio_codecs.NNLS_ITERS)
  short = G.nnls64(feats, WEIGHTS, PINV, INV_L, BETA, 50)
  assert nnls_failures(short, ref, feats, audio_codecs.NNLS_ITERS)
  # an all-zero output does not pass
  assert nnls_failures(np.zeros_like(ref), ref, feats, audio_codecs.NNLS_ITERS)
  # the widest band of MelGAN's filterbank, which the per-step rounding counts
  assert int((WEIGHTS != 0).sum(axis=0).max()) == 21


def test_tables_match_fp64_recomputation():
  w64 = WEIGHTS.astype(np.float64)
  assert PINV.dtype == np.float32 and PINV.shape == (128, 513)
  np.testing.assert_array_equal(PINV, np.linalg.pinv(w64).astype(np.float32))
  # W [513, 128] has full column rank, so its pseudo-inverse is a left inverse: P W = I
  assert np.linalg.matrix_rank(w64) == 128
  assert np.abs(PINV.astype(np.float64) @ w64 - np.eye(128)).max() < 1e-4
  sigma = np.linalg.svd(w64, compute_uv=False)[0]
  assert INV_L == float(np.float32(1.0 / sigma ** 2))
  assert abs(1.0 / INV_L - 9.907) < 1e-3
  assert BETA.dtype == np.float32 and BETA.shape == (audio_codecs.NNLS_ITERS,)
  np.testing.assert_array_equal(BETA, G.fista_betas(audio_codecs.NNLS_ITERS).astype(np.float32))
  t1 = (1 + np.sqrt(5)) / 2
  assert BETA[0] == 0.0 and BETA[1] == np.float32((t1 - 1) / ((1 + np.sqrt(1 + 4 * t1 * t1)) / 2))
  assert (np.diff(BETA) > 0).all() and BETA[-1] < 1


def test_philox_uniform_helper_agrees_with_philox4x32_10():
  seed = (7 << 32) | 12345
  n = 4 * 50
  # with the sampler's tag its uniforms are the ones normal() turns into Box-Muller pairs
  u = G.uniform(seed, n, tag=0x6d7364).reshape(-1, 4)
  f32 = np.float32
  ra = np.sqrt(f32(-2.0) * np.log(np.clip(u[:, 0], f32(1e-12), f32(1.0))))
  a1 = (f32(2.0) * u[:, 1]).astype(np.float64) * np.pi
  np.testing.assert_array_equal((ra * np.cos(a1).astype(np.float32)).astype(np.float32),
                                philox.normal(seed, 0, n).reshape(-1, 4)[:, 0])
  # the phase stream: word e % 4 at counter (e / 4, 0, 0, PHASE_TAG); a partial last group
  u = G.uniform(seed, 4 * 3 + 2)
  for e in (0, 5, 13):
    r = philox.philox4x32_10(e // 4, 0, 0, G.PHASE_TAG, seed & 0xFFFFFFFF, seed >> 32)
    assert u[e] == (np.float32(r[e % 4]) + np.float32(0.5)) * np.float32(2.0 ** -32)
  assert u.shape == (14,) and ((u > 0) & (u <= 1)).all()
  assert G.PHASE_TAG != 0x6d7364


def test_save_audio_round_trips_16_bit_samples(tmp_path):
  rng = np.random.default_rng(2)
  x = rng.uniform(-1, 1, 5000).astype(np.float32)
  x[:6] = [-1.0, 1.0, 1.7, -3.0, 0.99999, np.nan]
  path = str(tmp_path / 'a.wav')
  song.save_audio(path, x)
  got = song.load_audio(path)
  q = np.clip(np.rint(np.nan_to_num(x.astype(np.float64)) * 32768), -32768, 32767) / 32768
  np.testing.assert_array_equal(got, q.astype(np.float32))
  assert got[1] == got[2] == np.float32(32767 / 32768) and got[3] == -1.0 and got[5] == 0.0
  # a quantised signal comes back bit for bit, through a file object too
  buf = io.BytesIO()
  song.save_audio(buf, got)
  np.testing.assert_array_equal(song.load_audio(buf.getvalue()), got)
  with pytest.raises(ValueError):
    song.save_audio(io.BytesIO(), np.zeros((2, 10)))


def test_griffin_lim_argument_errors_need_no_device():
  with pytest.raises(ValueError, match='must be'):
    audio_codecs.griffin_lim(np.zeros((4, 64), np.float32))
  with pytest.raises(ValueError, match='must be'):
    audio_codecs.griffin_lim(np.zeros(128, np.float32))
  with pytest.raises(ValueError, match='must be'):
    audio_codecs.griffin_lim(np.zeros((1, 2, 3, 128), np.float32))
  with pytest.raises(ValueError, match='momentum'):
    audio_codecs.griffin_lim(np.zeros((4, 128), np.float32), momentum=-0.5)
  with pytest.raises(ValueError, match='momentum'):
    audio_codecs.griffin_lim(np.zeros((4, 128), np.float32), momentum=float('nan'))
  with pytest.raises(ValueError, match='n_iter'):
    audio_codecs.griffin_lim(np.zeros((4, 128), np.float32), n_iter=-1)
  with pytest.raises(NotImplementedError, match='griffin_lim'):
    audio_codecs.MelGAN().decode(np.zeros((4, 128), np.float32))


# ---- the shared-header refactor leaves the existing kernels' SASS unchanged ---------------------

PARENT = '371413184d8e1c6c8c43d8c87afdf0143a80cee3'   # the last commit before the shared headers
HEADERS = 'a730110b2aaf35e5f81c1077848a0c8dbc55ee03'  # the commit that introduced them
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = 'music_spectrogram_diffusion_b200/csrc'
# kernels changed on purpose since the shared headers came in: compared as that commit built them
CHANGED_SINCE = {'sampler_step_kernel'}
# kernels changed on purpose later, not compared: the token embedding now gives an id outside the table
# a zero row, as the reference's one-hot embedding does (tests/test_gpu_row_kernels.py checks it bit for bit)
CHANGED_LATER = {'embed_tokens_kernel'}


def _sass(root, src, out_dir):
  """{kernel: SASS} of one source file."""
  cubin = os.path.join(out_dir, src.replace('.cu', '.cubin'))
  cmd = [_native._nvcc()] + _native.NVCC_FLAGS + ['-I', os.path.join(root, 'include'), '-cubin',
                                                  os.path.join(root, CSRC, src), '-o', cubin]
  subprocess.run(cmd, check=True, capture_output=True)
  cuobjdump = shutil.which('cuobjdump') or os.path.join(os.path.dirname(_native._nvcc()), 'cuobjdump')
  sass = subprocess.run([cuobjdump, '-sass', cubin], check=True, capture_output=True,
                        text=True).stdout
  # anonymous-namespace names carry a hash of the source's path
  sass = re.sub(r'_GLOBAL__N__[0-9a-f]+_', '_GLOBAL__N__', sass)
  parts = re.split(r'^\s+Function : (\S+)\s*$', sass, flags=re.M)
  return dict(zip(parts[1::2], parts[2::2]))


def _checkout(commit, dest):
  (dest / CSRC).mkdir(parents=True)
  (dest / 'include').mkdir()
  listing = subprocess.run(['git', '-C', REPO, 'ls-tree', '--name-only', commit, CSRC + '/'],
                           check=True, capture_output=True, text=True).stdout.split()
  for path in listing + ['include/msd_b200.h']:
    blob = subprocess.run(['git', '-C', REPO, 'show', f'{commit}:{path}'], check=True,
                          capture_output=True).stdout
    (dest / path).write_bytes(blob)
  return str(dest)


def test_shared_headers_leave_encoder_and_sampler_sass_unchanged(tmp_path):
  if shutil.which('git') is None or shutil.which(_native._nvcc()) is None:
    pytest.skip('needs git and nvcc')
  for commit in (PARENT, HEADERS):
    if subprocess.run(['git', '-C', REPO, 'cat-file', '-e', commit + '^{commit}'],
                      capture_output=True).returncode != 0:
      pytest.skip('the commits around the shared headers are not in this checkout')
  old = _checkout(PARENT, tmp_path / 'parent')
  at_headers = _checkout(HEADERS, tmp_path / 'headers')
  for src in ('audio_mel.cu', 'elementwise.cu'):
    a = _sass(old, src, old)
    b = _sass(REPO, src, str(tmp_path))
    assert any(('audio_mel_kernel' if src == 'audio_mel.cu' else 'sampler_step') in k for k in a)
    assert a.keys() == b.keys(), f'{src}: kernels differ from the parent commit'
    changed = [k for k in a if any(n in k for n in CHANGED_SINCE)]
    if changed:
      b.update({k: v for k, v in _sass(at_headers, src, at_headers).items() if k in changed})
    for k in a:
      if not any(n in k for n in CHANGED_LATER):
        assert a[k] == b[k], f'{src}: SASS of {k} differs from the parent commit'
