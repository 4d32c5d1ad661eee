"""-m gpu: Griffin-Lim decoding (msd_op_griffin_lim_*) against the fp64 oracle one op and one
iteration at a time, the whole decode's determinism and batch independence, the ops' argument
checks, and a synthesized song rendered to a WAV file."""
import ctypes
import io

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import _native, audio_codecs, engine, song
from oracle import griffin_lim_oracle as G
from oracle import mel_oracle as MO
from tests.test_gpu_song_batch import _model, _notes, tiny  # noqa: F401  (fixture)
from tests.test_griffin_lim import decode_features, nnls_failures

pytestmark = pytest.mark.gpu

WIN = audio_codecs.hann_window()
WEIGHTS = audio_codecs.linear_to_mel_weight_matrix()
PINV, INV_L, BETA = audio_codecs.griffin_lim_host_tables()
MAX_RATIO = {}   # err / bound per check, reported by the last test


def _ratio(name, err, bound):
  err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
  assert np.isfinite(err).all()
  r = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1.0),
                            np.where(err > 0, np.inf, 0.0))))
  MAX_RATIO[name] = max(MAX_RATIO.get(name, 0.0), r)
  assert r <= 1.0, (name, r)
  return r


@pytest.fixture(scope='module')
def dev(cuda_device):
  return cuda_device


@pytest.fixture(scope='module')
def features():
  """[F, 128] f32: a 3 s song, a silent stretch and a loud full-band burst."""
  return decode_features()


def _tables(dev):
  window, weights = audio_codecs.mel_tables(dev)
  pinv, inv_l, beta = audio_codecs.griffin_lim_tables(dev)
  return window, weights, pinv, inv_l, beta


def test_phase_init_is_cos_sin_of_the_philox_uniforms(dev):
  for seed in (0, (1 << 40) + 5):
    for frames in (37, 1):   # 37 * 513 and 513 are odd: a partial last group of 4
      got = engine.op_griffin_lim_init(2, frames, seed, dev).cpu().numpy()
      assert got.shape == (2, frames, 513)
      np.testing.assert_array_equal(got[0], got[1])
      u = G.uniform(seed, frames * 513).astype(np.float64).reshape(frames, 513)
      for part, ref in ((got[0].real, np.cos(2 * np.pi * u)), (got[0].imag, np.sin(2 * np.pi * u))):
        ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
        _ratio('phase init (2 ulp)', np.abs(part - ref), 2 * ulp)


@pytest.mark.parametrize('n_iter', [0, 1, 3, 10, audio_codecs.NNLS_ITERS])
def test_nnls_against_oracle(dev, features, n_iter):
  _, weights, pinv, inv_l, beta = _tables(dev)
  feats = torch.from_numpy(features).to(dev)
  got = engine.op_griffin_lim_magnitude(feats[None], weights, pinv, inv_l, beta, n_iter)[0]
  got = got.cpu().numpy().astype(np.float64)
  ref = G.nnls64(features, WEIGHTS, PINV, INV_L, BETA, n_iter)
  assert (got >= 0).all()
  err = np.abs(got - ref).max(axis=1)
  scale = np.abs(ref).max(axis=1)
  _ratio(f'nnls {n_iter} steps', err, G.nnls_bound(features, WEIGHTS, PINV, INV_L, ref, n_iter))
  print(f'nnls {n_iter} steps: max err / max|S| per frame {float((err / scale).max()):.3e}, '
        f'log fit {G.log_fit(got, features, WEIGHTS):.4e} (oracle '
        f'{G.log_fit(ref, features, WEIGHTS):.4e})')
  assert nnls_failures(got, ref, features, n_iter) == []
  # rows and frames are independent: frames 5.. of a 3-row launch equal those frames alone
  rows = torch.stack([feats, feats.flip(0), feats])
  batch = engine.op_griffin_lim_magnitude(rows, weights, pinv, inv_l, beta, n_iter)
  alone = engine.op_griffin_lim_magnitude(feats[None, 5:], weights, pinv, inv_l, beta, n_iter)
  assert torch.equal(batch[2, 5:], alone[0]) and torch.equal(batch[0], batch[2])


def _state(dev, features, seed=1):
  """(S, angles, tprev) f32/complex64 on the device: S from the oracle's NNLS, random phases,
  and a tprev of the magnitude's scale."""
  S = G.nnls64(features, WEIGHTS, PINV, INV_L, BETA, audio_codecs.NNLS_ITERS).astype(np.float32)
  F = S.shape[0]
  angles = engine.op_griffin_lim_init(1, F, seed, dev)[0]
  rng = np.random.default_rng(seed)
  tprev = (S * np.exp(2j * np.pi * rng.uniform(size=S.shape))).astype(np.complex64)
  return torch.from_numpy(S).to(dev), angles, torch.from_numpy(tprev).to(dev)


def test_one_iteration_against_oracle(dev, features):
  window = _tables(dev)[0]
  S, angles, tprev = _state(dev, features)
  S64 = S.cpu().numpy().astype(np.float64)
  a64 = angles.cpu().numpy().astype(np.complex128)
  t64 = tprev.cpu().numpy().astype(np.complex128)
  for momentum in (0.99, 0.0):
    ang, tp = angles.clone()[None], tprev.clone()[None]
    engine.op_griffin_lim_iterate(S[None], window, ang, tp, momentum, 1)
    ref_ang, ref_tp, _, _ = G.gl_iteration64(S64, a64, t64, WIN, momentum)
    tb, ab, mag, angb = G.iteration_bounds(S64, a64, t64, WIN, momentum)
    _ratio('iteration tprev', np.abs(tp[0].cpu().numpy() - ref_tp), tb)
    held = mag > ab
    skipped = int((~held).sum())
    print(f'momentum {momentum}: angles checked at {int(held.sum())} elements, skipped {skipped} '
          f'where |a| is within its bound')
    # the bound is a worst case over the frame's energy: quiet bins of loud frames fall inside it
    assert skipped < 0.5 * held.size
    _ratio('iteration angles', np.abs(ang[0].cpu().numpy() - ref_ang)[held], angb[held])
    # unit modulus wherever |a| is well above the 1e-16 floor
    assert np.allclose(np.abs(ang[0].cpu().numpy())[held], 1.0, atol=1e-6)
    # the bounds above are worst cases over a frame's energy; on the loud bins (within 1 % of
    # their frame's largest) fp32 is held far tighter, which a twiddle or scaling slip would break:
    # an fp32 numpy evaluation of the same iteration stays within 1e-5 relative there
    loud = np.abs(ref_tp) >= 1e-2 * np.abs(ref_tp).max(axis=1, keepdims=True)
    rel = float((np.abs(tp[0].cpu().numpy() - ref_tp)[loud] / np.abs(ref_tp)[loud]).max())
    MAX_RATIO['iteration tprev, loud bins (1e-4 relative)'] = max(
        MAX_RATIO.get('iteration tprev, loud bins (1e-4 relative)', 0.0), rel / 1e-4)
    assert rel <= 1e-4, rel
    a_loud = mag >= 1e-2 * mag.max(axis=1, keepdims=True)
    dang = float(np.abs(ang[0].cpu().numpy() - ref_ang)[a_loud].max())
    MAX_RATIO['iteration angles, loud bins (1e-4)'] = max(
        MAX_RATIO.get('iteration angles, loud bins (1e-4)', 0.0), dang / 1e-4)
    assert dang <= 1e-4, dang


def test_iterations_compose_and_do_not_depend_on_tiling(dev, features):
  window = _tables(dev)[0]
  S, angles, tprev = _state(dev, features, seed=2)
  # two launches in one call (the ping-pong) equal two calls of one (the copy back)
  a1, t1 = angles.clone()[None], tprev.clone()[None]
  a2, t2 = angles.clone()[None], tprev.clone()[None]
  engine.op_griffin_lim_iterate(S[None], window, a1, t1, 0.99, 3)
  for _ in range(3):
    engine.op_griffin_lim_iterate(S[None], window, a2, t2, 0.99, 1)
  assert torch.equal(a1, a2) and torch.equal(t1, t2)
  # frames 17.. of a row alone equal the same frames inside a longer row, away from the new edge:
  # a frame sees its neighbours only, so after one iteration frames 19.. agree bit for bit
  a3, t3 = angles.clone()[None, 17:].contiguous(), tprev.clone()[None, 17:].contiguous()
  engine.op_griffin_lim_iterate(S[None, 17:].contiguous(), window, a3, t3, 0.99, 1)
  a4, t4 = angles.clone()[None], tprev.clone()[None]
  engine.op_griffin_lim_iterate(S[None], window, a4, t4, 0.99, 1)
  assert torch.equal(a3[0, 2:], a4[0, 19:]) and torch.equal(t3[0, 2:], t4[0, 19:])


def test_istft_against_oracle(dev, features):
  window = _tables(dev)[0]
  S, angles, _ = _state(dev, features, seed=3)
  got = engine.op_griffin_lim_istft(S[None], window, angles[None])[0].cpu().numpy()
  S64 = S.cpu().numpy().astype(np.float64)
  a64 = angles.cpu().numpy().astype(np.complex128)
  ref = G.istft64(S64 * a64, WIN)
  assert got.shape == (S.shape[0] * 320,) and got[0] == 0.0
  _ratio('istft', np.abs(got - ref), G.istft_bound(S64, a64, WIN))


def test_whole_decode(dev, features):
  y = audio_codecs.griffin_lim(features, n_iter=32, momentum=0.99, seed=5)
  assert y.dtype == np.float32 and y.shape == (features.shape[0] * 320,)
  ref, S = G.decode64(features, WIN, WEIGHTS, PINV, INV_L, BETA, audio_codecs.NNLS_ITERS, 32, 0.99,
                      seed=5)
  sc_gpu = G.spectral_convergence(y, S, WIN)
  sc_ref = G.spectral_convergence(ref, S, WIN)
  print(f'spectral convergence: gpu {sc_gpu:.5f}, oracle {sc_ref:.5f}')
  assert abs(sc_gpu - sc_ref) <= 0.01 * sc_ref
  codec = audio_codecs.MelGAN()
  enc_gpu = codec.encode(y)
  enc_ref = codec.encode(ref.astype(np.float32))
  # in the log domain, where the oracle's re-encoded mel is above 1e-3 (below, a tiny absolute
  # difference is a large log one)
  audible = enc_ref > np.log(1e-3)
  diff = np.abs(enc_gpu - enc_ref)[audible]
  print(f're-encoded at {int(audible.sum())} audible bins: mean |diff| {diff.mean():.2e} nats, '
        f'max {diff.max():.2e}')
  assert diff.mean() <= 1e-2
  # the decode is near its features: re-encoding gives the frames back, roughly
  assert enc_gpu.shape == features.shape
  loud = features > np.log(1e-2)
  print(f're-encoded vs features where loud: mean |diff| {np.abs(enc_gpu - features)[loud].mean():.3f}')
  # deterministic, and independent of the batch
  np.testing.assert_array_equal(audio_codecs.griffin_lim(features, seed=5), y)
  other = features[::-1].copy()
  batch = audio_codecs.griffin_lim(np.stack([other, features, other + 0.5]), seed=5)
  assert batch.shape == (3, y.shape[0])
  np.testing.assert_array_equal(batch[1], y)
  # a CUDA tensor stays on its device and agrees with the numpy path
  t = audio_codecs.griffin_lim(torch.from_numpy(features).to(dev), seed=5)
  assert t.is_cuda and t.device == dev
  np.testing.assert_array_equal(t.cpu().numpy(), y)
  empty = audio_codecs.griffin_lim(np.zeros((0, 128), np.float32))
  assert empty.shape == (0,)


def test_ops_refuse_bad_arguments(dev):
  lib = _native.load()
  f = torch.zeros(1, 4, 513, dtype=torch.float32, device=dev)
  c = torch.zeros(1, 4, 513, dtype=torch.complex64, device=dev)
  w = torch.zeros(640, dtype=torch.float32, device=dev)
  p = ctypes.c_void_p(f.data_ptr())
  pc = ctypes.c_void_p(c.data_ptr())
  pw = ctypes.c_void_p(w.data_ptr())
  s = ctypes.c_void_p(0)
  null = ctypes.c_void_p(0)
  big = (1 << 31) // 3 + 1
  mag = lib.msd_op_griffin_lim_magnitude
  assert mag(null, 1, 4, p, p, 0.1, p, 1, p, s) == -1
  assert mag(p, 1, 4, p, p, 0.1, null, 1, p, s) == -1
  assert mag(p, -1, 4, p, p, 0.1, p, 1, p, s) == -1
  assert mag(p, 1, -4, p, p, 0.1, p, 1, p, s) == -1
  assert mag(p, 1, 4, p, p, 0.1, p, -1, p, s) == -1
  assert mag(p, 3, big, p, p, 0.1, p, 1, p, s) == -1
  assert mag(p, 0, 4, p, p, 0.1, p, 1, p, s) == 0
  assert mag(p, 1, 0, p, p, 0.1, p, 1, p, s) == 0
  init = lib.msd_op_griffin_lim_init
  assert init(1, 4, 0, null, s) == -1
  assert init(-1, 4, 0, pc, s) == -1 and init(1, -4, 0, pc, s) == -1
  assert init(3, big, 0, pc, s) == -1
  assert init(0, 4, 0, pc, s) == 0 and init(1, 0, 0, pc, s) == 0
  it = lib.msd_op_griffin_lim_iterate
  assert it(p, 1, 4, pw, pc, pc, null, 0.5, 1, s) == -1
  assert it(p, 1, 4, null, pc, pc, pc, 0.5, 1, s) == -1
  assert it(p, 1, 4, pw, pc, pc, pc, -0.5, 1, s) == -1
  assert it(p, 1, 4, pw, pc, pc, pc, float('nan'), 1, s) == -1
  assert it(p, 1, 4, pw, pc, pc, pc, 0.5, -1, s) == -1
  assert it(p, -1, 4, pw, pc, pc, pc, 0.5, 1, s) == -1
  assert it(p, 3, big, pw, pc, pc, pc, 0.5, 1, s) == -1
  assert it(p, 0, 4, pw, pc, pc, pc, 0.5, 1, s) == 0 and it(p, 1, 4, pw, pc, pc, pc, 0.5, 0, s) == 0
  ist = lib.msd_op_griffin_lim_istft
  assert ist(p, null, 1, 4, pw, p, s) == -1
  assert ist(p, pc, 1, -4, pw, p, s) == -1
  assert ist(p, pc, 3, big, pw, p, s) == -1
  assert ist(p, pc, 0, 4, pw, p, s) == 0
  torch.cuda.synchronize()
  with pytest.raises(ValueError):
    engine.op_griffin_lim_iterate(f, w, c, c, -1.0, 1)
  with pytest.raises(ValueError):
    engine.op_griffin_lim_istft(f, w, c.real.contiguous())


def test_synthesized_song_to_wav(dev, tiny):
  t5, params = tiny
  model = _model(t5, params, 1, steps=3)
  out = song.synthesize_song(model, _notes(2.5, 60), seed=1)
  audio = audio_codecs.griffin_lim(out['full_pred_encoded'][:out['num_frames']])
  buf = io.BytesIO()
  song.save_audio(buf, audio)
  back = song.load_audio(buf.getvalue())
  assert back.shape == (out['num_frames'] * 320,)
  assert np.isfinite(back).all()


def test_zz_report_max_error_over_bound():
  assert MAX_RATIO
  for name, r in MAX_RATIO.items():
    print(f'griffin_lim {name}: max err/bound = {r:.4f}')
