"""-m gpu: MelGAN.encode on the CUDA kernel (msd_op_audio_mel) against the fp64 oracle, its
frame invariance, its argument checks, and songs primed with a recording."""
import ctypes

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import _native, audio_codecs, engine, song
from oracle import mel_oracle as MO
from tests.test_gpu_song_batch import C, _model, _nseg, _notes, tiny  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

SR = 16000
WIN = audio_codecs.hann_window()
WEIGHTS = audio_codecs.linear_to_mel_weight_matrix()
MAX_RATIO = []   # err / bound of every checked element set, reported by the last test


def _floor(device):
  """logf(1e-5f) as the device computes it."""
  return torch.log(torch.tensor(1e-5, dtype=torch.float32, device=device)).item()


def _check_against_oracle(x, got, device, weights=WEIGHTS):
  """got [F, 128] (the kernel's log-mels of x [n]) against the fp64 oracle with the same float32
  tables.  In the linear domain, |exp(out) - clip(m64)| <= bound (MO.error_bound) wherever the
  kernel did not clip to the floor; where it did, the oracle is within the bound of the floor, and
  wherever the oracle is further below the floor than the bound, out is exactly logf(1e-5f)."""
  got = np.asarray(got, np.float64)
  m64 = MO.mel_linear64(x, WIN, weights)
  bound = MO.error_bound(x, WIN, weights)
  assert got.shape == m64.shape
  assert np.isfinite(got).all()
  floor = _floor(device)
  at_floor = got == floor
  ratio = np.abs(np.exp(got) - np.clip(m64, *MO.CLIP)) / bound
  r = float(ratio[~at_floor].max()) if (~at_floor).any() else 0.0
  MAX_RATIO.append(r)
  assert r < 1.0, r
  assert (m64[at_floor] <= MO.CLIP[0] + bound[at_floor]).all()
  assert at_floor[m64 < MO.CLIP[0] - bound].all()
  return r


def _signals(n, seed=0):
  rng = np.random.default_rng(seed)
  t = np.arange(n) / SR
  sig = {f'noise{s:g}': s * rng.uniform(-1, 1, n) for s in (1e-6, 1e-3, 1.0)}
  sig['tone440'] = np.sin(2 * np.pi * 440 * t)
  sig['tone3k'] = 0.3 * np.sin(2 * np.pi * 3000 * t + 0.2)
  sig['chirp'] = np.sin(2 * np.pi * (50 * t + 700 * t * t))
  imp = np.zeros(n)
  imp[[100, 5000, n // 2]] = [1.0, -0.5, 0.25]
  sig['impulse'] = imp
  sig['clipped'] = np.clip(3 * np.sin(2 * np.pi * 220 * t), -1, 1)
  mixed = rng.normal(0, 0.1, n)
  mixed[n // 4:n // 2] = 0.0   # a silent stretch
  sig['silent_stretch'] = mixed
  return {k: v.astype(np.float32) for k, v in sig.items()}


def test_accuracy_on_test_signals(cuda_device):
  codec = audio_codecs.MelGAN()
  for name, x in _signals(SR * 4 + 123).items():
    got = codec.encode(x)
    assert isinstance(got, np.ndarray) and got.dtype == np.float32
    _check_against_oracle(x, got, cuda_device)
  # silence: exactly the floor everywhere
  silent = codec.encode(np.zeros(SR, np.float32))
  assert silent.shape == (50, 128)
  assert (silent == np.float32(_floor(cuda_device))).all()


@pytest.mark.parametrize('n', [0, 1, 319, 320, 321, 641])
def test_lengths(cuda_device, n):
  x = np.random.default_rng(n).uniform(-1, 1, n).astype(np.float32)
  got = audio_codecs.MelGAN().encode(x)
  assert got.shape == (MO.num_frames(n), 128)
  if n:
    _check_against_oracle(x, got, cuda_device)
  t = audio_codecs.MelGAN().encode(torch.from_numpy(x).to(cuda_device))
  assert t.is_cuda and t.shape == (MO.num_frames(n), 128)
  assert np.array_equal(t.cpu().numpy(), got)
  assert audio_codecs.MelGAN().encode(np.zeros((3, n), np.float32)).shape == (3, MO.num_frames(n), 128)


def test_ten_minutes(cuda_device):
  n = SR * 600 + 77
  rng = np.random.default_rng(10)
  envelope = 10.0 ** rng.uniform(-6, 0, n // SR + 1).repeat(SR)[:n]
  x = (envelope * rng.uniform(-1, 1, n)).astype(np.float32)
  got = audio_codecs.MelGAN().encode(torch.from_numpy(x).to(cuda_device))
  assert got.shape == (30001, 128)
  _check_against_oracle(x, got.cpu().numpy(), cuda_device)


def test_rows_equal_single_rows_bitwise(cuda_device):
  """2-D input: each row is encoded as it is alone (a frame does not depend on row or batch)."""
  sig = list(_signals(SR * 2 + 5, seed=2).values())
  batch = np.stack(sig)
  got = audio_codecs.MelGAN().encode(batch)
  assert got.shape == (len(sig), MO.num_frames(batch.shape[1]), 128)
  for r, x in enumerate(sig):
    assert np.array_equal(got[r], audio_codecs.MelGAN().encode(x)), r
  dev = audio_codecs.MelGAN().encode(torch.from_numpy(batch).to(cuda_device))
  assert dev.is_cuda and np.array_equal(dev.cpu().numpy(), got)


def test_whole_song_equals_per_segment_encodes_bitwise(cuda_device):
  codec = audio_codecs.MelGAN()
  model = type('M', (), {'audio_codec': codec, 'sequence_length': {'targets': 256}})()
  for n in (320 * 256 * 3 + 4321, 320 * 256 * 2 - 320, 320 * 256 * 2):
    x = np.random.default_rng(n).normal(0, 0.2, n).astype(np.float32)
    got = song.encode_song_audio(model, x)
    want, total = MO.encode_song_by_segments(x, codec.encode)
    assert got['num_frames'] == total
    assert want.dtype == np.float32
    assert np.array_equal(got['full_gt_encoded'], want), n


def test_shift_by_whole_hops_shifts_the_frames(cuda_device):
  codec = audio_codecs.MelGAN()
  x = np.random.default_rng(3).normal(0, 0.3, SR * 3 + 211).astype(np.float32)
  ref = codec.encode(x)
  for k in (1, 7, 300):
    y = np.concatenate([np.random.default_rng(k).normal(0, 0.3, 320 * k).astype(np.float32), x])
    assert np.array_equal(codec.encode(y)[k:], ref), k


def test_output_past_the_written_frames_is_untouched(cuda_device):
  rows, n = 3, 320 * 40 + 9
  audio = torch.randn(rows, n, device=cuda_device)
  win, weights = audio_codecs.mel_tables(cuda_device)
  frames = MO.num_frames(n)
  want = engine.op_audio_mel(audio, win, weights)
  out = torch.full((rows * frames * 128 + 4096,), -12345.0, device=cuda_device)
  lib = _native.load()
  assert lib.msd_op_audio_mel(ctypes.c_void_p(audio.data_ptr()), rows, n,
                              ctypes.c_void_p(win.data_ptr()), ctypes.c_void_p(weights.data_ptr()),
                              ctypes.c_void_p(out.data_ptr()), None) == 0
  torch.cuda.synchronize()
  assert torch.equal(out[:rows * frames * 128].view(rows, frames, 128), want)
  assert (out[rows * frames * 128:] == -12345.0).all()


def test_a_table_too_wide_for_shared_memory(cuda_device):
  """A dense filterbank (every weight non-zero) is read from global memory: same arithmetic."""
  w = np.random.default_rng(4).uniform(0.01, 1.0, (513, 128)).astype(np.float32)
  x = np.random.default_rng(5).normal(0, 0.3, SR).astype(np.float32)
  win, _ = audio_codecs.mel_tables(cuda_device)
  got = engine.op_audio_mel(torch.from_numpy(x)[None].to(cuda_device), win,
                            torch.from_numpy(w).to(cuda_device))[0].cpu().numpy()
  _check_against_oracle(x, got, cuda_device, weights=w)


def test_wrapper_and_entry_point_refuse_bad_arguments(cuda_device):
  win, weights = audio_codecs.mel_tables(cuda_device)
  good = torch.zeros(2, 1000, device=cuda_device)
  for bad in (good.double(), good[:, ::2], good.cpu(), good[0]):
    with pytest.raises(ValueError):
      engine.op_audio_mel(bad, win, weights)
  with pytest.raises(ValueError):
    engine.op_audio_mel(good, win[:320], weights)
  with pytest.raises(ValueError):
    engine.op_audio_mel(good, win, weights.t().contiguous())
  with pytest.raises(ValueError):
    audio_codecs.MelGAN().encode(torch.zeros(1000))
  lib = _native.load()
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  out = torch.empty(2, 4, 128, device=cuda_device)
  assert lib.msd_op_audio_mel(None, 2, 1000, p(win), p(weights), p(out), None) == -1
  assert lib.msd_op_audio_mel(p(good), 2, 1000, p(win), None, p(out), None) == -1
  assert lib.msd_op_audio_mel(p(good), -1, 1000, p(win), p(weights), p(out), None) == -1
  assert lib.msd_op_audio_mel(p(good), 2, -5, p(win), p(weights), p(out), None) == -1
  # 2^16 rows x 2^16 frames: more output frames than int32 can count (refused before any launch)
  assert lib.msd_op_audio_mel(p(good), 1 << 16, 320 << 16, p(win), p(weights), p(out), None) == -1
  assert b'2^31' in lib.msd_last_error()
  torch.cuda.synchronize()


# ---- songs primed with a recording (tiny config, C = 128 context frames) ----------------------
def _recording(n, seed):
  t = np.arange(n) / SR
  rng = np.random.default_rng(seed)
  return (0.4 * np.sin(2 * np.pi * 330 * t) + rng.normal(0, 0.05, n)).astype(np.float32)


def test_primed_song_equals_the_chain_driven_by_hand(cuda_device, tiny):
  t5, params = tiny
  model = _model(t5, params, 1)
  notes = _notes(4.0, 60)
  lengths = model.sequence_length
  for n in (320 * 60 + 123, SR * 5):   # context shorter than C, and a full C frames
    a = _recording(n, n)
    got = song.synthesize_song(model, notes, seed=3, context_audio=a)
    mel = audio_codecs.MelGAN().encode(a)
    first, count = song.primer_frames(n, C)
    assert count == min(C, n // 320 - 1)
    pred = np.zeros((1, C, 128), np.float32)
    pred[0, :count] = mel[first:first + count]
    mask = np.zeros((1, C), np.int32)
    mask[0, :count] = 1
    toks = got['tokens']
    full = []
    for i in range(len(toks)):
      pred, _ = model.predict({
          'encoder_input_tokens': toks[i:i + 1], 'encoder_continuous_inputs': pred,
          'encoder_continuous_mask': mask if i == 0 else np.ones((1, C), np.int32),
          'decoder_target_tokens': np.zeros((1, lengths['targets'], 128), np.float32)}, seed=3)
      full.append(pred[0])
    assert np.array_equal(got['full_pred_encoded'], np.concatenate(full)), n
    plain = song.synthesize_song(model, notes, seed=3)
    n_t = lengths['targets']
    assert not np.array_equal(got['full_pred_encoded'][:n_t], plain['full_pred_encoded'][:n_t])
  with pytest.raises(ValueError):
    song.synthesize_song(model, notes, context_audio=np.zeros(639, np.float32))
  with pytest.raises(ValueError):
    song.synthesize_song(model, notes, always_mask_context=True, context_audio=_recording(SR, 1))


def test_primed_songs_at_batch1_equal_synthesize_song(cuda_device, tiny):
  t5, params = tiny
  model = _model(t5, params, 1)
  notes = [_notes(4.0, 60), _notes(2.2, 62), _notes(6.5, 64)]
  audios = [_recording(SR * 3, 1), None, _recording(320 * 10 + 7, 2)]
  seeds = [4, 5, 31337]
  results, agg = song.synthesize_songs(model, notes, seeds, context_audios=audios)
  assert agg['segments'] == sum(_nseg(model, n) for n in notes)
  for r, n, a, s in zip(results, notes, audios, seeds):
    want = song.synthesize_song(model, n, seed=s, context_audio=a)
    np.testing.assert_array_equal(r['full_pred_encoded'], want['full_pred_encoded'])
  plain, _ = song.synthesize_songs(model, notes, seeds)
  np.testing.assert_array_equal(plain[1]['full_pred_encoded'], results[1]['full_pred_encoded'])
  assert not np.array_equal(plain[0]['full_pred_encoded'], results[0]['full_pred_encoded'])
  with pytest.raises(ValueError):
    song.synthesize_songs(model, notes, seeds, context_audios=audios[:2])
  with pytest.raises(ValueError):
    song.synthesize_songs(model, notes, seeds, always_mask_context=True, context_audios=audios)


def test_zz_report_max_error_over_bound():
  assert MAX_RATIO
  print(f'audio_mel: max err/bound over {len(MAX_RATIO)} checks = {max(MAX_RATIO):.4f}')
