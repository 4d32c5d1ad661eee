"""-m gpu: per-row noise streams (msd_sample_rows) and the multi-song driver on the CUDA engine."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import config, engine, inference, song, weights
from music_spectrogram_diffusion_b200 import midi_tokens as M
from tests import helpers as H

pytestmark = pytest.mark.gpu

T = N = C = 128
SEEDS3 = (0, 31337, (9 << 32) | 5)


@pytest.fixture(scope='module')
def tiny():
  t5 = config.t5_tiny()
  return t5, weights.synthetic_params(t5, T, N, C, seed=0)


def _engine(t5, params, B, steps, rng='jax', precision='bf16', lengths=(T, N, C)):
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = steps
  diff.classifier_free_guidance.eval_condition_weight = 2.0
  eng = engine.Engine(engine.make_msd_config(t5, diff, *lengths, max_batch=B, rng=rng,
                                             precision=precision), 0)
  eng.load_weights(params)
  return eng


def _encode(eng, toks, ctx, cmask, device):
  b = H.torch_batch(toks, ctx, cmask, device)
  eng.encode(b['encoder_input_tokens'], b['encoder_continuous_inputs'], b['encoder_continuous_mask'])


def _per_row_jax_draws(seeds, steps, n_row, device):
  """init_z [B, n_row] and noise [steps, B, n_row]: row b is seeds[b]'s own batch-1 draw."""
  z0 = torch.stack([engine.op_jax_normal(s, -1, n_row, device) for s in seeds])
  noise = torch.stack([torch.stack([engine.op_jax_normal(s, i, n_row, device) for s in seeds])
                       for i in range(steps)])
  return z0, noise


def _check_rows_follow_their_own_jax_streams(eng, seeds, steps, n_frames, device):
  shape = (len(seeds), n_frames, 128)
  got = eng.sample_rows(seeds).clone()
  z0, noise = _per_row_jax_draws(seeds, steps, n_frames * 128, device)
  want = eng.sample(z0.view(shape).contiguous(), noise.view((steps,) + shape).contiguous()).clone()
  assert torch.isfinite(got).all()
  assert torch.equal(got, want), (got - want).abs().max().item()


@pytest.mark.parametrize('precision', ['bf16', 'fp32_accurate'])
def test_per_row_noise_is_each_seeds_batch1_jax_stream(cuda_device, tiny, precision):
  """Row b of sample_rows(seeds) == sample() with row b of init_z = normal(PRNGKey(seeds[b]),
  [N*128]) and row b of noise[i] = normal(fold_in(PRNGKey(seeds[b]), i), [N*128]) injected."""
  t5, params = tiny
  steps = 6
  eng = _engine(t5, params, 3, steps, precision=precision)
  _encode(eng, *H.make_batch(3, T, C), cuda_device)
  _check_rows_follow_their_own_jax_streams(eng, SEEDS3, steps, N, cuda_device)
  # the per-row key tables are rebuilt when the seeds change (and kept when they do not)
  _check_rows_follow_their_own_jax_streams(eng, (5, 0, 31337), steps, N, cuda_device)
  _check_rows_follow_their_own_jax_streams(eng, (5, 0, 31337), steps, N, cuda_device)
  eng.close()


def test_per_row_noise_at_base_size(cuda_device):
  """The same property on base_with_context (256 frames, 2048 tokens), 3 rows."""
  t5 = config.t5_base()
  lengths = config.TASK_FEATURE_LENGTHS_CONTEXT
  Tb, Nb, Cb = lengths['inputs'], lengths['targets'], lengths['targets_context']
  params = weights.synthetic_params(t5, Tb, Nb, Cb, seed=0)
  steps = 4
  eng = _engine(t5, params, 3, steps, lengths=(Tb, Nb, Cb))
  _encode(eng, *H.make_batch(3, Tb, Cb, seed=3), cuda_device)
  _check_rows_follow_their_own_jax_streams(eng, SEEDS3, steps, Nb, cuda_device)
  eng.close()


@pytest.mark.parametrize('rng', ['jax', 'philox'])
def test_batch1_per_row_sampling_is_msd_sample(cuda_device, tiny, rng):
  t5, params = tiny
  steps = 5
  eng = _engine(t5, params, 3, steps, rng=rng)
  toks, ctx, cmask = H.make_batch(1, T, C, seed=2)
  _encode(eng, toks, ctx, cmask, cuda_device)
  for s in SEEDS3:
    a = eng.sample_rows([s]).clone()
    b = eng.sample(seed=s).clone()
    assert torch.equal(a, b), (rng, s)
  # B identical rows under one repeated seed are identical; one seed over the batch is not
  rep = lambda a: np.repeat(a, 3, axis=0)
  _encode(eng, rep(toks), rep(ctx), rep(cmask), cuda_device)
  rows = eng.sample_rows([7, 7, 7]).clone()
  assert torch.equal(rows[0], rows[1]) and torch.equal(rows[0], rows[2])
  one = eng.sample(seed=7).clone()   # right after sample_rows: back on the whole-batch stream
  assert not torch.equal(one[0], one[1]) and not torch.equal(one[1], one[2])
  eng.close()


@pytest.mark.parametrize('rng', ['jax', 'philox'])
def test_rows_are_independent(cuda_device, tiny, rng):
  """Changing row 2's tokens, context and seed leaves the other rows bit-identical; permuting the
  rows permutes the output bit-identically."""
  t5, params = tiny
  steps = 6
  eng = _engine(t5, params, 4, steps, rng=rng)
  toks, ctx, cmask = H.make_batch(4, T, C, seed=5, ctx_masks=[0, 1, 1, 0])
  seeds = [3, 11, 29, (1 << 40) + 2]
  _encode(eng, toks, ctx, cmask, cuda_device)
  base = eng.sample_rows(seeds).clone()
  t2, c2, m2 = H.make_batch(4, T, C, seed=6, ctx_masks=[1, 1, 0, 1])
  toks_b, ctx_b, cmask_b = toks.copy(), ctx.copy(), cmask.copy()
  toks_b[2], ctx_b[2], cmask_b[2] = t2[2], c2[2], m2[2]
  _encode(eng, toks_b, ctx_b, cmask_b, cuda_device)
  changed = eng.sample_rows([seeds[0], seeds[1], 12345, seeds[3]]).clone()
  assert not torch.equal(changed[2], base[2])
  for r in (0, 1, 3):
    assert torch.equal(changed[r], base[r]), r
  for perm in ([3, 2, 1, 0], [1, 3, 0, 2], [2, 0, 3, 1]):
    _encode(eng, toks[perm], ctx[perm], cmask[perm], cuda_device)
    got = eng.sample_rows([seeds[p] for p in perm]).clone()
    assert torch.equal(got, base[perm]), perm
  eng.close()


def test_sample_rows_refusals(cuda_device, tiny):
  t5, params = tiny
  eng = _engine(t5, params, 2, 3)
  out = torch.empty(2, N, 128, device=cuda_device)
  seeds = (ctypes.c_uint64 * 2)(1, 2)
  assert eng.lib.msd_sample_rows(eng._h, seeds, ctypes.c_void_p(out.data_ptr()), None) == -1
  assert b'msd_encode' in eng.lib.msd_last_error()
  _encode(eng, *H.make_batch(2, T, C), cuda_device)
  assert eng.lib.msd_sample_rows(eng._h, None, ctypes.c_void_p(out.data_ptr()), None) == -1
  assert eng.lib.msd_sample_rows(eng._h, seeds, None, None) == -1
  with pytest.raises(ValueError):
    eng.sample_rows([1, 2, 3])
  eng.close()


def _model(t5, params, slots, steps=5):
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = steps
  diff.classifier_free_guidance.eval_condition_weight = 2.0
  lengths = {'inputs': T, 'targets': N, 'targets_context': C}
  return inference.InferenceModel.from_config(t5, diff, lengths, 'synthetic:0', slots,
                                              params=params)


def _notes(seconds, pitch):
  return M.make_notes([(0.1, seconds - 0.3, pitch, 100, 0, False),
                       (0.7, 1.2, pitch + 7, 90, 41, False), (1.0, 1.3, 38, 110, 0, True)])


def _nseg(model, notes):
  return song._tokenize(model, notes, None)[1]


def test_predict_on_device_with_seeds(cuda_device, tiny):
  t5, params = tiny
  model = _model(t5, params, 2)
  toks, ctx, cmask = (torch.from_numpy(a).to(cuda_device) for a in H.make_batch(2, T, C))
  with pytest.raises(ValueError):
    model.predict_on_device(toks, ctx, cmask, seeds=[1])
  with pytest.raises(ValueError):
    model.predict_on_device(toks, ctx, cmask, seeds=[1, 2], init_z=torch.zeros(2, N, 128))
  got = model.predict_on_device(toks, ctx, cmask, seeds=[1, 2])
  assert got.shape == (2, N, 128)
  assert torch.equal(got, model.engine.sample_rows([1, 2]))
  # without seeds: unchanged (one seed over the whole batch)
  assert torch.equal(model.predict_on_device(toks, ctx, cmask, seed=4),
                     model.engine.sample(seed=4))


def test_songs_at_batch1_are_the_single_song_chains(cuda_device, tiny):
  t5, params = tiny
  model = _model(t5, params, 1)
  a, b = _notes(4.0, 60), _notes(6.5, 64)
  assert (_nseg(model, a), _nseg(model, b)) == (2, 3)
  results, agg = song.synthesize_songs(model, [a, b], seeds=[4, 31337])
  assert agg['rounds'] == 5 and agg['segments'] == 5 and agg['x_realtime'] > 0
  for r, notes, s in ((results[0], a, 4), (results[1], b, 31337)):
    want = song.synthesize_song(model, notes, seed=s)
    np.testing.assert_array_equal(r['full_pred_encoded'], want['full_pred_encoded'])
    np.testing.assert_array_equal(r['tokens'], want['tokens'])
    assert r['num_frames'] == want['num_frames']
    assert r['model_timing']['prediction_seconds_per_chunk'] > 0


def test_song_order_does_not_change_any_song(cuda_device, tiny):
  """4 slots, 4 songs of 2 segments: every order of the songs gives each song the same bits."""
  t5, params = tiny
  model = _model(t5, params, 4, steps=4)
  notes = [_notes(4.0, 60 + 3 * k) for k in range(4)]
  assert all(_nseg(model, n) == 2 for n in notes)
  seeds = [0, 9, 0, (3 << 32) | 1]
  ref = None
  for perm in itertools.permutations(range(4)):
    results, agg = song.synthesize_songs(model, [notes[p] for p in perm], [seeds[p] for p in perm])
    assert agg['rounds'] == 2
    got = {p: r['full_pred_encoded'] for p, r in zip(perm, results)}
    if ref is None:
      ref = got
      assert not np.array_equal(ref[0], ref[2])   # same seed, different notes
      continue
    for p in range(4):
      np.testing.assert_array_equal(got[p], ref[p], err_msg=str(perm))


def test_batched_songs_follow_their_batch1_chains(cuda_device, tiny):
  """2 slots, songs of 2, 1 and 3 segments against each song alone at batch 1: the noise is the
  same, only batch-size dependent kernel choices differ."""
  t5, params = tiny
  steps = 20
  batched = _model(t5, params, 2, steps)
  single = _model(t5, params, 1, steps)
  notes = [_notes(4.0, 60), _notes(2.2, 62), _notes(6.5, 64)]
  assert [_nseg(batched, n) for n in notes] == [2, 1, 3]
  seeds = [5, 6, 7]
  results, agg = song.synthesize_songs(batched, notes, seeds)
  assert agg['rounds'] == 4 and agg['segments'] == 6
  span = 4.0 - np.log(1e-5)
  for k, (r, n, s) in enumerate(zip(results, notes, seeds)):
    want = song.synthesize_song(single, n, seed=s)['full_pred_encoded']
    assert r['full_pred_encoded'].shape == want.shape
    err = np.abs(r['full_pred_encoded'] - want) / span * 2.0
    H.assert_trajectory_close(err, f'song {k} batched with 2 slots vs alone')
