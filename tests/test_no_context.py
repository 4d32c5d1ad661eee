"""CPU: the no-context diffusion model (models.DiffusionModel + network.Transformer) -- gin surface,
parameter tree, its oracle against the context model's, and the song scheduling of independent
segments, driven by a stand-in predict function."""
import os
import types

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import (audio_codecs, config, engine, inference, song,
                                              weights)
from music_spectrogram_diffusion_b200 import midi_tokens as M
from oracle import msd_oracle as O
from tests import helpers as H
from tests import no_context_oracle as NC

HERE = os.path.dirname(os.path.abspath(__file__))
GIN = os.path.join(HERE, 'golden', 'base_no_context.gin')
GIN_CONTEXT = os.path.join(HERE, 'golden', 'base_with_context.gin')
REF_ROOT = os.path.join(HERE, 'golden', 'reference_gin')


# ---- gin -----------------------------------------------------------------------------------
def test_gin_fixture_builds_the_no_context_surface():
  m = inference.InferenceModel('synthetic:0', inference.parse_training_gin_file(GIN, []),
                               batch_size=3)
  assert m.sequence_length == {'inputs': 2048, 'targets': 256}
  assert (m.inputs_length, m.targets_length) == (2048, 256)
  assert m.targets_context_length is None and not m.has_context
  # inference.py:113-157: no continuous inputs; decoder_input_tokens because the no-context
  # feature converter lists it
  assert m.input_shapes == {'encoder_input_tokens': (3, 2048), 'decoder_target_tokens': (3, 256, 128),
                            'decoder_input_tokens': (3, 256, 128)}
  assert m.input_types == {'encoder_input_tokens': np.int32, 'decoder_target_tokens': np.float32,
                           'decoder_input_tokens': np.float32}
  assert set(m.model.FEATURE_CONVERTER_CLS.MODEL_FEATURES) == {
      'encoder_input_tokens', 'decoder_target_tokens', 'decoder_input_tokens', 'decoder_target_mask'}
  assert set(m.model.FEATURE_CONVERTER_CLS.TASK_FEATURES) == {'inputs', 'targets'}
  t5 = m.model.module_config
  assert (t5.vocab_size, t5.emb_dim, t5.num_heads, t5.num_decoder_layers) == (1536, 768, 12, 12)
  assert t5.decoder_cross_attend_style == 'concat_encodings'
  cfg = engine.make_msd_config(t5, m.model.diffusion_config, 2048, 256, m.targets_context_length, 3)
  assert cfg.context_length == 0 and cfg.inputs_length == 2048


def _ref_gin(model_file, task_file):
  return (f"include 'music_spectrogram_diffusion/gin/models/diffusion/{model_file}'\n"
          f"include 'music_spectrogram_diffusion/gin/tasks/mt3/{task_file}'\n")


@pytest.mark.parametrize('size', ['t5_small', 't5_base'])
def test_stored_basic_gins_resolve_to_the_no_context_model(monkeypatch, size):
  monkeypatch.setattr(inference, '_GIN_SEARCH_ROOTS', [REF_ROOT])
  m = inference.InferenceModel('synthetic:0', _ref_gin(f'basic/{size}.gin', 'mega.gin'))
  want = getattr(config, size)()
  t5 = m.model.module_config
  assert (t5.emb_dim, t5.num_heads, t5.num_encoder_layers, t5.num_decoder_layers, t5.mlp_dim) == (
      want.emb_dim, want.num_heads, want.num_encoder_layers, want.num_decoder_layers, want.mlp_dim)
  assert m.sequence_length == {'inputs': 2048, 'targets': 256}
  assert m.targets_context_length is None
  assert 'encoder_continuous_inputs' not in m.input_shapes
  # the context family next to it still takes a context
  c = inference.InferenceModel('synthetic:0', _ref_gin(f'context/{size}.gin', 'context_mega.gin'))
  assert c.targets_context_length == 256 and c.has_context


def test_mismatched_model_and_lengths_raise(monkeypatch):
  extra = "TASK_FEATURE_LENGTHS = {'inputs': 2048, 'targets': 256, 'targets_context': 256}"
  with pytest.raises(ValueError, match='DiffusionModel') as e:
    inference.InferenceModel('synthetic:0', inference.parse_training_gin_file(GIN, [extra]))
  assert 'ContextDiffusionModel' in str(e.value) and 'models.DiffusionModel' in str(e.value)
  extra = "TASK_FEATURE_LENGTHS = {'inputs': 2048, 'targets': 256}"
  with pytest.raises(ValueError, match='ContextDiffusionModel') as e:
    inference.InferenceModel('synthetic:0', inference.parse_training_gin_file(GIN_CONTEXT, [extra]))
  assert 'models.DiffusionModel' in str(e.value)
  monkeypatch.setattr(inference, '_GIN_SEARCH_ROOTS', [REF_ROOT])
  with pytest.raises(ValueError):
    inference.InferenceModel('synthetic:0', _ref_gin('basic/t5_small.gin', 'context_mega.gin'))
  with pytest.raises(ValueError):
    inference.InferenceModel('synthetic:0', _ref_gin('context/t5_small.gin', 'mega.gin'))


def test_from_config_without_targets_context():
  m = inference.InferenceModel.from_config(config.t5_tiny(), config.DiffusionConfig(),
                                           {'inputs': 128, 'targets': 128}, batch_size=2)
  assert m.targets_context_length is None
  assert set(m.input_shapes) == {'encoder_input_tokens', 'decoder_target_tokens',
                                 'decoder_input_tokens'}


def test_library_accepts_context_length_zero():
  """msd_step_table validates a configuration as msd_create does: context_length 0 is accepted, a
  negative one refused; the sampler table does not depend on it."""
  from music_spectrogram_diffusion_b200 import _native
  t5, d = config.t5_base(), config.DiffusionConfig()
  for ctx in (0, None):
    assert engine.make_msd_config(t5, d, 2048, 256, ctx, 1).context_length == 0
  with_ctx = engine.step_table_for(engine.make_msd_config(t5, d, 2048, 256, 256, 1))
  np.testing.assert_array_equal(engine.step_table_for(engine.make_msd_config(t5, d, 2048, 256, 0, 1)),
                                with_ctx)
  bad = engine.make_msd_config(t5, d, 2048, 256, 0, 1)
  bad.context_length = -128
  with pytest.raises(_native.MsdError, match='context_length'):
    engine.step_table_for(bad)


# ---- parameter tree ----------------------------------------------------------------------------
@pytest.mark.parametrize('style', ['concat_encodings', 'sum_cross_attends'])
def test_parameter_tree(style):
  """The context trees (411,665,664 base / 104,035,840 small) minus their context encoders
  (85,248,768 / 19,079,680), for either cross-attention style."""
  for make, total, with_ctx in ((config.t5_base, 326_416_896, 411_665_664),
                                (config.t5_small, 84_956_160, 104_035_840)):
    t5 = make()
    t5.decoder_cross_attend_style = style
    for ctx in (0, None):
      shapes = weights.param_shapes(t5, 2048, 256, ctx)
      assert weights.num_params(shapes) == total
    if style == 'concat_encodings':
      assert weights.num_params(weights.param_shapes(t5, 2048, 256, 256)) == with_ctx
    names = [n for n, _ in shapes]
    assert len(set(names)) == len(names)
    assert 'encoder/layers_0/attention/query/kernel' in names
    assert 'encoder/token_embedder/embedding' in names and 'encoder/encoder_norm/scale' in names
    assert 'decoder/layers_0/MultiHeadDotProductAttention_0/key/kernel' in names
    assert not any(n.startswith(('token_encoder/', 'continuous_encoder/')) for n in names)
    assert not any('MultiHeadDotProductAttention_1' in n for n in names)


def test_synthetic_and_checked_trees():
  t5 = config.t5_tiny()
  p = weights.synthetic_params(t5, 128, 128, None, seed=2)
  q = weights.synthetic_params(t5, 128, 128, 0, seed=2)
  assert p.keys() == q.keys() and all(np.array_equal(p[k], q[k]) for k in p)
  assert set(p) == {n for n, _ in weights.param_shapes(t5, 128, 128, 0)}
  weights.check_params(p, t5, 128, 128, None)
  with pytest.raises(ValueError, match='missing encoder/'):
    weights.check_params(weights.synthetic_params(t5, 128, 128, 128), t5, 128, 128, None)
  # existing calls are unchanged: the default is the context tree
  assert 'continuous_encoder/input_proj/kernel' in weights.synthetic_params(t5, 128, 128)


# ---- the oracle: the no-context model is the context model with a masked-out context -------------
T = N = C = 128


@pytest.mark.parametrize('style', ['concat_encodings', 'sum_cross_attends'])
def test_oracle_equals_context_model_with_masked_context(style):
  """fp64: a context model given an all-zero context mask and the same weights computes what the
  no-context model does.  Masked keys get a -1e10 bias, so their exp is exactly 0, and
  sum_cross_attends zeroes the fully masked source."""
  t5 = config.t5_tiny()
  t5.decoder_cross_attend_style = style
  steps, B = 4, 2
  nc = weights.synthetic_params(t5, T, N, None, seed=3)
  ctx_tree = NC.as_context_tree(nc, weights.synthetic_params(t5, T, N, C, seed=4))
  assert set(ctx_tree) == {n for n, _ in weights.param_shapes(t5, T, N, C)}
  Pn, Pc = O.params_to(nc, torch.float64), O.params_to(ctx_tree, torch.float64)
  oc = H.oracle_config(t5, steps, 2.0)
  toks, ctx, _ = H.make_batch(B, T, C)
  cmask = np.zeros((B, C), np.int32)
  batch = {k: v for k, v in H.torch_batch(toks, ctx, cmask).items()}
  batch['encoder_continuous_inputs'] = batch['encoder_continuous_inputs'].to(torch.float64)
  enc_n = NC.encode(Pn, oc, batch['encoder_input_tokens'], torch.float64)
  enc_c = O.encode(Pc, oc, batch['encoder_input_tokens'],
                   O.scale_features(batch['encoder_continuous_inputs'], oc, clip=True),
                   batch['encoder_continuous_mask'])
  assert len(enc_n) == 1
  assert torch.equal(enc_n[0][0], enc_c[0][0]) and torch.equal(enc_n[0][1], enc_c[0][1])

  def rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()

  z = torch.randn(B, N, 128, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
  for flag in (1.0, 0.0):
    t = torch.full((B,), 0.75, dtype=torch.float64)
    got = O.decode(Pn, oc, [(e * flag, m * flag) for e, m in enc_n], z, t)
    want = O.decode(Pc, oc, [(e * flag, m * flag) for e, m in enc_c], z, t)
    assert rel(got, want) <= 1e-12, (flag, rel(got, want))
  init_z, noise = (x.to(torch.float64) for x in H.make_noise(steps, B, N))
  got, scores = NC.predict_batch_with_aux(Pn, oc, batch, init_z, noise)
  want, _ = O.predict_batch_with_aux(Pc, oc, batch, init_z, noise)
  assert got.shape == (B, N, 128) and not scores.any()
  assert rel(got, want) <= 1e-12, rel(got, want)


# ---- song scheduling ---------------------------------------------------------------------------
FRAMES, DIMS, INPUTS = 8, 4, 16
LENGTHS = [3, 1, 4, 2, 2]


class FakeSegments:
  """Row r of the output depends on row r of the tokens and seeds[r] only."""

  def __init__(self, frames=FRAMES, dims=DIMS, clock=None):
    self.frames, self.dims, self.clock = frames, dims, clock
    self.calls = []

  def __call__(self, toks, seeds):
    assert toks.dtype == torch.int32 and toks.shape[0] == len(seeds)
    self.calls.append((toks.clone(), list(seeds)))
    if self.clock is not None:
      self.clock.advance(len(self.calls))   # round k takes k + 1 seconds
    tok = (toks.long().sum(1) % 97).to(torch.float32)[:, None, None]
    sd = torch.tensor([float(s % 1013) for s in seeds])[:, None, None]
    pos = torch.arange(self.frames * self.dims, dtype=torch.float32).view(1, self.frames, self.dims)
    return torch.tanh(0.01 * tok + 0.001 * sd + 1e-3 * pos)


def _songs(lengths, seed=0):
  rng = np.random.default_rng(seed)
  return [torch.from_numpy(rng.integers(3, 1000, (n, INPUTS)).astype(np.int32)) for n in lengths]


@pytest.mark.parametrize('slots', [1, 3, 5, 12, 20])
def test_rounds_rows_seeds_and_reassembly(slots):
  segs = _songs(LENGTHS)
  seeds = [0, 7, 31337, (9 << 32) | 5, 7]
  fake = FakeSegments()
  mels, rounds = song.batch_segments(fake, segs, slots, DIMS, torch.device('cpu'), seeds)
  total = sum(LENGTHS)
  assert len(rounds) == len(fake.calls) == -(-total // slots)
  order = [(s, k) for s, n in enumerate(LENGTHS) for k in range(n)]
  assert [r for rd in rounds for r in rd['rows']] == order
  assert all(len(rd['rows']) == slots for rd in rounds[:-1])
  for rd, (toks, call_seeds) in zip(rounds, fake.calls):
    assert call_seeds == [seeds[s] for s, _ in rd['rows']]
    assert torch.equal(toks, torch.stack([segs[s][k] for s, k in rd['rows']]))
    assert rd['seconds'] >= 0
  for s, n in enumerate(LENGTHS):
    want = torch.cat([FakeSegments()(segs[s][k:k + 1], [seeds[s]]) for k in range(n)], dim=1)
    assert mels[s].shape == (1, n * FRAMES, DIMS)
    assert torch.equal(mels[s], want), s


def test_batch_segments_rejects_bad_arguments():
  segs = _songs([2, 1])
  with pytest.raises(ValueError):
    song.batch_segments(FakeSegments(), segs, 2, DIMS, torch.device('cpu'), [0])
  with pytest.raises(ValueError):
    song.batch_segments(FakeSegments(), segs, 0, DIMS, torch.device('cpu'), [0, 0])
  mels, rounds = song.batch_segments(FakeSegments(), [segs[0][:0]], 4, DIMS, torch.device('cpu'), [0])
  assert rounds == [] and mels[0].shape == (1, 0, DIMS)


class _Clock:
  def __init__(self):
    self.now = 1000.0

  def time(self):
    return self.now

  def advance(self, seconds):
    self.now += seconds


def _fake_model(slots, lengths, clock=None):
  """What the song drivers read off a no-context InferenceModel, with the stand-in predictor."""
  fake = FakeSegments(lengths['targets'], 128, clock)

  def predict_on_device(toks, ctx, mask, seed=0, init_z=None, noise=None, seeds=None):
    assert ctx is None and mask is None
    assert seeds is not None and init_z is None and noise is None
    return fake(toks, seeds)

  model = types.SimpleNamespace(
      audio_codec=audio_codecs.MelGAN(), sequence_length=lengths, codec=inference.build_codec(),
      batch_size=slots, engine=types.SimpleNamespace(device=torch.device('cpu')),
      predict_on_device=predict_on_device)
  return model, fake


def _notes(seconds):
  return M.make_notes([(0.1, seconds - 0.2, 60, 100, 0, False), (0.5, 1.0, 38, 110, 0, True)])


LENGTHS_NC = {'inputs': 128, 'targets': 32}   # 0.64 s segments


def test_synthesize_songs_runs_independent_rows(monkeypatch):
  clock = _Clock()
  monkeypatch.setattr(song.time, 'time', clock.time)
  model, fake = _fake_model(4, LENGTHS_NC, clock)
  notes = [_notes(2.0), M.make_notes([(0.05, 0.4, 60, 100, 0, False)]), _notes(3.0)]
  nseg = [song._tokenize(model, n, None)[1] for n in notes]
  assert nseg[1] == 1 and min(nseg[0], nseg[2]) > 1
  results, agg = song.synthesize_songs(model, notes, seeds=[1, 2, 3])
  total = sum(nseg)
  assert agg['segments'] == total and agg['rounds'] == len(fake.calls) == -(-total // 4)
  assert agg['wall_seconds'] == pytest.approx(sum(range(1, agg['rounds'] + 1)))
  rows = [(s, k) for s, n in enumerate(nseg) for k in range(n)]
  for s, (r, n) in enumerate(zip(results, nseg)):
    assert set(r) == {'full_pred_encoded', 'num_frames', 'tokens', 'model_timing'}
    assert r['full_pred_encoded'].shape == (n * 32, 128) and r['tokens'].shape == (n, 128)
    want = torch.cat([FakeSegments(32, 128)(torch.from_numpy(r['tokens'][k:k + 1].astype(np.int32)),
                                            [s + 1]) for k in range(n)], dim=1)
    np.testing.assert_array_equal(r['full_pred_encoded'], want[0].numpy())
    # the mean of the rounds (round j takes j + 1 s) that carried a segment after the song's first
    later = sorted({i // 4 for i, (t, k) in enumerate(rows) if t == s and k != 0})
    per_chunk = r['model_timing']['prediction_seconds_per_chunk']
    if later:
      assert per_chunk == pytest.approx(np.mean([j + 1 for j in later]))
      assert r['model_timing']['predictions_seconds_per_audio_second'] == pytest.approx(per_chunk / 0.64)
    else:
      assert np.isnan(per_chunk)


def test_synthesize_song_batches_its_segments():
  model, fake = _fake_model(3, LENGTHS_NC)
  notes = _notes(4.0)
  n = song._tokenize(model, notes, None)[1]
  assert n > 3
  r = song.synthesize_song(model, notes, seed=9)
  assert len(fake.calls) == -(-n // 3)
  assert all(s == 9 for _, seeds in fake.calls for s in seeds)
  assert set(r) == {'full_pred_encoded', 'num_frames', 'tokens', 'model_timing'}
  assert r['full_pred_encoded'].shape == (n * 32, 128)
  results, _ = song.synthesize_songs(model, [notes], [9])
  np.testing.assert_array_equal(r['full_pred_encoded'], results[0]['full_pred_encoded'])
  r2 = song.synthesize_song(model, notes, seed=9, max_segments=2)
  assert r2['full_pred_encoded'].shape == (2 * 32, 128)


def test_context_arguments_are_refused():
  model, fake = _fake_model(2, LENGTHS_NC)
  notes = _notes(2.0)
  audio = np.zeros(16000, np.float32)
  with pytest.raises(ValueError, match='context'):
    song.synthesize_song(model, notes, context_audio=audio)
  with pytest.raises(ValueError, match='always_mask_context'):
    song.synthesize_song(model, notes, always_mask_context=True)
  with pytest.raises(ValueError, match='context_audios'):
    song.synthesize_songs(model, [notes], context_audios=[audio])
  with pytest.raises(ValueError, match='context_audios'):
    song.synthesize_songs(model, [notes], context_audios=[None])
  with pytest.raises(ValueError, match='always_mask_context'):
    song.synthesize_songs(model, [notes], always_mask_context=True)
  assert not fake.calls
