"""-m gpu: the no-context model (context_length 0: models.DiffusionModel + network.Transformer) on
the CUDA engine, against its oracle (tests/no_context_oracle.py), against the context engine with
a masked-out context, through the cross-attention call site, the song drivers and a T5X
checkpoint."""
import os

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import config, engine, inference, song, weights
from oracle import msd_oracle as O
from tests import helpers as H
from tests import no_context_oracle as NC
from tests.test_gpu_attention_views import HH, H as HEADS, N as BASE_N, T as BASE_T
from tests.test_gpu_attention_views import Out, Workspace, attend, check, randn
from tests.test_gpu_song_batch import _notes, _nseg

pytestmark = pytest.mark.gpu

T = N = C = 128
LENGTHS = {'inputs': T, 'targets': N}


@pytest.fixture(scope='module')
def tiny():
  t5 = config.t5_tiny()
  return t5, weights.synthetic_params(t5, T, N, None, seed=0)


def _tokens(B, T, seed=1):
  """Token rows with padding: full, half, and (from row 2 on) nearly empty."""
  toks, _, _ = H.make_batch(B, T, 128, seed=seed)
  if B > 2:
    toks[2, 3:] = 0
    toks[2, 2] = 1
  return toks


def _rel(a, b):
  return ((a - b).abs().max() / b.abs().max().clamp_min(1e-6)).item()


def _encode(eng, toks, device):
  eng.encode(torch.from_numpy(toks).to(device), None, None)


# ---- against the oracle --------------------------------------------------------------------------
@pytest.mark.parametrize('size', ['tiny', 't5_small'])
@pytest.mark.parametrize('conditioned', [True, False])
def test_decode_eps(cuda_device, size, conditioned):
  if size == 'tiny':
    t5, Ts, Ns, B = config.t5_tiny(), T, N, 3
  else:
    t5, Ts, Ns, B = config.t5_small(), 2048, 256, 2
  steps = 16
  params = weights.synthetic_params(t5, Ts, Ns, None, seed=1)
  toks = _tokens(B, Ts)
  if B == 2:
    toks[1, 40:] = 0     # nearly empty
    toks[1, 39] = 1
  eng = H.build_engine(t5, Ts, Ns, 0, B, steps, 2.0, params)
  _encode(eng, toks, cuda_device)
  oc = H.oracle_config(t5, steps, 2.0)
  P = O.params_to(params)
  encs = NC.encode(P, oc, torch.from_numpy(toks))
  z = torch.randn(B, Ns, 128, generator=torch.Generator().manual_seed(3))
  flag = 1.0 if conditioned else 0.0
  for step_i in (steps - 1, 5, 0):
    got = eng.decode_eps(z.to(cuda_device), step_i, conditioned).cpu()
    t = np.float32(step_i + 1.0) / np.float32(steps)
    want = O.decode(P, oc, [(e * flag, m * flag) for e, m in encs], z, torch.full((B,), float(t)))
    rel = ((got - want).abs().max() / want.abs().max()).item()
    print(f'{size} cond={conditioned} step {step_i}: rel max err {rel:.3e}')
    assert rel < 3e-2, f'step {step_i}: rel max err {rel}'
  eng.close()


@pytest.mark.parametrize('style', ['concat_encodings', 'sum_cross_attends'])
def test_sample_matches_oracle(cuda_device, style):
  t5 = config.t5_tiny()
  t5.decoder_cross_attend_style = style
  params = weights.synthetic_params(t5, T, N, None, seed=0)
  B, steps = 3, 12
  toks = _tokens(B, T)
  init_z, noise = H.make_noise(steps, B, N)
  eng = H.build_engine(t5, T, N, 0, B, steps, 2.0, params)
  _encode(eng, toks, cuda_device)
  mel = eng.sample(init_z.to(cuda_device), noise.to(cuda_device)).cpu()
  oc = H.oracle_config(t5, steps, 2.0)
  ref, _ = NC.predict_batch_with_aux(O.params_to(params), oc,
                                     {'encoder_input_tokens': torch.from_numpy(toks)}, init_z, noise)
  err = (mel - ref).abs() / (oc.max_value - oc.min_value) * 2.0
  assert torch.isfinite(mel).all()
  H.assert_trajectory_close(err, f'no-context tiny {style}')
  eng.close()


@pytest.mark.parametrize('style', ['concat_encodings', 'sum_cross_attends'])
def test_fp32_accurate_sample_matches_oracle(cuda_device, style):
  """The bounds of test_fp32_accurate_sample_matches_oracle (10x inside SURVEY 8d's fp32
  tolerance)."""
  t5 = config.t5_tiny()
  t5.decoder_cross_attend_style = style
  params = weights.synthetic_params(t5, T, N, None, seed=0)
  B, steps = 2, 12
  toks = _tokens(B, T)
  init_z, noise = H.make_noise(steps, B, N)
  eng = H.build_engine(t5, T, N, 0, B, steps, 2.0, params, precision='fp32_accurate')
  _encode(eng, toks, cuda_device)
  mel = eng.sample(init_z.to(cuda_device), noise.to(cuda_device)).cpu()
  oc = H.oracle_config(t5, steps, 2.0)
  ref, _ = NC.predict_batch_with_aux(O.params_to(params), oc,
                                     {'encoder_input_tokens': torch.from_numpy(toks)}, init_z, noise)
  err = (mel - ref).abs() / (oc.max_value - oc.min_value) * 2.0
  H.assert_trajectory_close(err, f'no-context fp32-accurate tiny {style}',
                            mean=1e-4, p99=1e-3, share_01=1e-5)
  eng.close()


# ---- against the context engine with a masked-out context ---------------------------------------
@pytest.mark.parametrize('style', ['concat_encodings', 'sum_cross_attends'])
def test_same_as_context_engine_with_masked_context(cuda_device, style):
  """A context engine sharing the weights and given all-zero context masks: the token rows of the
  encodings are the same bits (same kernels, same rows); decode_eps agrees within the oracle
  bound (the cross-attention runs over 128 more masked keys, which changes the rounding only)."""
  t5 = config.t5_tiny()
  t5.decoder_cross_attend_style = style
  nc = weights.synthetic_params(t5, T, N, None, seed=0)
  ctx_tree = NC.as_context_tree(nc, weights.synthetic_params(t5, T, N, C, seed=1))
  B, steps = 3, 16
  _, ctx, _ = H.make_batch(B, T, C)
  toks = _tokens(B, T)
  cmask = np.zeros((B, C), np.int32)
  a = H.build_engine(t5, T, N, 0, B, steps, 2.0, nc)
  b = H.build_engine(t5, T, N, C, B, steps, 2.0, ctx_tree)
  _encode(a, toks, cuda_device)
  tb = H.torch_batch(toks, ctx, cmask, cuda_device)
  b.encode(tb['encoder_input_tokens'], tb['encoder_continuous_inputs'], tb['encoder_continuous_mask'])
  ea, eb = a.encodings(), b.encodings()
  assert ea.shape == (B, T, t5.emb_dim) and eb.shape == (B, T + C, t5.emb_dim)
  assert torch.equal(ea, eb[:, :T])
  z = torch.randn(B, N, 128, generator=torch.Generator().manual_seed(3)).to(cuda_device)
  worst = 0.0
  for conditioned in (True, False):
    for step_i in (steps - 1, 5, 0):
      ga, gb = a.decode_eps(z, step_i, conditioned), b.decode_eps(z, step_i, conditioned)
      rel = _rel(ga.cpu(), gb.cpu())
      worst = max(worst, rel)
      if not conditioned:
        assert torch.equal(ga, gb)   # the unconditional pass skips the cross-attention in both
      assert rel < 3e-2, (conditioned, step_i, rel)
  print(f'{style}: largest rel |decode_eps(no context) - decode_eps(masked context)| = {worst:.3e}')
  a.close()
  b.close()


def test_encode_arguments(cuda_device, tiny):
  t5, params = tiny
  eng = H.build_engine(t5, T, N, 0, 1, 4, 2.0, params)
  toks = torch.from_numpy(_tokens(1, T)).to(cuda_device)
  with pytest.raises(ValueError):
    eng.encode(toks, torch.zeros(1, C, 128, device=cuda_device),
               torch.zeros(1, C, dtype=torch.int32, device=cuda_device))
  eng.encode(toks, None, None)
  assert eng.encodings().shape == (1, T, t5.emb_dim)
  eng.close()
  # a context engine still needs its context
  ctx_eng = H.build_engine(t5, T, N, C, 1, 4, 2.0, weights.synthetic_params(t5, T, N, C))
  with pytest.raises(ValueError):
    ctx_eng.encode(toks, None, None)
  assert ctx_eng.lib.msd_encode(ctx_eng._h, engine._ptr(toks), None, None, 1, None) == -1
  ctx_eng.close()
  # a context tree does not load into a no-context engine (no encoder/...)
  with pytest.raises(Exception, match='encoder/'):
    H.build_engine(t5, T, N, 0, 1, 4, 2.0, weights.synthetic_params(t5, T, N, C))


# ---- the cross-attention call site at base dimensions ---------------------------------------------
LAYERS, CACHE_B = 2, 8


@pytest.mark.parametrize('prec', ['bf16', 'fp32_accurate'])
@pytest.mark.parametrize('nb,kbr', [(1, 0), (8, 0), (8, BASE_T)])
def test_cross_attention_over_the_token_cache(cuda_device, prec, nb, kbr):
  """cross_attention without a context: K / V of layer 1 of a [L][B * T, 2 hh] cache (ld 2 hh, V
  at column hh), T = 2048 keys per batch row, mask rows of T / 32 words, kv_static = 1; kbr:
  kv_batch_rows (0: the launch's key count, as the engine passes it)."""
  dev = cuda_device
  dt = torch.float32 if prec == 'fp32_accurate' else torch.bfloat16
  rows = nb * BASE_N
  cache = torch.empty(LAYERS * CACHE_B * BASE_T * 2 * HH, dtype=dt, device=dev)
  q = torch.empty(rows * HH, dtype=dt, device=dev)
  mask = torch.ones(nb, BASE_T, dtype=torch.int32)
  for b, n in enumerate([2048, 1500, 40, 700, 2048, 3, 2048, 1024][:nb]):
    mask[b, n:] = 0
  mask = mask.to(dev)
  o_ld = HH
  out = Out(rows, 3 * HH if prec == 'fp32_accurate' else HH, dev)
  ws = Workspace(nb, BASE_N, dev)
  k_off = 1 * CACHE_B * BASE_T * 2 * HH
  g = torch.Generator(dev).manual_seed(61 + nb + kbr)
  for draw in range(2):
    cache.copy_(randn(cache.shape, g, 1.0, dt, dev))
    torch.as_strided(cache, (LAYERS * CACHE_B * BASE_T, HH), (2 * HH, 1), 0).mul_(0.5)
    q.copy_(randn(q.shape, g, 0.5, dt, dev))
    want, wabs = attend(prec, q, 0, HH, cache, k_off, k_off + HH, 2 * HH, nb, BASE_N, BASE_T, out, 0,
                        o_ld, ws, mask=mask, kbr=kbr, kv_static=1)
    check(prec, out, 0, o_ld, want, wabs, f'no-context cross {prec} nb={nb} kbr={kbr} draw {draw}')
    out.assert_untouched_outside()
  assert HEADS * 64 == HH


# ---- songs -----------------------------------------------------------------------------------------
def _model(t5, params, slots, steps=5, precision='bf16'):
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = steps
  diff.classifier_free_guidance.eval_condition_weight = 2.0
  return inference.InferenceModel.from_config(t5, diff, LENGTHS, 'synthetic:0', slots,
                                              params=params, precision=precision)


def _segment_batch(r, k):
  return {'encoder_input_tokens': r['tokens'][k:k + 1].astype(np.int32)}


def test_song_rounds_follow_batch1_segments(cuda_device, tiny):
  """6 segments at batch 4 (2 rounds) against each segment's predict(segment, seed) at batch 1."""
  t5, params = tiny
  steps = 20
  batched = _model(t5, params, 4, steps)
  single = _model(t5, params, 1, steps)
  notes = _notes(14.0, 60)
  assert _nseg(batched, notes) == 6
  r = song.synthesize_song(batched, notes, seed=11)
  assert set(r) == {'full_pred_encoded', 'num_frames', 'tokens', 'model_timing'}
  assert r['full_pred_encoded'].shape == (6 * N, 128)
  assert r['model_timing']['prediction_seconds_per_chunk'] > 0
  span = 4.0 - np.log(1e-5)
  for k in range(6):
    want, _ = single.predict(_segment_batch(r, k), seed=11)
    err = np.abs(r['full_pred_encoded'][k * N:(k + 1) * N] - want[0]) / span * 2.0
    H.assert_trajectory_close(err, f'segment {k} in a round of 4 vs alone at batch 1')


def test_song_at_batch1_is_predict_bit_for_bit(cuda_device, tiny):
  t5, params = tiny
  model = _model(t5, params, 1)
  notes = _notes(7.0, 62)
  n = _nseg(model, notes)
  assert n == 3
  r = song.synthesize_song(model, notes, seed=(5 << 32) | 3)
  for k in range(n):
    want, _ = model.predict(_segment_batch(r, k), seed=(5 << 32) | 3)
    np.testing.assert_array_equal(r['full_pred_encoded'][k * N:(k + 1) * N], want[0])
  with pytest.raises(ValueError):
    song.synthesize_song(model, notes, always_mask_context=True)


def test_several_songs(cuda_device, tiny):
  t5, params = tiny
  steps = 20
  batched = _model(t5, params, 4, steps)
  single = _model(t5, params, 1, steps)
  notes = [_notes(7.0, 60), _notes(4.0, 64), _notes(9.0, 67)]
  nseg = [_nseg(batched, n) for n in notes]
  assert nseg == [3, 2, 4]
  seeds = [0, 9, (3 << 32) | 1]
  results, agg = song.synthesize_songs(batched, notes, seeds)
  assert agg['segments'] == 9 and agg['rounds'] == 3 and agg['x_realtime'] > 0
  span = 4.0 - np.log(1e-5)
  for k, (r, nt, s) in enumerate(zip(results, notes, seeds)):
    want = song.synthesize_song(single, nt, seed=s)
    assert r['full_pred_encoded'].shape == want['full_pred_encoded'].shape
    np.testing.assert_array_equal(r['tokens'], want['tokens'])
    assert r['num_frames'] == want['num_frames']
    err = np.abs(r['full_pred_encoded'] - want['full_pred_encoded']) / span * 2.0
    H.assert_trajectory_close(err, f'song {k} among 3 at batch 4 vs alone')


def test_predict_on_device_and_predict(cuda_device, tiny):
  t5, params = tiny
  model = _model(t5, params, 2)
  toks = torch.from_numpy(_tokens(2, T)).to(cuda_device)
  got = model.predict_on_device(toks, None, None, seeds=[1, 2])
  assert torch.equal(got, model.engine.sample_rows([1, 2]))
  assert torch.equal(model.predict_on_device(toks, None, None, seed=4), model.engine.sample(seed=4))
  with pytest.raises(ValueError):
    model.predict_on_device(toks, torch.zeros(2, C, 128, device=cuda_device),
                            torch.zeros(2, C, dtype=torch.int32, device=cuda_device))
  # predict reads encoder_input_tokens only; other keys are ignored
  batch = {'encoder_input_tokens': toks.cpu().numpy()}
  mel, scores = model.predict(batch, seed=4)
  assert mel.shape == (2, N, 128) and not scores.any()
  np.testing.assert_array_equal(mel, model.engine.sample(seed=4).cpu().numpy())
  extra = dict(batch, decoder_target_tokens=np.zeros((2, N, 128), np.float32),
               decoder_input_tokens=np.zeros((2, N, 128), np.float32),
               encoder_continuous_inputs=np.zeros((2, 7, 3), np.float32))
  mel2, _ = model.predict(extra, seed=4)
  np.testing.assert_array_equal(mel, mel2)


def test_basic_gin_model_predicts_and_synthesizes(cuda_device):
  """InferenceModel from the basic (no-context) gin fixture at base size, 3 sampler steps: predict
  and a song of 3 segments in rounds of 2 rows."""
  gin = inference.parse_training_gin_file(
      os.path.join(os.path.dirname(__file__), 'golden', 'base_no_context.gin'),
      ['sampler/diffusion_utils.DiffusionSchedule.num_steps = 3'])
  model = inference.InferenceModel('synthetic:0', gin, batch_size=2)
  assert model.targets_context_length is None
  rng = np.random.default_rng(2)
  toks = rng.integers(3, 1391, (1, 2048)).astype(np.int32)
  toks[0, 1200:] = 0
  mel, _ = model.predict({'encoder_input_tokens': toks}, seed=0)
  assert mel.shape == (1, 256, 128) and np.isfinite(mel).all()
  notes = _notes(13.0, 60)
  n = _nseg(model, notes)
  assert n == 3
  r = song.synthesize_song(model, notes)
  assert set(r) == {'full_pred_encoded', 'num_frames', 'tokens', 'model_timing'}
  assert r['full_pred_encoded'].shape == (n * 256, 128) and np.isfinite(r['full_pred_encoded']).all()


# ---- checkpoints -------------------------------------------------------------------------------------
def test_inference_model_restores_t5x_checkpoint(cuda_device, tiny, tmp_path):
  from music_spectrogram_diffusion_b200 import t5x_checkpoint
  t5, params = tiny
  ck = t5x_checkpoint.save_t5x_checkpoint(str(tmp_path / 'checkpoint_500000'), params, step=500000,
                                          inline_below=300, chunk_rows=64)
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = 4
  a = inference.InferenceModel.from_config(t5, diff, LENGTHS, ck, 1)
  b = inference.InferenceModel.from_config(t5, diff, LENGTHS, 'synthetic:0', 1, params=params)
  rng = np.random.default_rng(9)
  batch = dict(encoder_input_tokens=rng.integers(3, 1391, (1, T)).astype(np.int32),
               decoder_target_tokens=np.zeros((1, N, 128), np.float32))
  ma, _ = a.predict(batch, seed=3)
  mb, _ = b.predict(batch, seed=3)
  np.testing.assert_array_equal(ma, mb)
  # a context checkpoint is not a no-context model's
  ck2 = t5x_checkpoint.save_t5x_checkpoint(str(tmp_path / 'ctx'), weights.synthetic_params(t5, T, N, C),
                                           step=1)
  with pytest.raises(ValueError, match='does not match the gin config'):
    inference.InferenceModel.from_config(t5, diff, LENGTHS, ck2, 1).predict(batch)
