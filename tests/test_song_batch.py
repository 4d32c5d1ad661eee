"""song.chain_songs / synthesize_songs scheduling on the CPU, driven by a stand-in predict_rows."""
import types

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import audio_codecs, inference, midi_tokens as M, song

FRAMES, DIMS, INPUTS = 8, 4, 16
LENGTHS = [3, 1, 4, 2, 2]


class FakeRows:
  """Row r of the output depends on row r of tokens / ctx / mask and seeds[r] only (elementwise
  float math, so the value of a row does not depend on the batch it is computed in)."""

  def __init__(self, frames=FRAMES):
    self.frames = frames
    self.calls = []

  def __call__(self, toks, ctx, mask, seeds):
    assert toks.dtype == torch.int32 and mask.dtype == torch.int32
    assert toks.shape[0] == ctx.shape[0] == mask.shape[0] == len(seeds)
    self.calls.append((toks.clone(), ctx.clone(), mask.clone(), list(seeds)))
    tok = (toks.long().sum(1) % 97).to(torch.float32)[:, None, None]
    sd = torch.tensor([float(s % 1013) for s in seeds])[:, None, None]
    m = mask.to(torch.float32)[:, :self.frames, None]
    return torch.tanh(0.5 * ctx[:, :self.frames] + 0.01 * tok + 0.001 * sd + 0.3 * m)


def _songs(lengths, seed=0):
  rng = np.random.default_rng(seed)
  return [torch.from_numpy(rng.integers(3, 1000, (n, INPUTS)).astype(np.int32)) for n in lengths]


def _serial(fake, segs, seed, always_mask_context=False, dims=DIMS):
  prev = torch.zeros(1, fake.frames, dims)
  outs = []
  for k in range(len(segs)):
    first = k == 0 or always_mask_context
    mask = torch.full((1, fake.frames), 0 if first else 1, dtype=torch.int32)
    prev = fake(segs[k][None], prev, mask, [seed])
    outs.append(prev)
  return torch.cat(outs, dim=1)


@pytest.mark.parametrize('always_mask_context', [False, True])
@pytest.mark.parametrize('slots', [1, 2, 3, 8])
def test_rounds_follow_the_schedule_and_equal_the_serial_chains(slots, always_mask_context):
  segs = _songs(LENGTHS)
  seeds = [0, 7, 31337, (9 << 32) | 5, 7]
  fake = FakeRows()
  mels, rounds = song.chain_songs(fake, segs, slots, FRAMES, DIMS, torch.device('cpu'), seeds,
                                  always_mask_context)
  # every song is its own serial chain of the same predict function
  for s, n in enumerate(LENGTHS):
    assert mels[s].shape == (1, n * FRAMES, DIMS)
    assert torch.equal(mels[s], _serial(FakeRows(), segs[s], seeds[s], always_mask_context)), s
  assert len(rounds) == len(fake.calls)
  assert sum(len(r['rows']) for r in rounds) == sum(LENGTHS)
  seen = {}
  entered = []
  for k, (rd, (toks, ctx, mask, rseeds)) in enumerate(zip(rounds, fake.calls)):
    rows = rd['rows']
    assert 1 <= len(rows) <= slots
    assert rd['seconds'] >= 0
    songs_here = [s for s, _ in rows]
    assert songs_here == sorted(songs_here)  # compacted, in order of entry
    for r, (s, seg) in enumerate(rows):
      if s not in seen:
        entered.append(s)
      else:
        assert seen[s] == (k - 1, seg - 1), (s, seen[s], k, seg)  # no gap between a song's rounds
      seen[s] = (k, seg)
      assert torch.equal(toks[r], segs[s][seg])
      assert rseeds[r] == seeds[s]
      want = 0 if (seg == 0 or always_mask_context) else 1
      assert (mask[r] == want).all(), (s, seg)
      if seg == 0:
        assert not ctx[r].any()
      else:
        assert torch.equal(ctx[r], mels[s][0, (seg - 1) * FRAMES:seg * FRAMES])
    # the batch shrinks only once every song has entered
    if len(rows) < slots:
      assert len(seen) == len(LENGTHS), (k, rows)
  assert entered == list(range(len(LENGTHS)))  # songs enter in order
  for s, n in enumerate(LENGTHS):
    assert seen[s][1] == n - 1


def test_each_song_enters_when_a_slot_frees():
  segs = _songs(LENGTHS)
  _, rounds = song.chain_songs(FakeRows(), segs, 2, FRAMES, DIMS, torch.device('cpu'), [0] * 5)
  assert [r['rows'] for r in rounds] == [
      [(0, 0), (1, 0)], [(0, 1), (2, 0)], [(0, 2), (2, 1)], [(2, 2), (3, 0)], [(2, 3), (3, 1)],
      [(4, 0)], [(4, 1)]]


def test_chain_songs_rejects_bad_arguments():
  segs = _songs([2, 1])
  with pytest.raises(ValueError):
    song.chain_songs(FakeRows(), segs, 2, FRAMES, DIMS, torch.device('cpu'), [0])
  with pytest.raises(ValueError):
    song.chain_songs(FakeRows(), segs, 0, FRAMES, DIMS, torch.device('cpu'), [0, 0])


def _fake_model(slots, lengths):
  """What synthesize_songs reads off an InferenceModel, with the stand-in predict function."""
  fake = FakeRows(lengths['targets'])

  def predict_on_device(toks, ctx, mask, seed=0, init_z=None, noise=None, seeds=None):
    assert seeds is not None and init_z is None and noise is None
    return fake(toks, ctx, mask, seeds)

  model = types.SimpleNamespace(
      audio_codec=audio_codecs.MelGAN(), sequence_length=lengths, codec=inference.build_codec(),
      batch_size=slots, engine=types.SimpleNamespace(device=torch.device('cpu')),
      predict_on_device=predict_on_device)
  return model, fake


def _notes(seconds):
  return M.make_notes([(0.1, seconds - 0.2, 60, 100, 0, False), (0.5, 1.0, 38, 110, 0, True)])


def test_synthesize_songs_returns_the_song_dicts_and_honours_max_segments():
  lengths = {'inputs': 128, 'targets': 32, 'targets_context': 32}   # 0.64 s segments
  model, fake = _fake_model(3, lengths)
  notes = [_notes(2.0), _notes(1.0), _notes(3.0), _notes(1.5)]
  full = [song._tokenize(model, n, None)[1] for n in notes]
  assert min(full) > 1
  results, agg = song.synthesize_songs(model, notes, seeds=[1, 2, 3, 4])
  assert agg['segments'] == sum(full) and agg['rounds'] == len(fake.calls)
  assert agg['wall_seconds'] >= 0 and agg['audio_seconds'] == pytest.approx(sum(full) * 0.64)
  for s, (r, n) in enumerate(zip(results, full)):
    assert set(r) == {'full_pred_encoded', 'num_frames', 'tokens', 'model_timing'}
    assert r['full_pred_encoded'].shape == (n * 32, 128)
    assert r['tokens'].shape == (n, 128) and r['num_frames'] <= n * 32
    assert set(r['model_timing']) == {'prediction_seconds_per_chunk',
                                      'predictions_seconds_per_audio_second'}
    assert r['model_timing']['prediction_seconds_per_chunk'] >= 0
    segs = torch.from_numpy(r['tokens'].astype(np.int32))
    want = _serial(FakeRows(32), segs, s + 1, dims=128)
    np.testing.assert_array_equal(r['full_pred_encoded'], want[0].numpy())
  results, agg = song.synthesize_songs(model, notes, max_segments=2)
  assert agg['segments'] == 2 * len(notes)
  for r in results:
    assert r['full_pred_encoded'].shape == (2 * 32, 128) and r['tokens'].shape[0] == 2
    assert r['num_frames'] <= 2 * 32
  # one segment: no timed segment after the first
  results, _ = song.synthesize_songs(model, notes[:1], max_segments=1)
  assert np.isnan(results[0]['model_timing']['prediction_seconds_per_chunk'])


def test_synthesize_songs_default_seed_and_seed_count():
  lengths = {'inputs': 128, 'targets': 32, 'targets_context': 32}
  model, fake = _fake_model(2, lengths)
  notes = [_notes(1.0), _notes(1.2), _notes(0.8)]
  song.synthesize_songs(model, notes, max_segments=1)
  assert all(s == 0 for call in fake.calls for s in call[3])
  with pytest.raises(ValueError):
    song.synthesize_songs(model, notes, seeds=[0, 1])
