"""Audio -> MelGAN mel features on the CPU: the float32 tables, frame counts, the song segmentation
(in the fp64 oracle), primer frames, WAV loading and priming in the chained-song scheduler."""
import io
import struct
import types
import wave

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import audio_codecs, midi_tokens, song
from oracle import mel_oracle as MO
from tests.test_song_batch import DIMS, FRAMES, FakeRows, _songs

LENGTHS = [3, 1, 4, 2, 2]
SEEDS = [0, 7, 31337, (9 << 32) | 5, 7]


def test_filterbank_shape_range_and_bands():
  w = audio_codecs.linear_to_mel_weight_matrix()
  assert w.dtype == np.float32 and w.shape == (513, 128)
  assert not w[0].any()
  assert w.min() >= 0.0 and w.max() <= 1.0
  for j in range(128):
    nz = np.nonzero(w[:, j])[0]
    assert len(nz) > 0, j
    assert nz[-1] - nz[0] + 1 == len(nz), j   # contiguous
  assert len(np.nonzero(w[:, 0])[0]) == 1
  assert (w != 0).sum() == 1012


def test_float32_tables_follow_the_fp64_formulas():
  w = audio_codecs.linear_to_mel_weight_matrix()
  assert np.abs(w - MO.linear_to_mel_weight_matrix64()).max() < 2e-5
  win = audio_codecs.hann_window()
  assert win.dtype == np.float32 and win.shape == (640,)
  assert win[0] == 0.0 and win[320] == 1.0
  assert np.abs(win - MO.hann_window64()).max() < 1e-6   # float32 cos argument, as TF


@pytest.mark.parametrize('n,frames', [(0, 0), (1, 1), (319, 1), (320, 1), (321, 2), (640, 2),
                                      (641, 3)])
def test_frame_counts(n, frames):
  assert MO.num_frames(n) == frames
  assert MO.frames64(np.ones(n)).shape == (frames, 640)
  assert MO.mel_linear64(np.ones(n), audio_codecs.hann_window(),
                         audio_codecs.linear_to_mel_weight_matrix()).shape == (frames, 128)


def test_frames_are_zero_padded_at_the_end_without_centring():
  x = np.arange(1, 700, dtype=np.float64)
  fr = MO.frames64(x)
  assert fr.shape == (3, 640)
  np.testing.assert_array_equal(fr[0], x[:640])
  np.testing.assert_array_equal(fr[1, :379], x[320:])
  assert not fr[1, 379:].any()
  np.testing.assert_array_equal(fr[2, :59], x[640:])


def test_primer_frames():
  # the last min(C, n // 320 - 1) frames whose 640-sample window lies inside the recording
  assert song.primer_frames(640, 256) == (0, 1)
  assert song.primer_frames(959, 256) == (0, 1)
  assert song.primer_frames(960, 256) == (0, 2)
  assert song.primer_frames(320 * 100, 256) == (0, 99)
  assert song.primer_frames(320 * 300 + 17, 256) == (43, 256)
  assert song.primer_frames(320 * 300 + 17, 128) == (171, 128)
  for n in (640, 1000, 320 * 300 + 17):
    first, count = song.primer_frames(n, 256)
    assert (first + count - 1) * 320 + 640 <= n < (first + count) * 320 + 640
  for n in (0, 1, 639):
    with pytest.raises(ValueError):
      song.primer_frames(n, 256)


class _OracleCodec:
  hop_size, n_dims = 320, 128

  def __init__(self):
    self.window = audio_codecs.hann_window()
    self.weights = audio_codecs.linear_to_mel_weight_matrix()

  def encode(self, x):
    return MO.encode64(x, self.window, self.weights)


@pytest.mark.parametrize('n', [320 * 256 * 2 - 320, 320 * 256 * 2, 320 * 256 * 3 + 4321, 5000])
def test_whole_song_encode_then_slice_equals_per_segment_encode(n):
  """encode_song_audio (one encode of the padded song, cut into segments) against the reference's
  per-segment route (each segment with its 16 extra frames, the last padded with 0.0), both on
  the fp64 oracle."""
  rng = np.random.default_rng(n)
  x = rng.uniform(-1, 1, n).astype(np.float32)
  model = types.SimpleNamespace(audio_codec=_OracleCodec(), sequence_length={'targets': 256})
  got = song.encode_song_audio(model, x)
  want, total = MO.encode_song_by_segments(x, model.audio_codec.encode)
  assert got['num_frames'] == total == midi_tokens.num_song_frames(n / 16000)
  assert got['full_gt_encoded'].shape == want.shape == (-(-total // 256) * 256, 128)
  # encode_song_audio keeps float32: the fp64 oracle's values rounded once
  np.testing.assert_allclose(got['full_gt_encoded'], want, rtol=2 ** -24, atol=1e-12)
  if total % 256:
    assert not want[total:].any()   # the feature converter's 0.0 padding
  assert (want[:total] != 0).all()


def test_segment_spans_follow_split_full_song():
  assert MO.segment_spans(600) == [(0, 271), (256, 527), (512, 600)]
  assert MO.segment_spans(256) == [(0, 256)]
  assert MO.segment_spans(257) == [(0, 257), (256, 257)]


def _wav(x_int, width, channels, rate=16000):
  buf = io.BytesIO()
  with wave.open(buf, 'wb') as w:
    w.setnchannels(channels)
    w.setsampwidth(width)
    w.setframerate(rate)
    if width == 1:
      raw = (x_int + 128).astype(np.uint8).tobytes()
    elif width == 3:
      v = x_int.astype(np.int64) & 0xFFFFFF
      raw = np.stack([v & 0xFF, (v >> 8) & 0xFF, v >> 16], -1).astype(np.uint8).tobytes()
    else:
      raw = x_int.astype({2: '<i2', 4: '<i4'}[width]).tobytes()
    w.writeframes(raw)
  return buf.getvalue()


@pytest.mark.parametrize('channels', [1, 2])
@pytest.mark.parametrize('width', [1, 2, 3, 4])
def test_load_audio_round_trips(width, channels, tmp_path):
  bits = 8 * width
  rng = np.random.default_rng(width * 10 + channels)
  top = 1 << (bits - 1)
  x_int = rng.integers(-top, top, (999, channels), dtype=np.int64)
  x_int[0] = -top
  x_int[1] = top - 1
  data = _wav(x_int.reshape(-1), width, channels)
  want = (x_int / float(top)).astype(np.float32)
  want = want[:, 0] if channels == 1 else want.mean(axis=1, dtype=np.float32)
  got = song.load_audio(data)
  assert got.dtype == np.float32 and got.shape == (999,)
  np.testing.assert_array_equal(got, want)
  path = tmp_path / 'a.wav'
  path.write_bytes(data)
  np.testing.assert_array_equal(song.load_audio(str(path)), want)
  assert np.abs(got).max() <= 1.0


def test_load_audio_refuses_other_rates_and_compressed_formats():
  with pytest.raises(ValueError, match='16000'):
    song.load_audio(_wav(np.zeros(10, np.int64), 2, 1, rate=44100))
  # an IMA ADPCM header (format tag 0x11)
  fmt = struct.pack('<HHIIHH', 0x11, 1, 16000, 8000, 256, 4) + struct.pack('<HH', 2, 505)
  data = b'data' + struct.pack('<I', 256) + bytes(256)
  chunk = b'WAVE' + b'fmt ' + struct.pack('<I', len(fmt)) + fmt + data
  adpcm = b'RIFF' + struct.pack('<I', len(chunk)) + chunk
  with pytest.raises(ValueError):
    song.load_audio(adpcm)
  with pytest.raises(ValueError):
    song.load_audio(b'not a wav file at all')


def _primers(songs, seed=1):
  """An (ctx, mask) primer for the songs listed, None for the others."""
  rng = np.random.default_rng(seed)
  out = [None] * len(LENGTHS)
  for s, count in songs.items():
    ctx = torch.zeros(1, FRAMES, DIMS)
    ctx[0, :count] = torch.from_numpy(rng.normal(size=(count, DIMS)).astype(np.float32))
    mask = torch.zeros(1, FRAMES, dtype=torch.int32)
    mask[0, :count] = 1
    out[s] = (ctx, mask)
  return out


@pytest.mark.parametrize('slots', [1, 2, 3, 8])
def test_primed_songs_get_their_context_on_the_first_segment_only(slots):
  segs = _songs(LENGTHS)
  primers = _primers({0: 3, 2: FRAMES, 3: 1})
  fake = FakeRows()
  mels, rounds = song.chain_songs(fake, segs, slots, FRAMES, DIMS, torch.device('cpu'), SEEDS,
                                  initial_context=primers)
  plain_fake = FakeRows()
  plain, plain_rounds = song.chain_songs(plain_fake, segs, slots, FRAMES, DIMS, torch.device('cpu'),
                                         SEEDS)
  # the schedule (compaction, order of entry) does not depend on the primers
  assert [r['rows'] for r in rounds] == [r['rows'] for r in plain_rounds]
  for rd, (_, ctx, mask, _) in zip(rounds, fake.calls):
    for r, (s, seg) in enumerate(rd['rows']):
      if seg == 0 and primers[s] is not None:
        assert torch.equal(ctx[r:r + 1], primers[s][0])
        assert torch.equal(mask[r:r + 1], primers[s][1])
        count = int(primers[s][1].sum())
        assert (mask[r, :count] == 1).all() and (mask[r, count:] == 0).all()
      elif seg == 0:
        assert not ctx[r].any() and not mask[r].any()
      else:
        assert (mask[r] == 1).all()
  for s in range(len(LENGTHS)):
    # a primed song is its own serial chain started from the primer
    prev, m = primers[s] if primers[s] is not None else (torch.zeros(1, FRAMES, DIMS),
                                                         torch.zeros(1, FRAMES, dtype=torch.int32))
    want = []
    single = FakeRows()
    for k in range(LENGTHS[s]):
      prev = single(segs[s][k][None], prev, m, [SEEDS[s]])
      m = torch.ones(1, FRAMES, dtype=torch.int32)
      want.append(prev)
    assert torch.equal(mels[s], torch.cat(want, dim=1)), s
    assert torch.equal(mels[s], plain[s]) == (primers[s] is None), s


def test_no_initial_context_reproduces_the_unprimed_rounds():
  segs = _songs(LENGTHS)
  runs = []
  for ic in ('absent', None, [None] * len(LENGTHS)):
    fake = FakeRows()
    kw = {} if ic == 'absent' else {'initial_context': ic}
    mels, rounds = song.chain_songs(fake, segs, 2, FRAMES, DIMS, torch.device('cpu'), SEEDS, **kw)
    runs.append((mels, [r['rows'] for r in rounds], fake.calls))
  for mels, rows, calls in runs[1:]:
    assert rows == runs[0][1]
    assert all(torch.equal(a, b) for a, b in zip(mels, runs[0][0]))
    for c, c0 in zip(calls, runs[0][2]):
      for a, b in zip(c[:3], c0[:3]):
        assert a.dtype == b.dtype and torch.equal(a, b)
      assert c[3] == c0[3]


def test_initial_context_is_checked():
  segs = _songs(LENGTHS)
  cpu = torch.device('cpu')
  with pytest.raises(ValueError):
    song.chain_songs(FakeRows(), segs, 2, FRAMES, DIMS, cpu, SEEDS, initial_context=[None])
  with pytest.raises(ValueError):
    song.chain_songs(FakeRows(), segs, 2, FRAMES, DIMS, cpu, SEEDS, always_mask_context=True,
                     initial_context=_primers({1: 2}))
  bad = [None] * len(LENGTHS)
  bad[0] = (torch.zeros(1, FRAMES + 1, DIMS), torch.zeros(1, FRAMES + 1, dtype=torch.int32))
  with pytest.raises(ValueError):
    song.chain_songs(FakeRows(), segs, 2, FRAMES, DIMS, cpu, SEEDS, initial_context=bad)
