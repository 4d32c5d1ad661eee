"""Full-song synthesis driver: notes (or a MIDI file) -> chained 5.12 s segments -> mel frames.

Library form of the loops the reference keeps in its colab ("Synthesize Audio" cell) and in
`beam/evaluation.py:156-276`: the first segment runs with a masked context, every later one
is conditioned on the previous segment's predicted mel; per-segment wall times are reported
with the reference's `model_timing` fields (first segment excluded, evaluation.py:217-220,
238-247).  The mel -> audio vocoder is outside this path (SURVEY §2); `audio_codecs.griffin_lim`
stands in for it.

Audio goes the other way through `MelGAN.encode` (the library's CUDA kernel): `load_audio` reads
a 16 kHz WAV file (or, with resample=True, a WAV file at any rate, resampled to 16 kHz on the GPU
as the reference's librosa does), `encode_song_audio` gives a recording's ground-truth mels segment by segment
(`full_gt_encoded`, evaluation.py:156-276), and `context_audio=` primes a song's first segment
with the end of a recording instead of a masked-out context.

The other way, `audio_codecs.griffin_lim` renders predicted features (`full_pred_encoded`) to
audio without the absent vocoder, and `save_audio` writes it as a 16-bit WAV file.

`synthesize_songs` runs several such chains at once: each round puts the next segment of every
active song into one batch, one song per row, and every row draws its noise from its own song's
seed (`InferenceModel.predict_on_device(..., seeds=)`), so a song comes out as it would alone.

A model without a context (the reference's no-context `DiffusionModel`, lengths without
`targets_context`) has no chain: a song's segments do not depend on each other, and the
reference's loop predicts each one on its own with the song's seed (evaluation.py:179-210).  Both
drivers then run every segment of every song as an independent batch row (`batch_segments`),
`batch_size` rows per round, so a 12-segment song takes 2 rounds at batch 8 instead of 12 calls.
"""

from __future__ import annotations

import io
import time
import wave
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from music_spectrogram_diffusion_b200 import audio_codecs, midi_file, midi_tokens

# predict_rows(tokens [R, inputs], ctx [R, context, n_dims], mask [R, context], seeds: R ints)
#   -> mel [R, targets, n_dims]; row r must depend on row r of the inputs and seeds[r] only
PredictRows = Callable[[torch.Tensor, torch.Tensor, torch.Tensor, Sequence[int]], torch.Tensor]
# predict_segments(tokens [R, inputs], seeds: R ints) -> mel [R, targets, n_dims] of a model
#   without a context; row r must depend on row r of the tokens and seeds[r] only
PredictSegments = Callable[[torch.Tensor, Sequence[int]], torch.Tensor]


def has_context(model) -> bool:
  """Whether the model conditions a segment on a context (ContextDiffusionModel: its lengths have
  `targets_context`) or not (DiffusionModel)."""
  return 'targets_context' in model.sequence_length


def _refuse_context(model, what: Optional[str]) -> None:
  if what is not None:
    raise ValueError(f'{what}: this model has no context (its TASK_FEATURE_LENGTHS '
                     f'{dict(model.sequence_length)} lack targets_context)')


def event_vocabulary_of(model) -> midi_tokens.EventVocabulary:
  """The model's event vocabulary: `InferenceModel.codec` is the tokeniser's own object."""
  return model.codec


def load_notes(midi: Union[str, bytes], sustain: bool = True) -> np.ndarray:
  data = open(midi, 'rb').read() if isinstance(midi, str) else midi
  song = midi_file.read_midi(data)
  if sustain:
    song = midi_file.apply_sustain(song)
  return song.notes


def load_audio(path_or_bytes: Union[str, bytes], resample: bool = False) -> np.ndarray:
  """A PCM WAV file (path or bytes) -> float32 [n] at 16 kHz in [-1, 1): 8-bit unsigned, 16-, 24-
  and 32-bit signed samples, scaled by 2^-(bits - 1); channels are averaged to mono as librosa's
  `load(mono=True)` does.

  By default the file must be at 16 kHz; any other rate raises ValueError.  With resample=True a
  file at any rate is read and mixed down the same way, then resampled to 16 kHz on the GPU as
  `librosa.load(sr=16000)` does (`audio_codecs.resample`: librosa 0.9's kaiser_best, bit for bit
  resampy's loop; preprocessors.py:150-155, 332-333, 518-521).  A 16 kHz file comes back
  unchanged."""
  src = io.BytesIO(path_or_bytes) if isinstance(path_or_bytes, (bytes, bytearray)) else path_or_bytes
  try:
    with wave.open(src, 'rb') as w:
      rate, width, channels = w.getframerate(), w.getsampwidth(), w.getnchannels()
      raw = w.readframes(w.getnframes())
  except (wave.Error, EOFError) as e:
    raise ValueError(f'not a PCM WAV file: {e}') from e
  if rate != 16000 and not resample:
    raise ValueError(f'sample rate {rate} Hz: MelGAN features need 16000 Hz audio; pass '
                     'resample=True to resample it as the reference does (librosa)')
  if width == 1:
    x = (np.frombuffer(raw, np.uint8).astype(np.float32) - 128.0) / 128.0
  elif width == 2:
    x = np.frombuffer(raw, '<i2').astype(np.float32) / 32768.0
  elif width == 3:
    b = np.frombuffer(raw, np.uint8).reshape(-1, 3).astype(np.int32)
    v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
    x = (np.where(v >= 1 << 23, v - (1 << 24), v) / float(1 << 23)).astype(np.float32)
  elif width == 4:
    x = (np.frombuffer(raw, '<i4').astype(np.float64) / float(1 << 31)).astype(np.float32)
  else:
    raise ValueError(f'{8 * width}-bit samples are not supported (8, 16, 24 or 32-bit PCM)')
  x = x.reshape(-1, channels)
  x = (x[:, 0] if channels == 1 else x.mean(axis=1, dtype=np.float32)).astype(np.float32)
  if rate != 16000:
    x = audio_codecs.resample(x, rate, 16000)
  return x


def save_audio(path_or_file, audio, sample_rate: int = 16000) -> None:
  """Writes mono audio [n] (numpy or a tensor, nominally in [-1, 1)) as a 16-bit PCM WAV file to
  a path or a writable binary file object: each sample is clipped to [-1, 1), scaled by 32768 and
  rounded to nearest, so `load_audio` of the file gives the audio quantised to 16 bits back
  exactly.  NaN is written as 0."""
  if torch.is_tensor(audio):
    audio = audio.detach().cpu().numpy()
  x = np.asarray(audio, np.float64)
  if x.ndim != 1:
    raise ValueError(f'save_audio: audio must be mono [n], got shape {x.shape}')
  if int(sample_rate) != sample_rate or sample_rate <= 0:
    raise ValueError(f'save_audio: sample_rate={sample_rate} must be a positive integer')
  q = np.clip(np.rint(np.nan_to_num(x, nan=0.0) * 32768.0), -32768, 32767).astype('<i2')
  with wave.open(path_or_file, 'wb') as w:
    w.setnchannels(1)
    w.setsampwidth(2)
    w.setframerate(int(sample_rate))
    w.writeframes(q.tobytes())


def encode_song_audio(model, samples: np.ndarray) -> Dict[str, Any]:
  """A song's recording -> its ground-truth mels, as the reference's full-song evaluation cuts them
  (`split_full_song` + `encode_audio`, preprocessors.py:60-81, 631-696, 863-921).

  The samples are padded by 320 - n % 320 (a whole hop when n is a multiple), giving num_frames
  hop-frames (`midi_tokens.num_song_frames`); segment s is frames [s * targets, (s + 1) * targets)
  encoded with the 16 frames after it, and the last one is padded with 0.0 to a full segment.  A
  frame depends on its own 640 samples only, so the song is encoded once and cut.
  Returns {'full_gt_encoded': f32 [segments * targets, n_dims], 'num_frames': int}."""
  ac = model.audio_codec
  per_segment = model.sequence_length['targets']
  x = np.asarray(samples, np.float32)
  if x.ndim != 1:
    raise ValueError(f'samples must be 1-D, got shape {x.shape}')
  x = np.pad(x, [0, ac.hop_size - len(x) % ac.hop_size])
  total = len(x) // ac.hop_size
  full = np.zeros((-(-total // per_segment) * per_segment, ac.n_dims), np.float32)
  full[:total] = ac.encode(x)
  return {'full_gt_encoded': full, 'num_frames': total}


def primer_frames(n_samples: int, context_frames: int, hop: int = 320,
                  window: int = 640) -> Tuple[int, int]:
  """(first, count): the recording's frames [first, first + count) that prime a song -- the last
  min(context_frames, n_samples // hop - 1) frames whose whole window lies inside the recording,
  as every context frame of training had real audio under it."""
  if n_samples < window:
    raise ValueError(f'a context recording needs at least {window} samples, got {n_samples}')
  usable = n_samples // hop - 1
  count = min(context_frames, usable)
  return usable - count, count


def audio_context(model, audio, device: Optional[torch.device] = None
                  ) -> Tuple[torch.Tensor, torch.Tensor]:
  """A recording (f32 [n] at 16 kHz, numpy or tensor) -> (ctx f32 [1, C, n_dims], mask int32
  [1, C]) on `device` (default: the model's): its last frames (`primer_frames`) front-filled,
  mask 1 over them and 0 after (the feature converter's sequence_mask layout)."""
  ac = model.audio_codec
  c = model.sequence_length.get('targets_context') or 0
  device = model.engine.device if device is None else device
  a = torch.as_tensor(audio).to(device, torch.float32).contiguous()
  if a.dim() != 1:
    raise ValueError(f'context audio must be 1-D, got shape {tuple(a.shape)}')
  first, count = primer_frames(a.shape[0], c, ac.hop_size)
  span = a[first * ac.hop_size:(first + count + 1) * ac.hop_size]
  ctx = torch.zeros(1, c, ac.n_dims, dtype=torch.float32, device=device)
  ctx[0, :count] = ac.encode(span)[:count]
  mask = torch.zeros(1, c, dtype=torch.int32, device=device)
  mask[0, :count] = 1
  return ctx, mask


def _tokenize(model, notes: np.ndarray, max_segments: Optional[int]):
  """(tokenize_song result, number of segments to synthesise)."""
  ac = model.audio_codec
  lengths = model.sequence_length
  toks = midi_tokens.tokenize_song(
      notes, event_vocabulary_of(model), inputs_length=lengths['inputs'],
      frames_per_segment=lengths['targets'], frame_rate=ac.frame_rate, sample_rate=ac.sample_rate,
      hop_size=ac.hop_size)
  nseg = len(toks.tokens) if max_segments is None else min(max_segments, len(toks.tokens))
  return toks, nseg


def synthesize_song(model, notes: np.ndarray, seed: int = 0, always_mask_context: bool = False,
                    max_segments: Optional[int] = None, context_audio=None) -> Dict[str, Any]:
  """model: an `InferenceModel` (anything with .predict, .sequence_length, .audio_codec, .codec).
  context_audio: a 16 kHz recording (f32 [n], at least 640 samples) whose end conditions the first
  segment (`audio_context`) instead of a masked-out context; not with always_mask_context.

  Returns {'full_pred_encoded': f32 [segments * targets_length, n_dims] in feature units,
  'num_frames': frames that belong to the song, 'tokens': the per-segment model inputs,
  'model_timing': {...}} -- the same keys `beam/evaluation.py` yields for this part.

  A model without a context runs the song's segments as independent rows through
  `synthesize_songs` (each as predict(segment, seed) computes it at batch 1, up to the kernels'
  batch-size dependent rounding; bit for bit at batch_size 1); context_audio and
  always_mask_context are refused for it."""
  if not has_context(model):
    _refuse_context(model, 'context_audio' if context_audio is not None else
                    'always_mask_context' if always_mask_context else None)
    results, _ = synthesize_songs(model, [notes], [seed], max_segments=max_segments)
    return results[0]
  ac = model.audio_codec
  lengths = model.sequence_length
  toks, nseg = _tokenize(model, notes, max_segments)
  ctx_len = lengths.get('targets_context') or 0
  pred = np.zeros((1, ctx_len, ac.n_dims), np.float32)
  primer_mask = None
  if context_audio is not None:
    if always_mask_context:
      raise ValueError('context_audio with always_mask_context: the context would be masked out')
    pred, primer_mask = (t.cpu().numpy() for t in audio_context(model, context_audio))
  full = np.zeros((1, 0, ac.n_dims), np.float32)
  seconds = []
  for i in range(nseg):
    batch = {
        'encoder_input_tokens': toks.tokens[i:i + 1],
        'encoder_continuous_inputs': pred[:1],
        # first segment: nothing to condition on (or the recording); later ones: a full chunk of
        # predicted context
        'encoder_continuous_mask': primer_mask if (i == 0 and primer_mask is not None) else (
            np.zeros if (i == 0 or always_mask_context) else np.ones)((1, ctx_len), np.int32),
        'decoder_target_tokens': np.zeros((1, lengths['targets'], ac.n_dims), np.float32),
    }
    tick = time.time()
    pred, _ = model.predict(batch, seed=seed)
    if i != 0:
      seconds.append(time.time() - tick)
    full = np.concatenate([full, pred[:1]], axis=1)
  seconds_per_chunk = lengths['targets'] * (ac.hop_size / ac.sample_rate)
  per_chunk = float(np.mean(seconds)) if seconds else float('nan')
  return {
      'full_pred_encoded': full[0],
      'num_frames': min(toks.num_frames, nseg * lengths['targets']),
      'tokens': toks.tokens[:nseg],
      'model_timing': {
          'prediction_seconds_per_chunk': per_chunk,
          'predictions_seconds_per_audio_second': per_chunk / seconds_per_chunk,
      },
  }


def chain_songs(predict_rows: PredictRows, token_segments: Sequence[torch.Tensor], slots: int,
                context_frames: int, n_dims: int, device: torch.device, seeds: Sequence[int],
                always_mask_context: bool = False,
                initial_context: Optional[Sequence[Optional[Tuple[torch.Tensor, torch.Tensor]]]] = None
                ) -> Tuple[List[torch.Tensor], List[Dict[str, Any]]]:
  """Chained synthesis of several songs, batched across rows (the scheduling core of
  `synthesize_songs`).

  token_segments[s]: int32 [n_segments_s, inputs_length], the model inputs of song s.  Each round
  has one row per active song (at most `slots`, compacted in order of entry): a song enters as
  soon as a slot is free, in order, and contributes its next segment to every round until it is
  done.  A row's context is its song's previous prediction, kept on `device`; a song's first
  segment (every segment with always_mask_context) gets an all-zero mask, later ones all-one
  masks (beam/evaluation.py:187-203).  initial_context[s], when given and not None, is song s's
  (ctx f32 [1, context_frames, n_dims], mask int32 [1, context_frames]) on `device`, used for its
  first segment instead of the masked-out context (`audio_context`).

  Returns (mel [1, n_segments_s * frames, n_dims] per song, rounds), rounds[k] = {'rows': [(song,
  segment), ...], 'seconds': host wall time of the round, synchronised with the device when the
  output is a CUDA tensor}."""
  if slots < 1:
    raise ValueError(f'slots={slots} must be positive')
  if len(seeds) != len(token_segments):
    raise ValueError(f'{len(seeds)} seeds for {len(token_segments)} songs')
  n_songs = len(token_segments)
  if initial_context is not None:
    if len(initial_context) != n_songs:
      raise ValueError(f'{len(initial_context)} initial contexts for {n_songs} songs')
    if always_mask_context and any(c is not None for c in initial_context):
      raise ValueError('an initial context with always_mask_context: it would be masked out')
    for c in initial_context:
      if c is not None and (tuple(c[0].shape) != (1, context_frames, n_dims)
                            or tuple(c[1].shape) != (1, context_frames)):
        raise ValueError(f'an initial context must be ([1, {context_frames}, {n_dims}], '
                         f'[1, {context_frames}]), got {tuple(c[0].shape)}, {tuple(c[1].shape)}')
  done = [0] * n_songs
  primed = lambda s: initial_context is not None and initial_context[s] is not None and done[s] == 0
  prev: List[Optional[torch.Tensor]] = [None] * n_songs
  outs: List[List[torch.Tensor]] = [[] for _ in range(n_songs)]
  rounds: List[Dict[str, Any]] = []
  active: List[int] = []
  entering = 0
  while True:
    while len(active) < slots and entering < n_songs:
      if len(token_segments[entering]) > 0:
        active.append(entering)
      entering += 1
    if not active:
      break
    toks = torch.stack([token_segments[s][done[s]] for s in active]).to(device, torch.int32)
    zero = torch.zeros(1, context_frames, n_dims, dtype=torch.float32, device=device)
    ctx = torch.cat([initial_context[s][0] if primed(s) else zero if prev[s] is None else prev[s]
                     for s in active])
    first = [done[s] == 0 or always_mask_context for s in active]
    mask = torch.tensor([[0 if f else 1] for f in first], dtype=torch.int32,
                        device=device).expand(len(active), context_frames).contiguous()
    if any(primed(s) for s in active):
      mask = torch.cat([initial_context[s][1].to(torch.int32) if primed(s) else mask[r:r + 1]
                        for r, s in enumerate(active)])
    if toks.is_cuda:
      torch.cuda.synchronize(device)
    tick = time.time()
    mel = predict_rows(toks, ctx, mask, [seeds[s] for s in active])
    if mel.is_cuda:
      torch.cuda.synchronize(mel.device)
    rounds.append({'rows': [(s, done[s]) for s in active], 'seconds': time.time() - tick})
    for r, s in enumerate(active):
      prev[s] = mel[r:r + 1]
      outs[s].append(prev[s])
      done[s] += 1
    active = [s for s in active if done[s] < len(token_segments[s])]
  empty = torch.zeros(1, 0, n_dims, dtype=torch.float32, device=device)
  return [torch.cat(o, dim=1) if o else empty for o in outs], rounds


def batch_segments(predict_segments: PredictSegments, token_segments: Sequence[torch.Tensor],
                   slots: int, n_dims: int, device: torch.device, seeds: Sequence[int]
                   ) -> Tuple[List[torch.Tensor], List[Dict[str, Any]]]:
  """Synthesis of several songs with a model without a context (the scheduling core of
  `synthesize_songs` for it): no segment depends on another, so every segment of every song is an
  independent row.  The rows -- song 0's segments in order, then song 1's, ... -- are packed in
  that order into rounds of `slots` rows (the last one may be shorter), and each row draws its
  noise from its song's seed.

  token_segments[s]: int32 [n_segments_s, inputs_length].  Returns the same as `chain_songs`: (mel
  [1, n_segments_s * frames, n_dims] per song, rounds), rounds[k] = {'rows': [(song, segment),
  ...], 'seconds': host wall time of the round, synchronised with the device when the output is
  a CUDA tensor}."""
  if slots < 1:
    raise ValueError(f'slots={slots} must be positive')
  if len(seeds) != len(token_segments):
    raise ValueError(f'{len(seeds)} seeds for {len(token_segments)} songs')
  rows = [(s, k) for s, segs in enumerate(token_segments) for k in range(len(segs))]
  outs: List[List[torch.Tensor]] = [[] for _ in token_segments]
  rounds: List[Dict[str, Any]] = []
  for first in range(0, len(rows), slots):
    part = rows[first:first + slots]
    toks = torch.stack([token_segments[s][k] for s, k in part]).to(device, torch.int32)
    if toks.is_cuda:
      torch.cuda.synchronize(device)
    tick = time.time()
    mel = predict_segments(toks, [seeds[s] for s, _ in part])
    if mel.is_cuda:
      torch.cuda.synchronize(mel.device)
    rounds.append({'rows': part, 'seconds': time.time() - tick})
    for r, (s, _) in enumerate(part):
      outs[s].append(mel[r:r + 1])
  empty = torch.zeros(1, 0, n_dims, dtype=torch.float32, device=device)
  return [torch.cat(o, dim=1) if o else empty for o in outs], rounds


def synthesize_songs(model, songs: Sequence[np.ndarray], seeds: Optional[Sequence[int]] = None,
                     always_mask_context: bool = False, max_segments: Optional[int] = None,
                     context_audios: Optional[Sequence[Any]] = None
                     ) -> Tuple[List[Dict[str, Any]], Dict[str, float]]:
  """`synthesize_song` for many songs at once: up to model.batch_size songs run side by side, one
  per batch row (`chain_songs`), each drawing its noise from its own seed, so every song comes out
  as `synthesize_song(model, notes, seed)` computes it up to the kernels' batch-size dependent
  rounding.  seeds: one per song, default 0 for every song (the reference's `predict(batch)`).
  context_audios: one recording or None per song, as synthesize_song's context_audio; the
  recordings are encoded on the device and stay there.

  A model without a context runs every segment of every song as an independent row instead
  (`batch_segments`): model.batch_size rows per round, each segment as `predict(segment, seed)`
  of its song computes it; context_audios and always_mask_context are refused for it.

  Returns (one dict per song with synthesize_song's keys, aggregate): model_timing of a song is
  the mean wall time of the rounds that carried its segments after its first; aggregate =
  {'rounds', 'segments', 'wall_seconds' (sum of the round times), 'audio_seconds',
  'x_realtime' (audio seconds per wall second)}."""
  if seeds is None:
    seeds = [0] * len(songs)
  if len(seeds) != len(songs):
    raise ValueError(f'{len(seeds)} seeds for {len(songs)} songs')
  if not has_context(model):
    _refuse_context(model, 'context_audios' if context_audios is not None else
                    'always_mask_context' if always_mask_context else None)
  if context_audios is not None and len(context_audios) != len(songs):
    raise ValueError(f'{len(context_audios)} context recordings for {len(songs)} songs')
  if always_mask_context and context_audios is not None and any(
      a is not None for a in context_audios):
    raise ValueError('context_audios with always_mask_context: the context would be masked out')
  ac = model.audio_codec
  lengths = model.sequence_length
  device = model.engine.device
  tokenized = [_tokenize(model, notes, max_segments) for notes in songs]
  segs = [torch.from_numpy(np.ascontiguousarray(t.tokens[:n], dtype=np.int32)).to(device)
          for t, n in tokenized]
  if has_context(model):
    primers = None if context_audios is None else [
        None if a is None else audio_context(model, a, device) for a in context_audios]
    mels, rounds = chain_songs(
        lambda toks, ctx, mask, row_seeds: model.predict_on_device(toks, ctx, mask, seeds=row_seeds),
        segs, model.batch_size, lengths.get('targets_context') or 0, ac.n_dims, device,
        [int(s) for s in seeds], always_mask_context, primers)
  else:
    mels, rounds = batch_segments(
        lambda toks, row_seeds: model.predict_on_device(toks, None, None, seeds=row_seeds),
        segs, model.batch_size, ac.n_dims, device, [int(s) for s in seeds])
  seconds_per_chunk = lengths['targets'] * (ac.hop_size / ac.sample_rate)
  later: List[List[float]] = [[] for _ in songs]
  for rd in rounds:
    # each round once per song, however many of the song's segments it carried
    for s in {s for s, k in rd['rows'] if k != 0}:
      later[s].append(rd['seconds'])
  results = []
  for s, ((toks, nseg), mel) in enumerate(zip(tokenized, mels)):
    per_chunk = float(np.mean(later[s])) if later[s] else float('nan')
    results.append({
        'full_pred_encoded': mel[0].cpu().numpy(),
        'num_frames': min(toks.num_frames, nseg * lengths['targets']),
        'tokens': toks.tokens[:nseg],
        'model_timing': {
            'prediction_seconds_per_chunk': per_chunk,
            'predictions_seconds_per_audio_second': per_chunk / seconds_per_chunk,
        },
    })
  segments = sum(n for _, n in tokenized)
  wall = float(sum(rd['seconds'] for rd in rounds))
  audio = segments * seconds_per_chunk
  return results, {'rounds': len(rounds), 'segments': segments, 'wall_seconds': wall,
                   'audio_seconds': audio, 'x_realtime': audio / wall if wall > 0 else float('nan')}
