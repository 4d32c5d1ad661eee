"""Full-song synthesis driver: notes (or a MIDI file) -> chained 5.12 s segments -> mel frames.

Library form of the loops the reference keeps in its colab ("Synthesize Audio" cell) and in
`beam/evaluation.py:156-276`: the first segment runs with a masked context, every later one
is conditioned on the previous segment's predicted mel; per-segment wall times are reported
with the reference's `model_timing` fields (first segment excluded, evaluation.py:217-220,
238-247).  The mel -> audio vocoder is outside this path (SURVEY §2).

`synthesize_songs` runs several such chains at once: each round puts the next segment of every
active song into one batch, one song per row, and every row draws its noise from its own song's
seed (`InferenceModel.predict_on_device(..., seeds=)`), so a song comes out as it would alone.
"""

from __future__ import annotations

import time
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from music_spectrogram_diffusion_b200 import midi_file, midi_tokens

# predict_rows(tokens [R, inputs], ctx [R, context, n_dims], mask [R, context], seeds: R ints)
#   -> mel [R, targets, n_dims]; row r must depend on row r of the inputs and seeds[r] only
PredictRows = Callable[[torch.Tensor, torch.Tensor, torch.Tensor, Sequence[int]], torch.Tensor]


def event_vocabulary_of(model) -> midi_tokens.EventVocabulary:
  """The model's event vocabulary: `InferenceModel.codec` is the tokeniser's own object."""
  return model.codec


def load_notes(midi: Union[str, bytes], sustain: bool = True) -> np.ndarray:
  data = open(midi, 'rb').read() if isinstance(midi, str) else midi
  song = midi_file.read_midi(data)
  if sustain:
    song = midi_file.apply_sustain(song)
  return song.notes


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
                    max_segments: Optional[int] = None) -> Dict[str, Any]:
  """model: an `InferenceModel` (anything with .predict, .sequence_length, .audio_codec, .codec).

  Returns {'full_pred_encoded': f32 [segments * targets_length, n_dims] in feature units,
  'num_frames': frames that belong to the song, 'tokens': the per-segment model inputs,
  'model_timing': {...}} -- the same keys `beam/evaluation.py` yields for this part."""
  ac = model.audio_codec
  lengths = model.sequence_length
  toks, nseg = _tokenize(model, notes, max_segments)
  ctx_len = lengths.get('targets_context') or 0
  pred = np.zeros((1, ctx_len, ac.n_dims), np.float32)
  full = np.zeros((1, 0, ac.n_dims), np.float32)
  seconds = []
  for i in range(nseg):
    batch = {
        'encoder_input_tokens': toks.tokens[i:i + 1],
        'encoder_continuous_inputs': pred[:1],
        # first segment: nothing to condition on; later ones: a full chunk of predicted context
        'encoder_continuous_mask': (np.zeros if (i == 0 or always_mask_context) else np.ones)(
            (1, ctx_len), np.int32),
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
                always_mask_context: bool = False) -> Tuple[List[torch.Tensor], List[Dict[str, Any]]]:
  """Chained synthesis of several songs, batched across rows (the scheduling core of
  `synthesize_songs`).

  token_segments[s]: int32 [n_segments_s, inputs_length], the model inputs of song s.  Each round
  has one row per active song (at most `slots`, compacted in order of entry): a song enters as
  soon as a slot is free, in order, and contributes its next segment to every round until it is
  done.  A row's context is its song's previous prediction, kept on `device`; a song's first
  segment (every segment with always_mask_context) gets an all-zero mask, later ones all-one
  masks (beam/evaluation.py:187-203).

  Returns (mel [1, n_segments_s * frames, n_dims] per song, rounds), rounds[k] = {'rows': [(song,
  segment), ...], 'seconds': host wall time of the round, synchronised with the device when the
  output is a CUDA tensor}."""
  if slots < 1:
    raise ValueError(f'slots={slots} must be positive')
  if len(seeds) != len(token_segments):
    raise ValueError(f'{len(seeds)} seeds for {len(token_segments)} songs')
  n_songs = len(token_segments)
  done = [0] * n_songs
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
    ctx = torch.cat([zero if prev[s] is None else prev[s] for s in active])
    first = [done[s] == 0 or always_mask_context for s in active]
    mask = torch.tensor([[0 if f else 1] for f in first], dtype=torch.int32,
                        device=device).expand(len(active), context_frames).contiguous()
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


def synthesize_songs(model, songs: Sequence[np.ndarray], seeds: Optional[Sequence[int]] = None,
                     always_mask_context: bool = False, max_segments: Optional[int] = None
                     ) -> Tuple[List[Dict[str, Any]], Dict[str, float]]:
  """`synthesize_song` for many songs at once: up to model.batch_size songs run side by side, one
  per batch row (`chain_songs`), each drawing its noise from its own seed, so every song comes out
  as `synthesize_song(model, notes, seed)` computes it up to the kernels' batch-size dependent
  rounding.  seeds: one per song, default 0 for every song (the reference's `predict(batch)`).

  Returns (one dict per song with synthesize_song's keys, aggregate): model_timing of a song is
  the mean wall time of the rounds that carried its segments after its first; aggregate =
  {'rounds', 'segments', 'wall_seconds' (sum of the round times), 'audio_seconds',
  'x_realtime' (audio seconds per wall second)}."""
  if seeds is None:
    seeds = [0] * len(songs)
  if len(seeds) != len(songs):
    raise ValueError(f'{len(seeds)} seeds for {len(songs)} songs')
  ac = model.audio_codec
  lengths = model.sequence_length
  device = model.engine.device
  tokenized = [_tokenize(model, notes, max_segments) for notes in songs]
  segs = [torch.from_numpy(np.ascontiguousarray(t.tokens[:n], dtype=np.int32)).to(device)
          for t, n in tokenized]
  mels, rounds = chain_songs(
      lambda toks, ctx, mask, row_seeds: model.predict_on_device(toks, ctx, mask, seeds=row_seeds),
      segs, model.batch_size, lengths.get('targets_context') or 0, ac.n_dims, device,
      [int(s) for s in seeds], always_mask_context)
  seconds_per_chunk = lengths['targets'] * (ac.hop_size / ac.sample_rate)
  later: List[List[float]] = [[] for _ in songs]
  for rd in rounds:
    for s, k in rd['rows']:
      if k != 0:
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
