"""Many songs at once vs one after another: song.synthesize_songs at --batch-size slots against the
same songs through song.synthesize_song at batch 1, in one process.  base_with_context with
synthetic weights, CFG 2.0.  Songs are synthetic arrangements of different lengths (seeded).
Prints one JSON line: aggregate x-realtime of both arms and their ratio, per-song agreement of the
two arms in normalised [-1, 1] units, and the card name / power limit read in the same run.
Needs a GPU; there is no CPU path."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from music_spectrogram_diffusion_b200 import config, inference, midi_tokens as M, song, weights


def synthetic_song(rng, n_segments, seconds_per_segment):
  """A three-instrument arrangement that tokenises into exactly n_segments segments."""
  dur = n_segments * seconds_per_segment - 0.5
  rows = []
  for prog in (0, 33, 48):
    t = 0.0
    while t < dur - 0.5:
      d = float(rng.uniform(0.1, 0.8))
      rows.append((t, min(t + d, dur), int(rng.integers(40, 80)), int(rng.integers(40, 120)), prog,
                   False))
      t += float(rng.uniform(0.1, 0.5))
  return M.make_notes(rows)


def gpu_card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    name, power = (s.strip() for s in out[0].split(','))
    return {'gpu': name, 'power_limit': power}
  except Exception as e:  # pylint: disable=broad-except
    return {'gpu': torch.cuda.get_device_name(0), 'power_limit': f'unavailable ({e})'}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--songs', type=int, default=8)
  ap.add_argument('--min-segments', type=int, default=4)
  ap.add_argument('--max-segments', type=int, default=12)
  ap.add_argument('--batch-size', type=int, default=8)
  ap.add_argument('--diffusion-steps', type=int, default=1000)
  ap.add_argument('--song-seed', type=int, default=0, help='generator of the synthetic songs')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    print(json.dumps({'error': 'no CUDA device: songs_bench measures the H100 path only'}))
    sys.exit(2)

  t5 = config.t5_base()
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = args.diffusion_steps
  diff.classifier_free_guidance.eval_condition_weight = 2.0
  lengths = dict(config.TASK_FEATURE_LENGTHS_CONTEXT)
  params = weights.synthetic_params(t5, lengths['inputs'], lengths['targets'],
                                    lengths['targets_context'], 128, seed=0)
  batched = inference.InferenceModel.from_config(t5, diff, lengths, 'synthetic:0', args.batch_size,
                                                 params=params)
  single = inference.InferenceModel.from_config(t5, diff, lengths, 'synthetic:0', 1, params=params)
  ac = batched.audio_codec
  seconds_per_segment = lengths['targets'] * ac.hop_size / ac.sample_rate
  rng = np.random.default_rng(args.song_seed)
  nsegs = [int(n) for n in rng.integers(args.min_segments, args.max_segments + 1, args.songs)]
  songs = [synthetic_song(rng, n, seconds_per_segment) for n in nsegs]
  seeds = [0] * len(songs)   # the reference's predict(batch) default, every song

  # warm-up outside the timed window: one round at every batch size the batched run will use, one
  # batch-1 segment on the single-song model
  slots = args.batch_size
  dev = batched.engine.device
  _, rounds = song.chain_songs(lambda t, c, m, s: torch.zeros(len(s), 1, 1), [torch.zeros(n, 1)
                               for n in nsegs], slots, 1, 1, torch.device('cpu'), seeds)
  sizes = sorted({len(r['rows']) for r in rounds})
  C, T, nd = lengths['targets_context'], lengths['inputs'], ac.n_dims
  for b in sizes:
    batched.predict_on_device(torch.full((b, T), 1, dtype=torch.int32, device=dev),
                              torch.zeros(b, C, nd, device=dev),
                              torch.zeros(b, C, dtype=torch.int32, device=dev), seeds=[0] * b)
  song.synthesize_song(single, songs[0], max_segments=1)
  torch.cuda.synchronize()

  t0 = time.time()
  res_b, agg = song.synthesize_songs(batched, songs, seeds)
  torch.cuda.synchronize()
  wall_b = time.time() - t0
  assert agg['segments'] == sum(nsegs), (agg, nsegs)
  print(f'batched: {wall_b:.1f} s for {sum(nsegs)} segments', file=sys.stderr)
  t0 = time.time()
  res_s = [song.synthesize_song(single, n, seed=s) for n, s in zip(songs, seeds)]
  torch.cuda.synchronize()
  wall_s = time.time() - t0

  span = ac.max_value - ac.min_value
  agreement = []
  for rb, rs in zip(res_b, res_s):
    e = np.abs(rb['full_pred_encoded'].astype(np.float64) - rs['full_pred_encoded']) / span * 2.0
    agreement.append({'mean': float(e.mean()), 'p99': float(np.quantile(e, 0.99)),
                      'share_01': float((e > 0.1).mean())})
  audio = sum(nsegs) * seconds_per_segment
  out = {
      'songs': len(songs), 'segments_per_song': nsegs, 'segments': sum(nsegs),
      'diffusion_steps': args.diffusion_steps, 'batch_size': slots, 'model': 'base_with_context',
      'batch_sizes_used': sizes,
      'batched': {'x_realtime': round(audio / wall_b, 3), 'wall_seconds': round(wall_b, 3),
                  'rounds': agg['rounds'], 'round_seconds': round(agg['wall_seconds'], 3)},
      'serial': {'x_realtime': round(audio / wall_s, 3), 'wall_seconds': round(wall_s, 3)},
      'batched_over_serial': round(wall_s / wall_b, 3),
      'agreement': agreement,
      'agreement_worst': {k: max(a[k] for a in agreement) for k in ('mean', 'p99', 'share_01')},
  }
  out.update(gpu_card())
  print(json.dumps(out))


if __name__ == '__main__':
  main()
