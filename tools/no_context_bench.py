"""The no-context model (models.DiffusionModel + network.Transformer) against base_with_context, in
one process on one GPU.  Base size, synthetic weights, CFG 2.0.

1. Per-segment throughput: --segments segments x --diffusion-steps steps, device-resident
   Engine.encode + Engine.sample_rows timed with CUDA events, the two models alternated
   --reps times; frames/s of each, plus the encode share.
2. One --song-segments-segment synthetic song: the context model chained at batch 1
   (song.synthesize_song) against the no-context model, whose segments are independent rows, at
   each --song-batch size; x-realtime of each.

Prints one JSON line with the card name and power limit read in the same run.  Needs a GPU; there
is no CPU path."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from music_spectrogram_diffusion_b200 import config, engine, inference, song, weights
from tools.songs_bench import gpu_card, synthetic_song


def _diffusion(steps):
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = steps
  diff.classifier_free_guidance.eval_condition_weight = 2.0
  return diff


def throughput(args, t5, lengths_ctx, params_ctx, params_nc):
  T, N, C = lengths_ctx['inputs'], lengths_ctx['targets'], lengths_ctx['targets_context']
  B = args.segments
  diff = _diffusion(args.diffusion_steps)
  engines = {}
  for name, ctx_len, params in (('no_context', 0, params_nc), ('with_context', C, params_ctx)):
    eng = engine.Engine(engine.make_msd_config(t5, diff, T, N, ctx_len, max_batch=B), 0)
    eng.load_weights(params)
    engines[name] = eng
  dev = engines['no_context'].device
  rng = np.random.default_rng(0)
  toks = torch.from_numpy(rng.integers(3, 1391, (B, T)).astype(np.int32)).to(dev)
  ctx = torch.from_numpy(rng.uniform(-11.0, 4.0, (B, C, 128)).astype(np.float32)).to(dev)
  cmask = torch.ones(B, C, dtype=torch.int32, device=dev)
  seeds = list(range(B))
  out = torch.empty(B, N, 128, dtype=torch.float32, device=dev)

  def run(name):
    eng = engines[name]
    e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    e0.record()
    if name == 'no_context':
      eng.encode(toks, None, None)
    else:
      eng.encode(toks, ctx, cmask)
    e1.record()
    eng.sample_rows(seeds, out=out)
    e2.record()
    e2.synchronize()
    return e0.elapsed_time(e1) / 1e3, e1.elapsed_time(e2) / 1e3

  for name in engines:   # warm-up: modules, the step graph of this batch size
    run(name)
  times = {name: [] for name in engines}
  for _ in range(args.reps):
    for name in engines:
      times[name].append(run(name))
  res = {}
  for name, ts in times.items():
    enc = [t[0] for t in ts]
    tot = [t[0] + t[1] for t in ts]
    res[name] = {'frames_per_s': [round(B * N / t, 1) for t in tot],
                 'encode_ms': [round(1e3 * t, 2) for t in enc],
                 'step_ms': [round(1e3 * t[1] / args.diffusion_steps, 4) for t in ts]}
  for eng in engines.values():
    eng.close()
  return res


def one_song(args, t5, lengths_ctx, params_ctx, params_nc):
  diff = _diffusion(args.diffusion_steps)
  lengths_nc = {'inputs': lengths_ctx['inputs'], 'targets': lengths_ctx['targets']}
  chained = inference.InferenceModel.from_config(t5, diff, lengths_ctx, 'synthetic:0', 1,
                                                 params=params_ctx)
  ac = chained.audio_codec
  seconds_per_segment = lengths_ctx['targets'] * ac.hop_size / ac.sample_rate
  notes = synthetic_song(np.random.default_rng(1), args.song_segments, seconds_per_segment)
  n = song._tokenize(chained, notes, None)[1]
  assert n == args.song_segments, (n, args.song_segments)
  audio = n * seconds_per_segment

  def timed(model):
    song.synthesize_song(model, notes, max_segments=1)   # warm-up
    if model.batch_size > 1:
      # every batch size the rounds use: full rounds and the remainder
      sizes = {model.batch_size, n % model.batch_size or model.batch_size}
      dev = model.engine.device
      for b in sizes:
        model.predict_on_device(torch.ones(b, lengths_ctx['inputs'], dtype=torch.int32, device=dev),
                                None, None, seeds=[0] * b)
    torch.cuda.synchronize()
    t0 = time.time()
    r = song.synthesize_song(model, notes)
    torch.cuda.synchronize()
    wall = time.time() - t0
    return {'x_realtime': round(audio / wall, 3), 'wall_seconds': round(wall, 3)}, r

  res = {'segments': n, 'audio_seconds': round(audio, 2)}
  res['with_context_chained_batch1'], _ = timed(chained)
  del chained
  torch.cuda.empty_cache()
  for b in args.song_batch:
    model = inference.InferenceModel.from_config(t5, diff, lengths_nc, 'synthetic:0', b,
                                                 params=params_nc)
    res[f'no_context_batch{b}'], _ = timed(model)
    res[f'no_context_batch{b}']['rounds'] = -(-n // b)
    del model
    torch.cuda.empty_cache()
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--segments', type=int, default=8)
  ap.add_argument('--diffusion-steps', type=int, default=1000)
  ap.add_argument('--reps', type=int, default=3, help='alternated timings of each model')
  ap.add_argument('--song-segments', type=int, default=12)
  ap.add_argument('--song-batch', type=int, nargs='+', default=[8, 12])
  ap.add_argument('--no-song', action='store_true')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    print(json.dumps({'error': 'no CUDA device: no_context_bench measures the H100 path only'}))
    sys.exit(2)
  out = dict(gpu_card())
  t5 = config.t5_base()
  lengths = dict(config.TASK_FEATURE_LENGTHS_CONTEXT)
  T, N, C = lengths['inputs'], lengths['targets'], lengths['targets_context']
  params_ctx = weights.synthetic_params(t5, T, N, C, 128, seed=0)
  params_nc = weights.synthetic_params(t5, T, N, None, 128, seed=0)
  out.update({'model': 'base', 'cfg_weight': 2.0, 'diffusion_steps': args.diffusion_steps,
              'segments': args.segments})
  out['throughput'] = throughput(args, t5, lengths, params_ctx, params_nc)
  if not args.no_song:
    out['song'] = one_song(args, t5, lengths, params_ctx, params_nc)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
