"""In-graph kernel timeline of one diffusion step (CUPTI through torch.profiler): start offset,
duration and critical-path contribution of every kernel of a replayed step graph (bench.py's
`graph_timeline`, which the bench line also carries as `in_graph`), written out in full."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from music_spectrogram_diffusion_b200 import inference

ap = argparse.ArgumentParser()
ap.add_argument('--model', default='base')
ap.add_argument('--segments', type=int, default=8)
ap.add_argument('--diffusion-steps', type=int, default=12)
ap.add_argument('--precision', default='bf16')
ap.add_argument('--out', default='graph_timeline.json')
args = ap.parse_args()
t5, diff, lengths = bench.model_configs(args)
model = inference.InferenceModel.from_config(t5, diff, lengths, 'synthetic:0', args.segments, 0,
                                             precision=args.precision)
eng = model.engine
dev = eng.device
b = bench.synthetic_batch(args.segments, lengths, 100)
eng.encode(torch.from_numpy(b['encoder_input_tokens']).to(dev),
           torch.from_numpy(b['encoder_continuous_inputs']).to(dev),
           torch.from_numpy(b['encoder_continuous_mask']).to(dev))
summary, rows = bench.graph_timeline(eng)
os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
json.dump({'summary': summary, 'kernels': rows}, open(args.out, 'w'), indent=0)
print(json.dumps(summary))
for r in (rows or [])[:40]:
  print(r)
