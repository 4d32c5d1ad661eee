"""Runs encode + a few uncaptured diffusion steps of the bench workload; meant to be wrapped in
ncu."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from music_spectrogram_diffusion_b200 import inference

ap = argparse.ArgumentParser()
ap.add_argument('--model', default='base')
ap.add_argument('--segments', type=int, default=8)
ap.add_argument('--diffusion-steps', type=int, default=1000)
ap.add_argument('--reps', type=int, default=1)
args = ap.parse_args()
t5, diff, lengths = bench.model_configs(args)
model = inference.InferenceModel.from_config(t5, diff, lengths, 'synthetic:0', args.segments, 0)
eng = model.engine
dev = eng.device
b = bench.synthetic_batch(args.segments, lengths, 100)
eng.encode(torch.from_numpy(b['encoder_input_tokens']).to(dev),
           torch.from_numpy(b['encoder_continuous_inputs']).to(dev),
           torch.from_numpy(b['encoder_continuous_mask']).to(dev))
torch.cuda.synchronize()
prof = eng.profile_step(step_i=args.diffusion_steps // 2, reps=args.reps)
print(json.dumps(prof))
