"""Per-launch table of the decoder GEMMs as one replayed diffusion step runs them (CUPTI through
torch.profiler, as bench.py's `graph_timeline`): for each launch site (input projection, QKV,
self-out, cross-q, cross-out, wi, wo, output projection) its M x N x K, epilogue, tile width, grid,
mean in-graph duration, its summed critical-path share of the step, TFLOP/s and the share of the
989 TFLOP/s dense-bf16 data-sheet bound.  The GEMM launches are labelled by their order in the
step (run_decoder / decoder_layers of engine.cu), which the script checks against the launch
count."""
import argparse, json, os, re, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from music_spectrogram_diffusion_b200 import inference

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense bf16

ap = argparse.ArgumentParser()
ap.add_argument('--model', default='base')
ap.add_argument('--segments', type=int, default=8)
ap.add_argument('--diffusion-steps', type=int, default=12)
ap.add_argument('--out', default=None, help='also write the table as JSON here')
args = ap.parse_args()
t5, diff, lengths = bench.model_configs(args)
model = inference.InferenceModel.from_config(t5, diff, lengths, 'synthetic:0', args.segments, 0)
eng = model.engine
dev = eng.device
b = bench.synthetic_batch(args.segments, lengths, 100)
eng.encode(torch.from_numpy(b['encoder_input_tokens']).to(dev),
           torch.from_numpy(b['encoder_continuous_inputs']).to(dev),
           torch.from_numpy(b['encoder_continuous_mask']).to(dev))

# launch sites in step order: (label, M, N, K, epilogue)
B, Nf, d = args.segments, lengths['targets'], t5.emb_dim
hh, F, nd = t5.num_heads * t5.head_dim, t5.mlp_dim, 128
R, Rc = 2 * B * Nf, B * Nf  # both guidance passes; the conditional pass cross-attends
layer = [('qkv', R, 3 * hh, d, 'bf16 + row scale + bias'), ('self-out', R, d, hh, 'resid + prep'),
         ('cross-q', Rc, hh, d, 'bf16 + row scale'), ('cross-out', Rc, d, hh, 'resid + prep'),
         ('wi', R, 2 * F, d, 'gated GELU + row scale + bias'), ('wo', R, d, F, 'resid + prep')]
sites = [('in-proj', B * Nf, d, 3 * nd, 'position (rows duplicated)')]
for l in range(t5.num_decoder_layers):
  sites += [s if not (l + 1 == t5.num_decoder_layers and s[0] == 'wo') else ('wo', R, d, F, 'resid')
            for s in layer]
sites.append(('out-proj', R, nd, 3 * d, 'f32'))

for _ in range(2):
  eng.sample(seed=1)
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
  eng.sample(seed=2)
  torch.cuda.synchronize()
path = os.path.join(tempfile.mkdtemp(), 'trace.json')
prof.export_chrome_trace(path)
ev = sorted((e for e in json.load(open(path))['traceEvents'] if e.get('cat') == 'kernel'),
            key=lambda e: e['ts'])
steps = int(eng.cfg.num_steps)
pre = next(k for k in range(4) if (len(ev) - k) % steps == 0)
nodes = (len(ev) - pre) // steps
step = ev[pre + (steps // 2) * nodes:][:nodes]
t0, prev_end = step[0]['ts'], step[0]['ts']
gemms = []
for e in step:
  end = e['ts'] + e['dur']
  crit = max(0.0, end - prev_end)
  prev_end = max(prev_end, end)
  m = re.search(r'gemm_bf16_wgmma_kernel<(\d+)>', e['name'])
  if m:
    gemms.append((int(m.group(1)), e.get('args', {}).get('grid'), e['dur'], crit))
assert len(gemms) == len(sites), f'{len(gemms)} GEMM launches in the step, expected {len(sites)}'
step_us = prev_end - t0

table = {}
for (label, M, N, K, epi), (bn, grid, dur, crit) in zip(sites, gemms):
  r = table.setdefault(label, dict(site=label, M=M, N=N, K=K, epilogue=epi, bn=set(), grid=set(),
                                   launches=0, dur_us=0.0, critical_us=0.0))
  r['bn'].add(bn); r['grid'].add(str(grid))
  r['launches'] += 1; r['dur_us'] += dur; r['critical_us'] += crit
rows = []
for r in table.values():
  n = r['launches']
  flop = 2.0 * r['M'] * r['N'] * r['K']
  mean = r['dur_us'] / n
  tf = flop / (mean * 1e-6) / 1e12
  rows.append(dict(r, bn='/'.join(map(str, sorted(r['bn']))), grid=' '.join(sorted(r['grid'])),
                   mean_us=round(mean, 2), dur_us=round(r['dur_us'], 1),
                   critical_us=round(r['critical_us'], 1), tflops=round(tf, 1),
                   share_of_bound=round(tf / PEAK_TFLOPS, 3)))
gemm_crit = sum(r['critical_us'] for r in rows)
print(f'{torch.cuda.get_device_name()}: step {step_us:.1f} us in graph, {len(gemms)} GEMM launches, '
      f'GEMM critical path {gemm_crit:.1f} us')
print('| launch | M x N x K | epilogue | BN | grid | launches | mean us | critical us / step | TFLOP/s | share of 989 |')
print('|---|---|---|---|---|---|---|---|---|---|')
for r in rows:
  print(f"| {r['site']} | {r['M']} x {r['N']} x {r['K']} | {r['epilogue']} | {r['bn']} | {r['grid']} | "
        f"{r['launches']} | {r['mean_us']} | {r['critical_us']} | {r['tflops']} | {r['share_of_bound']} |")
if args.out:
  os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
  json.dump({'step_us': step_us, 'gemm_critical_us': gemm_crit, 'rows': rows}, open(args.out, 'w'), indent=1)
