"""GPU diagnostic (not a test): structured probes of the wgmma GEMM / attention kernels that
make layout mistakes (swizzle, descriptor strides, major-ness) visible in the output."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from music_spectrogram_diffusion_b200 import engine, _native

dev = torch.device('cuda', 0)

def report(name, got, want, tol):
  d = (got - want).abs()
  bad = d > tol
  print(f'[{name}] max={d.max().item():.4e} mean={d.mean().item():.4e} bad={bad.float().mean().item():.4f} finite={torch.isfinite(got).all().item()}')
  if bad.any():
    idx = bad.nonzero()[:12]
    for ix in idx:
      ix = tuple(int(v) for v in ix)
      print('   ', ix, 'got', float(got[ix]), 'want', float(want[ix]))
    if got.dim() == 2:
      rows = bad.any(dim=1).nonzero().flatten()
      cols = bad.any(dim=0).nonzero().flatten()
      print('    bad rows (first 20):', rows[:20].tolist(), ' n=', len(rows))
      print('    bad cols (first 20):', cols[:20].tolist(), ' n=', len(cols))

def probe_gemm():
  for block_n in (0, 64, 96, 128, 192, 256):
    print('--- gemm block_n', block_n)
    for (M, N, K) in [(128, 64, 64), (256, 128, 64), (256, 192, 128), (256, 256, 256), (128, 256, 768), (1024, 768, 768), (4096, 2304, 768)]:
      if block_n and N % block_n:
        continue
      # selection probe: A one-hot -> out[m, n] = W[m % K, n]
      a = torch.zeros(M, K); a[torch.arange(M), torch.arange(M) % K] = 1.0
      w = ((torch.arange(K)[:, None] + 2 * torch.arange(N)[None, :]) % 251).float()
      try:
        got = engine.op_dense_epilogue(a.to(dev), w.to(dev), 'f32', block_n).cpu()
        report(f'gemm-select {M}x{N}x{K}', got, w[torch.arange(M) % K], 0.5)
      except Exception as e:
        print('gemm-select', (M, N, K), 'EXC', e)
        return False
      g = torch.Generator().manual_seed(0)
      a = torch.randn(M, K, generator=g).bfloat16().float()
      w = (torch.randn(K, N, generator=g) / np.sqrt(K)).bfloat16().float()
      try:
        got = engine.op_dense_epilogue(a.to(dev), w.to(dev), 'f32', block_n).cpu()
        report(f'gemm-rand {M}x{N}x{K}', got, a @ w, 1e-2)
      except Exception as e:
        print('gemm-rand', (M, N, K), 'EXC', e)
        return False
  return True

def probe_attn():
  for (nb, H, Lq, Lk) in [(1, 1, 128, 128), (1, 1, 128, 256), (2, 2, 256, 384)]:
    w = H * 64
    g = torch.Generator().manual_seed(1)
    # uniform attention (q = 0): out = mean over keys of V -> isolates the PV (MN-major V) MMA
    q = torch.zeros(nb, Lq, w)
    k = torch.randn(nb, Lk, w, generator=g).bfloat16().float()
    v = ((torch.arange(Lk)[None, :, None] % 7) + (torch.arange(w)[None, None, :] % 5)).float().expand(nb, Lk, w).contiguous()
    try:
      got = engine.op_attention(q.to(dev), k.to(dev), v.to(dev), None, H).cpu()
      report(f'attn-uniform {nb},{H},{Lq},{Lk}', got, v.mean(dim=1, keepdim=True).expand_as(got), 5e-2)
    except Exception as e:
      print('attn-uniform EXC', e); return False
    # one-hot attention: q.k large for key == (query % Lk) -> out[i] = V[i % Lk]: isolates S = QK^T
    q = torch.zeros(nb, Lq, w); kk = torch.zeros(nb, Lk, w)
    # use 64-dim codes: key j has code c_j (random +-1), query i uses 3*c_{i%Lk}
    codes = (torch.randint(0, 2, (Lk, 64), generator=g).float() * 2 - 1)
    for h in range(H):
      kk[:, :, h*64:(h+1)*64] = codes
      q[:, :, h*64:(h+1)*64] = 3.0 * codes[torch.arange(Lq) % Lk]
    v = torch.randn(nb, Lk, w, generator=g).bfloat16().float()
    try:
      got = engine.op_attention(q.to(dev), kk.to(dev), v.to(dev), None, H).cpu()
      logits = torch.einsum('bqhd,bkhd->bhqk', q.view(nb, Lq, H, 64), kk.view(nb, Lk, H, 64))
      want = torch.einsum('bhqk,bkhd->bqhd', torch.softmax(logits, -1), v.view(nb, Lk, H, 64)).reshape(nb, Lq, w)
      report(f'attn-onehot {nb},{H},{Lq},{Lk}', got.reshape(nb*Lq, w), want.reshape(nb*Lq, w), 5e-2)
    except Exception as e:
      print('attn-onehot EXC', e); return False
    q = torch.randn(nb, Lq, w, generator=g).bfloat16().float() * 0.5
    try:
      got = engine.op_attention(q.to(dev), k.to(dev), v.to(dev), None, H).cpu()
      logits = torch.einsum('bqhd,bkhd->bhqk', q.view(nb, Lq, H, 64), k.view(nb, Lk, H, 64))
      want = torch.einsum('bhqk,bkhd->bqhd', torch.softmax(logits, -1), v.view(nb, Lk, H, 64)).reshape(nb, Lq, w)
      report(f'attn-rand {nb},{H},{Lq},{Lk}', got.reshape(nb*Lq, w), want.reshape(nb*Lq, w), 5e-2)
    except Exception as e:
      print('attn-rand EXC', e); return False
  return True

if __name__ == '__main__':
  _native.load()
  print(torch.cuda.get_device_name(0))
  ok = probe_gemm()
  if '--all' in sys.argv:
    probe_attn()
