"""GEMM micro-benchmark over the decoder's shapes and tile widths, 0 = automatic (GPU)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from music_spectrogram_diffusion_b200 import _native
lib = _native.load()
torch.zeros(1, device='cuda')
EPI = {0: 'bf16', 1: 'f32', 2: 'resid', 3: 'gated'}
shapes = [('qkv', 4096, 2304, 768, 0), ('wi', 4096, 4096, 768, 3), ('wo', 4096, 768, 2048, 2),
          ('out', 4096, 768, 768, 2), ('crossq', 2048, 768, 768, 0), ('crossout', 2048, 768, 768, 2),
          ('big', 8192, 8192, 8192, 0),
          ('big_k768', 8192, 8192, 768, 0)]
for name, M, N, K, epi in shapes:
  for bn in (0, 256, 192, 128, 96, 64):
    if bn and N % bn: continue
    if bn == 96 and epi in (0, 3): continue  # 96 only for fp32 outputs
    ms = ctypes.c_float(0)
    rc = lib.msd_bench_gemm(M, N, K, epi, bn, 20, ctypes.byref(ms))
    if rc != 0:
      print(name, bn, 'ERR', lib.msd_last_error().decode()); continue
    tf = 2.0 * M * N * K / (ms.value * 1e-3) / 1e12
    print(f'{name:9s} M={M} N={N} K={K} epi={EPI[epi]:5s} bn={bn:3d}: {ms.value*1e3:8.1f} us  {tf:7.1f} TF/s')
