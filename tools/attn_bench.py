"""Attention micro-benchmark over the decoder's shapes (GPU): back-to-back launches, warm.
Environment: MSD_ATTN_BKV / MSD_ATTN_SPLITS / MSD_ATTN_TAIL select the variant."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from music_spectrogram_diffusion_b200 import _native
lib = _native.load()
torch.zeros(1, device='cuda')
shapes = [('self  B=8', 16, 12, 256, 256), ('cross B=8', 8, 12, 256, 2304),
          ('self  B=1', 2, 12, 256, 256), ('cross B=1', 1, 12, 256, 2304),
          ('tokenenc B=8', 8, 12, 2048, 2048)]
for name, nb, H, Lq, Lk in shapes:
  ms = ctypes.c_float(0)
  rc = lib.msd_bench_attention(nb, H, Lq, Lk, 20, ctypes.byref(ms))
  if rc != 0:
    print(name, 'ERR', lib.msd_last_error().decode()); continue
  tf = 4.0 * nb * H * Lq * Lk * 64 / (ms.value * 1e-3) / 1e12
  print(f'{name:13s} nb={nb:2d} Lq={Lq} Lk={Lk}: {ms.value * 1e3:8.1f} us  {tf:7.1f} TF/s', flush=True)
