"""-m gpu: the tile width the GEMM picks on its own (block_n 0), as
msd_op_gemm_view reports it.  The CTAs are persistent, one per SM, so a launch takes
ceil(tiles / SMs) tile times and a tile costs about BN + 64 column-units: the width with the least
ceil(tiles / SMs) * (BN + 64) runs, the wider one on a tie, and 96 only when the output is fp32.
At 132 SMs (H100 SXM) that is 192 for the decoder's QKV, 96 for its cross-attention output
projection and 256 for large square products."""
import pytest
import torch

from music_spectrogram_diffusion_b200 import engine

pytestmark = pytest.mark.gpu

# (M, N, epilogue, width at 132 SMs)
SHAPES = [
    (4096, 2304, 'bf16', 192),       # QKV
    (4096, 768, 'f32', 192),         # self-attention out / wo
    (2048, 768, 'bf16', 128),        # cross-q
    (2048, 768, 'f32', 96),          # cross-attention out
    (4096, 4096, 'gated_gelu', 256),  # wi
    (4096, 128, 'f32', 64),          # output projection
    (8192, 8192, 'bf16', 256),
    (16384, 2304, 'bf16', 256),      # encoder QKV
]


def _rule(m, n, epilogue, sms):
  best, best_cost = 0, 0
  for bn in (256, 192, 128, 96, 64):
    if n % bn or (bn == 96 and epilogue != 'f32'):
      continue
    cost = -(-(m // 128) * (n // bn) // sms) * (bn + 64)
    if best == 0 or cost < best_cost:
      best, best_cost = bn, cost
  return best


@pytest.mark.parametrize('m,n,epilogue,at_132', SHAPES)
def test_gemm_picks_the_width_with_the_fewest_waves(m, n, epilogue, at_132):
  dev = torch.device('cuda:0')
  sms = torch.cuda.get_device_properties(dev).multi_processor_count
  k = 64
  a = torch.zeros(m, k, dtype=torch.bfloat16, device=dev)
  w = torch.zeros(n, k, dtype=torch.bfloat16, device=dev)
  cols = n // 2 if epilogue == 'gated_gelu' else n
  out = torch.full((m, cols), float('nan'), dtype=torch.float32 if epilogue == 'f32' else torch.bfloat16,
                   device=dev)
  bn = engine.op_gemm_view(a, 0, k, w, 0, k, m, n, k, epilogue, out, 0, cols)
  torch.cuda.synchronize()
  assert bn == _rule(m, n, epilogue, sms)
  if sms == 132:
    assert bn == at_132
  assert bool((out == 0).all())  # zero operands: every tile was written
