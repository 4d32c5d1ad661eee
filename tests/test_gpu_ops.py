"""-m gpu: operator-level parity of the sm_90a kernels against the oracle's restatement of
msd/layers.py (same shape of test as layers_test.py:375-387 / 285-330 / 450-484, at sizes the
tensor-core kernels accept)."""
import numpy as np
import pytest
import torch

from oracle import msd_oracle as O
from tests import test_gpu_attention_views as AV
from tests.helpers import bf16_round

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('block_n', [0, 64, 96, 128, 192, 256])
@pytest.mark.parametrize('M,N,K', [(128, 768, 64), (256, 768, 128), (512, 2304, 768),
                                   (384, 768, 384), (2048 + 128, 1536, 2048),
                                   # the decoder's fp32-output projections at base width and B = 8,
                                   # where block_n 0 picks 192 (4096 rows) or 96 (2048 rows) at 132 SMs
                                   (4096, 768, 768), (4096, 768, 2048), (2048, 768, 768), (2048, 768, 1536)])
def test_dense_general(cuda_device, M, N, K, block_n):
  from music_spectrogram_diffusion_b200 import engine
  if block_n and N % block_n:
    pytest.skip('tile width does not divide N')
  g = torch.Generator().manual_seed(M + N + K)
  a = bf16_round(torch.randn(M, K, generator=g))
  w = bf16_round(torch.randn(K, N, generator=g) / np.sqrt(K))
  got = engine.op_dense_epilogue(a.to(cuda_device), w.to(cuda_device), 'f32', block_n).cpu()
  want = O.dense_general(a.double(), w.double()).float()
  err = (got - want).abs().max().item()
  assert err < 2e-4 * np.sqrt(K), f'max err {err}'


@pytest.mark.parametrize('nb,heads,Lq,Lk,tail,masked', [
    (2, 2, 128, 256, 1, False), (2, 3, 256, 384, 1, True), (2, 3, 256, 384, 2, True),
    (1, 2, 256, 2304, 5, True), (2, 2, 256, 768, 2, 'head'), (3, 2, 128, 256, 1, True),
    (8, 12, 256, 768, 0, False), (8, 12, 256, 2304, 0, True)])
def test_dot_product_attention_tail_split(cuda_device, monkeypatch, nb, heads, Lq, Lk, tail, masked):
  """128-key instance: long/short CTA pairs (the last `tail` key blocks go to a second CTA, merged
  by the combine kernel; tail 0 = the automatic choice); run twice to check that a launch leaves
  nothing behind."""
  from music_spectrogram_diffusion_b200 import engine
  monkeypatch.setenv('MSD_ATTN_BKV', '128')
  monkeypatch.setenv('MSD_ATTN_SPLITS', '1')
  monkeypatch.setenv('MSD_ATTN_TAIL', str(tail))
  g = torch.Generator().manual_seed(nb * 77 + Lk + tail)
  w = heads * 64
  q = bf16_round(torch.randn(nb, Lq, w, generator=g) * 0.5)
  k = bf16_round(torch.randn(nb, Lk, w, generator=g) * 0.5)
  v = bf16_round(torch.randn(nb, Lk, w, generator=g))
  mask = None
  if masked:
    mask = (torch.rand(nb, Lk, generator=g) > 0.3).to(torch.int32)
    if masked == 'head':
      mask[0, :Lk - 128] = 0                   # the long CTA of batch 0 has nothing to attend to
    else:
      mask[0, Lk // 2:] = 0                    # the short CTA of batch 0 has nothing to attend to
    if nb > 2:
      mask[2, :] = 0                           # neither has -> zeros
  q, k, v = q.to(cuda_device), k.to(cuda_device), v.to(cuda_device)
  mask = None if mask is None else mask.to(cuda_device)
  want, wabs = AV.reference(q, k, v, mask)
  for run in range(2):
    got = engine.op_attention(q, k, v, mask, heads)
    AV.check_rounding_bound(got, want, wabs, f'nb={nb} Lk={Lk} tail={tail} masked={masked} run {run}')


def _pack_gated_cols(b0, b1):
  """Accumulator column order of the gated projection: 32 columns of wi_0, 32 of wi_1, ..."""
  F = b0.shape[-1]
  return torch.stack([b0.view(F // 32, 32), b1.view(F // 32, 32)], dim=1).reshape(2 * F)


@pytest.mark.parametrize('gated', [False, True])
@pytest.mark.parametrize('M,d,K,N2,split_row,bn1,bn2', [
    (4096, 768, 768, 2304, 2048, 0, 0),      # self-attention projection -> QKV of the B = 8 step
    (4096, 768, 2048, 2048, 4096, 192, 256),  # wo -> next layer (explicit widths)
    (512, 768, 768, 768, 256, 64, 64),        # batch 1: 12 column tiles of partial row sums
    (4096, 768, 768, 768, 4096, 64, 0),       # 192 tiles of 64 columns: more CTAs than SMs
    (1280, 768, 512, 768, 600, 256, 0),       # 8 chunks per tile (ring refills), ragged split row
    (384, 512, 512, 1024, 128, 128, 0),       # odd number of 128-row blocks, other width
    (256, 256, 128, 256, 0, 256, 128)])       # one column tile, every row in the "hi" group
def test_deferred_normalisation_pair(cuda_device, M, d, K, N2, split_row, bn1, bn2, gated):
  """EPI_RESID_PREP + the row-scale / bias-row epilogues (kernels.h GemmPrep / GemmRowScale): the
  pre-norm (+FiLM) of layers.py:632-666 split into a column gain where x is produced and a row
  scale where the next accumulator is drained.  Checked (a) tightly against the same split written
  in fp64 and (b) against the plain formulation norm -> FiLM -> dense of the oracle."""
  from music_spectrogram_diffusion_b200 import engine
  g = torch.Generator().manual_seed(M + d + K + N2 + gated)
  a = bf16_round(torch.randn(M, K, generator=g))
  w_out = bf16_round(torch.randn(K, d, generator=g) / np.sqrt(K))
  x = torch.randn(M, d, generator=g) * 3
  x[5] *= 30.0                                   # one row with a very different scale
  gamma = 1 + 0.1 * torch.randn(2, d, generator=g)
  fs = 0.2 * torch.randn(2, d, generator=g)
  fb = 0.2 * torch.randn(2, d, generator=g)
  gain = gamma * (1 + fs)                        # rows < split_row use [0], the others [1]
  w2 = bf16_round(torch.randn(d, N2, generator=g) / np.sqrt(d))
  w2b = bf16_round(torch.randn(d, N2, generator=g) / np.sqrt(d)) if gated else None
  sel = (torch.arange(M) >= split_row).long()
  # the bias row is one vector for the whole call: use group 0's FiLM bias for every row
  bias0 = fb[0].double() @ w2.double()
  bias1 = fb[0].double() @ w2b.double() if gated else None
  bias = (_pack_gated_cols(bias0, bias1) if gated else bias0).float()
  dev = cuda_device
  x_out, y = engine.op_dense_deferred_norm(
      a.to(dev), w_out.to(dev), x.to(dev), gain[0].to(dev), gain[1].to(dev), split_row, w2.to(dev),
      None if w2b is None else w2b.to(dev), bias.to(dev), bn1, bn2)
  x_out, y = x_out.cpu(), y.cpu()
  # stage 1: the residual stream
  xw = (x.double() + O.dense_general(a.double(), w_out.double()))
  assert (x_out - xw.float()).abs().max().item() < 2e-4 * np.sqrt(K) * 4
  # (a) the split formulation in fp64 from the device's own x_out
  xo = x_out.double()
  inv = torch.rsqrt((xo * xo).mean(-1, keepdim=True) + 1e-6)
  opnd = bf16_round((xo * gain[sel].double()).float()).double()
  u = inv * (opnd @ w2.double()) + bias0
  if gated:
    u1 = inv * (opnd @ w2b.double()) + bias1
    want = (O.gelu_tanh(u) * u1).float()
    tol = 2.0 ** -8 * want.abs() + 1.5e-3 * u1.abs().float() + 2e-3
  else:
    want = u.float()
    tol = 2.0 ** -8 * want.abs() + 2e-3
  err = (y - want).abs()
  assert (err <= tol).all(), (err - tol).max().item()
  # (b) the reference order of operations: rmsnorm * scale, FiLM, dense (fp64), bf16-level agreement
  n = O.layer_norm(xw.float(), torch.ones(d)).double() * gain[sel].double() + fb[0].double()
  r = n @ w2.double()
  ref = (O.gelu_tanh(r) * (n @ w2b.double())).float() if gated else r.float()
  rel = (y - ref).abs().mean().item() / ref.abs().mean().item()
  assert rel < 1e-2, rel


@pytest.mark.parametrize('bkv,draw', [(64, 1), (64, 0), (128, 1), (128, 0)])
@pytest.mark.parametrize('splits', [0, 1, 3])
@pytest.mark.parametrize('nb,heads,Lq,Lk,masked', [
    (1, 1, 128, 128, False), (2, 2, 128, 256, False), (2, 3, 256, 384, True),
    (1, 2, 256, 2304, True), (3, 2, 128, 128, True), (2, 2, 256, 768, True),
    (16, 12, 256, 256, False), (8, 12, 256, 2304, True)])
def test_dot_product_attention(cuda_device, monkeypatch, nb, heads, Lq, Lk, masked, splits, bkv, draw):
  """Both instances of the kernel (64-key and 128-key blocks).  splits: 0 = automatic split-KV
  choice, 1 = single pass, 3 = forced 3-way split through the combine kernel; draw: two
  independent random draws of the inputs and the mask.  The last two shapes are the B = 8 decoder's
  self- and cross-attention.  Run twice: a launch leaves nothing behind in the workspace."""
  from music_spectrogram_diffusion_b200 import engine
  if splits == 3 and (Lk // bkv) % 3:
    pytest.skip('key blocks not divisible by 3')
  monkeypatch.setenv('MSD_ATTN_BKV', str(bkv))
  if splits:
    monkeypatch.setenv('MSD_ATTN_SPLITS', str(splits))
  g = torch.Generator().manual_seed(nb * 1000 + Lk + 7 * (1 - draw))
  w = heads * 64
  q = bf16_round(torch.randn(nb, Lq, w, generator=g) * 0.5)
  k = bf16_round(torch.randn(nb, Lk, w, generator=g) * 0.5)
  v = bf16_round(torch.randn(nb, Lk, w, generator=g))
  mask = None
  if masked:
    mask = (torch.rand(nb, Lk, generator=g) > 0.3).to(torch.int32)
    mask[0, Lk // 2:] = 0                      # a run of fully masked key blocks
    if nb > 2:
      mask[2, :] = 0                           # a row with nothing to attend to -> zeros
  q, k, v = q.to(cuda_device), k.to(cuda_device), v.to(cuda_device)
  mask = None if mask is None else mask.to(cuda_device)
  want, wabs = AV.reference(q, k, v, mask)
  for run in range(2):
    got = engine.op_attention(q, k, v, mask, heads)
    AV.check_rounding_bound(got, want, wabs,
                            f'nb={nb} Lk={Lk} splits={splits} bkv={bkv} draw={draw} run {run}')


@pytest.mark.parametrize('rows,d,film', [(128, 128, False), (256, 768, True), (100, 512, True)])
def test_layer_norm_film(cuda_device, rows, d, film):
  from music_spectrogram_diffusion_b200 import engine
  g = torch.Generator().manual_seed(rows + d)
  x = torch.randn(rows, d, generator=g) * 3
  gamma = 1 + 0.1 * torch.randn(d, generator=g)
  fv = torch.randn(2 * d, generator=g) * 0.2 if film else None
  want = O.layer_norm(x, gamma)
  if film:
    want = want * (fv[:d] + 1.0) + fv[d:]
  got = engine.op_rmsnorm_film(x.to(cuda_device), gamma.to(cuda_device),
                               None if fv is None else fv.to(cuda_device)).cpu()
  err = (got - want).abs().max().item()
  assert err < 4e-2, f'max err {err}'   # bf16 output rounding of O(4) values
  assert (got - bf16_round(want)).abs().max().item() < 2e-2


# ---- fused GEMM epilogues (kernels.h GemmEpilogue), each at the decoder's B = 8 height ----------
def _dense_inputs(M, N, K, seed):
  g = torch.Generator().manual_seed(seed)
  a = bf16_round(torch.randn(M, K, generator=g))
  w = bf16_round(torch.randn(K, N, generator=g) / np.sqrt(K))
  return g, a, w


@pytest.mark.parametrize('block_n', [0, 64, 128, 192, 256])
@pytest.mark.parametrize('M,N,K', [(4096, 2304, 768), (512, 768, 768), (4096, 768, 2048)])
def test_epilogue_bf16(cuda_device, M, N, K, block_n):
  """EPI_BF16 (q/k/v projections, layers.py:262-264): bf16(a w) against the fp64 product."""
  from music_spectrogram_diffusion_b200 import engine
  if block_n and N % block_n:
    pytest.skip('tile width does not divide N')
  _, a, w = _dense_inputs(M, N, K, M + N + K + 1)
  got = engine.op_dense_epilogue(a.to(cuda_device), w.to(cuda_device), 'bf16', block_n).cpu()
  want = O.dense_general(a.double(), w.double()).float()
  assert torch.equal(got, bf16_round(got))                       # really a bf16 result
  # one bf16 rounding of an O(1) value + fp32 accumulation error
  assert (got - want).abs().max().item() < 2.0 ** -8 * max(1.0, want.abs().max().item()) + 2e-4 * np.sqrt(K)


@pytest.mark.parametrize('block_n', [0, 64, 96, 128, 192, 256])
@pytest.mark.parametrize('M,N,K', [(4096, 768, 768), (512, 768, 2048), (4096, 768, 2048)])
def test_epilogue_residual_f32(cuda_device, M, N, K, block_n):
  """EPI_RESID_F32 (x + out-projection / wo, network.py:186-193, 252-256), TMA-loaded residual
  chunks and TMA stores; in place like the engine uses it."""
  from music_spectrogram_diffusion_b200 import engine
  if block_n and N % block_n:
    pytest.skip('tile width does not divide N')
  g, a, w = _dense_inputs(M, N, K, M + N + K + 2)
  resid = torch.randn(M, N, generator=g) * 3
  got = engine.op_dense_epilogue(a.to(cuda_device), w.to(cuda_device), 'resid_f32', block_n,
                                 resid=resid.to(cuda_device)).cpu()
  want = (O.dense_general(a.double(), w.double()) + resid.double()).float()
  assert (got - want).abs().max().item() < 2e-4 * np.sqrt(K)


@pytest.mark.parametrize('block_n', [0, 64, 128, 256])
@pytest.mark.parametrize('dup', [False, True])
@pytest.mark.parametrize('shifted', [False, True])
def test_epilogue_position_f32(cuda_device, block_n, dup, shifted):
  """EPI_POS_F32: input projection + position table rows (network.py:327-334 terminal-relative
  roll, 420-427), optionally duplicated into the unconditional rows (dup_rows)."""
  from music_spectrogram_diffusion_b200 import engine
  nseq, L, N, K = 8, 256, 768, 384
  M = nseq * L
  g, a, w = _dense_inputs(M, N, K, 4242 + block_n)
  pos = torch.randn(L, N, generator=g)
  shift = torch.tensor([0, 40, 255, 1, 128, 0, 77, 200], dtype=torch.int32) if shifted else None
  got = engine.op_dense_epilogue(a.to(cuda_device), w.to(cuda_device), 'pos_f32', block_n,
                                 pos=pos.to(cuda_device),
                                 pos_shift=None if shift is None else shift.to(cuda_device),
                                 dup_rows=M if dup else 0).cpu()
  y = O.dense_general(a.double(), w.double()).view(nseq, L, N)
  for s_ in range(nseq):
    sh = int(shift[s_]) if shifted else 0
    # row r of sequence s gets pos[(r - shift) mod L] == roll(arange(L), shift)[r]
    y[s_] += pos.double()[torch.roll(torch.arange(L), sh, 0)]
  want = y.view(M, N).float()
  assert got.shape[0] == (2 * M if dup else M)
  assert (got[:M] - want).abs().max().item() < 2e-4 * np.sqrt(K)
  if dup:
    assert torch.equal(got[M:], got[:M])


@pytest.mark.parametrize('block_n', [0, 64, 128, 256])
@pytest.mark.parametrize('M,F,K', [(4096, 2048, 768), (512, 1024, 512)])
def test_epilogue_gated_gelu(cuda_device, M, F, K, block_n):
  """EPI_GATED_GELU: gelu_tanh(x wi_0) * (x wi_1) (layers.py:483-509) with the wi_0 / wi_1 rows
  interleaved in 32-column groups and tanh.approx in the epilogue; the tanh.approx error
  (abs ~5e-4 on tanh) is bounded here in isolation."""
  from music_spectrogram_diffusion_b200 import engine
  if block_n and (2 * F) % block_n:
    pytest.skip('tile width does not divide 2F')
  g, a, w0 = _dense_inputs(M, F, K, M + F + K + 3)
  w1 = bf16_round(torch.randn(K, F, generator=g) / np.sqrt(K))
  a = a * 2.0   # pre-activations with a few sigma of range (|u| up to ~8)
  got = engine.op_dense_epilogue(a.to(cuda_device), w0.to(cuda_device), 'gated_gelu', block_n,
                                 w1=w1.to(cuda_device)).cpu()
  h0, h1 = O.dense_general(a.double(), w0.double()), O.dense_general(a.double(), w1.double())
  want = (O.gelu_tanh(h0) * h1).float()
  err = (got - want).abs()
  tol = 2.0 ** -8 * want.abs() + 1.5e-3 * h1.abs().float() + 1e-3   # bf16 rounding + tanh.approx * |gate|
  assert (err <= tol).all(), (err - tol).max().item()
  assert err.mean().item() < 4e-3


@pytest.mark.parametrize('M,F,K', [(512, 2048, 768), (256, 256, 128)])
def test_epilogue_gated_gelu_split_precision(cuda_device, M, F, K):
  """EPI_GATED_GELU_SPLIT3 (fp32-accurate mode): unrounded fp32 operands through the 3 x bf16
  split GEMM, exact tanh, [hi | lo | hi] output: ~2^-16 relative."""
  from music_spectrogram_diffusion_b200 import engine
  g = torch.Generator().manual_seed(M + F + K)
  a = torch.randn(M, K, generator=g) * 2.0
  w0 = torch.randn(K, F, generator=g) / np.sqrt(K)
  w1 = torch.randn(K, F, generator=g) / np.sqrt(K)
  got = engine.op_dense_epilogue(a.to(cuda_device), w0.to(cuda_device), 'gated_gelu_split3', 0,
                                 w1=w1.to(cuda_device)).cpu()
  want = (O.gelu_tanh(O.dense_general(a.double(), w0.double())) *
          O.dense_general(a.double(), w1.double())).float()
  err = (got - want).abs().max().item()
  assert err < 3e-4 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize('splits', [0, 1, 3])
@pytest.mark.parametrize('nb,heads,Lq,Lk,masked', [
    (1, 1, 128, 128, False), (2, 3, 256, 384, True), (1, 2, 256, 2304, True),
    (3, 2, 128, 256, True), (2, 12, 256, 256, False)])
def test_dot_product_attention_fp32(cuda_device, monkeypatch, nb, heads, Lq, Lk, masked, splits):
  """The fp32 attention of the fp32-accurate mode against the oracle on UNROUNDED fp32 inputs,
  large logits included (no 1/sqrt(d) scaling in this model).  splits: 0 = automatic split-KV
  choice, 1 = single pass, 3 = forced 3-way split + combine."""
  from music_spectrogram_diffusion_b200 import engine
  if splits == 3 and (Lk // 64) % 3:
    pytest.skip('key blocks not divisible by 3')
  if splits:
    monkeypatch.setenv('MSD_ATTN_SPLITS', str(splits))
  g = torch.Generator().manual_seed(nb * 31 + Lk)
  w = heads * 64
  q = torch.randn(nb, Lq, w, generator=g) * 0.7
  k = torch.randn(nb, Lk, w, generator=g) * 0.7
  v = torch.randn(nb, Lk, w, generator=g)
  mask = bias = m4 = None
  if masked:
    mask = (torch.rand(nb, Lk, generator=g) > 0.3).to(torch.int32)
    mask[0, Lk // 2:] = 0
    if nb > 2:
      mask[2, :] = 0
    m4 = O.make_attention_mask(torch.ones(nb, Lq), mask.float())
    bias = torch.where(m4 > 0, torch.zeros_like(m4), torch.full_like(m4, -1e10))
  want = O.dot_product_attention(q.double().view(nb, Lq, heads, 64), k.double().view(nb, Lk, heads, 64),
                                 v.double().view(nb, Lk, heads, 64),
                                 None if bias is None else bias.double()).reshape(nb, Lq, w).float()
  if masked:
    want = O.zero_activations_if_masked(want, m4)
  got = engine.op_attention_f32(q.to(cuda_device), k.to(cuda_device), v.to(cuda_device),
                                None if mask is None else mask.to(cuda_device), heads).cpu()
  err = (got - want).abs().max().item()
  assert torch.isfinite(got).all() and err < 1e-4, err


def test_device_threefry_bits_are_exact(cuda_device):
  """Integer work is bit-exact: the uint32 words of the device jax.random stream (before the
  float transform) == jax_rng.random_bits for PRNGKey(seed) and for fold_in(key, i)."""
  from music_spectrogram_diffusion_b200 import engine, jax_rng as J
  for seed, step, n in ((0, -1, 4096), (7, 0, 65536), (123456789, 999, 2 * 256 * 128),
                        ((5 << 32) | 77, 3, 8), (31337, 500, 8 * 256 * 128)):
    key = J.prng_key(seed) if step < 0 else J.fold_in(J.prng_key(seed), step)
    want = J.random_bits(key, n)
    got = engine.op_jax_bits(seed, step, n, cuda_device).cpu().numpy().view(np.uint32)
    np.testing.assert_array_equal(got, want)
