"""-m gpu: the attention kernels through the operand views the engine launches them with
(engine.cu: run_encoder, cross_attention, decoder_layers) at base dimensions, against
fp64 attention computed from the same views.

Every case fills the output buffer with a sentinel first (everything outside the written slice
must be bit-identical afterwards, including MARGIN rows past its end), fills the split-KV
workspace with NaN (a partial the combine reads but no split wrote shows up), and runs two input
draws into the same buffers (a value left over from the first draw fails the second).

bf16 results are held to `rounding_bound`, derived from the kernel's rounding points:
  |got - want| <= 2^-8 (sum_j w_j |v_j| + |want|) + 2^-12 sum_j w_j |v_j| + 1e-5,
w = the fp64 softmax.  bf16 keeps 8 significant bits, so one rounding to nearest is off by at most
2^-8 relative.  P is rounded to bf16 before the PV product (<= 2^-8 sum w|v| on the output; the
row sum l is kept from the unrounded fp32 values) and the output is rounded to bf16 (<= 2^-8
|want|): the first term is these two worst cases added, with no slack.  The second term covers
everything done in fp32 (ex2.approx, the logits' and PV's fp32 accumulation, the running-max
rescale, the split combine, and the product of the two roundings), each 2^-13 or far less.
Measured on an H100 (80 GB HBM3, 700 W power limit) the largest err / bound is 0.91, in the
peaked-logit cases: there most of the weight sits on a few keys whose P is not exactly 1, so their
rounding errors do not average out, and the output rounding adds on top.  With q, k at 0.5 sigma
the largest is 0.74 (tests/test_gpu_ops.py: 0.70), with q at 1 sigma 0.81.
Unlike a flat absolute bound, this one is as tight for a row whose output is 0.05 as for one
whose output is 1, and dropping a key that carries 1 % of the softmax weight breaks it.
"""
import pytest
import torch

from oracle import msd_oracle as O

pytestmark = pytest.mark.gpu

HH, H, N, T, C = 768, 12, 256, 2048, 256     # base: heads * 64, heads, targets, inputs, context
MKV = T + C
CACHE_B = 8                                  # batch rows of the cross K/V cache (max_batch)
LAYERS = 2                                   # cache layers; the cases attend layer 1
SENTINEL = -7.25                             # bf16-exact, far outside any output here
MARGIN = 64                                  # rows after every output view that nothing may write
OFFSETS = (0, 1, 7, 8, 31, 32, 63, 64, 127)  # in-block key positions of the one-key cases


# ---- the bound ---------------------------------------------------------------------------------
def rounding_bound(want: torch.Tensor, wabs: torch.Tensor) -> torch.Tensor:
  """Largest |got - want| of a correct bf16 attention output (module docstring)."""
  return 2.0 ** -8 * (wabs + want.abs()) + 2.0 ** -12 * wabs + 1e-5


def check_rounding_bound(got: torch.Tensor, want: torch.Tensor, wabs: torch.Tensor, what: str = '') -> float:
  """Asserts the bound elementwise; prints and returns the largest err / bound."""
  got, want, wabs = got.double(), want.double().to(got.device), wabs.double().to(got.device)
  assert torch.isfinite(got).all(), what
  ratio = ((got - want).abs() / rounding_bound(want, wabs)).max().item()
  print(f'[err/bound] {what}: {ratio:.3f}')
  assert ratio <= 1.0, (what, ratio)
  return ratio


def reference(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, keymask):
  """fp64 attention of q [nb, Lq, w], k / v [nb, Lk, w] with key mask [nb, Lk] (> 0 = attend) or
  None: (softmax(q k^T + bias) v, softmax(q k^T + bias) |v|), rows without an attendable key 0."""
  nb, lq, w = q.shape
  lk = k.shape[1]
  heads = w // 64

  def split(t, n):
    return t.double().reshape(nb, n, heads, 64)

  bias = m4 = None
  if keymask is not None:
    m4 = O.make_attention_mask(torch.ones(nb, lq, dtype=torch.float64, device=q.device),
                               (keymask > 0).double())
    bias = torch.where(m4 > 0, torch.zeros_like(m4), torch.full_like(m4, -1e10))
  want = O.dot_product_attention(split(q, lq), split(k, lk), split(v, lk), bias).reshape(nb, lq, w)
  wabs = O.dot_product_attention(split(q, lq), split(k, lk), split(v, lk).abs(), bias).reshape(nb, lq, w)
  if m4 is not None:
    want = O.zero_activations_if_masked(want, m4)
    wabs = O.zero_activations_if_masked(wabs, m4)
  return want, wabs


# ---- buffers and views ---------------------------------------------------------------------------
def view(t: torch.Tensor, off: int, ld: int, rows: int, cols: int) -> torch.Tensor:
  """rows x cols of the flat buffer t from element `off` with row stride ld (a strided view)."""
  return torch.as_strided(t, (rows, cols), (ld, 1), off)


def kv_rows(t, off, ld, nb, kbr, row0, lk):
  """K or V of batch b: rows b * kbr + row0 + [0, lk) of the view, as [nb, lk, HH]."""
  return view(t, off, ld, nb * kbr, HH).reshape(nb, kbr, HH)[:, row0:row0 + lk]


def operand_dtype(prec):
  return torch.float32 if prec == 'fp32_accurate' else torch.bfloat16


class Out:
  """A sentinel-filled bf16 output buffer [rows + MARGIN, ld] that remembers what was written."""

  def __init__(self, rows, ld, device):
    self.t = torch.full(((rows + MARGIN) * ld,), SENTINEL, dtype=torch.bfloat16, device=device)
    self.written = torch.zeros(self.t.numel(), dtype=torch.bool, device=device)
    self.rows, self.ld = rows, ld

  def slices(self, prec, o_col, o_ld):
    """The slice(s) a launch writes: [view] (bf16) or [hi, lo, hi] (fp32-accurate, o_ld = third)."""
    if prec == 'fp32_accurate':
      return [view(self.t, o_col + j * o_ld, 3 * o_ld, self.rows, HH) for j in range(3)]
    return [view(self.t, o_col, o_ld, self.rows, HH)]

  def mark(self, prec, o_col, o_ld):
    n = 3 if prec == 'fp32_accurate' else 1
    step = 3 * o_ld if n == 3 else o_ld
    for j in range(n):
      view(self.written, o_col + j * o_ld, step, self.rows, HH).fill_(True)

  def assert_untouched_outside(self):
    bits = torch.tensor(SENTINEL, dtype=torch.bfloat16).view(torch.int16).item()
    outside = self.t[~self.written].view(torch.int16)
    assert outside.numel() > 0 and bool((outside == bits).all()), \
        f'{int((outside != bits).sum())} elements outside the written slices changed'


class Workspace:
  """Split-KV partials (engine.attention_workspace), NaN-filled once."""

  def __init__(self, nb, lq, device):
    from music_spectrogram_diffusion_b200 import engine
    self.part_o, self.part_ml = engine.attention_workspace(nb, lq, H, device)
    self.part_o.fill_(float('nan'))
    self.part_ml.fill_(float('nan'))


def attend(prec, q, q_off, ldq, kv, k_off, v_off, ldkv, nb, lq, lk, out, o_col, o_ld, ws,
           mask=None, word0=0, kbr=0, row0=0, kv_static=0, splits=0, tail=0):
  """One launch through msd_op_attention_view; returns the fp64 reference of the same views
  (want, wabs) as [nb * lq, HH]."""
  from music_spectrogram_diffusion_b200 import engine
  engine.op_attention_view(q, q_off, ldq, kv, k_off, ldkv, kv, v_off, ldkv, nb, H, lq, lk, out.t, o_col,
                           o_ld, ws.part_o, ws.part_ml, key_mask=mask, mask_word0=word0,
                           kv_batch_rows=kbr, kv_row0=row0, kv_static=kv_static, splits=splits,
                           tail=tail, precision=prec)
  out.mark(prec, o_col, o_ld)
  qv = view(q, q_off, ldq, nb * lq, HH).reshape(nb, lq, HH)
  kb = kbr or lk
  kk = kv_rows(kv, k_off, ldkv, nb, kb, row0, lk)
  vv = kv_rows(kv, v_off, ldkv, nb, kb, row0, lk)
  km = None if mask is None else mask[:, word0 * 32:word0 * 32 + lk]
  want, wabs = reference(qv, kk, vv, km)
  return want.reshape(nb * lq, HH), wabs.reshape(nb * lq, HH)


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
  """One unit in the last place of bf16 at |x| (8 significant bits); 0 at 0."""
  _, e = torch.frexp(x.double())
  return torch.ldexp((x != 0).double(), (e - 8).to(torch.int32))


def check(prec, out, o_col, o_ld, want, wabs, what):
  """bf16: the rounding bound.  fp32-accurate: hi + lo within 1e-4 of fp64 (the existing fp32
  criterion), the third slice == the first bit for bit, lo == bf16(v - hi) within one bf16 ulp
  (plus the fp32 kernel's own error, taken as 2^-16 sum w|v|).  Returns the checked value."""
  sl = out.slices(prec, o_col, o_ld)
  if prec != 'fp32_accurate':
    check_rounding_bound(sl[0].float(), want, wabs, what)
    return sl[0].float()
  hi, lo, hi2 = sl
  assert torch.equal(hi2.view(torch.int16), hi.view(torch.int16)), what
  v = hi.double() + lo.double()
  err = (v - want).abs().max().item()
  print(f'[fp32] {what}: max |hi + lo - want| = {err:.2e}')
  assert torch.isfinite(v).all() and err < 1e-4, (what, err)
  lo_ref = (want - hi.double()).to(torch.bfloat16).double()
  tol = bf16_ulp(lo_ref) + 2.0 ** -16 * wabs
  assert bool(((lo.double() - lo_ref).abs() <= tol).all()), (what, ((lo.double() - lo_ref).abs() - tol).max().item())
  return v.float()


def randn(shape, g, scale, dtype, device):
  return (torch.randn(shape, generator=g, device=device) * scale).to(dtype)


def fill_qkv(qkv, rows, g, qk_scale=0.5):
  """Fused [rows, 3 HH] buffer: q | k at qk_scale sigma, v at 1 sigma."""
  qkv.copy_(randn(qkv.shape, g, qk_scale, qkv.dtype, qkv.device))
  v = view(qkv, 2 * HH, 3 * HH, rows, HH)
  v.copy_(randn((rows, HH), g, 1.0, qkv.dtype, qkv.device))


def fill_cache(cache, g, k_scale=0.5):
  """[LAYERS][CACHE_B * MKV, 2 HH] = (k | v) rows; every layer random, so a wrong layer shows."""
  rows = cache.numel() // (2 * HH)
  cache.copy_(randn(cache.shape, g, 1.0, cache.dtype, cache.device))
  view(cache, 0, 2 * HH, rows, HH).mul_(k_scale)


def cross_mask(nb, device):
  """Key masks [nb, MKV] of the engine's shape: padded token segments, a fully masked, a partly
  filled and a scattered context; one segment with scattered token bits too."""
  m = torch.ones(nb, MKV, dtype=torch.int32)
  tok_len = [2048, 1500, 2048, 700, 2048, 2048, 40, 2048]
  for b in range(nb):
    m[b, tok_len[b % 8]:T] = 0
  if nb == 1:
    m[0, T + 100:] = 0
  if nb > 2:
    m[2, T:] = 0
  if nb > 5:
    m[5, T + 100:] = 0
  if nb > 7:
    gen = torch.Generator().manual_seed(7)
    m[7] = (torch.rand(MKV, generator=gen) > 0.3).to(torch.int32)
  return m.to(device)


def cache_offsets(layer, b_rows=CACHE_B):
  k_off = layer * b_rows * MKV * 2 * HH
  return k_off, k_off + HH


# ---- decoder self-attention over the fused QKV buffer ------------------------------------------
@pytest.mark.parametrize('prec', ['bf16', 'fp32_accurate'])
@pytest.mark.parametrize('nb,splits', [(16, 0), (1, 0), (1, 2)])
def test_decoder_self_attention_fused_qkv(cuda_device, prec, nb, splits):
  """decoder_layers: Q, K, V are column views (offsets 0 / hh / 2hh, ld 3 hh) of the QKV
  projection's output; nb = 16 is both guidance passes of B = 8."""
  dev = cuda_device
  rows = nb * N
  qkv = torch.empty(rows * 3 * HH, dtype=operand_dtype(prec), device=dev)
  o_ld = HH
  out = Out(rows, 3 * o_ld if prec == 'fp32_accurate' else o_ld, dev)
  ws = Workspace(nb, N, dev)
  g = torch.Generator(dev).manual_seed(11 + nb)
  for draw in range(2):
    fill_qkv(qkv.view(rows, 3 * HH), rows, g)
    want, wabs = attend(prec, qkv, 0, 3 * HH, qkv, HH, 2 * HH, 3 * HH, nb, N, N, out, 0, o_ld, ws,
                        splits=splits)
    check(prec, out, 0, o_ld, want, wabs, f'self {prec} nb={nb} splits={splits} draw {draw}')
    out.assert_untouched_outside()


# ---- the two encoders ------------------------------------------------------------------------------
@pytest.mark.parametrize('bkv', [64, 128])
def test_token_encoder_self_attention(cuda_device, monkeypatch, bkv):
  """run_encoder over the tokens: Lq = Lk = 2048, mask rows of Mkv / 32 = 72 words, segment 1
  padded after 700 tokens.  The kernel applies the key mask only, so the padded query rows are
  defined too and are compared with the rest."""
  monkeypatch.setenv('MSD_ATTN_BKV', str(bkv))
  dev = cuda_device
  nb, rows = 2, 2 * T
  qkv = torch.empty(rows * 3 * HH, dtype=torch.bfloat16, device=dev)
  mask = torch.ones(nb, MKV, dtype=torch.int32)
  mask[1, 700:T] = 0
  mask[:, T:] = (torch.rand(nb, C, generator=torch.Generator().manual_seed(3)) > 0.5).to(torch.int32)
  mask = mask.to(dev)
  out = Out(rows, HH, dev)
  ws = Workspace(nb, T, dev)
  g = torch.Generator(dev).manual_seed(21 + bkv)
  for draw in range(2):
    fill_qkv(qkv.view(rows, 3 * HH), rows, g)
    want, wabs = attend('bf16', qkv, 0, 3 * HH, qkv, HH, 2 * HH, 3 * HH, nb, T, T, out, 0, HH, ws,
                        mask=mask)
    check('bf16', out, 0, HH, want, wabs, f'token encoder bkv={bkv} draw {draw}')
    out.assert_untouched_outside()


@pytest.mark.parametrize('bkv', [64, 128])
def test_context_encoder_self_attention(cuda_device, monkeypatch, bkv):
  """run_encoder over the context: the mask pointer starts T / 32 = 64 words into rows of 72.
  Segment 1's context is fully masked (exact zeros), segment 2 holds 100 of 256 frames."""
  monkeypatch.setenv('MSD_ATTN_BKV', str(bkv))
  dev = cuda_device
  nb, rows = 3, 3 * C
  qkv = torch.empty(rows * 3 * HH, dtype=torch.bfloat16, device=dev)
  mask = (torch.rand(nb, MKV, generator=torch.Generator().manual_seed(4)) > 0.5).to(torch.int32)
  mask[0, T:] = 1
  mask[1, T:] = 0
  mask[2, T:] = 0
  mask[2, T:T + 100] = 1
  mask = mask.to(dev)
  out = Out(rows, HH, dev)
  ws = Workspace(nb, C, dev)
  g = torch.Generator(dev).manual_seed(31 + bkv)
  for draw in range(2):
    fill_qkv(qkv.view(rows, 3 * HH), rows, g)
    want, wabs = attend('bf16', qkv, 0, 3 * HH, qkv, HH, 2 * HH, 3 * HH, nb, C, C, out, 0, HH, ws,
                        mask=mask, word0=T // 32)
    got = check('bf16', out, 0, HH, want, wabs, f'context encoder bkv={bkv} draw {draw}')
    assert bool((got[C:2 * C] == 0).all())
    assert bool((got[2 * C:] != 0).any())
    out.assert_untouched_outside()


# ---- cross-attention over the per-layer K/V cache ----------------------------------------------
CROSS_CASES = [(1, 0, 0), (8, 0, 0), (8, 0, 5)]   # (nb, splits, tail): 6 automatic splits, unsplit, tail


@pytest.mark.parametrize('logits', ['normal', 'peaked'])
@pytest.mark.parametrize('bkv', [64, 128])
@pytest.mark.parametrize('nb,splits,tail', CROSS_CASES)
def test_concat_cross_attention_from_the_cache(cuda_device, monkeypatch, nb, splits, tail, bkv, logits):
  """cross_attention, concat_encodings: K / V of layer 1 of a 2-layer cache (ld 2 hh, V at
  column hh), kv_static = 1 (K / V and the mask read ahead of the dependency wait).  'peaked': q
  and k at 2 sigma, logits with sigma ~ 32 (no 1/sqrt(d) in this model), so the running max moves
  across key blocks and splits."""
  monkeypatch.setenv('MSD_ATTN_BKV', str(bkv))
  dev = cuda_device
  scale = 2.0 if logits == 'peaked' else 0.5
  rows = nb * N
  cache = torch.empty(LAYERS * CACHE_B * MKV * 2 * HH, dtype=torch.bfloat16, device=dev)
  q = torch.empty(rows * HH, dtype=torch.bfloat16, device=dev)
  mask = cross_mask(nb, dev)
  out = Out(rows, HH, dev)
  ws = Workspace(nb, N, dev)
  k_off, v_off = cache_offsets(1)
  g = torch.Generator(dev).manual_seed(41 + nb + bkv + tail)
  for draw in range(2):
    fill_cache(cache, g, scale)
    q.copy_(randn(q.shape, g, scale, q.dtype, dev))
    want, wabs = attend('bf16', q, 0, HH, cache, k_off, v_off, 2 * HH, nb, N, MKV, out, 0, HH, ws,
                        mask=mask, kv_static=1, splits=splits, tail=tail)
    check('bf16', out, 0, HH, want, wabs, f'concat cross nb={nb} tail={tail} bkv={bkv} {logits} draw {draw}')
    out.assert_untouched_outside()


@pytest.mark.parametrize('nb', [1, 8])
def test_concat_cross_attention_from_the_cache_fp32(cuda_device, nb):
  """The same views through the fp32 kernel (fp32-accurate mode), output [hi | lo | hi]."""
  dev = cuda_device
  rows = nb * N
  cache = torch.empty(LAYERS * CACHE_B * MKV * 2 * HH, dtype=torch.float32, device=dev)
  q = torch.empty(rows * HH, dtype=torch.float32, device=dev)
  mask = cross_mask(nb, dev)
  out = Out(rows, 3 * HH, dev)
  ws = Workspace(nb, N, dev)
  k_off, v_off = cache_offsets(1)
  g = torch.Generator(dev).manual_seed(51 + nb)
  for draw in range(2):
    fill_cache(cache, g)
    q.copy_(randn(q.shape, g, 0.5, q.dtype, dev))
    want, wabs = attend('fp32_accurate', q, 0, HH, cache, k_off, v_off, 2 * HH, nb, N, MKV, out, 0, HH, ws,
                        mask=mask, kv_static=1)
    check('fp32_accurate', out, 0, HH, want, wabs, f'concat cross fp32 nb={nb} draw {draw}')
    out.assert_untouched_outside()


def sum_cross_launches(prec, q, cache, nb, out, o_ld, ws1, ws2, mask, splits=(0, 0)):
  """sum_cross_attends: tokens then context from one [tokens | context] cache (kv_batch_rows =
  Mkv), Q from columns 0 / hh of a 2 hh-wide buffer, O into columns [0, hh) / [hh, 2 hh)."""
  k_off, v_off = cache_offsets(1)
  ref_t = attend(prec, q, 0, 2 * HH, cache, k_off, v_off, 2 * HH, nb, N, T, out, 0, o_ld, ws1,
                 mask=mask, kbr=MKV, row0=0, kv_static=1, splits=splits[0])
  ref_c = attend(prec, q, HH, 2 * HH, cache, k_off, v_off, 2 * HH, nb, N, C, out, HH, o_ld, ws2,
                 mask=mask, word0=T // 32, kbr=MKV, row0=T, kv_static=1, splits=splits[1])
  return ref_t, ref_c


@pytest.mark.parametrize('prec', ['bf16', 'fp32_accurate'])
@pytest.mark.parametrize('nb', [1, 3])
def test_sum_cross_attends_from_the_cache(cuda_device, prec, nb):
  """Both launches of the sum_cross_attends block into one [rows, 2 hh] buffer ([rows, 3 x 2 hh]
  in fp32-accurate mode).  nb = 3: segment 2's context is fully masked, so its context half is
  exactly zero while its token half is not."""
  dev = cuda_device
  rows = nb * N
  dt = operand_dtype(prec)
  cache = torch.empty(LAYERS * CACHE_B * MKV * 2 * HH, dtype=dt, device=dev)
  q = torch.empty(rows * 2 * HH, dtype=dt, device=dev)
  mask = cross_mask(nb, dev)
  o_ld = 2 * HH
  out = Out(rows, 3 * o_ld if prec == 'fp32_accurate' else o_ld, dev)
  ws1, ws2 = Workspace(nb, N, dev), Workspace(nb, N, dev)
  g = torch.Generator(dev).manual_seed(61 + nb)
  for draw in range(2):
    fill_cache(cache, g)
    q.copy_(randn(q.shape, g, 0.5, dt, dev))
    (wt, at), (wc, ac) = sum_cross_launches(prec, q, cache, nb, out, o_ld, ws1, ws2, mask)
    tok = check(prec, out, 0, o_ld, wt, at, f'sum_cross tokens {prec} nb={nb} draw {draw}')
    ctx = check(prec, out, HH, o_ld, wc, ac, f'sum_cross context {prec} nb={nb} draw {draw}')
    if nb == 3:
      assert bool((ctx[2 * N:] == 0).all())
      assert bool((tok[2 * N:] != 0).any())
    out.assert_untouched_outside()


# ---- sharper families ------------------------------------------------------------------------------
def one_key_positions(blocks):
  return [blk * 128 + off for blk in blocks for off in OFFSETS]


@pytest.mark.parametrize('bkv', [64, 128])
@pytest.mark.parametrize('splits,tail', [(0, 0), (1, 0), (2, 0), (3, 0), (6, 0), (1, 5)])
def test_one_attendable_key_concat_cross(cuda_device, monkeypatch, bkv, splits, tail):
  """Batch row b may attend one key only, at in-block positions {0, 1, 7, 8, 31, 32, 63, 64, 127}
  of the first, a middle and the last 128-key block: its softmax weight is exactly 1, so every
  query row's output is that key's V row bit for bit, on every split path.  Pins the fragment
  column -> mask bit mapping and the K / V / O row and column offsets."""
  monkeypatch.setenv('MSD_ATTN_BKV', str(bkv))
  dev = cuda_device
  keys = one_key_positions((0, MKV // 128 // 2 - 1, MKV // 128 - 1))
  nb = len(keys)
  rows = nb * N
  cache = torch.empty(LAYERS * nb * MKV * 2 * HH, dtype=torch.bfloat16, device=dev)
  q = torch.empty(rows * HH, dtype=torch.bfloat16, device=dev)
  mask = torch.zeros(nb, MKV, dtype=torch.int32)
  mask[torch.arange(nb), torch.tensor(keys)] = 1
  mask = mask.to(dev)
  out = Out(rows, HH, dev)
  ws = Workspace(nb, N, dev)
  k_off, v_off = cache_offsets(1, nb)
  g = torch.Generator(dev).manual_seed(71 + bkv + splits + tail)
  for draw in range(2):
    fill_cache(cache, g, 2.0 if draw else 0.5)
    q.copy_(randn(q.shape, g, 1.0, q.dtype, dev))
    attend('bf16', q, 0, HH, cache, k_off, v_off, 2 * HH, nb, N, MKV, out, 0, HH, ws, mask=mask,
           kv_static=1, splits=splits, tail=tail)
    v = kv_rows(cache, v_off, 2 * HH, nb, MKV, 0, MKV)[torch.arange(nb), torch.tensor(keys)]   # [nb, HH]
    got = out.slices('bf16', 0, HH)[0].reshape(nb, N, HH)
    bad = (got.view(torch.int16) != v[:, None, :].view(torch.int16)).any(-1).any(-1)
    assert not bool(bad.any()), [keys[i] for i in torch.nonzero(bad).flatten().tolist()]
    out.assert_untouched_outside()


@pytest.mark.parametrize('bkv', [64, 128])
@pytest.mark.parametrize('splits', [0, 2])
def test_one_attendable_key_sum_cross_context(cuda_device, monkeypatch, bkv, splits):
  """The one-key family in the context source of sum_cross_attends (kv_row0 = T, mask from word
  T / 32, Q from column hh, O into columns [hh, 2 hh)): the context half is the key's V row bit
  for bit; the token half stays an ordinary attention within the rounding bound."""
  monkeypatch.setenv('MSD_ATTN_BKV', str(bkv))
  dev = cuda_device
  keys = one_key_positions((0, 1))
  nb = len(keys)
  rows = nb * N
  cache = torch.empty(LAYERS * nb * MKV * 2 * HH, dtype=torch.bfloat16, device=dev)
  q = torch.empty(rows * 2 * HH, dtype=torch.bfloat16, device=dev)
  mask = torch.zeros(nb, MKV, dtype=torch.int32)
  mask[:, :1000] = 1
  mask[torch.arange(nb), T + torch.tensor(keys)] = 1
  mask = mask.to(dev)
  out = Out(rows, 2 * HH, dev)
  ws1, ws2 = Workspace(nb, N, dev), Workspace(nb, N, dev)
  k_off, v_off = cache_offsets(1, nb)
  g = torch.Generator(dev).manual_seed(81 + bkv + splits)
  for draw in range(2):
    fill_cache(cache, g)
    q.copy_(randn(q.shape, g, 1.0, q.dtype, dev))
    wt, at = attend('bf16', q, 0, 2 * HH, cache, k_off, v_off, 2 * HH, nb, N, T, out, 0, 2 * HH, ws1,
                    mask=mask, kbr=MKV, row0=0, kv_static=1)
    attend('bf16', q, HH, 2 * HH, cache, k_off, v_off, 2 * HH, nb, N, C, out, HH, 2 * HH, ws2,
           mask=mask, word0=T // 32, kbr=MKV, row0=T, kv_static=1, splits=splits)
    check('bf16', out, 0, 2 * HH, wt, at, f'sum_cross one-key tokens bkv={bkv} draw {draw}')
    v = kv_rows(cache, v_off, 2 * HH, nb, MKV, T, C)[torch.arange(nb), torch.tensor(keys)]
    got = out.slices('bf16', HH, 2 * HH)[0].reshape(nb, N, HH)
    bad = (got.view(torch.int16) != v[:, None, :].view(torch.int16)).any(-1).any(-1)
    assert not bool(bad.any()), [keys[i] for i in torch.nonzero(bad).flatten().tolist()]
    out.assert_untouched_outside()


# ---- the hook's own guard rails ----------------------------------------------------------------
def test_views_outside_their_tensors_are_refused_before_launch(cuda_device):
  """A mistaken view is a Python error, never an out-of-bounds access."""
  from music_spectrogram_diffusion_b200 import engine
  dev = cuda_device
  nb, rows = 1, N
  qkv = torch.zeros(rows * 3 * HH, dtype=torch.bfloat16, device=dev)
  out = torch.zeros(rows * HH, dtype=torch.bfloat16, device=dev)
  po, pml = engine.attention_workspace(nb, N, H, dev)
  mask = torch.ones(nb, MKV, dtype=torch.int32, device=dev)

  def call(**kw):
    a = dict(q=qkv, q_off=0, ldq=3 * HH, k=qkv, k_off=HH, ldk=3 * HH, v=qkv, v_off=2 * HH, ldv=3 * HH,
             nb=nb, heads=H, lq=N, lk=N, out=out, o_col=0, o_ld=HH, part_o=po, part_ml=pml)
    a.update(kw)
    engine.op_attention_view(**a)

  call()                                                    # the valid launch runs
  for kw in (dict(v_off=2 * HH + 8),                        # V columns past the row
             dict(lq=2 * N),                                # Q rows past the end
             dict(o_col=8),                                 # O columns past its row
             dict(kv_batch_rows=N, kv_row0=128),            # key rows past the batch row
             dict(key_mask=mask, mask_word0=MKV // 32 - 4),  # mask words past the row
             dict(key_mask=mask, mask_word0=2),             # unaligned mask start
             dict(part_o=po[:-1]),                          # workspace too small
             dict(splits=13)):
    with pytest.raises(ValueError):
      call(**kw)
