"""-m gpu: the row kernels that run between the GEMMs, launched the way the engine launches them:
the norm kernel (rmsnorm_film_kernel) in each of its launch forms through msd_op_rmsnorm_view, and
the encoder's front end (the key-mask words, the context roll and the token embedding) through
msd_op_encoder_inputs.

Every output buffer starts as a bf16- (or int-) exact sentinel with margin rows past its view; after
each launch everything outside the slice the launch writes is bit-identical to before.

Norm (LayerNorm layers.py:632-649, FiLM 652-666), at d = 128 k for every instance k = 1..8 and
1, 7, 8, 9, 100 and 4096 rows (8 rows per block), in the engine's forms:
  * plain (encoder pre-norms, norm_into): ldo = d;
  * FiLM (decoder pre-norms with MSD_FUSED_NORM=0): scale | bias rows read at film + (*step) 2 Ld 2d
    + j 2d for the layer rows j = 2l and 2l + 1, at device steps 0, middle and last of a table of
    independent random rows (a neighbouring row is off by O(1)).  The table sits one step into its
    buffer, so a launch that reads a wrong step still reads defined values;
  * split3 (the fp32-accurate pre-norms, and the decoder final norm engine.cu run_decoder): [hi | lo |
    hi] with ldo = 3d, with and without FiLM;
  * remap (the encoders' final norms, launch_rmsnorm_rows_remap): row b src_len + t to row b Mkv +
    dst_off + t at dst_off 0 (tokens) and T (context), with and without split3.
The rows mix scales 1e-3 (mean square about eps, so eps = 1e-6 is tested), 1 and 1e3, an all-zero
row (output exactly 0) and a row with one element 1e4 times the others.  The reference is fp64 from
the same fp32 inputs; each element's bound follows the kernel's rounding points (u = 2^-24):
  * the sum of squares: each lane chains 4 ITERS products, then 5 shuffle adds: (4 ITERS + 6) u
    relative (all terms are non-negative);
  * / D and + 1e-6: u each; rsqrtf within 2 ulp (4 u): inv within (e_ss + 2 u) / 2 + 4 u;
  * x inv g: two products, 2 u;
  * FiLM: 1 + fs, the product and the add, u each;
  * bf16 output: half a bf16 ulp at the value; an exact 0 must stay 0.
split3 also checks that the third block is bit-equal to the first, that |lo| <= half an ulp of hi and
hi == bf16(hi + lo) except where |lo| is exactly that half ulp (a tie of the pair, which rounds to
even), and that hi + lo is within the fp32 bound plus 2^-17 |y|: lo = bf16(y - hi) keeps 8 bits of a
residual below 2^-8 |y|, so it is off by up to 2^-17 |y| (2^-18 does not hold: 0.998 * 2^-17 is
reached by random fp32 values).

Masks and embedding are integer or single-rounding outputs and are compared bit for bit: the key-mask
words with tokens > 0 | ctx_mask > 0, ctx_seq_len with the reference's get_sequence_length
(network.py:28-39) % C, and the encoder's input rows with fp32 one_hot(id) @ emb + pos (an id outside
[0, vocab) embeds as zeros).

Measured on an H100 80GB HBM3 at a 700 W power limit, the largest err / bound per group (printed as
'[err/bound] <group>: ...'): plain 0.9998, film 1.0000 (below 1 in the fifth digit), split3 0.9998,
film_split3 1.0000, remap 0.9998, remap_split3 0.9998; the fp32 value hi + lo of the split forms:
split3 0.928, film_split3 0.997, remap_split3 0.923.  The bf16 outputs sit at their rounding's worst
case (an fp32 value next to a bf16 midpoint rounds by almost half an ulp, and the fp32 error is a
small part of the bound), so they are held to within a rounding-level error; the split values are
held to within the 2^-17 |y| of lo's rounding.  Masks, the roll and the embedding rows are exact.
"""
import ctypes

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import _native, config, engine, weights
from oracle import msd_oracle as O
from tests import helpers as H
from tests.test_gpu_gemm_views import Buffers, view

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS = float(np.float32(1e-6))      # the kernel adds 1e-6f
SENTINEL = -7.25
STEPS, LD = 5, 2                   # FiLM table of a 2-layer decoder: [STEPS][2 LD][2 d]
TEST_STEPS = (0, STEPS // 2, STEPS - 1)
ROWS = (1, 7, 8, 9, 100, 4096)
DS = tuple(128 * k for k in range(1, 9))
VOCAB = 1536


# ---- bounds --------------------------------------------------------------------------------------
def half_ulp_bf16(x: torch.Tensor) -> torch.Tensor:
  """Half a bf16 ulp at |x| (8 significant bits), 0 at 0."""
  x = x.abs().double()
  _, e = torch.frexp(x)
  return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), (e - 9).to(torch.int32)))


def check(got, want, bound, group, what):
  """|got - want| <= bound elementwise; a bound of 0 asks for equality."""
  got = got.double()
  assert bool(torch.isfinite(got).all()), what
  err = (got - want).abs()
  ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300),
                      torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, float('inf'))))
  r = ratio.max().item()
  print(f'[err/bound] {group}: {what}: {r:.4f}')
  assert r <= 1.0, (what, r)


def norm_reference(x, gamma, film_row=None):
  """fp64 rmsnorm(x) gamma (then FiLM with the scale | bias row film_row [2 d]) and the bound on the
  kernel's fp32 value before its output rounding."""
  d = x.shape[1]
  X = x.double()
  inv = torch.rsqrt((X * X).mean(-1, keepdim=True) + EPS)
  y = X * inv * gamma.double()
  e_ss = (4 * (d // 128) + 6) * U
  rel_inv = 0.5 * (e_ss + 2 * U) + 4 * U
  e = y.abs() * (rel_inv + 2 * U)
  if film_row is not None:
    s = 1.0 + film_row[:d].double()
    want = y * s + film_row[d:].double()
    e = e * s.abs() + (y * s).abs() * 2 * U + (want.abs() + e * s.abs()) * U
  else:
    want = y
  return want, e * (1 + 2.0 ** -16)   # second-order terms


def norm_rows(rows, d, g, device):
  """Rows cycling through scales 1e-3 (mean square ~ eps), 1, 1e3, an all-zero row and a unit row
  with one element 1e4 times the others."""
  x = torch.randn(rows, d, generator=g, dtype=torch.float64, device=device)
  scale = torch.tensor([1e-3, 1.0, 1e3, 0.0, 1.0], dtype=torch.float64, device=device)
  x *= scale[torch.arange(rows, device=device) % 5].unsqueeze(1)
  spikes = torch.arange(4, max(rows, 4), 5, device=device)
  x[spikes, (37 * spikes) % d] *= 1e4
  return x.float().contiguous()


# ---- the norm kernel ------------------------------------------------------------------------------
FORMS = {  # name: (FiLM, split3, remap)
    'plain': (False, False, False),
    'film': (True, False, False),
    'split3': (False, True, False),          # also the decoder final norm (ldo = 3d, no FiLM)
    'film_split3': (True, True, False),
    'remap': (False, False, True),
    'remap_split3': (False, True, True),
}


def remap_shape(rows):
  """(B, src_len) with B * src_len == rows, and the other source's length in the encodings."""
  return {1: (1, 1), 7: (1, 7), 8: (2, 4), 9: (3, 3), 100: (4, 25), 4096: (2, 2048)}[rows], 5


def check_norm_out(out_rows, want, e, d, split3, group, what):
  """out_rows: the bf16 rows the launch wrote, [rows, d] or [rows, 3 d]."""
  hi = out_rows[:, :d]
  check(hi, want, half_ulp_bf16(want.abs() + e) + e, group, what)
  if not split3:
    return
  lo, hi2 = out_rows[:, d:2 * d], out_rows[:, 2 * d:]
  assert torch.equal(hi.view(torch.int16), hi2.view(torch.int16)), f'{what}: third block != first'
  h, l = hi.double(), lo.double()
  half = half_ulp_bf16(h)
  assert bool((l.abs() <= half).all()), f'{what}: |lo| above half an ulp of hi'
  pair = (h + l).float().to(torch.bfloat16)
  tie = l.abs() == half
  same = pair.view(torch.int16) == hi.view(torch.int16)
  assert bool((same | tie).all()), f'{what}: hi != bf16(hi + lo) at {int((~(same | tie)).sum())} elements'
  check(h + l, want, e + 2.0 ** -17 * (want.abs() + e), group + ' fp32', what)


@pytest.mark.parametrize('form', sorted(FORMS))
@pytest.mark.parametrize('rows', ROWS)
@pytest.mark.parametrize('d', DS)
def test_rmsnorm_view(cuda_device, d, rows, form):
  dev = cuda_device
  has_film, split3, remap = FORMS[form]
  g = torch.Generator(dev).manual_seed(1000 * d + rows + 7 * sorted(FORMS).index(form))
  x = norm_rows(rows, d, g, dev)
  gamma = (1 + 0.5 * torch.randn(d, generator=g, device=dev)).contiguous()
  width = 3 * d if split3 else d
  ldo = width
  bufs = Buffers(dev)
  if remap:
    (B, src_len), other = remap_shape(rows)
    for dst_off in (0, other):
      dst_len = src_len + other
      out = bufs.add(f'out{dst_off}', B * dst_len, ldo, torch.bfloat16, SENTINEL)
      writes = [(f'out{dst_off}', (b * dst_len + dst_off) * ldo, ldo, src_len, width) for b in range(B)]
      bufs.launch(lambda: engine.op_rmsnorm_view(x, gamma, out, 0, ldo, split3=split3, src_len=src_len,
                                                 dst_len=dst_len, dst_off=dst_off), writes)
      got = torch.cat([view(out, off, ldo, n, c) for _, off, _, n, c in writes])
      want, e = norm_reference(x, gamma)
      check_norm_out(got, want, e, d, split3, form, f'd={d} rows={rows} dst_off={dst_off}')
    return
  out = bufs.add('out', rows, ldo, torch.bfloat16, SENTINEL)
  writes = [('out', 0, ldo, rows, width)]
  if not has_film:
    bufs.launch(lambda: engine.op_rmsnorm_view(x, gamma, out, 0, ldo, split3=split3), writes)
    want, e = norm_reference(x, gamma)
    check_norm_out(view(out, 0, ldo, rows, width), want, e, d, split3, form, f'd={d} rows={rows}')
    return
  # FiLM rows [STEPS][2 LD][2 d], one step of padding ahead of the table
  stride = 2 * LD * 2 * d
  film = (0.5 * torch.randn((STEPS + 1) * stride, generator=g, device=dev)).contiguous()
  step = torch.zeros(1, dtype=torch.int32, device=dev)
  for s in TEST_STEPS:
    step.fill_(s)
    for j in (2 * LD - 2, 2 * LD - 1):      # layer LD - 1: its self-attention and MLP pre-norms
      off = stride + j * 2 * d
      bufs.launch(lambda: engine.op_rmsnorm_view(x, gamma, out, 0, ldo, film=film, film_offset=off,
                                                 film_step_stride=stride, step=step, split3=split3), writes)
      row = film[off + s * stride:off + s * stride + 2 * d]
      want, e = norm_reference(x, gamma, row)
      check_norm_out(view(out, 0, ldo, rows, width), want, e, d, split3, form,
                     f'd={d} rows={rows} step={s} j={j}')


def test_rmsnorm_view_refuses_bad_launches(cuda_device):
  """The hook refuses, with a message, every launch the kernel cannot run as described."""
  dev = cuda_device
  x = torch.ones(16, 256, device=dev)
  gamma = torch.ones(256, device=dev)
  out = torch.zeros(16 * 3 * 256, dtype=torch.bfloat16, device=dev)
  film = torch.zeros(4 * 512, device=dev)
  step = torch.zeros(1, dtype=torch.int32, device=dev)
  p = lambda t: ctypes.c_void_p(t.data_ptr())
  ok = dict(x=p(x), rows=16, d=256, gamma=p(gamma), out=p(out), out_off=0, ldo=256)
  bad = [dict(x=None), dict(gamma=None), dict(out=None), dict(d=200), dict(d=1152), dict(rows=0),
         dict(ldo=128), dict(split3=1, ldo=512), dict(out_off=-8), dict(film=p(film)),
         dict(film=p(film), step=p(step), film_offset=-4), dict(src_len=3), dict(src_len=8, dst_len=8, dst_off=4),
         dict(src_len=8, dst_len=16, ldo=512), dict(src_len=8, dst_len=16, film=p(film), step=p(step)),
         dict(dst_off=-1, src_len=8, dst_len=16)]
  lib = _native.load()
  args = _native.MsdRmsnormViewArgs(**ok)
  assert lib.msd_op_rmsnorm_view(ctypes.byref(args), None) == 0
  for change in bad:
    args = _native.MsdRmsnormViewArgs(**dict(ok, **change))
    assert lib.msd_op_rmsnorm_view(ctypes.byref(args), None) == -1, change
    assert b'msd_op_rmsnorm_view' in lib.msd_last_error(), change
  assert lib.msd_op_rmsnorm_view(None, None) == -1


# ---- the encoder front end ------------------------------------------------------------------------
def sequence_length(row: np.ndarray) -> int:
  """network.py:28-39: the first index of a 0, or the full length when row[0] != 0 and no 0 is
  found (argmax of an all-False array is 0)."""
  length = int(np.argmax(row == 0))
  if length == 0 and row[0] != 0:
    length = row.shape[0]
  return length


def mask_words(m: np.ndarray) -> np.ndarray:
  """[B, L] bool -> [B, L / 32] uint32, bit j of word w = m[:, 32 w + j]."""
  b, n = m.shape
  w = m.reshape(b, n // 32, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)
  return w.sum(-1).astype(np.uint32)


def context_masks(B, C, rng):
  """Rows whose first zero lands at 0, 31, 32, 33 and C - 1, an all-zero row, a row with no zero,
  a zero followed by ones, and a random row; nonzero values include negatives (not attended, but
  not padding either)."""
  first = [0, 31, 32, 33, C - 1, 'zeros', 'ones', 'zero_then_ones', C // 2 + 5]
  out = np.empty((B, C), np.int32)
  for b in range(B):
    f = first[(b + (2 if B == 1 else 0)) % len(first)]
    if f == 'zeros':
      out[b] = 0
    elif f == 'ones':
      out[b] = 1
    elif f == 'zero_then_ones':
      out[b] = 1
      out[b, 0] = 0
    else:
      out[b, :f] = rng.choice([-3, -1, 1, 2, 5], f)
      out[b, f] = 0
      out[b, f + 1:] = rng.choice([-1, 0, 1, 4], C - f - 1)
  return out


def embed_reference(tokens, emb, pos):
  """fp32 one_hot(id) @ emb + pos: the embedding row (zeros outside [0, vocab)) plus the position
  row, one fp32 add."""
  valid = (tokens >= 0) & (tokens < emb.shape[0])
  rows = emb[torch.where(valid, tokens, torch.zeros_like(tokens)).long()]
  rows = torch.where(valid.unsqueeze(-1), rows, torch.zeros_like(rows))
  return rows + pos[:tokens.shape[1]].unsqueeze(0)


def run_encoder_inputs(dev, tokens, cmask, emb, pos, terminal_relative):
  """One msd_op_encoder_inputs launch into sentinel buffers: (bits uint32 [B, words], ctx_seq_len,
  x [B, T, d])."""
  B, T = tokens.shape
  C = 0 if cmask is None else cmask.shape[1]
  d = emb.shape[1]
  words = (T + C) // 32
  bufs = Buffers(dev)
  bits = bufs.add('bits', B, words, torch.int32, -0x5A5A5A5B)
  seq = bufs.add('seq', 1, B, torch.int32, -77)
  x = bufs.add('x', B * T, d, torch.float32, SENTINEL)
  bufs.launch(lambda: engine.op_encoder_inputs(tokens, cmask, emb, pos, terminal_relative, bits, seq, x),
              [('bits', 0, words, B, words), ('seq', 0, B, 1, B), ('x', 0, d, B * T, d)])
  return (bits[:B * words].view(B, words).cpu().numpy().view(np.uint32), seq[:B].cpu().numpy(),
          x[:B * T * d].view(B, T, d))


@pytest.mark.parametrize('terminal_relative', [1, 0])
@pytest.mark.parametrize('B', [1, 3, 9])
@pytest.mark.parametrize('C', [0, 128, 256])
@pytest.mark.parametrize('T', [128, 2048])
def test_encoder_masks(cuda_device, T, C, B, terminal_relative):
  """Key-mask words of [tokens | context] and the terminal-relative roll, bit for bit.  T = 2048 has
  each of the 8 warps build 8 words; C = 0 is the no-context model (ctx_mask NULL)."""
  if C == 0 and terminal_relative:
    pytest.skip('terminal-relative positions need a context')
  dev = cuda_device
  rng = np.random.default_rng(T + C + B + terminal_relative)
  toks = rng.integers(-3, VOCAB + 3, (B, T)).astype(np.int32)
  toks[rng.random((B, T)) < 0.4] = 0
  cmask = context_masks(B, C, rng) if C else None
  g = torch.Generator(dev).manual_seed(1)
  emb = torch.randn(VOCAB, 128, generator=g, device=dev)
  pos = torch.randn(T, 128, generator=g, device=dev)
  tokens = torch.from_numpy(toks).to(dev)
  bits, seq, x = run_encoder_inputs(dev, tokens, None if cmask is None else torch.from_numpy(cmask).to(dev),
                                    emb, pos, terminal_relative)
  want = mask_words(toks > 0)
  if C:
    want = np.concatenate([want, mask_words(cmask > 0)], axis=1)
  np.testing.assert_array_equal(bits, want)
  want_seq = [sequence_length(cmask[b]) % C if terminal_relative else 0 for b in range(B)]
  np.testing.assert_array_equal(seq, np.array(want_seq, np.int32))
  if C and terminal_relative:
    # the pattern set reaches every edge: roll 0 from the all-ones, all-zeros and leading-zero rows
    assert B < 9 or sorted(want_seq) == sorted([0, 31, 32, 33, C - 1, 0, 0, 0, C // 2 + 5])
  assert torch.equal(x, embed_reference(tokens, emb, pos))


@pytest.mark.parametrize('T', [128, 2048])
@pytest.mark.parametrize('d', [128, 768, 1024])
def test_token_embedding(cuda_device, d, T):
  """The encoder's input rows, bit for bit: ids 0, 1, vocab - 1 and random ids in range take their
  embedding row; vocab, vocab + 5, 2^31 - 1 and -1 take none (the reference's one-hot product gives
  zeros), so x = pos there."""
  dev = cuda_device
  B = 2
  rng = np.random.default_rng(d + T)
  toks = rng.integers(0, VOCAB, (B, T)).astype(np.int32)
  special = [0, 1, VOCAB - 1, VOCAB, VOCAB + 5, 2 ** 31 - 1, -1]
  for i, v in enumerate(special):
    toks[0, 3 + 11 * i] = v
    toks[1, T - 1 - 5 * i] = v
  g = torch.Generator(dev).manual_seed(d)
  emb = torch.randn(VOCAB, d, generator=g, device=dev)
  pos = torch.randn(T, d, generator=g, device=dev)
  tokens = torch.from_numpy(toks).to(dev)
  _, _, x = run_encoder_inputs(dev, tokens, None, emb, pos, 0)
  want = embed_reference(tokens, emb, pos)
  assert torch.equal(x, want)
  outside = (tokens < 0) | (tokens >= VOCAB)
  assert int(outside.sum()) == 2 * 4
  assert torch.equal(x[outside], pos.expand(B, T, d)[outside])


def test_out_of_vocabulary_ids_encode_as_the_reference(cuda_device):
  """test_gpu_model.test_encode's set-up with ids >= vocab on attended positions: the reference's
  one-hot embedding gives them a zero row (only the position row), and so must the engine."""
  T = N = C = 128
  t5 = config.t5_tiny()
  params = weights.synthetic_params(t5, T, N, C, seed=0)
  B = 3
  toks, ctx, cmask = H.make_batch(B, T, C, ctx_masks=[1, 0, 1])
  cmask[2, 40:] = 0
  toks[0, 5] = t5.vocab_size
  toks[0, 17] = t5.vocab_size + 100
  toks[2, 3] = 2 ** 31 - 1
  toks[1, 9] = t5.vocab_size
  eng = H.build_engine(t5, T, N, C, B, 4, 2.0, params)
  b = H.torch_batch(toks, ctx, cmask, cuda_device)
  eng.encode(b['encoder_input_tokens'], b['encoder_continuous_inputs'], b['encoder_continuous_mask'])
  got = eng.encodings().cpu()
  oc = H.oracle_config(t5, 4, 2.0)
  cb = H.torch_batch(toks, ctx, cmask)
  encs = O.encode(O.params_to(params), oc, cb['encoder_input_tokens'],
                  O.scale_features(cb['encoder_continuous_inputs'], oc, clip=True),
                  cb['encoder_continuous_mask'])
  want = torch.cat([encs[0][0], encs[1][0]], dim=1)
  valid = torch.cat([encs[0][1], encs[1][1]], dim=1) > 0
  assert bool(valid[0, 5]) and bool(valid[2, 3])
  err = ((got - want).abs() * valid.unsqueeze(-1)).max().item()
  assert torch.isfinite(got).all()
  assert err < 6e-2, f'max err on valid positions {err}'
  eng.close()
