"""-m gpu: the GEMM through every launch form the engine uses (engine.cu: decoder_layers
in both norm forms, run_decoder, msd_encode), on caller-owned buffers with the engine's strides,
offsets, step-indexed tables and deferred-normalisation arguments (msd_op_gemm_view,
msd_op_prep_rows), and the load-time conditioning tables behind them (msd_get_conditioning_tables).

Base dimensions: d = 768, hh = 768, F = 2048, N = 256, n_dims = 128.  The step tables (column
gains, the two bias-row tables) are built from FiLM rows that are independent random draws per
step, read at device steps 0, 6 and 12 of 13: reading a neighbouring row is off by O(1), never by a
rounding-level amount.  Every output and prep.a buffer starts as a bf16-exact sentinel with MARGIN
rows past its view, every partial-row-sum slot as NaN; after each launch everything outside the
slice it writes is bit-identical to before (an ss slot read but not written shows up as NaN).
Three draws run into the same buffers, one per step.

(a) Tight, per launch: fp64 from the device's own upstream outputs (its x, prep.a, ss), held to a
per-element bound from the kernel's rounding points (u = 2^-24):
  * accumulation: the tensor core rounds its fp32 partial sum at most once per k16 MMA, by at
    most 2u of the sum so far, so |acc - exact| <= (K / 16) 2u sum_k |a_k w_k|;
  * row scale: rsqrtf is within 2 ulp (2^-22 relative), the fp32 sum of <= 12 partials and the
    scaling by 1/d and +1e-6 add < 8u, so inv_r is within 3 * 2^-22 relative; the product with
    the accumulator and the bias add round once each (u |.|);
  * gated GELU: tanh.approx.f32 is within 2^-10.9 absolute, its fp32 argument within 3u relative;
    r's error passes through gelu' <= 1.13, g's through |gelu(r)|;
  * bf16 output: one rounding to nearest, half an ulp at the value (<= 2^-8 |y|), f32 output u |y|;
  * prep.a = bf16(x g): u |x g| + half an ulp; the per-tile sums of squares: each lane chains
    BN / 4 fmas, then two shuffles, (BN / 4 + 4) u sum x^2; prep_rows: (d / 32 + 8) u sum x^2.
(b) Loose, one whole fused decoder layer against the plain order of operations in fp64 from the
layer input and the raw FiLM rows (rmsnorm -> gamma (1 + fs) + fb -> dense), with a random fixed
"attention output": the only extra error is the bf16 operand rounding, 2^-8 inv_r sum_k |x_k g_k w_k|
per projection, carried through the layer.

Measured on an H100 80GB HBM3 at a 700 W power limit, the largest err / bound per group (printed
as '[err/bound] <group>: ...'): prep.a 1.000 and prep_rows 1.000 (an fp32 product x g that lands on
a bf16 rounding midpoint meets that rounding's worst case exactly), row scale 0.993, row scale +
bias 0.994, gated 0.919, partial sums 0.198, f32 epilogues 0.326, split precision 0.103, loose
layer 0.252, conditioning tables 0.969.  The fp32 outputs sit well inside their bounds because
the accumulation term is a worst case over K / 16 roundings; the bf16 outputs are held to within
a few percent of their output rounding alone.
"""
import math

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import _native, config, engine, weights
from oracle import msd_oracle as O

pytestmark = pytest.mark.gpu

D, HH, F, N, ND, C = 768, 768, 2048, 256, 128, 256
STEPS, LD = 13, 2                  # step tables of a 2-layer decoder, num_steps not a multiple of 8
TEST_STEPS = (0, 6, STEPS - 1)
GSTRIDE = 2 * LD * D               # engine: gtab step stride
SENTINEL = -7.25
MARGIN = 64
KSS = 16                           # partial-sum slots per table (engine: kSsParts)
U = 2.0 ** -24
E_TANH = 2.0 ** -10.9
WIDTHS = (64, 96, 128, 192, 256)


# ---- bounds ------------------------------------------------------------------------------------
def half_ulp_bf16(x: torch.Tensor) -> torch.Tensor:
  """Half a bf16 ulp at |x| (8 significant bits)."""
  _, e = torch.frexp(x.abs().double())
  return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (e - 9).to(torch.int32))


def acc_err(k: int, abs_sum: torch.Tensor) -> torch.Tensor:
  return (k / 16) * 2 * U * abs_sum


def check(got, want, bound, group, what):
  got = got.double()
  assert bool(torch.isfinite(got).all()), what
  ratio = ((got - want).abs() / bound).max().item()
  print(f'[err/bound] {group}: {what}: {ratio:.3f}')
  assert ratio <= 1.0, (what, ratio)


def check_bf16(got, want, e_pre, group, what):
  check(got, want, half_ulp_bf16(want.abs() + e_pre) + e_pre, group, what)


def gelu64(x):
  return O.gelu_tanh(x)


def gated_split(acc: torch.Tensor):
  """[M, 2F] accumulator columns (32 of wi_0, 32 of wi_1, ...) -> (r, g) [M, F]."""
  m, n2 = acc.shape
  a = acc.reshape(m, n2 // 64, 2, 32)
  return a[:, :, 0].reshape(m, n2 // 2), a[:, :, 1].reshape(m, n2 // 2)


def gated_bound(r, g, e_r, e_g):
  """Pre-rounding error of gelu(r) g from errors e_r, e_g of its inputs."""
  uarg = 0.7978845608028654 * (r + 0.044715 * r ** 3)
  return (1.13 * e_r * g.abs() + gelu64(r).abs() * e_g +
          0.5 * (r * g).abs() * (E_TANH + 3 * U * uarg.abs()) + 4 * U * (gelu64(r) * g).abs())


# ---- buffers ---------------------------------------------------------------------------------
def view(t, off, ld, rows, cols):
  return torch.as_strided(t, (rows, cols), (ld, 1), off)


class Buffers:
  """Flat device buffers by name; `launch` checks that a call writes nothing outside its slices."""

  def __init__(self, device):
    self.t = {}
    self.dev = device

  def add(self, name, rows, ld, dtype, fill=SENTINEL):
    self.t[name] = torch.full(((rows + MARGIN) * ld,), fill, dtype=dtype, device=self.dev)
    return self.t[name]

  def __getitem__(self, name):
    return self.t[name]

  def launch(self, fn, writes):
    """writes: [(name, off, ld, rows, cols)] the call may write."""
    before = {k: v.clone() for k, v in self.t.items()}
    ret = fn()
    for name, t in self.t.items():
      mask = torch.ones(t.numel(), dtype=torch.bool, device=self.dev)
      for (wn, off, ld, rows, cols) in writes:
        if wn == name:
          view(mask, off, ld, rows, cols).fill_(False)
      bits = torch.int16 if t.element_size() == 2 else torch.int32
      same = t[mask].view(bits) == before[name][mask].view(bits)
      assert bool(same.all()), f'{name}: {int((~same).sum())} elements outside the written slices changed'
    return ret


def ss_view(t, stride, parts, rows):
  return view(t, 0, stride, parts, rows)


def inv_rows(tab, parts, stride, rows, d=D):
  """fp64 rsqrt(mean x^2 + eps) from the device's partial sums: [rows]."""
  ss = ss_view(tab, stride, parts, rows).double().sum(0)
  return torch.rsqrt(ss / d + 1e-6)


def rand_bf16(shape, g, scale, device):
  return (torch.randn(shape, generator=g, device=device) * scale).to(torch.bfloat16)


# ---- the per-step conditioning, from raw FiLM rows ---------------------------------------------
class StepTables:
  """Per layer: gamma_self, gamma_cross, gamma_mlp [d]; per step and layer FiLM rows (fs | fb) of
  the two FiLM layers, independent draws; the derived tables as the engine lays them out."""

  def __init__(self, w_qkv, w_wi, g, device):
    self.gamma = torch.rand(LD, 3, D, generator=g, device=device, dtype=torch.float64) + 0.5
    self.fs = torch.randn(STEPS, LD, 2, D, generator=g, device=device, dtype=torch.float64) * 0.3
    self.fb = torch.randn(STEPS, LD, 2, D, generator=g, device=device, dtype=torch.float64) * 0.3
    gain = torch.empty(STEPS, 2 * LD, D, dtype=torch.float64, device=device)
    for l in range(LD):
      gain[:, 2 * l] = self.gamma[l, 0] * (1 + self.fs[:, l, 0])
      gain[:, 2 * l + 1] = self.gamma[l, 2] * (1 + self.fs[:, l, 1])
    self.gtab = gain.float().contiguous()
    self.ln_cross = [self.gamma[l, 1].float().contiguous() for l in range(LD)]
    self.btab_qkv = torch.stack([self.fb[:, l, 0] @ w_qkv[l].double().T for l in range(LD)], 1).float().contiguous()
    self.btab_wi = torch.stack([self.fb[:, l, 1] @ w_wi[l].double().T for l in range(LD)], 1).float().contiguous()

  # (tensor, element offset, step stride) as the engine passes them
  def g_self(self, l):
    return (self.gtab, 2 * l * D, GSTRIDE)

  def g_mlp(self, l):
    return (self.gtab, (2 * l + 1) * D, GSTRIDE)

  def b_qkv(self, l):
    return (self.btab_qkv, l * 3 * HH, LD * 3 * HH)

  def b_wi(self, l):
    return (self.btab_wi, l * 2 * F, LD * 2 * F)


def at_step(tab, s, n):
  """The n values a launch reads from (tensor, offset, step stride) at step s, fp64."""
  t, off, stride = tab
  return t.view(-1)[off + s * stride:off + s * stride + n].double()


# ---- one fused decoder layer, launch by launch -----------------------------------------------
FORMS = {'guided': (2, 1), 'unguided': (1, 1), 'unconditioned': (1, 0)}   # (passes, conditioned)


def widths_for(plan, epi_bf16):
  """block_n of each GEMM under a plan: 'auto', a forced width (auto where it is not allowed)."""
  if plan == 'auto' or plan == 'mixed':
    return 0
  if plan == 96 and epi_bf16:
    return 0
  return plan


def bn_for(plan, n, bf16_out):
  w = widths_for(plan, bf16_out)
  return w if (w == 0 or n % w == 0) else 0


class Layer:
  def __init__(self, B, form, nsrc, device, seed):
    passes, cond = FORMS[form]
    self.B, self.nsrc = B, nsrc
    self.R = passes * B * N
    self.Rc = B * N if cond else 0
    self.ss_stride = self.R + 128
    g = torch.Generator(device).manual_seed(seed)
    self.g = g
    self.dev = device
    k = lambda n, kk, sc=1.0: rand_bf16((n, kk), g, sc / math.sqrt(kk), device)
    self.w_qkv = [k(3 * HH, D) for _ in range(LD)]
    self.w_out = k(D, HH)
    self.w_cq = k(nsrc * HH, D)
    self.w_co = k(D, nsrc * HH)
    self.w_wi = [k(2 * F, D) for _ in range(LD)]
    self.w_wo = k(D, F)
    self.tabs = StepTables(self.w_qkv, self.w_wi, g, device)
    self.step = torch.zeros(1, dtype=torch.int32, device=device)
    b = Buffers(device)
    R = self.R
    b.add('x', R, D, torch.float32)
    b.add('x_last', R, D, torch.float32)
    b.add('xn', R, D, torch.bfloat16)
    b.add('qkv', R, 3 * HH, torch.bfloat16)
    b.add('attn', R, HH, torch.bfloat16)
    b.add('qc', R, nsrc * HH, torch.bfloat16)
    b.add('attn2', R, nsrc * HH, torch.bfloat16)
    b.add('hmid', R, F, torch.bfloat16)
    for s in ('ss_x', 'ss_so', 'ss_co'):
      b.t[s] = torch.full((KSS * self.ss_stride,), float('nan'), device=device)
    self.b = b

  # -- the launches, each with its tight check ------------------------------------------------
  def gemm(self, a, a_off, lda, w, m, n, k, epi, out, ldo, **kw):
    return engine.op_gemm_view(a, a_off, lda, w, 0, k, m, n, k, epi, out, 0, ldo, step=self.step, **kw)

  def rs(self, lo, plo, hi, phi, split, bias):
    return dict(ss_lo=self.b[lo], parts_lo=plo, ss_hi=self.b[hi], parts_hi=phi, split_row=split,
                ss_stride=self.ss_stride, inv_d=1.0 / D, bias=bias)

  def inv(self, lo, plo, hi, phi, split, m):
    i_lo = inv_rows(self.b[lo], plo, self.ss_stride, m)
    i_hi = inv_rows(self.b[hi], phi, self.ss_stride, m)
    rows = torch.arange(m, device=self.dev)
    return torch.where(rows < split, i_lo, i_hi)

  def check_scaled(self, got, a, w, inv, bias, k, group, what):
    """bf16 out = bf16(inv acc + bias): returns the fp64 pre-rounding value and its error bound."""
    acc = a.double() @ w.double().T
    aw = a.double().abs() @ w.double().abs().T
    y = inv[:, None] * acc + (0 if bias is None else bias[None, :])
    e = inv[:, None] * acc_err(k, aw) + 3 * 2.0 ** -22 * (inv[:, None] * acc).abs() + U * (
        (inv[:, None] * acc).abs() + y.abs())
    if got is not None:
      check_bf16(got, y, e, group, what)
    return y, e

  def resid_prep(self, a, a_off, lda, w, m, k, g_lo, g_hi, split, ss, bn, group, what, x_name='x'):
    """EPI_RESID_PREP in place on x: checks x, prep.a, the partial sums; returns the parts."""
    b, s = self.b, int(self.step.item())
    x_old = view(b[x_name], 0, D, m, D).double()
    bn_run = b.launch(lambda: self.gemm(a, a_off, lda, w, m, D, k, 'resid_prep', b[x_name], D,
                                        block_n=bn, resid=b[x_name],
                                        prep=dict(g_lo=g_lo, g_hi=g_hi, split_row=split, a=b['xn'], lda=D,
                                                  ss=b[ss], ss_stride=self.ss_stride)),
                      [(x_name, 0, D, m, D), ('xn', 0, D, m, D), (ss, 0, self.ss_stride, D // max(bn, 1) if bn else KSS, m)])
    parts = D // bn_run
    av = view(a, a_off, lda, m, k).double()
    acc = av @ w.double().T
    want = x_old + acc
    xd = view(b[x_name], 0, D, m, D)
    check(xd, want, acc_err(k, av.abs() @ w.double().abs().T) + U * want.abs() + 1e-30,
          'f32 epilogues', f'{what}: x')
    xd = xd.double()
    rows = torch.arange(m, device=self.dev)[:, None]
    gv = torch.where(rows < split, at_step(g_lo, s, D)[None, :], at_step(g_hi, s, D)[None, :])
    xg = xd * gv
    check_bf16(view(b['xn'], 0, D, m, D), xg, U * xg.abs(), 'prep.a', f'{what}: prep.a')
    got_ss = ss_view(b[ss], self.ss_stride, parts, m).double()
    want_ss = (xd ** 2).reshape(m, parts, bn_run).sum(-1).T
    check(got_ss, want_ss, (bn_run / 4 + 4) * U * want_ss + 1e-30, 'partial sums', f'{what}: ss')
    assert bool(torch.isnan(view(b[ss], 0, self.ss_stride, KSS, m)[parts:]).all()), f'{what}: extra ss slots'
    return parts, bn_run

  def run(self, plan, s, draw, loose):
    """One draw at step s: the layer's launches in the engine's order with tight checks, then the
    loose comparison of the whole layer.  Returns {launch: tile width} of what ran."""
    B, R, Rc, nsrc, b, T = self.B, self.R, self.Rc, self.nsrc, self.b, self.tabs
    g, dev = self.g, self.dev
    tag = f'B={B} R={R} Rc={Rc} nsrc={nsrc} plan={plan} step={s}'
    self.step.fill_(s)
    for name in ('ss_x', 'ss_so', 'ss_co'):
      b[name].fill_(float('nan'))
    x0 = torch.randn(R, D, generator=g, device=dev) * (0.5 + draw)
    view(b['x'], 0, D, R, D).copy_(x0)
    view(b['attn'], 0, HH, R, HH).copy_(rand_bf16((R, HH), g, 1.0, dev))
    view(b['attn2'], 0, nsrc * HH, R, nsrc * HH).copy_(rand_bf16((R, nsrc * HH), g, 1.0, dev))
    ran = {}
    # 1. layer 0's prep: no GEMM produced the stream
    b.launch(lambda: engine.op_prep_rows(b['x'], T.gtab, 0, GSTRIDE, self.step, R, D, b['xn'], D, b['ss_x']),
             [('xn', 0, D, R, D), ('ss_x', 0, self.ss_stride, 1, R)])
    xg = x0.double() * at_step(T.g_self(0), s, D)[None, :]
    check_bf16(view(b['xn'], 0, D, R, D), xg, U * xg.abs(), 'prep_rows', f'{tag}: prep_rows a')
    want_ss = (x0.double() ** 2).sum(1)
    check(b['ss_x'][:R], want_ss, (D / 32 + 8) * U * want_ss, 'prep_rows', f'{tag}: prep_rows ss')
    # 2. QKV with row scale (1 partial) and the layer's step-indexed bias row
    xn0 = view(b['xn'], 0, D, R, D).clone()
    bn = bn_for(plan, 3 * HH, True)
    ran['qkv'] = b.launch(lambda: self.gemm(b['xn'], 0, D, self.w_qkv[0], R, 3 * HH, D, 'bf16', b['qkv'], 3 * HH,
                                            block_n=bn, rs=self.rs('ss_x', 1, 'ss_x', 1, R, T.b_qkv(0))),
                          [('qkv', 0, 3 * HH, R, 3 * HH)])
    inv0 = self.inv('ss_x', 1, 'ss_x', 1, R, R)
    self.check_scaled(view(b['qkv'], 0, 3 * HH, R, 3 * HH), xn0, self.w_qkv[0], inv0,
                      at_step(T.b_qkv(0), s, 3 * HH), D, 'row scale + bias', f'{tag}: qkv')
    # 3. self-attention out-projection: ln_cross (step stride 0) below Rc, g_mlp from Rc on
    g_mlp = T.g_mlp(0)
    g_lo = (T.ln_cross[0], 0, 0) if Rc > 0 else g_mlp
    bn_so = 192 if plan == 'mixed' else bn_for(plan, D, False)
    parts_so, ran['self_out'] = self.resid_prep(b['attn'], 0, HH, self.w_out, R, HH, g_lo, g_mlp, Rc, 'ss_so',
                                                bn_so, 'resid_prep', f'{tag}: self_out')
    x1 = view(b['x'], 0, D, R, D).double().clone()
    # 4.-5. cross-attention block over the first Rc rows
    parts_co = parts_so
    if Rc > 0:
      xn1 = view(b['xn'], 0, D, Rc, D).clone()
      bn = bn_for(plan, nsrc * HH, True)
      ran['cross_q'] = b.launch(
          lambda: self.gemm(b['xn'], 0, D, self.w_cq, Rc, nsrc * HH, D, 'bf16', b['qc'], nsrc * HH, block_n=bn,
                            rs=self.rs('ss_so', parts_so, 'ss_so', parts_so, Rc, None)),
          [('qc', 0, nsrc * HH, Rc, nsrc * HH)])
      inv1 = self.inv('ss_so', parts_so, 'ss_so', parts_so, Rc, Rc)
      self.check_scaled(view(b['qc'], 0, nsrc * HH, Rc, nsrc * HH), xn1, self.w_cq, inv1, None, D,
                        'row scale', f'{tag}: cross_q')
      bn_co = 64 if plan == 'mixed' else bn_for(plan, D, False)
      parts_co, ran['cross_out'] = self.resid_prep(b['attn2'], 0, nsrc * HH, self.w_co, Rc, nsrc * HH, g_mlp,
                                                   g_mlp, Rc, 'ss_co', bn_co, 'resid_prep', f'{tag}: cross_out')
      assert bool(torch.isnan(view(b['ss_co'], 0, self.ss_stride, KSS, R)[:, Rc:]).all())
    x2 = view(b['x'], 0, D, R, D).double().clone()
    # 6. MLP wi, gated: rows < Rc scaled by ss_co, the others by ss_so
    xn2 = view(b['xn'], 0, D, R, D).clone()
    bn = bn_for(plan, 2 * F, True)
    rs = (self.rs('ss_co', parts_co, 'ss_so', parts_so, Rc, T.b_wi(0)) if Rc > 0 else
          self.rs('ss_so', parts_so, 'ss_so', parts_so, R, T.b_wi(0)))
    ran['wi'] = b.launch(lambda: self.gemm(b['xn'], 0, D, self.w_wi[0], R, 2 * F, D, 'gated_gelu', b['hmid'], F,
                                           block_n=bn, rs=rs), [('hmid', 0, F, R, F)])
    inv2 = (self.inv('ss_co', parts_co, 'ss_so', parts_so, Rc, R) if Rc > 0 else
            self.inv('ss_so', parts_so, 'ss_so', parts_so, R, R))
    y, e = self.check_scaled(None, xn2, self.w_wi[0], inv2, at_step(T.b_wi(0), s, 2 * F), D, '', '')
    (r, gg), (er, eg) = gated_split(y), gated_split(e)
    h = gelu64(r) * gg
    check_bf16(view(b['hmid'], 0, F, R, F), h, gated_bound(r, gg, er, eg), 'gated', f'{tag}: wi')
    # 7. MLP wo: into the next layer's gain (partials d / bn), then that layer's QKV; and the last
    # layer's plain residual form from the same stream
    view(b['x_last'], 0, D, R, D).copy_(view(b['x'], 0, D, R, D))
    hm = view(b['hmid'], 0, F, R, F).clone()
    g_next = T.g_self(1)
    bn_wo = bn_for(plan, D, False)
    parts_x, ran['wo'] = self.resid_prep(b['hmid'], 0, F, self.w_wo, R, F, g_next, g_next, R, 'ss_x', bn_wo,
                                         'resid_prep', f'{tag}: wo')
    xn3 = view(b['xn'], 0, D, R, D).clone()
    bn = bn_for(plan, 3 * HH, True)
    b.launch(lambda: self.gemm(b['xn'], 0, D, self.w_qkv[1], R, 3 * HH, D, 'bf16', b['qkv'], 3 * HH, block_n=bn,
                               rs=self.rs('ss_x', parts_x, 'ss_x', parts_x, R, T.b_qkv(1))),
             [('qkv', 0, 3 * HH, R, 3 * HH)])
    inv3 = self.inv('ss_x', parts_x, 'ss_x', parts_x, R, R)
    self.check_scaled(view(b['qkv'], 0, 3 * HH, R, 3 * HH), xn3, self.w_qkv[1], inv3,
                      at_step(T.b_qkv(1), s, 3 * HH), D, 'row scale + bias', f'{tag}: qkv layer 1')
    b.launch(lambda: self.gemm(b['hmid'], 0, F, self.w_wo, R, D, F, 'resid_f32', b['x_last'], D, block_n=bn_wo,
                               resid=b['x_last']), [('x_last', 0, D, R, D)])
    acc = hm.double() @ self.w_wo.double().T
    want = x2 + acc
    check(view(b['x_last'], 0, D, R, D), want,
          acc_err(F, hm.double().abs() @ self.w_wo.double().abs().T) + U * want.abs() + 1e-30,
          'f32 epilogues', f'{tag}: wo last layer')
    ran.update(parts_so=parts_so, parts_co=parts_co, parts_x=parts_x)
    if loose:
      self.loose(x0.double(), s, tag)
    return ran

  def loose(self, x0, s, tag):
    """The layer in the plain order of operations from its input and the raw FiLM rows."""
    b, T, R, Rc, nsrc = self.b, self.tabs, self.R, self.Rc, self.nsrc

    def rms(x):
      return torch.rsqrt((x * x).mean(1) + 1e-6)

    def proj(x, ex, gain, bias, w):
      """(rmsnorm(x) gain + bias) w, and the error bound of the split form from bf16 operands,
      the input's error ex (through the operand and, at most as much again, the row scale) and
      the tight form's fp32 terms."""
      inv = rms(x)
      wd = w.double()
      acc = (x * inv[:, None] * gain[None, :]) @ wd.T
      b = 0 if bias is None else (bias @ wd.T)[None, :]
      e = inv[:, None] * ((2.0 ** -8 * (x * gain[None, :]).abs() + 2 * ex * gain.abs()[None, :]) @ wd.abs().T)
      e = e * (1 + 2.0 ** -6) + inv[:, None] * acc_err(D, (x * gain[None, :]).abs() @ wd.abs().T)
      return acc + b, e + 2.0 ** -20 * (acc.abs() + abs(b))

    fs, fb, gam = T.fs[s, 0], T.fb[s, 0], T.gamma[0]
    y, e = proj(x0, 0, gam[0] * (1 + fs[0]), fb[0], self.w_qkv[0])
    # the device's QKV of this draw was overwritten by layer 1's; rebuild layer 0's from a fresh launch
    qkv = torch.empty(R * 3 * HH, dtype=torch.bfloat16, device=self.dev)
    xn = torch.empty(R * D, dtype=torch.bfloat16, device=self.dev)
    ssx = torch.empty(self.ss_stride * KSS, device=self.dev)
    xin = x0.float().contiguous()
    engine.op_prep_rows(xin, T.gtab, 0, GSTRIDE, self.step, R, D, xn, D, ssx)
    self.gemm(xn, 0, D, self.w_qkv[0], R, 3 * HH, D, 'bf16', qkv, 3 * HH,
              rs=dict(ss_lo=ssx, parts_lo=1, ss_hi=ssx, parts_hi=1, split_row=R, ss_stride=self.ss_stride,
                      inv_d=1.0 / D, bias=T.b_qkv(0)))
    check_bf16(qkv.view(R, 3 * HH), y, e, 'loose layer', f'{tag}: loose qkv')
    at = b['attn'][:R * HH].view(R, HH).double()
    x1 = x0 + at @ self.w_out.double().T
    ex1 = acc_err(HH, at.abs() @ self.w_out.double().abs().T) + U * x1.abs()
    x2, ex2 = x1.clone(), ex1.clone()
    if Rc > 0:
      y, e = proj(x1[:Rc], ex1[:Rc], gam[1], None, self.w_cq)
      check_bf16(b['qc'][:Rc * nsrc * HH].view(Rc, nsrc * HH), y, e, 'loose layer', f'{tag}: loose cross_q')
      a2 = b['attn2'][:Rc * nsrc * HH].view(Rc, nsrc * HH).double()
      x2[:Rc] = x1[:Rc] + a2 @ self.w_co.double().T
      ex2[:Rc] += acc_err(nsrc * HH, a2.abs() @ self.w_co.double().abs().T) + U * x2[:Rc].abs()
    y, e = proj(x2, ex2, gam[2] * (1 + fs[1]), fb[1], self.w_wi[0])
    (r, gg), (er, eg) = gated_split(y), gated_split(e)
    h = gelu64(r) * gg
    eh = gated_bound(r, gg, er, eg)
    check_bf16(b['hmid'][:R * F].view(R, F), h, eh, 'loose layer', f'{tag}: loose wi')
    wo = self.w_wo.double()
    x3 = x2 + h @ wo.T
    ex3 = ((eh + half_ulp_bf16(h.abs() + eh)) @ wo.abs().T + ex2 + acc_err(F, h.abs() @ wo.abs().T) +
           U * x3.abs())
    check(b['x_last'][:R * D].view(R, D), x3, ex3, 'loose layer', f'{tag}: loose x after wo')


LAYER_CASES = ([(B, 'guided', nsrc, plan) for B in (1, 3, 8) for nsrc in (1, 2)
                for plan in ('auto', 'mixed') + WIDTHS] +
               [(3, 'unguided', nsrc, plan) for nsrc in (1, 2) for plan in ('auto', 'mixed', 64)] +
               [(3, 'unconditioned', 1, plan) for plan in ('auto', 96, 256)])


@pytest.mark.parametrize('B,form,nsrc,plan', LAYER_CASES)
def test_fused_decoder_layer_launches(cuda_device, B, form, nsrc, plan):
  """decoder_layers in the deferred form, one layer plus the next layer's QKV, every launch as the
  engine makes it (plan: the engine's automatic tile widths, one width forced wherever it is
  allowed, or 'mixed': self-out at 192 and cross-out at 64 columns, so the MLP's two row-scale
  tables have 4 and 12 partial sums)."""
  layer = Layer(B, form, nsrc, cuda_device, seed=1000 * B + 10 * nsrc + len(str(plan)))
  for draw, s in enumerate(TEST_STEPS):
    ran = layer.run(plan, s, draw, loose=(plan == 'auto'))
    print(f'[tiles] B={B} {form} nsrc={nsrc} plan={plan}: {ran}')
  if plan == 'mixed' and layer.Rc > 0 and layer.Rc < layer.R:
    assert ran['parts_co'] != ran['parts_so']


def test_split_row_inside_a_block(cuda_device):
  """The kernel picks g_lo / g_hi and the ss_lo / ss_hi pair per row: a split at row 200, inside
  the second 128-row block, with 12 and 4 partial sums (the engine's splits fall on block bounds)."""
  dev = cuda_device
  layer = Layer(1, 'guided', 1, dev, seed=77)
  b, T, R = layer.b, layer.tabs, layer.R
  split = 200
  for draw, s in enumerate(TEST_STEPS):
    layer.step.fill_(s)
    for name in ('ss_x', 'ss_so', 'ss_co'):
      b[name].fill_(float('nan'))
    view(b['x'], 0, D, R, D).copy_(torch.randn(R, D, generator=layer.g, device=dev))
    view(b['attn'], 0, HH, R, HH).copy_(rand_bf16((R, HH), layer.g, 1.0, dev))
    tag = f'split {split} step {s}'
    # two producers over all rows at different widths; the consumer takes rows < split from the first
    layer.resid_prep(b['attn'], 0, HH, layer.w_out, R, HH, (T.ln_cross[0], 0, 0), T.g_mlp(0), split, 'ss_co',
                     64, 'resid_prep', f'{tag}: producer 64')
    p_lo = D // 64
    ss_lo_copy = b['ss_co'].clone()
    view(b['x'], 0, D, R, D).copy_(torch.randn(R, D, generator=layer.g, device=dev))
    p_hi, _ = layer.resid_prep(b['attn'], 0, HH, layer.w_out, R, HH, T.g_mlp(0), T.g_mlp(0), split, 'ss_so',
                               192, 'resid_prep', f'{tag}: producer 192')
    b['ss_co'].copy_(ss_lo_copy)
    xn = view(b['xn'], 0, D, R, D).clone()
    b.launch(lambda: layer.gemm(b['xn'], 0, D, layer.w_wi[0], R, 2 * F, D, 'gated_gelu', b['hmid'], F,
                                rs=layer.rs('ss_co', p_lo, 'ss_so', p_hi, split, T.b_wi(0))),
             [('hmid', 0, F, R, F)])
    inv = layer.inv('ss_co', p_lo, 'ss_so', p_hi, split, R)
    y, e = layer.check_scaled(None, xn, layer.w_wi[0], inv, at_step(T.b_wi(0), s, 2 * F), D, '', '')
    (r, gg), (er, eg) = gated_split(y), gated_split(e)
    check_bf16(view(b['hmid'], 0, F, R, F), gelu64(r) * gg, gated_bound(r, gg, er, eg), 'gated', f'{tag}: wi')


# ---- split-precision GEMMs -----------------------------------------------------------------------
def split3(v: torch.Tensor):
  """[hi | lo | hi] bf16 of fp32 rows (the A operand of a split-precision GEMM)."""
  hi = v.to(torch.bfloat16)
  lo = (v - hi.float()).to(torch.bfloat16)
  return torch.cat([hi, lo, hi], 1).contiguous()


def split3_w(w: torch.Tensor):
  """[hi | hi | lo] bf16 of fp32 weight rows [N, K]."""
  hi = w.to(torch.bfloat16)
  lo = (w - hi.float()).to(torch.bfloat16)
  return torch.cat([hi, hi, lo], 1).contiguous()


def check_f32_gemm(got, a, w, k, add, group, what):
  acc = a.double() @ w.double().T
  want = acc + (0 if add is None else add)
  bound = acc_err(k, a.double().abs() @ w.double().abs().T) + U * want.abs() + 1e-30
  check(got, want, bound, group, what)
  return want


@pytest.mark.parametrize('B', [1, 3, 8])
def test_spec_out_split_precision(cuda_device, B):
  """run_decoder's last GEMM: EPI_F32, N = n_dims = 128, K = 3d over [hi | lo | hi] rows of the
  decoder norm's output against the [hi | hi | lo] spec_out weights; its output is the eps every
  sampler step consumes.  Also within 2^-14 relative of the fp32 product."""
  dev = cuda_device
  R = 2 * B * N
  g = torch.Generator(dev).manual_seed(90 + B)
  b = Buffers(dev)
  b.add('xn', R, 3 * D, torch.bfloat16)
  b.add('eps', R, ND, torch.float32)
  w32 = torch.randn(ND, D, generator=g, device=dev) / math.sqrt(D)
  w = split3_w(w32)
  for draw in range(2):
    v = O.layer_norm(torch.randn(R, D, generator=g, device=dev) * (1 + draw),
                     1 + 0.1 * torch.randn(D, generator=g, device=dev))
    view(b['xn'], 0, 3 * D, R, 3 * D).copy_(split3(v))
    a = view(b['xn'], 0, 3 * D, R, 3 * D).clone()
    b.launch(lambda: engine.op_gemm_view(b['xn'], 0, 3 * D, w, 0, 3 * D, R, ND, 3 * D, 'f32', b['eps'], 0, ND),
             [('eps', 0, ND, R, ND)])
    got = view(b['eps'], 0, ND, R, ND)
    check_f32_gemm(got, a, w, 3 * D, None, 'split precision', f'spec_out B={B} draw {draw}')
    exact = v.double() @ w32.double().T
    rel = ((got.double() - exact).abs() / (v.double().abs() @ w32.double().abs().T)).max().item()
    assert rel < 2.0 ** -14, rel


@pytest.mark.parametrize('guided', [True, False])
@pytest.mark.parametrize('B', [1, 3, 8])
def test_input_projections(cuda_device, B, guided):
  """dec_in_proj: EPI_POS_F32 over the [hi | lo | hi] z rows (lda = 3 n_dims = 384), position rows
  of N, duplicated to the unconditional rows (dup_rows = B N) with guidance.  ctx_in_proj: the
  same over B context segments of C frames, each position table rolled by ctx_seq_len[b]."""
  dev = cuda_device
  g = torch.Generator(dev).manual_seed(100 + B + 7 * guided)
  R = (2 if guided else 1) * B * N
  b = Buffers(dev)
  b.add('z', B * N, 3 * ND, torch.bfloat16)
  b.add('x', R, D, torch.float32)
  b.add('ctx', B * C, 3 * ND, torch.bfloat16)
  b.add('ex', B * C, D, torch.float32)
  w = split3_w(torch.randn(D, ND, generator=g, device=dev) / math.sqrt(ND))
  wc = split3_w(torch.randn(D, ND, generator=g, device=dev) / math.sqrt(ND))
  pos = torch.randn(N, D, generator=g, device=dev)
  cpos = torch.randn(C, D, generator=g, device=dev)
  shift = torch.tensor([0, 100, 255, 1, 128, 37, 200, 5][:B], dtype=torch.int32, device=dev)
  dup = B * N if guided else 0
  for draw in range(2):
    view(b['z'], 0, 3 * ND, B * N, 3 * ND).copy_(split3(torch.randn(B * N, ND, generator=g, device=dev)))
    view(b['ctx'], 0, 3 * ND, B * C, 3 * ND).copy_(split3(torch.rand(B * C, ND, generator=g, device=dev) * 2 - 1))
    z = view(b['z'], 0, 3 * ND, B * N, 3 * ND).clone()
    b.launch(lambda: engine.op_gemm_view(b['z'], 0, 3 * ND, w, 0, 3 * ND, B * N, D, 3 * ND, 'pos_f32', b['x'], 0, D,
                                         pos=pos, dup_rows=dup),
             [('x', 0, D, B * N + dup, D)])
    want = check_f32_gemm(view(b['x'], 0, D, B * N, D), z, w, 3 * ND, pos.double().repeat(B, 1),
                          'f32 epilogues', f'dec_in_proj B={B} guided={guided} draw {draw}')
    if dup:
      assert torch.equal(view(b['x'], 0, D, B * N, D).view(torch.int32),
                         view(b['x'], B * N * D, D, B * N, D).view(torch.int32))
    cz = view(b['ctx'], 0, 3 * ND, B * C, 3 * ND).clone()
    b.launch(lambda: engine.op_gemm_view(b['ctx'], 0, 3 * ND, wc, 0, 3 * ND, B * C, D, 3 * ND, 'pos_f32', b['ex'],
                                         0, D, pos=cpos, pos_shift=shift),
             [('ex', 0, D, B * C, D)])
    rows = torch.arange(B * C, device=dev)
    pr = (rows % C - shift.long()[rows // C]) % C
    check_f32_gemm(view(b['ex'], 0, D, B * C, D), cz, wc, 3 * ND, cpos.double()[pr],
                   'f32 epilogues', f'ctx_in_proj B={B} draw {draw}')
    del want


@pytest.mark.parametrize('B,nsrc', [(1, 1), (3, 2), (8, 1), (8, 2)])
def test_fp32_accurate_decoder_launches(cuda_device, B, nsrc):
  """decoder_layers / cross_attention in the fp32-accurate mode: every dense is a 3 x bf16
  split product (K tripled); q / k / v and the cross q come out fp32 (EPI_F32), the residual
  projections add in place (EPI_RESID_F32, cross-out over the first B N rows of 2 B N), the gated
  MLP writes [hi | lo | hi] into ldo = 3F (EPI_GATED_GELU_SPLIT3, exact tanh)."""
  dev = cuda_device
  g = torch.Generator(dev).manual_seed(200 + B + nsrc)
  R, Rc = 2 * B * N, B * N
  b = Buffers(dev)
  b.add('xn', R, 3 * D, torch.bfloat16)
  b.add('qkv', R, 3 * HH, torch.float32)
  b.add('attn', R, 3 * HH, torch.bfloat16)
  b.add('qc', R, nsrc * HH, torch.float32)
  b.add('attn2', R, 3 * nsrc * HH, torch.bfloat16)
  b.add('x', R, D, torch.float32)
  b.add('hmid', R, 3 * F, torch.bfloat16)

  def wt(n, k):
    return split3_w(torch.randn(n, k, generator=g, device=dev) / math.sqrt(k))
  w_qkv, w_out, w_cq, w_co, w_wi, w_wo = (wt(3 * HH, D), wt(D, HH), wt(nsrc * HH, D), wt(D, nsrc * HH),
                                          wt(2 * F, D), wt(D, F))

  def gv(a, a_off, lda, w, m, n, k, epi, out, ldo, **kw):
    return engine.op_gemm_view(b[a], a_off, lda, w, 0, k, m, n, k, epi, b[out], 0, ldo, **kw)
  for draw in range(2):
    view(b['x'], 0, D, R, D).copy_(torch.randn(R, D, generator=g, device=dev))
    view(b['xn'], 0, 3 * D, R, 3 * D).copy_(split3(O.layer_norm(torch.randn(R, D, generator=g, device=dev),
                                                                 torch.ones(D, device=dev))))
    view(b['attn'], 0, 3 * HH, R, 3 * HH).copy_(split3(torch.randn(R, HH, generator=g, device=dev)))
    view(b['attn2'], 0, 3 * nsrc * HH, R, 3 * nsrc * HH).copy_(
        split3(torch.randn(R, nsrc * HH, generator=g, device=dev)))
    tag = f'acc B={B} nsrc={nsrc} draw {draw}'
    xn = view(b['xn'], 0, 3 * D, R, 3 * D).clone()
    b.launch(lambda: gv('xn', 0, 3 * D, w_qkv, R, 3 * HH, 3 * D, 'f32', 'qkv', 3 * HH), [('qkv', 0, 3 * HH, R, 3 * HH)])
    check_f32_gemm(view(b['qkv'], 0, 3 * HH, R, 3 * HH), xn, w_qkv, 3 * D, None, 'split precision', f'{tag}: qkv')
    x0 = view(b['x'], 0, D, R, D).double().clone()
    at = view(b['attn'], 0, 3 * HH, R, 3 * HH).clone()
    b.launch(lambda: gv('attn', 0, 3 * HH, w_out, R, D, 3 * HH, 'resid_f32', 'x', D, resid=b['x']),
             [('x', 0, D, R, D)])
    check_f32_gemm(view(b['x'], 0, D, R, D), at, w_out, 3 * HH, x0, 'split precision', f'{tag}: self_out')
    b.launch(lambda: gv('xn', 0, 3 * D, w_cq, Rc, nsrc * HH, 3 * D, 'f32', 'qc', nsrc * HH),
             [('qc', 0, nsrc * HH, Rc, nsrc * HH)])
    check_f32_gemm(view(b['qc'], 0, nsrc * HH, Rc, nsrc * HH), xn[:Rc], w_cq, 3 * D, None, 'split precision',
                   f'{tag}: cross_q')
    x1 = view(b['x'], 0, D, R, D).double().clone()
    a2 = view(b['attn2'], 0, 3 * nsrc * HH, Rc, 3 * nsrc * HH).clone()
    b.launch(lambda: gv('attn2', 0, 3 * nsrc * HH, w_co, Rc, D, 3 * nsrc * HH, 'resid_f32', 'x', D, resid=b['x']),
             [('x', 0, D, Rc, D)])
    check_f32_gemm(view(b['x'], 0, D, Rc, D), a2, w_co, 3 * nsrc * HH, x1[:Rc], 'split precision',
                   f'{tag}: cross_out')
    b.launch(lambda: gv('xn', 0, 3 * D, w_wi, R, 2 * F, 3 * D, 'gated_gelu_split3', 'hmid', 3 * F),
             [('hmid', 0, 3 * F, R, 3 * F)])
    acc = xn.double() @ w_wi.double().T
    e = acc_err(3 * D, xn.double().abs() @ w_wi.double().abs().T) + U * acc.abs()
    (r, gg), (er, eg) = gated_split(acc), gated_split(e)
    h = gelu64(r) * gg
    eh = 1.13 * er * gg.abs() + gelu64(r).abs() * eg + 8 * U * (r * gg).abs()   # exact tanhf: a few ulp
    hm = view(b['hmid'], 0, 3 * F, R, 3 * F)
    hi, lo, hi2 = hm[:, :F], hm[:, F:2 * F], hm[:, 2 * F:]
    assert torch.equal(hi.view(torch.int16), hi2.view(torch.int16)), tag
    # hi + lo keeps ~16 bits: the lo half's own rounding is half a bf16 ulp of |v - hi|
    check(hi.double() + lo.double(), h, eh + half_ulp_bf16((h - hi.double()).abs() + eh) + 1e-30,
          'split precision', f'{tag}: wi split3')
    x2 = view(b['x'], 0, D, R, D).double().clone()
    hmc = hm.clone()
    b.launch(lambda: gv('hmid', 0, 3 * F, w_wo, R, D, 3 * F, 'resid_f32', 'x', D, resid=b['x']), [('x', 0, D, R, D)])
    check_f32_gemm(view(b['x'], 0, D, R, D), hmc, w_wo, 3 * F, x2, 'split precision', f'{tag}: wo')


# ---- load-time conditioning tables -------------------------------------------------------------
def timing_signal(num_steps, d, max_time=2e4):
  """The engine's get_timing_signal_1d per step (diffusion_utils.py:69-97): fp64 values from the
  float32 position the engine forms, and a bound on the engine's float rounding of the argument
  (its exp argument k * incf, expf, and the product: (2 |k inc| + 4) u relative)."""
  half = d // 2
  t = np.arange(1, num_steps + 1, dtype=np.float32) / np.float32(num_steps)
  pos = (t * np.float32(max_time)).astype(np.float64)
  inc = math.log(max_time) / (half - 1.0)
  k = np.arange(half, dtype=np.float64)
  arg = pos[:, None] * np.exp(-k * inc)[None, :]
  sig = np.concatenate([np.sin(arg), np.cos(arg)], 1)
  rel = (2 * k * inc + 4) * U
  err = np.concatenate([rel * arg + U, rel * arg + U], 1)
  return sig, err


def swish64(x):
  return x / (1 + np.exp(-x))


def restate_tables(params, cfg, steps):
  """fp64 restatement of the engine's load-time tables, with the film table's error bound."""
  d, L = cfg.emb_dim, cfg.num_decoder_layers
  P = {k: v.astype(np.float64) for k, v in params.items()}
  sig, e0 = timing_signal(steps, d)
  out = dict()

  def dense(x, ex, w, act):
    y = x @ w
    e = ex @ np.abs(w) + w.shape[0] * U * (np.abs(x) @ np.abs(w))
    if act:
      y = swish64(y)
      e = 1.1 * e + 4 * U * np.abs(y)
    return y, e
  c1, e1 = dense(sig, e0, P['decoder/time_emb_dense0/kernel'], True)
  c2, e2 = dense(c1, e1, P['decoder/time_emb_dense1/kernel'], True)
  film = np.zeros((steps, 2 * L, 2 * d))
  efilm = np.zeros_like(film)
  for l in range(L):
    for f in range(2):
      film[:, 2 * l + f], efilm[:, 2 * l + f] = dense(
          c2, e2, P[f'decoder/layers_{l}/FiLMLayer_{f}/DenseGeneral_0/kernel'], False)
  return film, efilm + U * np.abs(film)


def packed_qkv(params, l):
  p = f'decoder/layers_{l}/self_attention/'
  w = np.concatenate([params[p + n + '/kernel'].T for n in ('query', 'key', 'value')], 0)
  return torch.from_numpy(w).to(torch.bfloat16).double().numpy()


def packed_wi(params, l):
  w0 = params[f'decoder/layers_{l}/mlp/wi_0/kernel']   # [d, F]
  w1 = params[f'decoder/layers_{l}/mlp/wi_1/kernel']
  Fm = w0.shape[1]
  r = np.arange(2 * Fm)
  col = (r >> 6) * 32 + (r & 31)
  w = np.where(((r & 63) < 32)[:, None], w0.T[col], w1.T[col])
  return torch.from_numpy(np.ascontiguousarray(w)).to(torch.bfloat16).double().numpy()


@pytest.mark.parametrize('size', ['tiny', 'base'])
def test_conditioning_tables(cuda_device, size):
  """msd_load_weights' tables (launch_sgemm_f32 with swish, launch_film_gain, launch_film_bias)
  at every step and layer, 13 steps (film_bias handles 8 at a time) and 2 decoder layers:
    film      against the fp64 time MLP and FiLM dense (bound carried from the timing signal's
              float argument and fp32 accumulation over K = d and 4d);
    gain      against gamma (1 + fs) in fp64 from the engine's own film rows (2 roundings);
    bias_*    against fb times the packed bf16 weights in fp64 from the engine's film rows
              (fp32 accumulation over K = d), wi with its 32-column gate interleave."""
  if size == 'tiny':
    t5, T, Nn, Cc = config.t5_tiny(), 128, 128, 128
  else:
    t5, T, Nn, Cc = config.t5_base(), 2048, 256, 256
    t5.num_encoder_layers, t5.num_decoder_layers = 1, 2
  params = weights.synthetic_params(t5, T, Nn, Cc, seed=5)
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = STEPS
  eng = engine.Engine(engine.make_msd_config(t5, diff, T, Nn, Cc, max_batch=1), 0)
  eng.load_weights(params)
  tabs = eng.conditioning_tables()
  eng.close()
  d, L = t5.emb_dim, t5.num_decoder_layers
  film64, efilm = restate_tables(params, t5, STEPS)
  ratio = np.max(np.abs(tabs['film'] - film64) / efilm)
  print(f'[err/bound] conditioning tables: {size} film: {ratio:.3f}')
  assert ratio <= 1.0, ratio
  film = tabs['film'].astype(np.float64)
  for l in range(L):
    for f, ln in ((0, 'pre_self_attention_layer_norm'), (1, 'pre_mlp_layer_norm')):
      gamma = params[f'decoder/layers_{l}/{ln}/scale'].astype(np.float64)
      want = gamma[None, :] * (1 + film[:, 2 * l + f, :d])
      r = np.max(np.abs(tabs['gain'][:, 2 * l + f] - want) / (2 * U * np.abs(want) + 1e-30))
      print(f'[err/bound] conditioning tables: {size} gain l={l} f={f}: {r:.3f}')
      assert r <= 1.0, (l, f, r)
    for name, w, f in (('bias_qkv', packed_qkv(params, l), 0), ('bias_wi', packed_wi(params, l), 1)):
      fb = film[:, 2 * l + f, d:]
      want = fb @ w.T
      bound = d * U * (np.abs(fb) @ np.abs(w).T) + U * np.abs(want) + 1e-30
      r = np.max(np.abs(tabs[name][:, l] - want) / bound)
      print(f'[err/bound] conditioning tables: {size} {name} l={l}: {r:.3f}')
      assert r <= 1.0, (name, l, r)


def test_conditioning_tables_without_deferred_normalisation(cuda_device):
  """The fp32-accurate mode keeps the stand-alone norms: the film table is there, the gain and bias
  tables are refused."""
  t5 = config.t5_tiny()
  diff = config.DiffusionConfig()
  diff.sampler.schedule.num_steps = STEPS
  eng = engine.Engine(engine.make_msd_config(t5, diff, 128, 128, 128, max_batch=1, precision='fp32_accurate'), 0)
  eng.load_weights(weights.synthetic_params(t5, 128, 128, 128, seed=5))
  assert eng.conditioning_tables(deferred=False)['film'].shape == (STEPS, 2 * t5.num_decoder_layers, 2 * t5.emb_dim)
  with pytest.raises(_native.MsdError, match='deferred normalisation is off'):
    eng.conditioning_tables()
  eng.close()


# ---- the hooks' own guard rails --------------------------------------------------------------
def test_views_outside_their_tensors_are_refused_before_launch(cuda_device):
  """A mistaken view is a Python error, never an out-of-bounds access."""
  dev = cuda_device
  M = 256
  a = torch.zeros(M * D, dtype=torch.bfloat16, device=dev)
  w = torch.zeros(2 * F * D, dtype=torch.bfloat16, device=dev)
  x = torch.zeros(M * D, device=dev)
  xn = torch.zeros(M * D, dtype=torch.bfloat16, device=dev)
  out = torch.zeros(M * F, dtype=torch.bfloat16, device=dev)
  ss = torch.zeros(KSS * M, device=dev)
  gt = torch.ones(STEPS * GSTRIDE, device=dev)
  bt = torch.zeros(STEPS * LD * 2 * F, device=dev)
  step = torch.full((1,), STEPS - 1, dtype=torch.int32, device=dev)

  def prep(**kw):
    p = dict(g_lo=(gt, D, GSTRIDE), g_hi=(gt, D, GSTRIDE), split_row=M, a=xn, lda=D, ss=ss, ss_stride=M)
    p.update(kw)
    return p

  def resid_prep(**kw):
    a_ = dict(a=a, a_off=0, lda=D, b=w, b_off=0, ldb=D, m=M, n=D, k=D, epilogue='resid_prep', out=x, out_off=0,
              ldo=D, resid=x, step=step, prep=prep())
    a_.update(kw)
    return engine.op_gemm_view(**a_)

  def gated(**kw):
    rs = dict(ss_lo=ss, parts_lo=1, ss_hi=ss, parts_hi=1, split_row=M, ss_stride=M, inv_d=1.0 / D,
              bias=(bt, F * 2, LD * 2 * F))
    rs.update(kw.pop('rs', {}))
    a_ = dict(a=a, a_off=0, lda=D, b=w, b_off=0, ldb=D, m=M, n=2 * F, k=D, epilogue='gated_gelu', out=out,
              out_off=0, ldo=F, step=step, rs=rs)
    a_.update(kw)
    return engine.op_gemm_view(**a_)

  resid_prep()                                              # the valid launches run
  gated()
  engine.op_prep_rows(x, gt, 0, GSTRIDE, step, M, D, xn, D, ss)
  for call, kw in ((resid_prep, dict(a_off=8)),                         # A rows past the end
                   (resid_prep, dict(m=2 * M)),                         # rows past every buffer
                   (resid_prep, dict(b_off=2 * F * D - D * D + 8)),     # B past the end
                   (resid_prep, dict(out_off=8, resid_off=8)),          # out / resid past the end
                   (resid_prep, dict(prep=prep(g_hi=(gt, 3 * D + 8, GSTRIDE)))),  # gain past its row
                   (resid_prep, dict(prep=prep(ss=ss[:D // 64 * M - 1]))),       # too few ss slots
                   (resid_prep, dict(prep=prep(ss_stride=M - 128))),             # ss rows overlap
                   (resid_prep, dict(prep=None)),                       # epilogue 6 without prep
                   (gated, dict(rs=dict(parts_hi=KSS + 1))),            # row scale reads past ss
                   (gated, dict(rs=dict(bias=(bt, 2 * F + 8, LD * 2 * F)))),     # bias past the table
                   (gated, dict(ldo=F - 8)),                            # out columns past the row
                   (gated, dict(step=torch.full((1,), STEPS, dtype=torch.int32, device=dev)))):  # step row past the end
    with pytest.raises(ValueError):
      call(**kw)
  with pytest.raises(ValueError):   # gains of a step past the table
    engine.op_prep_rows(x, gt, 3 * D + 8, GSTRIDE, step, M, D, xn, D, ss)
  with pytest.raises(ValueError):   # operand rows past a_out
    engine.op_prep_rows(x, gt, 0, GSTRIDE, step, M, D, xn[:-8], D, ss)
