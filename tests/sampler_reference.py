"""fp64 running-error restatement of the sampler's float32 arithmetic, shared by
tests/test_sampler_table.py (the host step table) and tests/test_gpu_sampler_step.py (the kernel).

An `R` carries a float32 computation in fp64: `v` is the exact value of the operations applied so
far to the exact inputs, `e` bounds |float32 result - v|.  Each operation adds the errors its inputs
carry, propagated through its exact derivative bound, plus its own rounding at the float32 result:
a basic operation rounds once (<= u |r|, u = 2^-24), a libm call (expf, logf, log1pf, expm1f, sqrtf
counted as basic) is within one ulp (<= 2u |r|).  A fused multiply-add rounds once where a*b + c
rounds twice, so counting a*b + c as two roundings also covers nvcc's FMA contraction.  Non-finite
values carry no bound: the tests compare them exactly.
"""
import math

import numpy as np
import torch

from oracle import msd_oracle as O

U = 2.0 ** -24
F64 = torch.float64


def _t(x):
  return torch.as_tensor(np.asarray(x, dtype=np.float64) if not isinstance(x, torch.Tensor) else x,
                         dtype=F64)


class R:
  def __init__(self, v, e=None):
    self.v = _t(v)
    e = torch.zeros_like(self.v) if e is None else _t(e)
    self.e = torch.where(torch.isfinite(self.v), e, torch.zeros_like(e))

  @staticmethod
  def _round(v, e, k=1.0):
    return R(v, e + k * U * (v.abs() + e))

  def __neg__(self):
    return R(-self.v, self.e)

  def __add__(self, o):
    o = lift(o)
    return R._round(self.v + o.v, self.e + o.e)

  def __sub__(self, o):
    o = lift(o)
    return R._round(self.v - o.v, self.e + o.e)

  def __mul__(self, o):
    o = lift(o)
    return R._round(self.v * o.v, self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e)

  def __truediv__(self, o):
    o = lift(o)
    v = self.v / o.v
    den = o.v.abs() - o.e
    e = torch.where(den > 0, (self.e + v.abs() * o.e) / den.clamp_min(1e-300), torch.full_like(v, math.inf))
    return R._round(v, e)

  __radd__ = __add__
  __rmul__ = __mul__

  def __rsub__(self, o):
    return lift(o) - self

  def __rtruediv__(self, o):
    return lift(o) / self


def lift(x):
  return x if isinstance(x, R) else R(x)


def sqrt(a):
  v = a.v.sqrt()
  return R._round(v, a.e / (v + (a.v - a.e).clamp_min(0).sqrt()).clamp_min(1e-300))


def exp(a):
  v = a.v.exp()
  return R._round(v, v * torch.expm1(a.e), 2)


def expm1(a):
  v = torch.expm1(a.v)
  return R._round(v, (a.v + a.e).exp() * a.e, 2)


def log(a):
  v = a.v.log()
  den = a.v - a.e
  e = torch.where(den > 0, a.e / den.clamp_min(1e-300), torch.full_like(v, math.inf))
  return R._round(v, e, 2)


def log1p(a):
  v = torch.log1p(a.v)
  den = 1 + a.v - a.e
  e = torch.where(den > 0, a.e / den.clamp_min(1e-300), torch.full_like(v, math.inf))
  return R._round(v, e, 2)


def where(c, a, b):
  a, b = lift(a), lift(b)
  c = _t(c).bool() if not isinstance(c, torch.Tensor) else c
  return R(torch.where(c, a.v, b.v), torch.where(c, a.e, b.e))


def clip1(a):
  """fminf(fmaxf(a, -1), 1) with NaN kept (jnp.clip): 1-Lipschitz, so the error passes unchanged;
  an infinite value clips to exactly +-1."""
  v = a.v.clamp(-1.0, 1.0)
  return R(v, torch.where(torch.isinf(a.v), torch.zeros_like(a.e), a.e.clamp_max(2.0)))


def sigmoidf(x):
  return 1.0 / (1.0 + exp(-x))


def log_sigmoidf(x):
  return where(x.v < 0, x - log1p(exp(x)), -log1p(exp(-x)))


# ---- the host table (engine.cu build_step_table) from its float logsnr columns --------------
SAMPLERS = {'ddpm': 0, 'ddim': 1}
MODEL_OUTPUTS = ('eps', 'x0', 'v')


def table_mirror(lt, ls, ltr, sampler, logvar, model_output):
  """Columns 0-4 and 8-13 of build_step_table, as R over the steps, from the float32 logsnr
  columns lt (6), ls (7), ltr (14) taken as exact.  logvar: 'large', 'small' or 'medium:<frac>'."""
  lt, ls, ltr = R(lt), R(ls), R(ltr)
  col = {}
  col[0] = sqrt(1.0 + exp(-lt))
  col[1] = 1.0 / sqrt(1.0 + exp(lt))
  if sampler == 'ddpm':
    alpha_st = sqrt((1.0 + exp(-lt)) / (1.0 + exp(-ls)))
    alpha_s = sqrt(sigmoidf(ls))
    d = lt - ls
    rr = exp(d)
    omr = -expm1(d)
    if logvar == 'large':
      var = omr * sigmoidf(-lt)
    elif logvar == 'small':
      var = omr * sigmoidf(-ls)
    else:
      frac = np.float32(logvar.split(':')[1])
      x = ls - lt
      l1mr = where(x.v > float(np.log(np.float32(2.0))), log1p(-exp(-x)), log(-expm1(-x)))
      min_lv, max_lv = l1mr + log_sigmoidf(-ls), l1mr + log_sigmoidf(-lt)
      var = exp(float(frac) * max_lv + float(np.float32(1.0) - frac) * min_lv)
    col[2], col[3], col[4] = rr * alpha_st, omr * alpha_s, sqrt(var)
  else:
    col[2], col[3], col[4] = sqrt(sigmoidf(-ls)), sqrt(sigmoidf(ls)), R(torch.zeros_like(lt.v))
  A, Bc = sqrt(1.0 + exp(-ltr)), 1.0 / sqrt(1.0 + exp(ltr))
  C, D = sqrt(1.0 + exp(ltr)), 1.0 / sqrt(1.0 + exp(-ltr))
  zero, one = R(torch.zeros_like(lt.v)), R(torch.ones_like(lt.v))
  if model_output == 'eps':
    col[8], col[9], col[10], col[11] = zero, one, A, -A * Bc
  elif model_output == 'x0':
    col[8], col[9], col[10], col[11] = C, -C * D, zero, one
  else:
    al, sg = sqrt(sigmoidf(ltr)), sqrt(sigmoidf(-ltr))
    col[10], col[11] = al, -sg
    col[8], col[9] = C * (1.0 - D * al), C * D * sg
  col[12] = sqrt(1.0 + exp(lt))
  col[13] = 1.0 / sqrt(1.0 + exp(-lt))
  return col


def clip_to(a, lo, hi):
  """fminf(fmaxf(a, lo), hi) with NaN kept; an infinite value clips to exactly lo / hi."""
  v = a.v.clamp(lo, hi)
  return R(v, torch.where(torch.isinf(a.v), torch.zeros_like(a.e), a.e.clamp_max(hi - lo)))


def frac_f32(logvar):
  """logvar with the medium fraction as the float32 the config stores (and the reference's float32
  arithmetic multiplies by)."""
  if logvar.startswith('medium:'):
    return f'medium:{float(np.float32(logvar.split(":")[1]))!r}'
  return logvar


def kernel_mirror(z, mo, lt, ls, ltr, sampler, logvar, model_output, passes, weight, clip_x0,
                  last, noise=None):
  """sampler_step_body (csrc/elementwise.cu) on exact float32 inputs z [n], mo [passes, n] and
  noise [n] (or None), with the step's coefficients built from the float logsnr values lt, ls, ltr
  as the host table builds them: returns R of the new z."""
  c = table_mirror(np.array([lt]), np.array([ls]), np.array([ltr]), sampler, logvar, model_output)
  z = R(z)
  mo = [R(m) for m in mo]
  p0, p1, q0, q1 = c[8], c[9], c[10], c[11]
  eps_model = model_output == 'eps'

  def eps_of(m):
    return m if eps_model else p1 * m + p0 * z
  e = eps_of(mo[0])
  if passes == 2:
    w = np.float32(weight)
    e = float(w) * e + float(np.float32(1) - w) * eps_of(mo[1])
    x0 = c[0] * (z - e * c[1])
  elif model_output == 'x0':
    x0 = mo[0]
  elif eps_model:
    x0 = q0 * (z - mo[0] * (-q1 / q0))
  else:
    x0 = q1 * mo[0] + q0 * z
  if clip_x0:
    x0 = clip1(x0)
    if sampler == 'ddim':
      e = c[12] * (z - x0 * c[13])
  if last:
    return x0
  if sampler == 'ddim':
    return c[3] * x0 + c[2] * e
  zn = c[2] * z + c[3] * x0
  return zn if noise is None else zn + c[4] * R(noise)


def oracle_step(z, mo, lt, ls, ltr, sampler, logvar, model_output, passes, weight, clip_x0, last,
                noise=None):
  """O.eval_step for one step in fp64 with the model output given (mo [passes, n]) and the logsnr
  values lt, ls, ltr (the device table's columns 6, 7, 14)."""
  z = _t(z)
  mo = [_t(m) for m in mo]
  x0, eps = O.x0_and_eps_from_model_output(z, mo[0], ltr, model_output)
  if passes == 2:
    w = float(np.float32(weight))
    _, eu = O.x0_and_eps_from_model_output(z, mo[1], ltr, model_output)
    eps = w * eps + (1.0 - w) * eu
    x0 = O.predict_x0_from_eps(z, eps, lt)
  if clip_x0:
    x0 = torch.clamp(x0, -1.0, 1.0)
    eps = O.predict_eps_from_x0(z, x0, lt)
  if last:
    return x0
  if sampler == 'ddim':
    s = torch.tensor(ls, dtype=F64)
    return torch.sqrt(torch.sigmoid(s)) * x0 + torch.sqrt(torch.sigmoid(-s)) * eps
  d = O.diffusion_reverse(x0, z, ls, lt, frac_f32(logvar))
  return d['mean'] + d['std'] * (0.0 if noise is None else _t(noise))
