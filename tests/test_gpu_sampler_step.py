"""-m gpu: the sampler kernel (sampler_step_kernel), its initial state (init_z_kernel) and the
encoder's feature front end (scale_split_kernel), one launch at a time, on caller-owned buffers
(msd_op_sampler_step, msd_op_init_z, msd_op_scale_split).

Reference: O.eval_step restated in fp64 for one step (sampler_reference.oracle_step) with the model
output as an input, the same float32 z / model output / noise, and the device table's logsnr columns
6, 7 and 14.  The table is then the only thing kernel and test share; tests/test_sampler_table.py
checks it against the oracle.  The bound is per element: the running error of the kernel's float32
evaluation including the host's evaluation of the coefficients it reads (sampler_reference.
kernel_mirror), i.e. a sum over rounding points of |term| u, written in terms of |z|, |eps| eps_scale
etc. rather than |x0|, so the 22026x cancellation of the first reverse step is counted where it
happens.  FMA contraction only removes roundings; the clip is 1-Lipschitz.  A non-finite reference
value (Inf or NaN in the model output) must come out as the same non-finite value.

Exact checks: z_split == [bf16(z) | bf16(z - bf16(z)) | bf16(z)] of the kernel's own z; mel_out
(sentinel-filled) changes only at step 0, and there it is scale_to_features(z) within its rounding;
nothing past n in z, z_split or mel_out changes.

Generated noise: with z = 0 and an eps-model output of 0, x0 = 0 and the new z is sigma * noise up
to one rounding, so the draw is recovered and compared: Philox with oracle/philox.normal within
MAX_PHILOX_ULP ulp of max(|x|, 1) (sincospif and logf against numpy's float64 sin / cos and float32
log), jax with jax_rng at the tolerance of test_jax_random_stream_on_device_matches_numpy.

The RunArgs path (the step graph's): one launch leaves run.step = s - 1 and run.done = 0; k launches
in one call are bit-identical to k single launches, each of which matches the reference fed the
device's previous z, with a different table row and noise row per step.  At B = 8, N = 256 (256
blocks) and at 8 x 2048 x 128 (2048 blocks, more than one wave).

Measured on an H100 80GB HBM3 at a 700 W power limit, the largest err / bound per group: reverse
steps 0.466, last step 0.650, mel_out 0.694, RunArgs chain 0.249, scale_split 0.478; Philox draws
within 3.54 ulp (step noise), 3.29 (per-row noise), 2.00 / 3.00 (init_z whole-batch / per row).

The guidance-split exchange (xrole != 0) and the L2 prefetch are not exercised here.
"""
import math
import zlib

import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import engine, jax_rng as J
from oracle import msd_oracle as O
from oracle import philox as P
from tests import sampler_reference as S
from tests.test_sampler_table import make_cfg

pytestmark = pytest.mark.gpu

ND = 128
STEPS = 12
TEST_STEPS = (STEPS - 1, STEPS // 2, 1, 0)
SENT = -3.5                      # bf16-exact sentinel
MARGIN = 64
FMIN, FMAX = float(np.float32(math.log(1e-5))), 4.0
MAX_PHILOX_ULP = 4
PASSES = ((1, 1.0), (2, 2.0), (2, 0.5))
VARIANTS = (('ddpm', 'large'), ('ddpm', 'small'), ('ddpm', 'medium:0.3'), ('ddim', 'large'))
WORST = {}


def report(group, ratio):
  WORST[group] = max(WORST.get(group, 0.0), ratio)
  print(f'[err/bound] {group}: {ratio:.3f} (worst so far {WORST[group]:.3f})')


def table(sampler, logvar, model_output, clip_x0=True, steps=STEPS):
  cfg, _ = make_cfg(steps, sampler, logvar, model_output, 'cosine', 'cosine', clip_x0)
  return engine.step_table_for(cfg)


def guarded(n, dtype, dev, fill=SENT):
  return torch.full((n + MARGIN,), fill, dtype=dtype, device=dev)


def same(a, b):
  """Equal, NaN == NaN."""
  return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def check_split(z, zs, n):
  """z_split rows == [bf16(z) | bf16(z - bf16(z)) | bf16(z)] of the kernel's own z."""
  zr = z[:n].view(-1, ND)
  hi = zr.to(torch.bfloat16)
  lo = (zr - hi.float()).to(torch.bfloat16)
  got = zs[:3 * n].view(-1, 3, ND)
  for k, want in ((0, hi), (1, lo), (2, hi)):
    assert same(got[:, k].float(), want.float()), f'z_split slot {k}'
  assert bool((zs[3 * n:] == SENT).all()), 'z_split written past n'


def check_against(got, ref, mirror, group):
  got = got.double().cpu()
  fin = torch.isfinite(ref)
  assert torch.equal(torch.isnan(got), torch.isnan(ref)), \
      f'{group}: NaN at {torch.nonzero(torch.isnan(got) != torch.isnan(ref)).flatten()[:8].tolist()}'
  assert torch.equal(got[torch.isinf(ref)], ref[torch.isinf(ref)]), group
  assert bool(((mirror.v[fin] - ref[fin]).abs() <= 1e-6 * mirror.e[fin] + 1e-12 * ref[fin].abs()).all()), \
      f'{group}: the mirror does not evaluate the oracle formula'
  bound = mirror.e[fin] * (1 + 1e-9) + 1e-40
  err = (got[fin] - ref[fin]).abs()
  ratio = (err / bound).max().item() if fin.any() else 0.0
  report(group, ratio)
  assert ratio <= 1.0, (group, ratio, int((err / bound).argmax()))


def crafted_inputs(n, passes, model_output, tab_row, gen):
  """z and model outputs: normal draws at two scales (1 and 16, half the elements each) plus
  crafted elements in the first row: x0 at exactly / just outside / far outside +-1, zeros, +-Inf,
  and one NaN in each pass's model output."""
  z = torch.randn(n, generator=gen, dtype=torch.float64)
  mo = torch.randn(passes, n, generator=gen, dtype=torch.float64)
  z[n // 2:] *= 16
  mo[:, n // 2:] *= 16
  p0, p1, q0, q1 = (float(tab_row[k]) for k in (8, 9, 10, 11))
  targets = [1.0, -1.0, 1 + 2 ** -20, -1 - 2 ** -20, 1 + 2 ** -10, -1 - 2 ** -10, 40.0, -40.0]
  for j, x0 in enumerate(targets):
    if model_output == 'x0':
      m = x0
    elif model_output == 'eps':
      m = (z[j].item() - x0 / q0) / (-q1 / q0)
    else:
      m = (x0 - q0 * z[j].item()) / q1
    mo[:, j] = m   # both passes alike: the guidance combine leaves it (up to rounding)
  k = len(targets)
  z[k], mo[:, k] = 0.0, 0.0
  z[k + 1] = 0.0
  mo[0, k + 2], mo[0, k + 3] = math.inf, -math.inf
  mo[0, k + 4] = math.nan
  mo[passes - 1, k + 5] = math.nan
  return z.float(), mo.float()


def run_step(eps, z0, tab, dev, step, n, passes, weight, clip_x0, ddim, noise=None, mel=True, **kw):
  z = guarded(n, torch.float32, dev)
  z[:n] = z0.to(dev)
  zs = guarded(3 * n, torch.bfloat16, dev)
  mel_out = guarded(n, torch.float32, dev) if mel else None
  coef = torch.from_numpy(tab).to(dev)
  st = torch.tensor([step], dtype=torch.int32, device=dev)
  engine.op_sampler_step(eps.to(dev).reshape(-1).contiguous(), z, zs, coef, n, passes, weight, clip_x0, ddim,
                         FMIN, FMAX, step=st, noise=noise, mel_out=mel_out, **kw)
  return z, zs, mel_out


@pytest.mark.parametrize('sampler,logvar', VARIANTS)
@pytest.mark.parametrize('clip_x0', [True, False])
@pytest.mark.parametrize('passes,weight', PASSES)
@pytest.mark.parametrize('model_output', S.MODEL_OUTPUTS)
def test_sampler_step_matches_fp64(cuda_device, sampler, logvar, clip_x0, passes, weight, model_output):
  tab = table(sampler, logvar, model_output, clip_x0)
  gen = torch.Generator().manual_seed(zlib.crc32(repr((sampler, logvar, clip_x0, passes, weight, model_output)).encode()))
  for idx, step in enumerate(TEST_STEPS):
    B, N = ((3, 256), (1, 256), (8, 256), (3, 128))[idx]
    n = B * N * ND
    z0, mo = crafted_inputs(n, passes, model_output, tab[step], gen)
    noise = torch.randn(STEPS, n, generator=gen)   # a different row per step
    z, zs, mel = run_step(mo, z0, tab, cuda_device, step, n, passes, weight, clip_x0, sampler == 'ddim',
                          noise=noise.to(cuda_device))
    lt, ls, ltr = (float(tab[step, k]) for k in (6, 7, 14))
    args = (lt, ls, ltr, sampler, logvar, model_output, passes, weight, clip_x0, step == 0)
    nz = None if sampler == 'ddim' or step == 0 else noise[step]
    ref = S.oracle_step(z0, mo, *args, noise=nz)
    mirror = S.kernel_mirror(z0, mo, *args, noise=nz)
    check_against(z[:n], ref, mirror, f'step {"last" if step == 0 else "reverse"}')
    assert bool((z[n:] == SENT).all()), 'z written past n'
    check_split(z, zs, n)
    check_mel(z, mel, n, step)


def check_mel(z, mel, n, step):
  if step != 0:
    assert bool((mel == SENT).all()), f'mel_out written at step {step}'
    return
  assert bool((mel[n:] == SENT).all()), 'mel_out written past n'
  zn = z[:n].double().cpu()
  oc = O.OracleConfig(min_value=FMIN, max_value=FMAX)
  ref = O.scale_to_features(zn, oc)
  span = S.R(FMAX) - FMIN
  mirror = (S.R(zn) + 1.0) * 0.5 * span + FMIN
  check_against(mel[:n], ref, mirror, 'mel_out')


def test_sampler_step_nan_propagates_through_clip(cuda_device):
  """jnp.clip / torch.clamp keep a NaN: a NaN model output must not come out as x0 = -1."""
  tab = table('ddpm', 'large', 'x0')
  n = 1024
  mo = torch.zeros(1, n)
  mo[0, 5] = math.nan
  z, _, _ = run_step(mo, torch.zeros(n), tab, cuda_device, 0, n, 1, 1.0, True, False)
  assert math.isnan(z[5].item()), z[5].item()
  assert bool((z[:n][torch.arange(n, device=cuda_device) != 5] == 0).all())


# ---- generated noise -----------------------------------------------------------------------
def philox_ulp(got, want):
  scale = np.spacing(np.maximum(np.abs(want), np.float32(1)).astype(np.float32)).astype(np.float64)
  return (np.abs(got - want.astype(np.float64)) / scale).max()


def check_draw(kind, got, want, group):
  if kind == 0:
    d = philox_ulp(got, want)
    WORST[group] = max(WORST.get(group, 0.0), d)
    print(f'[ulp] {group}: {d:.2f}')
    assert d <= MAX_PHILOX_ULP, (group, d)
  else:
    np.testing.assert_allclose(got, want, rtol=3e-6, atol=3e-7, err_msg=group)


def keys_for(seed, steps):
  return torch.from_numpy(J.step_keys(seed, steps).reshape(-1).view(np.int32).copy())


@pytest.mark.parametrize('rng_kind', [0, 1])
@pytest.mark.parametrize('per_row', [False, True])
def test_generated_noise_matches_numpy(cuda_device, rng_kind, per_row):
  dev = cuda_device
  tab = table('ddpm', 'large', 'eps')
  B, N = 3, 256
  n_row = N * ND
  n = B * n_row
  seed = (7 << 32) | 12345
  seeds = [seed, 99, (1 << 63) + 5]
  stride = 2 * (STEPS + 1) + 6   # a padded row stride
  row_keys = torch.zeros(B * stride, dtype=torch.int32)
  for b, s in enumerate(seeds):
    row_keys[b * stride:b * stride + 2 * (STEPS + 1)] = keys_for(s, STEPS)
  kw = dict(rng_kind=rng_kind, seed=seed, rng_keys=keys_for(seed, STEPS).to(dev),
            n_row=n_row, row_keys=row_keys.to(dev), row_key_stride=stride,
            row_seeds=torch.tensor([s - (1 << 64) if s >= 1 << 63 else s for s in seeds], dtype=torch.int64,
                                   device=dev))
  for step in (STEPS - 1, 5, 1):
    z = guarded(n, torch.float32, dev, 0.0)
    zs = guarded(3 * n, torch.bfloat16, dev)
    coef = torch.from_numpy(tab).to(dev)
    eps = torch.zeros(n, device=dev)
    out = engine.op_sampler_step(eps, z, zs, coef, n, 1, 1.0, True, False, FMIN, FMAX, run_step=step,
                                 per_row=per_row, **kw)
    assert out == (step - 1, 0), out
    check_split(torch.cat([z[:n], torch.full((MARGIN,), SENT, device=dev)]), zs, n)
    assert bool((z[n:] == 0).all())
    sigma = np.float64(tab[step, 4])
    got = z[:n].double().cpu().numpy() / sigma
    for b in range(B):
      s = seeds[b] if per_row else seed
      lo, cnt = (b * n_row, n_row) if per_row else (0, n)
      if not per_row and b:
        break
      if rng_kind == 0:
        want = P.normal(s, step + 1, cnt)
      else:
        want = J.step_noise(s, step, (cnt,))
      check_draw(rng_kind, got[lo:lo + cnt], want, f'{"philox" if rng_kind == 0 else "jax"} noise'
                 f'{" per row" if per_row else ""}')


# ---- the RunArgs path ----------------------------------------------------------------------
@pytest.mark.parametrize('B,N', [(8, 256), (8, 2048)])
@pytest.mark.parametrize('noise_kind', ['injected', 'philox_rows'])
def test_run_args_steps_chain(cuda_device, B, N, noise_kind):
  dev = cuda_device
  sampler, logvar, model_output = 'ddpm', 'large', 'v'
  tab = table(sampler, logvar, model_output)
  coef = torch.from_numpy(tab).to(dev)
  n = B * N * ND
  gen = torch.Generator().manual_seed(B * N)
  z0 = torch.randn(n, generator=gen)
  mo = torch.randn(2, n, generator=gen)
  eps = mo.reshape(-1).to(dev)
  seeds = list(range(11, 11 + B))
  if noise_kind == 'injected':
    noise = torch.randn(STEPS, n, generator=gen)
    kw = dict(noise=noise.to(dev))
  else:
    noise = None
    kw = dict(per_row=True, n_row=N * ND, row_seeds=torch.tensor(seeds, dtype=torch.int64, device=dev),
              rng_kind=0)
  first, k = 5, 6   # steps 5 .. 0: the last one writes the mel
  # k single launches, each against the reference fed the device's previous z
  z = guarded(n, torch.float32, dev)
  z[:n] = z0.to(dev)
  zs = guarded(3 * n, torch.bfloat16, dev)
  mel = guarded(n, torch.float32, dev)
  for step in range(first, first - k, -1):
    prev = z[:n].cpu()
    out = engine.op_sampler_step(eps, z, zs, coef, n, 2, 2.0, True, False, FMIN, FMAX, run_step=step,
                                 mel_out=mel, **kw)
    assert out == (step - 1, 0), out
    if noise is not None:
      nz = noise[step]
    else:
      nz = torch.from_numpy(np.concatenate([P.normal(s, step + 1, N * ND) for s in seeds]))
    lt, ls, ltr = (float(tab[step, kk]) for kk in (6, 7, 14))
    args = (lt, ls, ltr, sampler, logvar, model_output, 2, 2.0, True, step == 0)
    nz = None if step == 0 else nz
    ref = S.oracle_step(prev, mo, *args, noise=nz)
    mirror = S.kernel_mirror(prev, mo, *args, noise=nz)
    if noise is None and step != 0:
      # the generated draw differs from numpy's by a few ulp: the reference takes the device's
      # draw within that bound as an input error of sigma * noise
      sig = abs(float(tab[step, 4]))
      mirror = S.R(mirror.v, mirror.e + sig * MAX_PHILOX_ULP * 2.0 ** -23 * np.maximum(np.abs(nz.numpy()), 1))
    check_against(z[:n], ref, mirror, 'run chain')
    check_mel(z, mel, n, step)
  single = (z.clone(), zs.clone(), mel.clone())
  # the same k steps as k launches of one call: bit-identical
  z = guarded(n, torch.float32, dev)
  z[:n] = z0.to(dev)
  zs = guarded(3 * n, torch.bfloat16, dev)
  mel = guarded(n, torch.float32, dev)
  out = engine.op_sampler_step(eps, z, zs, coef, n, 2, 2.0, True, False, FMIN, FMAX, run_step=first,
                               launches=k, mel_out=mel, **kw)
  assert out == (first - k, 0), out
  for a, b in zip((z, zs, mel), single):
    assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                       b.view(torch.int16) if b.dtype == torch.bfloat16 else b.view(torch.int32))


# ---- init_z, scale_split, the engine's table -----------------------------------------------
def test_init_z_copy_and_streams(cuda_device):
  dev = cuda_device
  B, N = 3, 256
  n_row = N * ND
  n = B * n_row
  src = torch.randn(n)
  src[:4] = torch.tensor([math.inf, -math.inf, math.nan, 0.0])
  z = guarded(n, torch.float32, dev)
  zs = guarded(3 * n, torch.bfloat16, dev)
  engine.op_init_z(z, zs, n, init_z=src.to(dev))
  assert torch.equal(z[:n].cpu().view(torch.int32), src.view(torch.int32))
  check_split(z, zs, n)
  seed = (3 << 32) | 17
  seeds = [seed, 2024, 5]
  stride = 4
  row_keys = torch.zeros(B * stride, dtype=torch.int32)
  for b, s in enumerate(seeds):
    row_keys[b * stride:b * stride + 2] = keys_for(s, 0)
  row_seeds = torch.tensor(seeds, dtype=torch.int64, device=dev)
  for kind in (0, 1):
    name = 'philox' if kind == 0 else 'jax'
    # whole batch
    engine.op_init_z(z, zs, n, seed=seed, rng_kind=kind, rng_keys=keys_for(seed, 0).to(dev))
    want = P.normal(seed, 0, n) if kind == 0 else J.init_z(seed, (n,))
    check_draw(kind, z[:n].double().cpu().numpy(), want, f'{name} init_z')
    check_split(z, zs, n)
    # per row: row b is the seed's own batch-1 draw
    engine.op_init_z(z, zs, n, rng_kind=kind, rng_keys=row_keys.to(dev), n_row=n_row, row_key_stride=stride,
                     row_seeds=row_seeds)
    check_split(z, zs, n)
    rows = z[:n].clone()
    for b, s in enumerate(seeds):
      want = P.normal(s, 0, n_row) if kind == 0 else J.init_z(s, (n_row,))
      check_draw(kind, rows[b * n_row:(b + 1) * n_row].double().cpu().numpy(), want, f'{name} init_z per row')
      z1 = guarded(n_row, torch.float32, dev)
      zs1 = guarded(3 * n_row, torch.bfloat16, dev)
      engine.op_init_z(z1, zs1, n_row, seed=s, rng_kind=kind, rng_keys=keys_for(s, 0).to(dev))
      assert torch.equal(z1[:n_row], rows[b * n_row:(b + 1) * n_row]), (name, b)


def test_scale_split_matches_fp64(cuda_device):
  rows = 64
  g = torch.Generator().manual_seed(4)
  f = (torch.rand(rows, ND, generator=g) * (FMAX - FMIN + 4) + FMIN - 2).double()
  f32 = np.float32
  special = [FMIN, FMAX, float(np.nextafter(f32(FMIN), f32(-10))), float(np.nextafter(f32(FMIN), f32(10))),
             float(np.nextafter(f32(FMAX), f32(-10))), float(np.nextafter(f32(FMAX), f32(10))),
             -1e30, 1e30, math.inf, -math.inf, math.nan, 0.0]
  f[0, :len(special)] = torch.tensor(special, dtype=torch.float64)
  feat = f.float()
  out = torch.full((rows * 3 * ND + MARGIN,), SENT, dtype=torch.bfloat16, device=cuda_device)
  engine.op_scale_split(feat.to(cuda_device), FMIN, FMAX, out=out)
  assert bool((out[rows * 3 * ND:] == SENT).all())
  sp = out[:rows * 3 * ND].view(rows, 3, ND).float().cpu()
  assert same(sp[:, 0], sp[:, 2])
  got = sp[:, 0].double() + sp[:, 1].double()
  oc = O.OracleConfig(min_value=FMIN, max_value=FMAX)
  ref = O.scale_features(feat.double(), oc, clip=True)
  inv = S.R(1.0) / (S.R(FMAX) - FMIN)
  mirror = (S.clip_to(S.R(feat), FMIN, FMAX) - FMIN) * inv * 2.0 - 1.0
  # the split keeps 16 significant bits: hi + lo is within 2^-17 |hi| <= 2^-16 |v| of the float value
  mirror = S.R(mirror.v, mirror.e + 2.0 ** -16 * (mirror.v.abs() + mirror.e))
  check_against(got, ref, mirror, 'scale_split')
  # hi is bf16 of the float value, lo its remainder: |lo| <= half an ulp of hi
  fin = torch.isfinite(sp[:, 0])
  assert bool((sp[:, 1][fin].abs() <= sp[:, 0][fin].abs() * 2.0 ** -8 + 1e-38).all())


def test_engine_table_equals_step_table_for(cuda_device):
  for sampler, logvar, mo in (('ddpm', 'medium:0.3', 'v'), ('ddim', 'large', 'x0'), ('ddpm', 'large', 'eps')):
    cfg, _ = make_cfg(STEPS, sampler, logvar, mo, (1e-4, 0.02), (1e-4, 0.02, 1000))
    eng = engine.Engine(cfg, 0)
    try:
      assert np.array_equal(eng.step_table().view(np.int32), engine.step_table_for(cfg).view(np.int32))
    finally:
      eng.close()


def test_sampler_step_refuses_bad_arguments(cuda_device):
  dev = cuda_device
  tab = torch.from_numpy(table('ddpm', 'large', 'eps')).to(dev)
  n = 1024
  z, zs, eps = torch.zeros(n, device=dev), torch.zeros(3 * n, dtype=torch.bfloat16, device=dev), \
      torch.zeros(2 * n, device=dev)
  st = torch.tensor([3], dtype=torch.int32, device=dev)
  common = (eps, z, zs, tab, n)
  with pytest.raises(ValueError):
    engine.op_sampler_step(*common, 3, 1.0, True, False, FMIN, FMAX, step=st)          # passes
  with pytest.raises(ValueError):
    engine.op_sampler_step(*common, 1, 1.0, True, False, FMIN, FMAX, run_step=STEPS)   # step
  with pytest.raises(ValueError):
    engine.op_sampler_step(*common, 1, 1.0, True, False, FMIN, FMAX, run_step=2, launches=4)
  with pytest.raises(ValueError):
    engine.op_sampler_step(*common, 1, 1.0, True, False, FMIN, FMAX, step=st, rng_kind=1)   # no keys
  with pytest.raises(ValueError):
    engine.op_sampler_step(*common, 1, 1.0, True, False, FMIN, FMAX, run_step=3, per_row=True, n_row=12,
                           row_seeds=torch.zeros(100, dtype=torch.int64, device=dev))
  lib = engine._native.load()
  run_out = (engine.ctypes.c_int32 * 2)()
  for passes, step, per_row, n_row in ((3, 1, 0, 0), (1, STEPS, 0, 0), (1, 1, 1, 12)):
    rc = lib.msd_op_sampler_step(engine._ptr(eps), engine._ptr(z), engine._ptr(zs), None, None, engine._ptr(tab),
                                 STEPS, None, n, ND, passes, 1.0, 1, 0, FMIN, FMAX, 0, 0, None, n_row, None, 0,
                                 None, step, per_row, 1, run_out, None)
    assert rc == -1, (passes, step, per_row)
  assert z.abs().sum().item() == 0
