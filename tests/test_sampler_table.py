"""The sampler's per-step table (engine.cu build_step_table, through msd_step_table: no GPU) against
the oracle for every sampler variant.

Grid: ddpm with logvar large / small / medium:{0, 0.3, 1} and ddim; model_output eps / x0 / v;
cosine or linear sampler schedule; cosine, linear-1000 or linear-num_steps train schedule;
num_steps 1, 2, 12 and 1000; plus a linear sampler schedule steep enough to saturate at
logsnr = -20, so that consecutive steps have logsnr_s == logsnr_t (1 - r = 0; the medium logvar
then takes log1mexp(0) = -inf).

Checks:
  * the logsnr columns 6 (t), 7 (s) and 14 (train schedule at t) against O.sampler_logsnr /
    O.train_logsnr in float32.  Both evaluate the same float32 formula with different libm
    implementations (glibc vs numpy), so they agree to a few ulp, except where -2 log(tan(.))
    cancels near logsnr = 0; the distance is measured in ulp of max(|logsnr|, 1).  Largest
    distance measured over the grid (glibc 2.39, numpy 2.3): 2.5; bound MAX_LOGSNR_ULP = 3.
  * every other coefficient in fp64 from the table's own float logsnr columns through the oracle's
    formulas (diffusion_reverse, predict_x0_from_eps / predict_eps_from_x0, the x0 / eps
    coefficients of x0_and_eps_from_model_output, the ddim sqrt(sigmoid(+-ls))).  The bound is the
    running error of the host's float32 evaluation (sampler_reference.table_mirror): every float
    operation rounds within u |r|, every libm call within 2u |r|, input errors propagate through
    the exact derivative bound.  This is where cancellation shows: column 8 of the v model,
    C (1 - D al), loses everything to the subtraction at high logsnr, and its bound says so.
    Largest err / bound over the grid, by column: 0: 0.94, 1: 0.65, 2: 0.72, 3: 0.56, 4: 0.52,
    8: 0.98, 9: 0.52, 10: 0.94, 11: 0.62, 12: 0.98, 13: 0.67.
  * column 5 (is_last) exactly, column 15 zero; a non-finite oracle value (the saturated medium
    case with frac 0 or 1: 0 * -inf) must be the same non-finite value in the table.
"""
import numpy as np
import pytest
import torch

from music_spectrogram_diffusion_b200 import config, engine
from oracle import msd_oracle as O
from tests import sampler_reference as S

LOGVARS = ('large', 'small', 'medium:0', 'medium:0.3', 'medium:1')
SAMPLER_VARIANTS = [('ddpm', lv) for lv in LOGVARS] + [('ddim', 'large')]
LINEAR = (1e-4, 0.02)
STEEP = (0.9, 0.999)             # cumprod(1 - beta) < e^-20 within a few steps: logsnr clips at -20
MAX_LOGSNR_ULP = 3


def make_cfg(steps, sampler, logvar, model_output, sched, train, clip_x0=True):
  """(msd_config, OracleConfig).  sched: 'cosine' | (start, stop); train: 'cosine' | (start, stop,
  num_steps)."""
  d = config.DiffusionConfig()
  d.sampler.name, d.sampler.logvar_type, d.sampler.clip_x0 = sampler, logvar, clip_x0
  d.model_output = model_output
  okw = dict(num_steps=steps, sampler=sampler, logvar_type=logvar, model_output=model_output,
             clip_x0=clip_x0)
  if sched == 'cosine':
    d.sampler.schedule = config.DiffusionSchedule('cosine', num_steps=steps)
  else:
    d.sampler.schedule = config.DiffusionSchedule('linear', sched[0], sched[1], steps)
    okw.update(schedule='linear', schedule_start=sched[0], schedule_stop=sched[1])
  if train != 'cosine':
    d.train_schedule = config.DiffusionSchedule('linear', *train)
    okw.update(train_schedule='linear', train_schedule_start=train[0], train_schedule_stop=train[1],
               train_schedule_num_steps=train[2])
  cfg = engine.make_msd_config(config.t5_tiny(), d, 128, 256, 256, max_batch=1)
  return cfg, O.OracleConfig(**okw)


def ulp_distance(got, want):
  """|got - want| in ulp of max(|want|, 1) (float32)."""
  scale = np.spacing(np.maximum(np.abs(want), np.float32(1)).astype(np.float32)).astype(np.float64)
  return np.abs(got.astype(np.float64) - want.astype(np.float64)) / scale


def oracle_columns(tab, oc):
  """fp64 coefficients through the oracle's own formulas, at the table's float logsnr columns."""
  lt, ls, ltr = (tab[:, k].astype(np.float64) for k in (6, 7, 14))
  n = tab.shape[0]
  one, zero = torch.ones(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
  col = {}
  # predict_x0_from_eps at the sampler's logsnr_t: x0 = c0 (z - eps c1)
  col[0] = O.predict_x0_from_eps(one, zero, lt)
  col[1] = -O.predict_x0_from_eps(zero, one, lt) / col[0]
  if oc.sampler == 'ddpm':
    lv = oc.logvar_type
    if lv.startswith('medium:'):
      # the reference multiplies float32 logvars by the Python frac, i.e. by float32(frac)
      lv = f'medium:{float(np.float32(lv.split(":")[1]))!r}'
    col[2] = O.diffusion_reverse(zero, one, ls, lt, lv)['mean']
    rev = O.diffusion_reverse(one, zero, ls, lt, lv)
    col[3], col[4] = rev['mean'], rev['std']
  else:
    # eval_step's ddim update: sqrt(sigmoid(ls)) x0 + sqrt(sigmoid(-ls)) eps
    lst = torch.from_numpy(ls)
    col[2], col[3], col[4] = torch.sqrt(torch.sigmoid(-lst)), torch.sqrt(torch.sigmoid(lst)), zero
  # eps = p0 z + p1 out, x0 = q0 z + q1 out (linear in z and out)
  x0_z, eps_z = O.x0_and_eps_from_model_output(one, zero, ltr, oc.model_output)
  x0_o, eps_o = O.x0_and_eps_from_model_output(zero, one, ltr, oc.model_output)
  col[8], col[9], col[10], col[11] = eps_z, eps_o, x0_z, x0_o
  # predict_eps_from_x0 at logsnr_t: eps = e1 (z - x0 e2)
  col[12] = O.predict_eps_from_x0(one, zero, lt)
  col[13] = -O.predict_eps_from_x0(zero, one, lt) / col[12]
  return {k: v.expand(n).double() for k, v in col.items()}


def check_table(steps, sampler, logvar, model_output, sched, train, worst):
  cfg, oc = make_cfg(steps, sampler, logvar, model_output, sched, train)
  tab = engine.step_table_for(cfg)
  assert tab.shape == (steps, 16) and tab.dtype == np.float32
  what = f'{sampler}/{logvar}/{model_output}/{sched}/{train}/{steps}'
  f32 = np.float32
  t = (np.arange(steps, dtype=f32) + f32(1)) / f32(steps)
  s = np.arange(steps, dtype=f32) / f32(steps)
  for k, want in ((6, O.sampler_logsnr(t, oc)), (7, O.sampler_logsnr(s, oc)), (14, O.train_logsnr(t, oc))):
    d = ulp_distance(tab[:, k], np.asarray(want, f32)).max()
    worst['logsnr_ulp'] = max(worst.get('logsnr_ulp', 0.0), d)
    assert d <= MAX_LOGSNR_ULP, (what, k, d)
  assert np.array_equal(tab[:, 5], (np.arange(steps) == 0).astype(f32)), what
  assert np.all(tab[:, 15] == 0), what
  want = oracle_columns(tab, oc)
  mirror = S.table_mirror(tab[:, 6], tab[:, 7], tab[:, 14], sampler, logvar, model_output)
  for k in (0, 1, 2, 3, 4, 8, 9, 10, 11, 12, 13):
    got = torch.from_numpy(tab[:, k].astype(np.float64))
    w = want[k]
    fin = torch.isfinite(w)
    # a non-finite oracle value must come out as the same non-finite value
    assert torch.equal(torch.isnan(got), torch.isnan(w)), (what, k)
    assert torch.equal(got[torch.isinf(w)], w[torch.isinf(w)]), (what, k)
    # the mirror evaluates the oracle's formula: the two fp64 values agree far inside the bound
    m = mirror[k]
    assert bool(((m.v[fin] - w[fin]).abs() <= 1e-6 * m.e[fin] + 1e-12 * w[fin].abs()).all()), (what, k)
    bound = m.e[fin] * (1 + 1e-9) + 1e-45
    ratio = ((got[fin] - w[fin]).abs() / bound).max().item() if fin.any() else 0.0
    worst[k] = max(worst.get(k, 0.0), ratio)
    assert ratio <= 1.0, (what, k, ratio)


def report(worst):
  cols = ' '.join(f'{k}:{v:.3f}' for k, v in sorted((k, v) for k, v in worst.items() if isinstance(k, int)))
  print(f'[err/bound] step table columns {cols}; logsnr ulp {worst.get("logsnr_ulp", 0):.2f}')


@pytest.mark.parametrize('steps', [1, 2, 12, 1000])
@pytest.mark.parametrize('sampler,logvar', SAMPLER_VARIANTS)
def test_step_table_matches_oracle(steps, sampler, logvar):
  worst = {}
  for model_output in S.MODEL_OUTPUTS:
    for sched in ('cosine', LINEAR):
      for train in ('cosine', LINEAR + (1000,), LINEAR + (steps,)):
        check_table(steps, sampler, logvar, model_output, sched, train, worst)
  report(worst)


@pytest.mark.filterwarnings('ignore:divide by zero encountered in log')   # the oracle's log(0) -> clip
@pytest.mark.parametrize('steps', [12, 1000])
@pytest.mark.parametrize('logvar', LOGVARS)
def test_step_table_saturated_schedule(steps, logvar):
  """A linear sampler schedule that clips at logsnr = -20: the last steps have ls == lt, r = 1,
  1 - r = 0, sigma 0 (large / small, medium:0.3: exp(-inf)) or NaN (medium:0 / medium:1, whose
  0 * -inf the reference computes too)."""
  cfg, oc = make_cfg(steps, 'ddpm', logvar, 'eps', STEEP, 'cosine')
  tab = engine.step_table_for(cfg)
  flat = tab[:, 6] == tab[:, 7]
  assert flat.sum() >= 2 and np.all(tab[flat, 6] == np.float32(-20)), tab[:, 6:8]
  worst = {}
  for model_output in S.MODEL_OUTPUTS:
    check_table(steps, 'ddpm', logvar, model_output, STEEP, 'cosine', worst)
  frac = logvar.split(':')[1] if ':' in logvar else None
  if frac in ('0', '1'):
    assert np.all(np.isnan(tab[flat, 4]))
  else:
    assert np.all(tab[flat, 4] == 0)
  assert np.all(tab[flat, 3] == 0) and np.all(tab[flat, 2] == 1)
  report(worst)


def test_step_table_refuses_what_create_refuses():
  cfg, _ = make_cfg(4, 'ddpm', 'large', 'eps', 'cosine', 'cosine')
  for field, bad in (('sampler', 2), ('logvar_type', 3), ('model_output', 3), ('head_dim', 32)):
    c = type(cfg).from_buffer_copy(cfg)
    setattr(c, field, bad)
    with pytest.raises(engine._native.MsdError):
      engine.step_table_for(c)
  c = type(cfg).from_buffer_copy(cfg)
  c.logvar_type, c.logvar_frac = 2, 1.5
  with pytest.raises(engine._native.MsdError):
    engine.step_table_for(c)
