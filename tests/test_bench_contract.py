"""bench.py contract pieces that run without a GPU: the reference arm's JSON line, the
rank-0-only rule under torchrun, and the algorithmic FLOP model behind `roofline` / `whole_step`
(SURVEY App. C)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from music_spectrogram_diffusion_b200 import config  # noqa: E402


def _run(extra_env=None):
  env = dict(os.environ)
  env.pop('RANK', None)
  env.pop('WORLD_SIZE', None)
  env.update(extra_env or {})
  return subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference',
                         '--model', 'tiny', '--steps', '1', '--warmup', '0', '--diffusion-steps', '4'],
                        env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)


def test_reference_arm_prints_one_contract_line():
  out = _run()
  assert out.returncode == 0, out.stderr[-500:]
  lines = [l for l in out.stdout.splitlines() if l.startswith('{')]
  assert len(lines) == 1
  j = json.loads(lines[0])
  assert j['impl'] == 'reference' and j['metric'] == 'mel-frames/sec' and j['unit'] == 'frames/s'
  assert j['higher_is_better'] is True and j['scaling'] == 'weak' and j['vs_baseline'] is None
  assert j['n_gpus'] == 1 and j['steps'] == 1 and j['warmup'] == 0 and j['value'] > 0
  assert 'workload' in j['config'] and 'model' not in j['config']
  cb = j['cpu_baseline']
  assert cb['kind'] == 'port' and cb['cores'] >= 1 and cb['value'] == j['value'] and cb['sample']
  assert j['e2e'] == {'value': j['value'], 'unit': 'frames/s', 'h2d_bytes_per_step': 0,
                      'd2h_bytes_per_step': 0}


def test_reference_arm_runs_on_rank_zero_only():
  out = _run({'RANK': '1', 'WORLD_SIZE': '2', 'LOCAL_RANK': '1'})
  assert out.returncode == 0 and not [l for l in out.stdout.splitlines() if l.startswith('{')]


def test_reference_arm_refuses_to_dump_outputs(tmp_path):
  out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference',
                        '--model', 'tiny', '--dump-outputs', str(tmp_path / 'd')],
                       cwd=ROOT, capture_output=True, text=True, timeout=300)
  assert out.returncode != 0 and '--dump-outputs' in out.stderr
  assert not (tmp_path / 'd').exists()


@pytest.mark.gpu
def test_dump_outputs_is_float32_and_repeatable(tmp_path):
  """--dump-outputs writes the last timed step's mel frames; same arguments, same bytes."""
  import numpy as np
  got = []
  for name in ('a', 'b'):
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--model', 'tiny',
                          '--segments', '2', '--steps', '2', '--warmup', '1', '--diffusion-steps', '8',
                          '--no-song', '--no-cpu-baseline', '--no-traffic', '--no-timeline',
                          '--dump-outputs', str(tmp_path / name)],
                         cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-800:]
    j = json.loads([l for l in out.stdout.splitlines() if l.startswith('{')][-1])
    assert j['steps'] == 2
    assert sorted(os.listdir(tmp_path / name)) == ['mel.npy']
    got.append(np.load(tmp_path / name / 'mel.npy'))
  assert got[0].dtype == np.float32 and got[0].shape == (2, 128, 128)
  assert np.isfinite(got[0]).all() and np.array_equal(got[0], got[1])


def test_flop_model_matches_the_survey_derivation():
  lengths = dict(config.TASK_FEATURE_LENGTHS_CONTEXT)
  per_step, once = bench.flops_model(config.t5_base(), lengths)
  assert abs(per_step / 1e9 - 120.997) < 0.01          # cond 74.994 + uncond 46.003 GF per segment
  assert abs(once / 1e9 - 613.7) < 0.2                 # encoders + hoisted cross K/V
  assert abs((per_step * 1000 + once) / 256 / 1e9 - 475.04) < 0.05   # GFLOP per mel frame
  assert abs(bench.as_written_flops(config.t5_base(), lengths) / 1e9 - 280.9) < 0.2
  small, _ = bench.flops_model(config.t5_small(), lengths)
  assert abs(small / 1e9 - 29.93) < 0.05
