"""The GEMM's drains read their per-tile constants (bias row, column gains) from shared memory,
staged by asynchronous copies, so no instance issues a read-only-path global load (`LDG...CONSTANT`)
whose latency a store would wait behind; and every instance fits its register budget without
spilling.  Compiled here for sm_90a; needs nvcc and cuobjdump, no GPU."""
import os
import re
import shutil
import subprocess

import pytest

from music_spectrogram_diffusion_b200 import _native

WIDTHS = (64, 96, 128, 192, 256)


def _tool(name):
  cand = os.path.join(os.path.dirname(_native._nvcc()), name)
  return cand if os.path.isabs(cand) and os.path.exists(cand) else shutil.which(name)


@pytest.fixture(scope='module')
def gemm_build(tmp_path_factory):
  nvcc, cuobjdump = _tool('nvcc'), _tool('cuobjdump')
  if nvcc is None or cuobjdump is None:
    pytest.skip('nvcc / cuobjdump not available')
  obj = str(tmp_path_factory.mktemp('gemm_sass') / 'gemm_wgmma.o')
  cmd = [nvcc] + _native.NVCC_FLAGS + ['-Xptxas', '-v', '-I', _native._INCLUDE, '-c',
                                       os.path.join(_native._CSRC, 'gemm_wgmma.cu'), '-o', obj]
  r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True)
  sass = subprocess.run([cuobjdump, '-sass', obj], stdout=subprocess.PIPE, text=True, check=True).stdout
  return r.stdout, sass


def _sass_of(sass, bn):
  m = re.search(r'Function : (\S*gemm_bf16_wgmma_kernelILi%d\S*)\n(.*?)(?=\n\s*Function :|\Z)' % bn,
                sass, re.S)
  assert m, f'no SASS for gemm_bf16_wgmma_kernel<{bn}>'
  return m.group(2)


@pytest.mark.parametrize('bn', WIDTHS)
def test_gemm_drain_issues_no_read_only_global_loads(gemm_build, bn):
  body = _sass_of(gemm_build[1], bn)
  assert 'LDGSTS' in body  # the constants are staged
  ldg_constant = re.findall(r'LDG\S*CONSTANT', body)
  assert not ldg_constant, f'gemm_bf16_wgmma_kernel<{bn}>: {len(ldg_constant)} x {ldg_constant[0]}'


@pytest.mark.parametrize('bn', WIDTHS)
def test_gemm_fits_its_registers_without_spills(gemm_build, bn):
  log = gemm_build[0]
  m = re.search(r"Compiling entry function '\S*gemm_bf16_wgmma_kernelILi%d\S*'.*?"
                r'(\d+) bytes spill stores, (\d+) bytes spill loads\s*\n.*?Used (\d+) registers' % bn,
                log, re.S)
  assert m, f'no ptxas report for gemm_bf16_wgmma_kernel<{bn}>'
  stores, loads, regs = map(int, m.groups())
  assert stores == 0 and loads == 0, f'<{bn}>: {stores} B spill stores, {loads} B spill loads'
  assert regs <= 168, f'<{bn}>: {regs} registers'
