"""ctypes binding of libmsd_b200.so (C ABI in include/msd_b200.h) + in-tree build.

The library is the product: there is NO Python/CPU fallback.  `load()` raises if
the shared object has not been built (``python -c "import __graft_entry__ as g;
g.build()"``), and every entry point raises `MsdError` on a non-zero return.
"""

from __future__ import annotations

import ctypes
import os
import subprocess
import sys
from typing import List, Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, 'csrc')
_INCLUDE = os.path.join(os.path.dirname(_HERE), 'include')
LIB_NAME = 'libmsd_b200.so'
LIB_PATH = os.path.join(_HERE, LIB_NAME)
SOURCES = ['gemm_wgmma.cu', 'attention_wgmma.cu', 'attention_f32.cu', 'elementwise.cu',
           'engine.cu', 'audio_mel.cu', 'audio_resample.cu']
HEADERS = ['common.cuh', 'kernels.h', 'wgmma.cuh']
NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo',
    '-std=c++17', '-Xcompiler', '-fPIC',
]


class MsdError(RuntimeError):
  pass


def _nvcc() -> str:
  for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
    if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
      return cand
  return 'nvcc'


def _stale() -> bool:
  if not os.path.exists(LIB_PATH):
    return True
  t = os.path.getmtime(LIB_PATH)
  deps = [os.path.join(_CSRC, f) for f in SOURCES + HEADERS]
  deps.append(os.path.join(_INCLUDE, 'msd_b200.h'))
  return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
  """Compile csrc/*.cu for sm_90a into the in-tree shared library."""
  if not force and not _stale():
    return LIB_PATH
  objdir = os.path.join(_HERE, 'build')
  os.makedirs(objdir, exist_ok=True)
  objs: List[str] = []
  procs = []
  for src in SOURCES:
    obj = os.path.join(objdir, src.replace('.cu', '.o'))
    cmd = [_nvcc()] + NVCC_FLAGS + ['-I', _INCLUDE, '-c', os.path.join(_CSRC, src), '-o', obj]
    if verbose:
      print(' '.join(cmd), file=sys.stderr)
    procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs.append(obj)
  for src, p in procs:
    out, _ = p.communicate()
    if p.returncode != 0:
      raise MsdError(f'nvcc failed on {src}:\n{out.decode()}')
  cmd = [_nvcc(), '-shared', '-o', LIB_PATH] + objs
  r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
  if r.returncode != 0:
    raise MsdError(f'link failed:\n{r.stdout.decode()}')
  return LIB_PATH


class MsdConfig(ctypes.Structure):
  """struct msd_config (include/msd_b200.h)."""
  _fields_ = [
      ('vocab_size', ctypes.c_int32), ('emb_dim', ctypes.c_int32),
      ('num_heads', ctypes.c_int32), ('head_dim', ctypes.c_int32),
      ('num_encoder_layers', ctypes.c_int32), ('num_decoder_layers', ctypes.c_int32),
      ('mlp_dim', ctypes.c_int32), ('inputs_length', ctypes.c_int32),
      ('targets_length', ctypes.c_int32), ('context_length', ctypes.c_int32),
      ('n_dims', ctypes.c_int32), ('num_steps', ctypes.c_int32),
      ('max_batch', ctypes.c_int32), ('sampler', ctypes.c_int32),
      ('logvar_type', ctypes.c_int32), ('clip_x0', ctypes.c_int32),
      ('context_positions', ctypes.c_int32),
      ('max_decoder_noise_time', ctypes.c_float),
      ('eval_condition_weight', ctypes.c_float),
      ('feature_min', ctypes.c_float), ('feature_max', ctypes.c_float),
      ('model_output', ctypes.c_int32), ('sampler_schedule', ctypes.c_int32),
      ('train_schedule', ctypes.c_int32), ('train_num_steps', ctypes.c_int32),
      ('logvar_frac', ctypes.c_float), ('sampler_beta_start', ctypes.c_float),
      ('sampler_beta_stop', ctypes.c_float), ('train_beta_start', ctypes.c_float),
      ('train_beta_stop', ctypes.c_float), ('cross_attend_style', ctypes.c_int32),
      ('rng_kind', ctypes.c_int32), ('precision', ctypes.c_int32),
  ]


class MsdTensor(ctypes.Structure):
  """struct msd_tensor (include/msd_b200.h)."""
  _fields_ = [
      ('name', ctypes.c_char_p), ('data', ctypes.c_void_p),
      ('ndim', ctypes.c_int32), ('shape', ctypes.c_int64 * 4),
  ]


# Every symbol include/msd_b200.h declares: (name, restype, argtypes)
_P = ctypes.c_void_p
_I = ctypes.c_int32
SYMBOLS = [
    ('msd_last_error', ctypes.c_char_p, []),
    ('msd_abi_version', ctypes.c_int, []),
    ('msd_create', ctypes.c_int, [ctypes.POINTER(MsdConfig), ctypes.c_int, ctypes.POINTER(_P)]),
    ('msd_destroy', None, [_P]),
    ('msd_load_weights', ctypes.c_int, [_P, ctypes.POINTER(MsdTensor), _I]),
    ('msd_encode', ctypes.c_int, [_P, _P, _P, _P, _I, _P]),
    ('msd_sample', ctypes.c_int, [_P, _P, _P, ctypes.c_uint64, _P, _P]),
    ('msd_sample_rows', ctypes.c_int, [_P, _P, _P, _P]),
    ('msd_p2p_export', ctypes.c_int, [_P, _P]),
    ('msd_p2p_attach', ctypes.c_int, [_P, _P, _I]),
    ('msd_p2p_detach', ctypes.c_int, [_P]),
    ('msd_decode_eps', ctypes.c_int, [_P, _P, _I, _I, _P, _P]),
    ('msd_get_encodings', ctypes.c_int, [_P, _P, _P]),
    ('msd_get_step_table', ctypes.c_int, [_P, _P]),
    ('msd_step_table', ctypes.c_int, [ctypes.POINTER(MsdConfig), _P]),
    ('msd_profile_step', ctypes.c_int, [_P, _I, _I, _P]),
    ('msd_launch_count', ctypes.c_uint64, []),
    ('msd_op_dense', ctypes.c_int, [_P, _P, _I, _I, _I, _P, _P]),
    ('msd_op_dense_variant', ctypes.c_int, [_P, _P, _I, _I, _I, _P, _I, _I, _P]),
    ('msd_bench_gemm', ctypes.c_int, [_I, _I, _I, _I, _I, _I, _I, ctypes.POINTER(ctypes.c_float)]),
    ('msd_bench_attention', ctypes.c_int, [_I, _I, _I, _I, _I, ctypes.POINTER(ctypes.c_float)]),
    ('msd_op_attention', ctypes.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    ('msd_op_rmsnorm_film', ctypes.c_int, [_P, _P, _P, _I, _I, _P, _P]),
    ('msd_op_jax_normal', ctypes.c_int, [ctypes.c_uint64, _I, ctypes.c_int64, _P, _P]),
    ('msd_op_jax_bits', ctypes.c_int, [ctypes.c_uint64, _I, ctypes.c_int64, _P, _P]),
    ('msd_op_dense_epilogue', ctypes.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _I, _P, _I, _P, _P]),
    ('msd_op_dense_deferred_norm', ctypes.c_int,
     [_P, _P, _P, _I, _I, _I, _P, _P, _I, _P, _P, _I, _P, _I, _I, _P, _P, _P]),
    ('msd_op_attention_f32', ctypes.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    ('msd_op_attention_view', ctypes.c_int,
     [_I, _P, ctypes.c_int64, _I, _P, ctypes.c_int64, _I, _P, ctypes.c_int64, _I, _I, _I, _I, _I, _I, _I,
      _P, _I, _I, _I, _P, ctypes.c_int64, _I, _P, _P, _I, _I, _P]),
    ('msd_op_gemm_view', ctypes.c_int,
     [_P, ctypes.c_int64, _I, _P, ctypes.c_int64, _I, _I, _I, _I, _I, _I, _I,
      _P, ctypes.c_int64, _I, _P, ctypes.c_int64, _P, _I, _P, _I,
      _P, _P, ctypes.c_int64, _P, ctypes.c_int64, _I, _P, _I, _P, _I,
      _P, _I, _P, _I, _I, _I, ctypes.c_float, _P, ctypes.c_int64, ctypes.POINTER(_I), _P]),
    ('msd_op_prep_rows', ctypes.c_int, [_P, _P, ctypes.c_int64, _P, _I, _I, _P, _I, _P, _P]),
    ('msd_get_conditioning_tables', ctypes.c_int, [_P, _P, _P, _P, _P]),
    ('msd_op_sampler_step', ctypes.c_int,
     [_P, _P, _P, _P, _P, _P, _I, _P, ctypes.c_int64, _I, _I, ctypes.c_float, _I, _I, ctypes.c_float,
      ctypes.c_float, ctypes.c_uint64, _I, _P, ctypes.c_int64, _P, ctypes.c_int64, _P, _I, _I, _I,
      ctypes.POINTER(_I), _P]),
    ('msd_op_init_z', ctypes.c_int,
     [_P, _P, _P, ctypes.c_int64, _I, ctypes.c_uint64, _I, _P, ctypes.c_int64, ctypes.c_int64, _P, _P]),
    ('msd_op_scale_split', ctypes.c_int,
     [_P, _P, ctypes.c_int64, _I, ctypes.c_float, ctypes.c_float, _P]),
    ('msd_op_audio_mel', ctypes.c_int, [_P, _I, ctypes.c_int64, _P, _P, _P, _P]),
    ('msd_op_audio_resample', ctypes.c_int,
     [_P, _I, ctypes.c_int64, _I, _I, _P, _I, _I, _P, _I, _P, ctypes.c_int64, _P]),
]
ABI_VERSION = 6  # MSD_B200_ABI_VERSION of include/msd_b200.h this binding was written against

_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
  """dlopen the in-tree library (fails loudly when it is missing)."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise MsdError(
        f'{LIB_PATH} is missing: the CUDA extension has not been built. '
        'Run `python -c "import __graft_entry__ as g; g.build()"`. '
        'There is no CPU fallback.')
  lib = ctypes.CDLL(LIB_PATH)
  for name, restype, argtypes in SYMBOLS:
    fn = getattr(lib, name)  # AttributeError if the symbol is not exported
    fn.restype = restype
    fn.argtypes = argtypes
  got = lib.msd_abi_version()
  if got != ABI_VERSION:
    raise MsdError(f'{LIB_PATH} implements ABI {got}, this binding expects {ABI_VERSION}: the '
                   'shared object is stale, rebuild it (python -c "import __graft_entry__ as g; g.build()")')
  _lib = lib
  return lib


def check(rc: int, what: str) -> None:
  if rc != 0:
    msg = load().msd_last_error()
    raise MsdError(f'{what} failed ({rc}): {msg.decode() if msg else "?"}')
