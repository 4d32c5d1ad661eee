"""Thin host wrapper over the C ABI: torch tensors are storage only.

`Engine` owns one `msd_ctx` (one GPU).  It mirrors the operator surface the
reference exposes one level below `InferenceModel.predict`:
  encode      <-> module.apply(..., method=module.encode)   models.py:365-371
  decode_eps  <-> module.apply(..., method=module.decode)   models.py:378-386
  sample      <-> diffusion_utils.eval_scan + scale_to_features  models.py:393-395
"""

from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional

import numpy as np
import torch

from music_spectrogram_diffusion_b200 import _native
from music_spectrogram_diffusion_b200.config import DiffusionConfig, T5Config


PRECISIONS = {'bf16': 0, 'fp32_accurate': 1}


def make_msd_config(t5: T5Config, diffusion: DiffusionConfig, inputs_length: int,
                    targets_length: int, context_length: int, max_batch: int,
                    n_dims: int = 128, feature_min: float = math.log(1e-5),
                    feature_max: float = 4.0, rng: str = 'jax',
                    precision: str = 'bf16') -> _native.MsdConfig:
  """Translate the reference's config objects into `struct msd_config`.  rng: 'jax' (the
  threefry stream of jax.random.PRNGKey(seed), as the reference draws its noise) or 'philox'.
  precision: 'bf16' (tensor-core operands in bf16, the fast path) or 'fp32_accurate' (3 x bf16
  split-precision dense layers + fp32 attention: what T5Config.dtype = float32 asks for).
  context_length 0 (or None) selects the no-context model, models.DiffusionModel with
  network.Transformer (gin/models/diffusion/basic)."""
  context_length = int(context_length or 0)
  if rng not in ('jax', 'philox'):
    raise ValueError(f'unknown rng {rng!r}')
  if precision not in PRECISIONS:
    raise ValueError(f'unknown precision {precision!r} (expected one of {sorted(PRECISIONS)})')
  if tuple(t5.mlp_activations) != ('gelu', 'linear'):
    raise NotImplementedError(
        f'mlp_activations={t5.mlp_activations}: only the gated-GELU MLP of the '
        'diffusion configs (gin/models/diffusion/context/t5_base.gin:79) is built')
  styles = {'concat_encodings': 0, 'sum_cross_attends': 1}
  if t5.decoder_cross_attend_style not in styles:
    raise ValueError(f'Unknown decoder_cross_attend_style: {t5.decoder_cross_attend_style}')
  if diffusion.model_output == 'x0_and_eps':
    raise NotImplementedError(
        'model_output="x0_and_eps" needs a 2*n_dims output head; the context network emits n_dims '
        'channels (network.py:452-456), so the reference cannot run it on this path either')
  if diffusion.model_output not in ('eps', 'x0', 'v'):
    raise ValueError('Unknown model_output: %s' % diffusion.model_output)
  sched, tsched = diffusion.sampler.schedule, diffusion.train_schedule
  names = {'cosine': 0, 'linear': 1}
  for sc in (sched, tsched):
    if sc.name not in names:
      raise ValueError('Schedule %s not identified.' % sc.name)
    if sc.name == 'linear' and (sc.start is None or sc.stop is None or not sc.num_steps):
      raise ValueError('linear schedule needs start, stop and num_steps')
  if diffusion.sampler.name not in ('ddpm', 'ddim'):
    raise ValueError('Unknown sampler type: %s' % diffusion.sampler.name)
  sampler = {'ddpm': 0, 'ddim': 1}[diffusion.sampler.name]
  lv = diffusion.sampler.logvar_type
  logvar_frac = 0.0
  if lv.startswith('medium:'):
    logvar, logvar_frac = 2, float(lv.split(':')[1])
    if not 0 <= logvar_frac <= 1:
      raise ValueError(f'logvar_type {lv!r}: frac must be in [0, 1]')
  elif lv in ('large', 'small'):
    logvar = {'large': 0, 'small': 1}[lv]
  else:
    raise ValueError(f'unknown logvar_type {lv!r}')
  ctxpos = {'regular': 0, 'terminal_relative': 1}[t5.context_positions]
  return _native.MsdConfig(
      vocab_size=t5.vocab_size, emb_dim=t5.emb_dim, num_heads=t5.num_heads,
      head_dim=t5.head_dim, num_encoder_layers=t5.num_encoder_layers,
      num_decoder_layers=t5.num_decoder_layers, mlp_dim=t5.mlp_dim,
      inputs_length=inputs_length, targets_length=targets_length,
      context_length=context_length, n_dims=n_dims, num_steps=int(sched.num_steps),
      max_batch=max_batch, sampler=sampler, logvar_type=logvar,
      clip_x0=int(bool(diffusion.sampler.clip_x0)), context_positions=ctxpos,
      max_decoder_noise_time=float(t5.max_decoder_noise_time),
      eval_condition_weight=float(diffusion.classifier_free_guidance.eval_condition_weight),
      feature_min=float(feature_min), feature_max=float(feature_max),
      model_output={'eps': 0, 'x0': 1, 'v': 2}[diffusion.model_output],
      sampler_schedule=names[sched.name], train_schedule=names[tsched.name],
      train_num_steps=int(tsched.num_steps or 0), logvar_frac=logvar_frac,
      sampler_beta_start=float(sched.start or 0.0), sampler_beta_stop=float(sched.stop or 0.0),
      train_beta_start=float(tsched.start or 0.0), train_beta_stop=float(tsched.stop or 0.0),
      cross_attend_style=styles[t5.decoder_cross_attend_style],
      rng_kind={'philox': 0, 'jax': 1}[rng], precision=PRECISIONS[precision])


def _ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
  return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _stream(device: torch.device) -> ctypes.c_void_p:
  return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Engine:
  """One msd_ctx on one GPU."""

  def __init__(self, cfg: _native.MsdConfig, device: int = 0):
    self.lib = _native.load()
    if not torch.cuda.is_available():
      raise _native.MsdError('no CUDA device: the sm_90a library cannot run (no CPU fallback)')
    self.cfg = cfg
    self.device = torch.device('cuda', device)
    torch.cuda.set_device(self.device)
    torch.zeros(1, device=self.device)  # make sure the primary context exists
    handle = ctypes.c_void_p()
    _native.check(self.lib.msd_create(ctypes.byref(cfg), device, ctypes.byref(handle)),
                  'msd_create')
    self._h = handle
    self._batch = 0

  def close(self) -> None:
    if getattr(self, '_h', None):
      self.lib.msd_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  # -- weights ---------------------------------------------------------------
  def load_weights(self, params: Dict[str, np.ndarray]) -> None:
    names = sorted(params)
    arr = (_native.MsdTensor * len(names))()
    keep = []
    for i, k in enumerate(names):
      a = np.ascontiguousarray(params[k], dtype=np.float32)
      keep.append(a)
      arr[i].name = k.encode()
      arr[i].data = a.ctypes.data
      arr[i].ndim = a.ndim
      for j, s in enumerate(a.shape):
        arr[i].shape[j] = s
    _native.check(self.lib.msd_load_weights(self._h, arr, len(names)), 'msd_load_weights')

  # -- operator surface --------------------------------------------------------
  def encode(self, tokens: torch.Tensor, ctx_features: Optional[torch.Tensor],
             ctx_mask: Optional[torch.Tensor]) -> None:
    """ctx_features / ctx_mask: the context, or None for both with a no-context model
    (context_length 0)."""
    b = tokens.shape[0]
    assert tokens.dtype == torch.int32 and tokens.is_cuda and tokens.is_contiguous()
    assert tokens.shape == (b, self.cfg.inputs_length), tokens.shape
    if self.cfg.context_length == 0:
      if ctx_features is not None or ctx_mask is not None:
        raise ValueError('this model has no context (context_length 0): pass None for '
                         'ctx_features and ctx_mask')
    else:
      if ctx_features is None or ctx_mask is None:
        raise ValueError(f'this model takes a context of {self.cfg.context_length} frames: '
                         'ctx_features and ctx_mask are required')
      assert ctx_features.dtype == torch.float32 and ctx_features.is_contiguous()
      assert ctx_mask.dtype == torch.int32 and ctx_mask.is_contiguous()
      assert ctx_features.shape == (b, self.cfg.context_length, self.cfg.n_dims)
      assert ctx_mask.shape == (b, self.cfg.context_length)
    _native.check(self.lib.msd_encode(self._h, _ptr(tokens), _ptr(ctx_features), _ptr(ctx_mask),
                                      b, _stream(self.device)), 'msd_encode')
    self._batch = b

  def encodings(self) -> torch.Tensor:
    out = torch.empty(self._batch, self.cfg.inputs_length + self.cfg.context_length,
                      self.cfg.emb_dim, dtype=torch.float32, device=self.device)
    _native.check(self.lib.msd_get_encodings(self._h, _ptr(out), _stream(self.device)),
                  'msd_get_encodings')
    return out

  def decode_eps(self, z: torch.Tensor, step_i: int, conditioned: bool) -> torch.Tensor:
    assert z.dtype == torch.float32 and z.is_cuda and z.is_contiguous()
    assert z.shape == (self._batch, self.cfg.targets_length, self.cfg.n_dims)
    out = torch.empty_like(z)
    _native.check(self.lib.msd_decode_eps(self._h, _ptr(z), step_i, int(conditioned), _ptr(out),
                                          _stream(self.device)), 'msd_decode_eps')
    return out

  def sample(self, init_z: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None,
             seed: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    shape = (self._batch, self.cfg.targets_length, self.cfg.n_dims)
    if init_z is not None:
      assert init_z.dtype == torch.float32 and init_z.is_contiguous() and init_z.shape == shape
    if noise is not None:
      assert noise.dtype == torch.float32 and noise.is_contiguous()
      assert noise.shape == (self.cfg.num_steps,) + shape, noise.shape
    if out is None:
      out = torch.empty(shape, dtype=torch.float32, device=self.device)
    _native.check(self.lib.msd_sample(self._h, _ptr(init_z), _ptr(noise), seed, _ptr(out),
                                      _stream(self.device)), 'msd_sample')
    return out

  def sample_rows(self, seeds, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Like sample(seed=...), but row b of the encoded batch draws its noise from seeds[b] alone:
    row b comes out as sample(seed=seeds[b]) would draw it at batch 1 (msd_sample_rows)."""
    seeds = [int(s) for s in seeds]
    if len(seeds) != self._batch:
      raise ValueError(f'{len(seeds)} seeds for an encoded batch of {self._batch}')
    shape = (self._batch, self.cfg.targets_length, self.cfg.n_dims)
    if out is None:
      out = torch.empty(shape, dtype=torch.float32, device=self.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape == shape
    arr = (ctypes.c_uint64 * len(seeds))(*[s & 0xFFFFFFFFFFFFFFFF for s in seeds])
    _native.check(self.lib.msd_sample_rows(self._h, arr, _ptr(out), _stream(self.device)),
                  'msd_sample_rows')
    return out

  # -- guidance split over two GPUs (msd_p2p_*, include/msd_b200.h) --------------------------
  def p2p_export(self) -> bytes:
    buf = ctypes.create_string_buffer(64)
    _native.check(self.lib.msd_p2p_export(self._h, buf), 'msd_p2p_export')
    return buf.raw

  def p2p_attach(self, peer_handle: bytes, role: str) -> None:
    """role: 'cond' (this GPU runs the conditional pass) or 'uncond'."""
    if len(peer_handle) != 64:
      raise ValueError('peer handle must be the 64 bytes msd_p2p_export returned on the other rank')
    self._peer_handle = ctypes.create_string_buffer(peer_handle, 64)
    _native.check(self.lib.msd_p2p_attach(self._h, self._peer_handle,
                                          {'cond': 1, 'uncond': 2}[role]), 'msd_p2p_attach')

  def p2p_detach(self) -> None:
    _native.check(self.lib.msd_p2p_detach(self._h), 'msd_p2p_detach')

  KERNEL_CLASSES = ('gemm', 'attention', 'rmsnorm_film', 'sampler', 'other')

  def profile_step(self, step_i: int = 500, reps: int = 3) -> Dict[str, Dict[str, float]]:
    """Per-kernel-class CUDA-event timing of one diffusion step (uncaptured)."""
    out = np.zeros((5, 4), dtype=np.float64)
    _native.check(self.lib.msd_profile_step(self._h, step_i, reps, out.ctypes.data),
                  'msd_profile_step')
    return {name: dict(ms=float(out[i, 0]), launches=float(out[i, 1]), flops=float(out[i, 2]),
                       bytes=float(out[i, 3]))
            for i, name in enumerate(self.KERNEL_CLASSES)}

  def step_table(self) -> np.ndarray:
    tab = np.zeros((self.cfg.num_steps, 16), dtype=np.float32)
    _native.check(self.lib.msd_get_step_table(self._h, tab.ctypes.data), 'msd_get_step_table')
    return tab

  def conditioning_tables(self, deferred: bool = True) -> Dict[str, np.ndarray]:
    """The load-time conditioning tables (msd_get_conditioning_tables), float32:
    film [steps, 2 L, 2 d] and, with deferred=True (bf16 mode), gain [steps, 2 L, d],
    bias_qkv [steps, L, 3 hh] and bias_wi [steps, L, 2 F]."""
    c = self.cfg
    s, L, d, hh = c.num_steps, c.num_decoder_layers, c.emb_dim, c.num_heads * c.head_dim
    shapes = dict(film=(s, 2 * L, 2 * d))
    if deferred:
      shapes.update(gain=(s, 2 * L, d), bias_qkv=(s, L, 3 * hh), bias_wi=(s, L, 2 * c.mlp_dim))
    out = {k: np.zeros(v, dtype=np.float32) for k, v in shapes.items()}
    ptrs = [ctypes.c_void_p(out[k].ctypes.data) if k in out else None
            for k in ('film', 'gain', 'bias_qkv', 'bias_wi')]
    _native.check(self.lib.msd_get_conditioning_tables(self._h, *ptrs), 'msd_get_conditioning_tables')
    return out


def launch_count() -> int:
  return int(_native.load().msd_launch_count())


# ---- operator-level hooks (unit parity with msd/layers.py) --------------------
def op_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
                 key_mask: Optional[torch.Tensor], heads: int) -> torch.Tensor:
  lib = _native.load()
  nb, lq, _ = q.shape
  lk = k.shape[1]
  out = torch.empty_like(q)
  _native.check(lib.msd_op_attention(_ptr(q.contiguous()), _ptr(k.contiguous()),
                                     _ptr(v.contiguous()), _ptr(key_mask), nb, heads, lq, lk,
                                     _ptr(out), _stream(q.device)), 'msd_op_attention')
  return out


def op_rmsnorm_film(x: torch.Tensor, gamma: torch.Tensor,
                    film: Optional[torch.Tensor]) -> torch.Tensor:
  """LayerNorm (layers.py:632-649), then FiLM with the scale | bias vector film [2 d] (None = none):
  f32 (bf16-rounded) [rows, d], through op_rmsnorm_view."""
  rows, d = x.shape
  out = torch.empty(rows, d, dtype=torch.bfloat16, device=x.device)
  step = None if film is None else torch.zeros(1, dtype=torch.int32, device=x.device)
  op_rmsnorm_view(x.contiguous(), gamma.contiguous(), out, 0, d,
                  film=None if film is None else film.contiguous(), step=step)
  return out.float()


EPILOGUES = {'bf16': 0, 'f32': 1, 'resid_f32': 2, 'gated_gelu': 3, 'pos_f32': 4, 'gated_gelu_split3': 5}


def op_dense_epilogue(a: torch.Tensor, w: torch.Tensor, epilogue: str, block_n: int = 0,
                      w1: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None,
                      pos: Optional[torch.Tensor] = None, pos_shift: Optional[torch.Tensor] = None,
                      dup_rows: int = 0) -> torch.Tensor:
  """The GEMM with one of its fused epilogues (kernels.h GemmEpilogue); see msd_op_dense_epilogue."""
  lib = _native.load()
  m, k = a.shape
  n = w.shape[1]
  out = torch.empty(m + dup_rows, n, dtype=torch.float32, device=a.device)
  pos_rows = 0 if pos is None else pos.shape[0]
  keep = [t.contiguous() if t is not None else None for t in (a, w, w1, resid, pos, pos_shift)]
  _native.check(lib.msd_op_dense_epilogue(_ptr(keep[0]), _ptr(keep[1]), _ptr(keep[2]), m, n, k,
                                          EPILOGUES[epilogue], block_n, _ptr(keep[3]), _ptr(keep[4]),
                                          pos_rows, _ptr(keep[5]), dup_rows, _ptr(out),
                                          _stream(a.device)), 'msd_op_dense_epilogue')
  return out


def op_dense_deferred_norm(a: torch.Tensor, w_out: torch.Tensor, x: torch.Tensor, g_lo: torch.Tensor,
                           g_hi: torch.Tensor, split_row: int, w2: torch.Tensor,
                           w2b: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
                           block_n1: int = 0, block_n2: int = 0):
  """Residual projection with the deferred-normalisation epilogue + the projection consuming it
  (msd_op_dense_deferred_norm): returns (x_out [M, d], y [M, N2])."""
  lib = _native.load()
  m, k = a.shape
  d = w_out.shape[1]
  n2 = w2.shape[1]
  x_out = torch.empty(m, d, dtype=torch.float32, device=a.device)
  y = torch.empty(m, n2, dtype=torch.float32, device=a.device)
  keep = [t.contiguous() if t is not None else None for t in (a, w_out, x, g_lo, g_hi, w2, w2b, bias)]
  _native.check(lib.msd_op_dense_deferred_norm(_ptr(keep[0]), _ptr(keep[1]), _ptr(keep[2]), m, d, k,
                                               _ptr(keep[3]), _ptr(keep[4]), split_row, _ptr(keep[5]),
                                               _ptr(keep[6]), n2, _ptr(keep[7]), block_n1, block_n2,
                                               _ptr(x_out), _ptr(y), _stream(a.device)),
                'msd_op_dense_deferred_norm')
  return x_out, y


def op_attention_f32(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
                     key_mask: Optional[torch.Tensor], heads: int) -> torch.Tensor:
  lib = _native.load()
  nb, lq, _ = q.shape
  lk = k.shape[1]
  out = torch.empty_like(q)
  _native.check(lib.msd_op_attention_f32(_ptr(q.contiguous()), _ptr(k.contiguous()),
                                         _ptr(v.contiguous()), _ptr(key_mask), nb, heads, lq, lk,
                                         _ptr(out), _stream(q.device)), 'msd_op_attention_f32')
  return out


ATTN_MAX_SPLITS = 12   # split-KV workspace of msd_op_attention_view, in splits


def attention_workspace(nb: int, lq: int, heads: int, device: torch.device):
  """(part_o, part_ml) f32 buffers for op_attention_view with up to ATTN_MAX_SPLITS splits."""
  rows = nb * lq * heads * ATTN_MAX_SPLITS
  return (torch.empty(rows * 64, dtype=torch.float32, device=device),
          torch.empty(rows * 2, dtype=torch.float32, device=device))


def _check_view(name: str, t: torch.Tensor, off: int, ld: int, rows: int, cols: int, elem: int) -> None:
  """The view (rows x cols from element `off`, row stride `ld`) lies inside t, no row wraps."""
  if not t.is_contiguous():
    raise ValueError(f'{name}: tensor must be contiguous')
  align = 16 // elem
  if off < 0 or ld <= 0 or off % align or ld % align:
    raise ValueError(f'{name}: offset {off} / leading dimension {ld} must be non-negative multiples '
                     f'of {align} elements')
  row0, col0 = divmod(off, ld)
  if col0 + cols > ld:
    raise ValueError(f'{name}: columns [{col0}, {col0 + cols}) exceed the leading dimension {ld}')
  if (row0 + rows) * ld > t.numel():
    raise ValueError(f'{name}: rows [{row0}, {row0 + rows}) of {ld} elements exceed the '
                     f'{t.numel()} elements of the tensor')


def op_attention_view(q: torch.Tensor, q_off: int, ldq: int, k: torch.Tensor, k_off: int, ldk: int,
                      v: torch.Tensor, v_off: int, ldv: int, nb: int, heads: int, lq: int, lk: int,
                      out: torch.Tensor, o_col: int, o_ld: int, part_o: torch.Tensor,
                      part_ml: torch.Tensor, key_mask: Optional[torch.Tensor] = None,
                      mask_word0: int = 0, kv_batch_rows: int = 0, kv_row0: int = 0,
                      kv_static: int = 0, splits: int = 0, tail: int = 0,
                      precision: str = 'bf16') -> None:
  """The attention kernel over views of caller-owned device buffers (msd_op_attention_view):
  q / k / v are bf16 (precision 'bf16') or f32 ('fp32_accurate') tensors addressed by element
  offset + leading dimension, out is bf16 and is written in place (fp32_accurate: [hi | lo | hi]
  with o_ld the width of one third), key_mask int32 [nb, mask_len].  Every view is checked to lie
  inside its tensor before the library is called."""
  if precision not in PRECISIONS:
    raise ValueError(f'unknown precision {precision!r}')
  acc = PRECISIONS[precision]
  dt, elem = (torch.float32, 4) if acc else (torch.bfloat16, 2)
  width = heads * 64
  if nb <= 0 or heads <= 0 or lq <= 0 or lk <= 0 or lq % 128 or lk % 128:
    raise ValueError(f'nb={nb}, heads={heads}: Lq={lq} and Lk={lk} must be positive multiples of 128')
  for name, t in (('q', q), ('k', k), ('v', v)):
    if t.dtype != dt or not t.is_cuda:
      raise ValueError(f'{name}: expected a {dt} CUDA tensor, got {t.dtype} on {t.device}')
  if out.dtype != torch.bfloat16 or not out.is_cuda:
    raise ValueError('out: expected a bf16 CUDA tensor')
  kbr = kv_batch_rows if kv_batch_rows > 0 else lk
  if kv_batch_rows < 0 or kv_row0 < 0 or kv_row0 + lk > kbr:
    raise ValueError(f'key rows [{kv_row0}, {kv_row0 + lk}) exceed the {kbr} rows per batch')
  _check_view('q', q, q_off, ldq, nb * lq, width, elem)
  _check_view('k', k, k_off, ldk, nb * kbr, width, elem)
  _check_view('v', v, v_off, ldv, nb * kbr, width, elem)
  if acc:
    if o_col + width > o_ld:
      raise ValueError(f'out: columns [{o_col}, {o_col + width}) exceed the third of width {o_ld}')
    _check_view('out', out, o_col, 3 * o_ld, nb * lq, 2 * o_ld + width, 2)
  else:
    _check_view('out', out, o_col, o_ld, nb * lq, width, 2)
  mask_len = 0
  if key_mask is not None:
    if key_mask.dtype != torch.int32 or not key_mask.is_contiguous() or key_mask.dim() != 2 \
        or key_mask.shape[0] != nb:
      raise ValueError(f'key_mask: expected contiguous int32 [{nb}, mask_len]')
    mask_len = key_mask.shape[1]
    if mask_len % 128 or mask_word0 < 0 or mask_word0 % 4 or mask_word0 + lk // 32 > mask_len // 32:
      raise ValueError(f'key_mask: words [{mask_word0}, {mask_word0 + lk // 32}) outside rows of '
                       f'{mask_len // 32} words (mask_len and the start word: multiples of 128 / 4)')
  elif mask_word0:
    raise ValueError('mask_word0 without a key_mask')
  need = nb * lq * heads * ATTN_MAX_SPLITS
  for name, t, n in (('part_o', part_o, need * 64), ('part_ml', part_ml, need * 2)):
    if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() < n:
      raise ValueError(f'{name}: expected a contiguous f32 tensor of at least {n} elements')
  if not 0 <= splits <= ATTN_MAX_SPLITS or tail < 0 or (acc and tail):
    raise ValueError(f'splits={splits} must be in [0, {ATTN_MAX_SPLITS}]; tail={tail} >= 0 (bf16 only)')
  args = _native.MsdAttentionViewArgs(
      precision=acc, q=_ptr(q), q_off=q_off, ldq=ldq, k=_ptr(k), k_off=k_off, ldk=ldk, v=_ptr(v), v_off=v_off,
      ldv=ldv, nb=nb, heads=heads, Lq=lq, Lk=lk, kv_batch_rows=kv_batch_rows, kv_row0=kv_row0,
      key_mask=_ptr(key_mask), mask_len=mask_len, mask_word0=mask_word0, kv_static=int(kv_static),
      out=_ptr(out), o_col=o_col, o_ld=o_ld, part_o=_ptr(part_o), part_ml=_ptr(part_ml), splits=splits,
      tail=tail)
  _native.check(_native.load().msd_op_attention_view(ctypes.byref(args), _stream(q.device)),
                'msd_op_attention_view')


GEMM_EPILOGUES = dict(EPILOGUES, resid_prep=6)
_F32_OUT = ('f32', 'resid_f32', 'pos_f32', 'resid_prep')


def _check_dev(name: str, t: torch.Tensor, dtype: torch.dtype, device: torch.device) -> None:
  if t.dtype != dtype or t.device != device:
    raise ValueError(f'{name}: expected a {dtype} tensor on {device}, got {t.dtype} on {t.device}')


def _check_vector(name: str, t: torch.Tensor, off: int, n: int, device: torch.device) -> None:
  """n float32 values of t from element `off`."""
  _check_dev(name, t, torch.float32, device)
  _check_view(name, t, off, off + n, 1, n, 4)


def _step_value(step: Optional[torch.Tensor], device: torch.device) -> int:
  """The device step index a launch will read (0 without one)."""
  if step is None:
    return 0
  _check_dev('step', step, torch.int32, device)
  if step.numel() != 1:
    raise ValueError('step: expected one int32 element')
  s = int(step.item())
  if s < 0:
    raise ValueError(f'step: {s} is negative')
  return s


def op_gemm_view(a: torch.Tensor, a_off: int, lda: int, b: torch.Tensor, b_off: int, ldb: int,
                 m: int, n: int, k: int, epilogue: str, out: torch.Tensor, out_off: int, ldo: int,
                 block_n: int = 0, resid: Optional[torch.Tensor] = None,
                 resid_off: int = 0, pos: Optional[torch.Tensor] = None,
                 pos_shift: Optional[torch.Tensor] = None, dup_rows: int = 0,
                 step: Optional[torch.Tensor] = None, prep: Optional[dict] = None,
                 rs: Optional[dict] = None) -> int:
  """The GEMM over views of caller-owned device buffers, with every argument the engine's decoder
  sets (msd_op_gemm_view); returns the tile width that ran.  a / b: bf16, out = a[m, k] b[n, k]^T
  through `epilogue` (GEMM_EPILOGUES) into out (f32 or bf16 by epilogue) at out_off / ldo.
  prep (epilogue 'resid_prep'): dict(g_lo=(t, off, step_stride), g_hi=(t, off, step_stride),
  split_row, a, lda, ss, ss_stride).  rs (row scale on 'bf16' / 'gated_gelu'): dict(ss_lo, parts_lo,
  ss_hi, parts_hi, split_row, ss_stride, inv_d, bias=(t, off, step_stride) or None).
  Every view is checked to lie inside its tensor before the library is called; step-indexed
  vectors at the step `step` holds, prep.ss for the narrowest tile the launch may run (N / 64
  partial sums, or N / block_n)."""
  if epilogue not in GEMM_EPILOGUES:
    raise ValueError(f'unknown epilogue {epilogue!r} (expected one of {sorted(GEMM_EPILOGUES)})')
  dev = a.device
  if m <= 0 or n <= 0 or k <= 0 or m % 128 or k % 64:
    raise ValueError(f'm={m}, n={n}, k={k}: m must be a positive multiple of 128, k of 64')
  for name, t in (('a', a), ('b', b)):
    _check_dev(name, t, torch.bfloat16, dev)
  _check_view('a', a, a_off, lda, m, k, 2)
  _check_view('b', b, b_off, ldb, n, k, 2)
  f32_out = epilogue in _F32_OUT
  _check_dev('out', out, torch.float32 if f32_out else torch.bfloat16, dev)
  cols = {'gated_gelu': n // 2, 'gated_gelu_split3': 3 * (n // 2)}.get(epilogue, n)
  _check_view('out', out, out_off, ldo, m + (dup_rows if epilogue == 'pos_f32' else 0), cols,
              4 if f32_out else 2)
  if resid is not None:
    _check_dev('resid', resid, torch.float32, dev)
    _check_view('resid', resid, resid_off, ldo, m, n, 4)
  elif epilogue in ('resid_f32', 'resid_prep'):
    raise ValueError(f'epilogue {epilogue!r} needs resid')
  pos_rows = 0
  if epilogue == 'pos_f32':
    if pos is None:
      raise ValueError("epilogue 'pos_f32' needs pos")
    _check_dev('pos', pos, torch.float32, dev)
    pos_rows = pos.shape[0]
    _check_view('pos', pos, 0, n, pos_rows, n, 4)
    if pos_shift is not None:
      _check_dev('pos_shift', pos_shift, torch.int32, dev)
      if pos_shift.numel() < -(-m // pos_rows):
        raise ValueError(f'pos_shift: {pos_shift.numel()} entries for {-(-m // pos_rows)} sequences')
  s = _step_value(step, dev)
  pa = _native.MsdGemmPrep()
  if prep is not None:
    if epilogue != 'resid_prep':
      raise ValueError('prep goes with the resid_prep epilogue')
    gains = {}
    for key in ('g_lo', 'g_hi'):
      t, off, stride = prep[key]
      if stride and step is None:
        raise ValueError(f'prep.{key}: a step stride needs the device step')
      _check_vector(f'prep.{key}', t, off + s * stride, n, dev)
      gains[key] = ctypes.c_void_p(t.data_ptr() + 4 * off)
      gains[key + '_step_stride'] = stride
    _check_dev('prep.a', prep['a'], torch.bfloat16, dev)
    _check_view('prep.a', prep['a'], 0, prep['lda'], m, n, 2)
    _check_dev('prep.ss', prep['ss'], torch.float32, dev)
    if prep['ss_stride'] < m:
      raise ValueError(f'prep.ss_stride {prep["ss_stride"]} < m = {m}')
    _check_view('prep.ss', prep['ss'], 0, prep['ss_stride'], n // (block_n or 64), m, 4)
    pa = _native.MsdGemmPrep(**gains, split_row=prep['split_row'], a=_ptr(prep['a']), lda=prep['lda'],
                             ss=_ptr(prep['ss']), ss_stride=prep['ss_stride'])
  elif epilogue == 'resid_prep':
    raise ValueError("epilogue 'resid_prep' needs prep")
  ra = _native.MsdGemmRowScale()
  if rs is not None:
    if epilogue not in ('bf16', 'gated_gelu'):
      raise ValueError('the row scale goes with the bf16 and gated_gelu epilogues')
    sums = {}
    for key in ('lo', 'hi'):
      t, parts = rs['ss_' + key], rs['parts_' + key]
      _check_dev(f'rs.ss_{key}', t, torch.float32, dev)
      if parts <= 0 or rs['ss_stride'] < m:
        raise ValueError(f'rs: parts_{key} = {parts} / ss_stride {rs["ss_stride"]} (m = {m})')
      _check_view(f'rs.ss_{key}', t, 0, rs['ss_stride'], parts, m, 4)
      sums['ss_' + key], sums['parts_' + key] = _ptr(t), parts
    if rs.get('bias') is not None:
      t, off, stride = rs['bias']
      if stride and step is None:
        raise ValueError('rs.bias: a step stride needs the device step')
      _check_vector('rs.bias', t, off + s * stride, n, dev)
      sums['col_bias'], sums['bias_step_stride'] = ctypes.c_void_p(t.data_ptr() + 4 * off), stride
    ra = _native.MsdGemmRowScale(**sums, split_row=rs['split_row'], ss_stride=rs['ss_stride'],
                                 inv_d=rs['inv_d'])
  args = _native.MsdGemmViewArgs(
      a=_ptr(a), a_off=a_off, lda=lda, b=_ptr(b), b_off=b_off, ldb=ldb, M=m, N=n, K=k,
      epilogue=GEMM_EPILOGUES[epilogue], block_n=block_n, out=_ptr(out), out_off=out_off,
      ldo=ldo, resid=_ptr(resid), resid_off=resid_off, pos=_ptr(pos), pos_rows=pos_rows,
      pos_shift=_ptr(pos_shift), dup_rows=dup_rows, step=_ptr(step), prep=pa, rs=ra)
  bn = ctypes.c_int32(0)
  _native.check(_native.load().msd_op_gemm_view(ctypes.byref(args), ctypes.byref(bn), _stream(dev)),
                'msd_op_gemm_view')
  return bn.value


def op_prep_rows(x: torch.Tensor, g: torch.Tensor, g_off: int, g_step_stride: int, step: torch.Tensor,
                 rows: int, d: int, a_out: torch.Tensor, lda: int, ss_out: torch.Tensor) -> None:
  """The first decoder layer's prep (msd_op_prep_rows): a_out [rows, lda] bf16 = bf16(x * g_step),
  ss_out[:rows] = row sums of x^2; x f32 rows of d, g_step the d gains at g_off + step *
  g_step_stride.  Views are checked before the library is called."""
  dev = x.device
  _check_dev('x', x, torch.float32, dev)
  _check_view('x', x, 0, d, rows, d, 4)
  _check_vector('g', g, g_off + _step_value(step, dev) * g_step_stride, d, dev)
  _check_dev('a_out', a_out, torch.bfloat16, dev)
  _check_view('a_out', a_out, 0, lda, rows, d, 2)
  _check_vector('ss_out', ss_out, 0, rows, dev)
  _native.check(_native.load().msd_op_prep_rows(
      _ptr(x), ctypes.c_void_p(g.data_ptr() + 4 * g_off), g_step_stride, _ptr(step), rows, d,
      _ptr(a_out), lda, _ptr(ss_out), _stream(dev)), 'msd_op_prep_rows')


def op_rmsnorm_view(x: torch.Tensor, gamma: torch.Tensor, out: torch.Tensor, out_off: int, ldo: int,
                    film: Optional[torch.Tensor] = None, film_offset: int = 0, film_step_stride: int = 0,
                    step: Optional[torch.Tensor] = None, split3: bool = False, src_len: int = 0,
                    dst_len: int = 0, dst_off: int = 0) -> None:
  """The norm kernel in any form the engine launches it (msd_op_rmsnorm_view): x f32 [rows, d] ->
  rmsnorm(x) gamma, with FiLM (scale | bias rows [2 d] of film at film_offset + step * film_step_stride)
  when film is given, written in place to the bf16 out at out_off + r * ldo (split3: [hi | lo | hi]).
  src_len > 0 remaps row b * src_len + t to b * dst_len + dst_off + t.  Views are checked before the
  library is called."""
  dev = x.device
  _check_dev('x', x, torch.float32, dev)
  if x.dim() != 2:
    raise ValueError(f'x: expected [rows, d], got {tuple(x.shape)}')
  rows, d = x.shape
  if rows <= 0 or d % 128 or not 0 < d <= 1024:
    raise ValueError(f'x: {rows} rows of d = {d}: d must be k * 128 <= 1024')
  _check_view('x', x, 0, d, rows, d, 4)
  _check_vector('gamma', gamma, 0, d, dev)
  _check_dev('out', out, torch.bfloat16, dev)
  width = 3 * d if split3 else d
  out_rows = rows
  if src_len:
    if src_len < 0 or rows % src_len or dst_off < 0 or dst_off + src_len > dst_len:
      raise ValueError(f'remap of {rows} rows in sequences of {src_len} to rows [{dst_off}, '
                       f'{dst_off + src_len}) of {dst_len}')
    if film is not None:
      raise ValueError('a remapped launch takes no FiLM')
    if ldo != width:
      raise ValueError(f'a remapped launch writes rows of {width} values: ldo must be {width}')
    out_rows = rows // src_len * dst_len
  _check_view('out', out, out_off, ldo, out_rows, width, 2)
  if film is not None:
    if step is None:
      raise ValueError('FiLM rows need the device step')
    _check_vector('film', film, film_offset + _step_value(step, dev) * film_step_stride, 2 * d, dev)
    if film_offset % 4 or film_step_stride % 4 or film_step_stride < 0:
      raise ValueError(f'film: offset {film_offset} / step stride {film_step_stride} must be '
                       'non-negative multiples of 4')
  args = _native.MsdRmsnormViewArgs(
      x=_ptr(x), rows=rows, d=d, gamma=_ptr(gamma), out=_ptr(out), out_off=out_off, ldo=ldo, film=_ptr(film),
      film_step_stride=film_step_stride, film_offset=film_offset, step=_ptr(step), split3=int(bool(split3)),
      src_len=src_len, dst_len=dst_len, dst_off=dst_off)
  _native.check(_native.load().msd_op_rmsnorm_view(ctypes.byref(args), _stream(dev)), 'msd_op_rmsnorm_view')


def op_encoder_inputs(tokens: torch.Tensor, ctx_mask: Optional[torch.Tensor], embedding: torch.Tensor,
                      pos: torch.Tensor, terminal_relative: bool, bits: torch.Tensor,
                      ctx_seq_len: torch.Tensor, x: torch.Tensor) -> None:
  """The encoder's front end as msd_encode runs it (msd_op_encoder_inputs): from tokens int32 [B, T]
  and ctx_mask int32 [B, C] (None: no context, C = 0), writes the key-mask words bits int32 storage
  [B, (T + C) / 32], the context roll ctx_seq_len int32 [B] and the token encoder's input rows x f32
  [B, T, d] = one_hot(tokens) embedding [vocab, d] + pos [T, d].  Buffers are checked before the
  library is called."""
  dev = tokens.device
  _check_dev('tokens', tokens, torch.int32, dev)
  if tokens.dim() != 2 or not tokens.is_contiguous():
    raise ValueError(f'tokens: expected a contiguous [B, T], got {tuple(tokens.shape)}')
  b, t = tokens.shape
  c = 0
  if ctx_mask is not None:
    _check_dev('ctx_mask', ctx_mask, torch.int32, dev)
    if ctx_mask.dim() != 2 or ctx_mask.shape[0] != b or not ctx_mask.is_contiguous():
      raise ValueError(f'ctx_mask: expected a contiguous [{b}, C], got {tuple(ctx_mask.shape)}')
    c = ctx_mask.shape[1]
  if b < 1 or t <= 0 or t % 128 or c % 128 or (ctx_mask is not None and c == 0):
    raise ValueError(f'B = {b} must be >= 1, T = {t} and C = {c} positive multiples of 128')
  if terminal_relative and c == 0:
    raise ValueError('terminal_relative positions need a context')
  _check_dev('embedding', embedding, torch.float32, dev)
  if embedding.dim() != 2 or not embedding.is_contiguous() or embedding.shape[0] < 1:
    raise ValueError(f'embedding: expected a contiguous [vocab, d], got {tuple(embedding.shape)}')
  vocab, d = embedding.shape
  if d % 4:
    raise ValueError(f'd = {d} must be a multiple of 4')
  _check_flat('pos', pos, torch.float32, dev, t * d)
  _check_flat('bits', bits, torch.int32, dev, b * (t + c) // 32)
  _check_flat('ctx_seq_len', ctx_seq_len, torch.int32, dev, b)
  _check_flat('x', x, torch.float32, dev, b * t * d)
  args = _native.MsdEncoderInputsArgs(
      tokens=_ptr(tokens), ctx_mask=_ptr(ctx_mask), B=b, T=t, C=c, terminal_relative=int(bool(terminal_relative)),
      embedding=_ptr(embedding), pos=_ptr(pos), d=d, vocab=vocab, bits=_ptr(bits), ctx_seq_len=_ptr(ctx_seq_len),
      x=_ptr(x))
  _native.check(_native.load().msd_op_encoder_inputs(ctypes.byref(args), _stream(dev)), 'msd_op_encoder_inputs')


STEP_COLS = 16   # floats per diffusion step in the sampler table (msd_get_step_table)


def step_table_for(cfg: _native.MsdConfig) -> np.ndarray:
  """The sampler's per-step table [num_steps, STEP_COLS] float32 for cfg (msd_step_table): what
  Engine.step_table() returns for a context created from cfg, computed on the host without a GPU."""
  if not isinstance(cfg, _native.MsdConfig):
    raise TypeError(f'cfg: expected an MsdConfig, got {type(cfg).__name__}')
  if cfg.num_steps <= 0:
    raise ValueError(f'num_steps = {cfg.num_steps} must be positive')
  tab = np.zeros((cfg.num_steps, STEP_COLS), dtype=np.float32)
  _native.check(_native.load().msd_step_table(ctypes.byref(cfg), tab.ctypes.data), 'msd_step_table')
  return tab


def _check_flat(name: str, t: torch.Tensor, dtype: torch.dtype, device: torch.device, n: int) -> None:
  """t is a contiguous `dtype` tensor on `device` with at least n elements."""
  _check_dev(name, t, dtype, device)
  if not t.is_contiguous():
    raise ValueError(f'{name}: tensor must be contiguous')
  if t.numel() < n:
    raise ValueError(f'{name}: {t.numel()} elements, the launch reads or writes {n}')


def _check_state(z: torch.Tensor, z_split: torch.Tensor, n: int, n_dims: int) -> None:
  if n <= 0 or n_dims <= 0 or n % 4 or n_dims % 4 or n % n_dims:
    raise ValueError(f'n = {n} must be a positive multiple of n_dims = {n_dims}, both multiples of 4')
  if not z.is_cuda:
    raise ValueError(f'z: expected a CUDA tensor, got one on {z.device}')
  _check_flat('z', z, torch.float32, z.device, n)
  _check_flat('z_split', z_split, torch.bfloat16, z.device, 3 * n)


def _check_streams(n: int, steps: int, rng_kind: int, rng_keys: Optional[torch.Tensor], n_row: int,
                   row_keys: Optional[torch.Tensor], row_key_stride: int,
                   row_seeds: Optional[torch.Tensor], per_row: bool, device: torch.device) -> None:
  """The key / seed tables a generated draw of n elements reads: rng_kind 1 reads key rows
  0 .. steps of rng_keys (int32 storage of uint32 words, 2 per row); per-row streams read row b's
  table at row_keys + b * row_key_stride, or its Philox seed row_seeds[b] (int64 storage)."""
  if rng_kind not in (0, 1):
    raise ValueError(f'rng_kind = {rng_kind} must be 0 (philox) or 1 (jax)')
  if not per_row:
    if rng_kind == 1:
      if rng_keys is None or n % 8 or n >= 1 << 32:
        raise ValueError('the jax stream needs rng_keys and a draw of k * 8 < 2^32 elements')
      _check_flat('rng_keys', rng_keys, torch.int32, device, 2 * (steps + 1))
    return
  if n_row <= 0 or n_row % 8 or n % n_row or n >= 1 << 32:
    raise ValueError(f'per-row streams: n_row = {n_row} must be a multiple of 8 dividing n = {n} < 2^32')
  rows = n // n_row
  if rng_kind == 1:
    if row_keys is None or row_key_stride < 2 * (steps + 1):
      raise ValueError(f'per-row jax streams need row_keys with a stride >= {2 * (steps + 1)}')
    _check_flat('row_keys', row_keys, torch.int32, device, (rows - 1) * row_key_stride + 2 * (steps + 1))
  else:
    if row_seeds is None:
      raise ValueError('per-row Philox streams need row_seeds')
    _check_flat('row_seeds', row_seeds, torch.int64, device, rows)


def op_sampler_step(eps: torch.Tensor, z: torch.Tensor, z_split: torch.Tensor, coef: torch.Tensor,
                    n: int, passes: int, cond_weight: float, clip_x0: bool, ddim: bool,
                    feat_min: float, feat_max: float, n_dims: int = 128,
                    step: Optional[torch.Tensor] = None, run_step: Optional[int] = None,
                    launches: int = 1, mel_out: Optional[torch.Tensor] = None,
                    noise: Optional[torch.Tensor] = None, seed: int = 0, rng_kind: int = 0,
                    rng_keys: Optional[torch.Tensor] = None, per_row: bool = False, n_row: int = 0,
                    row_keys: Optional[torch.Tensor] = None, row_key_stride: int = 0,
                    row_seeds: Optional[torch.Tensor] = None):
  """The sampler kernel on caller-owned device buffers (msd_op_sampler_step): updates z[:n] and
  z_split[:3 n] in place (and mel_out[:n] at step 0).  eps f32 [passes * n], coef f32 [steps, 16],
  noise f32 [steps, n] or None (generated: seed / rng_keys, or the per-row tables).
  Exactly one of `step` (device int32: one launch, the step read from there) and `run_step` (the
  graph's RunArgs path: `launches` launches from that step) is given; the latter returns the
  (step, done) the RunArgs hold afterwards.  Every buffer is checked before the library is called."""
  if (step is None) == (run_step is None):
    raise ValueError('give exactly one of step (device) and run_step (RunArgs path)')
  if passes not in (1, 2):
    raise ValueError(f'passes = {passes} must be 1 or 2')
  _check_state(z, z_split, n, n_dims)
  dev = z.device
  _check_flat('eps', eps, torch.float32, dev, passes * n)
  _check_dev('coef', coef, torch.float32, dev)
  if coef.dim() != 2 or coef.shape[1] != STEP_COLS or coef.shape[0] <= 0 or not coef.is_contiguous():
    raise ValueError(f'coef: expected a contiguous [num_steps, {STEP_COLS}] table, got {tuple(coef.shape)}')
  steps = coef.shape[0]
  if step is not None:
    first = _step_value(step, dev)
    if per_row or launches != 1:
      raise ValueError('per-row streams and several launches take the RunArgs path (run_step)')
  else:
    first = int(run_step)
  if launches < 1 or first >= steps or first - launches + 1 < 0:
    raise ValueError(f'{launches} launch(es) from step {first} leave the table of {steps} steps')
  if mel_out is not None:
    _check_flat('mel_out', mel_out, torch.float32, dev, n)
  if noise is not None:
    _check_flat('noise', noise, torch.float32, dev, steps * n)
  else:
    _check_streams(n, steps, rng_kind, rng_keys, n_row, row_keys, row_key_stride, row_seeds, per_row, dev)
  streams = _native.MsdNoiseStreams(
      seed=int(seed) & 0xFFFFFFFFFFFFFFFF, rng_kind=rng_kind, rng_keys=_ptr(rng_keys), n_row=n_row,
      row_keys=_ptr(row_keys), row_key_stride=row_key_stride, row_seeds=_ptr(row_seeds))
  args = _native.MsdSamplerStepArgs(
      eps=_ptr(eps), z=_ptr(z), z_split=_ptr(z_split), mel_out=_ptr(mel_out), noise=_ptr(noise),
      coef=_ptr(coef), num_steps=steps, step=_ptr(step), n=n, n_dims=n_dims, passes=passes,
      cond_weight=float(cond_weight), clip_x0=int(bool(clip_x0)), ddim=int(bool(ddim)),
      feat_min=float(feat_min), feat_max=float(feat_max), streams=streams,
      run_step=0 if run_step is None else first, per_row=int(bool(per_row)), launches=launches)
  run_out = (ctypes.c_int32 * 2)()
  _native.check(_native.load().msd_op_sampler_step(ctypes.byref(args), run_out, _stream(dev)),
                'msd_op_sampler_step')
  return None if run_step is None else (run_out[0], run_out[1])


def op_init_z(z: torch.Tensor, z_split: torch.Tensor, n: int, n_dims: int = 128,
              init_z: Optional[torch.Tensor] = None, seed: int = 0, rng_kind: int = 0,
              rng_keys: Optional[torch.Tensor] = None, n_row: int = 0, row_key_stride: int = 0,
              row_seeds: Optional[torch.Tensor] = None) -> None:
  """The sampler's initial state (msd_op_init_z): z[:n] = init_z[:n], or the draw of Philox stream 0
  of seed (rng_kind 0) / of key row 0 of rng_keys (rng_kind 1); n_row > 0: row b's own draw from
  row_seeds[b] / row_keys + b * row_key_stride (rng_keys is then the per-row table).  z_split[:3 n]
  gets the [hi | lo | hi] split.  Buffers are checked before the library is called."""
  _check_state(z, z_split, n, n_dims)
  dev = z.device
  if init_z is not None:
    _check_flat('init_z', init_z, torch.float32, dev, n)
  else:
    _check_streams(n, 0, rng_kind, rng_keys, n_row, rng_keys, row_key_stride, row_seeds, n_row > 0, dev)
  streams = _native.MsdNoiseStreams(
      seed=int(seed) & 0xFFFFFFFFFFFFFFFF, rng_kind=rng_kind, rng_keys=_ptr(rng_keys), n_row=n_row,
      row_keys=_ptr(rng_keys), row_key_stride=row_key_stride, row_seeds=_ptr(row_seeds))
  args = _native.MsdInitZArgs(init_z=_ptr(init_z), z=_ptr(z), z_split=_ptr(z_split), n=n, n_dims=n_dims,
                              streams=streams)
  _native.check(_native.load().msd_op_init_z(ctypes.byref(args), _stream(dev)), 'msd_op_init_z')


def op_scale_split(feat: torch.Tensor, feat_min: float, feat_max: float,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
  """The encoder's context-feature front end (msd_op_scale_split): feat f32 [rows, n_dims] ->
  bf16 [rows, 3 n_dims] = [hi | lo | hi] of scale_features(feat, clip=True), written into out (which
  may be larger: only its first rows * 3 n_dims elements are written) or a new tensor."""
  if feat.dim() != 2 or not feat.is_cuda:
    raise ValueError(f'feat: expected a [rows, n_dims] CUDA tensor, got {tuple(feat.shape)} on {feat.device}')
  rows, nd = feat.shape
  if rows <= 0 or nd <= 0 or nd % 4:
    raise ValueError(f'feat: {rows} rows of {nd}: n_dims must be a positive multiple of 4')
  _check_flat('feat', feat, torch.float32, feat.device, rows * nd)
  if out is None:
    out = torch.empty(rows, 3 * nd, dtype=torch.bfloat16, device=feat.device)
  _check_flat('out', out, torch.bfloat16, feat.device, rows * 3 * nd)
  _native.check(_native.load().msd_op_scale_split(_ptr(feat), _ptr(out), rows, nd, float(feat_min),
                                                  float(feat_max), _stream(feat.device)),
                'msd_op_scale_split')
  return out


def op_jax_bits(seed: int, step: int, n: int, device: torch.device) -> torch.Tensor:
  """Raw uint32 words of the device jax.random stream (as int32 storage; view as uint32)."""
  out = torch.empty(n, dtype=torch.int32, device=device)
  _native.check(_native.load().msd_op_jax_bits(seed, step, n, _ptr(out), _stream(device)),
                'msd_op_jax_bits')
  return out


def op_jax_normal(seed: int, step: int, n: int, device: torch.device) -> torch.Tensor:
  """Device draw of the jax.random stream (step < 0: init_z; else the noise of scan index step)."""
  out = torch.empty(n, dtype=torch.float32, device=device)
  _native.check(_native.load().msd_op_jax_normal(seed, step, n, _ptr(out), _stream(device)),
                'msd_op_jax_normal')
  return out


def op_audio_mel(audio: torch.Tensor, window: torch.Tensor, weights: torch.Tensor) -> torch.Tensor:
  """MelGAN log-mel features of audio [rows, n] (msd_op_audio_mel): f32 [rows, ceil(n / 320), 128]
  from the window f32 [640] and mel weights f32 [513, 128] (audio_codecs.mel_tables), all
  contiguous f32 tensors on one CUDA device.  Enqueued on the device's current stream."""
  for name, t, shape in (('audio', audio, None), ('window', window, (640,)),
                         ('weights', weights, (513, 128))):
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
      raise ValueError(f'{name}: expected a contiguous float32 CUDA tensor, got {t.dtype} on '
                       f'{t.device} (contiguous: {t.is_contiguous()})')
    if t.device != audio.device:
      raise ValueError(f'{name} is on {t.device}, audio on {audio.device}')
    if shape is not None and tuple(t.shape) != shape:
      raise ValueError(f'{name}: expected shape {shape}, got {tuple(t.shape)}')
  if audio.dim() != 2:
    raise ValueError(f'audio: expected [rows, n], got {tuple(audio.shape)}')
  rows, n = audio.shape
  out = torch.empty(rows, -(-n // 320), 128, dtype=torch.float32, device=audio.device)
  if out.numel() == 0:
    return out
  with torch.cuda.device(audio.device):
    _native.check(_native.load().msd_op_audio_mel(_ptr(audio), rows, n, _ptr(window), _ptr(weights),
                                                   _ptr(out), _stream(audio.device)),
                  'msd_op_audio_mel')
  return out


def op_audio_resample(audio: torch.Tensor, orig_sr: int, target_sr: int, window: torch.Tensor,
                      precision: int, segments: torch.Tensor) -> torch.Tensor:
  """audio [rows, n] resampled from orig_sr to target_sr as resampy's kaiser_best loop does it
  (msd_op_audio_resample): f32 [rows, int(n * target_sr / orig_sr)] (resampy's length, not yet
  padded to librosa's).  audio is a contiguous f32 CUDA tensor; window (the unscaled half window,
  audio_codecs.resample_window) f64 [window_len] with 2^precision entries per zero crossing, and
  segments (audio_codecs.time_register_segments) f64 [S, 3], on the same device.  Enqueued on the
  device's current stream."""
  for name, t, dtype, dim in (('audio', audio, torch.float32, 2), ('window', window, torch.float64, 1),
                              ('segments', segments, torch.float64, 2)):
    if t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
      raise ValueError(f'{name}: expected a contiguous {dtype} CUDA tensor, got {t.dtype} on '
                       f'{t.device} (contiguous: {t.is_contiguous()})')
    if t.device != audio.device:
      raise ValueError(f'{name} is on {t.device}, audio on {audio.device}')
    if t.dim() != dim:
      raise ValueError(f'{name}: expected {dim} dimensions, got {tuple(t.shape)}')
  if segments.shape[1] != 3 or segments.shape[0] < 1:
    raise ValueError(f'segments: expected [S >= 1, 3], got {tuple(segments.shape)}')
  if int(orig_sr) != orig_sr or int(target_sr) != target_sr or orig_sr <= 0 or target_sr <= 0:
    raise ValueError(f'rates must be positive integers, got {orig_sr} -> {target_sr}')
  rows, n = audio.shape
  out = torch.empty(rows, int(n * (float(target_sr) / orig_sr)), dtype=torch.float32,
                    device=audio.device)
  if out.numel() == 0:
    return out
  with torch.cuda.device(audio.device):
    _native.check(_native.load().msd_op_audio_resample(
        _ptr(audio), rows, n, int(orig_sr), int(target_sr), _ptr(window), window.shape[0],
        precision, _ptr(segments), segments.shape[0], _ptr(out), out.shape[1],
        _stream(audio.device)), 'msd_op_audio_resample')
  return out


def _check_gl(name: str, t: torch.Tensor, dtype, shape, device) -> None:
  if t.dtype != dtype or not t.is_cuda or not t.is_contiguous():
    raise ValueError(f'{name}: expected a contiguous {dtype} CUDA tensor, got {t.dtype} on '
                     f'{t.device} (contiguous: {t.is_contiguous()})')
  if t.device != device:
    raise ValueError(f'{name} is on {t.device}, expected {device}')
  if shape is not None and tuple(t.shape) != tuple(shape):
    raise ValueError(f'{name}: expected shape {tuple(shape)}, got {tuple(t.shape)}')


def op_griffin_lim_magnitude(features: torch.Tensor, weights: torch.Tensor, pinv: torch.Tensor,
                             inv_lipschitz: float, beta: torch.Tensor, n_iter: int) -> torch.Tensor:
  """Linear magnitudes of MelGAN features [rows, F, 128] (msd_op_griffin_lim_magnitude): f32
  [rows, F, 513], the non-negative least-squares fit of exp(features) by S @ weights after n_iter
  FISTA steps from max(0, exp(features) @ pinv).  weights f32 [513, 128], pinv f32 [128, 513] and
  beta f32 [>= n_iter] (audio_codecs.griffin_lim_tables) on the features' device.  Enqueued on the
  device's current stream."""
  if features.dim() != 3 or features.shape[2] != 128:
    raise ValueError(f'features: expected [rows, F, 128], got {tuple(features.shape)}')
  dev = features.device
  _check_gl('features', features, torch.float32, None, dev)
  _check_gl('weights', weights, torch.float32, (513, 128), dev)
  _check_gl('pinv', pinv, torch.float32, (128, 513), dev)
  _check_gl('beta', beta, torch.float32, None, dev)
  if int(n_iter) != n_iter or n_iter < 0 or beta.dim() != 1 or beta.shape[0] < max(n_iter, 1):
    raise ValueError(f'n_iter={n_iter} must be >= 0 with beta [>= max(n_iter, 1)], got beta '
                     f'{tuple(beta.shape)}')
  rows, frames = features.shape[:2]
  out = torch.empty(rows, frames, 513, dtype=torch.float32, device=dev)
  if out.numel() == 0:
    return out
  with torch.cuda.device(dev):
    _native.check(_native.load().msd_op_griffin_lim_magnitude(
        _ptr(features), rows, frames, _ptr(weights), _ptr(pinv), float(inv_lipschitz), _ptr(beta),
        int(n_iter), _ptr(out), _stream(dev)), 'msd_op_griffin_lim_magnitude')
  return out


def op_griffin_lim_init(rows: int, frames: int, seed: int, device: torch.device) -> torch.Tensor:
  """Random initial phases (msd_op_griffin_lim_init): complex64 [rows, frames, 513] of modulus 1
  from the Philox stream of seed, the same for every row."""
  if rows < 0 or frames < 0:
    raise ValueError(f'rows={rows}, frames={frames} must be >= 0')
  out = torch.empty(rows, frames, 513, dtype=torch.complex64, device=device)
  if out.numel() == 0:
    return out
  with torch.cuda.device(device):
    _native.check(_native.load().msd_op_griffin_lim_init(
        rows, frames, int(seed) & 0xFFFFFFFFFFFFFFFF, _ptr(out), _stream(device)),
        'msd_op_griffin_lim_init')
  return out


def op_griffin_lim_iterate(mag: torch.Tensor, window: torch.Tensor, angles: torch.Tensor,
                           tprev: torch.Tensor, momentum: float, n_iter: int,
                           work: Optional[torch.Tensor] = None) -> None:
  """n_iter fast Griffin-Lim iterations (msd_op_griffin_lim_iterate) on angles and tprev,
  complex64 [rows, F, 513], in place, against the magnitudes mag f32 [rows, F, 513] with the
  codec's window f32 [640].  work (complex64, the same shape) is scratch; one is allocated when it
  is None.  Enqueued on the device's current stream."""
  if mag.dim() != 3 or mag.shape[2] != 513:
    raise ValueError(f'mag: expected [rows, F, 513], got {tuple(mag.shape)}')
  if not momentum >= 0:
    raise ValueError(f'momentum={momentum} must be >= 0')
  if int(n_iter) != n_iter or n_iter < 0:
    raise ValueError(f'n_iter={n_iter} must be an integer >= 0')
  dev = mag.device
  _check_gl('mag', mag, torch.float32, None, dev)
  _check_gl('window', window, torch.float32, (640,), dev)
  _check_gl('angles', angles, torch.complex64, mag.shape, dev)
  _check_gl('tprev', tprev, torch.complex64, mag.shape, dev)
  if work is None:
    work = torch.empty_like(angles)
  _check_gl('work', work, torch.complex64, mag.shape, dev)
  if mag.numel() == 0 or n_iter == 0:
    return
  with torch.cuda.device(dev):
    _native.check(_native.load().msd_op_griffin_lim_iterate(
        _ptr(mag), mag.shape[0], mag.shape[1], _ptr(window), _ptr(angles), _ptr(tprev), _ptr(work),
        float(momentum), int(n_iter), _stream(dev)), 'msd_op_griffin_lim_iterate')


def op_griffin_lim_istft(mag: torch.Tensor, window: torch.Tensor, angles: torch.Tensor) -> torch.Tensor:
  """audio f32 [rows, 320 F] = ISTFT(mag angles) (msd_op_griffin_lim_istft): mag f32 and angles
  complex64 [rows, F, 513], window f32 [640], on one CUDA device."""
  if mag.dim() != 3 or mag.shape[2] != 513:
    raise ValueError(f'mag: expected [rows, F, 513], got {tuple(mag.shape)}')
  dev = mag.device
  _check_gl('mag', mag, torch.float32, None, dev)
  _check_gl('window', window, torch.float32, (640,), dev)
  _check_gl('angles', angles, torch.complex64, mag.shape, dev)
  out = torch.empty(mag.shape[0], mag.shape[1] * 320, dtype=torch.float32, device=dev)
  if out.numel() == 0:
    return out
  with torch.cuda.device(dev):
    _native.check(_native.load().msd_op_griffin_lim_istft(
        _ptr(mag), _ptr(angles), mag.shape[0], mag.shape[1], _ptr(window), _ptr(out), _stream(dev)),
        'msd_op_griffin_lim_istft')
  return out
