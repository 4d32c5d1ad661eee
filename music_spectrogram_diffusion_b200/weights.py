"""Parameter tree of ContinuousContextTransformer (or, without a context, Transformer): names,
shapes, synthetic init.

Names follow the flax tree the reference creates (SURVEY App. B):
  setup() attribute names   msd/models/diffusion/network.py:530-535
  layer / norm / dense names  network.py:127-152, 174-252, 278-301, 321-355,
                              380-456; msd/layers.py:262-264, 371-377, 485-508
  no-context Transformer      network.py:460-468: token encoder `encoder`, no continuous
                              encoder, one cross-attention source (`..._0` only)
A real T5X checkpoint flattens to exactly these '/'-joined keys under
``target/`` (read by ``t5x_checkpoint.py``); the tree can also be synthesised
(no checkpoint is available offline) or loaded from an ``.npz``.
"""

from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np

from music_spectrogram_diffusion_b200.config import T5Config

ParamDict = Dict[str, np.ndarray]


def _attention(prefix: str, d: int, hd_total: int) -> List[Tuple[str, Tuple[int, ...]]]:
  return [
      (f'{prefix}/query/kernel', (d, hd_total)),
      (f'{prefix}/key/kernel', (d, hd_total)),
      (f'{prefix}/value/kernel', (d, hd_total)),
      (f'{prefix}/out/kernel', (hd_total, d)),
  ]


def _mlp(prefix: str, d: int, f: int, n_act: int) -> List[Tuple[str, Tuple[int, ...]]]:
  out = []
  for i in range(n_act):
    name = 'wi' if n_act == 1 else f'wi_{i}'
    out.append((f'{prefix}/{name}/kernel', (d, f)))
  out.append((f'{prefix}/wo/kernel', (f, d)))
  return out


def param_shapes(cfg: T5Config, inputs_length: int, targets_length: int,
                 context_length: Optional[int], n_dims: int = 128
                 ) -> List[Tuple[str, Tuple[int, ...]]]:
  """Ordered (name, shape) list of every parameter on the inference path.  context_length 0 or
  None: the no-context network.Transformer tree."""
  d, hh, f = cfg.emb_dim, cfg.num_heads * cfg.head_dim, cfg.mlp_dim
  na = len(cfg.mlp_activations)
  ctx = bool(context_length)
  tok = 'token_encoder' if ctx else 'encoder'
  s: List[Tuple[str, Tuple[int, ...]]] = []
  s.append((f'{tok}/token_embedder/embedding', (cfg.vocab_size, d)))
  s.append((f'{tok}/Embed_0/embedding', (inputs_length, d)))
  for enc in (tok, 'continuous_encoder') if ctx else (tok,):
    if enc == 'continuous_encoder':
      s.append(('continuous_encoder/input_proj/kernel', (n_dims, d)))
      s.append(('continuous_encoder/Embed_0/embedding', (context_length, d)))
    for l in range(cfg.num_encoder_layers):
      p = f'{enc}/layers_{l}'
      s.append((f'{p}/pre_attention_layer_norm/scale', (d,)))
      s += _attention(f'{p}/attention', d, hh)
      s.append((f'{p}/pre_mlp_layer_norm/scale', (d,)))
      s += _mlp(f'{p}/mlp', d, f, na)
    s.append((f'{enc}/encoder_norm/scale', (d,)))
  s.append(('decoder/time_emb_dense0/kernel', (d, 4 * d)))
  s.append(('decoder/time_emb_dense1/kernel', (4 * d, 4 * d)))
  s.append(('decoder/Embed_0/embedding', (targets_length, d)))
  s.append(('decoder/continuous_inputs_projection/kernel', (n_dims, d)))
  for l in range(cfg.num_decoder_layers):
    p = f'decoder/layers_{l}'
    s.append((f'{p}/pre_self_attention_layer_norm/scale', (d,)))
    s.append((f'{p}/FiLMLayer_0/DenseGeneral_0/kernel', (4 * d, 2 * d)))
    s += _attention(f'{p}/self_attention', d, hh)
    s.append((f'{p}/pre_cross_attention_layer_norm/scale', (d,)))
    # one attention per source for sum_cross_attends (network.py:199-216): without a context
    # there is one source and either style has only `_0`
    if cfg.decoder_cross_attend_style == 'concat_encodings' or not ctx:
      s += _attention(f'{p}/MultiHeadDotProductAttention_0', d, hh)
    else:
      s += _attention(f'{p}/MultiHeadDotProductAttention_0', d, hh)
      s += _attention(f'{p}/MultiHeadDotProductAttention_1', d, hh)
    s.append((f'{p}/pre_mlp_layer_norm/scale', (d,)))
    s.append((f'{p}/FiLMLayer_1/DenseGeneral_0/kernel', (4 * d, 2 * d)))
    s += _mlp(f'{p}/mlp', d, f, na)
  s.append(('decoder/decoder_norm/scale', (d,)))
  s.append(('decoder/spec_out_dense/kernel', (d, n_dims)))
  return s


def num_params(shapes) -> int:
  return int(sum(int(np.prod(sh)) for _, sh in shapes))


def _sinusoidal(max_len: int, features: int, rng: np.random.Generator) -> np.ndarray:
  """'fixed_permuted_offset' table, msd/layers.py:51-106 (numpy rng)."""
  position = np.arange(0, max_len)[:, np.newaxis]
  scale_factor = -np.log(10000.0) / (features // 2 - 1)
  div_term = np.exp(np.arange(0, features // 2) * scale_factor)
  rads = position * div_term
  sin_off = rng.uniform(0, 2 * np.pi, [features // 2])
  cos_off = rng.uniform(0, 2 * np.pi, [features // 2])
  pe = np.zeros((max_len, features), dtype=np.float32)
  pe[:, :features // 2] = np.sin(rads + sin_off)
  pe[:, features // 2:2 * (features // 2)] = np.cos(rads + cos_off)
  return pe[:, rng.permutation(features)].astype(np.float32)


def synthetic_params(cfg: T5Config, inputs_length: int = 2048,
                     targets_length: int = 256, context_length: Optional[int] = 256,
                     n_dims: int = 128, seed: int = 0) -> ParamDict:
  """Seeded random-init tree with the reference's initialiser statistics.

  Dense kernels N(0, 1/fan_in) (variance_scaling(1,'fan_in'), layers.py:206,
  411); query kernels additionally / sqrt(head_dim) (layers.py:254-258); norm
  scales 1 + 0.1 N(0,1) so they are not the identity; token embedding N(0,1)
  (network.py:282); FiLM kernels x0.1 to keep activations O(1).
  """
  rng = np.random.default_rng(seed)
  out: ParamDict = {}
  for name, shape in param_shapes(cfg, inputs_length, targets_length,
                                  context_length, n_dims):
    if name.endswith('/scale'):
      w = 1.0 + 0.1 * rng.standard_normal(shape)
    elif name.endswith('token_embedder/embedding'):
      w = rng.standard_normal(shape)
    elif name.endswith('Embed_0/embedding'):
      w = _sinusoidal(shape[0], shape[1], rng)
    else:
      w = rng.standard_normal(shape) / math.sqrt(shape[0])
      if name.endswith('/query/kernel'):
        w = w / math.sqrt(cfg.head_dim)
      if 'FiLMLayer' in name:
        w = w * 0.1
    out[name] = np.ascontiguousarray(w, dtype=np.float32)
  return out


def check_params(params: ParamDict, cfg: T5Config, inputs_length: int, targets_length: int,
                 context_length: Optional[int], n_dims: int = 128) -> None:
  """Raises if a restored tree lacks a parameter of the inference path or has a wrong shape
  (the reference fails inside t5x's restore with a shape-mismatch error, inference.py:171-181).
  Extra entries (optimizer slots, unrelated modules) are ignored."""
  problems = []
  for name, shape in param_shapes(cfg, inputs_length, targets_length, context_length, n_dims):
    if name not in params:
      problems.append(f'missing {name} {shape}')
    elif tuple(params[name].shape) != tuple(shape):
      problems.append(f'{name}: checkpoint shape {tuple(params[name].shape)} != model shape {shape}')
  if problems:
    head = '; '.join(problems[:6])
    raise ValueError(f'checkpoint does not match the gin config ({len(problems)} problems): {head}')


def save_npz(path: str, params: ParamDict) -> None:
  np.savez(path, **{k.replace('/', '.'): v for k, v in params.items()})


def load_npz(path: str) -> ParamDict:
  with np.load(path) as z:
    return {k.replace('.', '/'): np.ascontiguousarray(z[k], dtype=np.float32)
            for k in z.files}
