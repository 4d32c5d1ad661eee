"""CPU restatement of the reference's DDPM sampling hot path (the ORACLE).

THIS FILE IS TEST INFRASTRUCTURE, NOT PRODUCT.  It restates, line by line, the
arithmetic of ``music_spectrogram_diffusion`` (reference files cited as
``msd/<file>:<lines>``) for the path

    InferenceModel.predict -> ContextDiffusionModel.predict_batch_with_aux
      -> ContinuousContextTransformer.encode / .decode -> eval_scan (DDPM)

in plain torch-CPU tensor ops (fp32 by default, fp64 on request), with the graph
exactly AS WRITTEN by the reference (cross-attention K/V re-projected on every
step, the unconditional pass run in full, FiLM recomputed from the timestep on
every call).  The CUDA product takes exact algebraic shortcuts (hoisted K/V,
elided unconditional cross-attention, tabulated FiLM); tests prove those
shortcuts equal this file.

PARITY STATUS: **parity unpinned** for the network and the sampler.  The
reference's JAX/Flax/T5X stack is not importable in this image (no jax, flax,
t5x, gin, seqio, tensorflow; no network), so this restatement cannot be checked
against outputs of the reference itself.  What IS pinned: the reference's own
known-answer tests for the primitives on the path, ``msd/layers_test.py``
``test_dot_product_attention`` (375-387), ``test_multihead_dot_product_attention``
(285-330), ``test_make_attention_mask_multiply_pairwise_fn`` (117-125) and
``DenseTest`` (450-484), re-expressed with the same ``np.random.seed(0)`` draws
in ``tests/test_oracle_kat.py``.  Third-party semantics relied upon (not in
/root/reference): ``flax.linen.gelu`` (tanh approximation), ``flax.linen.swish``
(x*sigmoid(x)), ``jax.nn.softmax`` (max-subtracted), ``lax.dot_general`` in true
fp32 (the CPU/XLA behaviour; TPUs default to bf16 passes).

Noise: ``jax.random`` (threefry) is third-party; parity runs inject ``init_z``
and the per-step ``noise`` explicitly into both this oracle and the CUDA path.
"""

from __future__ import annotations

import dataclasses
import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

Tensor = torch.Tensor
Params = Dict[str, Tensor]


# -----------------------------------------------------------------------------
# Config (mirrors msd/models/diffusion/network.py:54-72 and
# msd/models/diffusion/diffusion_utils.py:25-59; plain dataclasses, no gin).
# -----------------------------------------------------------------------------
@dataclasses.dataclass
class OracleConfig:
  vocab_size: int = 1536
  emb_dim: int = 768
  num_heads: int = 12
  num_encoder_layers: int = 12
  num_decoder_layers: int = 12
  head_dim: int = 64
  mlp_dim: int = 2048
  mlp_activations: Tuple[str, ...] = ('gelu', 'linear')
  max_decoder_noise_time: float = 2e4
  decoder_cross_attend_style: str = 'concat_encodings'
  context_positions: str = 'terminal_relative'
  # diffusion
  num_steps: int = 1000
  schedule: str = 'cosine'          # sampler schedule name ('cosine' | 'linear')
  schedule_start: Optional[float] = None   # linear schedule: beta range
  schedule_stop: Optional[float] = None
  train_schedule: str = 'cosine'
  train_schedule_start: Optional[float] = None
  train_schedule_stop: Optional[float] = None
  train_schedule_num_steps: Optional[int] = None
  model_output: str = 'eps'         # 'eps' | 'x0' | 'v'
  sampler: str = 'ddpm'
  clip_x0: bool = True
  logvar_type: str = 'large'
  eval_condition_weight: float = 5.0
  # codec (msd/audio_codecs.py:204-213)
  n_dims: int = 128
  min_value: float = math.log(1e-5)
  max_value: float = 4.0


# -----------------------------------------------------------------------------
# L1 primitives (msd/layers.py)
# -----------------------------------------------------------------------------
def dense_general(x: Tensor, kernel: Tensor) -> Tensor:
  """Bias-free dense over the last axis.  msd/layers.py:397-442."""
  return x.to(kernel.dtype) @ kernel


def layer_norm(x: Tensor, scale: Tensor, epsilon: float = 1e-6) -> Tensor:
  """T5 RMS norm, no mean subtraction / bias.  msd/layers.py:632-649."""
  mean2 = torch.mean(x * x, dim=-1, keepdim=True)
  y = x * torch.rsqrt(mean2 + epsilon)
  return y * scale


def gelu_tanh(x: Tensor) -> Tensor:
  """flax.linen.gelu default (approximate=True); named by msd/layers.py:451."""
  return 0.5 * x * (1.0 + torch.tanh(
      math.sqrt(2.0 / math.pi) * (x + 0.044715 * x * x * x)))


def swish(x: Tensor) -> Tensor:
  """flax.linen.swish, used at msd/models/diffusion/network.py:385,391."""
  return x * torch.sigmoid(x)


_ACTIVATIONS: Dict[str, Callable[[Tensor], Tensor]] = {
    'gelu': gelu_tanh,
    'linear': lambda x: x,
    'relu': torch.relu,
    'swish': swish,
}


def dot_product_attention(query: Tensor, key: Tensor, value: Tensor,
                          bias: Optional[Tensor] = None) -> Tensor:
  """softmax(QK^T + bias) V with NO 1/sqrt(d).  msd/layers.py:109-181.

  query [b,q,h,d], key/value [b,k,h,d], bias broadcastable to [b,h,q,k].
  """
  attn_weights = torch.einsum('bqhd,bkhd->bhqk', query, key)
  if bias is not None:
    attn_weights = attn_weights + bias.to(attn_weights.dtype)
  attn_weights = torch.softmax(attn_weights, dim=-1)
  return torch.einsum('bhqk,bkhd->bqhd', attn_weights, value)


def multi_head_dot_product_attention(
    inputs_q: Tensor, inputs_kv: Tensor, mask: Optional[Tensor],
    p: Params, prefix: str, num_heads: int, head_dim: int) -> Tensor:
  """msd/layers.py:188-379 (non-decode branch).

  Kernels: query/key/value [features, heads*head_dim], out [heads*head_dim,
  features] (layout pinned by msd/layers_test.py:285-330).  mask [b,1,q,k].
  """
  b, ql, _ = inputs_q.shape
  kl = inputs_kv.shape[1]
  query = dense_general(inputs_q, p[f'{prefix}/query/kernel'])
  key = dense_general(inputs_kv, p[f'{prefix}/key/kernel'])
  value = dense_general(inputs_kv, p[f'{prefix}/value/kernel'])
  query = query.reshape(b, ql, num_heads, head_dim)
  key = key.reshape(b, kl, num_heads, head_dim)
  value = value.reshape(b, kl, num_heads, head_dim)
  if mask is not None:
    # msd/layers.py:341-348: mask -> additive bias 0 / -1e10.
    attention_bias = torch.where(
        mask > 0, torch.zeros_like(mask), torch.full_like(mask, -1e10))
  else:
    attention_bias = None
  x = dot_product_attention(query, key, value, bias=attention_bias)
  x = x.reshape(b, ql, num_heads * head_dim)
  return dense_general(x, p[f'{prefix}/out/kernel'])


def mlp_block(x: Tensor, p: Params, prefix: str,
              activations: Sequence[str]) -> Tensor:
  """msd/layers.py:459-510: product of activated wi_k projections, then wo."""
  acts = []
  for idx, name in enumerate(activations):
    dense_name = 'wi' if len(activations) == 1 else f'wi_{idx}'
    h = dense_general(x, p[f'{prefix}/{dense_name}/kernel'])
    acts.append(_ACTIVATIONS[name](h))
  h = acts[0]
  for a in acts[1:]:
    h = h * a
  return dense_general(h, p[f'{prefix}/wo/kernel'])


def film_layer(x: Tensor, conditioning_emb: Tensor, kernel: Tensor) -> Tensor:
  """msd/layers.py:652-666: x * (scale + 1) + bias, always float32 there."""
  scale_bias = dense_general(conditioning_emb, kernel)
  scale, bias = torch.chunk(scale_bias, 2, dim=-1)
  return x * (scale + 1.0) + bias


def make_attention_mask(query_input: Tensor, key_input: Tensor) -> Tensor:
  """msd/layers.py:672-704 with multiply as pairwise fn -> [b,1,q,k]."""
  mask = query_input.unsqueeze(-1) * key_input.unsqueeze(-2)
  return mask.unsqueeze(-3)


def zero_activations_if_masked(y: Tensor, mask: Tensor) -> Tensor:
  """msd/layers.py:882-902."""
  is_not_empty = torch.any(mask.squeeze(1) == 1, dim=-1, keepdim=True)
  return y * is_not_empty.to(y.dtype)


def embed(ids: Tensor, embedding: Tensor) -> Tensor:
  """msd/layers.py:556-559 with one_hot=True: one_hot(ids) @ embedding, a gather in exact arithmetic.
  An id outside [0, vocab) matches no row of the one-hot and embeds as zeros."""
  ids = ids.long()
  valid = (ids >= 0) & (ids < embedding.shape[0])
  rows = embedding[torch.where(valid, ids, torch.zeros_like(ids))]
  return torch.where(valid.unsqueeze(-1), rows, torch.zeros_like(rows))


def sinusoidal_table(max_len: int, features: int, rng: np.random.Generator,
                     min_scale: float = 1.0, max_scale: float = 10000.0,
                     permute_bands: bool = True,
                     random_phase_offsets: bool = True) -> np.ndarray:
  """msd/layers.py:51-106 with numpy's rng standing in for jax.random.

  Position tables are checkpoint PARAMETERS in the reference
  (msd/models/diffusion/network.py:84-91); this is only used to synthesise
  plausible ones.
  """
  position = np.arange(0, max_len)[:, np.newaxis]
  scale_factor = -np.log(max_scale / min_scale) / (features // 2 - 1)
  div_term = min_scale * np.exp(np.arange(0, features // 2) * scale_factor)
  rads = position * div_term
  if random_phase_offsets:
    sin_offsets = rng.uniform(0, 2 * np.pi, [features // 2])
    cos_offsets = rng.uniform(0, 2 * np.pi, [features // 2])
  else:
    sin_offsets = 0.
    cos_offsets = 0.
  pe = np.zeros((max_len, features), dtype=np.float32)
  pe[:, :features // 2] = np.sin(rads + sin_offsets)
  pe[:, features // 2:2 * (features // 2)] = np.cos(rads + cos_offsets)
  if permute_bands:
    pe = pe[:, rng.permutation(features)]
  return pe.astype(np.float32)


# -----------------------------------------------------------------------------
# L2 network (msd/models/diffusion/network.py)
# -----------------------------------------------------------------------------
def get_sequence_length(sequence: Tensor) -> int:
  """msd/models/diffusion/network.py:28-39 (one row)."""
  seq = sequence.reshape(-1)
  zeros = (seq == 0).nonzero()
  length = int(zeros[0]) if zeros.numel() else 0
  if length == 0 and seq[0] != 0:
    length = seq.shape[0]
  return length


def encoder_layer(x: Tensor, inputs_mask: Tensor, p: Params, prefix: str,
                  cfg: OracleConfig) -> Tensor:
  """msd/models/diffusion/network.py:109-158."""
  inputs = x
  encoder_mask = make_attention_mask(inputs_mask, inputs_mask).to(x.dtype)
  h = layer_norm(inputs, p[f'{prefix}/pre_attention_layer_norm/scale'])
  h = multi_head_dot_product_attention(
      h, h, encoder_mask, p, f'{prefix}/attention', cfg.num_heads, cfg.head_dim)
  h = h + inputs
  y = layer_norm(h, p[f'{prefix}/pre_mlp_layer_norm/scale'])
  y = mlp_block(y, p, f'{prefix}/mlp', cfg.mlp_activations)
  return y + h


def token_encoder(tokens: Tensor, tokens_mask: Tensor, p: Params,
                  cfg: OracleConfig) -> Tensor:
  """msd/models/diffusion/network.py:261-303."""
  seq_length = tokens.shape[1]
  x = embed(tokens, p['token_encoder/token_embedder/embedding'])
  x = x + p['token_encoder/Embed_0/embedding'][:seq_length][None]
  for lyr in range(cfg.num_encoder_layers):
    x = encoder_layer(x, tokens_mask, p, f'token_encoder/layers_{lyr}', cfg)
  return layer_norm(x, p['token_encoder/encoder_norm/scale'])


def continuous_encoder(inputs: Tensor, inputs_mask: Tensor, p: Params,
                       cfg: OracleConfig) -> Tensor:
  """msd/models/diffusion/network.py:306-357."""
  b, max_positions, _ = inputs.shape
  x = dense_general(inputs, p['continuous_encoder/input_proj/kernel'])
  table = p['continuous_encoder/Embed_0/embedding']
  if cfg.context_positions == 'regular':
    pos = torch.arange(max_positions).expand(b, max_positions)
  elif cfg.context_positions == 'terminal_relative':
    rows = []
    for i in range(b):
      seq_len = get_sequence_length(inputs_mask[i])
      # network.py:42-51: jnp.roll(arange, seq_len)
      rows.append(torch.roll(torch.arange(max_positions), seq_len, 0))
    pos = torch.stack(rows)
  else:
    raise ValueError(cfg.context_positions)
  x = x + table[pos]
  for lyr in range(cfg.num_encoder_layers):
    x = encoder_layer(x, inputs_mask, p, f'continuous_encoder/layers_{lyr}', cfg)
  return layer_norm(x, p['continuous_encoder/encoder_norm/scale'])


def encode(p: Params, cfg: OracleConfig, input_tokens: Tensor,
           continuous_inputs: Tensor, continuous_mask: Tensor
           ) -> List[Tuple[Tensor, Tensor]]:
  """ContinuousContextTransformer.encode, network.py:537-559.

  `continuous_inputs` is already scaled to [-1, 1] (models.py:361-363).
  """
  dtype = continuous_inputs.dtype
  tokens_mask = (input_tokens > 0).to(dtype)
  tokens_encoded = token_encoder(input_tokens, tokens_mask, p, cfg)
  cmask = continuous_mask.to(dtype)
  continuous_encoded = continuous_encoder(continuous_inputs, cmask, p, cfg)
  return [(tokens_encoded, tokens_mask), (continuous_encoded, cmask)]


def get_timing_signal_1d(position: Tensor, num_channels: int,
                         min_timescale: float = 1.0,
                         max_timescale: float = 2.0e4) -> Tensor:
  """msd/models/diffusion/diffusion_utils.py:69-97."""
  num_timescales = float(num_channels // 2)
  log_timescale_increment = (
      np.log(max_timescale / min_timescale) / (num_timescales - 1.0))
  # reference builds the arange in float32 (line 90) then multiplies.
  inv_timescales = min_timescale * torch.exp(
      torch.arange(int(num_timescales), dtype=torch.float32).to(position.dtype)
      * -log_timescale_increment)
  scaled_time = position.unsqueeze(1) * inv_timescales.unsqueeze(0)
  return torch.cat([torch.sin(scaled_time), torch.cos(scaled_time)], dim=1)


def conditioning_embedding(time: Tensor, p: Params, cfg: OracleConfig) -> Tensor:
  """network.py:377-394 -> [batch, 1, 4*emb]."""
  c = get_timing_signal_1d(time * cfg.max_decoder_noise_time, cfg.emb_dim,
                           max_timescale=cfg.max_decoder_noise_time)
  c = swish(dense_general(c, p['decoder/time_emb_dense0/kernel']))
  c = swish(dense_general(c, p['decoder/time_emb_dense1/kernel']))
  return c.unsqueeze(1)


def decoder_layer(inputs: Tensor,
                  encodings_and_encdec_masks: List[Tuple[Tensor, Tensor]],
                  conditioning_emb: Tensor, p: Params, prefix: str,
                  cfg: OracleConfig) -> Tensor:
  """msd/models/diffusion/network.py:161-258."""
  x = layer_norm(inputs, p[f'{prefix}/pre_self_attention_layer_norm/scale'])
  x = film_layer(x, conditioning_emb,
                 p[f'{prefix}/FiLMLayer_0/DenseGeneral_0/kernel'])
  x = multi_head_dot_product_attention(
      x, x, None, p, f'{prefix}/self_attention', cfg.num_heads, cfg.head_dim)
  x = x + inputs

  y = layer_norm(x, p[f'{prefix}/pre_cross_attention_layer_norm/scale'])
  if cfg.decoder_cross_attend_style == 'sum_cross_attends':
    ys = []
    for n, (encoded, encdec_mask) in enumerate(encodings_and_encdec_masks):
      y_n = multi_head_dot_product_attention(
          y, encoded, encdec_mask, p,
          f'{prefix}/MultiHeadDotProductAttention_{n}',
          cfg.num_heads, cfg.head_dim)
      ys.append(zero_activations_if_masked(y_n, encdec_mask))
    y = sum(ys) + x
  elif cfg.decoder_cross_attend_style == 'concat_encodings':
    encoded = torch.cat([e for e, _ in encodings_and_encdec_masks], dim=1)
    encdec_mask = torch.cat([m for _, m in encodings_and_encdec_masks], dim=-1)
    y = multi_head_dot_product_attention(
        y, encoded, encdec_mask, p,
        f'{prefix}/MultiHeadDotProductAttention_0', cfg.num_heads, cfg.head_dim)
    y = zero_activations_if_masked(y, encdec_mask)
    y = y + x
  else:
    raise ValueError(cfg.decoder_cross_attend_style)

  z = layer_norm(y, p[f'{prefix}/pre_mlp_layer_norm/scale'])
  z = film_layer(z, conditioning_emb,
                 p[f'{prefix}/FiLMLayer_1/DenseGeneral_0/kernel'])
  z = mlp_block(z, p, f'{prefix}/mlp', cfg.mlp_activations)
  return z + y


def decode(p: Params, cfg: OracleConfig,
           encodings_and_masks: List[Tuple[Tensor, Tensor]],
           input_tokens: Tensor, noise_time: Tensor) -> Tensor:
  """ContinuousContextTransformer.decode -> Decoder.__call__,
  network.py:561-573, 360-457."""
  batch, seq_length, _ = input_tokens.shape
  assert noise_time.shape == (batch,)
  dtype = input_tokens.dtype
  conditioning_emb = conditioning_embedding(noise_time, p, cfg)
  position_encodings = p['decoder/Embed_0/embedding'][:seq_length][None]
  decoder_mask = torch.ones(batch, seq_length, dtype=dtype)
  encs = [(x, make_attention_mask(decoder_mask, m.to(dtype)))
          for x, m in encodings_and_masks]
  y = dense_general(input_tokens,
                    p['decoder/continuous_inputs_projection/kernel'])
  y = y + position_encodings
  for lyr in range(cfg.num_decoder_layers):
    y = decoder_layer(y, encs, conditioning_emb, p, f'decoder/layers_{lyr}', cfg)
  y = layer_norm(y, p['decoder/decoder_norm/scale'])
  return dense_general(y, p['decoder/spec_out_dense/kernel'])


# -----------------------------------------------------------------------------
# L3 sampler (msd/models/diffusion/diffusion_utils.py)
# -----------------------------------------------------------------------------
def get_logsnr_t(t, schedule: str = 'cosine', dtype=np.float32, start=None, stop=None,
                 num_steps=None):
  """diffusion_utils.py:166-202.  Cosine (181-187): a, b are float64 numpy scalars in the
  reference; `a*t+b` and the log/tan run in the array dtype (float32).  Linear (189-199):
  float64 table of log(alphas_cumprod) - log1p(-alphas_cumprod) clipped to [-20, 20], then
  `jnp.interp` over linspace(0, 1, num_steps) in the array dtype."""
  logsnr_min, logsnr_max = -20.0, 20.0
  t = np.asarray(t, dtype=dtype)
  if schedule == 'cosine':
    b = np.arctan(np.exp(-0.5 * logsnr_max))
    a = np.arctan(np.exp(-0.5 * logsnr_min)) - b
    arg = (dtype(a) * t + dtype(b)).astype(dtype)
    return (dtype(-2.0) * np.log(np.tan(arg))).astype(dtype)
  if schedule == 'linear':
    assert num_steps is not None and num_steps > 0 and start is not None and stop is not None
    betas = np.linspace(start, stop, num_steps, dtype=np.float64)
    alphas_cumprod = np.cumprod(1. - betas, axis=0)
    logsnr = np.log(alphas_cumprod) - np.log1p(-alphas_cumprod)
    logsnr = np.clip(logsnr, logsnr_min, logsnr_max)
    xp = np.linspace(0, 1, num_steps).astype(dtype)
    fp = logsnr.astype(dtype)
    # jnp.interp: i = clip(searchsorted(xp, x, 'right'), 1, n-1); f = fp[i-1] + (x-xp[i-1])/dx*df
    i = np.clip(np.searchsorted(xp, t, side='right'), 1, len(xp) - 1)
    df = fp[i] - fp[i - 1]
    dx = xp[i] - xp[i - 1]
    delta = t - xp[i - 1]
    f = np.where(dx == 0, fp[i], fp[i - 1] + (delta / np.where(dx == 0, dtype(1), dx)) * df)
    f = np.where(t < xp[0], fp[0], np.where(t > xp[-1], fp[-1], f))
    return f.astype(dtype)
  raise ValueError('Schedule %s not identified.' % schedule)


def sampler_logsnr(t, cfg: 'OracleConfig', dtype=np.float32):
  return get_logsnr_t(t, cfg.schedule, dtype, cfg.schedule_start, cfg.schedule_stop, cfg.num_steps)


def train_logsnr(t, cfg: 'OracleConfig', dtype=np.float32):
  return get_logsnr_t(t, cfg.train_schedule, dtype, cfg.train_schedule_start,
                      cfg.train_schedule_stop, cfg.train_schedule_num_steps)


def log1mexp(x: Tensor) -> Tensor:
  """diffusion_utils.py:100-106: log(1 - exp(-x)) for x > 0."""
  return torch.where(x > math.log(2.0), torch.log1p(-torch.exp(-x)), torch.log(-torch.expm1(-x)))


def predict_x0_from_v(z: Tensor, v: Tensor, logsnr: float) -> Tensor:
  """diffusion_utils.py:225-233: x0 = alpha z - sigma v."""
  ls = torch.tensor(logsnr, dtype=z.dtype)
  return torch.sqrt(torch.sigmoid(ls)) * z - torch.sqrt(torch.sigmoid(-ls)) * v


def x0_and_eps_from_model_output(z: Tensor, model_output: Tensor, logsnr: float,
                                 kind: str) -> Tuple[Tensor, Tensor]:
  """_get_x0_and_eps_from_model_output, diffusion_utils.py:288-321 (logsnr from the TRAIN
  schedule).  'x0_and_eps' splits a 2*n_dims output; the context network's spec_out_dense
  emits n_dims channels (network.py:452-456), so that branch cannot be reached on this path."""
  if kind == 'eps':
    return predict_x0_from_eps(z, model_output, logsnr), model_output
  if kind == 'x0':
    return model_output, predict_eps_from_x0(z, model_output, logsnr)
  if kind == 'v':
    x0 = predict_x0_from_v(z, model_output, logsnr)
    return x0, predict_eps_from_x0(z, x0, logsnr)
  raise ValueError('Unknown model_output: %s' % kind)


def predict_x0_from_eps(z: Tensor, eps: Tensor, logsnr: float) -> Tensor:
  """diffusion_utils.py:215-222."""
  ls = torch.tensor(logsnr, dtype=z.dtype)
  return torch.sqrt(1.0 + torch.exp(-ls)) * (
      z - eps * torch.rsqrt(1.0 + torch.exp(ls)))


def predict_eps_from_x0(z: Tensor, x0: Tensor, logsnr: float) -> Tensor:
  """diffusion_utils.py:205-212."""
  ls = torch.tensor(logsnr, dtype=z.dtype)
  return torch.sqrt(1.0 + torch.exp(ls)) * (
      z - x0 * torch.rsqrt(1.0 + torch.exp(-ls)))


def diffusion_reverse(x0: Tensor, z_t: Tensor, logsnr_s: float, logsnr_t: float,
                      logvar_type: str) -> Dict[str, Tensor]:
  """diffusion_utils.py:120-163."""
  dt = z_t.dtype
  ls = torch.tensor(logsnr_s, dtype=dt)
  lt = torch.tensor(logsnr_t, dtype=dt)
  alpha_st = torch.sqrt((1. + torch.exp(-lt)) / (1. + torch.exp(-ls)))
  alpha_s = torch.sqrt(torch.sigmoid(ls))
  r = torch.exp(lt - ls)
  one_minus_r = -torch.expm1(lt - ls)
  mean = r * alpha_st * z_t + one_minus_r * alpha_s * x0
  if logvar_type == 'small':
    var = one_minus_r * torch.sigmoid(-ls)
  elif logvar_type == 'large':
    var = one_minus_r * torch.sigmoid(-lt)
  elif logvar_type.startswith('medium:'):
    frac = float(logvar_type.split(':')[1])
    assert 0 <= frac <= 1
    log_one_minus_r = log1mexp(ls - lt)
    min_logvar = log_one_minus_r + torch.nn.functional.logsigmoid(-ls)
    max_logvar = log_one_minus_r + torch.nn.functional.logsigmoid(-lt)
    var = torch.exp(frac * max_logvar + (1 - frac) * min_logvar)
  else:
    raise ValueError('unknown logvar_type %s' % logvar_type)
  return {'mean': mean, 'std': torch.sqrt(var), 'var': var}


def sampler_coefficients(i: int, num_steps: int, dtype=np.float64) -> Dict[str, float]:
  """Scalars of one reverse step (SURVEY App. A.4), in `dtype` arithmetic.

  Used for the known-answer test and to cross-check the CUDA step table.
  """
  t = dtype(i + 1.0) / dtype(num_steps)
  s = dtype(i) / dtype(num_steps)
  lt = dtype(get_logsnr_t(t, dtype=dtype))
  ls = dtype(get_logsnr_t(s, dtype=dtype))
  sig = lambda v: dtype(1.0) / (dtype(1.0) + np.exp(-v))
  alpha_st = np.sqrt((1. + np.exp(-lt)) / (1. + np.exp(-ls)))
  alpha_s = np.sqrt(sig(ls))
  r = np.exp(lt - ls)
  one_minus_r = -np.expm1(lt - ls)
  return {
      't': float(t), 'logsnr_t': float(lt), 'logsnr_s': float(ls),
      'c_z': float(r * alpha_st), 'c_x0': float(one_minus_r * alpha_s),
      'sigma': float(np.sqrt(one_minus_r * sig(-lt))),
      'x0_scale': float(np.sqrt(1. + np.exp(-lt))),
      'eps_scale': float(1.0 / np.sqrt(1. + np.exp(lt))),
  }


PredFn = Callable[[Tensor, Tensor, bool], Tensor]


def eval_step(z_t: Tensor, i: int, noise_i: Optional[Tensor], pred_fn: PredFn,
              cfg: OracleConfig) -> Tensor:
  """One reverse step, diffusion_utils.py:398-453 (body)."""
  f32 = np.float32
  t = f32(i + 1.0) / f32(cfg.num_steps)
  s = f32(i) / f32(cfg.num_steps)
  logsnr_t = float(sampler_logsnr(t, cfg))
  logsnr_s = float(sampler_logsnr(s, cfg))
  batch = z_t.shape[0]
  time = torch.full((batch,), float(t), dtype=z_t.dtype)

  # _get_x0_and_eps_from_model_output (288-321) uses the TRAIN schedule.
  logsnr_train = float(train_logsnr(t, cfg))
  pred_x0, pred_eps = x0_and_eps_from_model_output(z_t, pred_fn(z_t, time, True), logsnr_train,
                                                   cfg.model_output)
  if cfg.eval_condition_weight != 1:
    cond_wt = cfg.eval_condition_weight
    uncond_wt = 1. - cond_wt
    _, uncond_eps = x0_and_eps_from_model_output(z_t, pred_fn(z_t, time, False), logsnr_train,
                                                 cfg.model_output)
    pred_eps = cond_wt * pred_eps + uncond_wt * uncond_eps
    pred_x0 = predict_x0_from_eps(z_t, pred_eps, logsnr_t)
  if cfg.clip_x0:
    pred_x0 = torch.clamp(pred_x0, -1.0, 1.0)
    pred_eps = predict_eps_from_x0(z_t, pred_x0, logsnr_t)
  if cfg.sampler == 'ddim':
    # diffusion_utils.py:369-379
    ls = torch.tensor(logsnr_s, dtype=z_t.dtype)
    z_s = (torch.sqrt(torch.sigmoid(ls)) * pred_x0 +
           torch.sqrt(torch.sigmoid(-ls)) * pred_eps)
    return pred_x0 if i == 0 else z_s
  if cfg.sampler != 'ddpm':
    raise ValueError(cfg.sampler)
  # ddpm_step, diffusion_utils.py:382-395
  if i == 0:
    return pred_x0
  dist = diffusion_reverse(pred_x0, z_t, logsnr_s, logsnr_t, cfg.logvar_type)
  return dist['mean'] + dist['std'] * noise_i


def eval_scan(init_z: Tensor, noise: Optional[Tensor], pred_fn: PredFn,
              cfg: OracleConfig, trajectory: Optional[list] = None) -> Tensor:
  """diffusion_utils.py:456-476 with the RNG replaced by explicit tensors.

  `noise[i]` is the N(0,1) draw the reference takes from fold_in(rng, i) at
  step i (i = num_steps-1 .. 1; noise[0] is never used).  `noise` may also be
  a callable i -> tensor (lets long runs generate the draws on the fly).
  """
  z = init_z
  for i in range(cfg.num_steps - 1, -1, -1):
    if noise is None or i == 0:
      noise_i = None
    else:
      noise_i = noise(i) if callable(noise) else noise[i]
    z = eval_step(z, i, noise_i, pred_fn, cfg)
    if trajectory is not None:
      trajectory.append(z.clone())
  return z


# -----------------------------------------------------------------------------
# L4 model wrapper (msd/models/diffusion/models.py) + codec scaling
# -----------------------------------------------------------------------------
def scale_features(features: Tensor, cfg: OracleConfig,
                   output_range=(-1.0, 1.0), clip: bool = False) -> Tensor:
  """msd/audio_codecs.py:166-174."""
  min_out, max_out = output_range
  if clip:
    features = torch.clamp(features, cfg.min_value, cfg.max_value)
  zero_one = (features - cfg.min_value) / (cfg.max_value - cfg.min_value)
  return zero_one * (max_out - min_out) + min_out


def scale_to_features(outputs: Tensor, cfg: OracleConfig,
                      input_range=(-1.0, 1.0), clip: bool = False) -> Tensor:
  """msd/audio_codecs.py:176-183."""
  min_out, max_out = input_range
  if clip:
    outputs = torch.clamp(outputs, min_out, max_out)
  zero_one = (outputs - min_out) / (max_out - min_out)
  return zero_one * (cfg.max_value - cfg.min_value) + cfg.min_value


def predict_batch_with_aux(p: Params, cfg: OracleConfig, batch: Dict[str, Tensor],
                           init_z: Tensor, noise: Optional[Tensor],
                           trajectory: Optional[list] = None
                           ) -> Tuple[Tensor, Tensor]:
  """ContextDiffusionModel.predict_batch_with_aux, models.py:340-400,
  with explicit `init_z` / `noise` instead of the jax rng."""
  dtype = init_z.dtype
  ctx = scale_features(batch['encoder_continuous_inputs'].to(dtype), cfg,
                       clip=True)
  encodings_and_masks = encode(p, cfg, batch['encoder_input_tokens'], ctx,
                               batch['encoder_continuous_mask'])

  def pred_fn(z: Tensor, time: Tensor, include_conditioning: bool) -> Tensor:
    flag = 1.0 if include_conditioning else 0.0
    # models.py:376-377: encodings AND masks are multiplied by the flag.
    step_encs = [(e * flag, m * flag) for e, m in encodings_and_masks]
    return decode(p, cfg, step_encs, z, time)

  pred_x0 = eval_scan(init_z, noise, pred_fn, cfg, trajectory)
  decodes = scale_to_features(pred_x0, cfg)
  scores = torch.zeros(init_z.shape[0], dtype=dtype)
  return decodes, scores


def params_to(p: Dict[str, np.ndarray], dtype=torch.float32) -> Params:
  """numpy param dict -> torch-CPU tensors of `dtype`."""
  return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dtype)
          for k, v in p.items()}
