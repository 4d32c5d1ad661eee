"""CPU restatement of the reference's no-context diffusion model, on top of oracle/msd_oracle.py.

    DiffusionModel.predict_batch_with_aux     msd/models/diffusion/models.py:149-205
      -> Transformer.encode / .decode         msd/models/diffusion/network.py:470-496
      -> eval_scan (DDPM)

Transformer has the same Decoder as ContinuousContextTransformer and a TokenEncoder named
`encoder` (network.py:460-468); there is no continuous encoder and no context scaling.  Like the
oracle, this is test infrastructure: the graph as written, fp32 by default, fp64 on request.
"""

from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from oracle import msd_oracle as O

Tensor = torch.Tensor


def token_encoder(tokens: Tensor, tokens_mask: Tensor, p: O.Params, cfg: O.OracleConfig,
                  prefix: str = 'encoder') -> Tensor:
  """TokenEncoder (network.py:261-303) under `prefix`."""
  seq_length = tokens.shape[1]
  x = O.embed(tokens, p[f'{prefix}/token_embedder/embedding'])
  x = x + p[f'{prefix}/Embed_0/embedding'][:seq_length][None]
  for lyr in range(cfg.num_encoder_layers):
    x = O.encoder_layer(x, tokens_mask, p, f'{prefix}/layers_{lyr}', cfg)
  return O.layer_norm(x, p[f'{prefix}/encoder_norm/scale'])


def encode(p: O.Params, cfg: O.OracleConfig, input_tokens: Tensor,
           dtype: torch.dtype = torch.float32) -> List[Tuple[Tensor, Tensor]]:
  """Transformer.encode, network.py:470-482: one (encodings, mask) source."""
  tokens_mask = (input_tokens > 0).to(dtype)
  return [(token_encoder(input_tokens, tokens_mask, p, cfg), tokens_mask)]


def predict_batch_with_aux(p: O.Params, cfg: O.OracleConfig, batch: Dict[str, Tensor],
                           init_z: Tensor, noise: Optional[Tensor],
                           trajectory: Optional[list] = None) -> Tuple[Tensor, Tensor]:
  """DiffusionModel.predict_batch_with_aux, models.py:149-205, with explicit `init_z` / `noise`
  instead of the jax rng.  Reads batch['encoder_input_tokens'] only."""
  dtype = init_z.dtype
  encodings_and_masks = encode(p, cfg, batch['encoder_input_tokens'], dtype)

  def pred_fn(z: Tensor, time: Tensor, include_conditioning: bool) -> Tensor:
    flag = 1.0 if include_conditioning else 0.0
    # models.py:181-182: encodings AND masks are multiplied by the flag
    step_encs = [(e * flag, m * flag) for e, m in encodings_and_masks]
    return O.decode(p, cfg, step_encs, z, time)

  pred_x0 = O.eval_scan(init_z, noise, pred_fn, cfg, trajectory)
  return O.scale_to_features(pred_x0, cfg), torch.zeros(init_z.shape[0], dtype=dtype)


def as_context_tree(params: Dict, context_params: Dict) -> Dict:
  """The no-context tree `params` as a ContinuousContextTransformer tree: the token encoder
  renamed `token_encoder/`, the continuous encoder (and, for sum_cross_attends, the
  `MultiHeadDotProductAttention_1` kernels) taken from `context_params`, every other weight
  shared."""
  out = {('token_' + k if k.startswith('encoder/') else k): v for k, v in params.items()}
  for k, v in context_params.items():
    if k not in out:
      out[k] = v
  return out
