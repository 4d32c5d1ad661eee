"""Multi-GPU drivers: one process per GPU (torch.distributed), no collective inside the
diffusion loop.

Two partitionings of the reference's serve path (SURVEY §8e):
  * independent segments (BASELINE configs 3-4): `predict_sharded` gives each rank a contiguous
    block of segments; weights are replicated; the only communication is the final gather.
  * one song (config 5): segment k+1's context is segment k's FINAL mel
    (msd/beam/evaluation.py:179-223, colab ipynb:895-935), so the chain is strictly serial.
    `synthesize_song` relays the chain round-robin over the ranks and hands the 128 KB mel
    GPU-to-GPU with send/recv (NCCL over NVLink on an H100 box, gloo in the CPU tests) instead of
    through host numpy; it does not (cannot) make one song faster than one GPU's batch-1 speed,
    it removes the host round trip and frees the other ranks for other songs.
  * one song, faster (config 5, SURVEY 8e-iii): `CfgSplitPair` runs the conditional decoder pass
    of every reverse step on one GPU and the unconditional pass on a second one; the two sampler
    kernels swap their 128 KB of predicted noise per step by direct NVLink stores + a flag word
    (msd_p2p_*: no NCCL call inside the loop) and apply the identical update, so both ranks hold
    the same mel and the chain needs no hand-off at all.  torch.distributed only carries the two
    64-byte IPC handles at set-up.
The functions take a `predict_fn(tokens, ctx, ctx_mask, seed) -> mel` so the protocol is
testable on CPU with gloo and a stand-in predict function.
"""

from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

PredictFn = Callable[[torch.Tensor, torch.Tensor, torch.Tensor, int], torch.Tensor]


def shard_range(n_items: int, world: int, rank: int) -> Tuple[int, int]:
  """Contiguous block [lo, hi) of `n_items` for `rank`; sizes differ by at most one."""
  base, rem = divmod(n_items, world)
  lo = rank * base + min(rank, rem)
  return lo, lo + base + (1 if rank < rem else 0)


def predict_sharded(predict_fn: PredictFn, tokens: torch.Tensor, ctx: torch.Tensor,
                    ctx_mask: torch.Tensor, seed: int = 0,
                    group: Optional[dist.ProcessGroup] = None) -> torch.Tensor:
  """Every rank holds the full batch description; rank r computes its block and all ranks
  receive the full [n_segments, frames, n_dims] result (all_gather of equal-padded blocks)."""
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  rank = dist.get_rank(group) if dist.is_initialized() else 0
  n = tokens.shape[0]
  lo, hi = shard_range(n, world, rank)
  if hi > lo:
    # NOTE: the noise of a batch is one jax.random draw over the whole [b, frames, dims] block
    # (diffusion_utils.py:462), so the result depends on how segments are grouped into calls; the
    # same seed is used for every block, like a reference run at that per-host batch size.
    mine = predict_fn(tokens[lo:hi], ctx[lo:hi], ctx_mask[lo:hi], seed)
  else:
    mine = None
  if world == 1:
    return mine
  per = (n + world - 1) // world
  ref = mine if mine is not None else None
  shape_tail = tuple(ctx.shape[1:]) if ref is None else tuple(ref.shape[1:])
  device = ctx.device if ref is None else ref.device
  pad = torch.zeros((per,) + shape_tail, dtype=torch.float32, device=device)
  if mine is not None:
    pad[:hi - lo] = mine
  out = [torch.empty_like(pad) for _ in range(world)]
  dist.all_gather(out, pad, group=group)
  parts = []
  for r in range(world):
    a, b = shard_range(n, world, r)
    parts.append(out[r][:b - a])
  return torch.cat(parts, dim=0)


def synthesize_song(predict_fn: PredictFn, token_segments: Sequence[torch.Tensor],
                    context_frames: int, n_dims: int, device: torch.device, seed: int = 0,
                    always_mask_context: bool = False,
                    group: Optional[dist.ProcessGroup] = None) -> Optional[torch.Tensor]:
  """Chained synthesis of one song, segments relayed round-robin over the ranks.

  Mirrors InferSong.process (msd/beam/evaluation.py:156-223): the first segment runs with an
  all-zero context mask, every later one with the previous prediction as context and an all-one
  mask.  Returns the concatenated mel [1, n_segments * frames, n_dims] on rank 0, None elsewhere.
  """
  world = dist.get_world_size(group) if dist.is_initialized() else 1
  rank = dist.get_rank(group) if dist.is_initialized() else 0
  n_seg = len(token_segments)
  prev = torch.zeros(1, context_frames, n_dims, dtype=torch.float32, device=device)
  mine: List[Tuple[int, torch.Tensor]] = []
  for k in range(n_seg):
    owner = k % world
    if owner == rank:
      if k > 0 and world > 1:
        dist.recv(prev, src=(k - 1) % world, group=group)
      first = (k == 0) or always_mask_context
      mask = torch.zeros(1, context_frames, dtype=torch.int32, device=device) if first else \
          torch.ones(1, context_frames, dtype=torch.int32, device=device)
      toks = token_segments[k].to(device).reshape(1, -1)
      # one constant seed for every segment, as beam/evaluation.py:209 (`predict(batch)`, i.e.
      # seed 0 each time) and song.synthesize_song do: the relay is the same song on any world size
      pred = predict_fn(toks, prev, mask, seed)
      mine.append((k, pred))
      prev = pred[:1].clone()  # own buffer: later recv()s must not overwrite a stored result
      if k + 1 < n_seg and world > 1:
        dist.send(prev, dst=(k + 1) % world, group=group)
  if world == 1:
    return torch.cat([p for _, p in mine], dim=1)
  # gather on rank 0 in segment order
  if rank == 0:
    out: List[Optional[torch.Tensor]] = [None] * n_seg
    for k, p in mine:
      out[k] = p
    for k in range(n_seg):
      if k % world != 0:
        buf = torch.empty_like(mine[0][1])
        dist.recv(buf, src=k % world, group=group)
        out[k] = buf
    return torch.cat(out, dim=1)
  for k, p in mine:
    dist.send(p.contiguous(), dst=0, group=group)
  return None


class CfgSplitPair:
  """Ranks `cond_rank` and `uncond_rank` of `group` share every reverse step of their (identical)
  predict calls: one runs the conditional decoder pass, the other the unconditional one, and the
  sampler kernels exchange the predicted noise GPU-to-GPU (engine.Engine.p2p_*).  Use as a context
  manager around the chained-song loop; other ranks of the group are not involved."""

  def __init__(self, model, cond_rank: int = 0, uncond_rank: int = 1,
               group: Optional[dist.ProcessGroup] = None):
    self.model, self.group = model, group
    self.rank = dist.get_rank(group)
    self.cond_rank, self.uncond_rank = cond_rank, uncond_rank
    self.active = self.rank in (cond_rank, uncond_rank)

  def __enter__(self):
    handles: List[Optional[bytes]] = [None] * dist.get_world_size(self.group)
    mine = self.model.engine.p2p_export() if self.active else b''
    dist.all_gather_object(handles, mine, group=self.group)
    if self.active:
      peer = self.uncond_rank if self.rank == self.cond_rank else self.cond_rank
      self.model.engine.p2p_attach(handles[peer], 'cond' if self.rank == self.cond_rank else 'uncond')
    dist.barrier(group=self.group)   # nobody samples before both sides are attached
    return self

  def __exit__(self, *exc):
    if self.active:
      torch.cuda.synchronize(self.model.engine.device)
    dist.barrier(group=self.group)   # both sides are done with each other's buffer
    if self.active:
      self.model.engine.p2p_detach()
    return False


def synthesize_song_cfg_split(model, token_segments: Sequence[torch.Tensor], context_frames: int,
                              n_dims: int, seed: int = 0, always_mask_context: bool = False,
                              group: Optional[dist.ProcessGroup] = None,
                              timings: Optional[List[float]] = None) -> Optional[torch.Tensor]:
  """One chained song (InferSong.process, beam/evaluation.py:156-223) on ranks 0 and 1 of `group`
  with the guidance split; every other rank returns None at once.  Both participating ranks
  return the full mel [1, n_segments * frames, n_dims] (they compute identical copies).  When
  `timings` is given, the wall seconds of every segment but the first are appended (the
  reference's model_timing protocol, evaluation.py:217-220)."""
  import time
  rank = dist.get_rank(group)
  with CfgSplitPair(model, 0, 1, group) as pair:
    if not pair.active:
      return None
    device = model.engine.device
    prev = torch.zeros(1, context_frames, n_dims, dtype=torch.float32, device=device)
    outs = []
    for k, toks in enumerate(token_segments):
      first = (k == 0) or always_mask_context
      mask = (torch.zeros if first else torch.ones)(1, context_frames, dtype=torch.int32, device=device)
      torch.cuda.synchronize(device)
      tick = time.time()
      pred = model.predict_on_device(toks.to(device).reshape(1, -1), prev, mask, seed)
      torch.cuda.synchronize(device)
      if timings is not None and k > 0:
        timings.append(time.time() - tick)
      outs.append(pred)
      prev = pred[:1]
    return torch.cat(outs, dim=1)
