"""Drop-in for `music_spectrogram_diffusion.inference` (msd/inference.py) on the CUDA engine.

Keeps the reference's call surface:
  parse_training_gin_file(gin_file, gin_bindings) -> str          inference.py:32-65
  InferenceModel(checkpoint_path, gin_config, batch_size=1)       inference.py:68-111
    .sequence_length / .inputs_length / .targets_length / .targets_context_length
    .audio_codec / .codec / .model.FEATURE_CONVERTER_CLS / .batch_size / .partitioner
    .input_shapes / .input_types                                   inference.py:113-157
    .predict(batch, seed=0) -> (pred_mel f32 [B, targets, n_dims], scores f32 [B])   200-203
and replaces the jitted `predict_batch_with_aux` with libmsd_b200.so (ctypes; torch only
allocates device/pinned buffers).  There is no CPU fallback.

Both diffusion model families of the reference run: `models.ContextDiffusionModel` +
`network.ContinuousContextTransformer` (TASK_FEATURE_LENGTHS with `targets_context`, the
gin/models/diffusion/context configs) and the no-context `models.DiffusionModel` +
`network.Transformer` (lengths without `targets_context`, gin/models/diffusion/basic).  As in the
reference, the lengths decide which inputs the model takes (inference.py:113-157).

Checkpoints: `checkpoint_path` may be a T5X checkpoint directory such as
`.../base_with_context/checkpoint_500000` (msgpack index + one zarr array per parameter, read by
`t5x_checkpoint.py` without t5x/tensorstore), an `.npz` written by `weights.save_npz` (flax
names, fp32) or `synthetic:<seed>` (random init; no pretrained checkpoint is available offline).

Noise: with `rng='jax'` (default) `seed` means what it means in the reference -- init_z =
normal(PRNGKey(seed)), step noise = normal(fold_in(key, i)) -- drawn on the GPU from a restated
jax.random threefry2x32 stream (`jax_rng.py`: pinned on the Random123 vectors and the values the
JAX docs print for PRNGKey(0); the fold_in composition is unverified offline).  `rng='philox'`
selects the library's own Philox4x32-10 stream (restated in oracle/philox.py).  Parity runs can
also inject noise through `predict(..., init_z=, noise=)`.
"""

from __future__ import annotations

import dataclasses
import math
import os
from typing import Any, Dict, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch

from music_spectrogram_diffusion_b200 import (audio_codecs, config, engine, gin_lite, midi_tokens,
                                              t5x_checkpoint, weights)

_GIN_SEARCH_ROOTS = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]


def parse_training_gin_file(gin_file: str, gin_bindings: Sequence[str]) -> str:
  """Read a training `config.gin` and append override bindings (inference.py:32-65).

  The reference rewrites the `__main__` import for gin's dynamic registration; imports are
  irrelevant to gin_lite, so the text is passed through with the bindings appended.
  """
  with open(gin_file) as f:
    cfg = f.read()
  return cfg + '\n' + '\n'.join(gin_bindings) + '\n'


# ---- minimal stand-ins for objects callers poke at --------------------------------------
class _NoContextFeatureConverterSpec:
  """Batch-dict schema of ContinuousOutpusEncDecFeatureConverter (msd/feature_converters.py:23-39),
  the feature converter of the no-context DiffusionModel (models.py:38)."""
  TASK_FEATURES = {'inputs': np.int32, 'targets': np.float32}
  MODEL_FEATURES = {
      'encoder_input_tokens': np.int32,
      'decoder_target_tokens': np.float32,
      'decoder_input_tokens': np.float32,
      'decoder_target_mask': np.bool_,
  }


class _FeatureConverterSpec:
  """Batch-dict schema of ContinuousContextFeatureConverter
  (msd/models/diffusion/feature_converters.py:26-43)."""
  TASK_FEATURES = {'inputs': np.int32, 'targets': np.float32, 'targets_context': np.float32}
  MODEL_FEATURES = {
      'encoder_input_tokens': np.int32,
      'encoder_continuous_inputs': np.float32,
      'encoder_continuous_mask': np.bool_,
      'decoder_target_tokens': np.float32,
      'decoder_target_mask': np.bool_,
  }


@dataclasses.dataclass
class _Model:
  """What callers read off `InferenceModel.model` (models.py:208-221)."""
  module_config: config.T5Config
  diffusion_config: config.DiffusionConfig
  audio_codec: audio_codecs.AudioCodec
  FEATURE_CONVERTER_CLS: Any = _FeatureConverterSpec


class _Partitioner:
  """The colab monkey-patches `.partitioner.partition` (ipynb:233-247); keep it harmless."""

  def partition(self, fn, *args, **kwargs):
    return fn


def build_codec(num_velocity_bins: int = 127, steps_per_second: int = 100,
                max_shift_seconds: int = 10) -> midi_tokens.EventVocabulary:
  """vocabularies.build_codec (msd/vocabularies.py:118-144): the event codec of a
  VocabularyConfig -- shift [0, max], pitch 128, velocity [0, bins], tie 1, program 128, drum 128.
  The same object `midi_tokens` tokenises with (one vocabulary implementation, not two)."""
  return midi_tokens.mt3_event_vocabulary(midi_tokens.VocabularyConfig(
      steps_per_second=steps_per_second, max_shift_seconds=max_shift_seconds,
      num_velocity_bins=num_velocity_bins))


def num_embeddings(codec: midi_tokens.EventVocabulary, extra_ids: int = 100) -> int:
  """vocabularies.num_embeddings (279-281): 3 specials + classes + extra ids, up to k*128."""
  vocab_size = 3 + codec.num_classes + extra_ids
  return 128 * math.ceil(vocab_size / 128)


# MODEL macro -> whether the model takes a context (TASK_FEATURE_LENGTHS has `targets_context`)
_DIFFUSION_MODELS = {'DiffusionModel': False, 'ContextDiffusionModel': True}


def _check_model_lengths(model: Any, lengths: Mapping[str, int]) -> None:
  """models.DiffusionModel runs without a context and models.ContextDiffusionModel with one; the
  task's lengths must say the same (the reference fails later, inside its feature converter)."""
  if not isinstance(model, gin_lite.ConfigurableRef):
    return
  name = model.name.rsplit('.', 1)[-1]
  if name not in _DIFFUSION_MODELS:
    return
  with_context = 'targets_context' in lengths
  if _DIFFUSION_MODELS[name] != with_context:
    raise ValueError(
        f'MODEL = @{model.name}() needs TASK_FEATURE_LENGTHS '
        f'{"with" if _DIFFUSION_MODELS[name] else "without"} targets_context, got {dict(lengths)}: '
        'models.ContextDiffusionModel takes inputs, targets and targets_context, '
        'models.DiffusionModel inputs and targets only')


def _build_from_gin(gin_config: str) -> Tuple[config.T5Config, config.DiffusionConfig,
                                              Dict[str, int], midi_tokens.EventVocabulary]:
  g = gin_lite.parse_config(gin_config, _GIN_SEARCH_ROOTS)
  lengths = dict(g.query_macro('TASK_FEATURE_LENGTHS'))
  _check_model_lengths(g.macros.get('MODEL'), lengths)

  vb = g.bindings_for('vocabularies.VocabularyConfig')
  kw = {}
  for name in ('num_velocity_bins', 'steps_per_second', 'max_shift_seconds'):
    if name in vb:
      kw[name] = int(g.resolve(vb[name]))
  codec = build_codec(**kw)

  t5 = config.T5Config()
  for k, v in g.bindings_for('network.T5Config').items():
    v = g.resolve(v)
    if isinstance(v, gin_lite.ConfigurableRef):
      if v.name.endswith('num_embeddings'):
        v = num_embeddings(codec)
      else:
        raise ValueError(f'unsupported reference {v!r} for T5Config.{k}')
    if not hasattr(t5, k):
      raise ValueError(f'network.T5Config has no field {k!r}')
    setattr(t5, k, tuple(v) if isinstance(v, list) else v)

  def schedule(scope: str) -> config.DiffusionSchedule:
    s = config.DiffusionSchedule()
    for k, v in g.bindings_for('diffusion_utils.DiffusionSchedule', scope).items():
      setattr(s, k, g.resolve(v))
    return s

  diff = config.DiffusionConfig()
  cfgc = config.ClassifierFreeGuidanceConfig()
  for k, v in g.bindings_for('diffusion_utils.ClassifierFreeGuidanceConfig').items():
    setattr(cfgc, k, g.resolve(v))
  diff.classifier_free_guidance = cfgc
  samp = config.SamplerConfig()
  for k, v in g.bindings_for('diffusion_utils.SamplerConfig').items():
    v = g.resolve(v)
    if isinstance(v, gin_lite.ConfigurableRef):
      v = schedule(v.scope)
    setattr(samp, k, v)
  diff.sampler = samp
  for k, v in g.bindings_for('diffusion_utils.DiffusionConfig').items():
    v = g.resolve(v)
    if isinstance(v, gin_lite.ConfigurableRef):
      if k == 'train_schedule':
        v = schedule(v.scope)
      elif k == 'sampler':
        v = samp
      elif k == 'classifier_free_guidance':
        v = cfgc
    setattr(diff, k, v)
  if diff.sampler.schedule.num_steps is None:
    diff.sampler.schedule.num_steps = 1000
  return t5, diff, lengths, codec


class InferenceModel:
  """Wrapper of the CUDA engine with the reference's `InferenceModel` surface."""

  def __init__(self, checkpoint_path: str, gin_config: str, batch_size: int = 1,
               device: int = 0, rng: str = 'jax', precision: str = 'bf16'):
    t5, diff, lengths, codec = _build_from_gin(gin_config)
    self._init_common(checkpoint_path, t5, diff, lengths, codec, batch_size, device, rng=rng,
                      precision=precision)

  @classmethod
  def from_config(cls, t5: config.T5Config, diffusion: config.DiffusionConfig,
                  sequence_length: Mapping[str, int], checkpoint_path: str = 'synthetic:0',
                  batch_size: int = 1, device: int = 0,
                  params: Optional[Dict[str, np.ndarray]] = None,
                  rng: str = 'jax', precision: str = 'bf16') -> 'InferenceModel':
    self = cls.__new__(cls)
    self._init_common(checkpoint_path, t5, diffusion, dict(sequence_length), build_codec(),
                      batch_size, device, params, rng, precision)
    return self

  def _init_common(self, checkpoint_path, t5, diff, lengths, codec, batch_size, device,
                   params=None, rng='jax', precision='bf16'):
    if rng not in ('jax', 'philox'):
      raise ValueError(f'unknown rng {rng!r}')
    if precision not in engine.PRECISIONS:
      raise ValueError(f'unknown precision {precision!r}')
    self.rng = rng
    self.precision = precision
    self.checkpoint_path = checkpoint_path
    self.batch_size = batch_size
    self.partitioner = _Partitioner()
    self.sequence_length = lengths
    self.inputs_length = lengths['inputs']
    self.targets_length = lengths['targets']
    # None: the no-context DiffusionModel (network.Transformer), as in the reference
    self.targets_context_length = lengths.get('targets_context', None)
    self.audio_codec = audio_codecs.MelGAN()
    self.codec = codec
    self.model = _Model(t5, diff, self.audio_codec)
    if self.targets_context_length is None:
      self.model.FEATURE_CONVERTER_CLS = _NoContextFeatureConverterSpec
    self._engine: Optional[engine.Engine] = None
    self._device_index = device
    self._params = params
    self._pinned: Dict[str, torch.Tensor] = {}
    self._dev: Dict[str, torch.Tensor] = {}

  # ---- reference properties ---------------------------------------------------
  @property
  def has_context(self) -> bool:
    """Whether the model takes a context (ContextDiffusionModel) or not (DiffusionModel)."""
    return self.targets_context_length is not None

  @property
  def input_shapes(self):
    shapes = {
        'encoder_input_tokens': (self.batch_size, self.inputs_length),
        'decoder_target_tokens': (self.batch_size, self.targets_length, self.audio_codec.n_dims),
    }
    if self.has_context:
      shapes.update({
          'encoder_continuous_inputs':
              (self.batch_size, self.targets_context_length, self.audio_codec.n_dims),
          'encoder_continuous_mask': (self.batch_size, self.targets_context_length),
      })
    if 'decoder_input_tokens' in self.model.FEATURE_CONVERTER_CLS.MODEL_FEATURES:
      shapes['decoder_input_tokens'] = shapes['decoder_target_tokens']
    return shapes

  @property
  def input_types(self):
    types = {
        'encoder_input_tokens': np.int32,
        'decoder_target_tokens': np.float32,
    }
    if self.has_context:
      types.update({
          'encoder_continuous_inputs': np.float32,
          'encoder_continuous_mask': np.int32,
      })
    if 'decoder_input_tokens' in self.model.FEATURE_CONVERTER_CLS.MODEL_FEATURES:
      types['decoder_input_tokens'] = types['decoder_target_tokens']
    return types

  def _encoder_inputs(self):
    """The batch keys the engine's encode reads."""
    return ('encoder_input_tokens', 'encoder_continuous_inputs',
            'encoder_continuous_mask') if self.has_context else ('encoder_input_tokens',)

  @property
  def step(self):
    return 0

  # ---- engine -------------------------------------------------------------------
  def _restore_from_checkpoint(self) -> Dict[str, np.ndarray]:
    if self._params is not None:
      return self._params
    cp = self.checkpoint_path
    if cp.startswith('synthetic:'):
      return weights.synthetic_params(self.model.module_config, self.inputs_length,
                                      self.targets_length, self.targets_context_length,
                                      self.audio_codec.n_dims, seed=int(cp.split(':', 1)[1]))
    if cp.endswith('.npz'):
      return weights.load_npz(cp)
    if t5x_checkpoint.is_t5x_checkpoint(cp):
      params = t5x_checkpoint.load_t5x_checkpoint(cp)
      weights.check_params(params, self.model.module_config, self.inputs_length,
                           self.targets_length, self.targets_context_length,
                           self.audio_codec.n_dims)
      return params
    raise FileNotFoundError(
        f'checkpoint {cp!r}: expected a T5X checkpoint directory, an .npz (weights.save_npz) '
        'or synthetic:<seed>')

  def _get_engine(self) -> engine.Engine:
    if self._engine is None:
      cfg = engine.make_msd_config(
          self.model.module_config, self.model.diffusion_config, self.inputs_length,
          self.targets_length, self.targets_context_length, self.batch_size,
          self.audio_codec.n_dims, self.audio_codec.min_value, self.audio_codec.max_value,
          rng=self.rng, precision=self.precision)
      eng = engine.Engine(cfg, self._device_index)
      eng.load_weights(self._restore_from_checkpoint())
      self._params = None  # the engine holds the packed copy
      dev = eng.device
      for name in self._encoder_inputs():
        shape = self.input_shapes[name]
        dt = torch.int32 if self.input_types[name] == np.int32 else torch.float32
        self._pinned[name] = torch.empty(shape, dtype=dt).pin_memory()
        self._dev[name] = torch.empty(shape, dtype=dt, device=dev)
      out_shape = self.input_shapes['decoder_target_tokens']
      self._dev['mel'] = torch.empty(out_shape, dtype=torch.float32, device=dev)
      self._pinned['mel'] = torch.empty(out_shape, dtype=torch.float32).pin_memory()
      self._engine = eng
    return self._engine

  @property
  def engine(self) -> engine.Engine:
    return self._get_engine()

  def predict_on_device(self, tokens: torch.Tensor, ctx_features: Optional[torch.Tensor],
                        ctx_mask: Optional[torch.Tensor], seed: int = 0,
                        init_z: Optional[torch.Tensor] = None,
                        noise: Optional[torch.Tensor] = None,
                        seeds: Optional[Sequence[int]] = None) -> torch.Tensor:
    """Device tensors in, device mel out (no host round trip); used by the multi-GPU drivers
    to hand a segment's prediction to the next segment's context GPU-to-GPU.

    seeds: one seed per row; row b then draws its noise from seeds[b] alone, i.e. comes out as
    predict_on_device(row b, seed=seeds[b]) at batch 1 would draw it (Engine.sample_rows), so
    unrelated segments (e.g. of different songs) can share a batch.  `seed` is then unused, and
    injected init_z / noise are not accepted.  A no-context model takes None for ctx_features and
    ctx_mask."""
    eng = self._get_engine()
    b = tokens.shape[0]
    if b > self.batch_size:
      raise ValueError(f'batch of {b} exceeds batch_size={self.batch_size}')
    if seeds is not None and (init_z is not None or noise is not None):
      raise ValueError('per-row seeds draw their own noise: init_z / noise cannot be injected')
    if seeds is not None and len(seeds) != b:
      raise ValueError(f'{len(seeds)} seeds for a batch of {b}')
    if self.has_context:
      if ctx_features is None or ctx_mask is None:
        raise ValueError('this model takes a context: ctx_features and ctx_mask are required')
      ctx_features = ctx_features.to(torch.float32).contiguous()
      ctx_mask = ctx_mask.to(torch.int32).contiguous()
    elif ctx_features is not None or ctx_mask is not None:
      raise ValueError('the no-context model takes no ctx_features / ctx_mask (pass None)')
    eng.encode(tokens.to(torch.int32).contiguous(), ctx_features, ctx_mask)
    if seeds is not None:
      return eng.sample_rows(seeds)
    return eng.sample(init_z, noise, seed=seed).clone()

  def predict(self, batch: Mapping[str, np.ndarray], seed: int = 0,
              init_z: Optional[np.ndarray] = None, noise: Optional[np.ndarray] = None
              ) -> Tuple[np.ndarray, np.ndarray]:
    """Host numpy batch in -> (pred_mel [B, targets, n_dims] in feature units, zeros [B]).
    A no-context model reads encoder_input_tokens only and ignores the other keys, as the
    reference's DiffusionModel.predict_batch_with_aux does (models.py:149-205)."""
    eng = self._get_engine()
    dev = eng.device
    b = int(np.asarray(batch['encoder_input_tokens']).shape[0])
    if b > self.batch_size:
      raise ValueError(f'batch of {b} exceeds batch_size={self.batch_size}')
    want = self.input_shapes
    for name in self._encoder_inputs():
      arr = np.asarray(batch[name])
      if tuple(arr.shape[1:]) != tuple(want[name][1:]):
        raise ValueError(f'{name}: shape {arr.shape} does not match {want[name]}')
      pin = self._pinned[name][:b]
      pin.copy_(torch.from_numpy(np.ascontiguousarray(arr.astype(self.input_types[name]))))
      self._dev[name][:b].copy_(pin, non_blocking=True)
    tgt = batch.get('decoder_target_tokens')
    if tgt is not None and tuple(np.asarray(tgt).shape[1:]) != tuple(
        want['decoder_target_tokens'][1:]):
      raise ValueError('decoder_target_tokens: only its shape is used and it must be '
                       f'{want["decoder_target_tokens"]}')
    if self.has_context:
      eng.encode(self._dev['encoder_input_tokens'][:b], self._dev['encoder_continuous_inputs'][:b],
                 self._dev['encoder_continuous_mask'][:b])
    else:
      eng.encode(self._dev['encoder_input_tokens'][:b], None, None)
    z0 = None if init_z is None else torch.from_numpy(
        np.ascontiguousarray(init_z, dtype=np.float32)).to(dev)
    nz = None if noise is None else torch.from_numpy(
        np.ascontiguousarray(noise, dtype=np.float32)).to(dev)
    mel_dev = self._dev['mel'][:b]
    eng.sample(z0, nz, seed=seed, out=mel_dev)
    pin = self._pinned['mel'][:b]
    pin.copy_(mel_dev, non_blocking=True)
    torch.cuda.current_stream(dev).synchronize()
    return pin.numpy().copy(), np.zeros((b,), np.float32)
