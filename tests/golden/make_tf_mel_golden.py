"""Dumps REFERENCE MelGAN features by running the reference's own `MelGAN.encode` (TensorFlow).

This is the route from "parity unpinned" to pinned for the audio -> mel kernel: on a machine that
has `tensorflow` and a checkout of magenta/music-spectrogram-diffusion, run

    python tests/golden/make_tf_mel_golden.py --reference /path/to/music-spectrogram-diffusion

It writes `tests/golden/tf_melgan_encode.npz`; `tests/test_tf_mel_golden.py` consumes the file
whenever it is present and skips otherwise.  TensorFlow is not installable in the build image (no
network), so the file is NOT committed yet; the script is written against the reference sources
and tf.signal's documented behaviour, not executed.

What is dumped (all float32):
  tf_window                  tf.signal.hann_window(640, periodic=True)
  tf_weights                 tf.signal.linear_to_mel_weight_matrix(128, 513, 16000, 0.0, 8000.0)
  audio_<name> / mel_<name>  seeded signals (SIGNALS) and MelGAN().encode(audio) of each
                             (audio_codecs.py:226-247)
"""
import argparse
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, 'tf_melgan_encode.npz')
SR = 16000


def signals():
  """Seeded test signals: noise from 1e-6 to full scale, tones, a chirp, an impulse, clipping,
  silence, and lengths around the hop and the window."""
  rng = np.random.default_rng(20240)
  n = SR * 3 + 77
  t = np.arange(n) / SR
  sig = {f'noise{k}': 10.0 ** -k * rng.uniform(-1, 1, n) for k in (6, 3, 0)}
  sig['tone440'] = np.sin(2 * np.pi * 440 * t)
  sig['chirp'] = np.sin(2 * np.pi * (50 * t + 700 * t * t))
  imp = np.zeros(n)
  imp[4321] = 1.0
  sig['impulse'] = imp
  sig['clipped'] = np.clip(3 * np.sin(2 * np.pi * 220 * t), -1, 1)
  sig['silence'] = np.zeros(SR)
  for m in (1, 319, 320, 321, 641):
    sig[f'len{m}'] = rng.uniform(-1, 1, m)
  return {k: v.astype(np.float32) for k, v in sig.items()}


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  ap.add_argument('--reference', required=True, help='checkout of music-spectrogram-diffusion')
  args = ap.parse_args()
  sys.path.insert(0, args.reference)
  import tensorflow as tf  # pylint: disable=import-outside-toplevel
  from music_spectrogram_diffusion import audio_codecs  # pylint: disable=import-outside-toplevel
  codec = audio_codecs.MelGAN()
  out = {
      'tf_window': tf.signal.hann_window(640, periodic=True).numpy().astype(np.float32),
      'tf_weights': tf.signal.linear_to_mel_weight_matrix(128, 513, 16000, 0.0, 8000.0)
                    .numpy().astype(np.float32),
  }
  for name, x in signals().items():
    out[f'audio_{name}'] = x
    out[f'mel_{name}'] = np.asarray(codec.encode(tf.constant(x)), np.float32)
  np.savez(OUT, **out)
  print(f'wrote {OUT}: {len(out)} arrays')


if __name__ == '__main__':
  main()
