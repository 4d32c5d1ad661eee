"""CPU: pins the oracle on the reference's own known-answer tests for the hot-path primitives
(msd/layers_test.py), re-expressed with the same np.random.seed(0) draws, plus the float64
sampler scalars of SURVEY App. A.4."""
import numpy as np
import pytest
import torch

from oracle import msd_oracle as O


def _softmax(x, axis=-1):
  x = x - x.max(axis=axis, keepdims=True)
  e = np.exp(x)
  return e / e.sum(axis=axis, keepdims=True)


def test_dot_product_attention_kat():
  """layers_test.py:375-387 (test_dot_product_attention): einsum/softmax, bias, NO scaling."""
  b, q, h, d, k = 2, 3, 4, 5, 6
  np.random.seed(0)
  query = np.random.randn(b, q, h, d)
  key = np.random.randn(b, k, h, d)
  value = np.random.randn(b, k, h, d)
  bias = np.random.randn(b, h, q, k)
  got = O.dot_product_attention(torch.from_numpy(query), torch.from_numpy(key),
                                torch.from_numpy(value), torch.from_numpy(bias)).numpy()
  logits = np.einsum('bqhd,bkhd->bhqk', query, key)
  weights = _softmax(logits + bias, axis=-1)
  expected = np.einsum('bhqk,bkhd->bqhd', weights, value)
  np.testing.assert_allclose(got, expected, atol=1e-6)


@pytest.mark.parametrize('f', [20, 22])
def test_multihead_dot_product_attention_kat(f):
  """layers_test.py:285-330: kernel layouts [f, h*d] / [h*d, f], no bias, no scale."""
  b, q, h, d, k = 2, 3, 4, 5, 6
  np.random.seed(0)
  inputs_q = np.random.randn(b, q, f)
  inputs_kv = np.random.randn(b, k, f)
  query_kernel = np.random.randn(f, h, d)
  key_kernel = np.random.randn(f, h, d)
  value_kernel = np.random.randn(f, h, d)
  out_kernel = np.random.randn(h, d, f)
  p = {
      'a/query/kernel': torch.from_numpy(query_kernel.reshape(f, -1)),
      'a/key/kernel': torch.from_numpy(key_kernel.reshape(f, -1)),
      'a/value/kernel': torch.from_numpy(value_kernel.reshape(f, -1)),
      'a/out/kernel': torch.from_numpy(out_kernel.reshape(-1, f)),
  }
  y = O.multi_head_dot_product_attention(torch.from_numpy(inputs_q), torch.from_numpy(inputs_kv),
                                         None, p, 'a', h, d).numpy()
  query = np.einsum('bqf,fhd->bqhd', inputs_q, query_kernel)
  key = np.einsum('bkf,fhd->bkhd', inputs_kv, key_kernel)
  value = np.einsum('bkf,fhd->bkhd', inputs_kv, value_kernel)
  logits = np.einsum('bqhd,bkhd->bhqk', query, key)
  weights = _softmax(logits, axis=-1)
  combined = np.einsum('bhqk,bkhd->bqhd', weights, value)
  y_expected = np.einsum('bqhd,hdf->bqf', combined, out_kernel)
  np.testing.assert_allclose(y, y_expected, rtol=1e-5, atol=1e-5)


def test_make_attention_mask_multiply_pairwise_fn():
  """layers_test.py:117-125."""
  decoder_target_tokens = torch.tensor([[7, 0, 0], [8, 5, 0]])
  m = (decoder_target_tokens > 0).float()
  attn_mask = O.make_attention_mask(m, m)
  expected = np.array([[[[1, 0, 0], [0, 0, 0], [0, 0, 0]]],
                       [[[1, 1, 0], [1, 1, 0], [0, 0, 0]]]])
  assert attn_mask.shape == (2, 1, 3, 3)
  np.testing.assert_array_equal(attn_mask.numpy(), expected)


def test_dense_general_kat():
  """layers_test.py:450-484 (DenseTest): bias-free x @ kernel, incl. joined axes."""
  np.random.seed(0)
  x = np.random.randn(2, 3, 4)
  w = np.random.randn(4, 5)
  got = O.dense_general(torch.from_numpy(x), torch.from_numpy(w)).numpy()
  np.testing.assert_allclose(got, x @ w, rtol=1e-12)
  # two contracted axes == contraction over the flattened axis (how `out` is stored)
  x2 = np.random.randn(2, 3, 4, 5)
  w2 = np.random.randn(4, 5, 6)
  got2 = O.dense_general(torch.from_numpy(x2.reshape(2, 3, 20)),
                         torch.from_numpy(w2.reshape(20, 6))).numpy()
  np.testing.assert_allclose(got2, np.einsum('abcd,cde->abe', x2, w2), rtol=1e-10)


def test_zero_activations_if_masked():
  y = torch.ones(2, 3, 4)
  mask = torch.zeros(2, 1, 3, 5)
  mask[1, 0, :, 2] = 1
  out = O.zero_activations_if_masked(y, mask)
  assert out[0].abs().sum() == 0 and torch.equal(out[1], y[1])


# SURVEY App. A.4: float64 known answers computed from diffusion_utils.py:120-187, 215-222
A4 = {
    999: dict(logsnr_t=-20.0, logsnr_s=-12.855470, c_z=0.028092, c_x0=0.001615, sigma=0.999605,
              x0_scale=22026.4658, eps_scale=1.0),
    998: dict(logsnr_t=-12.855470, logsnr_s=-11.497462, c_z=0.507120, c_x0=0.002367,
              sigma=0.861873, x0_scale=618.7718, eps_scale=0.999999),
    500: dict(logsnr_t=-0.006283, logsnr_s=0.0, c_z=0.995301, c_x0=0.004429, sigma=0.056048,
              x0_scale=1.4164, eps_scale=0.708217),
    1: dict(logsnr_t=11.497462, logsnr_s=12.855470, c_z=0.257174, c_x0=0.742826, sigma=0.002747,
            x0_scale=1.0, eps_scale=0.003187),
}


@pytest.mark.parametrize('i', sorted(A4))
def test_sampler_scalars_a4(i):
  c = O.sampler_coefficients(i, 1000, dtype=np.float64)
  for k, v in A4[i].items():
    np.testing.assert_allclose(c[k], v, rtol=1e-4, atol=2e-6, err_msg=f'i={i} {k}')


def test_cosine_logsnr_constants():
  b = np.arctan(np.exp(-10.0))
  a = np.arctan(np.exp(10.0)) - b
  np.testing.assert_allclose(a, 1.5707055269354342, rtol=1e-14)
  np.testing.assert_allclose(b, 4.539992973129278e-05, rtol=1e-12)
  np.testing.assert_allclose(np.log(2e4) / 383, 0.02585766984996378, rtol=1e-14)
  assert abs(float(O.get_logsnr_t(1.0, dtype=np.float64)) + 20.0) < 1e-9
  assert abs(float(O.get_logsnr_t(0.0, dtype=np.float64)) - 20.0) < 1e-9


def test_timing_signal_shape_and_values():
  t = torch.tensor([0.001, 0.5, 1.0], dtype=torch.float64)
  sig = O.get_timing_signal_1d(t * 2e4, 768, max_timescale=2e4)
  assert sig.shape == (3, 768)
  inv = np.exp(-np.arange(384) * np.log(2e4) / 383)
  np.testing.assert_allclose(sig[1, :384].numpy(), np.sin(1e4 * inv), atol=1e-6)
  np.testing.assert_allclose(sig[1, 384:].numpy(), np.cos(1e4 * inv), atol=1e-6)


def test_scale_features_roundtrip():
  cfg = O.OracleConfig()
  f = torch.tensor([-20.0, np.log(1e-5), 0.0, 4.0, 9.0])
  s = O.scale_features(f, cfg, clip=True)
  np.testing.assert_allclose(s.numpy(), [-1.0, -1.0, (0 - cfg.min_value) / 15.512925 * 2 - 1, 1.0, 1.0],
                             atol=1e-6)
  back = O.scale_to_features(s, cfg)
  np.testing.assert_allclose(back.numpy()[1:4], f.numpy()[1:4], atol=1e-5)


def test_get_sequence_length_and_roll():
  """network.py:28-51."""
  assert O.get_sequence_length(torch.tensor([1, 1, 0, 0, 0])) == 2
  assert O.get_sequence_length(torch.tensor([1, 1, 1])) == 3
  assert O.get_sequence_length(torch.tensor([0, 0, 0])) == 0
  assert torch.roll(torch.arange(5), 2, 0).tolist() == [3, 4, 0, 1, 2]


def test_linear_schedule_matches_float64_interp():
  """diffusion_utils.py:189-199 restated in float32 against a float64 numpy evaluation."""
  n, start, stop = 1000, 1e-4, 0.02
  betas = np.linspace(start, stop, n, dtype=np.float64)
  ac = np.cumprod(1. - betas)
  table = np.clip(np.log(ac) - np.log1p(-ac), -20.0, 20.0)
  ts = np.array([0.0, 1e-3, 0.25, 0.5, 0.7512, 0.999, 1.0])
  want = np.interp(ts, np.linspace(0, 1, n), table)
  got = O.get_logsnr_t(ts, 'linear', np.float32, start, stop, n)
  np.testing.assert_allclose(got, want, rtol=3e-4, atol=3e-4)
  assert got[0] == np.float32(table[0]) and got[-1] == np.float32(table[-1])
  with pytest.raises(ValueError, match='not identified'):
    O.get_logsnr_t(0.5, 'sigmoid')


def test_medium_logvar_interpolates_between_small_and_large():
  """diffusion_utils.py:141-156: frac 0 == 'small', frac 1 == 'large', log-linear in between."""
  one = torch.ones(3, dtype=torch.float64)
  ls, lt = 1.7, 0.4
  small = O.diffusion_reverse(one, one, ls, lt, 'small')['var']
  large = O.diffusion_reverse(one, one, ls, lt, 'large')['var']
  np.testing.assert_allclose(O.diffusion_reverse(one, one, ls, lt, 'medium:0')['var'], small, rtol=1e-12)
  np.testing.assert_allclose(O.diffusion_reverse(one, one, ls, lt, 'medium:1')['var'], large, rtol=1e-12)
  mid = O.diffusion_reverse(one, one, ls, lt, 'medium:0.25')['var']
  np.testing.assert_allclose(mid, large ** 0.25 * small ** 0.75, rtol=1e-12)
  x = torch.tensor([1e-3, 0.3, 0.7, 5.0], dtype=torch.float64)
  np.testing.assert_allclose(O.log1mexp(x), np.log(1 - np.exp(-x.numpy())), rtol=1e-10)


def test_model_output_conversions_are_consistent():
  """diffusion_utils.py:205-233, 288-321: x0 / eps / v describe the same point."""
  g = torch.Generator().manual_seed(0)
  z = torch.randn(4, 8, dtype=torch.float64, generator=g)
  eps = torch.randn(4, 8, dtype=torch.float64, generator=g)
  ls = -0.8
  x0, e = O.x0_and_eps_from_model_output(z, eps, ls, 'eps')
  assert e is eps
  x0b, eb = O.x0_and_eps_from_model_output(z, x0, ls, 'x0')
  np.testing.assert_allclose(eb, eps, rtol=1e-10)
  alpha, sigma = np.sqrt(1 / (1 + np.exp(-ls))), np.sqrt(1 / (1 + np.exp(ls)))
  np.testing.assert_allclose(alpha * x0 + sigma * eps, z, rtol=1e-10)   # z = alpha x0 + sigma eps
  v = alpha * eps - sigma * x0
  x0c, ec = O.x0_and_eps_from_model_output(z, v, ls, 'v')
  np.testing.assert_allclose(x0c, x0, rtol=1e-9)
  np.testing.assert_allclose(ec, eps, rtol=1e-9)
  with pytest.raises(ValueError, match='Unknown model_output'):
    O.x0_and_eps_from_model_output(z, eps, ls, 'x0_and_eps')


def test_embed_is_the_one_hot_product():
  """layers.py Embed with one_hot=True (network.py:278-284): one_hot(ids) @ embedding with the
  one-hot built as ids[..., None] == iota, so an id >= vocab or < 0 matches no row and embeds as
  zeros (not a clamped or wrapped row)."""
  vocab, d = 11, 6
  g = torch.Generator().manual_seed(0)
  emb = torch.randn(vocab, d, dtype=torch.float64, generator=g)
  ids = torch.tensor([[0, 1, vocab - 1, vocab, vocab + 5, 2 ** 31 - 1, -1, -vocab],
                      [5, -2 ** 31, 3, vocab - 1, 0, vocab, 7, 2]], dtype=torch.int32)
  one_hot = (ids.long().unsqueeze(-1) == torch.arange(vocab)).double()
  want = one_hot @ emb
  got = O.embed(ids, emb)
  assert got.shape == want.shape and got.dtype == torch.float64
  assert torch.equal(got, want)
  outside = (ids < 0) | (ids >= vocab)
  assert outside.sum() == 7 and bool((got[outside] == 0).all())
  assert torch.equal(got[~outside], emb[ids[~outside].long()])
