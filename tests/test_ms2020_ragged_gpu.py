"""GPU: a ragged encode that hands back the decoded values (tfcb_compress_ragged_decoded, `return_decoded=True`), and
MS2020Model.compress_images / decompress_images built on it.

The contract: the strings are those of the plain ragged encode, and the decoded values are bit for bit what the
ragged decode returns for them -- including where float quantisation is not the identity on the integer the coder
sees (|y - loc| >= 2^31 saturates, NaN becomes 0).  MS2020 over a list of images then needs num_slices + 1 encode
launches and no decode, and num_slices + 1 decode launches to decompress, whatever the number of images.
"""
import numpy as np
import pytest
import torch

import oracle
import util

pytestmark = pytest.mark.gpu

SPECIAL_LENGTHS = [0, 1, 31, 32, 33, 4097, 200_003]
SPECIAL_VALUES = [3e9, -3e9, 2.0e9, -2.1e9, float("inf"), float("-inf"), float("nan")]  # (2.0e9, -2.1e9: exact)


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import gen_ops
  return gen_ops


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


def _overflow_tables():
  cdfs = [util.laplace_cdf(n, 12, s) for n, s in ((41, 3.0), (31, 2.0), (61, 8.0), (9, 0.7), (21, 1.5), (101, 20.0))]
  lookup = util.make_lookup_1d(cdfs, [12] * len(cdfs), [True] * len(cdfs))
  coff = torch.tensor([-(len(c) - 1) // 2 for c in cdfs], dtype=torch.int32).cuda()
  return lookup, coff


def _loc_per_symbol(lens, nrows, q, index_mode):
  """The offset the decoder adds to every symbol: loc itself (index mode) or quant_offset[j mod nrows], j counted
  from 0 in every stream (channel mode); zero without one."""
  total = sum(lens)
  if q is None:
    return torch.zeros(total, device="cuda")
  if index_mode:
    return q
  rows = np.concatenate([np.arange(n) % nrows for n in lens]) if total else np.zeros(0, np.int64)
  return q[torch.from_numpy(rows).cuda()]


def _check_decoded(ops, F, lookup, coff, lens, y, q, index, strings, dec):
  """`dec` against the ragged decode of `strings`, as int32 bit patterns, and against round(y - loc) + loc where
  float quantisation is exact."""
  hd = ops.create_range_decoder(strings, lookup)
  ref = F.decode_ragged(hd, lens, index=index, quant_offset=q, cdf_offset=coff)
  assert bool(ops.entropy_decode_finalize(hd).all())
  assert dec.dtype == torch.float32 and dec.shape == ref.shape
  assert torch.equal(dec.view(torch.int32), ref.view(torch.int32))
  loc = _loc_per_symbol(lens, coff.numel(), q, index is not None)
  d = y - loc
  exact = d.abs() < 2.0**31  # (False for NaN)
  assert torch.equal(dec[exact], (torch.round(d) + loc)[exact])
  return exact


@pytest.mark.parametrize("with_offsets", [True, False])
@pytest.mark.parametrize("mode", ["channel", "index"])
def test_kernel_emits_what_the_decoder_returns(ops, F, mode, with_offsets):
  rng = np.random.default_rng(70 + 2 * (mode == "index") + with_offsets)
  lookup, coff = _overflow_tables()
  nrows = coff.numel()
  lens = SPECIAL_LENGTHS + [int(v) for v in rng.integers(0, 700, 300 - len(SPECIAL_LENGTHS))]
  rng.shuffle(lens)
  total = sum(lens)
  y = torch.from_numpy((rng.standard_normal(total) * 6).astype(np.float32)).cuda()
  y[torch.from_numpy(rng.random(total) < 0.01).cuda()] *= 500  # escapes
  # saturating and non-finite values, only in streams of at least 1000 symbols: the short ones stay comparable
  # with the oracle's integer coder below
  starts = np.concatenate([[0], np.cumsum(lens)])
  long_streams = [i for i, n in enumerate(lens) if n >= 1000]
  for k, i in enumerate(long_streams):
    at = rng.choice(lens[i], size=min(lens[i], 40), replace=False) + starts[i]
    for j, a in enumerate(at):
      y[int(a)] = SPECIAL_VALUES[(j + k) % len(SPECIAL_VALUES)]
  if mode == "channel":
    index = None
    q = torch.from_numpy(rng.uniform(-0.5, 0.5, nrows).astype(np.float32)).cuda() if with_offsets else None
  else:
    index = torch.from_numpy(rng.integers(0, nrows, total).astype(np.int32)).cuda()
    q = torch.from_numpy(rng.uniform(-2, 2, total).astype(np.float32)).cuda() if with_offsets else None

  strings, dec = F.compress_ragged(lookup, lens, y, q, coff, index=index, decoded=True)
  plain = F.compress_ragged(lookup, lens, y, q, coff, index=index)
  assert torch.equal(strings.offsets_dev, plain.offsets_dev)
  assert strings.tolist() == plain.tolist()
  exact = _check_decoded(ops, F, lookup, coff, lens, y, q, index, strings, dec)
  assert int((~exact).sum()) >= 20 * len(long_streams)  # saturating and non-finite values did reach the kernel

  # the oracle: the short streams' strings against the reference coder of the symbols they decode to
  hd = ops.create_range_decoder(strings, lookup)
  sym = F.decode_ragged(hd, lens, index=index).cpu().numpy()
  idx = None if index is None else index.cpu().numpy()
  O = oracle.best()
  picked = [i for i, n in enumerate(lens) if n < 1000][:40]
  got = strings.tolist()
  for i in picked:
    sl = slice(int(starts[i]), int(starts[i + 1]))
    want = O.encode(lookup, sym[sl][None], None if idx is None else idx[sl][None])
    assert want == [got[i]], i


def test_a_long_stream_beside_one_symbol_streams(ops, F):
  """One 20 M-symbol stream beside 4 095 one-symbol streams, channel mode with quantisation offsets."""
  lookup, coff = _overflow_tables()
  lens = [20_000_000] + [1] * 4095
  total = sum(lens)
  g = torch.Generator(device="cuda").manual_seed(21)
  y = torch.randn(total, device="cuda", generator=g) * 5
  y[torch.rand(total, device="cuda", generator=g) < 0.001] *= 300
  y[::1_000_003] = float("nan")
  y[7::999_983] = -3e9
  q = torch.linspace(-0.4, 0.4, coff.numel(), device="cuda")
  strings, dec = F.compress_ragged(lookup, lens, y, q, coff, decoded=True)
  _check_decoded(ops, F, lookup, coff, lens, y, q, None, strings, dec)


# ------------------------------------------------------------------------------------------------
# Entropy models
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_batched_entropy_model_return_decoded(dtype):
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  torch.manual_seed(0)
  prior = D.NoisyLogistic(loc=torch.linspace(-1, 1, 8), scale=torch.linspace(0.5, 4, 8))
  em = E.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=True, bottleneck_dtype=dtype).cuda()
  xs = [(torch.randn(n, 8, device="cuda") * 5).to(dtype) for n in (1, 17, 0, 300, 64)]
  strings, items = em.compress_ragged(xs, return_decoded=True)
  assert strings.tolist() == em.compress_ragged(xs).tolist()
  back = em.decompress_ragged(strings, [(x.shape[0],) for x in xs])
  assert len(items) == len(xs)
  for it, b in zip(items, back):
    assert it.dtype == b.dtype == dtype and it.shape == b.shape
    assert torch.equal(it.view(torch.int16 if dtype == torch.float16 else torch.int32),
                       b.view(torch.int16 if dtype == torch.float16 else torch.int32))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_location_scale_model_return_decoded(dtype):
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  torch.manual_seed(1)
  ls = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 16, lambda i: torch.exp(i / 4 - 1), coding_rank=3,
                                          compression=True, bottleneck_dtype=dtype).cuda()
  xs = [(torch.randn(h, w, 5, device="cuda") * 6).to(dtype) for h, w in ((4, 4), (5, 3), (1, 9), (17, 2), (0, 3))]
  sc = [torch.rand(x.shape, device="cuda") * 16 for x in xs]
  loc = [(torch.randn(x.shape, device="cuda") * 3).to(dtype) for x in xs]
  strings, items = ls.compress_ragged(xs, sc, loc, return_decoded=True)
  assert strings.tolist() == ls.compress_ragged(xs, sc, loc).tolist()
  iv = torch.int16 if dtype == torch.float16 else torch.int32
  for it, b in zip(items, ls.decompress_ragged(strings, sc, loc)):
    assert it.dtype == b.dtype == dtype and it.shape == b.shape
    assert torch.equal(it.view(iv), b.view(iv))


# ------------------------------------------------------------------------------------------------
# MS2020Model
# ------------------------------------------------------------------------------------------------
SIZES = [(64, 64), (128, 64), (64, 128), (192, 64), (64, 192), (128, 128)]


@pytest.fixture(scope="module")
def ms2020():
  from compression_b200 import models
  torch.manual_seed(4)
  m = models.MS2020Model(num_filters=24, latent_depth=32, hyperprior_depth=16, num_slices=4, max_support_slices=2)
  return m.build("cuda", patch=(64, 64)).fix_tables()


def _images(sizes, seed):
  g = torch.Generator().manual_seed(seed)
  return [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in sizes]


def _same(a, b):
  if isinstance(a, torch.Tensor):
    return isinstance(b, torch.Tensor) and torch.equal(a, b)
  return a.shape == b.shape and a.tolist() == b.tolist()


def test_ms2020_compress_images_equals_compress(ms2020):
  m = ms2020
  images = _images(SIZES, 5)
  got = m.compress_images(images)
  assert len(got) == len(images)
  for g, x in zip(got, images):
    want = m.compress(x)
    assert len(g) == len(want) == 4 + m.num_slices
    assert all(_same(a, b) for a, b in zip(g, want))
  dec = m.decompress_images(got)
  for d, g, x in zip(dec, got, images):
    assert d.shape == x.shape and d.dtype == torch.uint8
    assert torch.equal(d, m.decompress(*g))


def test_ms2020_images_reject_bad_input(ms2020):
  with pytest.raises(ValueError):
    ms2020.compress_images([])
  with pytest.raises(ValueError):
    ms2020.compress_images([torch.zeros(64, 64, 3, dtype=torch.uint8), torch.zeros(64, 64, dtype=torch.uint8)])
  with pytest.raises(ValueError):
    ms2020.compress_images([torch.zeros(64, 64, 4, dtype=torch.uint8)])
  with pytest.raises(ValueError):
    ms2020.decompress_images([])


ENCODERS = [("functional", n) for n in ("compress_f32", "compress_ragged", "encode_channel_f32", "encode_index_f32")] + \
           [("gen_ops", n) for n in ("entropy_encode_channel", "entropy_encode_index")]
DECODERS = [("functional", n) for n in ("decode_ragged", "decode_channel_f32", "decode_index_f32")] + \
           [("gen_ops", n) for n in ("entropy_decode_channel", "entropy_decode_index")]


@pytest.mark.parametrize("n_images", [2, 6])
def test_ms2020_coder_calls_do_not_grow_with_the_image_count(ms2020, monkeypatch, n_images):
  from compression_b200 import functional, gen_ops
  mods = {"functional": functional, "gen_ops": gen_ops}
  calls = {"encode": 0, "decode": 0}

  def wrap(kind, fn):
    def counted(*a, **k):
      calls[kind] += 1
      return fn(*a, **k)
    return counted

  for kind, names in (("encode", ENCODERS), ("decode", DECODERS)):
    for mod, name in names:
      monkeypatch.setattr(mods[mod], name, wrap(kind, getattr(mods[mod], name)))
  images = _images((SIZES * 2)[:n_images], 6 + n_images)
  items = ms2020.compress_images(images)
  assert calls == {"encode": ms2020.num_slices + 1, "decode": 0}
  calls.update(encode=0, decode=0)
  out = ms2020.decompress_images(items)
  assert calls == {"encode": 0, "decode": ms2020.num_slices + 1}
  assert len(out) == n_images
