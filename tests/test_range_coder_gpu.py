"""GPU parity: CUDA range coder (through the C ABI) vs the oracle, bit exact.

Reference behaviour under test: cc/kernels/range_coder_kernels.cc:191-322,360-471 (stream drivers,
overflow coding), cc/lib/range_coder.cc:37-307 and cc/lib/range_coder.h:144-282 (coder).
"""
import numpy as np
import pytest
import torch

import oracle
import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import gen_ops
  return gen_ops


def _tables(rng, nrows, overflow_prob=0.5, pmin=1, pmax=16, maxbins=40, peaky=3):
  """Rows at precisions pmin..pmax with 1 to min(maxbins, 2^p) bins (a one-bin overflow row escapes every value)."""
  precs = [int(rng.integers(pmin, pmax + 1)) for _ in range(nrows)]
  cdfs = [util.random_cdf(rng, int(rng.integers(1, min(maxbins, 1 << p) + 1)), p, peaky=peaky) for p in precs]
  ovf = [bool(rng.random() < overflow_prob) for _ in range(nrows)]
  return cdfs, precs, ovf


def _values(rng, cdfs, ovf, S, N, index, esc_prob=0.3, big=50):
  nrows = len(cdfs)
  rows = index if index is not None else np.broadcast_to(np.arange(N) % nrows, (S, N))
  nb = np.asarray([len(c) - 1 for c in cdfs])[rows]
  is_ovf = np.asarray(ovf)[rows]
  inside = (rng.random((S, N)) * np.where(is_ovf, np.maximum(nb - 1, 1), nb)).astype(np.int64)
  wild = rng.integers(-big, big, size=(S, N)) + np.where(rng.random((S, N)) < 0.5, 0, nb)
  use_wild = is_ovf & (rng.random((S, N)) < esc_prob)
  return np.where(use_wild, wild, inside).astype(np.int32)


def _gpu_encode(ops, lookup, value, index, shape):
  h = ops.create_range_encoder(shape, lookup)
  if index is None:
    ops.entropy_encode_channel(h, torch.from_numpy(value).cuda())
  else:
    ops.entropy_encode_index(h, torch.from_numpy(index).cuda(), torch.from_numpy(value).cuda())
  return ops.entropy_encode_finalize(h)


@pytest.mark.parametrize("seed", range(24))
def test_encode_decode_matches_oracle_fuzz(ops, seed):
  rng = np.random.default_rng(seed)
  O = oracle.best()
  nrows = int(rng.integers(1, 9))
  S = int(rng.integers(1, 9))
  N = int(rng.integers(0, 700))
  cdfs, precs, ovf = _tables(rng, nrows)
  two_d = bool(rng.integers(0, 2)) or util.ambiguous_1d(precs, ovf)
  lookup = util.make_lookup_2d(cdfs, precs, ovf) if two_d else util.make_lookup_1d(
      cdfs, precs, ovf, pad=rng.integers(0, 3, size=nrows))
  index = rng.integers(0, nrows, size=(S, N)).astype(np.int32) if rng.integers(0, 2) else None
  value = _values(rng, cdfs, ovf, S, N, index)
  want = O.encode(lookup, value, index)
  got = _gpu_encode(ops, lookup, value, index, [S])
  assert got.tolist() == want
  # GPU decode of the oracle's strings
  hd = ops.create_range_decoder(want, lookup)
  if index is None:
    hd, dec = ops.entropy_decode_channel(hd, [N])
  else:
    hd, dec = ops.entropy_decode_index(hd, torch.from_numpy(index).cuda(), [N])
  ok = ops.entropy_decode_finalize(hd)
  assert np.array_equal(dec.cpu().numpy(), value)
  assert bool(ok.all())
  # oracle decode of the GPU strings
  back, ok2 = O.decode(lookup, got.tolist(), N, index)
  assert np.array_equal(back, value) and ok2.all()


def test_multi_call_handle_persistence(ops):
  """State persists across EntropyEncode*/Decode* calls on one handle (range_coder_kernels.cc:225-226); a handle
  finalized with nothing encoded gives the empty strings."""
  rng = np.random.default_rng(100)
  O = oracle.best()
  cdfs, precs, ovf = _tables(rng, 5)
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  S = 6
  for chunks in ([37, 1, 0, 256, 129], []):
    vals = [_values(rng, cdfs, ovf, S, n, None) for n in chunks]
    enc = O.encoder(lookup, S)
    h = ops.create_range_encoder([2, 3], lookup)
    for v in vals:
      enc.encode(v)
      ops.entropy_encode_channel(h, torch.from_numpy(v.reshape(2, 3, -1)).cuda())
    want = enc.finalize()
    got = ops.entropy_encode_finalize(h)
    assert got.shape == (2, 3)
    assert got.tolist() == want
    hd = ops.create_range_decoder(got, lookup)
    for v in vals:
      hd, dec = ops.entropy_decode_channel(hd, [v.shape[1]])
      assert dec.shape == (2, 3, v.shape[1])
      assert np.array_equal(dec.cpu().numpy().reshape(S, -1), v)
    assert bool(ops.entropy_decode_finalize(hd).all())


def test_finalize_tail_cases_and_tiny_streams(ops):
  """Every flush branch of RangeEncoder::Finalize (range_coder.cc:266-307) on short streams."""
  O = oracle.best()
  rng = np.random.default_rng(7)
  seen = set()
  for p in (1, 2, 5, 9, 12, 16):
    for nb in (2, 3, 17):
      if nb > (1 << p):
        continue
      cdf = util.random_cdf(rng, nb, p, peaky=4)
      lookup = util.make_lookup_1d([cdf], [p], [False])
      S, N = 64, int(rng.integers(1, 24))
      value = rng.integers(0, nb, size=(S, N)).astype(np.int32)
      want = O.encode(lookup, value)
      got = _gpu_encode(ops, lookup, value, None, [S]).tolist()
      assert got == want
      seen.update(len(w) - 2 * (len(w) // 2) for w in want)
  assert seen == {0, 1}


def test_top_hugging_intervals_state1(ops):
  """Symbols whose interval hugs the top of the range force long carry delays (state 1)."""
  O = oracle.best()
  for p in (8, 12, 16):
    total = 1 << p
    cdf = np.asarray([0, 1, total - 1, total], dtype=np.int32)  # bins: tiny, huge, tiny
    lookup = util.make_lookup_1d([cdf], [p], [False])
    rng = np.random.default_rng(p)
    S, N = 128, 600
    value = rng.choice(3, size=(S, N), p=[0.05, 0.5, 0.45]).astype(np.int32)
    want = O.encode(lookup, value)
    got = _gpu_encode(ops, lookup, value, None, [S])
    assert got.tolist() == want
    hd = ops.create_range_decoder(got, lookup)
    hd, dec = ops.entropy_decode_channel(hd, [N])
    assert np.array_equal(dec.cpu().numpy(), value)
    assert bool(ops.entropy_decode_finalize(hd).all())


def test_large_tables_and_long_streams(ops):
  """cfg2/cfg3-like shapes: many streams, long streams, wide tables (k-ary search > 1 round)."""
  O = oracle.best()
  rng = np.random.default_rng(11)
  cdfs = [util.laplace_cdf(n, 12, s) for n, s in ((41, 3.0), (301, 40.0), (1501, 250.0), (9, 0.7))]
  lookup = util.make_lookup_1d(cdfs, [12] * 4, [True] * 4)
  S, N = 32, 4096
  index = rng.integers(0, 4, size=(S, N)).astype(np.int32)
  value = np.empty((S, N), np.int32)
  for r, c in enumerate(cdfs):
    m = index == r
    value[m] = util.sample_symbols(rng, c, int(m.sum()))
  esc = rng.random((S, N)) < 0.01
  value[esc] = rng.integers(-3000, 3000, size=int(esc.sum()))
  want = O.encode(lookup, value, index, threads=8)
  got = _gpu_encode(ops, lookup, value, index, [S])
  assert got.tolist() == want
  hd = ops.create_range_decoder(got, lookup)
  hd, dec = ops.entropy_decode_index(hd, torch.from_numpy(index).cuda(), [N])
  assert np.array_equal(dec.cpu().numpy(), value)
  assert bool(ops.entropy_decode_finalize(hd).all())


def test_argument_errors(ops):
  cdf = np.asarray([0, 4, 8, 16], np.int32)
  lookup = util.make_lookup_1d([cdf], [4], [False])
  with pytest.raises(ops.InvalidArgumentError, match="value=3 not in range"):
    h = ops.create_range_encoder([1], lookup)
    ops.entropy_encode_channel(h, torch.tensor([[0, 3]], dtype=torch.int32).cuda())
    ops.entropy_encode_finalize(h)
  with pytest.raises(ops.InvalidArgumentError, match="index=2 not in range"):
    h = ops.create_range_encoder([1], lookup)
    ops.entropy_encode_index(h, torch.tensor([[0, 2]], dtype=torch.int32).cuda(),
                             torch.tensor([[0, 0]], dtype=torch.int32).cuda())
    ops.entropy_encode_finalize(h)
  for bad, msg in (([4, 1, 16], "CDF must start with 0"), ([4, 0, 3, 2, 16], "monotonically"),
                   ([4, 0, 3], "CDF must end with"), ([17, 0, 4], "precision"), ([4, 0], "prematurely")):
    with pytest.raises(ops.InvalidArgumentError, match=msg):
      ops.create_range_encoder([1], np.asarray(bad, np.int32))
  with pytest.raises(ops.InvalidArgumentError, match="should start with"):
    h = ops.create_range_encoder([2], lookup)
    ops.entropy_encode_channel(h, torch.zeros((3, 4), dtype=torch.int32).cuda())


def test_truncated_stream_fails_sanity(ops):
  O = oracle.best()
  rng = np.random.default_rng(3)
  cdf = util.random_cdf(rng, 30, 12)
  lookup = util.make_lookup_1d([cdf], [12], [False])
  value = util.sample_symbols(rng, cdf, 4000).reshape(4, 1000)
  strings = O.encode(lookup, value)
  cut = [s[:len(s) // 2] for s in strings]
  # decoding fewer symbols than encoded leaves unread bytes -> False (range_coder.h:146-148)
  hd = ops.create_range_decoder(strings, lookup)
  hd, _ = ops.entropy_decode_channel(hd, [10])
  assert not bool(ops.entropy_decode_finalize(hd).any())
  # truncated strings: the reference decoder has undefined behaviour here (its search can run past
  # the table); ours must stay in bounds and return *some* verdict per stream.
  hd = ops.create_range_decoder(cut, lookup)
  hd, dec = ops.entropy_decode_channel(hd, [1000])
  ok = ops.entropy_decode_finalize(hd).numpy()
  assert dec.shape == (4, 1000) and ok.shape == (4,)
  d = dec.cpu().numpy()
  assert d.min() >= 0 and d.max() < 30


@pytest.mark.parametrize("mode", ["index", "channel"])
def test_wide_rows(ops, mode):
  """Rows wider than the decoder's 64-key window (generic search path): flat and peaked
  tables of 65 ... 4000 bins (stride 2 ... 63), with and without overflow, uniform symbols (every bin is hit, both
  window edges, first and last bins, escapes); streams and decoded symbols against the oracle."""
  rng = np.random.default_rng(7 if mode == "index" else 8)
  sizes = [65, 66, 127, 128, 129, 191, 640, 1000, 1501, 2048, 4000, 40, 64]
  cdfs, precs, ovf = [], [], []
  for i, nb in enumerate(sizes):
    p = 16 if nb > 1500 else (12 if nb <= 1000 else 14)
    cdfs.append(util.random_cdf(rng, nb, p, peaky=1.0 if i % 2 else 6.0))
    precs.append(p)
    ovf.append(i % 3 == 0)
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  S, N = 6, 5000 if mode == "index" else 13 * 400
  if mode == "index":
    index = rng.integers(0, len(sizes), (S, N)).astype(np.int32)
  else:
    index = np.broadcast_to(np.arange(N, dtype=np.int32) % len(sizes), (S, N)).copy()
  hi = np.asarray([len(c) - 1 for c in cdfs])[index]           # bins per symbol's row
  ov = np.asarray(ovf)[index]
  value = (rng.random((S, N)) * (hi - ov)).astype(np.int32)    # overflow rows: regular symbols are [0, bins - 1)
  esc = ov & (rng.random((S, N)) < 0.02)
  value[esc] = rng.integers(-300, 3000, int(esc.sum())).astype(np.int32)
  edge = rng.random((S, N)) < 0.05
  value[edge & ~esc] = np.where(rng.random(int((edge & ~esc).sum())) < 0.5, 0, (hi - ov - 1)[edge & ~esc])
  O = oracle.best()
  want = O.encode(lookup, value, index if mode == "index" else None)
  h = ops.create_range_encoder([S], lookup)
  if mode == "index":
    ops.entropy_encode_index(h, torch.from_numpy(index).cuda(), torch.from_numpy(value).cuda())
  else:
    ops.entropy_encode_channel(h, torch.from_numpy(value).cuda())
  got = ops.entropy_encode_finalize(h)
  assert got.tolist() == want
  hd = ops.create_range_decoder(got, lookup)
  if mode == "index":
    hd, dec = ops.entropy_decode_index(hd, torch.from_numpy(index).cuda(), [N])
  else:
    hd, dec = ops.entropy_decode_channel(hd, [N])
  assert bool(ops.entropy_decode_finalize(hd).all())
  assert np.array_equal(dec.cpu().numpy(), value)
