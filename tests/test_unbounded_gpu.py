"""GPU: UnboundedIndexRangeEncode / Decode (gen_ops one-string ops and functional ragged batches) against the
oracle, byte for byte, including the reference's own tests, damaged strings and the whole int32 range."""
import os

import numpy as np
import pytest
import torch

import oracle
from oracle import unbounded as ubi
import unbounded_util as U

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "unbounded_golden.npz")
GRID = [(p, w) for p in (1, 5, 11, 16) for w in (1, 2, 3, 8, 15, 16)]


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import functional as F
  from compression_b200 import gen_ops
  return gen_ops, F


def _case(rng, p, w, rows, width, n, heavy=True):
  cdf, cdf_size, offset, params = U.build_tables(rng, rows, width, p)
  index = rng.integers(0, rows, n).astype(np.int32)
  d = U.sample(rng, params, index)
  if heavy:
    tail = (rng.pareto(0.7, n) * rng.choice([-1, 1], n)).astype(np.int64)
    d = np.where(rng.random(n) < 0.2, tail, d)
  data = np.clip(d + offset[index], U.INT32_MIN, U.INT32_MAX).astype(np.int32)
  keep = U.domain_ok(data, index, cdf_size, offset, w)
  return data[keep], index[keep], cdf, cdf_size, offset


def test_random_index_round_trip(ops):
  gen_ops, _ = ops
  rng = np.random.default_rng(1)
  cdf, cdf_size, offset, params = U.build_tables(rng, 10, 40, 14)
  index = rng.integers(0, 10, (1, 32, 32, 16)).astype(np.int32)
  data = (U.sample(rng, params, index) + offset[index]).astype(np.int32)
  data.reshape(-1)[0] = -3
  data.reshape(-1)[-1] = 40 + 5
  s = gen_ops.unbounded_index_range_encode(data, index, cdf, cdf_size, offset, 14, 3)
  assert s == ubi.best().encode(data, index, cdf, cdf_size, offset, 14, 3)
  back = gen_ops.unbounded_index_range_decode(s, index, cdf, cdf_size, offset, 14, 3)
  assert back.shape == index.shape and back.dtype == torch.int32
  assert np.array_equal(back.cpu().numpy(), data)


def test_encoder_and_decoder_debug(ops):
  gen_ops, _ = ops
  from compression_b200._lib import InvalidArgumentError
  cdf = np.array([[0, 16, 18, 32]], np.int32)
  args = dict(data=np.array(0, np.int32), index=np.array(0, np.int32), cdf=cdf, cdf_size=np.array([4], np.int32),
              offset=np.array([1], np.int32), precision=5, overflow_width=2)
  s = gen_ops.unbounded_index_range_encode(**args)
  assert s == ubi.best().encode(*args.values())
  dec = {k: v for k, v in args.items() if k != "data"}
  assert gen_ops.unbounded_index_range_decode(b"", **dec).shape == ()
  for change, msg in ((dict(index=np.array(-1, np.int32)), "'index' has a value not in"),
                      (dict(cdf_size=np.array([1], np.int32)), "'cdf_size' has a value not in"),
                      (dict(cdf_size=np.array([5], np.int32)), "'cdf_size' has a value not in"),
                      (dict(cdf=np.array([[1, 16, 18, 32]], np.int32)), "cdf[0]="),
                      (dict(cdf=np.array([[0, 16, 18, 31]], np.int32)), "cdf[^1]="),
                      (dict(cdf=np.array([[0, 18, 16, 32]], np.int32)), "monotonic"),
                      (dict(cdf=np.array([[0, 16, 18, 31]], np.int32)), "Each cdf should start from 0 and end at 32")):
    for fn, a in ((gen_ops.unbounded_index_range_encode, {**args, **change}),
                  (gen_ops.unbounded_index_range_decode, {"encoded": s, **{k: v for k, v in {**args, **change}.items()
                                                                          if k != "data"}})):
      with pytest.raises(InvalidArgumentError) as e:
        fn(**a)
      assert msg in str(e.value)


@pytest.mark.parametrize("p,w", GRID)
def test_fuzz_grid_equals_the_oracle_and_cross_decodes(ops, p, w):
  gen_ops, _ = ops
  rng = np.random.default_rng(1000 + 17 * p + w)
  O = ubi.best()
  for rows, width in ((1, 3), (13, 30)):
    data, index, cdf, cdf_size, offset = _case(rng, p, w, rows, width, 4000)
    s = gen_ops.unbounded_index_range_encode(data, index, cdf, cdf_size, offset, p, w)
    want = O.encode(data, index, cdf, cdf_size, offset, p, w)
    assert s == want
    assert np.array_equal(O.decode(s, index, cdf, cdf_size, offset, p, w), data)
    assert np.array_equal(
        gen_ops.unbounded_index_range_decode(want, index, cdf, cdf_size, offset, p, w).cpu().numpy(), data)


def test_golden_vectors(ops):
  gen_ops, _ = ops
  g = np.load(GOLDEN)
  for c in range(int(g["n_cases"])):
    k = lambda name: g[f"{c}_{name}"]
    p, w = int(k("p")), int(k("w"))
    s = gen_ops.unbounded_index_range_encode(k("data"), k("index"), k("cdf"), k("cdf_size"), k("offset"), p, w)
    assert s == k("encoded").tobytes(), c
    back = gen_ops.unbounded_index_range_decode(s, k("index"), k("cdf"), k("cdf_size"), k("offset"), p, w)
    assert np.array_equal(back.cpu().numpy(), k("data"))


def test_debug_level_zero_still_refuses_what_would_read_outside_the_tables(ops):
  gen_ops, F = ops
  from compression_b200._lib import InvalidArgumentError
  cdf = np.array([[0, 16, 18, 32], [0, 16, 16, 32]], np.int32)
  base = dict(cdf=cdf, cdf_size=np.array([4, 4], np.int32), offset=np.array([0, 0], np.int32), precision=5,
              overflow_width=2, debug_level=0)
  data = np.zeros(40, np.int32)
  for index, sizes, value, msg in (
      (np.r_[np.zeros(30), [2], np.zeros(9)], [4, 4], 0, "'index' has a value not in [0, 2): value=2 (string 0, "
       "element 30)"),
      (np.r_[np.zeros(7), [1], np.zeros(32)], [4, 9], 0, "'cdf_size' has a value not in [3, 4]: value=9"),
      (np.r_[np.zeros(33), [1], np.zeros(6)], [4, 4], 1, "zero probability"),  # row 1 bin 1 is empty
  ):
    d = data.copy()
    d[index == 1] = value
    a = dict(base, cdf_size=np.array(sizes, np.int32))
    with pytest.raises(InvalidArgumentError) as e:
      gen_ops.unbounded_index_range_encode(d, index.astype(np.int32), **a)
    assert msg in str(e.value)
    if "zero probability" not in msg:
      with pytest.raises(InvalidArgumentError) as e:
        gen_ops.unbounded_index_range_decode(b"\x12\x34", index.astype(np.int32), **a)
      assert msg.split(" (")[0] in str(e.value)
  # non-monotone rows that are never used for an empty bin are not checked at debug_level 0 (as the reference)
  ok = dict(base, cdf=np.array([[0, 16, 18, 32], [0, 20, 10, 32]], np.int32))
  s = gen_ops.unbounded_index_range_encode(np.zeros(3, np.int32), np.zeros(3, np.int32), **ok)
  assert s == ubi.best().encode(np.zeros(3, np.int32), np.zeros(3, np.int32),
                                                          *list(ok.values())[:-1], debug_level=0)


def test_empty_data(ops):
  gen_ops, _ = ops
  cdf = np.array([[0, 16, 18, 32]], np.int32)
  for shape in ((0,), (3, 0, 2)):
    z = np.zeros(shape, np.int32)
    assert gen_ops.unbounded_index_range_encode(z, z, cdf, [4], [1], 5, 2) == b""
    assert gen_ops.unbounded_index_range_decode(b"", z, cdf, [4], [1], 5, 2).shape == shape


@pytest.mark.parametrize("w", [1, 16])
def test_arena_worst_case(ops, w):
  """Every element escapes with the largest u (d = INT32_MIN: u = 2^32 - 1) through a 1-in-2^16 escape bin."""
  gen_ops, F = ops
  cdf = np.array([[0, 65535, 65536]], np.int32)
  n = 50_000
  data = np.full(n, U.INT32_MIN, np.int32)
  index = np.zeros(n, np.int32)
  s = gen_ops.unbounded_index_range_encode(data, index, cdf, [3], [0], 16, w)
  K = (32 + w - 1) // w
  assert len(s) * 8 <= n * (16 + w * (K // ((1 << w) - 1) + 1 + K)) + 64
  assert len(s) * 8 >= n * (16 + 32)  # the main symbol and 32 bits of digits at least
  back = gen_ops.unbounded_index_range_decode(s, index, cdf, [3], [0], 16, w)
  assert np.array_equal(back.cpu().numpy(), data)
  strings = F.unbounded_index_range_encode_ragged(np.tile(data, 3), np.tile(index, 3), [n, n, n], cdf, [3], [0], 16, w)
  assert strings.tolist() == [s] * 3


@pytest.mark.parametrize("w", [1, 2, 3, 8, 15, 16])
def test_every_int32_round_trips_and_the_reference_decoder_agrees_where_defined(ops, w):
  gen_ops, F = ops
  rng = np.random.default_rng(w)
  cdf = np.array([[0, 10, 20, 30, 32], [0, 1, 31, 32, 32]], np.int32)
  cdf_size = np.array([5, 4], np.int32)
  specials = np.array([U.INT32_MIN, U.INT32_MIN + 1, -1, 0, 1, U.INT32_MAX - 1, U.INT32_MAX, -(1 << 30), 1 << 30],
                      np.int64)
  for offset in ([0, 0], [U.INT32_MAX, -5], [U.INT32_MIN, 7], [-123456, 1 << 30]):
    offset = np.array(offset, np.int32)
    data = np.r_[specials, rng.integers(U.INT32_MIN, U.INT32_MAX, 2000, endpoint=True)].astype(np.int32)
    index = rng.integers(0, 2, data.size).astype(np.int32)
    s = gen_ops.unbounded_index_range_encode(data, index, cdf, cdf_size, offset, 5, w)
    back = gen_ops.unbounded_index_range_decode(s, index, cdf, cdf_size, offset, 5, w).cpu().numpy()
    assert np.array_equal(back, data)
    # one string per element, decoded by the reference decoder wherever its additions stay defined
    strings = F.unbounded_index_range_encode_ragged(data, index, [1] * data.size, cdf, cdf_size, offset, 5, w)
    O = ubi.best()
    checked = 0
    for i, one in enumerate(strings.tolist()):
      try:
        got = O.decode(one, index[i:i + 1], cdf, cdf_size, offset, 5, w)
      except oracle.OracleError as e:
        assert "overflows int32" in str(e)
        continue
      assert got[0] == data[i]
      checked += 1
    assert checked > data.size // 4


def test_ragged_equals_one_string_ops(ops):
  gen_ops, F = ops
  rng = np.random.default_rng(5)
  data, index, cdf, cdf_size, offset = _case(rng, 13, 4, 20, 50, 30_000)
  lengths = [0, 5, 0, 1, 12_000, 0, data.size - 12_006]
  strings = F.unbounded_index_range_encode_ragged(data, index, lengths, cdf, cdf_size, offset, 13, 4)
  got = strings.tolist()
  at = 0
  for n, s in zip(lengths, got):
    assert s == gen_ops.unbounded_index_range_encode(data[at:at + n], index[at:at + n], cdf, cdf_size, offset, 13, 4)
    at += n
  assert got[0] == b"" and got[2] == b""
  back = F.unbounded_index_range_decode_ragged(strings, index, lengths, cdf, cdf_size, offset, 13, 4)
  assert np.array_equal(back.cpu().numpy(), data)
  back = F.unbounded_index_range_decode_ragged(got, index, lengths, cdf, cdf_size, offset, 13, 4)
  assert np.array_equal(back.cpu().numpy(), data)


def test_one_long_string_among_many_short_ones(ops):
  gen_ops, F = ops
  rng = np.random.default_rng(6)
  data, index, cdf, cdf_size, offset = _case(rng, 16, 8, 64, 40, 1_100_000)
  n_long = 1_000_000
  lengths = [1] * 2000 + [n_long] + [1] * 2095
  data, index = data[:sum(lengths)], index[:sum(lengths)]
  strings = F.unbounded_index_range_encode_ragged(data, index, lengths, cdf, cdf_size, offset, 16, 8)
  want = ubi.best().encode_batch(data, index, lengths, cdf, cdf_size, offset, 16, 8,
                                                          threads=8)
  got = strings.tolist()
  assert got == want
  for i in (0, 1999, 2000, 2001, 4095):
    at = sum(lengths[:i])
    assert got[i] == gen_ops.unbounded_index_range_encode(data[at:at + lengths[i]], index[at:at + lengths[i]], cdf,
                                                          cdf_size, offset, 16, 8)
  back = F.unbounded_index_range_decode_ragged(strings, index, lengths, cdf, cdf_size, offset, 16, 8)
  assert np.array_equal(back.cpu().numpy(), data)


def test_launch_count_does_not_depend_on_the_number_of_strings(ops):
  _, F = ops
  from compression_b200 import _lib
  rng = np.random.default_rng(8)
  data, index, cdf, cdf_size, offset = _case(rng, 12, 3, 8, 20, 20_000)
  counts = []
  for k in (1, 7, 4096):
    lengths = np.diff(np.linspace(0, data.size, k + 1).astype(np.int64))
    for debug in (0, 1):
      before = _lib.launch_count()
      s = F.unbounded_index_range_encode_ragged(data, index, lengths, cdf, cdf_size, offset, 12, 3, debug)
      mid = _lib.launch_count()
      F.unbounded_index_range_decode_ragged(s, index, lengths, cdf, cdf_size, offset, 12, 3, debug)
      counts.append((k, debug, mid - before, _lib.launch_count() - mid))
  for k, debug, enc, dec in counts:
    assert (enc, dec) == (3 + debug, 1 + debug), counts


def _long_prefix(w, extra=1):
  """A string whose one escape has a width prefix of K + extra digits (no encoder writes more than K)."""
  K = (32 + w - 1) // w
  M = (1 << w) - 1
  total = K + extra
  prefix = [M] * (total // M) + [total % M]
  return oracle.port().encode_triples([18] + prefix, [32] + [v + 1 for v in prefix], [5] + [w] * len(prefix))


def test_damaged_strings(ops):
  gen_ops, F = ops
  from compression_b200._lib import InvalidArgumentError
  rng = np.random.default_rng(9)
  O = ubi.best()
  for p, w in ((14, 3), (8, 1), (16, 16), (5, 2), (11, 15)):
    data, index, cdf, cdf_size, offset = _case(rng, p, w, 6, 20, 500)
    good = O.encode(data, index, cdf, cdf_size, offset, p, w)
    damaged = [good[:len(good) // 3], b"", rng.bytes(len(good)), rng.bytes(7), b"\xff" * len(good)]
    for _ in range(6):
      f = bytearray(good)
      for _ in range(int(rng.integers(1, 4))):
        f[int(rng.integers(len(good)))] ^= 1 << int(rng.integers(8))
      damaged.append(bytes(f))
    for s in damaged:
      try:
        want = O.decode(s, index, cdf, cdf_size, offset, p, w)
      except oracle.OracleError as e:
        want = str(e)
      if isinstance(want, str) and "prefix longer" in want:
        with pytest.raises(InvalidArgumentError, match="overflow width prefix exceeds"):
          gen_ops.unbounded_index_range_decode(s, index, cdf, cdf_size, offset, p, w)
        continue
      got = gen_ops.unbounded_index_range_decode(s, index, cdf, cdf_size, offset, p, w).cpu().numpy()
      if not isinstance(want, str):
        assert np.array_equal(got, want)
  # over-long prefixes in strings 3 and 5 of a batch: the error names string 3 and its element
  cdf = np.array([[0, 16, 18, 32]], np.int32)
  for w in (1, 2, 3, 16):
    good = gen_ops.unbounded_index_range_encode(np.array([1, 1, 6], np.int32), np.zeros(3, np.int32), cdf, [4], [1],
                                                5, w)
    strings = [b"", b"\x00\x00", good, _long_prefix(w), b"\x20", _long_prefix(w, 5)]
    lengths = [0, 1, 3, 1, 1, 1]
    index = np.zeros(sum(lengths), np.int32)
    with pytest.raises(InvalidArgumentError) as e:
      F.unbounded_index_range_decode_ragged(strings, index, lengths, cdf, [4], [1], 5, w)
    assert "(string 3, element 0)" in str(e.value)
    with pytest.raises(InvalidArgumentError, match="overflow width prefix exceeds"):
      gen_ops.unbounded_index_range_decode(_long_prefix(w), np.zeros(1, np.int32), cdf, [4], [1], 5, w)
