"""UnboundedIndexRangeEncode / Decode oracles: the C port against the compiled reference, the golden file, and
the inputs on which the reference is undefined (both flavours must refuse them, never run them)."""
import os

import numpy as np
import pytest

import oracle
from oracle import unbounded as ubi
import unbounded_util as U

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "unbounded_golden.npz")
GRID = [(p, w) for p in (1, 5, 11, 16) for w in (1, 2, 3, 8, 15, 16)]


def flavours():
  return [ubi.port()] + ([ubi.ref()] if ubi.have_ref() else [])


def _case(rng, p, w, rows, width, n, heavy=False):
  cdf, cdf_size, offset, params = U.build_tables(rng, rows, width, p)
  index = rng.integers(0, rows, n).astype(np.int32)
  d = U.sample(rng, params, index)
  if heavy:  # Pareto-like tails in both directions
    tail = (rng.pareto(0.7, n) * rng.choice([-1, 1], n)).astype(np.int64)
    d = np.where(rng.random(n) < 0.2, tail, d)
  data = np.clip(d + offset[index], U.INT32_MIN, U.INT32_MAX).astype(np.int32)
  keep = U.domain_ok(data, index, cdf_size, offset, w)
  return data[keep], index[keep], cdf, cdf_size, offset


@pytest.mark.skipif(not ubi.have_ref(), reason="compiled reference not built")
@pytest.mark.parametrize("p,w", GRID)
def test_port_equals_reference(p, w):
  rng = np.random.default_rng(p * 100 + w)
  R, P = ubi.ref(), ubi.port()
  for rows, width, heavy in ((1, 3, False), (7, 12, True), (40, 70, True)):
    data, index, cdf, cdf_size, offset = _case(rng, p, w, rows, width, 3000, heavy)
    a = R.encode(data, index, cdf, cdf_size, offset, p, w)
    assert P.encode(data, index, cdf, cdf_size, offset, p, w) == a
    for O in (R, P):
      assert np.array_equal(O.decode(a, index, cdf, cdf_size, offset, p, w), data)


@pytest.mark.skipif(not ubi.have_ref(), reason="compiled reference not built")
def test_batch_threads_equal_one_string_ops():
  rng = np.random.default_rng(7)
  data, index, cdf, cdf_size, offset = _case(rng, 12, 4, 9, 30, 20000, True)
  lengths = [0, 1, 5000, 0, len(data) - 5001]
  R = ubi.ref()
  got = R.encode_batch(data, index, lengths, cdf, cdf_size, offset, 12, 4, threads=4)
  at = 0
  for n, s in zip(lengths, got):
    assert s == R.encode(data[at:at + n], index[at:at + n], cdf, cdf_size, offset, 12, 4)
    at += n
  assert got[0] == b""
  back = R.decode_batch(got, index, lengths, cdf, cdf_size, offset, 12, 4, threads=4)
  assert np.array_equal(back, data)


def test_golden():
  g = np.load(GOLDEN)
  for O in flavours():
    for c in range(int(g["n_cases"])):
      k = lambda name: g[f"{c}_{name}"]
      p, w = int(k("p")), int(k("w"))
      got = O.encode(k("data"), k("index"), k("cdf"), k("cdf_size"), k("offset"), p, w)
      assert got == k("encoded").tobytes(), (O.kind, c)
      assert np.array_equal(
          O.decode(got, k("index"), k("cdf"), k("cdf_size"), k("offset"), p, w), k("data"))


def _one(value, offset, w, m=2, p=5):
  cdf = np.array([[0, 16, 18, 32][:m + 2] if m == 2 else list(range(m + 2))], np.int32)
  return np.array([value], np.int32), np.zeros(1, np.int32), cdf, np.array([m + 2], np.int32), \
      np.array([offset], np.int32)


UNDEFINED = [
    ("data - offset", U.INT32_MIN, 1, 2),
    ("data - offset", U.INT32_MAX, -1, 2),
    ("-2 *", -(1 << 30), 0, 2),
    ("-2 *", U.INT32_MIN + 5, 0, 2),
    ("2 * (data", (1 << 30) + 2, 0, 2),
    ("shifts by 32", 2 + (1 << 15), 0, 16),  # u = 2^16 at w = 16
    ("shifts by 32", 2 + (1 << 29), 0, 3),   # u = 2^30 >= 2^(3 * 10)
]


@pytest.mark.parametrize("what,value,off,w", UNDEFINED)
def test_undefined_encodes_are_refused(what, value, off, w):
  for O in flavours():
    with pytest.raises(oracle.OracleError, match="undefined"):
      O.encode(*_one(value, off, w), 5, w)


def test_domain_edges_are_coded():
  for w in (1, 2, 3, 8, 15, 16):
    K = (32 + w - 1) // w
    top_u = (1 << ((K - 1) * w)) - 1  # the largest u the width loop handles
    edges = [-min((1 << 30) - 1, (top_u + 1) // 2), 2 + min((1 << 30) - 1, top_u // 2)]
    for v in edges:
      for O in flavours():
        s = O.encode(*_one(v, 0, w), 5, w)
        assert O.decode(s, *_one(v, 0, w)[1:], 5, w)[0] == v


def test_undefined_decodes_are_refused():
  for O in flavours():
    # a width prefix of K + 1 digits, and u / 2 + m or + offset beyond int32, from strings the GPU would write
    cdf = np.array([[0, 16, 18, 32]], np.int32)
    long_prefix = oracle.port().encode_triples([18, 3, 3, 3, 3, 3, 2], [32, 4, 4, 4, 4, 4, 3],
                                               [5, 2, 2, 2, 2, 2, 2])
    with pytest.raises(oracle.OracleError, match="prefix longer"):
      O.decode(long_prefix, np.zeros(1, np.int32), cdf, [4], [0], 5, 2)
    u = 0xFFFFFFFE  # even: u / 2 + m = 2^31 - 1 + 2
    triples = [(18, 32, 5)] + [(3, 4, 2)] * 5 + [(1, 2, 2)] + [(((u >> (2 * j)) & 3), ((u >> (2 * j)) & 3) + 1, 2) for j in range(16)]
    s = oracle.port().encode_triples(*zip(*triples))
    with pytest.raises(oracle.OracleError, match="max_value overflows"):
      O.decode(s, np.zeros(1, np.int32), cdf, [4], [0], 5, 2)
    u = 2 * 5  # 5 + m = 7; + offset INT32_MAX overflows
    triples = [(18, 32, 5), (2, 3, 2), (u & 3, (u & 3) + 1, 2), (u >> 2, (u >> 2) + 1, 2)]
    s = oracle.port().encode_triples(*zip(*triples))
    with pytest.raises(oracle.OracleError, match="offset overflows"):
      O.decode(s, np.zeros(1, np.int32), cdf, [4], [U.INT32_MAX], 5, 2)


def test_damaged_strings_decode_alike():
  if not ubi.have_ref():
    pytest.skip("compiled reference not built")
  rng = np.random.default_rng(11)
  R, P = ubi.ref(), ubi.port()
  for p, w in ((14, 3), (8, 1), (16, 16), (5, 2)):
    data, index, cdf, cdf_size, offset = _case(rng, p, w, 6, 20, 400, True)
    good = R.encode(data, index, cdf, cdf_size, offset, p, w)
    damaged = [good[:len(good) // 2], b"", rng.bytes(len(good))]
    flipped = bytearray(good)
    for _ in range(3):
      flipped[rng.integers(len(good))] ^= 1 << int(rng.integers(8))
    damaged.append(bytes(flipped))
    for s in damaged:
      res = []
      for O in (R, P):
        try:
          res.append(O.decode(s, index, cdf, cdf_size, offset, p, w))
        except oracle.OracleError as e:
          res.append(str(e))
      if isinstance(res[0], str) or isinstance(res[1], str):
        assert res[0] == res[1]
      else:
        assert np.array_equal(res[0], res[1])


def test_debug_checks_in_reference_order():
  cdf = np.array([[0, 16, 18, 32], [0, 1, 2, 32]], np.int32)
  for O in flavours():
    f = lambda **kw: O.encode(
        np.zeros(2, np.int32), kw.get("index", np.zeros(2, np.int32)), kw.get("cdf", cdf),
        kw.get("cdf_size", np.array([4, 4], np.int32)), np.ones(2, np.int32), 5, 2)
    for kw, msg in ((dict(index=np.array([0, 2], np.int32)), "'index' has a value not in"),
                    (dict(cdf_size=np.array([4, 5], np.int32)), "'cdf_size' has a value not in"),
                    (dict(cdf=np.array([[1, 16, 18, 32], [0, 1, 2, 32]], np.int32)), "cdf[0]="),
                    (dict(cdf=np.array([[0, 18, 16, 32], [0, 1, 2, 32]], np.int32)), "monotonic"),
                    (dict(index=np.array([0, 5], np.int32), cdf_size=np.array([1, 4], np.int32)), "'index'")):
      with pytest.raises(oracle.OracleError, match=msg.replace("[", r"\[").replace("^", r"\^")):
        f(**kw)
