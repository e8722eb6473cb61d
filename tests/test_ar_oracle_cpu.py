"""The CPU references of the autoregressive prior's parameter network (oracle/ar_oracle.py), checked without a GPU:
fma32 is correctly rounded, the float32 emulation stays within the derived bound of the float64 restatement, and
each plausible mistake in the kernel's order (a dropped term, another slice split, wrapped taps, the bias added
last, a float64 slope) changes the emulation's bits -- so the GPU test, which demands bit equality, would see it."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import ar_oracle as A

SHAPES = [(1, 1), (1, 4), (4, 1), (2, 2), (3, 5), (6, 9)]


def _weights(M, seed):
  """test_mbt2018_gpu._weights on the CPU: loc of a few units and scale indexes spread over the table range."""
  g = torch.Generator().manual_seed(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: torch.randn(*s, generator=g)
  b3 = torch.cat([0.5 * r(M), 24 + 4 * r(M)])
  return [r(5, 5, M, 2 * M) / math.sqrt(12 * M), 0.1 * r(2 * M), r(4 * M, n3) / math.sqrt(4 * M), 0.1 * r(n3),
          r(n3, n4) / math.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * M) / math.sqrt(n4), b3]


def _inputs(B, H, W, M, seed):
  rng = np.random.default_rng(seed)
  return (3 * rng.standard_normal((B, H, W, M))).astype(np.float32), \
      rng.standard_normal((B, H, W, 2 * M)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# fma32 against exact rational arithmetic
# ---------------------------------------------------------------------------------------------------------------
def _round32(v):
  """A nonzero Fraction rounded to the nearest float32, ties to even, with subnormals and overflow to inf."""
  sgn = -1 if v < 0 else 1
  a = abs(v)
  e = a.numerator.bit_length() - a.denominator.bit_length()
  if a < Fraction(2)**e:
    e -= 1
  q = Fraction(2)**(max(e, -126) - 23)  # the float32 quantum at this magnitude
  m = a / q
  n = m.numerator // m.denominator
  rem = m - n
  if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2):
    n += 1
  r = n * q
  return np.float32(sgn * (math.inf if r >= Fraction(2)**128 else float(r)))


def _exact_fma32(a, b, c):
  a, b, c = (np.float32(t) for t in (a, b, c))
  v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
  if v == 0:  # IEEE: an exact zero sum is +0 under round-to-nearest unless both addends are -0
    p_neg = bool(np.signbit(a)) != bool(np.signbit(b))
    both_neg = a * b == 0 and c == 0 and p_neg and bool(np.signbit(c))
    return np.float32(-0.0) if both_neg else np.float32(0.0)
  return _round32(v)


def _fma_cases():
  rng = np.random.default_rng(0)
  f = lambda x: np.asarray(x, np.float32)
  n = 6000
  # random magnitudes and signs
  ra = f(rng.standard_normal(n) * 2.0**rng.integers(-20, 20, n))
  rb = f(rng.standard_normal(n) * 2.0**rng.integers(-20, 20, n))
  rc = f(rng.standard_normal(n) * 2.0**rng.integers(-30, 30, n))
  # near-cancellation: c within a few ulps of -a*b, or exactly -fl32(a*b) (the result is the product's rounding error)
  na, nb = f(rng.standard_normal(n)), f(rng.standard_normal(n))
  nc = f(-(na.astype(np.float64) * nb) * (1 + rng.standard_normal(n) * 2.0**-22))
  nc[::2] = -(na[::2] * nb[::2])
  # subnormal operands and results, operands of different signs
  sa = f(rng.standard_normal(n) * 2.0**rng.integers(-75, -60, n))
  sb = f(rng.standard_normal(n) * 2.0**rng.integers(-75, -60, n))
  sc = f(rng.standard_normal(n) * 2.0**rng.integers(-149, -125, n))
  sc[::3] = f(rng.standard_normal(n // 3) * 2.0**-140)
  # signed zeros
  z = [(0.0, 1.5, 0.0), (-0.0, 1.5, 0.0), (-0.0, 1.5, -0.0), (0.0, -1.5, -0.0), (-0.0, -1.5, -0.0),
       (2.0, 3.0, -6.0), (-2.0, 3.0, 6.0), (1e-30, 1e-30, -0.0), (-1e-30, 1e-30, -0.0), (1e-30, 1e-30, 0.0),
       (2.0**-75, 2.0**-75, 0.0), (-(2.0**-75), 2.0**-76, -0.0), (2.0**-149, 0.5, 0.0), (3 * 2.0**-149, 0.5, -0.0)]
  za, zb, zc = (f([t[i] for t in z]) for i in range(3))
  return (np.concatenate([ra, na, sa, za]), np.concatenate([rb, nb, sb, zb]), np.concatenate([rc, nc, sc, zc]))


def test_fma32_is_correctly_rounded():
  a, b, c = _fma_cases()
  assert a.size >= 10**4
  got = A.fma32(a, b, c)
  want = np.array([_exact_fma32(*t) for t in zip(a, b, c)], np.float32)
  bad = np.flatnonzero(got.view(np.int32) != want.view(np.int32))
  assert bad.size == 0, [(a[i], b[i], c[i], got[i], want[i]) for i in bad[:5]]
  # the sets reach what they are meant to: subnormal results, exact zeros of both signs
  tiny = np.abs(want) < np.float32(2.0**-126)
  assert np.count_nonzero(tiny & (want != 0)) > 100
  assert np.any((want == 0) & np.signbit(want)) and np.any((want == 0) & ~np.signbit(want))


def test_fma32_avoids_the_double_rounding_of_float64():
  # a*b + c = 1 + 2^-24 + 2^-70: just above the float32 midpoint between 1 and 1 + 2^-23, so it rounds up; float64
  # rounds the sum onto the midpoint first, and the tie then goes to the even 1.0
  a, b, c = np.float32(-(1 + 2.0**-23)), np.float32(2.0**-24 * (1 - 2.0**-23)), np.float32(1 + 2.0**-23)
  exact = _exact_fma32(a, b, c)
  assert exact == np.float32(1 + 2.0**-23)
  naive = np.float32(float(a) * float(b) + float(c))
  assert naive == np.float32(1.0) and naive != exact
  assert A.fma32(a, b, c) == exact


# ---------------------------------------------------------------------------------------------------------------
# the float32 emulation within the derived bound of float64
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [6, 18, 30, 96])
def test_params32_is_within_the_derived_bound_of_float64(M):
  ws = _weights(M, 0)
  worst = 0.0
  for k, (H, W) in enumerate(SHAPES):
    y_hat, psi = _inputs(1, H, W, M, 10 * M + k)
    pos = list(range(H * W))
    loc, scale, index = A.params32(ws, y_hat, psi, pos, 64)
    loc64, scale64 = A.params64(ws, y_hat, psi, pos)
    bloc, bscale = A.bound64(ws, y_hat, psi, pos)
    for got, want, bound in ((loc, loc64, bloc), (scale, scale64, bscale)):
      err = np.abs(got.astype(np.float64) - want)
      assert np.all(err <= bound), (H, W, float((err - bound).max()))
    assert np.array_equal(index, A.table_index(scale, 64))
    # every layer within its own rounding bound, which is informative: 1e-4 of the layer's largest output
    for i, (err, bound, mag) in enumerate(A.layer_errors(ws, y_hat, psi, pos)):
      assert np.all(err <= bound), (H, W, i)
      assert bound.max() <= 1e-4 * mag.max(), (H, W, i, bound.max(), mag.max())
      worst = max(worst, err.max() / bound.max())
  assert worst > 1e-3  # the bounds are not vacuous: the observed error is a visible fraction of them


def test_bound64_is_informative_at_the_smallest_depth():
  # bound64 carries each layer's worst case through the following layers' Σ|W|; at M = 6 it stays near 1e-4 of the
  # output (at M = 96 it is ~10^3 times looser, which is why the per-layer check above exists)
  M = 6
  ws = _weights(M, 0)
  y_hat, psi = _inputs(1, 6, 9, M, 1)
  pos = list(range(54))
  _, scale64 = A.params64(ws, y_hat, psi, pos)
  bloc, bscale = A.bound64(ws, y_hat, psi, pos)
  assert max(bloc.max(), bscale.max()) <= 2e-4 * np.abs(scale64).max()


# ---------------------------------------------------------------------------------------------------------------
# mutations: what a bitwise comparison with the emulation catches
# ---------------------------------------------------------------------------------------------------------------
def _dense_ceil_slices(x, W, b, leaky):
  """ar_dense with ceil(K/8)-sized slices (the last ones shorter or empty) instead of s*K//8."""
  K = W.shape[0]
  n = -(-K // A.SLICES)
  acc = []
  for s in range(A.SLICES):
    p = np.zeros((x.shape[0], W.shape[1]), np.float32)
    for k in range(min(s * n, K), min((s + 1) * n, K)):
      p = A.fma32(x[:, k:k + 1], W[k][None], p)
    acc.append(p)
  v = np.broadcast_to(b, p.shape).astype(np.float32)
  for p in acc:
    v = v + p
  return np.where(v > 0, v, v * A.SLOPE32) if leaky else v


def _dense_bias_last(x, W, b, leaky):
  zero = np.zeros_like(b)
  v = A.dense32(x, W, zero, False) + b  # ((P_0 + ... + P_7) + bias): dense32 with a zero bias starts from +0
  return np.where(v > 0, v, v * A.SLOPE32) if leaky else v


def _dense_slope64(x, W, b, leaky):
  v = A.dense32(x, W, b, False)
  return np.where(v > 0, v, (v.astype(np.float64) * 0.01).astype(np.float32)) if leaky else v


def _dense_dropping(K_target, k_drop):
  """ar_dense that leaves term k_drop out of the layer whose input width is K_target."""
  def dense(x, W, b, leaky):
    if W.shape[0] != K_target:
      return A.dense32(x, W, b, leaky)
    keep = np.arange(W.shape[0]) != k_drop
    x2 = np.where(keep[None], x, np.float32(0))  # fma(0, w, acc) == acc for acc != -0 (never -0 here)
    return A.dense32(x2, W, b, leaky)
  return dense


def _taps_wrapping(y_hat, positions):
  """taps that read a right-hand neighbour past the row's end from the start of the next row (no xx < W test)."""
  y_hat = np.asarray(y_hat, np.float32)
  B, H, W, M = y_hat.shape
  flat = y_hat.reshape(B, H * W, M)
  out = np.zeros((B, len(positions), A.TAPS, M), np.float32)
  for i, p in enumerate(positions):
    py, px = divmod(int(p), W)
    for t in range(A.TAPS):
      yy, xx = py + t // 5 - 2, px + t % 5 - 2
      if yy >= 0 and xx >= 0 and 0 <= yy * W + xx < H * W:
        out[:, i, t] = flat[:, yy * W + xx]
  return out.reshape(B, len(positions), A.TAPS * M)


def _all_shapes(M, fn):
  """fn(ws, y_hat, psi, positions) over every position of every shape, at depth M."""
  ws = _weights(M, 0)
  for k, (H, W) in enumerate(SHAPES):
    y_hat, psi = _inputs(1, H, W, M, 100 + k)
    yield fn(ws, y_hat, psi, list(range(H * W)))


@pytest.mark.parametrize("M", [6, 18])
@pytest.mark.parametrize("name", ["ceil_slices", "bias_last", "slope64"])
def test_a_wrong_order_changes_the_bits(M, name):
  dense = {"ceil_slices": _dense_ceil_slices, "bias_last": _dense_bias_last, "slope64": _dense_slope64}[name]

  def differs(ws, y_hat, psi, pos):
    want = A.params32(ws, y_hat, psi, pos, 64)[:2]
    got = A.params32(ws, y_hat, psi, pos, 64, dense=dense)[:2]
    return any(not np.array_equal(g.view(np.int32), w.view(np.int32)) for g, w in zip(got, want))
  assert any(_all_shapes(M, differs))


@pytest.mark.parametrize("M", [6, 18])
@pytest.mark.parametrize("name", ["dropped_term", "wrapped_taps"])
def test_a_wrong_term_changes_the_bits_and_exceeds_the_float64_bound(M, name):
  n3 = 10 * M // 3
  if name == "dropped_term":  # one k of slice 3 of W2, whose input h1 is nonzero at every tested position
    kwargs = {"dense": _dense_dropping(n3, 3 * n3 // 8 + 1)}
  else:
    kwargs = {"gather": _taps_wrapping}

  def check(ws, y_hat, psi, pos):
    want = A.params32(ws, y_hat, psi, pos, 64)[:2]
    got = A.params32(ws, y_hat, psi, pos, 64, **kwargs)[:2]
    exact = A.params64(ws, y_hat, psi, pos)
    bound = A.bound64(ws, y_hat, psi, pos)
    bits = any(not np.array_equal(g.view(np.int32), w.view(np.int32)) for g, w in zip(got, want))
    beyond = any(np.any(np.abs(g.astype(np.float64) - e) > b) for g, e, b in zip(got, exact, bound))
    return bits, beyond
  results = list(_all_shapes(M, check))
  assert any(r[0] for r in results) and any(r[1] for r in results)


@pytest.mark.parametrize("M", [6, 18])
def test_the_dropped_term_is_nonzero(M):
  n3 = 10 * M // 3
  ws = _weights(M, 0)
  for k, (H, W) in enumerate(SHAPES):
    y_hat, psi = _inputs(1, H, W, M, 100 + k)
    pos = list(range(H * W))
    x = A.taps(y_hat, pos).reshape(H * W, -1)
    wc, bc, w1, b1 = A.unpack(ws)[:4]
    h1 = A.dense32(np.concatenate([A._psi_rows(psi, pos)[0], A.dense32(x, wc, bc, False)], -1), w1, b1, True)
    assert np.all(h1[:, 3 * n3 // 8 + 1] != 0)


# ---------------------------------------------------------------------------------------------------------------
# table indexes
# ---------------------------------------------------------------------------------------------------------------
def test_table_index_at_its_edges():
  ns = 64
  f = np.float32
  cases = [(-np.inf, 0), (-1e30, 0), (-1.5, 0), (-0.0, 0), (0.0, 0), (0.49, 0), (ns - 1, ns - 1), (ns - 0.5, ns - 1),
           (ns, ns - 1), (1e30, ns - 1), (np.inf, ns - 1), (np.nan, 0), (1.99, 1), (62.999996, 62)]
  s = np.array([c[0] for c in cases], f)
  assert A.table_index(s, ns).tolist() == [c[1] for c in cases]
  assert A.table_index(s, 17).tolist() == [min(c[1], 16) for c in cases]
  assert A.table_index(s, 1).tolist() == [0] * len(cases)
  assert A.table_index(s, ns).dtype == np.int32


def test_rint_to_int32_saturates_like_the_gpu():
  d = np.array([0.5, 1.5, 2.5, -0.5, -2.5, 2.0**31, -2.0**31, 3e9, -3e9, np.inf, -np.inf, np.nan, 2.0**31 - 128],
               np.float32)
  assert A.rint_to_int32(d).tolist() == [0, 2, 2, 0, -2, 2**31 - 1, -2**31, 2**31 - 1, -2**31, 2**31 - 1, -2**31,
                                         0, 2**31 - 128]
