"""Oracle of the mixture coder (DESIGN.md §3.18).

  cdf_from_masses  the exact integer map from masses m_0 .. m_L to the quantised CDF c_0 .. c_n (Python ints);
  masses_f64       float64 masses 2^32 * P(bin) of a mixture over a given support (scipy), to bound the device's;
  support_f32      the support (a, L) restated in numpy float32, expression for expression;
  lookup           the padded 2-D lookup [-p, c_0 .. c_n, 2^p ...] the compiled reference coder takes.
"""
import math

import numpy as np
from scipy import stats

FAMILIES = ("normal", "logistic")
TWO32 = 1 << 32


def quantile(family, tail_mass):
  """The family's upper quantile at tail_mass / 2, as float32 (the coder's t)."""
  if family == "logistic":
    return np.float32(math.log(2.0 / tail_mass - 1.0))
  return np.float32(stats.norm.isf(tail_mass / 2))


def cdf_from_masses(masses, precision):
  """c_0 .. c_n from m_0 .. m_L (n = L + 1): c_j = j + floor((2^p - n) S_j / T), S_j = sum_{i<j} m_i, T = S_n."""
  m = [int(x) for x in masses]
  n = len(m)
  T = sum(m)
  if T <= 0 or (1 << precision) < n:
    raise ValueError("masses must have a positive sum and at most 2^precision bins")
  out, S = [0], 0
  for j in range(1, n + 1):
    S += m[j - 1]
    out.append(j + ((1 << precision) - n) * S // T)
  return out


def escape_mass(bin_masses):
  """m_L = max(0, 2^32 - sum of the support's masses)."""
  return max(0, TWO32 - sum(int(x) for x in bin_masses))


def lookup(rows_cdf, precision, max_support):
  """int32 [rows, max_support + 3]: [-p, c_0 .. c_n] padded with 2^p."""
  out = np.full((len(rows_cdf), max_support + 3), 1 << precision, dtype=np.int32)
  out[:, 0] = -precision
  for r, c in enumerate(rows_cdf):
    out[r, 1:1 + len(c)] = c
  return out


def support_f32(family, w, mu, sg, tail_mass, max_support):
  """(a, L) of one element, with the coder's float32 expressions (numpy float32 arithmetic rounds to nearest)."""
  f = np.float32
  t = quantile(family, tail_mass)
  W = f(0)
  for x in w:
    W = f(W + f(x))
  winv = f(f(1) / W)
  lo, hi, mean = f(np.inf), f(-np.inf), f(0)
  for wk, mk, sk in zip(w, mu, sg):
    if not f(wk) > 0:
      continue
    ts = f(t * f(sk))
    lo = min(lo, f(f(mk) - ts))
    hi = max(hi, f(f(mk) + ts))
    mean = f(mean + f(f(f(wk) * winv) * f(mk)))
  af = f(np.floor(lo))
  width = f(f(f(np.ceil(hi)) - af) + f(1))
  if width <= max_support:
    L = int(width)
  else:
    L = max_support
    af = f(f(np.rint(mean)) - f((max_support - 1) // 2))
  a = int(min(max(af, f(-2**30)), f(2**30)))
  return a, L


def masses_f64(family, w, mu, sg, a, L):
  """2^32 * P(x) for x = a .. a + L - 1 under the normalised mixture, in float64.  Each component's bin probability
  is taken on the side of its median away from the bin (survival function above it), so neither tail cancels."""
  w = np.asarray(w, np.float64)
  w = w / w.sum()
  x = np.arange(a, a + L, dtype=np.float64)[:, None]
  mu = np.asarray(mu, np.float64)[None, :]
  sg = np.asarray(sg, np.float64)[None, :]
  zl, zh = (x - 0.5 - mu) / sg, (x + 0.5 - mu) / sg
  dist = stats.norm if family == "normal" else stats.logistic
  above = (x - mu) > 0
  p = np.where(above, dist.sf(zl) - dist.sf(zh), dist.cdf(zh) - dist.cdf(zl))
  return TWO32 * (p * w[None, :]).sum(axis=1)


def masses_bound(family, w, mu, sg, a, L):
  """(masses_f64, bound on |device mass - masses_f64|) in units of 2^-32 (DESIGN.md §3.18): 2^-16 of the mass for
  the float32 quotients, products and CDF evaluations, 2^-20 of 2^32 for the float32 CDF differences near 1/2 (where
  the CDF values themselves carry an ulp of 2^-25), and one unit for the truncation."""
  want = masses_f64(family, w, mu, sg, a, L)
  return want, 2.0**-16 * want + 2.0**-20 * TWO32 + 1.0
