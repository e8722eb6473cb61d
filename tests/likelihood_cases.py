"""Inputs shared by tests/test_likelihood_oracle_cpu.py and tests/test_likelihood_bounds_gpu.py: the deep-factorized
parameter regimes, the y and loc / scale sets that reach each regime of the rate-term kernels, and the channel counts
and row counts that reach each CTA geometry of `noisy_df_fwd_kernel` / `noisy_df_bwd_kernel`."""
import numpy as np
import torch

from compression_b200 import distributions as D
from oracle import likelihood_oracle as L

# cpb = C and subrows 256 .. 1; CTAs of 85 / 255 threads (not a multiple of 32); idle lanes at 129, 257, 513;
# 2 to 4 channel chunks from 257 up
DF_CHANNELS = [1, 2, 3, 85, 86, 100, 128, 129, 192, 255, 256, 257, 320, 384, 511, 512, 513, 1000]
# (C, rows) past the grid-stride thresholds: forward rows > (8192 // chunks) * subrows, backward rows >
# (512 // chunks) * subrows * 4; bls2017's y [64, 16, 16, 128] and bmshj2018's z [64, 4, 4, 192]
DF_LARGE = [(1, 2_200_000), (320, 4_500), (192, 5_000), (320, 3_000), (128, 64 * 16 * 16), (192, 64 * 4 * 4)]
DF_REGIMES = ["init", "random", "trained"]


def df_row_counts(C):
  """One row count below the CTA's sub-row count (1 where that is 1) and one that is not a multiple of it."""
  s = L.df_geometry(C, C, False)["subrows"]
  return [max(1, s // 2 + 1), 3 * s + 5]


def ulp32(r):
  """np.spacing(float32(|r|)) in float64."""
  return np.spacing(np.abs(np.asarray(r, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def df_packed(C, regime, seed):
  """Packed [C, 28] float32 parameters: the prior at initialisation, random as tests/test_likelihood_gpu.py draws
  them, or trained-like: softplus(matrices) log-uniform in [0.01, 50] (steep CDFs), biases in +-40 (the median far
  from 0), tanh(factors) in +-0.95."""
  torch.manual_seed(seed)
  if regime == "init":
    return D.NoisyDeepFactorized(batch_shape=(C,)).base._packed_parameters().detach().float()
  rng = np.random.default_rng(seed)
  if regime == "random":
    m = np.log1p(np.exp(np.log(np.expm1(10**(-1 / 3) / np.array([3.] * 12 + [1.] * 3))) + 0.5 * rng.normal(size=(C, 15))))
    b, f = rng.normal(size=(C, 7)), np.tanh(rng.normal(size=(C, 6)))
  else:
    m = np.exp(rng.uniform(np.log(0.01), np.log(50), (C, 15)))
    b, f = rng.uniform(-40, 40, (C, 7)), rng.uniform(-0.95, 0.95, (C, 6))
  return torch.tensor(np.concatenate([m, b, f], 1), dtype=torch.float32)


def df_medians(packed):
  """Per channel, the x where the CDF logits cross 0 (bisection in float64; l is increasing in x)."""
  w = L.df_params(packed.cpu())
  lo = torch.full((packed.shape[0],), -1e7, dtype=torch.float64)
  hi = -lo
  for _ in range(120):
    mid = (lo + hi) / 2
    up = L._mlp(w, mid) > 0
    hi, lo = torch.where(up, mid, hi), torch.where(up, lo, mid)
  return lo


def df_y(packed, rows, seed):
  """float32 y [rows, C]: a grid across the +-1/2 bin edges, bin centres, each channel's median and median -+ 1/2
  (l(y + 1/2) or l(y - 1/2) at 0: ties in the select), +-0, |y| log-uniform up to 1e4, and N(0, 6)."""
  C = packed.shape[0]
  g = np.random.default_rng(seed)
  n = rows * C
  k = np.arange(n)
  kind = (k // C * 7 + k % C) % 8
  grid = (g.integers(-40, 41, n) * 0.5 + np.array([0, 1e-6, -1e-6, 1e-3, -1e-3, .25, .5 - 2**-24, 0])[g.integers(0, 8, n)])
  centres = g.integers(-20, 21, n).astype(np.float64)
  med = np.tile(df_medians(packed).numpy(), rows)
  median = med + np.array([0, .5, -.5])[g.integers(0, 3, n)]
  signed_zero = np.where(g.random(n) < .5, 0.0, -0.0)
  tails = np.sign(g.random(n) - .5) * 10**(g.random(n) * 4)
  normal = g.normal(size=n) * 6
  y = np.select([kind == i for i in range(7)], [grid, centres, median, signed_zero, tails, normal, grid], normal)
  return torch.tensor(y.astype(np.float32).reshape(rows, C))


def ls_inputs(n, seed):
  """float32 (y, loc, scale), each [n], in blocks that reach every regime of the three bases:
    * general: y on a grid and N(0, 30), loc N(0, 2), scale log-uniform in [1e-2, 1e4] and the 0.11 the models use;
    * z = (y +- 1/2 - loc) / scale on both sides of log_ndtr's switch at -1, exactly -1, and |z| up to 40;
    * |z| beyond 37 (exp(-|z|) below eps) and beyond 745 (exp(-|z|) underflows);
    * z = 0 exactly (Laplace's abs at 0) and +-tiny (loc one float32 ulp from y + 1/2)."""
  g = np.random.default_rng(seed)
  k = np.arange(n)
  scale = np.exp(g.uniform(np.log(1e-2), np.log(1e4), n))
  scale[k % 11 == 0] = np.float32(0.11)
  y = np.where(k % 3 == 0, g.normal(size=n) * 30, g.integers(-80, 81, n) * .5 + g.choice([0, 1e-6, -1e-6, .25], n))
  loc = g.normal(size=n) * 2
  kind = k % 6
  # target z at y + 1/2: |z| up to 40 with a dense band around -1, or beyond 37 / 745
  z = np.where(g.random(n) < .5, g.uniform(-40, 40, n), -1 + g.uniform(-1e-3, 1e-3, n) * g.choice([1, 1e-6], n))
  z = np.where(kind == 2, np.sign(g.random(n) - .5) * np.exp(g.uniform(np.log(37), np.log(3000), n)), z)
  aim = np.isin(kind, (1, 2))
  loc = np.where(aim, y + .5 - z * scale, loc)
  # z exactly -1 at y - 1/2 or y + 1/2: power-of-two scale, y on the half-integer grid
  exact = kind == 3
  sc2 = 2.0**g.integers(-6, 8, n)
  side = g.choice([.5, -.5], n)
  scale = np.where(exact, sc2, scale)
  y = np.where(exact, g.integers(-40, 41, n) * .5, y)
  loc = np.where(exact, y + side + sc2, loc)
  # z = 0 and +-tiny
  zero = kind == 4
  y = np.where(zero, g.integers(-40, 41, n) * .5 + g.choice([0, .25], n), y)
  y32 = y.astype(np.float32)
  at = (y32.astype(np.float64) + g.choice([.5, -.5], n)).astype(np.float32)
  nudge = g.integers(-1, 2, n)
  toward = np.where(nudge > 0, np.float32(np.inf), np.float32(-np.inf))
  loc = np.where(zero, np.where(nudge == 0, at, np.nextafter(at, toward)), loc)
  return (torch.tensor(y32), torch.tensor(loc.astype(np.float32)), torch.tensor(scale.astype(np.float32)))
