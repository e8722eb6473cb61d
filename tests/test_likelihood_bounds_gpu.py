"""GPU: the fused rate-term kernels (csrc/likelihood.cu) against the float64 reference (oracle/likelihood_oracle.py),
element by element, at every CTA geometry of the deep-factorized kernels, past both grid-stride thresholds, at the
training shapes and in every regime of tests/likelihood_cases.py.

The kernels compute each element in double from the float32 inputs and round once, so they return float32(r) for the
reference value r unless r lies within the reference's own error of a rounding midpoint.  With
ulp32(r) = np.spacing(float32(|r|)):
  * log p, dy, dloc, dscale: |k - r| <= ulp32(r) / 2 + 2^-20 ulp32(r) + 2^-40 M;
  * the packed parameters' gradient: |k - r| <= ulp32(r) / 2 + sum over CTAs of ulp32(partial) / 2 + 2^-40 M, each
    CTA's partial row being rounded to float32 once and everything else summed in double;
  * a broadcast-scalar operand's gradient, summed in double from the float32 elementwise terms: ulp32(r) / 2 + the sum
    of the terms' own bars;
  * NaN and +-inf masks equal the reference's.
No element is excluded.  Each test reports how many elements fell in the midpoint band (k != float32(r))."""
import functools

import pytest
import torch

import likelihood_cases as cases
from compression_b200 import functional
from oracle import likelihood_oracle as L

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
INF, NAN = float("inf"), float("nan")
BASES = ["normal", "logistic", "laplace"]
BAND = {"elements": 0, "band": 0}


@pytest.fixture(scope="module", autouse=True)
def _report():
  yield
  print(f"\nrate-term bounds: {BAND['elements']} elements checked, {BAND['band']} in the midpoint band")


def _ulp32(r):
  f = r.abs().float()
  return (torch.nextafter(f, torch.full_like(f, INF)).double() - f.double())


def _masks(name, k, r):
  assert torch.equal(torch.isnan(k), torch.isnan(r)), f"{name}: NaN mask differs from the reference's"
  assert torch.equal(torch.isinf(k) & (k > 0), torch.isinf(r) & (r > 0)), f"{name}: +inf mask differs"
  assert torch.equal(torch.isinf(k) & (k < 0), torch.isinf(r) & (r < 0)), f"{name}: -inf mask differs"


def _elementwise_bar(r, M):
  u = _ulp32(r)
  return 0.5 * u + 2.0**-20 * u + L.EPS_BAR * M


def _check(name, k, r, bar):
  """k: the kernel's float32 result; r: the float64 reference; bar: the allowed |k - r| per element."""
  k, r, bar = k.detach().reshape(-1), r.detach().reshape(-1), bar.detach().reshape(-1)
  _masks(name, k, r)
  fin = torch.isfinite(r)
  err = (k.double() - r).abs()
  bad = fin & ~(err <= bar)  # a NaN bar fails
  if bad.any():
    i = torch.nonzero(bad)[:4, 0]
    raise AssertionError(f"{name}: {int(bad.sum())} of {r.numel()} elements beyond the bar: kernel "
                         f"{k[i].tolist()} reference {r[i].tolist()} bar {bar[i].tolist()} at {i.tolist()}")
  BAND["elements"] += int(fin.sum())
  BAND["band"] += int((fin & (k != r.float())).sum())


# ---------------------------------------------------------------------------------------------------------------
# deep factorized
# ---------------------------------------------------------------------------------------------------------------
def _run_df(y, packed, seed):
  dout = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed)).to(dev)
  yl, pl = y.clone().requires_grad_(True), packed.clone().requires_grad_(True)
  out = functional.noisy_deep_factorized_log_prob(yl, pl)
  dy, dp = torch.autograd.grad(out, [yl, pl], dout)
  ref = L.df_reference(y, packed, dout, partials=True, chunk_elems=1 << 19)
  _check("log p", out, ref["logp"], _elementwise_bar(ref["logp"], ref["M_logp"]))
  _check("dy", dy, ref["dy"], _elementwise_bar(ref["dy"], ref["M_dy"]))
  bar = 0.5 * _ulp32(ref["dpacked"]) + 0.5 * _ulp32(ref["partials"]).sum(0) + L.EPS_BAR * ref["M_dpacked"]
  _check("dpacked", dp, ref["dpacked"], bar)


@pytest.mark.parametrize("regime", cases.DF_REGIMES)
@pytest.mark.parametrize("C", cases.DF_CHANNELS)
def test_deep_factorized_at_every_geometry(C, regime):
  packed = cases.df_packed(C, regime, C)
  for rows in cases.df_row_counts(C):
    _run_df(cases.df_y(packed, rows, rows).to(dev), packed.to(dev), C + rows)


@pytest.mark.parametrize("C,rows", cases.DF_LARGE)
def test_deep_factorized_past_the_grid_stride_thresholds(C, rows):
  """Threads that walk more than one pass of the forward grid or more than 4 rows of the backward's, and the rate
  term's training shapes; parameters trained-like at the training shapes, random elsewhere."""
  regime = "trained" if (C, rows) in cases.DF_LARGE[-2:] else "random"
  packed = cases.df_packed(C, regime, rows)
  _run_df(cases.df_y(packed, rows, C).to(dev), packed.to(dev), rows)


def test_deep_factorized_non_finite_inputs():
  C, rows = 6, 40
  packed = cases.df_packed(C, "random", 1)
  y = cases.df_y(packed, rows, 2)
  y[0, 0], y[1, 1], y[2, 2], y[3, 3], y[4, 4] = INF, -INF, NAN, INF, -0.0
  y, packed = y.to(dev), packed.to(dev)
  dout = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).to(dev)
  yl, pl = y.clone().requires_grad_(True), packed.clone().requires_grad_(True)
  out = functional.noisy_deep_factorized_log_prob(yl, pl)
  dy, dp = torch.autograd.grad(out, [yl, pl], dout)
  ref = L.df_reference(y, packed, dout)
  _check("log p", out, ref["logp"], _elementwise_bar(ref["logp"], ref["M_logp"]))
  _check("dy", dy, ref["dy"], _elementwise_bar(ref["dy"], ref["M_dy"]))
  _masks("dpacked", dp, ref["dpacked"])
  assert bool(torch.isnan(dp[:4]).any(1).all()) and bool(torch.isfinite(dp[4:]).all())


# ---------------------------------------------------------------------------------------------------------------
# location-scale
# ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _ls(n):
  y, loc, scale = cases.ls_inputs(n, n % 1000)
  if n > 64:  # +-inf and NaN in each operand
    y[:3], loc[3:6], scale[6:9] = torch.tensor([INF, -INF, NAN]), torch.tensor([INF, -INF, NAN]), torch.tensor(
        [INF, NAN, INF])
  return y, loc, scale


def _run_ls(base, y, loc, scale, seed):
  """loc / scale: y-shaped, or 0-d (handed over as broadcast views, as the priors do)."""
  dout = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed)).to(dev)
  lo, sc, yl = (t.clone().requires_grad_(True) for t in (loc, scale, y))
  out = functional.noisy_loc_scale_log_prob(base, yl, lo.expand(y.shape) if lo.dim() == 0 else lo,
                                            sc.expand(y.shape) if sc.dim() == 0 else sc)
  dy, dloc, dscale = torch.autograd.grad(out, [yl, lo, sc], dout)
  ref = L.loc_scale_reference(base, y, loc, scale, dout)
  _check("log p", out, ref["logp"], _elementwise_bar(ref["logp"], ref["M_logp"]))
  bar_dy = _elementwise_bar(ref["dy"], ref["M_dy"])
  _check("dy", dy, ref["dy"], bar_dy)
  for name, k, r, bar in (("dloc", dloc, ref["dloc"], bar_dy),
                          ("dscale", dscale, ref["dscale"], _elementwise_bar(ref["dscale"], ref["M_dscale"]))):
    if k.dim():
      _check(name, k, r, bar)
    else:  # the float32 terms summed in double, rounded once
      s = r.sum()
      _check(name + " (0-d sum)", k, s, 0.5 * _ulp32(s) + bar.sum())


@pytest.mark.parametrize("n", [1, 2**21 - 1, 2**21 + 1, 64 * 16 * 16 * 192])
@pytest.mark.parametrize("base", BASES)
def test_location_scale_full_operands(base, n):
  """2^21 elements is one pass of the 8192 x 256 grid; bmshj2018's y [64, 16, 16, 192] takes two."""
  y, loc, scale = _ls(n)
  _run_ls(base, y.to(dev), loc.to(dev), scale.to(dev), n)


@pytest.mark.parametrize("operands", ["loc", "scale", "both"])
@pytest.mark.parametrize("base", BASES)
def test_location_scale_scalar_operands(base, operands):
  """0-d loc and / or scale over 4 M elements: their gradients are 4 M float32 terms summed in double."""
  n = 1 << 22
  y, loc, scale = _ls(n)
  keep = torch.isfinite(y) & torch.isfinite(loc) & torch.isfinite(scale)
  y, loc, scale = (t[keep].to(dev) for t in (y, loc, scale))
  if operands in ("loc", "both"):
    loc = torch.tensor(0.3, device=dev)
  if operands in ("scale", "both"):
    scale = torch.tensor(0.11 if operands == "both" else 2.5, device=dev)
  _run_ls(base, y, loc, scale, 7)
