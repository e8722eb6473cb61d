"""CPU: the float64 rate-term reference (oracle/likelihood_oracle.py) that tests/test_likelihood_bounds_gpu.py holds
the kernels to.

* Against 50 digits: in every regime of tests/likelihood_cases.py the reference's value and gradients are within
  2^-20 float32 ulp + 2^-40 M of the mpmath value, so a kernel within half an ulp of the reference returns the
  correctly rounded float32 value except where that value lies in this band around a rounding midpoint.
* Against the graph: on float64 priors the reference gives `_log_prob_graph`'s values and gradients (through the
  packing, for the raw parameters) and its NaN / inf masks.
* The restated CTA geometry gives the library's workspace size at every shape the GPU file uses."""
import numpy as np
import pytest
import torch

import likelihood_cases as cases
from compression_b200 import _lib
from compression_b200 import distributions as D
from oracle import likelihood_oracle as L

INF, NAN = float("inf"), float("nan")
BASES = {"normal": D.NoisyNormal, "logistic": D.NoisyLogistic, "laplace": D.NoisyLaplace}


def _within_50_digits(name, ref, exact, M):
  ref, exact, M = (np.asarray(v, dtype=np.float64) for v in (ref, exact, M))
  err = np.abs(ref - exact)
  bar = 2.0**-20 * cases.ulp32(exact) + L.EPS_BAR * M
  bad = ~(err <= bar)
  assert not bad.any(), (f"{name}: {int(bad.sum())} of {bad.size} beyond the bar, e.g. ref {ref[bad][:3]} exact "
                         f"{exact[bad][:3]} M {M[bad][:3]}")


@pytest.mark.parametrize("regime", cases.DF_REGIMES)
def test_deep_factorized_reference_against_50_digits(regime):
  C, rows = 6, 70
  packed = cases.df_packed(C, regime, 11)
  y = cases.df_y(packed, rows, 12)
  dout = torch.ones(rows, C)
  ref = L.df_reference(y, packed, dout)
  contrib, M_contrib = L.df_contributions(y, packed, dout)
  exact = [[L.mp_df(packed[c].tolist(), float(y[r, c])) for c in range(C)] for r in range(rows)]
  _within_50_digits("log p", ref["logp"], [[float(e[0]) for e in row] for row in exact], ref["M_logp"])
  _within_50_digits("dy", ref["dy"], [[float(e[1]) for e in row] for row in exact], ref["M_dy"])
  _within_50_digits("dpacked", contrib, [[[float(v) for v in e[2]] for e in row] for row in exact], M_contrib)


@pytest.mark.parametrize("base", list(BASES))
def test_location_scale_reference_against_50_digits(base):
  y, loc, scale = cases.ls_inputs(600, 21)
  ref = L.loc_scale_reference(base, y, loc, scale, torch.ones_like(y))
  exact = np.array([[float(v) for v in L.mp_loc_scale(base, *t)] for t in zip(y.tolist(), loc.tolist(),
                                                                              scale.tolist())])
  _within_50_digits("log p", ref["logp"], exact[:, 0], ref["M_logp"])
  _within_50_digits("dy", ref["dy"], exact[:, 1], ref["M_dy"])
  _within_50_digits("dloc", ref["dloc"], exact[:, 2], ref["M_dy"])
  _within_50_digits("dscale", ref["dscale"], exact[:, 3], ref["M_dscale"])


def test_location_scale_regimes_are_reached():
  y, loc, scale = (t.double() for t in cases.ls_inputs(6000, 21))
  z_p, z_m = (y + .5 - loc) / scale, (y - .5 - loc) / scale
  z = torch.cat([z_p, z_m])
  assert bool((z == -1).any()) and bool(((z > -1) & (z < -1 + 1e-6)).any()) and bool(((z < -1) & (z > -1 - 1e-6)).any())
  assert bool((z.abs() > 37).any()) and bool((z.abs() > 745).any()) and bool((z.abs() > 39).any())
  assert bool((z == 0).any()) and bool(((z != 0) & (z.abs() < 1e-6)).any())
  assert float(scale.min()) < 0.011 and float(scale.max()) > 9000 and bool((scale == np.float32(0.11)).any())


def _equal_masks(name, a, b):
  assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{name}: NaN mask"
  assert torch.equal(torch.isinf(a) & (a > 0), torch.isinf(b) & (b > 0)), f"{name}: +inf mask"
  assert torch.equal(torch.isinf(a) & (a < 0), torch.isinf(b) & (b < 0)), f"{name}: -inf mask"


def _close(name, a, b, M):
  """1e-14 of the value plus 1e-15 of its M (for a gradient, at least 16 times the sum of |terms|)."""
  _equal_masks(name, a, b)
  fin = torch.isfinite(b)
  tol = 1e-14 * b[fin].abs() + 1e-15 * M[fin]
  err = (a - b)[fin].abs()
  assert not bool((err > tol).any()), (name, float((err / tol).max()))


def _tensor_close(name, a, b, rtol):
  """Sums over rows: relative to the tensor's largest magnitude."""
  _equal_masks(name, a, b)
  fin = torch.isfinite(b)
  assert float((a - b)[fin].abs().max()) <= rtol * float(b[fin].abs().max()), name


@pytest.mark.parametrize("regime", ["random", "trained"])
def test_deep_factorized_reference_is_the_graph(regime):
  C, rows = 5, 64
  p = D.NoisyDeepFactorized(batch_shape=(C,), dtype=torch.float64)
  packed32 = cases.df_packed(C, regime, 3)
  with torch.no_grad():  # raw parameters with those transformed values
    b = p.base
    for m, sl in zip(b.matrices, (slice(0, 3), slice(3, 12), slice(12, 15))):
      m.copy_(torch.log(torch.expm1(packed32[:, sl].double())).reshape(m.shape))
    for t, sl in zip(b.biases, (slice(15, 18), slice(18, 21), slice(21, 22))):
      t.copy_(packed32[:, sl].double().reshape(t.shape))
    for t, sl in zip(b.factors, (slice(22, 25), slice(25, 28))):
      t.copy_(torch.atanh(packed32[:, sl].double()).reshape(t.shape))
  y = cases.df_y(packed32, rows, 4).double()
  y[0, 0], y[1, 1], y[2, 2], y[3, 3], y[4, 4] = INF, -INF, NAN, -0.0, 0.0
  dout = torch.randn(rows, C, dtype=torch.float64, generator=torch.Generator().manual_seed(5))
  params = list(p.parameters())
  yy = y.clone().requires_grad_(True)
  want = p._log_prob_graph(yy)
  g = torch.autograd.grad(want, [yy] + params, dout)
  packed = b._packed_parameters()
  ref = L.df_reference(y, packed, dout)
  raw = torch.autograd.grad(packed, params, ref["dpacked"])
  _close("log p", ref["logp"], want.detach(), ref["M_logp"])
  _close("dy", ref["dy"], g[0], ref["M_dy"])
  # rows without non-finite y: the channels that have one get NaN gradients in both
  for i, (u, v) in enumerate(zip(raw, g[1:])):
    _tensor_close(f"param {i}", u, v, 1e-13)
  assert bool(torch.isnan(g[1]).any())  # the channels with a non-finite y


@pytest.mark.parametrize("base", list(BASES))
def test_location_scale_reference_is_the_graph(base):
  y, loc, scale = (t.double() for t in cases.ls_inputs(3000, 8))
  y[:3], loc[3:6], scale[6:9] = torch.tensor([INF, -INF, NAN]), torch.tensor([INF, -INF, NAN]), torch.tensor(
      [INF, NAN, 0.11])
  dout = torch.randn(y.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
  lo, sc, yy = loc.clone().requires_grad_(True), scale.clone().requires_grad_(True), y.clone().requires_grad_(True)
  want = BASES[base](lo, sc, dtype=torch.float64)._log_prob_graph(yy)
  g = torch.autograd.grad(want, [yy, lo, sc], dout)
  ref = L.loc_scale_reference(base, y, loc, scale, dout)
  _close("log p", ref["logp"], want.detach(), ref["M_logp"])
  _close("dy", ref["dy"], g[0], ref["M_dy"])
  _close("dloc", ref["dloc"], g[1], ref["M_dy"])
  _close("dscale", ref["dscale"], g[2], ref["M_dscale"])


def _df_shapes():
  for C in cases.DF_CHANNELS:
    for rows in cases.df_row_counts(C):
      yield C, rows
  yield from cases.DF_LARGE


def test_workspace_size_is_the_restated_geometry():
  lib = _lib.lib()
  for C, rows in _df_shapes():
    assert lib.tfcb_noisy_deep_factorized_workspace_bytes(rows * C, C) == L.df_workspace_bytes(rows * C, C), (C, rows)


def test_large_shapes_pass_the_grid_stride_thresholds():
  """Forward rows > (8192 // chunks) subrows, backward rows > (512 // chunks) subrows 4: some thread walks a second
  row (forward) or more than 4 rows (backward); the small shapes stay in one pass."""
  fwd = bwd = False
  for C, rows in cases.DF_LARGE:
    g = L.df_geometry(rows * C, C, False)
    fwd |= rows > (8192 // g["chunks"]) * g["subrows"]
    bwd |= rows > (512 // g["chunks"]) * g["subrows"] * 4
  assert fwd and bwd
  for C in cases.DF_CHANNELS:
    g = L.df_geometry(C, C, True)
    assert g["subrows"] * g["cpb"] <= 256 and g["chunks"] * g["cpb"] >= C
    assert cases.df_row_counts(C)[0] <= max(1, g["subrows"])
