"""GPU: the fused rate-term kernels (csrc/likelihood.cu) behind UniformNoiseAdapter.log_prob.

The reference is the graph (`_log_prob_graph`) on a float64 copy of the prior with the same parameter values.  The
fused float32 result must be no worse than the float32 graph it replaces: per element
  |fused - ref64| <= max(2 |graph32 - ref64|, floor),
floor = 1e-6 max(1, |ref64|) for log p, dy, dloc, dscale and 2e-5 max|ref64| over each parameter tensor for the
deep-factorized parameter gradients.  NaN / inf masks of log p and dy equal the graph's."""
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import distributions as D
from compression_b200 import entropy_models as E

pytestmark = pytest.mark.gpu
dev = torch.device("cuda")
INF, NAN = float("inf"), float("nan")


def _check(name, fused, graph32, ref64, floor):
  f, g, r = fused.detach().double(), graph32.detach().double(), ref64.detach()
  assert f.shape == r.shape, name
  assert torch.equal(torch.isnan(f), torch.isnan(g)), f"{name}: NaN mask differs from the graph's"
  assert torch.equal(torch.isinf(f), torch.isinf(g)), f"{name}: inf mask differs from the graph's"
  assert torch.equal(torch.isinf(f) & (f > 0), torch.isinf(g) & (g > 0)), name
  fin = torch.isfinite(f) & torch.isfinite(r)
  err_f, err_g = (f - r).abs(), (g - r).abs()
  bar = torch.maximum(2 * err_g, floor)
  bad = fin & (err_f > bar)
  assert not bad.any(), (f"{name}: {int(bad.sum())} elements worse than the graph, e.g. fused {f[bad][:3].tolist()} "
                         f"graph {g[bad][:3].tolist()} ref {r[bad][:3].tolist()}")


def _elem_floor(r):
  return 1e-6 * r.detach().abs().clamp(min=1)


def _grads(fn, y, params, dout):
  y = y.detach().clone().requires_grad_(True)
  out = fn(y)
  gs = torch.autograd.grad(out, [y] + list(params), dout, allow_unused=True)
  return out.detach(), gs[0], gs[1:]


# ---------------------------------------------------------------------------------------------------------------
# deep factorized
# ---------------------------------------------------------------------------------------------------------------
def _df(C, seed, random=True):
  torch.manual_seed(seed)
  p = D.NoisyDeepFactorized(batch_shape=(C,), device=dev)
  if random:
    with torch.no_grad():
      for m in p.base.matrices:
        m.add_(0.5 * torch.randn_like(m))
      for b in p.base.biases:
        b.copy_(torch.randn_like(b))
      for f in p.base.factors:
        f.copy_(torch.randn_like(f))
  return p


def _df64(p):
  q = D.NoisyDeepFactorized(batch_shape=p.batch_shape, dtype=torch.float64, device=dev)
  with torch.no_grad():
    for a, b in zip(q.parameters(), p.parameters()):
      a.copy_(b.double())
  return q


def _df_inputs(C, rows, seed, tails=False):
  g = torch.Generator(device="cpu").manual_seed(seed)
  n = C * rows
  if tails:  # |y| log-uniform up to 1e3, both signs
    y = torch.sign(torch.rand(n, generator=g) - .5) * 10**(torch.rand(n, generator=g) * 3)
  else:  # a dense grid across the +-0.5 boundaries plus spread-out values
    k = torch.arange(n)
    grid = (k % 81 - 40).float() * .5 + torch.tensor([0., 1e-6, -1e-6, 1e-3, -1e-3, .25])[k % 6]
    y = torch.where(k % 3 == 0, torch.randn(n, generator=g) * 6, grid)
  return y.reshape(rows, C).to(dev)


def _compare_df(p, y, check_params=True):
  q = _df64(p)
  dout = torch.randn(y.shape, generator=torch.Generator().manual_seed(1)).to(dev)
  n0 = _lib.launch_count()
  f_out, f_dy, f_dp = _grads(p.log_prob, y, p.parameters(), dout)
  assert _lib.launch_count() - n0 == (3 if y.numel() else 0)  # forward; backward + partial reduction
  g_out, g_dy, g_dp = _grads(p._log_prob_graph, y, p.parameters(), dout)
  r_out, r_dy, r_dp = _grads(q._log_prob_graph, y.double(), q.parameters(), dout.double())
  _check("log_prob", f_out, g_out, r_out, _elem_floor(r_out))
  _check("dy", f_dy, g_dy, r_dy, _elem_floor(r_dy))
  if check_params:
    for i, (a, b, c) in enumerate(zip(f_dp, g_dp, r_dp)):
      _check(f"dparam{i}", a, b, c, 2e-5 * c.abs().max())
  return f_dy, f_dp


@pytest.mark.parametrize("C", [1, 3, 128, 192, 320])
def test_deep_factorized_accuracy(C):
  rows = 1031 if C < 100 else 37  # n not a multiple of any block size
  _compare_df(_df(C, C), _df_inputs(C, rows, C))


@pytest.mark.parametrize("C", [1, 128, 320])
def test_deep_factorized_tails_at_initialisation(C):
  _compare_df(_df(C, 7, random=False), _df_inputs(C, 300 if C > 1 else 20000, 3, tails=True))


def test_deep_factorized_nan_and_inf():
  C = 4
  p = _df(C, 2)
  y = _df_inputs(C, 64, 5)
  y[0, 0], y[1, 1], y[2, 2], y[3, 3] = INF, -INF, NAN, INF
  _compare_df(p, y, check_params=False)  # every parameter gradient of those channels is NaN, as in the graph
  dout = torch.ones_like(y)
  f = _grads(p.log_prob, y, p.parameters(), dout)[2]
  g = _grads(p._log_prob_graph, y, p.parameters(), dout)[2]
  for a, b in zip(f, g):
    assert torch.equal(torch.isnan(a), torch.isnan(b))


def test_deep_factorized_zero_size_and_shapes():
  p = _df(5, 3)
  y = torch.zeros(0, 5, device=dev, requires_grad=True)
  n0 = _lib.launch_count()
  out = p.log_prob(y)
  out.sum().backward()
  assert _lib.launch_count() == n0 and out.shape == (0, 5) and y.grad.shape == (0, 5)
  assert all(float(t.grad.abs().sum()) == 0 for t in p.parameters())
  # higher-rank batch shape, and C = 1 with any shape
  q = D.NoisyDeepFactorized(batch_shape=(2, 3), device=dev)
  y = torch.randn(4, 5, 2, 3, device=dev)
  torch.testing.assert_close(q.log_prob(y), q._log_prob_graph(y), rtol=1e-5, atol=1e-5)
  r = D.NoisyDeepFactorized(batch_shape=(), device=dev)
  y = torch.randn(7, 11, device=dev)
  torch.testing.assert_close(r.log_prob(y), r._log_prob_graph(y), rtol=1e-5, atol=1e-5)


def test_deep_factorized_backward_is_deterministic():
  p = _df(192, 11)
  y = _df_inputs(192, 4099, 2)
  dout = torch.randn(y.shape, device=dev)
  a = _grads(p.log_prob, y, p.parameters(), dout)
  b = _grads(p.log_prob, y, p.parameters(), dout)
  assert torch.equal(a[1], b[1])
  assert all(torch.equal(u, v) for u, v in zip(a[2], b[2]))


def test_second_order_gradient_raises():
  p = _df(4, 1)
  y = torch.randn(8, 4, device=dev, requires_grad=True)
  g, = torch.autograd.grad(p.log_prob(y).sum(), y, create_graph=True)
  with pytest.raises(RuntimeError):
    g.sum().backward()


# ---------------------------------------------------------------------------------------------------------------
# location-scale
# ---------------------------------------------------------------------------------------------------------------
KINDS = [(D.NoisyNormal, "normal"), (D.NoisyLogistic, "logistic"), (D.NoisyLaplace, "laplace")]


def _ls_inputs(n, seed):
  g = torch.Generator().manual_seed(seed)
  k = torch.arange(n)
  grid = (k % 161 - 80).float() * .5 + torch.tensor([0., 1e-6, -1e-6, 1e-3, -1e-3, .25])[k % 6]
  y = torch.where(k % 3 == 0, torch.randn(n, generator=g) * 30, grid)
  loc = torch.randn(n, generator=g) * 2
  scale = torch.exp(torch.rand(n, generator=g) * (torch.log(torch.tensor(256.)) - torch.log(torch.tensor(.11))) +
                    torch.log(torch.tensor(.11)))
  return y.to(dev), loc.to(dev), scale.to(dev)


def _compare_ls(cls, y, loc, scale, scalar_loc=False, scalar_scale=False, expect_launches=2):
  """loc / scale: y-shaped, or 0-d leaves handed to the prior as broadcast (stride-0) views."""
  dout = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).to(dev)

  def run(dtype, graph):
    lo = loc.detach().to(dtype).requires_grad_(True)
    sc = scale.detach().to(dtype).requires_grad_(True)
    p = cls(lo.expand(y.shape) if scalar_loc else lo, sc.expand(y.shape) if scalar_scale else sc, dtype=dtype)
    fn = p._log_prob_graph if graph else p.log_prob
    return _grads(fn, y.to(dtype), [lo, sc], dout.to(dtype))

  n0 = _lib.launch_count()
  f = run(torch.float32, False)
  assert _lib.launch_count() - n0 == (expect_launches if y.numel() else 0)
  g = run(torch.float32, True)
  r = run(torch.float64, True)
  _check("log_prob", f[0], g[0], r[0], _elem_floor(r[0]))
  _check("dy", f[1], g[1], r[1], _elem_floor(r[1]))
  _check("dloc", f[2][0], g[2][0], r[2][0], _elem_floor(r[2][0]))
  _check("dscale", f[2][1], g[2][1], r[2][1], _elem_floor(r[2][1]))


@pytest.mark.parametrize("cls,kind", KINDS)
def test_location_scale_accuracy(cls, kind):
  y, loc, scale = _ls_inputs(100_003, 1)
  _compare_ls(cls, y, loc, scale)


@pytest.mark.parametrize("cls,kind", KINDS)
def test_location_scale_scalar_operands(cls, kind):
  y, loc, scale = _ls_inputs(20_011, 2)
  y = y.reshape(20_011, 1).expand(20_011, 3).contiguous()
  _compare_ls(cls, y, torch.tensor(0.3, device=dev), scale.reshape(-1, 1).expand(-1, 3).contiguous(), scalar_loc=True)
  _compare_ls(cls, y, loc.reshape(-1, 1).expand(-1, 3).contiguous(), torch.tensor(2.5, device=dev), scalar_scale=True)
  for s in (0.11, 1.0, 256.0):
    _compare_ls(cls, y, torch.tensor(-0.7, device=dev), torch.tensor(s, device=dev), scalar_loc=True,
                scalar_scale=True)


@pytest.mark.parametrize("cls,kind", KINDS)
def test_location_scale_nan_inf_and_zero_size(cls, kind):
  y, loc, scale = _ls_inputs(1000, 4)
  y[:4] = torch.tensor([INF, -INF, NAN, 0.])
  loc[5], scale[6] = NAN, INF
  f = cls(loc, scale).log_prob(y)
  g = cls(loc, scale)._log_prob_graph(y)
  assert torch.equal(torch.isnan(f), torch.isnan(g)) and torch.equal(torch.isinf(f), torch.isinf(g))
  yy = y.clone().requires_grad_(True)
  dy_f, = torch.autograd.grad(cls(loc, scale).log_prob(yy).sum(), yy)
  dy_g, = torch.autograd.grad(cls(loc, scale)._log_prob_graph(yy).sum(), yy)
  assert torch.equal(torch.isnan(dy_f), torch.isnan(dy_g))
  e = torch.zeros(0, 3, device=dev)
  _compare_ls(cls, e, e, e + 1)


# ---------------------------------------------------------------------------------------------------------------
# routing, entropy models, models
# ---------------------------------------------------------------------------------------------------------------
def test_excluded_cases_give_the_graph_bits():
  torch.manual_seed(0)
  y = torch.randn(6, 8, device=dev) * 3
  cases = [
      D.NoisyDeepFactorized(batch_shape=(8,), num_filters=(3, 3, 3), device=dev),
      D.NoisyDeepFactorized(batch_shape=(8,), num_filters=(2, 4), device=dev),
      D.NoisyNormal(torch.zeros(8, device=dev), torch.ones(8, device=dev)),       # loc / scale broadcast over rows
      D.NoisyRoundedNormal(0., torch.ones(6, 8, device=dev)),
      D.NoisySoftRoundedNormal(loc=torch.zeros(6, 8, device=dev), scale=torch.ones(6, 8, device=dev)),
      D.NoisyRoundedDeepFactorized(batch_shape=(8,), device=dev),
  ]
  for p in cases:
    n0 = _lib.launch_count()
    assert torch.equal(p.log_prob(y), p._log_prob_graph(y))
    assert _lib.launch_count() == n0
  p = D.NoisyDeepFactorized(batch_shape=(8,), device=dev)
  assert torch.equal(p.log_prob(y.double()), p._log_prob_graph(y.double()))           # float64 input
  p64 = D.NoisyNormal(torch.zeros(6, 8, device=dev), torch.ones(6, 8, device=dev), dtype=torch.float64)
  assert torch.equal(p64.log_prob(y.double()), p64._log_prob_graph(y.double()))
  m = D.NoisyNormalMixture(torch.zeros(6, 8, 1, device=dev), torch.ones(6, 8, 1, device=dev),
                           torch.ones(6, 8, 1, device=dev))
  n0 = _lib.launch_count()
  m.log_prob(y)
  assert _lib.launch_count() == n0
  df = p.base  # DeepFactorized.log_prob without noise
  assert _lib.launch_count() == n0 and torch.isfinite(df.log_prob(y)).all()


def test_tables_are_untouched(monkeypatch):
  def tables(prior):
    em = E.ContinuousBatchedEntropyModel(prior, coding_rank=1, compression=True)
    return em.cdf.cpu().numpy().tobytes(), em.cdf_offset.cpu().numpy().tobytes()

  torch.manual_seed(5)
  p = _df(16, 5)
  with torch.no_grad():
    p.base.matrices[0].mul_(0.3)
  a = tables(p)
  monkeypatch.setattr(D, "_fused_log_prob_kind", lambda base, y: None)
  assert tables(p) == a
  monkeypatch.undo()
  em = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 64, lambda i: torch.exp(i / 63 * 7.8 - 2.2), coding_rank=1,
                                          compression=True)
  b = em.cdf.cpu().numpy().tobytes()
  monkeypatch.setattr(D, "_fused_log_prob_kind", lambda base, y: None)
  em2 = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 64, lambda i: torch.exp(i / 63 * 7.8 - 2.2), coding_rank=1,
                                           compression=True)
  assert em2.cdf.cpu().numpy().tobytes() == b


def _model_step(make, x, monkeypatch, fused):
  torch.manual_seed(123)
  m = make()
  if not fused:
    monkeypatch.setattr(D, "_fused_log_prob_kind", lambda base, y: None)
  torch.manual_seed(7)
  n0 = _lib.launch_count()
  loss, bpp, mse = m(x, training=True)
  loss.backward()
  launches = _lib.launch_count() - n0
  monkeypatch.undo()
  grads = {k: (None if v.grad is None else v.grad.detach().clone()) for k, v in m.named_parameters()}
  return float(loss), float(bpp), grads, launches


@pytest.mark.parametrize("which", ["bls2017", "bmshj2018", "ms2020"])
def test_models_training_step_matches_the_graph(which, monkeypatch):
  from compression_b200 import models
  make = {
      "bls2017": lambda: models.BLS2017Model(num_filters=32).build("cuda"),
      "bmshj2018": lambda: models.BMSHJ2018Model(num_filters=24).build("cuda", patch=(64, 64)),
      "ms2020": lambda: models.MS2020Model(num_filters=24, latent_depth=32, hyperprior_depth=16, num_slices=4,
                                           max_support_slices=2).build("cuda", patch=(64, 64)),
  }[which]
  x = torch.rand(2, 64, 64, 3, generator=torch.Generator().manual_seed(9)).mul(255).to(dev)
  det = torch.backends.cudnn.deterministic
  torch.backends.cudnn.deterministic = True
  try:
    lf, bf, gf, nf = _model_step(make, x, monkeypatch, True)
    lg, bg, gg, ng = _model_step(make, x, monkeypatch, False)
  finally:
    torch.backends.cudnn.deterministic = det
  assert nf > ng  # the fused kernels ran
  assert abs(lf - lg) <= 1e-5 * abs(lg) and abs(bf - bg) <= 1e-5 * abs(bg)
  assert sum(g is not None for g in gg.values()) > 0
  for k, g in gg.items():
    assert (g is None) == (gf[k] is None), k  # every parameter the graph trains still gets a gradient
    if g is None:
      continue
    # 5e-4 of the tensor's largest magnitude.  2e-5 holds for bls2017, but not for bmshj2018's hyper transforms,
    # measured on an H100: 2.8e-4 on hyper_analysis_transform.0.bias (gradients of at most 1.5e-5, sums of
    # cancelling per-pixel terms), 3.0e-5 on hyper_synthesis_transform.0.kernel.  What differs is the graph's float32
    # rate term; the fused one is computed in double and held to the float64 graph element by element above.
    tol = 5e-4 * float(g.abs().max())
    assert float((gf[k] - g).abs().max()) <= tol, (k, float((gf[k] - g).abs().max()), tol)


def test_entropy_models_with_expected_grads(monkeypatch):
  torch.manual_seed(2)
  prior = _df(8, 2)
  y = (torch.randn(4, 6, 8, device=dev) * 4)

  def batched(fused):
    if not fused:
      monkeypatch.setattr(D, "_fused_log_prob_kind", lambda base, y: None)
    em = E.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=False, expected_grads=True)
    yy = y.clone().requires_grad_(True)
    torch.manual_seed(0)
    _, bits = em(yy, training=True)
    gs = torch.autograd.grad(bits.sum(), [yy] + list(prior.parameters()))
    monkeypatch.undo()
    return bits.detach(), gs

  a, ga = batched(True)
  b, gb = batched(False)
  torch.testing.assert_close(a, b, rtol=1e-5, atol=0)
  for u, v in zip(ga, gb):
    # 5e-4, not 2e-5, of the largest magnitude: measured on an H100, 4.0e-5 (batched) and 1.25e-4 (location-scale,
    # gradients up to 374 at scale 0.11).  dydx = f(x + .5) - f(x - .5) of the graph carries the float32 rounding of
    # both log-likelihoods; the fused ones are computed in double
    assert float((u - v).abs().max()) <= 5e-4 * float(v.abs().max())

  scale_fn = lambda i: torch.exp(i / 63 * 7.8 - 2.2)

  def ls(fused):
    if not fused:
      monkeypatch.setattr(D, "_fused_log_prob_kind", lambda base, y: None)
    em = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 64, scale_fn, coding_rank=2, compression=False,
                                            expected_grads=True)
    yy = y.clone().requires_grad_(True)
    idx = (torch.rand(y.shape, generator=torch.Generator().manual_seed(4)) * 63).to(dev).requires_grad_(True)
    torch.manual_seed(0)
    _, bits = em(yy, idx, training=True)
    gs = torch.autograd.grad(bits.sum(), [yy, idx])
    monkeypatch.undo()
    return bits.detach(), gs

  a, ga = ls(True)
  b, gb = ls(False)
  torch.testing.assert_close(a, b, rtol=1e-5, atol=0)
  for u, v in zip(ga, gb):
    # 5e-4, not 2e-5, of the largest magnitude: measured on an H100, 4.0e-5 (batched) and 1.25e-4 (location-scale,
    # gradients up to 374 at scale 0.11).  dydx = f(x + .5) - f(x - .5) of the graph carries the float32 rounding of
    # both log-likelihoods; the fused ones are computed in double
    assert float((u - v).abs().max()) <= 5e-4 * float(v.abs().max())
