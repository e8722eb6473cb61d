"""ORACLE (test infrastructure): float64 reference of the fused rate-term kernels (compression_b200/csrc/likelihood.cu).

It takes the kernels' own inputs -- float32 y, the packed [C, 28] deep-factorized parameters of
`DeepFactorized._packed_parameters()`, or float32 loc / scale (y-shaped or 0-d) -- and evaluates
  log p(y) = log(F(y + 1/2) - F(y - 1/2))
in float64 torch as the graph of `UniformNoiseAdapter._log_prob_graph` writes it: the 1-3-3-1 MLP, `logsigmoid`,
`log_ndtr`, the two-branch Laplace form, the big / small select and `log1p(-exp(small - big)) + big`.  Gradients are
float64 autograd of that graph, so `torch.where`'s zero gradient for the branch not taken and the NaN / inf masks are
the graph's.

Each output comes with `M`, a magnitude such that the float64 evaluation (this one, or the kernels') is within a few
units of 2^-53 * M of the exact value.  For a gradient it is the sum of |terms| the final sum adds (the y + 1/2 and
y - 1/2 evaluations are separate autograd leaves), each weighted by how much the log difference amplifies relative
errors where F(y + 1/2) and F(y - 1/2) nearly agree.  The tests allow 2^-40 M on top of half a float32 ulp.

`df_geometry` restates the CTA geometry of `noisy_df_fwd_kernel` / `noisy_df_bwd_kernel`, and `df_reference` returns,
per CTA, the float64 sum of the parameter-gradient contributions the CTA writes as one float32 partial row.

The `mp_*` functions are a 50-digit mpmath path with explicit derivative formulas, for small sets on the CPU."""
import math

import torch
import torch.nn.functional as Fn

NUM_PARAMS = 28
M0, M1, M2, B0, B1, B2, F0, F1 = 0, 3, 12, 15, 18, 21, 22, 25
EPS_BAR = 2.0**-40  # weight of M in the bars (2^13 units of 2^-53)
MAX_THREADS, FWD_MAX_CTAS, BWD_MAX_CTAS, BWD_ROWS_PER_THREAD = 256, 8192, 512, 4


# ---- the graph's pieces -----------------------------------------------------------------------------------------
def _combine(lsf_p, lcdf_p, lsf_m, lcdf_m):
  right = lsf_p < lcdf_p
  big = torch.where(right, lsf_m, lcdf_p)
  small = torch.where(right, lsf_p, lcdf_m)
  return torch.where(torch.isinf(big), big, torch.log1p(-torch.exp(small - big)) + big), right


def _mlp(w, x):
  """CDF logits of the deep-factorized MLP; w: 28 tensors that broadcast with x."""
  a0 = []
  for i in range(3):
    h = w[M0 + i] * x + w[B0 + i]
    a0.append(h + w[F0 + i] * torch.tanh(h))
  a1 = []
  for i in range(3):
    h = w[M1 + 3 * i] * a0[0] + w[M1 + 3 * i + 1] * a0[1] + w[M1 + 3 * i + 2] * a0[2] + w[B1 + i]
    a1.append(h + w[F1 + i] * torch.tanh(h))
  return w[M2] * a1[0] + w[M2 + 1] * a1[1] + w[M2 + 2] * a1[2] + w[B2]


def _mlp_bounds(w, x):
  """(A, chain, act) for the MLP at x: A bounds the sum of |terms| behind l (its rounding error is a few eps * A);
  chain bounds, in units of eps, the relative error of the backward's factors 1 + f (1 - tanh(h)^2) from the
  rounding of h and tanh(h); act bounds the relative error of the activations a = h + f tanh(h) that the matrix
  gradients multiply."""
  tiny = torch.finfo(torch.float64).tiny
  chain, act = torch.zeros_like(x), torch.zeros_like(x)

  def unit(h, A, f):
    nonlocal chain, act
    t = torch.tanh(h)
    one_m = 1 - t * t
    chain = chain + (2 * (f * t).abs() * one_m * A + 2 * f.abs()) / (1 + f * one_m).abs().clamp(min=tiny)
    a = h + f * t
    act = act + 2 * A / a.abs().clamp(min=tiny)
    return a, 2 * A

  a0, A0 = zip(*[unit(w[M0 + i] * x + w[B0 + i], w[M0 + i].abs() * x.abs() + w[B0 + i].abs(), w[F0 + i])
                 for i in range(3)])
  a1, A1 = [], []
  for i in range(3):
    row = [w[M1 + 3 * i + j] for j in range(3)]
    a, A = unit(row[0] * a0[0] + row[1] * a0[1] + row[2] * a0[2] + w[B1 + i],
                sum(r.abs() * Aj for r, Aj in zip(row, A0)) + w[B1 + i].abs(), w[F1 + i])
    a1.append(a)
    A1.append(A)
  A = sum(w[M2 + j].abs() * A1[j] for j in range(3)) + w[B2].abs()
  return A, chain, act


def _log_difference_condition(lsf_p, lcdf_p, lsf_m, lcdf_m, mag):
  """(K, mag_d, e, right): K = e mag_d / (1 - e), the relative error of 1 - e in units of eps, where e = exp(small - big) and
  mag_d bounds the error of small - big; mag maps each of the four logs to its own magnitude."""
  right = lsf_p < lcdf_p
  big = torch.where(right, lsf_m, lcdf_p)
  small = torch.where(right, lsf_p, lcdf_m)
  mag_d = torch.where(right, mag["lsf_m"] + mag["lsf_p"], mag["lcdf_p"] + mag["lcdf_m"])
  e = torch.exp(small - big)
  K = e * mag_d / (-torch.expm1(small - big)).clamp(min=torch.finfo(torch.float64).tiny)
  return K, mag_d, e, right


# ---- deep factorized ---------------------------------------------------------------------------------------------
def df_geometry(n, C, backward):
  """`df_geometry` of likelihood.cu: cpb channels per CTA, subrows rows per CTA step, chunks on grid.y, grid_x CTAs
  per chunk.  A thread of CTA x, sub-row s, starts at row x * subrows + s and strides grid_x * subrows rows."""
  parts = -(-C // MAX_THREADS)
  cpb = -(-C // parts)
  subrows = MAX_THREADS // cpb
  chunks = -(-C // cpb)
  rows = n // C
  per_cta = subrows * (BWD_ROWS_PER_THREAD if backward else 1)
  cap = max(1, (BWD_MAX_CTAS if backward else FWD_MAX_CTAS) // chunks)
  grid_x = max(1, min(-(-rows // per_cta), cap))
  return {"cpb": cpb, "subrows": subrows, "chunks": chunks, "grid_x": grid_x}


def df_row_cta(rows, geometry, device="cpu"):
  """CTA index (blockIdx.x) whose threads walk each row."""
  return (torch.arange(rows, device=device) // geometry["subrows"]) % geometry["grid_x"]


def df_workspace_bytes(n, C):
  if n <= 0 or C <= 0:
    return 0
  return df_geometry(n, C, True)["grid_x"] * C * NUM_PARAMS * 4


def _df_pieces(w_p, w_m, x_p, x_m):
  l_p, l_m = _mlp(w_p, x_p), _mlp(w_m, x_m)
  lcdf_p, lsf_p, lcdf_m, lsf_m = Fn.logsigmoid(l_p), Fn.logsigmoid(-l_p), Fn.logsigmoid(l_m), Fn.logsigmoid(-l_m)
  out, _ = _combine(lsf_p, lcdf_p, lsf_m, lcdf_m)
  return out, (l_p, l_m, lsf_p, lcdf_p, lsf_m, lcdf_m)


def _df_bars(w, y, logs):
  """Per element: M of log p, and the weights R (dy) and R_dp (parameter contributions) of the y + 1/2 and y - 1/2
  terms of the gradients."""
  l_p, l_m, lsf_p, lcdf_p, lsf_m, lcdf_m = [t.detach() for t in logs]
  (A_p, chain_p, act_p), (A_m, chain_m, act_m) = _mlp_bounds(w, y + .5), _mlp_bounds(w, y - .5)
  sig = torch.sigmoid
  mag = {"lcdf_p": lcdf_p.abs() + sig(-l_p) * A_p, "lsf_p": lsf_p.abs() + sig(l_p) * A_p,
         "lcdf_m": lcdf_m.abs() + sig(-l_m) * A_m, "lsf_m": lsf_m.abs() + sig(l_m) * A_m}
  K, mag_d, e, right = _log_difference_condition(lsf_p, lcdf_p, lsf_m, lcdf_m, mag)
  M_out = torch.where(right, mag["lsf_m"], mag["lcdf_p"]) + torch.log1p(-e).abs() + K
  # per term: the log difference and its exp, the logsigmoid derivative at the argument the select uses (a relative
  # error sigmoid(-arg) * eps * A from l's rounding), the MLP's chain factors
  base = 16 + K + mag_d
  R_p = base + sig(torch.where(right, -l_p, l_p)) * A_p + chain_p
  R_m = base + sig(torch.where(right, -l_m, l_m)) * A_m + chain_m
  return M_out, (R_p, R_m), (R_p + act_p, R_m + act_m)


def df_params(packed):
  """The 28 columns of a packed [C, 28] tensor, in float64."""
  p = packed.detach().to(torch.float64)
  return [p[:, k] for k in range(NUM_PARAMS)]


def _df_chunk(w, yc, dc):
  """One block of rows [r, C]: log p, M, and with dc the gradients and per-element contributions."""
  if dc is None:
    with torch.no_grad():
      out, logs = _df_pieces(w, w, yc + .5, yc - .5)
      return {"logp": out, "M_logp": _df_bars(w, yc, logs)[0]}
  # per-row copies of the parameters, one set per evaluation, as the autograd leaves
  wp = [t.expand_as(yc).clone().requires_grad_(True) for t in w]
  wm = [t.expand_as(yc).clone().requires_grad_(True) for t in w]
  xp, xm = (yc + .5).requires_grad_(True), (yc - .5).requires_grad_(True)
  with torch.enable_grad():
    out, logs = _df_pieces(wp, wm, xp, xm)
    g = torch.autograd.grad(out, [xp, xm] + wp + wm, dc)
  with torch.no_grad():
    M_out, (R_p, R_m), (Q_p, Q_m) = _df_bars(w, yc, logs)
    cp, cm = torch.stack(g[2:2 + NUM_PARAMS], -1), torch.stack(g[2 + NUM_PARAMS:], -1)
    return {"logp": out.detach(), "M_logp": M_out, "dy": g[0] + g[1], "M_dy": g[0].abs() * R_p + g[1].abs() * R_m,
            "contrib": cp + cm, "M_contrib": cp.abs() * Q_p[..., None] + cm.abs() * Q_m[..., None]}


def df_reference(y, packed, dout=None, partials=False, chunk_elems=1 << 20):
  """float64 reference of noisy_deep_factorized_log_prob on the kernels' inputs.

  y: any shape with numel a multiple of C (channel of element i is i mod C); packed: [C, 28]; dout: y-shaped upstream
  gradient or None (forward only).  Returns float64 tensors shaped like y (`logp`, `M_logp`, `dy`, `M_dy`) and
  [C, 28] (`dpacked`; `M_dpacked`, the sum of the contributions' M).  With `partials`, also `partials`
  [grid_x, C, 28]: the sum of the contributions each CTA of the backward kernel writes as one float partial row.
  Rows are processed in blocks of about `chunk_elems` elements, so memory stays bounded at any size."""
  C = packed.shape[0]
  dev = packed.device
  w = df_params(packed)
  y64 = y.detach().to(dev, torch.float64).reshape(-1, C)
  d64 = None if dout is None else dout.detach().to(dev, torch.float64).reshape(-1, C)
  rows = y64.shape[0]
  res = {}
  if dout is not None:
    res["dpacked"] = torch.zeros(C, NUM_PARAMS, dtype=torch.float64, device=dev)
    res["M_dpacked"] = torch.zeros_like(res["dpacked"])
    if partials:
      g = df_geometry(y64.numel(), C, True)
      res["partials"] = torch.zeros(g["grid_x"], C, NUM_PARAMS, dtype=torch.float64, device=dev)
      cta = df_row_cta(rows, g, dev)
  step = max(1, chunk_elems // C)
  for r0 in range(0, rows, step):
    part = _df_chunk(w, y64[r0:r0 + step], None if d64 is None else d64[r0:r0 + step])
    for k in ("logp", "M_logp", "dy", "M_dy"):
      if k in part:
        res.setdefault(k, torch.empty_like(y64))[r0:r0 + step] = part[k]
    if dout is not None:
      res["dpacked"] += part["contrib"].sum(0)
      res["M_dpacked"] += part["M_contrib"].sum(0)
      if partials:
        res["partials"].index_add_(0, cta[r0:r0 + step], part["contrib"])
  for k in ("logp", "M_logp", "dy", "M_dy"):
    if k in res:
      res[k] = res[k].reshape(y.shape)
  return res


def df_contributions(y, packed, dout):
  """Per-element parameter-gradient contributions [rows, C, 28] and their M (small inputs)."""
  C = packed.shape[0]
  yc = y.detach().to(packed.device, torch.float64).reshape(-1, C)
  part = _df_chunk(df_params(packed), yc, dout.detach().to(yc).reshape(-1, C))
  return part["contrib"], part["M_contrib"]


# ---- location-scale ----------------------------------------------------------------------------------------------
def _std_log_cdf(base, z):
  if base == "normal":
    return torch.special.log_ndtr(z)
  if base == "logistic":
    return Fn.logsigmoid(z)
  return torch.where(z < 0, math.log(0.5) + z, torch.log1p(-0.5 * torch.exp(-z.abs())))


def _std_rel(base, x):
  """|d log s'(x) / dx| * |x|: the relative error of the log-CDF's derivative from a relative error eps in x."""
  if base == "normal":
    ds = torch.exp(-(torch.special.log_ndtr(x) + x * x / 2)) / math.sqrt(2 * math.pi)
    return (x + ds).abs() * x.abs()
  if base == "logistic":
    return torch.sigmoid(x) * x.abs()
  e = 0.5 * torch.exp(-x.abs())
  return torch.where(x > 0, (1 + e / (1 - e)) * x.abs(), torch.zeros_like(x))


def loc_scale_reference(base, y, loc, scale, dout=None):
  """float64 reference of noisy_loc_scale_log_prob(base, y, loc, scale) on the kernels' inputs: loc / scale
  y-shaped or 0-d.  Returns `logp`, `M_logp` and, with dout, the elementwise `dy`, `dloc`, `dscale` (the terms a 0-d
  operand's gradient sums) with `M_dy`, `M_dscale` (`M_dloc` is `M_dy`)."""
  dev = y.device
  x = y.detach().to(torch.float64)
  mu = loc.detach().to(dev, torch.float64).expand_as(x)
  sigma = scale.detach().to(dev, torch.float64).expand_as(x)
  leaves = [(x + .5), (x - .5), sigma.clone(), sigma.clone()]
  if dout is not None:
    leaves = [t.requires_grad_(True) for t in leaves]
  xp, xm, sp, sm = leaves
  with torch.set_grad_enabled(dout is not None):
    z_p, z_m = (xp - mu) / sp, (xm - mu) / sm
    s = lambda z: _std_log_cdf(base, z)
    lcdf_p, lsf_p, lcdf_m, lsf_m = s(z_p), s(-z_p), s(z_m), s(-z_m)
    out, _ = _combine(lsf_p, lcdf_p, lsf_m, lcdf_m)
    grads = torch.autograd.grad(out, leaves, dout.detach().to(x)) if dout is not None else None
  with torch.no_grad():
    z_p, z_m, lcdf_p, lsf_p, lcdf_m, lsf_m, out = (t.detach() for t in (z_p, z_m, lcdf_p, lsf_p, lcdf_m, lsf_m, out))
    # a relative error eps in z moves s(z) by |s'(z) z| eps
    d = {"normal": lambda v: torch.exp(-(torch.special.log_ndtr(v) + v * v / 2)) / math.sqrt(2 * math.pi),
         "logistic": lambda v: torch.sigmoid(-v),
         "laplace": lambda v: torch.where(v < 0, torch.ones_like(v),
                                          0.5 * torch.exp(-v.abs()) / (1 - 0.5 * torch.exp(-v.abs())))}[base]
    mag = {"lcdf_p": lcdf_p.abs() + (d(z_p) * z_p).abs(), "lsf_p": lsf_p.abs() + (d(-z_p) * z_p).abs(),
           "lcdf_m": lcdf_m.abs() + (d(z_m) * z_m).abs(), "lsf_m": lsf_m.abs() + (d(-z_m) * z_m).abs()}
    K, mag_d, e, right = _log_difference_condition(lsf_p, lcdf_p, lsf_m, lcdf_m, mag)
    res = {"logp": out, "M_logp": torch.where(right, mag["lsf_m"], mag["lcdf_p"]) + torch.log1p(-e).abs() + K}
    if dout is None:
      return res
    base_R = 16 + K + mag_d
    R_p = base_R + _std_rel(base, torch.where(right, -z_p, z_p))
    R_m = base_R + _std_rel(base, torch.where(right, -z_m, z_m))
    res["dy"] = grads[0] + grads[1]
    res["dloc"] = -res["dy"]
    res["M_dy"] = grads[0].abs() * R_p + grads[1].abs() * R_m
    res["dscale"] = grads[2] + grads[3]
    res["M_dscale"] = grads[2].abs() * R_p + grads[3].abs() * R_m
    return res


# ---- 50 digits ---------------------------------------------------------------------------------------------------
def _mp():
  import mpmath
  mpmath.mp.dps = 50
  return mpmath


def _mp_sigmoid(mp, v):
  return 1 / (1 + mp.exp(-v))


def mp_df(packed_row, y):
  """log p, d/dy and d/d(packed row) of one element at 50 digits; packed_row: 28 floats."""
  mp = _mp()
  w = [mp.mpf(float(v)) for v in packed_row]
  x = mp.mpf(float(y))

  def forward(xx):
    h0 = [w[M0 + i] * xx + w[B0 + i] for i in range(3)]
    t0 = [mp.tanh(h) for h in h0]
    a0 = [h0[i] + w[F0 + i] * t0[i] for i in range(3)]
    h1 = [sum(w[M1 + 3 * i + j] * a0[j] for j in range(3)) + w[B1 + i] for i in range(3)]
    t1 = [mp.tanh(h) for h in h1]
    a1 = [h1[i] + w[F1 + i] * t1[i] for i in range(3)]
    return sum(w[M2 + j] * a1[j] for j in range(3)) + w[B2], (xx, t0, a0, t1, a1)

  def backward(state, dl, acc):
    xx, t0, a0, t1, a1 = state
    acc[B2] += dl
    g1 = []
    for i in range(3):
      acc[M2 + i] += dl * a1[i]
      ga = dl * w[M2 + i]
      acc[F1 + i] += ga * t1[i]
      g1.append(ga * (1 + w[F1 + i] * (1 - t1[i]**2)))
      acc[B1 + i] += g1[i]
    dx = 0
    for j in range(3):
      ga = 0
      for i in range(3):
        acc[M1 + 3 * i + j] += g1[i] * a0[j]
        ga += g1[i] * w[M1 + 3 * i + j]
      acc[F0 + j] += ga * t0[j]
      g0 = ga * (1 + w[F0 + j] * (1 - t0[j]**2))
      acc[B0 + j] += g0
      acc[M0 + j] += g0 * xx
      dx += g0 * w[M0 + j]
    return dx

  l_p, s_p = forward(x + mp.mpf(0.5))
  l_m, s_m = forward(x - mp.mpf(0.5))
  sg = lambda v: _mp_sigmoid(mp, v)
  # the difference of survival functions on the right: both sides then subtract small numbers
  dF = sg(-l_m) - sg(-l_p) if l_p + l_m > 0 else sg(l_p) - sg(l_m)
  dl_p = sg(l_p) * sg(-l_p) / dF
  dl_m = -sg(l_m) * sg(-l_m) / dF
  acc = [mp.mpf(0)] * NUM_PARAMS
  dy = backward(s_p, dl_p, acc) + backward(s_m, dl_m, acc)
  return mp.log(dF), dy, acc


def mp_loc_scale(base, y, loc, scale):
  """log p, dy, dloc, dscale of one element at 50 digits (dout = 1).  Laplace's derivative at z = 0 exactly is the
  graph's: abs's zero subgradient leaves the log1p branch's term at 0."""
  mp = _mp()
  x, mu, sigma = mp.mpf(float(y)), mp.mpf(float(loc)), mp.mpf(float(scale))
  z_p, z_m = (x + mp.mpf(0.5) - mu) / sigma, (x - mp.mpf(0.5) - mu) / sigma
  if base == "normal":
    cdf = lambda z: mp.erfc(-z / mp.sqrt(2)) / 2
    pdf = lambda z: mp.exp(-z * z / 2) / mp.sqrt(2 * mp.pi)
  elif base == "logistic":
    cdf = lambda z: _mp_sigmoid(mp, z)
    pdf = lambda z: _mp_sigmoid(mp, z) * _mp_sigmoid(mp, -z)
  else:
    cdf = lambda z: mp.exp(z) / 2 if z < 0 else 1 - mp.exp(-z) / 2
    pdf = lambda z: mp.exp(-abs(z)) / 2
  sf = lambda z: cdf(-z)
  right = z_p + z_m > 0
  dF = sf(z_m) - sf(z_p) if right else cdf(z_p) - cdf(z_m)

  dens = lambda z: mp.mpf(0) if base == "laplace" and z == 0 else pdf(z)
  g_p, g_m = dens(z_p) / dF, -dens(z_m) / dF
  dy = (g_p + g_m) / sigma
  dscale = -(g_p * z_p + g_m * z_m) / sigma
  return mp.log(dF), dy, -dy, dscale
