"""GDN / IGDN at trained-model parameters on every kernel path, against two oracles.

The rest of the GDN suite draws gamma = 0.1 I + |N(0, 0.02^2)|, beta in [1, 1.5] and x ~ N(0, 1) per channel scale:
the initialiser plus a little noise.  There every product p_j gamma_jc is a small share of the norm
n_c = beta_c + sum_j p_j gamma_jc, so the per-product error of the tensor cores' 3xBF16 split averages away.  A
trained GDN layer looks different: beta falls toward its lower bound (1e-6), gamma keeps a few large entries and
many exact zeros, and the activations are heavy-tailed with exact zeros.  A few products then make up most of n.  The
synthetic families below reproduce those features (nothing is downloaded; the seeds are fixed):

  trained-like       beta log-uniform in [6e-6, 0.14]; gamma's diagonal e^N(-1, 1), 30 % of the off-diagonals
                     e^N(-5, 1.5^2), the rest exactly 0
  diagonal-dominant  gamma's diagonal e^N(-1, 1) plus U(0, 1e-4) everywhere, beta = 1e-6: n is one product
  permuted           trained-like gamma with its columns permuted: the dominant product is off the diagonal
  saturated          trained-like, a third of beta at exactly 1e-6 and a quarter of gamma's columns zero but for
                     one entry

and every input tensor holds the edges where kernels go wrong: whole pixels of exact zeros (n = beta, down to 1e-6),
10 % exact zeros inside pixels (more under rectify), channel scales e^N(0, 1.5^2), entries of magnitude 1e3, and
64 * 420 + 5 pixels (not a multiple of the 64-pixel tile, more tiles than one persistent wave at every width).

Oracle 1, the contract: oracle/gdn_oracle.py in float64.  Oracle 2, the same operation: gdn_oracle's float64
emulation of the tensor-core split (gdn_tc_forward_emulated / gdn_tc_backward_emulated).  Each tensor-core path is
held to the emulation element by element within a bound that covers only the kernels' fp32 accumulation and fp32
epilogues, k * 2^-24 * sum |terms| with k stated below; a kernel that loses a lo plane, a beta column or a dgamma
partial misses it by orders of magnitude (tests/test_gdn_split_model_cpu.py shows the bound can fail).  Against
float64 the tensor-core paths are held to the split's own error model (gdn_oracle.SPLIT_REL per product, carried
through q, dp and the sums), and the CUDA-core paths to the 1e-5 contract.  The measured maxima are printed."""
import math

import pytest
import torch

from oracle import gdn_oracle as O

pytestmark = pytest.mark.gpu

WIDTHS = [128, 192, 256, 320]
BIG = 64 * 420 + 5
U = O.U

# Bounds against the emulation, in units of 2^-24.  Each wgmma adds 16 exact bf16 products into the fp32 running sum
# and truncates what falls below its last bits; a contraction over K channels issues 3 K / 16 of them (hi.hi, lo.hi,
# hi.lo).  Measured on an H100 80GB HBM3 (700 W power limit), the worst case is one dominant product followed by many
# small ones (the diagonal-dominant family): up to 2.4 units of the running sum per instruction, so n and dp are held
# to k = 4 * 3 K / 16.  dgamma restarts its accumulator every kDgFlush = 8 chunks of 64 pixels (4 * 3 * 8
# instructions) and adds it into an fp32 partial: k = 4 * 96 + 8.  Epilogue arithmetic (beta + acc, rcp / division /
# sqrt / powf, the products forming q and dx) stays within K_EP units of the value it forms.
def k_acc(C_):
  return 4 * 3 * C_ // 16


K_DGAMMA = 4 * 3 * 4 * 8 + 8
K_EP = 8

MEASURED = {}  # the maxima of the cases run so far, by path (printed by each test as it runs)

FWD_CONFIGS = {  # name: (inverse, rectify, alpha, epsilon); gdn / igdn run the FAST variant, the others the general
    "gdn": (False, False, 1.0, 1.0),
    "igdn": (True, False, 1.0, 1.0),
    "gdn_rectify_sq_sqrt": (False, True, 2.0, 0.5),
    "igdn_rectify": (True, True, 1.0, 1.0),
}
POW_CONFIGS = {  # name: (inverse, rectify, alpha, epsilon, trainable alpha, trainable epsilon)
    "pow_gdn": (False, True, 1.3, 0.8, True, True),   # zeros under rectify and literal pow
    "pow_igdn": (True, False, 1.0, 0.7, False, True),  # fixed alpha = 1 keeps |u|
}


# ---- parameters ----------------------------------------------------------------------------------------------------

def initialiser_like(C_, seed):
  """The distribution of the rest of the GDN suite (for the comparison printed beside the trained families)."""
  g = torch.Generator().manual_seed(seed)
  gamma = 0.1 * torch.eye(C_) + (0.02 * torch.randn(C_, C_, generator=g)).abs()
  beta = 1.0 + 0.5 * torch.rand(C_, generator=g)
  return gamma, beta


def trained_like(C_, seed):
  g = torch.Generator().manual_seed(seed)
  beta = torch.exp(torch.empty(C_).uniform_(math.log(6e-6), math.log(0.14), generator=g))
  off = torch.exp(torch.randn(C_, C_, generator=g) * 1.5 - 5.0)
  off = torch.where(torch.rand(C_, C_, generator=g) < 0.3, off, torch.zeros(()))
  off.fill_diagonal_(0.0)
  gamma = off + torch.diag(torch.exp(torch.randn(C_, generator=g) - 1.0))
  return gamma, beta


def diagonal_dominant(C_, seed):
  g = torch.Generator().manual_seed(seed)
  gamma = torch.diag(torch.exp(torch.randn(C_, generator=g) - 1.0)) + 1e-4 * torch.rand(C_, C_, generator=g)
  return gamma, torch.full((C_,), 1e-6)


def permuted(C_, seed):
  gamma, beta = trained_like(C_, seed)
  perm = torch.randperm(C_, generator=torch.Generator().manual_seed(seed + 1))
  return gamma[:, perm].contiguous(), beta


def saturated(C_, seed):
  gamma, beta = trained_like(C_, seed)
  g = torch.Generator().manual_seed(seed + 2)
  beta[::3] = 1e-6
  for c in range(1, C_, 4):
    j = int(torch.randint(C_, (1,), generator=g))
    gamma[:, c] = 0.0
    gamma[j, c] = float(torch.exp(torch.randn(1, generator=g)))
  return gamma, beta


FAMILIES = {"trained": trained_like, "diagonal": diagonal_dominant, "permuted": permuted, "saturated": saturated}


def inputs(n_pix, C_, seed):
  """x [n_pix, C] with the edge cases listed in the module docstring, and dy ~ N(0, 1)."""
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(n_pix, C_, generator=g) * torch.exp(1.5 * torch.randn(C_, generator=g))
  x[torch.rand(n_pix, C_, generator=g) < 0.1] = 0.0
  x[::37] = 0.0   # whole pixels of zeros: n = beta
  x[-1] = 0.0
  big = torch.sign(torch.randn(n_pix, 4, generator=g)) * 1e3
  x[5::101, :4] = big[5::101]
  dy = torch.randn(n_pix, C_, generator=g)
  return x, dy


# ---- calls -------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


@pytest.fixture
def fp32_path(monkeypatch):
  """Runs the test on the CUDA-core kernels (TFCB_GDN_FP32=1)."""
  monkeypatch.setenv("TFCB_GDN_FP32", "1")


def _flags(F, inverse, rectify, pa=False, pe=False):
  return F._flags(inverse, rectify, pa, pe)


def run_backward(F, x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa=False, pe=False, exponents=False):
  """One tfcb_gdn_backward (or _exponents) call with a workspace of our own: (dx, dgamma, dbeta, dalpha_depsilon or
  None, q, launches).  q = dL/dn as the kernels left it at the start of the workspace."""
  from compression_b200 import _lib
  L = _lib.lib()
  n_pix, C_ = x.shape
  dx, dgamma, dbeta = torch.empty_like(x), torch.empty_like(gamma), torch.empty_like(beta)
  dae = torch.full((2,), float("nan"), device=x.device)
  p = lambda t: t.data_ptr()
  st = torch.cuda.current_stream().cuda_stream
  n0 = _lib.launch_count()
  if exponents:
    ws = torch.empty(int(L.tfcb_gdn_backward_exponents_workspace_bytes(n_pix, C_)), dtype=torch.uint8, device=x.device)
    _lib.check(L.tfcb_gdn_backward_exponents(p(x), p(gamma), p(beta), p(dy), p(dx), p(dgamma), p(dbeta), p(dae), p(ws),
                                             n_pix, C_, _flags(F, inverse, rectify, pa, pe), alpha, epsilon, st))
  else:
    ws = torch.empty(int(L.tfcb_gdn_backward_workspace_bytes(n_pix, C_)), dtype=torch.uint8, device=x.device)
    _lib.check(L.tfcb_gdn_backward(p(x), p(gamma), p(beta), p(dy), p(dx), p(dgamma), p(dbeta), p(ws), n_pix, C_,
                                   _flags(F, inverse, rectify, pa, pe), alpha, epsilon, st))
  launches = _lib.launch_count() - n0
  q = ws[:n_pix * C_ * 4].view(torch.float32).view(n_pix, C_).clone()
  return dx, dgamma, dbeta, (dae if exponents else None), q, launches


def run_forward(F, x, gamma, beta, inverse, rectify, alpha, epsilon, pa=False, pe=False):
  from compression_b200 import _lib
  n0 = _lib.launch_count()
  y = F.gdn_forward(x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe)
  return y, _lib.launch_count() - n0


def tc_backward_launches(C_, exponents):
  """dx + dgamma kernels (three passes at 256 / 320) + the two reductions (+ the exponent partials' reduction)."""
  return (4 if C_ <= 192 else 5) + (1 if exponents else 0)


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def dbeta_k(n_pix, C_):
  """dbeta's bound in units of 2^-24 of sum |q|: each staging thread adds 4 pixels' q per chunk in fp32, then a 4-level
  shuffle, then one rounding of the double reduction."""
  chunks = -(-n_pix // 64)
  parts = min(chunks, min(_sms(), 148)) if C_ <= 192 else min(chunks, max(1, min(_sms() // (C_ // (128 if C_ == 256 else 64)), 148)))
  return 4 * -(-chunks // parts) + 6


def exponent_sum_k(n_pix, C_):
  """The exponent gradients' summation bound in units of 2^-24 of sum |terms|: a thread adds at most C / 2 terms per
  tile it walks, each warpgroup walks at most ceil(tiles / SMs) tiles, then the shuffles and warps of its CTA."""
  tiles = -(-n_pix // 64)
  return (C_ // 2) * -(-tiles // _sms()) + 32


def _report(key, **vals):
  MEASURED.setdefault(key, {})
  for k, v in vals.items():
    MEASURED[key][k] = max(MEASURED[key].get(k, 0.0), v)
  print(f"GDN {key}: " + ", ".join(f"{k}={v:.3g}" for k, v in vals.items()))


def _max(t):
  return float(t.max()) if t.numel() else 0.0


# ---- the checks --------------------------------------------------------------------------------------------------

def check_masks(got, want):
  """NaN / inf positions equal the float64 oracle's wherever it is finite (here: everywhere)."""
  got = got.double()
  assert torch.isfinite(want).all()
  assert torch.isfinite(got).all(), int((~torch.isfinite(got)).sum())


def check_forward_tc(y, x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe, key):
  """y of a tensor-core forward: against the emulation within U * |y| * (k_acc * a / n + K_EP), and against float64
  within the split's error model."""
  C_ = x.shape[1]
  y_e, n, a = O.gdn_tc_forward_emulated(x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe)
  y64 = O.gdn_reference(x, gamma, beta, inverse, rectify, O._f32(alpha), O._f32(epsilon), device=x.device)
  check_masks(y, y64)
  err = (y.double() - y_e).abs()
  tol = U * y_e.abs() * (k_acc(C_) * a / n + K_EP)
  acc_dominated = a >= 0.25 * n
  k_meas = _max((err / (U * y_e.abs() * a / n))[acc_dominated & (y_e != 0)])
  assert bool((err <= tol).all()), ("forward vs emulation", float((err - tol).max()), k_meas)
  # float64: n is off by at most SPLIT_REL * a (the split) + accumulation + rounding of p; y by that relative to n
  delta = (O.SPLIT_REL + (k_acc(C_) + 4) * U) * a / n + U
  err64 = (y.double() - y64).abs()
  rel64 = _max((err64 / y64.abs())[y64 != 0])
  assert bool((err64 <= 1.25 * y64.abs() * (delta + K_EP * U)).all()), ("forward vs float64", rel64)
  assert bool((y[y64 == 0] == 0).all())
  return dict(fwd_vs_emulation_k=k_meas, fwd_vs_fp64_rel=rel64)


def _of_max(got, want):
  return float((got.double() - want).abs().max()) / (float(want.abs().max()) + 1e-300)


def exact_exponent_terms(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa):
  """Per-element terms of dL/dalpha and dL/depsilon in float64 from the exact graph (p, n, q, dp all float64)."""
  x64, g64, b64, dy64 = (t.double() for t in (x, gamma, beta, dy))
  u = torch.relu(x64) if rectify else x64
  al, ep = O._f32(alpha), O._f32(epsilon)
  p = u.abs() if (not pa and al == 1) else u**al
  if not pa and al == 1 and rectify:
    p = u
  n = p @ g64 + b64
  m = n**ep
  dm = ep * n**(ep - 1)
  q = dy64 * u * dm if inverse else -dy64 * u * dm / (m * m)
  dp = q @ g64.t()
  pos = u > 0
  ta = torch.where(pos, dp * p * torch.log(torch.where(pos, u, torch.ones_like(u))), torch.zeros_like(u))
  te = q * n * torch.log(n) / ep
  return ta, te


def check_backward_tc(got, x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe, key):
  """dx, dgamma, dbeta (and dalpha, depsilon) of a tensor-core backward and its q: against the emulation given q,
  and against float64 within the split's error model."""
  dx, dgamma, dbeta, dae, q = got
  n_pix, C_ = x.shape
  e = O.gdn_tc_backward_emulated(x, gamma, beta, dy, q, inverse, rectify, alpha, epsilon, pa, pe)
  n, a = e["n"], e["a"]
  kn = k_acc(C_)
  rel_n = a / n
  # q: n enters it at most squared
  q_tol = U * e["q"].abs() * (2 * kn * rel_n + K_EP)
  q_err = (q.double() - e["q"]).abs()
  assert bool((q_err <= q_tol).all()), ("q vs emulation", float((q_err - q_tol).max()))
  # dx = d + dpool * dp
  dx_unit = U * (e["d"].abs() * (rel_n + 1) + e["dpool"].abs() * e["a_dp"])
  dx_tol = U * (e["d"].abs() * (kn * rel_n + K_EP) + e["dpool"].abs() * kn * e["a_dp"] +
                K_EP * (e["dpool"] * e["dp"]).abs())
  dx_err = (dx.double() - e["dx"]).abs()
  assert bool((dx_err <= dx_tol).all()), ("dx vs emulation", float((dx_err / dx_tol.clamp_min(1e-300)).max()))
  dg_err = (dgamma.double() - e["dgamma"]).abs()
  assert bool((dg_err <= K_DGAMMA * U * e["a_dgamma"]).all()), ("dgamma vs emulation", _max(dg_err / (U * e["a_dgamma"])))
  db_err = (dbeta.double() - e["dbeta"]).abs()
  kb = dbeta_k(n_pix, C_)
  assert bool((db_err <= kb * U * e["a_dbeta"]).all()), ("dbeta vs emulation", _max(db_err / (U * e["a_dbeta"])), kb)
  meas = dict(q_vs_emulation_k=_max((q_err / (U * e["q"].abs() * (rel_n + 1)))[e["q"] != 0]),
              dx_vs_emulation_k=_max((dx_err / dx_unit)[dx_unit > 0]),
              dgamma_vs_emulation_k=_max((dg_err / (U * e["a_dgamma"]))[e["a_dgamma"] > 0]),
              dbeta_vs_emulation_k=_max((db_err / (U * e["a_dbeta"]))[e["a_dbeta"] > 0]))

  # float64, the contract's oracle, held to the split's error model carried through q, dp and the sums
  wx, wg, wb = O.gdn_reference_grads(x, gamma, beta, dy, inverse, rectify, O._f32(alpha), O._f32(epsilon),
                                     device=x.device)
  for got_t, want in ((dx, wx), (dgamma, wg), (dbeta, wb)):
    check_masks(got_t, want)
  delta = (O.SPLIT_REL + (kn + 4) * U) * rel_n + U       # n's relative error
  # q's relative error: n's, squared at most; with a literal-pow epsilon also powf's exponent -eps - 1 rounded to fp32
  q_rel = 2 * delta + K_EP * U + (U * torch.log(n).abs() if pe or float(epsilon) not in (1.0, 0.5) else 0)
  w = e["q"].abs() * q_rel                                # q's absolute error
  gam = gamma.to(x.device).double().abs()
  p = O.tc_pool(x, rectify, alpha, pa).double().abs()
  dp_err = O.SPLIT_REL * e["a_dp"] + w @ gam.t() + (kn + 4) * U * e["a_dp"]
  dx_b = (e["d"].abs() * (delta + K_EP * U) + e["dpool"].abs() * dp_err + K_EP * U * (e["dpool"] * e["dp"]).abs())
  dg_b = (O.SPLIT_REL + (K_DGAMMA + 4) * U) * e["a_dgamma"] + p.t() @ w
  db_b = w.sum(0) + kb * U * e["a_dbeta"]
  for name, got_t, want, bound in (("dx", dx, wx, dx_b), ("dgamma", dgamma, wg, dg_b), ("dbeta", dbeta, wb, db_b)):
    err = (got_t.double() - want).abs()
    assert bool((err <= 1.25 * bound + 1e-300).all()), (name, "vs float64", float((err - 1.25 * bound).max()))
    meas[f"{name}_vs_fp64_of_max"] = _of_max(got_t, want)

  if dae is not None:
    ta64, te64 = exact_exponent_terms(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa)
    ks = exponent_sum_k(n_pix, C_)
    u = (torch.relu(x) if rectify else x).double()
    log_u = torch.log(torch.where(u > 0, u, torch.ones_like(u))).abs()
    # dalpha = sum dp p ln u: dp off by kn units of a_dp (emulation) or by dp_err (float64)
    for name, idx, te, t64, per_em, per_64, on in (
        ("dalpha", 0, e["dalpha_terms"], ta64, p * log_u * kn * U * e["a_dp"], p * log_u * dp_err, pa),
        ("depsilon", 1, e["depsilon_terms"], te64,
         e["q"].abs() * (torch.log(n).abs() + 1) * (kn * a + n) * U / abs(O._f32(epsilon)),
         e["q"].abs() * (torch.log(n).abs() + 1) * (delta * n) / abs(O._f32(epsilon)) + te64.abs() * q_rel, pe)):
      if not on:
        continue
      got_v = float(dae[idx])
      em, f64, mag = float(te.sum()), float(t64.sum()), float(te.abs().sum())
      tol_em = float(per_em.sum()) + (ks + K_EP) * U * mag
      assert abs(got_v - em) <= tol_em, (name, "vs emulation", got_v, em, tol_em)
      tol_64 = 1.25 * (float(per_64.sum()) + (ks + K_EP) * U * mag)
      assert abs(got_v - f64) <= tol_64, (name, "vs float64", got_v, f64, tol_64)
      meas[f"{name}_vs_emulation_k"] = abs(got_v - em) / (U * mag)
      meas[f"{name}_vs_fp64_of_sum_abs"] = abs(got_v - f64) / mag
  return meas


# ---- float32 and literal-pow tensor cores -------------------------------------------------------------------------

def _tc_case(F, C_, family, cfg_name, pow_cfg, x=None, dy=None, key_extra=""):
  if pow_cfg:
    inverse, rectify, alpha, epsilon, pa, pe = POW_CONFIGS[cfg_name]
  else:
    (inverse, rectify, alpha, epsilon), pa, pe = FWD_CONFIGS[cfg_name], False, False
  gamma, beta = (t.cuda() for t in FAMILIES[family](C_, 1000 + C_))
  if x is None:
    x, dy = (t.cuda() for t in inputs(BIG, C_, 2000 + C_))
  key = f"tc{'_pow' if pow_cfg else ''} C={C_} {family} {cfg_name}{key_extra}"
  y, n_fwd = run_forward(F, x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe)
  assert n_fwd == 1
  meas = check_forward_tc(y, x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe, key)
  got = run_backward(F, x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe, exponents=pow_cfg)
  assert got[5] == tc_backward_launches(C_, pow_cfg), got[5]  # the tensor-core backward ran
  meas.update(check_backward_tc(got[:5], x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe, key))
  _report(key, **meas)


@pytest.mark.parametrize("cfg_name", sorted(FWD_CONFIGS))
@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("C_", WIDTHS)
def test_float32_tensor_cores_against_emulation_and_float64(F, C_, family, cfg_name):
  _tc_case(F, C_, family, cfg_name, False)


@pytest.mark.parametrize("cfg_name", sorted(POW_CONFIGS))
@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("C_", WIDTHS)
def test_literal_pow_tensor_cores_against_emulation_and_float64(F, C_, family, cfg_name):
  _tc_case(F, C_, family, cfg_name, True)


@pytest.mark.parametrize("C_", WIDTHS)
def test_initialiser_like_parameters_for_comparison(F, C_):
  """The suite's own distribution through the same checks, so the printed maxima can be compared."""
  FAMILIES["initialiser"] = initialiser_like
  try:
    g = torch.Generator().manual_seed(7)
    x = (torch.randn(BIG, C_, generator=g) * (0.05 + 3.95 * torch.rand(C_, generator=g))).cuda()
    dy = torch.randn(BIG, C_, generator=g).cuda()
    for cfg in ("gdn", "igdn"):
      _tc_case(F, C_, "initialiser", cfg, False, x, dy)
    _tc_case(F, C_, "initialiser", "pow_gdn", True, x, dy)
  finally:
    del FAMILIES["initialiser"]


@pytest.mark.parametrize("C_", [128, 192])
def test_dgamma_over_several_flushes(F, C_):
  """Enough pixels that every dgamma CTA flushes its accumulator into its partial more than once (kDgFlush chunks)."""
  n_pix = 64 * min(_sms(), 148) * 8 * 2 + 37
  x, dy = (t.cuda() for t in inputs(n_pix, C_, 3000 + C_))
  _tc_case(F, C_, "trained", "gdn", False, x, dy, key_extra=f" n_pix={n_pix}")


# ---- 16-bit activations --------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("C_", [128, 192])
def test_sixteen_bit_is_the_conversion_path_and_its_core_meets_the_emulation(F, C_, dtype):
  inverse, rectify, alpha, epsilon = FWD_CONFIGS["gdn_rectify_sq_sqrt"] if C_ == 192 else FWD_CONFIGS["gdn"]
  gamma, beta = (t.cuda() for t in trained_like(C_, 4000 + C_))
  x, dy = inputs(BIG, C_, 4100 + C_)
  x16, dy16 = x.to(dtype).cuda(), dy.to(dtype).cuda()
  assert F._gdn_native16(x16, C_, BIG, alpha, epsilon, False, False, dy16)
  y16, n_fwd = run_forward(F, x16, gamma, beta, inverse, rectify, alpha, epsilon)
  assert n_fwd == 1 and y16.dtype == dtype  # one kernel, no conversion passes
  y32 = F.gdn_forward(x16.float(), gamma, beta, inverse, rectify, alpha, epsilon)
  assert torch.equal(y16, y32.to(dtype))
  dx16, dg16, db16 = F.gdn_backward(x16, gamma, beta, dy16, inverse, rectify, alpha, epsilon)
  dx32, dg32, db32 = F.gdn_backward(x16.float(), gamma, beta, dy16.float(), inverse, rectify, alpha, epsilon)
  assert torch.equal(dx16, dx32.to(dtype)) and torch.equal(dg16, dg32) and torch.equal(db16, db32)
  # the float32 core they share, held to the emulation and to float64
  cfg = [k for k, v in FWD_CONFIGS.items() if v == (inverse, rectify, alpha, epsilon)][0]
  FAMILIES["trained16"] = lambda c, s: trained_like(c, 4000 + C_)
  try:
    _tc_case(F, C_, "trained16", cfg, False, x16.float(), dy16.float(), key_extra=f" {dtype}")
  finally:
    del FAMILIES["trained16"]


# ---- channels-first --------------------------------------------------------------------------------------------

CF_CASES = [  # one width per kernel family: (C, dtype, config, pow)
    (128, torch.float32, "gdn", False),
    (320, torch.float32, "igdn_rectify", False),
    (192, torch.float32, "pow_gdn", True),
    (256, torch.float32, "pow_igdn", True),
    (192, torch.bfloat16, "gdn_rectify_sq_sqrt", False),
]


@pytest.mark.parametrize("C_,dtype,cfg_name,pow_cfg", CF_CASES)
def test_channels_first_is_channels_last_bit_for_bit(F, C_, dtype, cfg_name, pow_cfg):
  if pow_cfg:
    inverse, rectify, alpha, epsilon, pa, pe = POW_CONFIGS[cfg_name]
  else:
    (inverse, rectify, alpha, epsilon), pa, pe = FWD_CONFIGS[cfg_name], False, False
  gamma, beta = (t.cuda() for t in saturated(C_, 5000 + C_))
  n_items, spatial = 5, 1077  # 5385 pixels: tiles span two items
  x, dy = inputs(n_items * spatial, C_, 5100 + C_)
  x, dy = x.to(dtype).cuda(), dy.to(dtype).cuda()
  cf = lambda t: t.view(n_items, spatial, C_).permute(0, 2, 1).contiguous()
  xc, dyc = cf(x), cf(dy)
  assert F._gdn_native_cf(xc, alpha, epsilon, pa, pe, dyc, exponent_grads=pow_cfg)
  y = F.gdn_forward(x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe)
  yc = F.gdn_forward(xc, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe, channels_first=True)
  assert torch.equal(cf(y), yc)
  if pow_cfg:
    a = F.gdn_backward_exponents(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe)
    b = F.gdn_backward_exponents(xc, gamma, beta, dyc, inverse, rectify, alpha, epsilon, pa, pe, channels_first=True)
  else:
    a = F.gdn_backward(x, gamma, beta, dy, inverse, rectify, alpha, epsilon)
    b = F.gdn_backward(xc, gamma, beta, dyc, inverse, rectify, alpha, epsilon, channels_first=True)
  assert torch.equal(cf(a[0]), b[0])
  for u, v in zip(a[1:], b[1:]):
    assert torch.equal(u, v)
  assert torch.isfinite(yc.float()).all() and torch.isfinite(b[1]).all()


# ---- CUDA cores ----------------------------------------------------------------------------------------------------

def _err_report(got, want):
  """(max |err| / max |want|, max elementwise relative error over entries with |want| >= 1 % of max |want|), as in
  test_gdn_gpu.py."""
  got, want = got.double(), want.double()
  scale = float(want.abs().max())
  err = (got - want).abs()
  big = want.abs() >= 1e-2 * scale
  return float(err.max()) / scale, float((err[big] / want.abs()[big]).max())


def _cuda_core_case(F, C_, family, cfg_name, pow_cfg):
  if pow_cfg:
    inverse, rectify, alpha, epsilon, pa, pe = POW_CONFIGS[cfg_name]
  else:
    (inverse, rectify, alpha, epsilon), pa, pe = FWD_CONFIGS[cfg_name], False, False
  gamma, beta = (t.cuda() for t in FAMILIES[family](C_, 6000 + C_))
  n_pix = BIG if C_ <= 192 else 5003
  x, dy = (t.cuda() for t in inputs(n_pix, C_, 6100 + C_))
  y, n_fwd = run_forward(F, x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe)
  assert n_fwd == 1
  y64 = O.gdn_reference(x, gamma, beta, inverse, rectify, O._f32(alpha), O._f32(epsilon), device=x.device)
  check_masks(y, y64)
  err = (y.double() - y64).abs()
  rel = _max((err / y64.abs())[y64 != 0])
  assert bool((err <= 1e-5 * y64.abs()).all()), ("forward", rel)  # BASELINE.json: within 1e-5 relative
  dx, dgamma, dbeta, dae, _, launches = run_backward(F, x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe,
                                                     exponents=pow_cfg)
  tiled = C_ % 32 == 0 and C_ <= 192
  assert launches == (5 if tiled else 2) + (2 if pow_cfg else 0), launches  # the CUDA-core kernels ran
  wx, wg, wb = O.gdn_reference_grads(x, gamma, beta, dy, inverse, rectify, O._f32(alpha), O._f32(epsilon),
                                     device=x.device)
  meas = dict(fwd_vs_fp64_rel=rel)
  for name, got, want in (("dx", dx, wx), ("dgamma", dgamma, wg), ("dbeta", dbeta, wb)):
    check_masks(got, want)
    of_max, rel_big = _err_report(got, want)
    assert of_max < 1e-5 and rel_big < 5e-4, (name, of_max, rel_big)
    meas[f"{name}_vs_fp64_of_max"] = of_max
    meas[f"{name}_vs_fp64_rel_big"] = rel_big
  if pow_cfg:
    ta, te = exact_exponent_terms(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa)
    for name, idx, terms, on in (("dalpha", 0, ta, pa), ("depsilon", 1, te, pe)):
      if on:
        e = abs(float(dae[idx]) - float(terms.sum())) / float(terms.abs().sum())
        assert e < 1e-5, (name, e)  # a sum with cancellation: relative to the sum of |terms|
        meas[f"{name}_vs_fp64_of_sum_abs"] = e
  _report(f"cuda-core C={C_} {family} {cfg_name}", **meas)


@pytest.mark.parametrize("cfg_name", sorted(FWD_CONFIGS) + sorted(POW_CONFIGS))
@pytest.mark.parametrize("family", ["trained", "diagonal"])
@pytest.mark.parametrize("C_", [128, 192])
def test_cuda_cores_under_fp32_switch_meet_the_contract(F, fp32_path, C_, family, cfg_name):
  _cuda_core_case(F, C_, family, cfg_name, cfg_name in POW_CONFIGS)


@pytest.mark.parametrize("cfg_name", sorted(FWD_CONFIGS) + sorted(POW_CONFIGS))
@pytest.mark.parametrize("family", ["trained", "saturated"])
@pytest.mark.parametrize("C_", [7, 64, 384])
def test_cuda_cores_at_other_widths_meet_the_contract(F, C_, family, cfg_name):
  _cuda_core_case(F, C_, family, cfg_name, cfg_name in POW_CONFIGS)
