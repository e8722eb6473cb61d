"""CPU references of the checkerboard context model with mixture priors (csrc/cb_mixture.cu, DESIGN §3.19), on top of
checkerboard_oracle's passes and ar_oracle's float32 emulation.

  - raw32 emulates a pass's dense layers bit for bit (ar_oracle.dense32's order; the last layer has 3KM outputs and
    no LeakyReLU); epilogue32 is the kernel's epilogue with numpy's correctly rounded exp in place of CUDA's expf,
    which is within EXPF_ULP ulp of it: weight_k = exp(fl32(l_k - m)), m the largest logit (NaN ignored), loc_k raw,
    scale_k = fmaxf(raw, 0.11f).
  - raw64 restates a pass in float64 with checkerboard_oracle's per-layer bound; epilogue_bound64 carries that bound
    through the epilogue.
  - encode32 is the two-pass encoder: y_hat = float(int32(rint(y))) (saturating, NaN -> 0), and the coding-order y
    with its mixtures.

Packed weights are the list [ctx kernel [5, 5, M, 2M], ctx bias, W1, b1, W2, b2, W3 [8M/3, 3KM], b3]; latents are
[B, H, W, M], psi [B, H, W, 2M]; raw outputs [B, n, 3KM] and mixture parameters [B, n, M, K] in coding order.
"""
import numpy as np

from oracle import ar_oracle as ar
from oracle import checkerboard_oracle as cb

EXPF_ULP = 2  # CUDA's expf: maximum ulp error over the full range (CUDA C++ Programming Guide, single precision)
SCALE_MIN = np.float32(0.11)


def raw32(ws, y_hat, psi, anchors):
  """The last layer's raw outputs [B, n, 3KM] of one pass, in coding order, bit for bit as the kernel writes them."""
  psi = ar._f32(psi)
  B, H, W, C = psi.shape
  pos = cb.positions(H, W, anchors)
  NO = ar._f32(ws[6]).shape[1]
  if not pos:  # the non-anchors of a 1x1 latent
    return np.zeros((B, 0, NO), np.float32)
  if anchors:
    return cb._anchor_out(ws, psi, pos, ar.dense32)
  x = cb.gather(y_hat, pos)
  P = x.shape[1]
  out = ar.network32(cb.packed_list(ws), x.reshape(B * P, -1), ar._psi_rows(psi, pos).reshape(B * P, -1))
  return out.reshape(B, P, NO)


def split(raw, K):
  """(logits, locs, scales) [..., M, K] of raw outputs [..., 3KM]: channel c at 3Kc .. 3Kc + 3K - 1."""
  r = raw.reshape(raw.shape[:-1] + (raw.shape[-1] // (3 * K), 3, K))
  return r[..., 0, :], r[..., 1, :], r[..., 2, :]


def epilogue32(raw, K):
  """(weight, loc, scale) [..., M, K] in float32.  weight uses float64 exp of the float32 difference, rounded once:
  the kernel's expf lies within EXPF_ULP ulp of it; loc and scale are exact."""
  l, mu, s = split(ar._f32(raw), K)
  m = np.fmax.reduce(l, axis=-1, keepdims=True)
  with np.errstate(invalid="ignore", over="ignore"):
    d = (l - m).astype(np.float32)  # one correctly rounded float32 subtraction
    w = np.exp(d.astype(np.float64)).astype(np.float32)
  return w, mu.copy(), np.fmax(s, SCALE_MIN)


def ulp32(x):
  """The spacing of float32 at |x| (the smallest subnormal at 0)."""
  a = np.abs(np.asarray(x, np.float32))
  return np.spacing(a).astype(np.float64)


def params32(ws, y_hat, psi, anchors, K):
  """(weight, loc, scale) [B, n, M, K] of one pass: loc and scale bit for bit, weight within EXPF_ULP ulp."""
  return epilogue32(raw32(ws, y_hat, psi, anchors), K)


def encode32(ws, y, psi, K):
  """The two-pass encoder: (y_hat [B, H, W, M], y [B, H W, M], weight, loc, scale [B, H W, M, K]) in coding order."""
  y = ar._f32(y)
  B, H, W, M = y.shape
  y_hat = ar.rint_to_int32(y).astype(np.float32)
  flat = y.reshape(B, H * W, M)
  parts = [params32(ws, y_hat, psi, anchors, K) for anchors in (True, False)]
  order = cb.coding_order(H, W)
  return (y_hat, flat[:, order]) + tuple(np.concatenate([p[i] for p in parts], 1) for i in range(3))


# ---------------------------------------------------------------------------------------------------------------
# float64: the restatement and its bound
# ---------------------------------------------------------------------------------------------------------------
def raw64(ws, y_hat, psi, anchors):
  """(raw outputs [B, n, 3KM] in float64, a-priori bound on |raw32 - exact|), as checkerboard_oracle.bound64."""
  wc, bc, w1, b1, w2, b2, w3, b3 = [w.astype(np.float64) for w in ar.unpack(cb.packed_list(ws))]
  x, ps, (B, P) = cb._inputs(y_hat, psi, anchors)
  ps = ps.astype(np.float64)
  if anchors:
    ctx, e = np.zeros_like(ps), np.zeros_like(ps)
  else:
    ctx, e = ar._dense_bound(x.astype(np.float64), np.zeros(x.shape), wc, bc, False)
  h, e = ar._dense_bound(np.concatenate([ps, ctx], -1), np.concatenate([np.zeros_like(ps), e], -1), w1, b1, True)
  h, e = ar._dense_bound(h, e, w2, b2, True)
  out, e = ar._dense_bound(h, e, w3, b3, False)
  return out.reshape(B, P, -1), e.reshape(B, P, -1)


def epilogue64(raw, K):
  """(weight, loc, scale) in float64: the same definitions without rounding."""
  l, mu, s = split(np.asarray(raw, np.float64), K)
  return np.exp(l - l.max(-1, keepdims=True)), mu, np.maximum(s, float(SCALE_MIN))


def epilogue_bound64(raw, bound, K):
  """Bounds on |epilogue32 of the float32 raw outputs - epilogue64 of the exact ones|, given |raw32 - raw| <= bound:
  loc and scale inherit the raw bound (fmax is 1-Lipschitz); a weight's exponent d = l_k - m is off by at most
  e_k + max_j e_j plus its float32 rounding, and the weight by exp(d + δ) - exp(d) plus EXPF_ULP ulp of the result."""
  l, _, _ = split(np.asarray(raw, np.float64), K)
  el, emu, es = split(np.asarray(bound, np.float64), K)
  d = l - l.max(-1, keepdims=True)
  delta = el + el.max(-1, keepdims=True)
  delta = delta + ar.U32 * (np.abs(d) + delta)
  hi = np.exp(d + delta)
  w_bound = (hi - np.exp(d)) + EXPF_ULP * np.spacing(np.abs(hi).astype(np.float32)).astype(np.float64)
  return w_bound, emu, es
