"""CPU references of the joint autoregressive prior's parameter network (csrc/autoregressive.cu), written from the
kernel's documented order of operations and the layer shapes of Minnen, Ballé & Toderici (2018).

Two references, for two different claims:
  - params32 / encode32 emulate the kernel's float32 arithmetic exactly: every dense output is
    ((bias + P_0) + ... + P_7) with P_s a correctly rounded fma chain from +0.0f over k in [s*K//8, (s+1)*K//8) in
    increasing k, LeakyReLU is `v > 0 ? v : fl32(v * 0.01f)`, and subnormals are kept (no flush to zero).  The kernel
    must agree with them bit for bit.
  - params64 restates the same mathematics in float64 and bound64 is an a-priori bound on |fl32 - exact| for the
    kernel's order, so params32 within bound64 of params64 shows that the emulated order computes the right function.

Packed weights are the list [ctx kernel [5, 5, M, 2M], ctx bias [2M], W1 [4M, 10M/3], b1, W2 [10M/3, 8M/3], b2,
W3 [8M/3, 2M], b3] as numpy float32 arrays (or tensors); the context layer reads the 12 causal taps of the kernel, its
first 12 * M * 2M floats.  Latents are [B, H, W, M], the hyper feature psi [B, H, W, 2M]; positions are raster
indexes p = y * W + x.  Everything is numpy, vectorised over images, positions and outputs: only the k-chain of a
slice is sequential.
"""
import numpy as np

SLICES = 8
TAPS = 12
SLOPE32 = np.float32(0.01)  # kArLeakySlope
U32 = 2.0**-24  # unit roundoff of float32
U64 = 2.0**-53


def _f32(x):
  return np.asarray(x.detach().cpu().numpy() if hasattr(x, "detach") else x, dtype=np.float32)


def fma32(a, b, c):
  """Correctly rounded float32 a * b + c, elementwise.  The product of two float32 values is exact in float64; the
  sum is formed in float64 with its exact error from TwoSum, rounded to odd at 53 bits, then rounded to nearest even
  at 24 bits, which is correct rounding (Boldo & Melquiond, "Emulation of FMA and correctly rounded sums: proved
  algorithms using rounding to odd", IEEE TC 2008).  float32(a * b + c) in float64 alone would round twice."""
  a, b, c = (np.asarray(t, np.float32).astype(np.float64) for t in (a, b, c))
  p = a * b
  s = p + c
  bb = s - p
  err = (p - (s - bb)) + (c - bb)
  even = (s.view(np.int64) & 1) == 0
  fix = (err != 0) & even & np.isfinite(s)
  s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
  return s.astype(np.float32)


def _bounds(K, s):
  return s * K // SLICES, (s + 1) * K // SLICES


def dense32(x, W, b, leaky):
  """The kernel's ar_dense: x [N, K], W [K, nout], b [nout] -> [N, nout] float32, in the kernel's exact order.
  The eight slices' chains run side by side; a slice shorter than the longest one leaves its accumulator alone."""
  x, W, b = _f32(x), _f32(W), _f32(b)
  N, K = x.shape
  nout = W.shape[1]
  k0 = np.array([_bounds(K, s)[0] for s in range(SLICES)])
  lens = np.array([_bounds(K, s)[1] for s in range(SLICES)]) - k0
  acc = np.zeros((N, SLICES, nout), np.float32)
  for i in range(int(lens.max())):
    live = i < lens
    k = np.where(live, k0 + i, 0)
    step = fma32(x[:, k][:, :, None], W[k][None], acc)
    acc = np.where(live[None, :, None], step, acc)
  v = np.broadcast_to(b, (N, nout)).astype(np.float32)
  for s in range(SLICES):
    v = v + acc[:, s]  # float32 + float32 in numpy: one correctly rounded addition
  if leaky:
    v = np.where(v > 0, v, v * SLOPE32)
  return v


def taps(y_hat, positions):
  """The 12 causal neighbours of a 5x5 type-A mask at each position, raster order, as [B, P, tap * M + channel]
  (the kernel's `taps` layout); zero where yy < 0 or xx is outside [0, W)."""
  y_hat = _f32(y_hat)
  B, H, W, M = y_hat.shape
  out = np.zeros((B, len(positions), TAPS, M), np.float32)
  for i, p in enumerate(positions):
    py, px = divmod(int(p), W)
    for t in range(TAPS):
      yy, xx = py + t // 5 - 2, px + t % 5 - 2
      if yy >= 0 and 0 <= xx < W:
        out[:, i, t] = y_hat[:, yy, xx]
  return out.reshape(B, len(positions), TAPS * M)


def unpack(ws):
  """[Wc [12M, 2M], bc, W1, b1, W2, b2, W3, b3] as float32 arrays, Wc read from the context kernel's first
  12 * M * 2M floats as ar_pack_weights lays them out."""
  ws = [_f32(w) for w in ws]
  M = ws[0].shape[2]
  wc = ws[0].reshape(-1)[:TAPS * M * 2 * M].reshape(TAPS * M, 2 * M)
  return [wc] + ws[1:]


def table_index(s, num_scales):
  """The kernel's ar_table_index: NaN-propagating max with 0, then min with num_scales - 1, truncated to int32;
  NaN -> 0 (the GPU's float-to-int conversion)."""
  s = np.asarray(s, np.float32)
  v = np.where(np.isnan(s), s, np.maximum(s, np.float32(0)))
  v = np.where(np.isnan(v), v, np.minimum(v, np.float32(num_scales - 1)))
  return np.where(np.isnan(v), 0, np.trunc(np.nan_to_num(v))).astype(np.int32)


def network32(ws, x_taps, psi_rows, dense=dense32):
  """[N, 12M] taps and [N, 2M] hyper features -> [N, 2M] = [loc, scale_index] in the kernel's float32 order."""
  wc, bc, w1, b1, w2, b2, w3, b3 = unpack(ws)
  ctx = dense(x_taps, wc, bc, False)
  h = dense(np.concatenate([_f32(psi_rows), ctx], -1), w1, b1, True)
  h = dense(h, w2, b2, True)
  return dense(h, w3, b3, False)


def _psi_rows(psi, positions):
  psi = _f32(psi)
  B, H, W, C = psi.shape
  return psi.reshape(B, H * W, C)[:, list(positions)]


def params32(ws, y_hat, psi, positions, num_scales, dense=dense32, gather=taps):
  """(loc, scale_index, index), each [B, len(positions), M], bit for bit as tfcb_ar_params gives them at each
  position (float32, float32, int32)."""
  x = gather(y_hat, positions)
  B, P = x.shape[:2]
  out = network32(ws, x.reshape(B * P, -1), _psi_rows(psi, positions).reshape(B * P, -1), dense)
  M = out.shape[1] // 2
  out = out.reshape(B, P, 2 * M)
  loc, scale = out[..., :M], out[..., M:]
  return loc, scale, table_index(scale, num_scales)


def rint_to_int32(d):
  """(int)rintf(d) on the GPU: round half to even, saturated to the int32 range, NaN -> 0."""
  d = np.asarray(d, np.float32).astype(np.float64)
  r = np.clip(np.rint(np.nan_to_num(d, nan=0.0)), -2.0**31, 2.0**31 - 1)
  return r.astype(np.int32)


def encode32(ws, y, psi, num_scales):
  """The encoder loop over every position in raster order: (y_hat, loc, index, scale_index) [B, H, W, M] with
  q = (int)rintf(y - loc) and y_hat = float(q) + loc in float32."""
  y = _f32(y)
  B, H, W, M = y.shape
  y_hat = np.zeros_like(y)
  loc, scale = np.zeros_like(y), np.zeros_like(y)
  index = np.zeros(y.shape, np.int32)
  fy, fyh, floc, fsc, fix = (t.reshape(B, H * W, M) for t in (y, y_hat, loc, scale, index))
  for p in range(H * W):
    l, s, i = params32(ws, y_hat, psi, [p], num_scales)
    q = rint_to_int32(fy[:, p] - l[:, 0])
    fyh[:, p] = q.astype(np.float32) + l[:, 0]
    floc[:, p], fsc[:, p], fix[:, p] = l[:, 0], s[:, 0], i[:, 0]
  return y_hat, loc, index, scale


# ---------------------------------------------------------------------------------------------------------------
# float64: the restatement and the bound of the float32 order's error
# ---------------------------------------------------------------------------------------------------------------
def _inputs64(y_hat, psi, positions):
  x = taps(y_hat, positions).astype(np.float64)
  B, P = x.shape[:2]
  return x.reshape(B * P, -1), _psi_rows(psi, positions).astype(np.float64).reshape(B * P, -1), (B, P)


def params64(ws, y_hat, psi, positions):
  """(loc, scale_index) [B, P, M] in float64, with the slope float(float32(0.01)) the kernel multiplies by."""
  wc, bc, w1, b1, w2, b2, w3, b3 = [w.astype(np.float64) for w in unpack(ws)]
  x, ps, (B, P) = _inputs64(y_hat, psi, positions)
  slope = float(SLOPE32)
  lk = lambda v: np.where(v > 0, v, v * slope)
  ctx = x @ wc + bc
  h = lk(np.concatenate([ps, ctx], -1) @ w1 + b1)
  h = lk(h @ w2 + b2)
  out = (h @ w3 + b3).reshape(B, P, -1)
  M = out.shape[-1] // 2
  return out[..., :M], out[..., M:]


def _gamma(m, u):
  return m * u / (1 - m * u)


def _dense_bound(x, e, W, b, leaky):
  """(exact output, its error bound) of one layer from the exact input x and the bound e on the float32 input's
  error.  The float32 order rounds every term at most n + 8 times (an fma chain of n = ceil(K/8) steps, then eight
  additions), so with |x̂| <= |x| + e:  e_out <= γ_{n+8} (|b| + Σ|W|(|x| + e)) + Σ|W| e;  the float64 restatement's
  own rounding adds γ⁶⁴_{K+1} of the same sum.  LeakyReLU is 1-Lipschitz and its float32 multiply adds u |0.01 v|."""
  K = W.shape[0]
  n = -(-K // SLICES)
  aW, ab = np.abs(W), np.abs(b)
  mag = ab + (np.abs(x) + e) @ aW
  v = x @ W + b
  bound = (_gamma(n + SLICES, U32) + _gamma(K + 1, U64)) * mag + e @ aW
  if leaky:
    slope = float(SLOPE32)
    bound = bound + (U32 + U64) * slope * (np.abs(v) + bound)
    v = np.where(v > 0, v, v * slope)
  return v, bound


def bound64(ws, y_hat, psi, positions):
  """(loc bound, scale_index bound) [B, P, M]: a-priori bounds on |params32 - exact| (and so, up to the float64
  rounding they include, on |params32 - params64|).  The taps and psi are read exactly: their error is zero."""
  wc, bc, w1, b1, w2, b2, w3, b3 = [w.astype(np.float64) for w in unpack(ws)]
  x, ps, (B, P) = _inputs64(y_hat, psi, positions)
  ctx, e = _dense_bound(x, np.zeros_like(x), wc, bc, False)
  x1 = np.concatenate([ps, ctx], -1)
  e1 = np.concatenate([np.zeros_like(ps), e], -1)
  h, e = _dense_bound(x1, e1, w1, b1, True)
  h, e = _dense_bound(h, e, w2, b2, True)
  _, e = _dense_bound(h, e, w3, b3, False)
  e = e.reshape(B, P, -1)
  M = e.shape[-1] // 2
  return e[..., :M], e[..., M:]


def layer_errors(ws, y_hat, psi, positions, dense=dense32):
  """Each layer of the float32 emulation against the same layer in float64 on the emulation's own float32 input:
  a list of four (|fl32 - float64|, bound, |float64|) arrays [B * P, outputs], the bound being _dense_bound's with
  an exact input.  bound64 carries every layer's worst case through the following layers' Σ|W|, which multiplies it
  by about 10^3 at M = 96 for weights of the tests' scale; this check bounds each layer by its own rounding alone."""
  wc, bc, w1, b1, w2, b2, w3, b3 = unpack(ws)
  x = taps(y_hat, positions)
  B, P = x.shape[:2]
  x = x.reshape(B * P, -1)
  ps = _psi_rows(psi, positions).reshape(B * P, -1)
  out = []
  for i, (W, b, leaky) in enumerate(((wc, bc, False), (w1, b1, True), (w2, b2, True), (w3, b3, False))):
    if i == 1:
      x = np.concatenate([ps, x], -1)  # [psi, ctx]
    got = dense(x, W, b, leaky)
    x64 = x.astype(np.float64)
    want, bound = _dense_bound(x64, np.zeros_like(x64), W.astype(np.float64), b.astype(np.float64), leaky)
    out.append((np.abs(got.astype(np.float64) - want), bound, np.abs(want)))
    x = got
  return out
