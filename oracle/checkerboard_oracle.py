"""CPU references of the checkerboard context model's parameter passes (csrc/checkerboard.cu), written from the
definitions of He, Zheng, Sun, Wang & Qin (CVPR 2021) and the kernel's documented order of operations, on top of
ar_oracle's float32 emulation.

  - Colours: (r, c) is an anchor when r + c is even.  Coding order: each image's anchors in raster order, then its
    non-anchors in raster order.
  - Context: 0 at an anchor (bias included); at a non-anchor bc + Wc · (ŷ at the 12 taps (dy, dx) in [-2, 2]^2 with
    dy + dx odd, raster order, zero outside the image).
  - params32 / encode32 emulate the kernel bit for bit (ar_oracle.dense32's order); params64 / bound64 restate the
    mathematics in float64 with ar_oracle's derived per-layer bound.

Packed weights are the list [ctx kernel [5, 5, M, 2M], ctx bias, W1, b1, W2, b2, W3, b3], as for ar_oracle; latents
are [B, H, W, M], psi [B, H, W, 2M], and coding-order outputs [B, n, M].
"""
import numpy as np

from oracle import ar_oracle as ar

TAPS = tuple((dy, dx) for dy in range(-2, 3) for dx in range(-2, 3) if (dy + dx) % 2)


def counts(H, W):
  """(anchors, non-anchors) per image."""
  return (H * W + 1) // 2, H * W // 2


def positions(H, W, anchors):
  """Raster indexes of one colour's positions, in coding order."""
  return [p for p in range(H * W) if (p // W + p % W) % 2 == (0 if anchors else 1)]


def coding_order(H, W):
  """Raster index of each coding-order row: the anchors, then the non-anchors."""
  return np.array(positions(H, W, True) + positions(H, W, False), np.int64)


def gather(y_hat, pos, taps=TAPS, wrap=False):
  """The checkerboard taps at each position as [B, P, tap * M + channel], zero outside the image.  `taps` and
  `wrap` (rows wrap into the neighbouring row) exist to show that a wrong gather changes the bits."""
  y_hat = ar._f32(y_hat)
  B, H, W, M = y_hat.shape
  flat = y_hat.reshape(B, H * W, M)
  out = np.zeros((B, len(pos), len(taps), M), np.float32)
  for i, p in enumerate(pos):
    py, px = divmod(int(p), W)
    for t, (dy, dx) in enumerate(taps):
      yy, xx = py + dy, px + dx
      if wrap:
        q = yy * W + xx
        if 0 <= q < H * W:
          out[:, i, t] = flat[:, q]
      elif 0 <= yy < H and 0 <= xx < W:
        out[:, i, t] = y_hat[:, yy, xx]
  return out.reshape(B, len(pos), len(taps) * M)


def packed_list(ws, taps=TAPS):
  """ws with the context kernel replaced by its checkerboard taps, [12, 1, M, 2M]: what cb_pack_weights packs, in a
  shape ar_oracle.unpack reads (its first 12 * M * 2M floats)."""
  k = ar._f32(ws[0])
  sel = np.stack([k[dy + 2, dx + 2] for dy, dx in taps])
  return [sel[:, None]] + [ar._f32(w) for w in ws[1:]]


def _anchor_out(ws, psi, pos, dense):
  _, _, w1, b1, w2, b2, w3, b3 = ar.unpack(packed_list(ws))
  psi_rows = ar._psi_rows(psi, pos)
  B, P, C = psi_rows.shape
  x1 = np.concatenate([psi_rows.reshape(B * P, C), np.zeros((B * P, C), np.float32)], -1)
  h = dense(x1, w1, b1, True)
  h = dense(h, w2, b2, True)
  return dense(h, w3, b3, False).reshape(B, P, -1)


def params32(ws, y_hat, psi, anchors, num_scales, dense=ar.dense32, gather_fn=gather):
  """(loc, scale_index, index) [B, n, M] of one pass, in coding order, bit for bit as tfcb_cb_params gives them."""
  psi = ar._f32(psi)
  B, H, W, C = psi.shape
  pos = positions(H, W, anchors)
  if not pos:  # the non-anchors of a 1x1 latent
    empty = np.zeros((B, 0, C // 2), np.float32)
    return empty, empty, empty.astype(np.int32)
  if anchors:
    out = _anchor_out(ws, psi, pos, dense)
    M = out.shape[-1] // 2
    return out[..., :M], out[..., M:], ar.table_index(out[..., M:], num_scales)
  return ar.params32(packed_list(ws), y_hat, psi, pos, num_scales, dense=dense, gather=gather_fn)


def encode32(ws, y, psi, num_scales):
  """The two-pass encoder: (y_hat [B, H, W, M], and y, loc, index, scale_index in coding order [B, H W, M])."""
  y = ar._f32(y)
  B, H, W, M = y.shape
  y_hat = np.zeros_like(y)
  flat_y, flat_hat = y.reshape(B, H * W, M), y_hat.reshape(B, H * W, M)
  parts = []
  for anchors in (True, False):
    pos = positions(H, W, anchors)
    loc, scale, index = params32(ws, y_hat, psi, anchors, num_scales)
    q = ar.rint_to_int32(flat_y[:, pos] - loc)
    flat_hat[:, pos] = q.astype(np.float32) + loc
    parts.append((flat_y[:, pos], loc, index, scale))
  return (y_hat,) + tuple(np.concatenate([a[i] for a in parts], 1) for i in range(4))


# ---------------------------------------------------------------------------------------------------------------
# float64: the restatement and ar_oracle's bound, per pass
# ---------------------------------------------------------------------------------------------------------------
def _inputs(y_hat, psi, anchors):
  psi = ar._f32(psi)
  B, H, W, C = psi.shape
  pos = positions(H, W, anchors)
  ps = ar._psi_rows(psi, pos).reshape(B * len(pos), C)
  x = None if anchors else gather(y_hat, pos).reshape(B * len(pos), -1)
  return x, ps, (B, len(pos))


def _layers(ws, y_hat, psi, anchors, dense_bound):
  wc, bc, w1, b1, w2, b2, w3, b3 = [w.astype(np.float64) for w in ar.unpack(packed_list(ws))]
  x, ps, (B, P) = _inputs(y_hat, psi, anchors)
  ps = ps.astype(np.float64)
  if anchors:
    ctx, e = np.zeros_like(ps), np.zeros_like(ps)
  else:
    x = x.astype(np.float64)
    ctx, e = dense_bound(x, np.zeros_like(x), wc, bc, False)
  h, e = dense_bound(np.concatenate([ps, ctx], -1), np.concatenate([np.zeros_like(ps), e], -1), w1, b1, True)
  h, e = dense_bound(h, e, w2, b2, True)
  out, e = dense_bound(h, e, w3, b3, False)
  M = out.shape[-1] // 2
  out, e = out.reshape(B, P, -1), e.reshape(B, P, -1)
  return (out[..., :M], out[..., M:]), (e[..., :M], e[..., M:])


def params64(ws, y_hat, psi, anchors):
  """(loc, scale_index) [B, n, M] of one pass in float64."""
  return _layers(ws, y_hat, psi, anchors, ar._dense_bound)[0]


def bound64(ws, y_hat, psi, anchors):
  """(loc bound, scale_index bound) [B, n, M]: ar_oracle's a-priori bound on |params32 - exact| for this pass."""
  return _layers(ws, y_hat, psi, anchors, ar._dense_bound)[1]


def layer_errors(ws, y_hat, psi, anchors, dense=ar.dense32):
  """Each layer of the float32 emulation against float64 on the emulation's own float32 input, as
  ar_oracle.layer_errors: a list of (|fl32 - float64|, bound, |float64|) arrays, three layers at the anchors and
  four at the non-anchors."""
  wc, bc, w1, b1, w2, b2, w3, b3 = ar.unpack(packed_list(ws))
  x, ps, _ = _inputs(y_hat, psi, anchors)
  layers = [(w1, b1, True), (w2, b2, True), (w3, b3, False)]
  if anchors:
    x = np.concatenate([ps, np.zeros_like(ps)], -1)
  else:
    layers.insert(0, (wc, bc, False))
  out = []
  for i, (Wt, b, leaky) in enumerate(layers):
    if i == 1 and not anchors:
      x = np.concatenate([ps, x], -1)
    got = dense(x, Wt, b, leaky)
    x64 = x.astype(np.float64)
    want, bound = ar._dense_bound(x64, np.zeros_like(x64), Wt.astype(np.float64), b.astype(np.float64), leaky)
    out.append((np.abs(got.astype(np.float64) - want), bound, np.abs(want)))
    x = got
  return out
