"""CPU references of the multistage context model's parameter passes (csrc/multistage.cu), written from the 2x2
schedule's definition and the kernel's documented order of operations, on top of ar_oracle's float32 emulation.

  - Stages: (r, c) has phase (r mod 2, c mod 2); the phases (0, 0), (1, 1), (0, 1), (1, 0) are stages 0 to 3.  Coding
    order: each image's stage 0 in raster order, then stages 1, 2 and 3.
  - Context: 0 at stage 0 (bias included); at stage s >= 1 bc_s + Wc_s · (ŷ at the stage's taps, the offsets (dy, dx)
    in [-2, 2]^2 whose neighbour lies in an earlier stage, raster order, zero outside the image).
  - params32 / encode32 emulate the kernel bit for bit (ar_oracle.dense32's order); params64 / bound64 restate the
    mathematics in float64 with ar_oracle's derived per-layer bound; context64 is the context feature of every
    position in float64, the training form's definition.

Weights are the list [ctx kernels (three [5, 5, M, 2M], stages 1-3), ctx biases (three [2M]), W1, b1, W2, b2, W3, b3];
latents are [B, H, W, M], psi [B, H, W, 2M], and coding-order outputs [B, n_s, M].
"""
import numpy as np

from oracle import ar_oracle as ar

PHASES = ((0, 0), (1, 1), (0, 1), (1, 0))


def stage_of(r, c):
  return PHASES.index((r % 2, c % 2))


TAPS = tuple(tuple((dy, dx) for dy in range(-2, 3) for dx in range(-2, 3)
                   if (dy, dx) != (0, 0) and stage_of(a + dy, b + dx) < s) for s, (a, b) in enumerate(PHASES))


def counts(H, W):
  """Positions of stages 0 to 3 per image."""
  return tuple(len(positions(H, W, s)) for s in range(4))


def positions(H, W, stage):
  """Raster indexes of one stage's positions, in coding order."""
  return [p for p in range(H * W) if stage_of(p // W, p % W) == stage]


def coding_order(H, W):
  """Raster index of each coding-order row: stage 0, 1, 2, 3."""
  return np.array([p for s in range(4) for p in positions(H, W, s)], np.int64)


def gather(y_hat, pos, taps):
  """The taps at each position as [B, P, tap * M + channel], zero outside the image."""
  y_hat = ar._f32(y_hat)
  B, H, W, M = y_hat.shape
  out = np.zeros((B, len(pos), len(taps), M), np.float32)
  for i, p in enumerate(pos):
    py, px = divmod(int(p), W)
    for t, (dy, dx) in enumerate(taps):
      if 0 <= py + dy < H and 0 <= px + dx < W:
        out[:, i, t] = y_hat[:, py + dy, px + dx]
  return out.reshape(B, len(pos), len(taps) * M)


def unpack(ws, stage):
  """[Wc_s [T_s M, 2M] (None at stage 0), bc_s, W1, b1, W2, b2, W3, b3] as float32 arrays."""
  kernels, biases = ws[0], ws[1]
  rest = [ar._f32(w) for w in ws[2:]]
  if stage == 0:
    return [None, None] + rest
  k = ar._f32(kernels[stage - 1])
  M = k.shape[2]
  wc = np.stack([k[dy + 2, dx + 2] for dy, dx in TAPS[stage]]).reshape(len(TAPS[stage]) * M, 2 * M)
  return [wc, ar._f32(biases[stage - 1])] + rest


def _psi_rows(psi, pos):
  psi = ar._f32(psi)
  B, H, W, C = psi.shape
  return psi.reshape(B, H * W, C)[:, list(pos)].reshape(B * len(pos), C)


def params32(ws, y_hat, psi, stage, num_scales, dense=ar.dense32):
  """(loc, scale_index, index) [B, n_s, M] of one stage, in coding order, bit for bit as tfcb_msc_params gives them."""
  psi = ar._f32(psi)
  B, H, W, C = psi.shape
  M = C // 2
  pos = positions(H, W, stage)
  if not pos:
    empty = np.zeros((B, 0, M), np.float32)
    return empty, empty, empty.astype(np.int32)
  wc, bc, w1, b1, w2, b2, w3, b3 = unpack(ws, stage)
  ps = _psi_rows(psi, pos)
  if stage == 0:
    ctx = np.zeros((B * len(pos), 2 * M), np.float32)
  else:
    ctx = dense(gather(y_hat, pos, TAPS[stage]).reshape(B * len(pos), len(TAPS[stage]) * M), wc, bc, False)
  h = dense(np.concatenate([ps, ctx], -1), w1, b1, True)
  h = dense(h, w2, b2, True)
  out = dense(h, w3, b3, False).reshape(B, len(pos), 2 * M)
  return out[..., :M], out[..., M:], ar.table_index(out[..., M:], num_scales)


def encode32(ws, y, psi, num_scales):
  """The four-pass encoder: (y_hat [B, H, W, M], and y, loc, index, scale_index in coding order [B, H W, M])."""
  y = ar._f32(y)
  B, H, W, M = y.shape
  y_hat = np.zeros_like(y)
  flat_y, flat_hat = y.reshape(B, H * W, M), y_hat.reshape(B, H * W, M)
  parts = []
  for stage in range(4):
    pos = positions(H, W, stage)
    loc, scale, index = params32(ws, y_hat, psi, stage, num_scales)
    q = ar.rint_to_int32(flat_y[:, pos] - loc)
    flat_hat[:, pos] = q.astype(np.float32) + loc
    parts.append((flat_y[:, pos], loc, index, scale))
  return (y_hat,) + tuple(np.concatenate([a[i] for a in parts], 1) for i in range(4))


# ---------------------------------------------------------------------------------------------------------------
# float64: the restatement, ar_oracle's bound and the context feature
# ---------------------------------------------------------------------------------------------------------------
def _layers(ws, y_hat, psi, stage):
  psi = ar._f32(psi)
  B, H, W, C = psi.shape
  M = C // 2
  pos = positions(H, W, stage)
  ws64 = [None if w is None else w.astype(np.float64) for w in unpack(ws, stage)]
  wc, bc, w1, b1, w2, b2, w3, b3 = ws64
  ps = _psi_rows(psi, pos).astype(np.float64)
  if stage == 0:
    ctx, e = np.zeros((len(ps), 2 * M)), np.zeros((len(ps), 2 * M))
  else:
    x = gather(y_hat, pos, TAPS[stage]).reshape(B * len(pos), len(TAPS[stage]) * M).astype(np.float64)
    ctx, e = ar._dense_bound(x, np.zeros_like(x), wc, bc, False)
  h, e = ar._dense_bound(np.concatenate([ps, ctx], -1), np.concatenate([np.zeros_like(ps), e], -1), w1, b1, True)
  h, e = ar._dense_bound(h, e, w2, b2, True)
  out, e = ar._dense_bound(h, e, w3, b3, False)
  out, e = out.reshape(B, len(pos), 2 * M), e.reshape(B, len(pos), 2 * M)
  return (out[..., :M], out[..., M:]), (e[..., :M], e[..., M:])


def params64(ws, y_hat, psi, stage):
  """(loc, scale_index) [B, n_s, M] of one stage in float64."""
  return _layers(ws, y_hat, psi, stage)[0]


def bound64(ws, y_hat, psi, stage):
  """(loc bound, scale_index bound) [B, n_s, M]: ar_oracle's a-priori bound on |params32 - exact| for this stage."""
  return _layers(ws, y_hat, psi, stage)[1]


def context64(ctx_kernels, ctx_biases, y_hat):
  """The context feature [B, H, W, 2M] of every position in float64: 0 at stage 0, bc_s + Wc_s · taps at stage s."""
  y_hat = np.asarray(y_hat, np.float64)
  B, H, W, M = y_hat.shape
  out = np.zeros((B, H, W, 2 * M))
  for r in range(H):
    for c in range(W):
      s = stage_of(r, c)
      if s == 0:
        continue
      k = np.asarray(ctx_kernels[s - 1], np.float64)
      v = np.broadcast_to(np.asarray(ctx_biases[s - 1], np.float64), (B, 2 * M)).copy()
      for dy, dx in TAPS[s]:
        if 0 <= r + dy < H and 0 <= c + dx < W:
          v += y_hat[:, r + dy, c + dx] @ k[dy + 2, dx + 2]
      out[:, r, c] = v
  return out
