"""CPU references of the space-channel multistage context model's group passes (csrc/multistage.cu, tfcb_mscc_*),
composed from multistage_oracle (the 2x2 schedule's stages, positions and taps) and space_channel_oracle (the channel
groups, the channel-context segment and the widths), on top of ar_oracle's float32 emulation.

  - Groups: counts (c_0, ..., c_{K-1}) summing to M; group k is channels [o_k, o_k + c_k).
  - Spatial context of group k at stage s: 0 at stage 0 (bias included); else bc_s + Wc_s · (the group's channels of
    ŷ at the stage's taps, raster order, zero outside the image).
  - Channel context of group k: given by the caller, [B, H, W, 2c_k] (none for k = 0).
  - Layer 1 reads [ψ (2M), channel ctx (2c_k, k >= 1), spatial ctx (2c_k)] of width K1; the widths are
    K1 -> 5 K1 / 6 -> 2 K1 / 3 -> 2c_k (rounded down), shared by the group's four stages.
  - Coding order: per image, group 0's stages 0, 1, 2, 3, then group 1's, ..., each stage in raster order with c_k
    channels per position.
  - params32 / encode32 emulate the kernel bit for bit (stage 0's zero segment computed literally, as
    space_channel_oracle does); params64 / bound64 restate each pass in float64 with ar_oracle's bound; context64 is
    a group's spatial context in float64, the training form's definition.

A group's weights are the list [ctx kernels (three [5, 5, c, 2c], stages 1-3), ctx biases (three [2c]), W1 [K1, N3],
b1, W2 [N3, N4], b2, W3 [N4, 2c], b3]; latents are [B, H, W, M], psi [B, H, W, 2M]; one pass's outputs are [B, n_s, c]
in coding order.
"""
import numpy as np

from oracle import ar_oracle as ar
from oracle import multistage_oracle as mso
from oracle import space_channel_oracle as sco

spans = sco.spans
widths = sco.widths


def coding_order(H, W, groups):
  """For each coding-order element of one image, its flat index p * M + channel into [H * W, M]."""
  M = sum(groups)
  out = []
  for o, c in spans(groups):
    for stage in range(4):
      for p in mso.positions(H, W, stage):
        out.extend(p * M + o + j for j in range(c))
  return np.array(out, np.int64)


def _inputs(group, y_hat, psi, ch_ctx, stage, gather_fn=mso.gather):
  """(taps [N, T_s c] or None, [ψ, channel ctx] rows [N, 2M + CH], (B, P)) of one pass's positions."""
  o, c = group
  psi = ar._f32(psi)
  B, H, W, C2 = psi.shape
  pos = mso.positions(H, W, stage)
  rows = [mso._psi_rows(psi, pos)]
  if o > 0:
    ch = ar._f32(ch_ctx)
    rows.append(ch.reshape(B, H * W, 2 * c)[:, pos].reshape(B * len(pos), 2 * c))
  taps = mso.TAPS[stage]
  x = None if stage == 0 else gather_fn(ar._f32(y_hat)[..., o:o + c], pos, taps).reshape(B * len(pos),
                                                                                         len(taps) * c)
  return x, np.concatenate(rows, -1), (B, len(pos))


def params32(ws, group, y_hat, psi, ch_ctx, stage, num_scales, dense=ar.dense32, gather_fn=mso.gather,
             segments=None):
  """(loc, scale_index, index) [B, n_s, c] of one stage of group (offset, channels), in coding order, bit for bit as
  tfcb_mscc_params gives them.  `segments` reorders layer 1's input segments ("psi", "ch", "ctx"), and `gather_fn`
  replaces the tap gather (it receives the group's channels of y_hat, the positions and the taps): both exist to
  show that a wrong layout changes the bits."""
  o, c = group
  wc, bc, w1, b1, w2, b2, w3, b3 = mso.unpack(ws, stage)
  x, head, (B, P) = _inputs(group, y_hat, psi, ch_ctx, stage, gather_fn)
  if P == 0:  # an empty stage (H = 1 or W = 1)
    empty = np.zeros((B, 0, c), np.float32)
    return empty, empty, empty.astype(np.int32)
  ctx = np.zeros((B * P, 2 * c), np.float32) if stage == 0 else dense(x, wc, bc, False)
  M2 = ar._f32(psi).shape[-1]
  parts = {"psi": head[:, :M2], "ch": head[:, M2:], "ctx": ctx}
  x1 = np.concatenate([parts[s] for s in (segments or ("psi", "ch", "ctx"))], -1)
  h = dense(x1, w1, b1, True)
  h = dense(h, w2, b2, True)
  out = dense(h, w3, b3, False).reshape(B, P, 2 * c)
  return out[..., :c], out[..., c:], ar.table_index(out[..., c:], num_scales)


def encode32(ws_list, groups, y, psi, channel_context, num_scales):
  """The group-by-group, stage-by-stage encoder: (y_hat [B, H, W, M], and y, loc, index, scale_index in coding order
  [B, H W M]).  channel_context(k, y_hat) gives group k's channel context for k >= 1 from the latents decoded so
  far."""
  y = ar._f32(y)
  B, H, W, M = y.shape
  y_hat = np.zeros_like(y)
  flat_y, flat_hat = y.reshape(B, H * W, M), y_hat.reshape(B, H * W, M)
  parts = []
  for k, (ws, (o, c)) in enumerate(zip(ws_list, spans(groups))):
    ch = channel_context(k, y_hat) if k else None
    for stage in range(4):
      pos = mso.positions(H, W, stage)
      loc, scale, index = params32(ws, (o, c), y_hat, psi, ch, stage, num_scales)
      yk = flat_y[:, pos, o:o + c]
      q = ar.rint_to_int32(yk - loc)
      flat_hat[:, pos, o:o + c] = q.astype(np.float32) + loc
      parts.append((yk, loc, index, scale))
  return (y_hat,) + tuple(np.concatenate([a[i].reshape(B, -1) for a in parts], 1) for i in range(4))


# ---------------------------------------------------------------------------------------------------------------
# float64: the restatement and ar_oracle's bound, per pass, and the training form's spatial context
# ---------------------------------------------------------------------------------------------------------------
def _layers64(ws, group, y_hat, psi, ch_ctx, stage):
  o, c = group
  wc, bc, w1, b1, w2, b2, w3, b3 = [None if w is None else w.astype(np.float64) for w in mso.unpack(ws, stage)]
  x, head, (B, P) = _inputs(group, y_hat, psi, ch_ctx, stage)
  head = head.astype(np.float64)
  if stage == 0:
    ctx, e = np.zeros((B * P, 2 * c)), np.zeros((B * P, 2 * c))
  else:
    x = x.astype(np.float64)
    ctx, e = ar._dense_bound(x, np.zeros_like(x), wc, bc, False)
  h, e = ar._dense_bound(np.concatenate([head, ctx], -1), np.concatenate([np.zeros_like(head), e], -1), w1, b1, True)
  h, e = ar._dense_bound(h, e, w2, b2, True)
  out, e = ar._dense_bound(h, e, w3, b3, False)
  out, e = out.reshape(B, P, -1), e.reshape(B, P, -1)
  return (out[..., :c], out[..., c:]), (e[..., :c], e[..., c:])


def params64(ws, group, y_hat, psi, ch_ctx, stage):
  """(loc, scale_index) [B, n_s, c] of one pass in float64."""
  return _layers64(ws, group, y_hat, psi, ch_ctx, stage)[0]


def bound64(ws, group, y_hat, psi, ch_ctx, stage):
  """(loc bound, scale_index bound) [B, n_s, c]: ar_oracle's a-priori bound on |params32 - exact| for this pass."""
  return _layers64(ws, group, y_hat, psi, ch_ctx, stage)[1]


def layer_errors(ws, group, y_hat, psi, ch_ctx, stage, dense=ar.dense32):
  """Each layer of the float32 emulation against float64 on the emulation's own float32 input, as
  ar_oracle.layer_errors: a list of (|fl32 - float64|, bound, |float64|), three layers at stage 0 and four at
  stages 1-3."""
  o, c = group
  wc, bc, w1, b1, w2, b2, w3, b3 = mso.unpack(ws, stage)
  x, head, (B, P) = _inputs(group, y_hat, psi, ch_ctx, stage)
  layers = [(w1, b1, True), (w2, b2, True), (w3, b3, False)]
  if stage == 0:
    x = np.concatenate([head, np.zeros((B * P, 2 * c), np.float32)], -1)
  else:
    layers.insert(0, (wc, bc, False))
  out = []
  for i, (Wt, b, leaky) in enumerate(layers):
    if i == 1 and stage:
      x = np.concatenate([head, x], -1)
    got = dense(x, Wt, b, leaky)
    x64 = x.astype(np.float64)
    want, bound = ar._dense_bound(x64, np.zeros_like(x64), Wt.astype(np.float64), b.astype(np.float64), leaky)
    out.append((np.abs(got.astype(np.float64) - want), bound, np.abs(want)))
    x = got
  return out


def context64(ctx_kernels, ctx_biases, y_hat, group):
  """Group (offset, channels)'s spatial context [B, H, W, 2c] in float64: multistage_oracle's context feature of its
  channels of y_hat."""
  o, c = group
  return mso.context64(ctx_kernels, ctx_biases, np.asarray(y_hat, np.float64)[..., o:o + c])
