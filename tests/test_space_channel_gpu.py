"""GPU: the space-channel context model (SpaceChannelModel, functional.scc_*).  Every group's passes equal the float32
emulation bit for bit, the one-group pass is tfcb_cb_params, the encoder is the emulated group-by-group encoder,
rows do not depend on the batch, the strings are the entropy model's of the coding-order tensors, the decoder
returns the encoder's latents without host synchronisation in a fixed number of launches, and the model's coding
calls fit together."""
import math

import numpy as np
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models
from oracle import space_channel_oracle as sco

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
SHAPES = [(1, 1), (1, 9), (7, 1), (2, 2), (32, 48)]
DEFAULT = (16, 16, 32, 64, 192)


@pytest.fixture(scope="module")
def em():
  scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                            compression=True).to("cuda")


def _weights(groups, seed):
  """Random per-group [ctx kernel, ctx bias, W1, b1, W2, b2, W3, b3] with loc of a few units and scale indexes
  spread over the table range."""
  g = torch.Generator().manual_seed(seed)
  M = sum(groups)
  out = []
  for k, c in enumerate(groups):
    k1, n3, n4 = sco.widths(M, k, c)
    r = lambda *s: torch.randn(*s, generator=g)
    ws = [r(5, 5, c, 2 * c) / math.sqrt(12 * c), 0.1 * r(2 * c), r(k1, n3) / math.sqrt(k1), 0.1 * r(n3),
          r(n3, n4) / math.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * c) / math.sqrt(n4),
          torch.cat([0.5 * r(c), 24 + 4 * r(c)])]
    out.append([w.cuda() for w in ws])
  return out


_PACKED = {}


def _packed(groups, seed=0):
  if (groups, seed) not in _PACKED:
    ws = _weights(groups, seed)
    M = sum(groups)
    _PACKED[(groups, seed)] = ([F.scc_pack_weights(M, s, *w) for s, w in zip(F.scc_spans(groups), ws)], ws)
  return _PACKED[(groups, seed)]


def _latents(B, H, W, M, seed):
  g = torch.Generator().manual_seed(1000 + seed)
  y = 3 * torch.randn(B, H, W, M, generator=g)
  big = torch.rand(B, H, W, M, generator=g) < 0.002  # a few escapes
  y[big] *= 40
  psi = torch.randn(B, H, W, 2 * M, generator=g)
  return y.cuda(), psi.cuda()


def _ch_ctx(groups):
  """A channel context the CPU reproduces exactly: channels of y_hat[..., :o_k] repeated and halved."""
  spans = F.scc_spans(groups)

  def fn(k, y_hat):
    o, c = spans[k]
    reps = -(-2 * c // o)
    if isinstance(y_hat, torch.Tensor):
      return y_hat[..., :o].repeat(1, 1, 1, reps)[..., :2 * c] * 0.5
    return np.tile(y_hat[..., :o], (1, 1, 1, reps))[..., :2 * c] * np.float32(0.5)

  return fn


def _np(t):
  return t.cpu().numpy()


def _bits(a):
  return np.asarray(a).view(np.int32)


def _encode(em, packed, groups, y, psi, ch_fn):
  y_hat, y_cc, loc, index, scale = F.scc_encode(packed, groups, y, psi, ch_fn, NUM_SCALES, scale_index=True)
  strings = F.compress_f32((y.shape[0],), em._lookup_host(), y_cc, loc, em.cdf_offset, index=index)
  return strings, y_hat, y_cc, loc, index, scale


def _decode(em, packed, groups, strings, psi, ch_fn):
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = F.scc_decode(handle, packed, groups, psi, ch_fn, NUM_SCALES, em.cdf_offset)
  return y_hat, gen_ops.entropy_decode_finalize(handle)


# ---------------------------------------------------------------------------------------------------------------
# 1. every group's passes are the float32 emulation, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [(6,), (1, 5), (2, 4, 6, 12), DEFAULT], ids=str)
def test_params_are_the_float32_emulation_bit_for_bit(groups):
  packed, ws = _packed(groups)
  M = sum(groups)
  shapes = SHAPES if M < 100 else [(1, 1), (1, 9), (7, 1), (2, 2), (5, 7)]
  for H, W in shapes:
    B = 3 if H * W < 100 else 1
    y, psi = _latents(B, H, W, M, M + H)
    y_hat = torch.round(y)
    fn = _ch_ctx(groups)
    for k, (p, w, g) in enumerate(zip(packed, ws, F.scc_spans(groups))):
      ch = fn(k, y_hat).contiguous() if k else None
      for anchors in (True, False):
        n = sco.cbo.counts(H, W)[0 if anchors else 1]
        got = F.scc_params(p, g, y_hat, psi, ch, anchors, NUM_SCALES)
        want = sco.params32(w, g, _np(y_hat), _np(psi), None if ch is None else _np(ch), anchors, NUM_SCALES)
        assert got[0].shape == (B, n, g[1])
        for a, b in zip(got, want):
          assert np.array_equal(_bits(_np(a)), _bits(b)), (groups, k, H, W, anchors)


def test_position_counts_off_the_tile_are_the_emulation():
  groups = (2, 4, 6, 12)
  packed, ws = _packed(groups)
  fn = _ch_ctx(groups)
  for B, (H, W) in ((3, (3, 5)), (5, (7, 11))):
    y, psi = _latents(B, H, W, 24, 40 + B)
    y_hat = torch.round(y)
    for k, (p, w, g) in enumerate(zip(packed, ws, F.scc_spans(groups))):
      ch = fn(k, y_hat).contiguous() if k else None
      for anchors in (True, False):
        assert (B * sco.cbo.counts(H, W)[0 if anchors else 1]) % 32
        got = F.scc_params(p, g, y_hat, psi, ch, anchors, NUM_SCALES)
        want = sco.params32(w, g, _np(y_hat), _np(psi), None if ch is None else _np(ch), anchors, NUM_SCALES)
        for a, b in zip(got, want):
          assert np.array_equal(_bits(_np(a)), _bits(b))


@pytest.mark.parametrize("M", [6, 96, 192])
def test_one_group_is_the_checkerboard_pass_bit_for_bit(M):
  (packed,), (ws,) = _packed((M,))
  cb_packed = F.cb_pack_weights(*ws)
  assert torch.equal(packed, cb_packed)
  for H, W in ((1, 1), (5, 7), (32, 48)):
    y, psi = _latents(2, H, W, M, 3 * M + H)
    y_hat = torch.round(y)
    for anchors in (True, False):
      got = F.scc_params(packed, (0, M), y_hat, psi, None, anchors, NUM_SCALES)
      want = F.cb_params(cb_packed, y_hat, psi, anchors, NUM_SCALES)
      for a, b in zip(got, want):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
  y, psi = _latents(2, 6, 7, M, 5)
  got = F.scc_encode([packed], (M,), y, psi, None, NUM_SCALES, scale_index=True)
  want = F.cb_encode(cb_packed, y, psi, NUM_SCALES, scale_index=True)
  for a, b in zip(got, want):
    assert torch.equal(a.reshape(-1).view(torch.int32), b.reshape(-1).view(torch.int32))


@pytest.mark.parametrize("groups", [(1, 5), (2, 4, 6, 12), DEFAULT], ids=str)
def test_encoder_is_the_emulated_encoder(groups):
  packed, ws = _packed(groups)
  M = sum(groups)
  B, H, W = 2, 5, 6
  y, psi = _latents(B, H, W, M, 21)
  fn = _ch_ctx(groups)
  got = F.scc_encode(packed, groups, y, psi, fn, NUM_SCALES, scale_index=True)
  want = sco.encode32(ws, groups, _np(y), _np(psi), fn, NUM_SCALES)
  for a, b in zip(got, want):
    assert np.array_equal(_bits(_np(a)), _bits(b))
  order = torch.from_numpy(sco.coding_order(H, W, groups)).cuda()
  assert torch.equal(got[1], y.reshape(B, -1)[:, order])
  assert torch.equal(got[0].reshape(B, -1)[:, order], torch.round(got[1] - got[2]) + got[2])


def test_rows_do_not_depend_on_the_batch():
  groups = DEFAULT
  packed, _ = _packed(groups)
  fn = _ch_ctx(groups)
  y, psi = _latents(6, 5, 7, 320, 5)
  for B in (3, 6):
    batch = F.scc_encode(packed, groups, y[:B], psi[:B], fn, NUM_SCALES, scale_index=True)
    for b in (0, B - 1):
      one = F.scc_encode(packed, groups, y[b:b + 1].clone(), psi[b:b + 1].clone(), fn, NUM_SCALES, scale_index=True)
      for g, w in zip(one, batch):
        assert torch.equal(g[0], w[b])


# ---------------------------------------------------------------------------------------------------------------
# 2. strings and the decoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [(2, 4, 6, 12), DEFAULT], ids=str)
@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (2, 2), (5, 7)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_strings_are_the_entropy_models_and_decode_to_the_encoders_latents(em, groups, shape):
  B, M = 3, sum(groups)
  y, psi = _latents(B, *shape, M, 7)
  y[0, 0, 0, :4] = torch.tensor([3e9, -3e9, 2.0**31, -2.0**31])  # saturated escapes
  packed, _ = _packed(groups)
  fn = _ch_ctx(groups)
  strings, y_hat_enc, y_cc, loc, index, scale = _encode(em, packed, groups, y, psi, fn)
  n = shape[0] * shape[1] * M
  assert torch.equal(em._flatten_indexes(em._normalize_indexes(scale)), index)
  want = em.compress(y_cc.view(B, n, 1, 1), scale.view(B, n, 1, 1), loc.view(B, n, 1, 1))
  assert strings.tolist() == want.tolist()
  y_hat, ok = _decode(em, packed, groups, strings, psi, fn)
  assert bool(ok.all())
  assert torch.equal(y_hat, y_hat_enc)


def test_batch_and_single_image_coding_interoperate(em):
  groups, (H, W), B = (2, 4, 6, 12), (5, 7), 6
  y, psi = _latents(B, H, W, 24, 3)
  packed, _ = _packed(groups)
  fn = _ch_ctx(groups)
  strings, y_hat_batch = _encode(em, packed, groups, y, psi, fn)[:2]
  for b, s in enumerate(strings.split()):  # batch encode, one-image decode
    y_hat, ok = _decode(em, packed, groups, s, psi[b:b + 1], fn)
    assert bool(ok.all()) and torch.equal(y_hat[0], y_hat_batch[b])
  singles = [_encode(em, packed, groups, y[b:b + 1], psi[b:b + 1], fn)[0] for b in range(B)]
  assert [s.tolist()[0] for s in singles] == strings.tolist()
  y_hat, ok = _decode(em, packed, groups, gen_ops.Strings.concat(singles), psi, fn)
  assert bool(ok.all()) and torch.equal(y_hat, y_hat_batch)


@pytest.mark.parametrize("B", [1, 4])
def test_decode_runs_without_host_sync_in_a_fixed_number_of_launches(em, B):
  groups = (2, 4, 6, 12)
  packed, _ = _packed(groups)
  fn = _ch_ctx(groups)
  counts = {}
  for shape in ((1, 1), (5, 7), (32, 48)):
    y, psi = _latents(B, *shape, 24, 13)
    strings, y_hat_enc = _encode(em, packed, groups, y, psi, fn)[:2]
    handle = gen_ops.create_range_decoder(strings, em._lookup_host())
    coff = em.cdf_offset.cuda()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
      y_hat = F.scc_decode(handle, packed, groups, psi, fn, NUM_SCALES, coff)
    finally:
      torch.cuda.set_sync_debug_mode(0)
    counts[shape] = _lib.launch_count() - n0
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert torch.equal(y_hat, y_hat_enc)
  # per group as the checkerboard decoder: 11 launches, 5 at 1x1 where the non-anchor passes are empty
  assert counts[(5, 7)] == counts[(32, 48)] == 11 * len(groups)
  assert counts[(1, 1)] == 5 * len(groups)


def test_damaged_strings_are_reported(em):
  groups, B, H, W = (2, 4, 6, 12), 3, 5, 7
  y, psi = _latents(B, H, W, 24, 17)
  packed, _ = _packed(groups)
  fn = _ch_ctx(groups)
  good = _encode(em, packed, groups, y, psi, fn)[0].tolist()
  padded = gen_ops.Strings.from_bytes([good[0] + bytes(range(64)), good[1], good[2]], (B,))
  truncated = gen_ops.Strings.from_bytes([good[0], good[1][:len(good[1]) // 2], good[2]], (B,))
  y_hat, ok = _decode(em, packed, groups, padded, psi, fn)
  assert torch.isfinite(y_hat).all() and ok.tolist() == [False, True, True]
  y_hat, ok = _decode(em, packed, groups, truncated, psi, fn)
  assert torch.isfinite(y_hat).all() and ok.tolist()[0] and ok.tolist()[2]


def test_bad_arguments_raise_before_any_launch(em):
  groups, B, H, W = (2, 4, 6, 12), 2, 3, 4
  y, psi = _latents(B, H, W, 24, 19)
  packed, _ = _packed(groups)
  fn = _ch_ctx(groups)
  strings = _encode(em, packed, groups, y, psi, fn)[0]
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  spans = F.scc_spans(groups)
  ch = fn(1, y).contiguous()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a batch of 1"):
    F.scc_decode(handle, packed, groups, psi[:1], fn, NUM_SCALES, em.cdf_offset)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.scc_params(packed[2], spans[1], y, psi, ch, True, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="ch_ctx"):
    F.scc_params(packed[1], spans[1], y, psi, None, True, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="ch_ctx"):
    F.scc_params(packed[1], spans[1], y, psi, ch[..., :3], True, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="no channel context"):
    F.scc_params(packed[0], spans[0], y, psi, ch, True, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="y_hat"):
    F.scc_params(packed[0], spans[0], None, psi, None, False, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="shape"):
    F.scc_encode(packed, groups, y[:, :2], psi, fn, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="groups must sum to M"):
    F.scc_encode(packed[::-1], groups[::-1][:3], y, psi, fn, NUM_SCALES)
  lib = _lib.lib()
  p = lambda t: None if t is None else t.data_ptr()
  o, c = spans[1]
  with pytest.raises(_lib.InvalidArgumentError, match="workspace of 4 floats"):
    _lib.check(lib.tfcb_scc_params(p(packed[1]), packed[1].numel(), 24, o, c, p(y), p(psi), p(ch), B, H, W, 0,
                                   NUM_SCALES, p(y), 4, 0, p(y), None, None, None, None, None, None))
  with pytest.raises(_lib.InvalidArgumentError, match="chctx"):
    _lib.check(lib.tfcb_scc_params(p(packed[1]), packed[1].numel(), 24, o, c, p(y), p(psi), None, B, H, W, 0,
                                   NUM_SCALES, p(y), 1 << 20, 0, p(y), None, None, None, None, None, None))
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# 3. the training path and the model
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_model():
  torch.manual_seed(0)
  return models.SpaceChannelModel(num_filters=24, latent_depth=24, groups=(2, 4, 6, 12)).build(
      "cuda", patch=(64, 64)).fix_tables()


def test_params_kernel_matches_the_training_path(small_model):
  m = small_model
  M = m.latent_depth
  g = torch.Generator().manual_seed(2)
  y_hat = torch.round(3 * torch.randn(2, 5, 6, M, generator=g)).cuda()
  psi = torch.randn(2, 5, 6, 2 * M, generator=g).cuda()
  allow = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
  torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
  try:
    with torch.no_grad():
      loc_t, scale_t = m.entropy_parameters_of(y_hat, psi)
      chs = [m._channel_context(k, y_hat) if k else None for k in range(len(m.groups))]
  finally:
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = allow
  for k, (o, c) in enumerate(m.spans):
    for anchors in (True, False):
      pos = sco.cbo.positions(5, 6, anchors)
      loc, scale, _ = F.scc_params(m._packed[k], (o, c), y_hat, psi, chs[k], anchors, NUM_SCALES)
      for got, want in ((loc, loc_t.view(2, 30, M)[:, pos, o:o + c]), (scale, scale_t.view(2, 30, M)[:, pos, o:o + c])):
        assert (got - want).abs().max().item() <= 1e-5 * (1 + want.abs().max().item())


def test_training_reaches_every_parameter(small_model):
  m = small_model
  m.zero_grad()
  x = torch.randint(0, 256, (2, 64, 64, 3), device="cuda").float()
  loss, bpp, mse = m(x, training=True)
  assert math.isfinite(float(bpp.detach())) and math.isfinite(float(mse.detach()))
  loss.backward()
  for name, prm in m.named_parameters():
    assert prm.grad is not None, name
    assert torch.isfinite(prm.grad).all(), name
  for cm in m.context_models:
    grad = cm.kernel.grad.abs().sum((2, 3)).cpu()
    assert torch.equal(grad > 0, models.checkerboard_mask(5) > 0)  # exactly the 12 taps learn
  m.zero_grad()


def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  out = []
  for h, w in sizes:
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 60 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None] * np.array([1.0, 0.7, 0.4])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)))
  return out


def test_model_round_trip_and_tfci(small_model):
  m = small_model
  x = _images([(64, 80)], 0)[0]
  packed = m.compress(x)
  assert len(packed) == 5
  x_hat = m.decompress(*packed)
  assert x_hat.shape == x.shape and x_hat.dtype == torch.uint8
  with torch.no_grad():
    y = m.analysis_transform(x[None].cuda().float())
    z = m.hyper_analysis_transform(y)
    psi = m._psi(m.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
    _, y_hat_enc, _, _ = m._encode_latents(y, psi)
    assert torch.equal(m._decode_latents(packed[0], psi), y_hat_enc)
    want = models._to_uint8(m.synthesis_transform(y_hat_enc)[:, :64, :80, :])[0]
  assert torch.equal(x_hat, want)
  assert torch.equal(m.decompress_from_tfci(m.compress_to_tfci(x)), x_hat)


def test_images_equal_the_one_image_calls_and_evaluate(small_model):
  m = small_model
  imgs = _images([(64, 80), (48, 64), (64, 80), (33, 47)], 1)
  items = m.compress_images(imgs)
  outs = m.decompress_images(items)
  for x, item, out in zip(imgs, items, outs):
    one = m.compress(x)
    assert one[0].tolist() == item[0].tolist() and one[1].tolist() == item[1].tolist()
    assert torch.equal(m.decompress(*one), out)
  batch = m.compress_batch(torch.stack([imgs[0], imgs[2]]))
  assert batch[0].tolist() == [items[0][0].tolist()[0], items[2][0].tolist()[0]]
  big = _images([(176, 192)], 2)
  d = m.evaluate_images(big)[0]
  e = m.evaluate(big[0])
  assert d["bpp"] == e["bpp"] and math.isfinite(e["psnr"])


def test_default_model_codes_an_image():
  torch.manual_seed(0)
  m = models.SpaceChannelModel(num_filters=32).build("cuda", patch=(64, 64)).fix_tables()
  assert m.latent_depth == 320 and m.groups == DEFAULT
  x = _images([(96, 128)], 3)[0]
  items = m.compress(x)
  assert m.decompress(*items).shape == x.shape
  with torch.no_grad():
    y = m.analysis_transform(x[None].cuda().float())
    psi = m._psi(m.side_entropy_model.quantize(m.hyper_analysis_transform(y)), tuple(y.shape[1:-1]))
    assert torch.equal(m._decode_latents(items[0], psi), m._encode_latents(y, psi)[1])
