"""GPU: the checkerboard context model (CheckerboardModel, functional.cb_*).  Both parameter passes equal the float32
emulation bit for bit, the encoder is the emulated two-pass encoder, rows do not depend on the batch, the strings are
the entropy model's of the coding-order tensors, the two-call decoder returns the encoder's latents without host
synchronisation in a fixed number of launches, and the model's coding calls fit together."""
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
from oracle import checkerboard_oracle as cbo

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
SHAPES = [(1, 1), (1, 2), (2, 1), (1, 9), (7, 1), (5, 7), (6, 8), (32, 48)]


@pytest.fixture(scope="module")
def em():
  scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                            compression=True).to("cuda")


def _weights(M, seed):
  """Random [ctx kernel, ctx bias, W1, b1, W2, b2, W3, b3] with loc of a few units and scale indexes spread over
  the table range (tests/test_mbt2018_gpu.py's scales)."""
  g = torch.Generator().manual_seed(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: torch.randn(*s, generator=g)
  b3 = torch.cat([0.5 * r(M), 24 + 4 * r(M)])
  ws = [r(5, 5, M, 2 * M) / math.sqrt(12 * M), 0.1 * r(2 * M), r(4 * M, n3) / math.sqrt(4 * M), 0.1 * r(n3),
        r(n3, n4) / math.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * M) / math.sqrt(n4), b3]
  return [w.cuda() for w in ws]


def _latents(B, H, W, M, seed):
  g = torch.Generator().manual_seed(1000 + seed)
  y = 3 * torch.randn(B, H, W, M, generator=g)
  big = torch.rand(B, H, W, M, generator=g) < 0.002  # a few escapes
  y[big] *= 40
  psi = torch.randn(B, H, W, 2 * M, generator=g)
  return y.cuda(), psi.cuda()


_PACKED = {}


def _packed(M, seed=0):
  if (M, seed) not in _PACKED:
    _PACKED[(M, seed)] = (F.cb_pack_weights(*_weights(M, seed)), _weights(M, seed))
  return _PACKED[(M, seed)]


def _encode(em, packed, y, psi):
  y_hat, y_cb, loc, index, scale = F.cb_encode(packed, y, psi, NUM_SCALES, scale_index=True)
  strings = F.compress_f32((y.shape[0],), em._lookup_host(), y_cb, loc, em.cdf_offset, index=index)
  return strings, y_hat, y_cb, loc, index, scale


def _decode(em, packed, strings, psi):
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = F.cb_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset)
  return y_hat, gen_ops.entropy_decode_finalize(handle)


def _np(t):
  return t.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------
# 1. both passes are the float32 emulation, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [6, 12, 18, 30, 42, 96, 192, 384])
def test_params_are_the_float32_emulation_bit_for_bit(M):
  packed, ws = _packed(M)
  shapes = [(1, 1), (1, 2), (2, 1), (1, 9), (7, 1), (5, 7), (6, 8), (32, 48)] if M <= 96 else [(1, 9), (5, 7), (7, 1)]
  for H, W in shapes:
    B = 2 if H * W < 100 else 1
    y, psi = _latents(B, H, W, M, M + H)
    y_hat = torch.round(y)
    for anchors in (True, False):
      got = F.cb_params(packed, y_hat, psi, anchors, NUM_SCALES)
      want = cbo.params32(ws, _np(y_hat), _np(psi), anchors, NUM_SCALES)
      for g, w in zip(got, want):
        assert np.array_equal(_np(g).view(np.int32), np.asarray(w).view(np.int32)), (M, H, W, anchors)


def test_tile_remainders_are_the_emulation():
  """B * n positions that are not multiples of the 32-position tile, at every position of the last tile."""
  M = 12
  packed, ws = _packed(M)
  for B, (H, W) in ((3, (3, 5)), (5, (7, 11)), (1, (11, 13))):
    y, psi = _latents(B, H, W, M, 40 + B)
    y_hat = torch.round(y)
    for anchors in (True, False):
      n = cbo.counts(H, W)[0 if anchors else 1]
      assert (B * n) % 32
      got = F.cb_params(packed, y_hat, psi, anchors, NUM_SCALES)
      want = cbo.params32(ws, _np(y_hat), _np(psi), anchors, NUM_SCALES)
      for g, w in zip(got, want):
        assert np.array_equal(_np(g).view(np.int32), np.asarray(w).view(np.int32))


@pytest.mark.parametrize("M", [12, 96])
def test_encoder_is_the_emulated_two_pass_encoder(M):
  packed, ws = _packed(M)
  B, H, W = 2, 6, 7
  y, psi = _latents(B, H, W, M, 21)
  got = F.cb_encode(packed, y, psi, NUM_SCALES, scale_index=True)
  want = cbo.encode32(ws, _np(y), _np(psi), NUM_SCALES)
  for g, w in zip(got, want):
    assert np.array_equal(_np(g).view(np.int32), np.asarray(w).view(np.int32))
  order = cbo.coding_order(H, W)
  assert torch.equal(got[1], y.view(B, H * W, M)[:, order])
  assert torch.equal(got[0].view(B, H * W, M)[:, order], torch.round(got[1] - got[2]) + got[2])


@pytest.mark.parametrize("M", [96, 192])
def test_rows_do_not_depend_on_the_batch(M):
  packed, _ = _packed(M)
  H, W = 5, 7
  y, psi = _latents(8, H, W, M, 5)
  for B in (3, 8):
    batch = F.cb_encode(packed, y[:B], psi[:B], NUM_SCALES, scale_index=True)
    for b in (0, B - 1):
      one = F.cb_encode(packed, y[b:b + 1].clone(), psi[b:b + 1].clone(), NUM_SCALES, scale_index=True)
      for g, w in zip(one, batch):
        assert torch.equal(g[0], w[b])


# ---------------------------------------------------------------------------------------------------------------
# 2. strings and the decoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [96, 192])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_strings_are_the_entropy_models_and_decode_to_the_encoders_latents(em, M, shape):
  B = 3
  y, psi = _latents(B, *shape, M, 7)
  packed, _ = _packed(M)
  strings, y_hat_enc, y_cb, loc, index, scale = _encode(em, packed, y, psi)
  HW = shape[0] * shape[1]
  assert torch.equal(em._flatten_indexes(em._normalize_indexes(scale)), index)
  want = em.compress(y_cb.view(B, HW, 1, M), scale.view(B, HW, 1, M), loc.view(B, HW, 1, M))
  assert strings.tolist() == want.tolist()
  y_hat, ok = _decode(em, packed, strings, psi)
  assert bool(ok.all())
  assert torch.equal(y_hat, y_hat_enc)


def test_escapes_up_to_the_saturated_value_round_trip(em):
  M, B, H, W = 96, 2, 5, 6
  y, psi = _latents(B, H, W, M, 23)
  y[0, 1, 2] = torch.tensor([3e9, -3e9, 2.0**31, -2.0**31, 1e6, -1e6] * (M // 6))  # a non-anchor
  y[0, 1, 3] = torch.tensor([-3e9, 3e9, 5e5, -5e5, 2.0**30, -7.0] * (M // 6))     # an anchor
  y[1] = 0.0
  packed, _ = _packed(M)
  strings, y_hat_enc, y_cb, loc, _, _ = _encode(em, packed, y, psi)
  assert torch.isfinite(y_hat_enc).all()
  y_hat, ok = _decode(em, packed, strings, psi)
  assert bool(ok.all())
  assert torch.equal(y_hat, y_hat_enc)


def test_batch_and_single_image_coding_interoperate(em):
  M, (H, W), B = 96, (5, 7), 8
  y, psi = _latents(B, H, W, M, 3)
  packed, _ = _packed(M)
  strings, y_hat_batch = _encode(em, packed, y, psi)[:2]
  for b, s in enumerate(strings.split()):  # batch encode, one-image decode
    y_hat, ok = _decode(em, packed, s, psi[b:b + 1])
    assert bool(ok.all()) and torch.equal(y_hat[0], y_hat_batch[b])
  singles = [_encode(em, packed, y[b:b + 1], psi[b:b + 1])[0] for b in range(B)]  # one-image encodes, batch decode
  assert [s.tolist()[0] for s in singles] == strings.tolist()
  y_hat, ok = _decode(em, packed, gen_ops.Strings.concat(singles), psi)
  assert bool(ok.all()) and torch.equal(y_hat, y_hat_batch)


@pytest.mark.parametrize("B", [1, 8])
def test_decode_runs_without_host_sync_in_a_fixed_number_of_launches(em, B):
  M = 96
  packed, _ = _packed(M)
  counts = {}
  for shape in ((1, 1), (5, 7), (32, 48)):
    y, psi = _latents(B, *shape, M, 13)
    strings, y_hat_enc = _encode(em, packed, y, psi)[:2]
    handle = gen_ops.create_range_decoder(strings, em._lookup_host())
    coff = em.cdf_offset.cuda()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
      y_hat = F.cb_decode(handle, packed, psi, NUM_SCALES, coff)
    finally:
      torch.cuda.set_sync_debug_mode(0)
    counts[shape] = _lib.launch_count() - n0
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert torch.equal(y_hat, y_hat_enc)
  # anchors: 3 parameter launches, a decode and a scatter; non-anchors: 4, a decode and a scatter.  At 1x1 the
  # non-anchor pass is empty and launches nothing.
  assert counts[(5, 7)] == counts[(32, 48)] == 11
  assert counts[(1, 1)] == 5


def test_damaged_strings_are_reported(em):
  M, B, H, W = 96, 3, 5, 7
  y, psi = _latents(B, H, W, M, 17)
  packed, _ = _packed(M)
  good = _encode(em, packed, y, psi)[0].tolist()
  padded = gen_ops.Strings.from_bytes([good[0] + bytes(range(64)), good[1], good[2]], (B,))
  truncated = gen_ops.Strings.from_bytes([good[0], good[1][:len(good[1]) // 2], good[2]], (B,))
  y_hat, ok = _decode(em, packed, padded, psi)
  assert torch.isfinite(y_hat).all() and ok.tolist() == [False, True, True]
  y_hat, ok = _decode(em, packed, truncated, psi)
  assert torch.isfinite(y_hat).all() and ok.tolist()[0] and ok.tolist()[2]
  m = models.CheckerboardModel(num_filters=24, latent_depth=M)
  m.entropy_model, m._packed, m.num_scales = em, packed, NUM_SCALES
  with pytest.raises(gen_ops.InvalidArgumentError, match="Sanity check failed"):
    m._decode_latents(padded, psi)


def test_bad_arguments_raise_before_any_launch(em):
  M, B, H, W = 96, 2, 3, 4
  y, psi = _latents(B, H, W, M, 19)
  packed, _ = _packed(M)
  strings = _encode(em, packed, y, psi)[0]
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a batch of 1"):
    F.cb_decode(handle, packed, psi[:1], NUM_SCALES, em.cdf_offset)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.cb_params(_packed(192)[0], y, psi, True, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="shape"):
    F.cb_encode(packed, y[:, :2], psi, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="y_hat"):
    F.cb_params(packed, None, psi, False, NUM_SCALES)
  lib = _lib.lib()
  p = lambda t: None if t is None else t.data_ptr()
  n = packed.numel()
  with pytest.raises(_lib.InvalidArgumentError, match="workspace of 4 floats"):
    _lib.check(lib.tfcb_cb_params(p(packed), n, M, p(y), p(psi), B, H, W, 0, NUM_SCALES, p(y), 4, 0, p(y), None,
                                  None, None, None, None, None))
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# 3. the training path
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_model():
  torch.manual_seed(0)
  return models.CheckerboardModel(num_filters=24, latent_depth=24).build("cuda", patch=(64, 64)).fix_tables()


def test_params_kernel_matches_the_training_path(small_model):
  m = small_model
  M = m.latent_depth
  g = torch.Generator().manual_seed(2)
  y_hat = torch.round(3 * torch.randn(2, 5, 6, M, generator=g)).cuda()
  psi = torch.randn(2, 5, 6, 2 * M, generator=g).cuda()
  allow = torch.backends.cudnn.allow_tf32
  torch.backends.cudnn.allow_tf32 = False
  try:
    with torch.no_grad():
      loc_t, scale_t = m.entropy_parameters_of(y_hat, psi)
  finally:
    torch.backends.cudnn.allow_tf32 = allow
  for anchors in (True, False):
    pos = cbo.positions(5, 6, anchors)
    loc, scale, _ = F.cb_params(m._packed, y_hat, psi, anchors, NUM_SCALES)
    for got, want in ((loc, loc_t.view(2, 30, M)[:, pos]), (scale, scale_t.view(2, 30, M)[:, pos])):
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
  grad = m.context_model.kernel.grad.abs().sum((2, 3)).cpu()
  assert torch.equal(grad > 0, models.checkerboard_mask(5) > 0)  # exactly the 12 taps learn
  m.zero_grad()


# ---------------------------------------------------------------------------------------------------------------
# 4. the model
# ---------------------------------------------------------------------------------------------------------------
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
  big = _images([(176, 192)], 2)
  d = m.evaluate_images(big)[0]
  e = m.evaluate(big[0])
  assert d["bpp"] == e["bpp"] and math.isfinite(e["psnr"])
