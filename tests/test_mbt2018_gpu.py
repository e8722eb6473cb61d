"""GPU: the joint autoregressive + hierarchical prior (MBT2018Model) on the parameter kernel and the device-stepped
encoder / decoder (functional.ar_*): encoder and decoder agree bit for bit, rows do not depend on the batch, the
strings are the standard index-mode stream, the parameter network is accurate, the decode loop never synchronises
with the host, damaged strings are reported, and the model's coding calls fit together."""
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
from oracle import ar_oracle

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
SHAPES = [(1, 1), (1, 9), (7, 1), (5, 7), (32, 48)]


@pytest.fixture(scope="module")
def em():
  scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                            compression=True).to("cuda")


def _weights(M, seed):
  """Random parameters [ctx kernel, ctx bias, W1, b1, W2, b2, W3, b3] with loc of a few units and scale indexes
  spread over the table range."""
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
    _PACKED[(M, seed)] = F.ar_pack_weights(*_weights(M, seed))
  return _PACKED[(M, seed)]


def _encode(em, packed, y, psi):
  y_hat, loc, index, scale = F.ar_encode(packed, y, psi, NUM_SCALES, scale_index=True)
  strings = F.compress_f32((y.shape[0],), em._lookup_host(), y, loc, em.cdf_offset, index=index)
  return strings, y_hat, loc, index, scale


def _decode(em, packed, strings, psi):
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = F.ar_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset)
  ok = gen_ops.entropy_decode_finalize(handle)
  return y_hat, ok


# ---------------------------------------------------------------------------------------------------------------
# 1. encoder = decoder, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [192, 96])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("B", [1, 3, 8])
def test_decoder_reproduces_the_encoders_latents(em, M, shape, B):
  for seed in (0, 1):
    y, psi = _latents(B, *shape, M, seed)
    packed = _packed(M, seed)
    strings, y_hat_enc, loc, _, _ = _encode(em, packed, y, psi)
    y_hat, ok = _decode(em, packed, strings, psi)
    assert bool(ok.all())
    assert torch.equal(y_hat, y_hat_enc)
    # the encoder's reconstruction is round(y - loc) + loc
    assert torch.equal(y_hat_enc, torch.round(y - loc) + loc)


# ---------------------------------------------------------------------------------------------------------------
# 2. batch invariance
# ---------------------------------------------------------------------------------------------------------------
def test_batch_and_single_image_coding_interoperate(em):
  M, (H, W), B = 96, (5, 7), 8
  y, psi = _latents(B, H, W, M, 3)
  packed = _packed(M)
  strings, y_hat_batch, _, _, _ = _encode(em, packed, y, psi)
  for b, s in enumerate(strings.split()):  # batch encode, one-image decode
    y_hat, ok = _decode(em, packed, s, psi[b:b + 1])
    assert bool(ok.all()) and torch.equal(y_hat[0], y_hat_batch[b])
  singles = [_encode(em, packed, y[b:b + 1], psi[b:b + 1]) for b in range(B)]  # one-image encodes, batch decode
  for b, one in enumerate(singles):
    assert one[0].tolist() == [strings.tolist()[b]]
  y_hat, ok = _decode(em, packed, gen_ops.Strings.concat([one[0] for one in singles]), psi)
  assert bool(ok.all()) and torch.equal(y_hat, y_hat_batch)


@pytest.mark.parametrize("M", [192, 96])
def test_params_rows_do_not_depend_on_the_batch(M):
  H, W, B = 4, 6, 8
  y_hat, psi = _latents(B, H, W, M, 5)
  y_hat = torch.round(y_hat)
  packed = _packed(M)
  for p in (0, 7, 23):
    batch = F.ar_params(packed, y_hat, psi, p, NUM_SCALES)
    for b in range(B):
      one = F.ar_params(packed, y_hat[b:b + 1].clone(), psi[b:b + 1].clone(), p, NUM_SCALES)
      for got, want in zip(one, batch):
        assert torch.equal(got[0], want[b]), (p, b)
    # the same row at every position of a batch of copies
    rep = F.ar_params(packed, y_hat[2:3].expand(B, -1, -1, -1).contiguous(), psi[2:3].expand(B, -1, -1, -1).contiguous(),
                      p, NUM_SCALES)
    for t in rep:
      assert all(torch.equal(t[b], t[0]) for b in range(B))


# ---------------------------------------------------------------------------------------------------------------
# 3. the strings are the standard index-mode stream
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [192, 96])
def test_strings_are_the_entropy_models_and_decode_on_the_naive_path(em, M):
  B, H, W = 3, 5, 7
  y, psi = _latents(B, H, W, M, 7)
  packed = _packed(M)
  strings, y_hat_enc, loc, index, scale = _encode(em, packed, y, psi)
  # the device conversion of scale_index is the entropy model's own
  flat = em._flatten_indexes(em._normalize_indexes(scale))
  assert torch.equal(flat, index)
  assert strings.tolist() == em.compress(y, scale, loc).tolist()
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = F.ar_decode_naive(handle, packed, psi, NUM_SCALES, em.cdf_offset)
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  assert torch.equal(y_hat, y_hat_enc)


def test_device_steps_and_naive_steps_mix_on_one_handle(em):
  M, B, H, W = 96, 2, 3, 5
  y, psi = _latents(B, H, W, M, 9)
  packed = _packed(M)
  strings, y_hat_enc, _, _, _ = _encode(em, packed, y, psi)
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = torch.zeros_like(y_hat_enc)
  F.ar_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset, y_hat=y_hat, p_begin=0, p_end=6)
  loc, _, index = F.ar_params(packed, y_hat, psi, 6, NUM_SCALES)
  y_hat.view(B, H * W, M)[:, 6] = F.decode_index_f32(handle, index, loc, em.cdf_offset)
  F.ar_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset, y_hat=y_hat, p_begin=7)
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  assert torch.equal(y_hat, y_hat_enc)


# ---------------------------------------------------------------------------------------------------------------
# 4. parameter network accuracy
# ---------------------------------------------------------------------------------------------------------------
def _reference64(ws, y_hat, psi, p):
  """float64 restatement of the context model and the entropy-parameter layers at position p."""
  ck, cb, w1, b1, w2, b2, w3, b3 = [w.double().cpu() for w in ws]
  B, H, W, M = y_hat.shape
  py, px = divmod(p, W)
  pad = torch.nn.functional.pad(y_hat.double().cpu(), (0, 0, 2, 2, 2, 2))
  patch = pad[:, py:py + 5, px:px + 5, :]  # [B, 5, 5, M] centred on p
  mask = models.causal_mask(5).double()[:, :, None, None]
  ctx = torch.einsum("byxc,yxcd->bd", patch, ck * mask) + cb
  lk = lambda v: torch.where(v > 0, v, 0.01 * v)
  h = lk(torch.cat([psi.double().cpu()[:, py, px], ctx], -1) @ w1 + b1)
  h = lk(h @ w2 + b2)
  out = h @ w3 + b3
  return out[:, :M], out[:, M:]


@pytest.mark.parametrize("M", [192, 96])
def test_params_match_a_float64_restatement(M):
  B, H, W = 2, 6, 9
  y_hat, psi = _latents(B, H, W, M, 11)
  y_hat = torch.round(y_hat)
  ws = _weights(M, 0)
  packed = _packed(M)
  positions = (0, 1, 10, 30, 53)
  bounds = ar_oracle.bound64(ws, y_hat, psi, positions)  # per element: the kernel order's derived error bound
  for i, p in enumerate(positions):
    loc, scale, _ = F.ar_params(packed, y_hat, psi, p, NUM_SCALES)
    rloc, rscale = _reference64(ws, y_hat, psi, p)
    # float32 with fixed-order sums of up to 12M terms: within 2e-5 of the output's scale, and within the bound
    for got, want, bound in ((loc, rloc, bounds[0]), (scale, rscale, bounds[1])):
      err = (got.double().cpu() - want).abs()
      assert err.max().item() <= 2e-5 * (1 + want.abs().max().item()), (p, err.max().item())
      assert bool((err <= torch.from_numpy(bound[:, i])).all()), p


@pytest.fixture(scope="module")
def small_model():
  torch.manual_seed(0)
  return models.MBT2018Model(num_filters=24, latent_depth=24).build("cuda", patch=(64, 64)).fix_tables()


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
  for p in range(30):
    loc, scale, _ = F.ar_params(m._packed, y_hat, psi, p, NUM_SCALES)
    py, px = divmod(p, 6)
    for got, want in ((loc, loc_t[:, py, px]), (scale, scale_t[:, py, px])):
      assert (got - want).abs().max().item() <= 1e-5 * (1 + want.abs().max().item())


def test_training_is_causal_finite_and_reaches_every_parameter(small_model):
  m = small_model
  M = m.latent_depth
  y = torch.randn(1, 4, 5, M, device="cuda")
  psi = torch.randn(1, 4, 5, 2 * M, device="cuda")
  with torch.no_grad():
    loc, scale = m.entropy_parameters_of(y, psi)
    for p in (0, 6, 13):
      y2 = y.clone()
      y2.view(1, 20, M)[:, p:] += 1.0
      loc2, scale2 = m.entropy_parameters_of(y2, psi)
      assert torch.equal(loc2.view(1, 20, M)[:, :p + 1], loc.view(1, 20, M)[:, :p + 1])
      assert torch.equal(scale2.view(1, 20, M)[:, :p + 1], scale.view(1, 20, M)[:, :p + 1])
  m.zero_grad()
  x = torch.randint(0, 256, (2, 64, 64, 3), device="cuda").float()
  loss, bpp, mse = m(x, training=True)
  assert math.isfinite(float(bpp.detach())) and math.isfinite(float(mse.detach()))
  loss.backward()
  for name, prm in m.named_parameters():
    assert prm.grad is not None, name
    assert torch.isfinite(prm.grad).all(), name
  assert m.context_model.kernel.grad.abs().sum() > 0
  m.zero_grad()


# ---------------------------------------------------------------------------------------------------------------
# 5. no host synchronisation in the loop; a fixed launch count
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1), (5, 7), (16, 24)])
def test_decode_loop_runs_without_host_sync_in_one_launch(em, shape):
  M, B = 96, 3
  y, psi = _latents(B, *shape, M, 13)
  packed = _packed(M)
  strings, y_hat_enc, _, _, _ = _encode(em, packed, y, psi)
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  coff = em.cdf_offset.cuda()
  y_hat = torch.zeros_like(y_hat_enc)
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  torch.cuda.set_sync_debug_mode("error")
  try:
    F.ar_decode(handle, packed, psi, NUM_SCALES, coff, y_hat=y_hat)
    F.ar_encode(packed, y, psi, NUM_SCALES, y_hat=torch.zeros_like(y))
  finally:
    torch.cuda.set_sync_debug_mode(0)
  assert _lib.launch_count() - n0 == 2
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  assert torch.equal(y_hat, y_hat_enc)


# ---------------------------------------------------------------------------------------------------------------
# 6. errors
# ---------------------------------------------------------------------------------------------------------------
def test_damaged_strings_decode_to_completion_and_are_reported(em):
  """Damaged strings decode to completion with the verdicts of the existing decoder (whose end-of-stream check
  need not catch every truncation or flipped byte); a string with bytes left over is always reported."""
  M, B, H, W = 96, 3, 5, 7
  y, psi = _latents(B, H, W, M, 17)
  packed = _packed(M)
  strings = _encode(em, packed, y, psi)[0]
  good = strings.tolist()
  truncated = [good[0], good[1][:len(good[1]) // 2], good[2]]
  flipped = [good[0], good[1], good[2][:4] + bytes(b ^ 0x5A for b in good[2][4:12]) + good[2][12:]]
  padded = [good[0] + bytes(range(64)), good[1], good[2]]
  for damaged in (truncated, flipped, padded):
    damaged = gen_ops.Strings.from_bytes(damaged, (B,))
    y_hat, ok = _decode(em, packed, damaged, psi)
    assert torch.isfinite(y_hat).all()
    handle = gen_ops.create_range_decoder(damaged, em._lookup_host())
    y_naive = F.ar_decode_naive(handle, packed, psi, NUM_SCALES, em.cdf_offset)
    assert torch.equal(y_hat, y_naive)
    assert ok.tolist() == gen_ops.entropy_decode_finalize(handle).tolist()
  _, ok = _decode(em, packed, gen_ops.Strings.from_bytes(padded, (B,)), psi)
  assert ok.tolist() == [False, True, True]
  m = models.MBT2018Model(num_filters=24, latent_depth=M)
  m.entropy_model, m._packed, m.num_scales = em, packed, NUM_SCALES
  with pytest.raises(gen_ops.InvalidArgumentError, match="Sanity check failed"):
    m._decode_latents(gen_ops.Strings.from_bytes(padded, (B,)), psi)


def test_bad_arguments_raise_before_any_launch(em):
  M, B, H, W = 96, 2, 3, 4
  y, psi = _latents(B, H, W, M, 19)
  packed = _packed(M)
  strings = _encode(em, packed, y, psi)[0]
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  lib = _lib.lib()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a batch of 1"):
    F.ar_decode(handle, packed, psi[:1], NUM_SCALES, em.cdf_offset)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.ar_decode(handle, _packed(192), psi, NUM_SCALES, em.cdf_offset)
  with pytest.raises(_lib.InvalidArgumentError, match="shape"):
    F.ar_encode(packed, y[:, :2], psi, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="positions"):
    F.ar_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset, p_begin=5, p_end=13)
  n = packed.numel()
  p = lambda t: None if t is None else t.data_ptr()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a batch of 3"):
    _lib.check(lib.tfcb_ar_decode(handle._h, p(packed), n, M, p(psi), 3, H, W, 0, H * W, NUM_SCALES,
                                  p(em.cdf_offset), p(y), None))
  with pytest.raises(_lib.InvalidArgumentError, match="rows for num_scales=65"):
    _lib.check(lib.tfcb_ar_decode(handle._h, p(packed), n, M, p(psi), B, H, W, 0, H * W, 65,
                                  p(em.cdf_offset), p(y), None))
  with pytest.raises(_lib.InvalidArgumentError, match="null"):
    _lib.check(lib.tfcb_ar_decode(handle._h, p(packed), n, M, p(psi), B, H, W, 0, H * W, NUM_SCALES, None, p(y),
                                  None))
  with pytest.raises(_lib.InvalidArgumentError, match="M=90"):
    _lib.check(lib.tfcb_ar_params(p(packed), n, 90, p(y), p(psi), B, H, W, 0, NUM_SCALES, None, None, None, None))
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# 7. integration
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
  string, side, x_shape, y_shape, z_shape = packed
  x_hat = m.decompress(*packed)
  assert x_hat.shape == x.shape and x_hat.dtype == torch.uint8
  # the decoder's latents are the encoder's, and x_hat is their synthesis
  xf = x[None].cuda().float()
  with torch.no_grad():
    y = m.analysis_transform(xf)
    z = m.hyper_analysis_transform(y)
    psi = m._psi(m.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
    _, y_hat_enc, _, _ = m._encode_latents(y, psi)
    y_hat = m._decode_latents(string, psi)
    assert torch.equal(y_hat, y_hat_enc)
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
    for a, b in zip(one[2:], item[2:]):
      assert torch.equal(a, b)
    assert torch.equal(m.decompress(*one), out)
  big = _images([(176, 192), (192, 176)], 2)  # MS-SSIM's five scales need at least 161 pixels a side
  per_image = m.evaluate_images(big)
  for x, d in zip(big, per_image):
    e = m.evaluate(x)
    assert d["bpp"] == e["bpp"] and d["msssim"] == e["msssim"]
    assert abs(d["psnr"] - e["psnr"]) < 1e-3
  assert math.isfinite(models.mean_metrics(per_image)["psnr"])
