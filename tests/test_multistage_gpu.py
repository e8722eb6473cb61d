"""GPU: the multistage context model (MultistageModel, functional.msc_*).  Every stage's parameters equal the float32
emulation bit for bit, the encoder is the emulated four-pass encoder, rows do not depend on the batch or the list,
the strings are the compiled reference coder's encoding of the coding-order symbols, the four-call decoder returns
the encoder's latents without host synchronisation in a fixed number of launches, substreams decode to the same
latents, and the model's coding calls fit together."""
import math

import numpy as np
import pytest
import torch

import oracle
from compression_b200 import _lib
from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models
from oracle import multistage_oracle as mso

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
SHAPES = [(1, 1), (1, 2), (2, 1), (1, 7), (6, 1), (3, 5), (6, 8), (32, 48)]


@pytest.fixture(scope="module")
def em():
  scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                            compression=True).to("cuda")


def _weights(M, seed):
  """Random [ctx kernels, ctx biases, W1, b1, W2, b2, W3, b3] with loc of a few units and scale indexes spread over
  the table range."""
  g = torch.Generator().manual_seed(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: torch.randn(*s, generator=g).cuda()
  b3 = torch.cat([0.5 * r(M), 24 + 4 * r(M)])
  return [[r(5, 5, M, 2 * M) / math.sqrt(12 * M) for _ in range(3)], [0.1 * r(2 * M) for _ in range(3)],
          r(4 * M, n3) / math.sqrt(4 * M), 0.1 * r(n3), r(n3, n4) / math.sqrt(n3), 0.1 * r(n4),
          8 * r(n4, 2 * M) / math.sqrt(n4), b3]


def _np_weights(ws):
  return [[k.cpu().numpy() for k in ws[0]], [b.cpu().numpy() for b in ws[1]]] + [w.cpu().numpy() for w in ws[2:]]


_PACKED = {}


def _packed(M, seed=0):
  if (M, seed) not in _PACKED:
    ws = _weights(M, seed)
    _PACKED[(M, seed)] = (F.msc_pack_weights(*ws), _np_weights(ws))
  return _PACKED[(M, seed)]


def _latents(B, H, W, M, seed):
  g = torch.Generator().manual_seed(1000 + seed)
  y = 3 * torch.randn(B, H, W, M, generator=g)
  big = torch.rand(B, H, W, M, generator=g) < 0.002  # a few escapes
  y[big] *= 40
  psi = torch.randn(B, H, W, 2 * M, generator=g)
  return y.cuda(), psi.cuda()


def _encode(em, packed, y, psi):
  y_hat, y_ms, loc, index, scale = F.msc_encode(packed, y, psi, NUM_SCALES, scale_index=True)
  strings = F.compress_f32((y.shape[0],), em._lookup_host(), y_ms, loc, em.cdf_offset, index=index)
  return strings, y_hat, y_ms, loc, index, scale


def _decode(em, packed, strings, psi, S=1):
  if S > 1:
    strings = gen_ops.split_substreams(strings, S)
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = F.msc_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset, substreams=S)
  return y_hat, gen_ops.entropy_decode_finalize(handle)


def _np(t):
  return t.cpu().numpy()


def _bits(a):
  return np.asarray(a).view(np.int32)


# ---------------------------------------------------------------------------------------------------------------
# 1. every stage is the float32 emulation, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [6, 12, 48, 96, 192])
def test_params_are_the_float32_emulation_bit_for_bit(M):
  packed, ws = _packed(M)
  shapes = SHAPES if M <= 48 else [(1, 7), (3, 5), (6, 1), (9, 11)]
  for H, W in shapes:
    B = 2 if H * W < 100 else 1
    y, psi = _latents(B, H, W, M, M + H)
    y_hat = torch.round(y)
    for s in range(4):
      got = F.msc_params(packed, y_hat, psi, s, NUM_SCALES)
      want = mso.params32(ws, _np(y_hat), _np(psi), s, NUM_SCALES)
      for g, w in zip(got, want):
        assert g.shape == w.shape and np.array_equal(_bits(_np(g)), _bits(w)), (M, H, W, s)


def test_ragged_params_equal_the_one_image_passes():
  M = 12
  packed, ws = _packed(M)
  shapes = [(1, 1), (3, 5), (1, 6), (7, 1), (6, 8), (2, 2)]  # tiles of 32 positions straddle images; empty stages
  lat = [_latents(1, h, w, M, i) for i, (h, w) in enumerate(shapes)]
  y_hats = [torch.round(y[0]) for y, _ in lat]
  psis = [p[0] for _, p in lat]
  for s in range(4):
    loc, scale, index, lengths = F.msc_params_ragged(packed, y_hats, psis, s, NUM_SCALES)
    assert lengths == [F.msc_counts(h, w)[s] * M for h, w in shapes]
    at = 0
    for yh, p, n in zip(y_hats, psis, lengths):
      want = mso.params32(ws, _np(yh[None]), _np(p[None]), s, NUM_SCALES)
      for g, w in zip((loc, scale, index), want):
        assert np.array_equal(_bits(_np(g[at:at + n])), _bits(w.reshape(-1)))
      at += n


@pytest.mark.parametrize("M", [12, 96])
def test_encoder_is_the_emulated_four_pass_encoder(M):
  packed, ws = _packed(M)
  B, H, W = 2, 5, 7
  y, psi = _latents(B, H, W, M, 21)
  got = F.msc_encode(packed, y, psi, NUM_SCALES, scale_index=True)
  want = mso.encode32(ws, _np(y), _np(psi), NUM_SCALES)
  for g, w in zip(got, want):
    assert np.array_equal(_bits(_np(g)), _bits(w))
  order = mso.coding_order(H, W)
  assert torch.equal(got[1], y.view(B, H * W, M)[:, order])
  assert torch.equal(got[0].view(B, H * W, M)[:, order], torch.round(got[1] - got[2]) + got[2])


def test_rows_do_not_depend_on_the_batch():
  M = 96
  packed, _ = _packed(M)
  H, W = 5, 7
  y, psi = _latents(8, H, W, M, 5)
  for B in (3, 8):
    batch = F.msc_encode(packed, y[:B], psi[:B], NUM_SCALES, scale_index=True)
    for b in (0, B - 1):
      one = F.msc_encode(packed, y[b:b + 1].clone(), psi[b:b + 1].clone(), NUM_SCALES, scale_index=True)
      for g, w in zip(one, batch):
        assert torch.equal(g[0], w[b])


# ---------------------------------------------------------------------------------------------------------------
# 2. strings and the decoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_strings_are_the_reference_coders_and_decode_to_the_encoders_latents(em, shape):
  M, B = 96, 3
  y, psi = _latents(B, *shape, M, 7)
  packed, _ = _packed(M)
  strings, y_hat_enc, y_ms, loc, index, scale = _encode(em, packed, y, psi)
  HW = shape[0] * shape[1]
  assert torch.equal(em._flatten_indexes(em._normalize_indexes(scale)), index)
  want = em.compress(y_ms.view(B, HW, 1, M), scale.view(B, HW, 1, M), loc.view(B, HW, 1, M))
  assert strings.tolist() == want.tolist()
  coff = em.cdf_offset
  sym = (torch.round(y_ms - loc).to(torch.int32) - coff[index.long()]).cpu().numpy().reshape(B, -1)
  ref = oracle.best().encode(em._lookup_host(), sym, index.cpu().numpy().reshape(B, -1))
  assert strings.tolist() == ref
  y_hat, ok = _decode(em, packed, strings, psi)
  assert bool(ok.all())
  assert torch.equal(y_hat, y_hat_enc)


def test_batch_and_single_image_coding_interoperate(em):
  M, (H, W), B = 96, (5, 7), 6
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


def test_ragged_coding_equals_the_one_image_calls(em):
  M = 48
  packed, _ = _packed(M)
  shapes = [(5, 7), (1, 1), (2, 9), (8, 1), (6, 6)]
  lat = [_latents(1, h, w, M, 30 + i) for i, (h, w) in enumerate(shapes)]
  ys, psis = [y[0] for y, _ in lat], [p[0] for _, p in lat]
  lookup, coff = em._lookup_host(), em.cdf_offset
  for S in (1, 3):
    y_hats, y_r, loc, index, lengths = F.msc_encode_ragged(packed, ys, psis, NUM_SCALES, substreams=S)
    strings = F.compress_ragged(lookup, lengths, y_r, loc, coff, index=index)
    if S > 1:
      strings = gen_ops.join_substreams(strings, S, (len(shapes),))
    for i, (y, p) in enumerate(zip(ys, psis)):
      one = F.msc_encode(packed, y[None], p[None], NUM_SCALES)
      assert torch.equal(y_hats[i], one[0][0])
      if S == 1:
        assert strings.tolist()[i] == F.compress_f32((1,), lookup, one[1], one[2], coff, index=one[3]).tolist()[0]
    split = gen_ops.split_substreams(strings, S) if S > 1 else strings
    handle = gen_ops.create_range_decoder(split, lookup)
    got = F.msc_decode_ragged(handle, packed, psis, NUM_SCALES, coff, substreams=S)
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    for g, w in zip(got, y_hats):
      assert torch.equal(g, w)


@pytest.mark.parametrize("S", [2, 5, 16])
def test_substreams_decode_to_the_one_stream_latents(em, S):
  M, B, H, W = 48, 2, 6, 7
  packed, _ = _packed(M)
  y, psi = _latents(B, H, W, M, 40 + S)
  strings1, y_hat1 = _encode(em, packed, y, psi)[:2]
  y_hat, y_s, loc, index = F.msc_encode(packed, y, psi, NUM_SCALES, substreams=S)
  assert torch.equal(y_hat, y_hat1)
  lengths = F.msc_substreams([H] * B, [W] * B, M, S)[0]
  parts = F.compress_ragged(em._lookup_host(), lengths, y_s, loc, em.cdf_offset, index=index)
  strings = gen_ops.join_substreams(parts, S, (B,))
  for one, many in zip(strings1.tolist(), strings.tolist()):
    header = len(many) - sum(len(p) for p in gen_ops.parse_substreams(many, S))
    assert len(many) <= len(one) + header + 4 * S
  got, ok = _decode(em, packed, strings, psi, S)
  assert bool(ok.all()) and torch.equal(got, y_hat1)
  handle = gen_ops.create_range_decoder(gen_ops.split_substreams(strings, S), em._lookup_host())
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="substreams"):
    F.msc_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset, substreams=S + 1)
  assert _lib.launch_count() == n0


@pytest.mark.parametrize("B", [1, 8])
def test_decode_runs_without_host_sync_in_a_fixed_number_of_launches(em, B):
  M = 96
  packed, _ = _packed(M)
  counts = {}
  for shape in ((1, 1), (1, 7), (5, 7), (32, 48)):
    y, psi = _latents(B, *shape, M, 13)
    strings, y_hat_enc = _encode(em, packed, y, psi)[:2]
    handle = gen_ops.create_range_decoder(strings, em._lookup_host())
    coff = em.cdf_offset.cuda()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
      y_hat = F.msc_decode(handle, packed, psi, NUM_SCALES, coff)
    finally:
      torch.cuda.set_sync_debug_mode(0)
    counts[shape] = _lib.launch_count() - n0
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert torch.equal(y_hat, y_hat_enc)
  # stage 0: 3 parameter launches, a decode and a scatter; stages 1-3: 4, a decode and a scatter.  An empty stage
  # launches nothing: at 1x1 stages 1-3 are empty, at 1x7 stages 1 and 3.
  assert counts[(5, 7)] == counts[(32, 48)] == 5 + 3 * 6
  assert counts[(1, 1)] == 5
  assert counts[(1, 7)] == 5 + 6


def test_encoder_launches_per_pass():
  M = 12
  packed, _ = _packed(M)
  y, psi = _latents(2, 5, 7, M, 2)
  n0 = _lib.launch_count()
  F.msc_encode(packed, y, psi, NUM_SCALES)
  assert _lib.launch_count() - n0 == 3 + 3 * 4


def test_bad_arguments_raise_before_any_launch(em):
  M, B, H, W = 96, 2, 3, 4
  y, psi = _latents(B, H, W, M, 19)
  packed, _ = _packed(M)
  strings = _encode(em, packed, y, psi)[0]
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  lib = _lib.lib()
  p = lambda t: None if t is None else t.data_ptr()
  n = packed.numel()
  work = torch.empty(1 << 16, dtype=torch.float32, device="cuda")
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a batch of 1"):
    F.msc_decode(handle, packed, psi[:1], NUM_SCALES, em.cdf_offset)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.msc_params(_packed(12)[0], y, psi, 0, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="shape"):
    F.msc_encode(packed, y[:, :2], psi, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="y_hat"):
    F.msc_params(packed, None, psi, 2, NUM_SCALES)
  for stage in (1, 2, 3):
    with pytest.raises(_lib.InvalidArgumentError, match="workspace of 4 floats"):
      _lib.check(lib.tfcb_msc_params(p(packed), n, M, p(y), p(psi), B, H, W, stage, NUM_SCALES, p(y), 4, 0, p(y),
                                     None, None, None, None, None, None))
    with pytest.raises(_lib.InvalidArgumentError, match="the encoder needs"):
      _lib.check(lib.tfcb_msc_params(p(packed), n, M, p(y), p(psi), B, H, W, stage, NUM_SCALES, p(work),
                                     work.numel(), 1, p(y), None, None, p(y), None, None, None))
  hs, ws = np.array([3, 2], np.int64), np.array([4, 2], np.int64)
  with pytest.raises(_lib.InvalidArgumentError, match="aligned"):
    _lib.check(lib.tfcb_msc_params_ragged(p(packed), n, M, p(y), p(psi), 2, hs.ctypes.data, ws.ctypes.data, 1,
                                          NUM_SCALES, p(work) + 4, work.numel() - 1, 0, None, None, None, None, None,
                                          None, None))
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# 3. the training path and the model
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_model():
  torch.manual_seed(0)
  return models.MultistageModel(num_filters=24, latent_depth=24).build("cuda", patch=(64, 64)).fix_tables()


def test_training_form_agrees_with_the_coding_kernels(small_model):
  m = small_model
  M, H, W = m.latent_depth, 5, 6
  g = torch.Generator().manual_seed(2)
  y_hat = torch.round(3 * torch.randn(2, H, W, M, generator=g)).cuda()
  psi = torch.randn(2, H, W, 2 * M, generator=g).cuda()
  allow = torch.backends.cudnn.allow_tf32
  torch.backends.cudnn.allow_tf32 = False
  try:
    with torch.no_grad():
      loc_t, scale_t = m.entropy_parameters_of(y_hat, psi)
  finally:
    torch.backends.cudnn.allow_tf32 = allow
  ws = [[_np(cm.kernel.detach()) for cm in m.context_models], [_np(cm.bias.detach()) for cm in m.context_models]]
  ws += [_np(t.detach()) for t in models._dense_weights(m.entropy_parameters)]
  for s in range(4):
    pos = mso.positions(H, W, s)
    loc, scale, _ = F.msc_params(m._packed, y_hat, psi, s, NUM_SCALES)
    lb, sb = mso.bound64(ws, _np(y_hat), _np(psi), s)
    # both sides are float32 evaluations of the same sums, each within the oracle's bound of the exact value
    for got, want, bound in ((loc, loc_t.view(2, H * W, M)[:, pos], lb), (scale, scale_t.view(2, H * W, M)[:, pos], sb)):
      assert np.all(np.abs(_np(got).astype(np.float64) - _np(want)) <= 2 * bound)


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
  for s, cm in enumerate(m.context_models, 1):  # exactly the stage's taps learn
    grad = cm.kernel.grad.abs().sum((2, 3)).cpu()
    assert torch.equal(grad > 0, models.multistage_mask(s) > 0)
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
  imgs = _images([(64, 80), (48, 64), (16, 16), (33, 47)], 1)
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


def test_model_substreams_decode_the_one_stream_images(small_model):
  m = small_model
  x = _images([(64, 80)], 3)[0]
  want = m.decompress(*m.compress(x))
  m4 = models.MultistageModel(num_filters=24, latent_depth=24, substreams=4).build("cuda", patch=(64, 64))
  keys = m4.state_dict().keys()  # (the weights: m also holds its coding tables)
  m4.load_state_dict({k: v for k, v in m.state_dict().items() if k in keys})
  m4.fix_tables()
  assert torch.equal(m4.decompress(*m4.compress(x)), want)
  items = m4.compress_images(_images([(64, 80), (40, 56)], 4))
  assert len(m4.decompress_images(items)) == 2
