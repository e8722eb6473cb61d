"""GPU: the checkerboard context model with mixture priors (CheckerboardMixtureModel, functional.cbm_*, DESIGN §3.19).
Both passes' locs and scales equal the float32 emulation bit for bit and the weights lie within expf's bound of it;
the strings are varint(len A) ‖ A ‖ N with A and N MixtureEntropyModel's strings of the coding-order latents under
the kernel's own mixtures; round trips are exact (escapes, saturated and non-finite latents included) whatever the
batch or list; damaged strings raise or decode without a fault; and the model's coding calls fit together."""
import math

import numpy as np
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models
from oracle import ar_oracle as ar
from oracle import cb_mixture_oracle as cmo
from oracle import checkerboard_oracle as cbo

pytestmark = pytest.mark.gpu

M = 12
SHAPES = [(1, 1), (1, 9), (7, 1), (5, 7), (3, 11), (32, 48)]  # (5, 7): 18 and 17 positions, off the 32-position tile


def _weights(M, K, seed):
  """Random [ctx kernel, ctx bias, W1, b1, W2, b2, W3, b3] with logits of a few units, locs of a few units and scales
  from below 0.11 to a few units."""
  g = torch.Generator().manual_seed(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: torch.randn(*s, generator=g)
  b3 = torch.stack([r(M, K), 0.5 * r(M, K), 1.5 + r(M, K)], 1).reshape(-1)
  ws = [r(5, 5, M, 2 * M) / math.sqrt(12 * M), 0.1 * r(2 * M), r(4 * M, n3) / math.sqrt(4 * M), 0.1 * r(n3),
        r(n3, n4) / math.sqrt(n3), 0.1 * r(n4), 2 * r(n4, 3 * K * M) / math.sqrt(n4), b3]
  return [w.cuda() for w in ws]


_PACKED = {}


def _packed(K, seed=0):
  if (K, seed) not in _PACKED:
    ws = _weights(M, K, seed)
    _PACKED[(K, seed)] = (F.cbm_pack_weights(*ws), ws)
  return _PACKED[(K, seed)]


def _latents(B, H, W, seed):
  g = torch.Generator().manual_seed(1000 + seed)
  y = 3 * torch.randn(B, H, W, M, generator=g)
  big = torch.rand(B, H, W, M, generator=g) < 0.01  # escapes: far outside every component's support
  y[big] *= 1000
  psi = torch.randn(B, H, W, 2 * M, generator=g)
  return y.cuda(), psi.cuda()


def _check_params(got, want):
  w, l, s = (t.cpu().numpy() for t in got)
  ww, wl, ws = want
  np.testing.assert_array_equal(l, wl)
  np.testing.assert_array_equal(s, ws)
  tol = (cmo.EXPF_ULP + 1) * cmo.ulp32(ww)  # expf's bound plus the oracle's own rounding of exp
  assert (np.abs(w.astype(np.float64) - ww.astype(np.float64)) <= tol).all()
  assert (w <= 1).all() and (w.max(-1) == 1).all() if w.size else True


@pytest.mark.parametrize("K", [1, 3, 8, 64])
@pytest.mark.parametrize("H,W", SHAPES)
def test_both_passes_match_the_float32_emulation(K, H, W):
  if K == 64 and H * W > 40:
    pytest.skip("K = 64 runs at the smaller shapes (the emulation is numpy)")
  packed, ws = _packed(K)
  y, psi = _latents(2, H, W, K + H)
  y_hat = torch.round(y)
  for anchors in (True, False):
    got = F.cbm_params(packed, K, y_hat, psi, anchors)
    n = cbo.counts(H, W)[0 if anchors else 1]
    assert got[0].shape == (2, n, M, K)
    _check_params(got, cmo.params32(ws, y_hat.cpu().numpy(), psi.cpu().numpy(), anchors, K))


def test_batch_and_ragged_passes_equal_one_image_calls():
  K = 3
  packed, _ = _packed(K)
  shapes = [(5, 7), (1, 1), (32, 48), (2, 3), (1, 9)]
  lat = [_latents(1, h, w, i) for i, (h, w) in enumerate(shapes)]
  y_hats, psis = [torch.round(y[0]) for y, _ in lat], [p[0] for _, p in lat]
  for anchors in (True, False):
    weight, loc, scale, lengths = F.cbm_params_ragged(packed, K, y_hats, psis, anchors)
    at = 0
    for yh, p, n in zip(y_hats, psis, lengths):
      one = F.cbm_params(packed, K, yh[None], p[None], anchors)
      for got, want in zip((weight, loc, scale), one):
        assert torch.equal(got[at:at + n], want.reshape(-1, K))
      at += n
    yb, pb = _latents(3, 5, 7, 9)
    batch = F.cbm_params(packed, K, torch.round(yb), pb, anchors)
    for b in range(3):
      one = F.cbm_params(packed, K, torch.round(yb[b:b + 1]), pb[b:b + 1], anchors)
      assert all(torch.equal(x[b:b + 1], o) for x, o in zip(batch, one))


@pytest.mark.parametrize("family", ["normal", "logistic"])
@pytest.mark.parametrize("K,S", [(1, 1), (3, 1), (8, 1), (3, 4)])
def test_strings_are_the_mixture_entropy_models_strings_of_both_colours(family, K, S):
  packed, _ = _packed(K)
  B, H, W = 2, 6, 7
  y, psi = _latents(B, H, W, 7 * K)
  y_hat, strings = F.cbm_encode(packed, K, y, psi, family=family, substreams=S)
  assert torch.equal(y_hat, torch.round(y))
  em = E.MixtureEntropyModel(family, coding_rank=2)
  order = torch.from_numpy(cbo.coding_order(H, W)).cuda()
  y_cb = y.reshape(B, H * W, M)[:, order]
  na = cbo.counts(H, W)[0]
  params = [F.cbm_params(packed, K, y_hat, psi, anchors) for anchors in (True, False)]
  for b, s in enumerate(strings.tolist()):
    a, n = F.cbm_split(s, b)
    assert s == gen_ops._varint(len(a)) + a + n
    for part, (w, l, sc), ys in ((a, params[0], y_cb[b, :na]), (n, params[1], y_cb[b, na:])):
      want = em.compress(ys[None], w[b:b + 1], l[b:b + 1], sc[b:b + 1], substreams=S).tolist()[0]
      assert part == want


def test_round_trips_are_exact_with_escapes_saturated_and_non_finite_latents():
  K = 3
  packed, ws = _packed(K)
  B, H, W = 2, 9, 8
  y, psi = _latents(B, H, W, 3)
  flat = y.view(-1)
  flat[5], flat[77], flat[200] = 3e9, -3e9, float("nan")  # saturate to int32's ends, NaN -> 0
  flat[301], flat[402] = float("inf"), float("-inf")
  flat[500] = 2.0**30 + 1e3
  y_hat, strings = F.cbm_encode(packed, K, y, psi)
  want = ar.rint_to_int32(y.cpu().numpy()).astype(np.float32)
  np.testing.assert_array_equal(y_hat.cpu().numpy(), want)
  np.testing.assert_array_equal(F.cbm_decode(strings, packed, K, psi).cpu().numpy(), want)
  enc = cmo.encode32(ws, y.cpu().numpy(), psi.cpu().numpy(), K)
  np.testing.assert_array_equal(enc[0], want)


@pytest.mark.parametrize("family", ["normal", "logistic"])
def test_an_images_string_is_the_same_alone_in_a_batch_and_in_a_ragged_list(family):
  K = 3
  packed, _ = _packed(K)
  shapes = [(5, 7), (1, 1), (12, 16), (1, 2), (2, 1)]
  lat = [_latents(1, h, w, 20 + i) for i, (h, w) in enumerate(shapes)]
  alone = [F.cbm_encode(packed, K, y, p, family=family)[1].tolist()[0] for y, p in lat]
  y_hats, strings = F.cbm_encode_ragged(packed, K, [y[0] for y, _ in lat], [p[0] for _, p in lat], family=family)
  assert strings.tolist() == alone
  for yh, (y, _) in zip(y_hats, lat):
    assert torch.equal(yh, torch.round(y[0]))
  dec = F.cbm_decode_ragged(strings, packed, K, [p[0] for _, p in lat], family=family)
  for d, (y, _) in zip(dec, lat):
    assert torch.equal(d, torch.round(y[0]))
  yb, pb = _latents(3, 5, 7, 40)
  batch = F.cbm_encode(packed, K, yb, pb, family=family)[1].tolist()
  assert batch == [F.cbm_encode(packed, K, yb[b:b + 1], pb[b:b + 1], family=family)[1].tolist()[0] for b in range(3)]


@pytest.mark.parametrize("S", [2, 16])
def test_substreams_decode_to_the_same_latents(S):
  K = 3
  packed, _ = _packed(K)
  y, psi = _latents(2, 32, 48, 50)
  y_hat, s1 = F.cbm_encode(packed, K, y, psi)
  _, sS = F.cbm_encode(packed, K, y, psi, substreams=S)
  assert s1.tolist() != sS.tolist()
  assert torch.equal(F.cbm_decode(sS, packed, K, psi, substreams=S), y_hat)
  shapes = [(5, 7), (1, 1), (32, 48)]
  lat = [_latents(1, h, w, 60 + i) for i, (h, w) in enumerate(shapes)]
  _, st = F.cbm_encode_ragged(packed, K, [y[0] for y, _ in lat], [p[0] for _, p in lat], substreams=S)
  for d, (y, _) in zip(F.cbm_decode_ragged(st, packed, K, [p[0] for _, p in lat], substreams=S), lat):
    assert torch.equal(d, torch.round(y[0]))


def test_damaged_strings_raise_or_decode_without_a_fault():
  K = 3
  packed, _ = _packed(K)
  y, psi = _latents(1, 6, 7, 70)
  y_hat, strings = F.cbm_encode(packed, K, y, psi)
  s = strings.tolist()[0]
  a, n = F.cbm_split(s)
  head = len(s) - len(a) - len(n)
  s4 = F.cbm_encode(packed, K, y, psi, substreams=4)[1].tolist()[0]
  n0 = _lib.launch_count()
  for bad, what in (((s[:head + len(a) - 1]), "runs past the end"), (b"", "truncated"), (b"\x80", "truncated"),
                    (b"\x81\x00" + s[head:], "minimal form"), (gen_ops._varint(len(s)) + s[head:], "runs past")):
    with pytest.raises(_lib.InvalidArgumentError, match=what):
      F.cbm_decode([bad], packed, K, psi)
  with pytest.raises(_lib.InvalidArgumentError, match="substream"):
    F.cbm_decode([s4], packed, K, psi, substreams=2)
  with pytest.raises(_lib.InvalidArgumentError, match="substream"):
    F.cbm_decode(strings, packed, K, psi, substreams=4)
  assert _lib.launch_count() == n0  # (the strings are split on the host before any device work)
  rng = np.random.default_rng(1)
  for trial in range(4):  # damage inside a range-coded part: not detectable, decodes to some latents
    b = bytearray(s)
    i = head + int(rng.integers(0, len(a) + len(n)))
    b[i] ^= 1 << int(rng.integers(0, 8))
    try:
      out = F.cbm_decode([bytes(b)], packed, K, psi)
    except _lib.InvalidArgumentError:  # (garbage anchors can give the non-anchors parameters the coder refuses)
      continue
    assert out.shape == y_hat.shape
  out = F.cbm_decode([s[:head + len(a) + len(n) // 2]], packed, K, psi)  # a shorter non-anchor part
  assert torch.equal(out.reshape(-1, M)[cbo.positions(6, 7, True)], y_hat.reshape(-1, M)[cbo.positions(6, 7, True)])


def test_launch_counts_are_fixed_whatever_the_batch_and_shapes():
  K = 3
  packed, _ = _packed(K)
  counts = set()
  for B, H, W in ((1, 5, 7), (3, 32, 48)):
    y, psi = _latents(B, H, W, B)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    y_hat, strings = F.cbm_encode(packed, K, y, psi)
    n1 = _lib.launch_count()
    F.cbm_decode(strings, packed, K, psi)
    n2 = _lib.launch_count()
    lengths = [H * W * M]
    n3 = _lib.launch_count()
    part = F.mixture_encode_ragged(y.reshape(-1)[:H * W * M].contiguous(), *[torch.ones(H * W * M, K).cuda()] * 3,
                                   lengths)
    n4 = _lib.launch_count()
    F.mixture_decode_ragged(part, *[torch.ones(H * W * M, K).cuda()] * 3, lengths)
    n5 = _lib.launch_count()
    # encode: 4 + 5 parameter launches and one mixture encode; decode: per colour a pass, a mixture decode, a scatter
    assert n1 - n0 == 9 + (n4 - n3), (n1 - n0, n4 - n3)
    assert n2 - n1 == 9 + 2 * (n5 - n4) + 2, (n2 - n1, n5 - n4)
    counts.add((n1 - n0, n2 - n1))
  assert counts == {(13, 13)}, counts  # the mixture coder's encode is four launches, its decode one


def test_host_checks_reject_before_any_launch():
  K = 3
  packed, _ = _packed(K)
  y, psi = _latents(1, 4, 4, 80)
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="family"):
    F.cbm_encode(packed, K, y, psi, family="laplace")
  with pytest.raises(_lib.InvalidArgumentError, match="K=4"):
    F.cbm_params(packed, 4, None, psi, True)
  with pytest.raises(_lib.InvalidArgumentError, match="multiple of 6"):
    F.cbm_params(packed, K, None, torch.zeros(1, 4, 4, 16).cuda(), True)
  with pytest.raises(_lib.InvalidArgumentError, match="y_hat"):
    F.cbm_params(packed, K, None, psi, False)
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for 1 images"):
    F.cbm_decode([b"", b""], packed, K, psi)
  lib = _lib.lib()
  nw = int(lib.tfcb_cbm_workspace_floats(M, K, 1, 4, 4, 1))
  work = torch.empty(nw, device="cuda")
  out = torch.empty(8 * M * K, device="cuda")
  p = F._p
  args = lambda **kw: dict(dict(packed=p(packed), pf=packed.numel(), M=M, K=K, yhat=None, psi=p(psi), B=1, H=4, W=4,
                                anchors=1, work=p(work), wf=nw, whole=0, w=p(out), l=p(out), s=p(out), y=None,
                                ycb=None, yho=None, stream=F._stream()), **kw)
  for kw, what in (({"M": 18}, "packed weights hold"), ({"K": 65}, "in \\[1, 64\\]"), ({"M": 10}, "multiple of 6"),
                   ({"packed": None}, "packed"), ({"psi": None}, "psi"), ({"wf": nw - 1}, "workspace"),
                   ({"w": None}, "weight"), ({"y": p(y)}, "encoder needs"), ({"H": 0}, "latent shape"),
                   ({"anchors": 0}, "yhat")):
    a = args(**kw)
    with pytest.raises(_lib.InvalidArgumentError, match=what):
      _lib.check(lib.tfcb_cbm_params(*a.values()))
  assert _lib.launch_count() == n0


# ---- CheckerboardMixtureModel ----
def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  out = []
  for h, w in sizes:
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 60 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None] * np.array([1.0, 0.7, 0.4])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)))
  return out


@pytest.fixture(scope="module", params=["normal", "logistic"])
def model(request):
  torch.manual_seed(0)
  return models.CheckerboardMixtureModel(num_filters=16, latent_depth=12, num_components=3,
                                         family=request.param).build("cuda", patch=(64, 64)).fix_tables()


def test_model_rate_matches_the_strings_and_training_has_gradients(model):
  """The string is within 1 % + 4 bytes of the graph's information content where the coder's bound holds (scales of
  about 0.5 and more, DESIGN §3.18): the last layer's scale outputs are moved to about 2.  At initialisation most
  scales sit at the 0.11 floor, where the 16-bit coder caps a symbol's cost and the graph counts more."""
  m = models.CheckerboardMixtureModel(num_filters=16, latent_depth=12, num_components=3,
                                      family=model.family).build("cuda", patch=(64, 64))
  m.load_state_dict(model.state_dict(), strict=False)
  last = m.entropy_parameters[-1]
  with torch.no_grad():
    last.kernel.mul_(0.1)
    last.bias.view(12, 3, 3)[:, 2, :] = 2.0
  model = m.fix_tables()
  x = _images([(256, 256)], 1)[0]
  item = model.compress(x)
  with torch.no_grad():
    xf = x[None].cuda().float()
    y = model.analysis_transform(xf)
    z_hat = model.side_entropy_model.quantize(model.hyper_analysis_transform(y))
    psi = model.hyper_synthesis_transform(z_hat)[:, :y.shape[1], :y.shape[2], :]
    _, bits = model.entropy_model(y, *model.mixture_parameters(torch.round(y), psi), training=False)
    model(xf, training=False)  # (the evaluation form of forward runs)
  got = 8 * len(item[0].tolist()[0])
  want = float(bits.sum())
  assert abs(got - want) <= 0.01 * want + 32, (got, want)
  model.zero_grad()
  loss, _, _ = model(x[None].cuda().float(), training=True)
  assert torch.isfinite(loss)
  loss.backward()
  missing = [n for n, p in model.named_parameters() if p.requires_grad and (p.grad is None or
                                                                            not torch.isfinite(p.grad).all())]
  assert not missing, missing
  model.zero_grad()


def test_model_round_trip_is_exact_and_the_string_does_not_depend_on_the_batch(model):
  x = _images([(64, 80)], 3)[0]
  item = model.compress(x)
  got = model.decompress(*item)
  with torch.no_grad():
    y = model.analysis_transform(x[None].cuda().float())
    want = torch.clamp(torch.round(model.synthesis_transform(torch.round(y))), 0, 255).to(torch.uint8)[0, :64, :80]
  assert torch.equal(got, want)
  batch = model.compress_batch(torch.stack([x, _images([(64, 80)], 4)[0], x]))
  assert batch[0].tolist()[0] == batch[0].tolist()[2] == item[0].tolist()[0]
  assert torch.equal(model.decompress_batch(*batch)[2], got)


def test_model_compress_images_tfci_and_evaluate(model):
  images = _images([(64, 80), (40, 56), (17, 33)], 5)
  items = model.compress_images(images)
  for x, it in zip(images, items):
    one = model.compress(x)
    assert it[0].tolist() == one[0].tolist() and it[1].tolist() == one[1].tolist()
  outs = model.decompress_images(items)
  for x, out in zip(images, outs):
    assert torch.equal(out, model.decompress(*model.compress(x)))
    assert torch.equal(model.decompress_from_tfci(model.compress_to_tfci(x)), out)
  big = _images([(176, 192), (184, 176)], 8)  # (MS-SSIM's five scales need 176 pixels a side)
  ev = [model.evaluate(x) for x in big]
  evs = model.evaluate_images(big)
  for a, b in zip(ev, evs):
    assert a["bpp"] == b["bpp"] and a["msssim"] == b["msssim"]
    assert math.isfinite(a["psnr"])


def test_model_substreams_decode_to_the_same_image(model):
  x = _images([(64, 80)], 6)[0]
  want = model.decompress(*model.compress(x))
  m4 = models.CheckerboardMixtureModel(num_filters=16, latent_depth=12, num_components=3, family=model.family,
                                       substreams=4).build("cuda", patch=(64, 64))
  m4.load_state_dict(model.state_dict(), strict=False)
  m4.fix_tables()
  assert torch.equal(m4.decompress(*m4.compress(x)), want)
  items = m4.compress_images(_images([(64, 80), (40, 56)], 7))
  assert len(m4.decompress_images(items)) == 2
