"""GPU: the context models over ragged lists of latents (functional.ar_* / cb_* / scc_*_ragged, §3.13).  Each image's
parameters, latents and strings equal the fixed-shape calls on that image alone, bit for bit, whatever shares the
launch; the decoders reproduce the encoders in launch counts that do not depend on the list; and the models' list
calls equal their one-image calls."""
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

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
DEFAULT = (16, 16, 32, 64, 192)
# latent shapes of a mixed list: 1x1 (no non-anchors), thin ones, repeats; 117 + 35 + 16 ... positions, so tiles of
# 32 positions straddle images
MIXED = [(1, 1), (1, 5), (5, 1), (2, 2), (3, 7), (17, 9), (3, 7), (32, 48), (1, 1)]
SMALL = [(1, 5), (3, 7), (1, 1), (5, 1), (2, 2), (3, 7), (7, 3)]


@pytest.fixture(scope="module")
def em():
  scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                            compression=True).to("cuda")


def _net(M, c, k1, g):
  """[ctx kernel, ctx bias, W1, b1, W2, b2, W3, b3] of one network, loc of a few units and scale indexes spread over
  the table."""
  n3, n4 = 5 * k1 // 6, 2 * k1 // 3
  r = lambda *s: torch.randn(*s, generator=g)
  ws = [r(5, 5, c, 2 * c) / math.sqrt(12 * c), 0.1 * r(2 * c), r(k1, n3) / math.sqrt(k1), 0.1 * r(n3),
        r(n3, n4) / math.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * c) / math.sqrt(n4), torch.cat([0.5 * r(c), 24 + 4 * r(c)])]
  return [w.cuda() for w in ws]


_CACHE = {}


def _ar_packed(M, cb):
  key = ("cb" if cb else "ar", M)
  if key not in _CACHE:
    w = _net(M, M, 4 * M, torch.Generator().manual_seed(M))
    _CACHE[key] = (F.cb_pack_weights if cb else F.ar_pack_weights)(*w)
  return _CACHE[key]


def _scc_packed(groups):
  if groups not in _CACHE:
    g = torch.Generator().manual_seed(sum(groups))
    M = sum(groups)
    _CACHE[groups] = [F.scc_pack_weights(M, (o, c), *_net(M, c, 2 * M + (2 * c if o else 0) + 2 * c, g))
                      for o, c in F.scc_spans(groups)]
  return _CACHE[groups]


def _latents(shapes, M, seed, escapes=False):
  g = torch.Generator().manual_seed(1000 + seed)
  ys, psis = [], []
  for H, W in shapes:
    y = 3 * torch.randn(H, W, M, generator=g)
    y[torch.rand(H, W, M, generator=g) < 0.002] *= 40
    ys.append(y.cuda())
    psis.append(torch.randn(H, W, 2 * M, generator=g).cuda())
  if escapes:
    ys[0].view(-1)[:4] = torch.tensor([3e9, -3e9, 2.0**31, -2.0**31], device="cuda")
  return ys, psis


def _ch_fn(groups):
  """A channel context of y_hat[..., :o_k] (repeated and halved), for batches and lists alike."""
  spans = F.scc_spans(groups)

  def one(k, y_hat):
    o, c = spans[k]
    reps = -(-2 * c // o)
    return (y_hat[..., :o].repeat(*([1] * (y_hat.dim() - 1)), reps)[..., :2 * c] * 0.5).contiguous()

  def fn(k, y_hat):
    return [one(k, y) for y in y_hat] if isinstance(y_hat, list) else one(k, y_hat)

  return fn


def _split(flat, lengths):
  return list(torch.split(flat, [int(n) for n in lengths]))


# ---------------------------------------------------------------------------------------------------------------
# 1. parameter passes: each image as the fixed-shape pass on that image alone
# ---------------------------------------------------------------------------------------------------------------
def _check_params(ragged, fixed, shapes, channels):
  loc, scale, index, lengths = ragged
  assert lengths == [n * channels for n in fixed[0]]
  for i, parts in enumerate(zip(_split(loc, lengths), _split(scale, lengths), _split(index, lengths))):
    for got, want in zip(parts, fixed[1][i]):
      assert torch.equal(got, want.reshape(-1)), (i, shapes[i])


@pytest.mark.parametrize("M", [6, 12, 192])
@pytest.mark.parametrize("shapes", [MIXED, [(3, 7)], [(17, 9)] * 3], ids=["mixed", "one", "repeated"])
def test_cb_params_ragged_equal_the_fixed_shape_pass(M, shapes):
  if M == 192 and len(shapes) > 3:
    shapes = [(1, 1), (1, 5), (5, 1), (3, 7), (9, 5)]
  packed = _ar_packed(M, cb=True)
  ys, psis = _latents(shapes, M, M)
  y_hats = [torch.round(y) for y in ys]
  for anchors in (True, False):
    ragged = F.cb_params_ragged(packed, y_hats, psis, anchors, NUM_SCALES)
    fixed = ([F.cb_counts(H, W)[0 if anchors else 1] for H, W in shapes],
             [F.cb_params(packed, yh[None], psi[None], anchors, NUM_SCALES) for yh, psi in zip(y_hats, psis)])
    _check_params(ragged, fixed, shapes, M)


@pytest.mark.parametrize("groups", [(6,), (1, 5), (2, 4, 6, 12), DEFAULT], ids=str)
def test_scc_params_ragged_equal_the_fixed_shape_pass(groups):
  M = sum(groups)
  shapes = MIXED if M < 100 else [(1, 1), (1, 5), (5, 1), (2, 2), (3, 7), (9, 5)]
  packed = _scc_packed(groups)
  ys, psis = _latents(shapes, M, M + 1)
  y_hats = [torch.round(y) for y in ys]
  fn = _ch_fn(groups)
  for k, (p, g) in enumerate(zip(packed, F.scc_spans(groups))):
    chs = fn(k, y_hats) if k else None
    for anchors in (True, False):
      ragged = F.scc_params_ragged(p, g, y_hats, psis, chs, anchors, NUM_SCALES)
      fixed = ([F.cb_counts(H, W)[0 if anchors else 1] for H, W in shapes],
               [F.scc_params(p, g, yh[None], psi[None], chs[i][None] if k else None, anchors, NUM_SCALES)
                for i, (yh, psi) in enumerate(zip(y_hats, psis))])
      _check_params(ragged, fixed, shapes, g[1])


# ---------------------------------------------------------------------------------------------------------------
# 2-3. encoders, strings and decoders
# ---------------------------------------------------------------------------------------------------------------
def _model_calls(kind, M=12, groups=(2, 4, 6)):
  """(encode_ragged, decode_ragged, encode_fixed, decode_fixed) of one context model on random weights."""
  if kind == "ar":
    p = _ar_packed(M, cb=False)
    return (lambda ys, psis: F.ar_encode_ragged(p, ys, psis, NUM_SCALES),
            lambda h, psis, coff: F.ar_decode_ragged(h, p, psis, NUM_SCALES, coff),
            lambda y, psi: (lambda r: (r[0], y, r[1], r[2]))(F.ar_encode(p, y, psi, NUM_SCALES)),
            lambda h, psi, coff: F.ar_decode(h, p, psi, NUM_SCALES, coff))
  if kind == "cb":
    p = _ar_packed(M, cb=True)
    return (lambda ys, psis: F.cb_encode_ragged(p, ys, psis, NUM_SCALES),
            lambda h, psis, coff: F.cb_decode_ragged(h, p, psis, NUM_SCALES, coff),
            lambda y, psi: F.cb_encode(p, y, psi, NUM_SCALES),
            lambda h, psi, coff: F.cb_decode(h, p, psi, NUM_SCALES, coff))
  p, fn = _scc_packed(groups), _ch_fn(groups)
  return (lambda ys, psis: F.scc_encode_ragged(p, groups, ys, psis, fn, NUM_SCALES),
          lambda h, psis, coff: F.scc_decode_ragged(h, p, groups, psis, fn, NUM_SCALES, coff),
          lambda y, psi: F.scc_encode(p, groups, y, psi, fn, NUM_SCALES),
          lambda h, psi, coff: F.scc_decode(h, p, groups, psi, fn, NUM_SCALES, coff))


KINDS = ["ar", "cb", "scc"]


def _ragged_strings(em, enc):
  y_hats, y, loc, index, lengths = enc
  return F.compress_ragged(em._lookup_host(), lengths, y, loc, em.cdf_offset, index=index)


def _decode(em, dec, strings, psis):
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hats = dec(handle, psis, em.cdf_offset)
  return y_hats, gen_ops.entropy_decode_finalize(handle)


@pytest.mark.parametrize("kind", KINDS)
def test_ragged_encoder_and_strings_equal_the_fixed_shape_encoder(em, kind):
  enc_r, _, enc_f, _ = _model_calls(kind)
  ys, psis = _latents(MIXED, 12, 3, escapes=True)
  enc = enc_r(ys, psis)
  strings = _ragged_strings(em, enc).tolist()
  y_hats, y, loc, index, lengths = enc
  assert lengths == [H * W * 12 for H, W in MIXED]
  for i, (yv, psi) in enumerate(zip(ys, psis)):
    yh_f, y_f, loc_f, index_f = enc_f(yv[None].contiguous(), psi[None].contiguous())
    assert torch.equal(y_hats[i], yh_f[0])
    for got, want in ((y, y_f), (loc, loc_f), (index, index_f)):
      assert torch.equal(_split(got, lengths)[i], want.reshape(-1))
    one = F.compress_f32((1,), em._lookup_host(), y_f, loc_f, em.cdf_offset, index=index_f)
    assert strings[i] == one.tolist()[0]


@pytest.mark.parametrize("kind", KINDS)
def test_one_shape_list_equals_the_batch_call(em, kind):
  enc_r, dec_r, enc_f, _ = _model_calls(kind)
  ys, psis = _latents([(5, 7)] * 3, 12, 4)
  enc = enc_r(ys, psis)
  batch = enc_f(torch.stack(ys), torch.stack(psis))
  assert torch.equal(torch.stack(enc[0]), batch[0])
  for got, want in zip(enc[1:4], batch[1:4]):
    assert torch.equal(got, want.reshape(-1))
  batch_strings = F.compress_f32((3,), em._lookup_host(), batch[1], batch[2], em.cdf_offset, index=batch[3])
  assert _ragged_strings(em, enc).tolist() == batch_strings.tolist()


@pytest.mark.parametrize("kind", KINDS)
def test_ragged_decoder_reproduces_the_encoder_and_mixes_with_fixed_strings(em, kind):
  enc_r, dec_r, enc_f, dec_f = _model_calls(kind)
  ys, psis = _latents(MIXED, 12, 5, escapes=True)
  enc = enc_r(ys, psis)
  strings = _ragged_strings(em, enc)
  y_hats, ok = _decode(em, dec_r, strings, psis)
  assert bool(ok.all())
  assert all(torch.equal(a, b) for a, b in zip(y_hats, enc[0]))
  for i, s in enumerate(strings.split()):  # ragged strings decode one image at a time
    h = gen_ops.create_range_decoder(s, em._lookup_host())
    y_hat = dec_f(h, psis[i][None].contiguous(), em.cdf_offset)
    assert bool(gen_ops.entropy_decode_finalize(h).all()) and torch.equal(y_hat[0], enc[0][i])
  singles = []  # fixed-shape strings decode as a list
  for yv, psi in zip(ys, psis):
    yh, y_f, loc_f, index_f = enc_f(yv[None].contiguous(), psi[None].contiguous())
    singles.append(F.compress_f32((1,), em._lookup_host(), y_f, loc_f, em.cdf_offset, index=index_f))
  y_hats, ok = _decode(em, dec_r, gen_ops.Strings.concat(singles), psis)
  assert bool(ok.all()) and all(torch.equal(a, b) for a, b in zip(y_hats, enc[0]))


def test_ar_list_longer_than_the_sm_count(em):
  enc_r, dec_r, _, _ = _model_calls("ar", M=6)
  n = torch.cuda.get_device_properties(0).multi_processor_count + 7
  shapes = [(1 + i % 3, 1 + (i * 5) % 4) for i in range(n)]
  ys, psis = _latents(shapes, 6, 6)
  enc = enc_r(ys, psis)
  y_hats, ok = _decode(em, dec_r, _ragged_strings(em, enc), psis)
  assert bool(ok.all()) and all(torch.equal(a, b) for a, b in zip(y_hats, enc[0]))


@pytest.mark.parametrize("kind", KINDS)
def test_permuting_the_list_permutes_the_outputs(em, kind):
  enc_r, dec_r, _, _ = _model_calls(kind)
  ys, psis = _latents(MIXED, 12, 8)
  perm = [7, 2, 0, 8, 5, 1, 3, 6, 4]
  a = enc_r(ys, psis)
  b = enc_r([ys[i] for i in perm], [psis[i] for i in perm])
  sa, sb = _ragged_strings(em, a).tolist(), _ragged_strings(em, b).tolist()
  for j, i in enumerate(perm):
    assert torch.equal(b[0][j], a[0][i]) and sb[j] == sa[i]
    for got, want in zip(b[1:4], a[1:4]):
      assert torch.equal(_split(got, b[4])[j], _split(want, a[4])[i])
  y_hats, ok = _decode(em, dec_r, _ragged_strings(em, b), [psis[i] for i in perm])
  assert bool(ok.all()) and all(torch.equal(y_hats[j], a[0][i]) for j, i in enumerate(perm))


@pytest.mark.parametrize("kind", KINDS)
def test_decode_is_host_sync_free_and_its_launches_do_not_depend_on_the_list(em, kind):
  enc_r, dec_r, _, _ = _model_calls(kind)
  counts = []
  for shapes in ([(5, 7)], [(5, 7)] * 4, [(1, 5), (3, 7), (17, 9), (2, 2), (32, 48), (5, 1)]):
    ys, psis = _latents(shapes, 12, 9)
    enc = enc_r(ys, psis)
    handle = gen_ops.create_range_decoder(_ragged_strings(em, enc), em._lookup_host())
    coff = em.cdf_offset.cuda()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
      y_hats = dec_r(handle, psis, coff)
    finally:
      torch.cuda.set_sync_debug_mode(0)
    counts.append(_lib.launch_count() - n0)
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert all(torch.equal(a, b) for a, b in zip(y_hats, enc[0]))
  want = {"ar": 1, "cb": 11, "scc": 33}[kind]
  assert counts == [want] * 3


@pytest.mark.parametrize("kind", KINDS)
def test_a_damaged_string_fails_only_its_image(em, kind):
  enc_r, dec_r, _, _ = _model_calls(kind)
  ys, psis = _latents(SMALL, 12, 10)
  strings = _ragged_strings(em, enc_r(ys, psis)).tolist()
  for i, truncate in ((1, False), (5, True)):
    bad = list(strings)
    bad[i] = bad[i][:len(bad[i]) // 2] if truncate else bad[i] + bytes(range(64))
    y_hats, ok = _decode(em, dec_r, gen_ops.Strings.from_bytes(bad, (len(bad),)), psis)
    assert all(bool(torch.isfinite(y).all()) for y in y_hats)
    ok = ok.tolist()
    assert all(ok[j] for j in range(len(bad)) if j != i)
    assert truncate or not ok[i]  # (a truncated string may still end in a state the check accepts)


def test_bad_arguments_raise_before_any_launch(em):
  p, lib = _ar_packed(12, cb=True), _lib.lib()
  ys, psis = _latents([(3, 7), (2, 2)], 12, 11)
  q = _scc_packed((2, 4, 6))
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="non-empty"):
    F.cb_encode_ragged(p, [], [], NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="empty latents"):
    F.ar_encode_ragged(_ar_packed(12, cb=False), [ys[0], ys[1][:0]], [psis[0], psis[1][:0]], NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="y"):
    F.cb_encode_ragged(p, [ys[0], ys[0]], psis, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="psi"):
    F.scc_encode_ragged(q, (2, 4, 6), ys, [psis[0], psis[1][..., :10]], _ch_fn((2, 4, 6)), NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="packed"):
    F.cb_params_ragged(p[:-1], None, psis, True, NUM_SCALES)
  strings = F.compress_ragged(em._lookup_host(), [21 * 12], ys[0].reshape(-1), ys[0].reshape(-1) * 0,
                              em.cdf_offset, index=torch.zeros(21 * 12, dtype=torch.int32, device="cuda"))
  h = gen_ops.create_range_decoder(strings, em._lookup_host())
  par = _ar_packed(12, cb=False)
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="strings"):
    F.cb_decode_ragged(h, p, psis, NUM_SCALES, em.cdf_offset)
  hs, ws = np.array([3, 2], dtype=np.int64), np.array([7, 2], dtype=np.int64)
  hp = lambda a: a.ctypes.data_as(__import__("ctypes").c_void_p)
  psi, y = torch.cat([t.reshape(-1) for t in psis]), torch.cat([t.reshape(-1) for t in ys])
  out = torch.empty_like(y)
  nw = int(lib.tfcb_scc_ragged_workspace_floats(12, 0, 12, 2, hp(hs), hp(ws), 1))
  work = torch.empty(nw, device="cuda")
  args = lambda packed_n, n_img, hs_, work_n: (F._p(p), packed_n, 12, 0, 12, None, F._p(psi), None, n_img, hp(hs_),
                                               hp(ws), 1, NUM_SCALES, F._p(work), work_n, 0, F._p(out), None, None, None,
                                               None, None, None)
  for a, msg in ((args(p.numel(), 2, hs, nw - 1), "workspace"), (args(p.numel() - 1, 2, hs, nw), "packed"),
                 (args(p.numel(), 0, hs, nw), "list"), (args(p.numel(), 2, np.array([3, 0], np.int64), nw), "shape")):
    with pytest.raises(_lib.InvalidArgumentError, match=msg):
      _lib.check(lib.tfcb_scc_params_ragged(*a))
  with pytest.raises(_lib.InvalidArgumentError, match="workspace"):
    _lib.check(lib.tfcb_ar_encode_ragged(F._p(par), par.numel(), 12,
                                         F._p(y), F._p(psi), 2, hp(hs), hp(ws), NUM_SCALES, F._p(work), 7, F._p(out),
                                         F._p(out), F._p(out), None, None))
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# 7. the models' list calls
# ---------------------------------------------------------------------------------------------------------------
def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  out = []
  for h, w in sizes:
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 60 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None] * np.array([1.0, 0.7, 0.4])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)))
  return out


@pytest.mark.parametrize("cls", [models.MBT2018Model, models.CheckerboardModel, models.SpaceChannelModel],
                         ids=lambda c: c.__name__)
def test_model_lists_equal_the_one_image_calls(cls):
  torch.manual_seed(0)
  kw = {"groups": (2, 4, 6)} if cls is models.SpaceChannelModel else {}
  m = cls(num_filters=24, latent_depth=12, **kw).build("cuda", patch=(64, 64)).fix_tables()
  # latents 5x3, 3x5, 1x1, 7x5, 3x3, 2x7: odd and distinct
  imgs = _images([(80, 48), (48, 80), (16, 16), (112, 65), (33, 47), (32, 100)], 1)
  items = m.compress_images(imgs)
  assert len({tuple(int(v) for v in it[3]) for it in items}) == len(imgs)
  outs = m.decompress_images(items)
  for x, item, out in zip(imgs, items, outs):
    one = m.compress(x)
    assert len(one) == len(item)
    for a, b in zip(one, item):
      assert (a.tolist() == b.tolist()) if not isinstance(a, torch.Tensor) else torch.equal(a, b)
    assert torch.equal(m.decompress(*one), out)
  big = _images([(176, 192), (192, 208)], 2)  # (MS-SSIM's five scales need 176 pixels a side)
  for x, d in zip(big, m.evaluate_images(big)):
    e = m.evaluate(x)
    assert d["bpp"] == e["bpp"] and d["msssim"] == e["msssim"]
    assert abs(d["psnr"] - e["psnr"]) <= 1e-4 * abs(e["psnr"])


def test_a_damaged_model_string_fails_the_sanity_check():
  torch.manual_seed(0)
  m = models.CheckerboardModel(num_filters=24, latent_depth=12).build("cuda", patch=(64, 64)).fix_tables()
  items = m.compress_images(_images([(80, 48), (48, 80), (33, 47)], 2))
  s = items[1][0].tolist()[0]
  items[1] = (gen_ops.Strings.from_bytes([s + bytes(range(64))], (1,)),) + tuple(items[1][1:])
  with pytest.raises(_lib.InvalidArgumentError, match="Sanity check failed"):
    m.decompress_images(items)
