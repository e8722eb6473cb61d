"""GPU: substreams (DESIGN §3.14).  Every substream is the compiled reference coder's encoding of its segment, the
gather is the NumPy permutation of the split, the five models decode the latents of S = 1 bit for bit at any S, the
strings stay within the rate bound, the context-model decoders make the launches of S = 1 without host
synchronisation, and damage is confined to the image it hits."""
import numpy as np
import pytest
import torch

import oracle
import util
from compression_b200 import _lib
from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models
from test_substreams_cpu import _split_np

pytestmark = pytest.mark.gpu
NUM_SCALES = 64


def _split_bytes(strings, S):
  return gen_ops.split_substreams(strings, S).tolist()


def _header_len(string, S):
  return len(string) - sum(len(p) for p in gen_ops.parse_substreams(string, S))


# ---------------------------------------------------------------------------------------------------------------
# bytes: each substream is the reference coder's string of its segment
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["channel", "index"])
@pytest.mark.parametrize("S", [2, 7, 64])
def test_substreams_are_the_reference_encoding_of_their_segments(mode, S):
  rng = np.random.default_rng(S)
  O = oracle.best()
  rows = 5
  cdfs = [util.laplace_cdf(33, 12, 0.5 + 0.4 * c) for c in range(rows)]
  lookup = util.make_lookup_1d(cdfs, [12] * rows, [True] * rows)
  units = [(3, rows), (41, rows), (1000, rows)] if mode == "channel" else [(3, 4), (41, 3), (1000, 7)]
  pos = [[n] for n, _ in units]
  wid = [[c] for _, c in units]
  n_sym = sum(n * c for n, c in units)
  value = rng.integers(-3, 30, n_sym).astype(np.int32)
  value[rng.random(n_sym) < 0.02] = -7  # escapes
  index = None if mode == "channel" else rng.integers(0, rows, n_sym).astype(np.int32)
  lengths, _ = F.substream_layout(pos, wid, S)
  _, _, perm = _split_np(pos, wid, S)  # single-phase: substream order is coding order
  assert np.array_equal(perm, np.arange(n_sym))
  got = F.compress_ragged(lookup, lengths, torch.from_numpy(value).cuda(),
                          index=None if index is None else torch.from_numpy(index).cuda()).tolist()
  offs = np.concatenate([[0], np.cumsum(lengths)])
  for k, s in enumerate(got):
    seg = slice(offs[k], offs[k + 1])
    want = O.encode(lookup, value[seg][None], None if index is None else index[seg][None])[0]
    assert s == want, k


@pytest.mark.parametrize("groups", [(12,), (2, 4, 6)])
def test_gathered_context_order_is_encoded_as_the_reference_does(groups):
  O = oracle.best()
  M = sum(groups)
  em = _em()
  y, psi = _latents(2, 3, 5, M, 1)
  packed = _pack(groups, M)
  S = 7
  out = _encode(groups, packed, y, psi, S)
  y_g, loc, index = (t.reshape(-1) for t in out[1:4])
  coff = em.cdf_offset
  sym = (torch.round(y_g - loc).to(torch.int32) - coff[index.long()]).cpu().numpy()
  idx = index.cpu().numpy()
  lengths = F.context_substreams(groups, [3, 3], [5, 5], S)[0]
  got = F.compress_ragged(em._lookup_host(), lengths, y_g, loc, coff, index=index).tolist()
  offs = np.concatenate([[0], np.cumsum(lengths)])
  for k, s in enumerate(got):
    seg = slice(offs[k], offs[k + 1])
    assert s == O.encode(em._lookup_host(), sym[seg][None], idx[seg][None])[0], k


# ---------------------------------------------------------------------------------------------------------------
# the gather
# ---------------------------------------------------------------------------------------------------------------
_EM = {}


def _em():
  if "em" not in _EM:
    scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
    _EM["em"] = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                                   compression=True).to("cuda")
  return _EM["em"]


def _latents(B, H, W, M, seed):
  g = torch.Generator().manual_seed(seed)
  return (3 * torch.randn(B, H, W, M, generator=g)).cuda(), torch.randn(B, H, W, 2 * M, generator=g).cuda()


def _pack(groups, M):
  torch.manual_seed(sum(groups))
  m = models.SpaceChannelModel(num_filters=8, latent_depth=M, groups=groups)
  m.build("cuda", patch=(16, 16))
  return m._pack()


def _encode(groups, packed, y, psi, S, scale_index=False):
  M = sum(groups)
  if len(groups) == 1:
    return F.cb_encode(packed[0], y, psi, NUM_SCALES, scale_index=scale_index, substreams=S)
  ctx = lambda k, y_hat: torch.zeros(y_hat.shape[:3] + (2 * groups[k],), device=y_hat.device)
  return F.scc_encode(packed, groups, y, psi, ctx, NUM_SCALES, scale_index=scale_index, substreams=S)


@pytest.mark.parametrize("groups", [(12,), (2, 4, 6), (16, 16, 32, 64, 192)])
@pytest.mark.parametrize("S", [2, 7, 64])
def test_gather_is_the_numpy_permutation(groups, S):
  M = sum(groups)
  packed = _pack(groups, M)
  B, H, W = 2, 5, 7  # 35 positions: no phase is a multiple of S
  y, psi = _latents(B, H, W, M, S)
  whole = _encode(groups, packed, y, psi, 1, scale_index=True)
  sub = _encode(groups, packed, y, psi, S, scale_index=True)
  assert torch.equal(whole[0], sub[0])
  _, _, perm = _split_np(*F.context_phases(groups, [H] * B, [W] * B), S)
  perm = torch.from_numpy(perm).cuda()
  for w, s in zip(whole[1:], sub[1:]):
    assert s.shape == w.shape and torch.equal(s.reshape(-1), w.reshape(-1)[perm])


@pytest.mark.parametrize("groups", [(12,), (2, 4, 6)])
def test_ragged_gather_is_the_numpy_permutation(groups):
  M = sum(groups)
  packed = _pack(groups, M)
  shapes = [(1, 1), (2, 3), (5, 7), (1, 9)]
  lat = [_latents(1, h, w, M, 3 + h) for h, w in shapes]
  ys, psis = [y[0] for y, _ in lat], [p[0] for _, p in lat]
  ctx = lambda k, y_hats: [torch.zeros(t.shape[:2] + (2 * groups[k],), device=t.device) for t in y_hats]
  for S in (1, 7):
    if len(groups) == 1:
      out = F.cb_encode_ragged(packed[0], ys, psis, NUM_SCALES, substreams=S)
    else:
      out = F.scc_encode_ragged(packed, groups, ys, psis, ctx, NUM_SCALES, substreams=S)
    if S == 1:
      whole = out
      continue
    pos, wid = F.context_phases(groups, [h for h, _ in shapes], [w for _, w in shapes])
    lengths, _, perm = _split_np(pos, wid, S)
    assert out[4] == lengths.tolist()
    perm = torch.from_numpy(perm).cuda()
    for w, s in zip(whole[1:4], out[1:4]):
      assert torch.equal(s, w[perm])


# ---------------------------------------------------------------------------------------------------------------
# the five models
# ---------------------------------------------------------------------------------------------------------------
def _model(name, S):
  torch.manual_seed(5)
  m = {"bls2017": lambda: models.BLS2017Model(num_filters=16, substreams=S),
       "bmshj2018": lambda: models.BMSHJ2018Model(num_filters=16, substreams=S),
       "ms2020": lambda: models.MS2020Model(num_filters=16, latent_depth=20, hyperprior_depth=8, num_slices=2,
                                            substreams=S),
       "checkerboard": lambda: models.CheckerboardModel(num_filters=16, latent_depth=12, substreams=S),
       "space_channel": lambda: models.SpaceChannelModel(num_filters=16, latent_depth=12, groups=(2, 4, 6),
                                                         substreams=S)}[name]()
  return m.build("cuda").fix_tables()


def _images(name=None):
  g = torch.Generator().manual_seed(9)
  # latents 1x1, 2x3 and 6x8 (the analysis transforms downsample by 16); MS2020 crops its slice transforms' support
  # only where y's sides are multiples of 4 (its hyper transforms downsample y by 4), so it takes 4x4, 4x8 and 8x12
  shapes = ((64, 64), (64, 128), (128, 192)) if name == "ms2020" else ((16, 16), (32, 48), (90, 128))
  return [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in shapes]


def _strings_of(item):
  return [s for s in item if isinstance(s, gen_ops.Strings)]


def _decode_capturing(model, fn):
  """fn()'s images, and the latents the synthesis transform received."""
  got = []
  hook = model.synthesis_transform.register_forward_pre_hook(lambda _, args: got.append(args[0].clone()))
  try:
    return fn(), got
  finally:
    hook.remove()


MODELS = ["bls2017", "bmshj2018", "ms2020", "checkerboard", "space_channel"]


@pytest.mark.parametrize("name", MODELS)
def test_models_decode_the_s1_latents_at_any_substream_count(name):
  imgs = _images(name)
  base = _model(name, 1)
  want = {}
  for mode in ("one", "batch", "list"):
    want[mode] = _run(base, mode, imgs)
  for S in (2, 7, 64):
    m = _model(name, S)
    for mode in ("one", "batch", "list"):
      (x_hat, y_hat, items), (x1, y1, items1) = _run(m, mode, imgs), want[mode]
      assert len(y_hat) == len(y1)
      for a, b in zip(y_hat, y1):
        assert torch.equal(a, b), (name, S, mode)
      for a, b in zip(x_hat, x1):
        assert (a.int() - b.int()).abs().max() <= 1
      for it, it1 in zip(items, items1):  # the rate bound, string by string
        assert len(it) == len(it1)
        for s, s1 in zip(_strings_of(it), _strings_of(it1)):
          for b, b1 in zip(s.tolist(), s1.tolist()):
            assert len(b) <= len(b1) + _header_len(b, S) + 4 * S


def _run(m, mode, imgs):
  if mode == "one":
    items = [m.compress(x) for x in imgs]
    x_hat, y_hat = _decode_capturing(m, lambda: [m.decompress(*it) for it in items])
  elif mode == "batch":
    x = torch.stack([imgs[1], imgs[1].flip(0)])
    items = [m.compress_batch(x)]
    x_hat, y_hat = _decode_capturing(m, lambda: list(m.decompress_batch(*items[0])))
  else:
    items = m.compress_images(imgs)
    x_hat, y_hat = _decode_capturing(m, lambda: m.decompress_images(items))
  return x_hat, y_hat, items


def test_tfci_round_trip_and_wrong_substream_count():
  x = torch.randint(0, 256, (192, 176, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
  m = _model("space_channel", 7)
  tfci = m.compress_to_tfci(x)
  assert m.decompress_from_tfci(tfci).shape == x.shape
  m1 = _model("space_channel", 1)
  assert torch.equal(m.decompress_from_tfci(tfci), m1.decompress_from_tfci(m1.compress_to_tfci(x)))
  other = _model("space_channel", 8)
  with pytest.raises(ValueError, match="string 0: written with 7 substreams, decoding expects 8"):
    other.decompress_from_tfci(tfci)
  m.evaluate(x)


@pytest.mark.parametrize("dtype", [torch.bfloat16])
def test_16bit_bottlenecks_decode_to_the_s1_values(dtype):
  g = torch.Generator().manual_seed(2)
  prior = D.NoisyLogistic(loc=torch.zeros(6), scale=torch.linspace(0.5, 4, 6))
  em = E.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=True, bottleneck_dtype=dtype).to("cuda")
  y = (6 * torch.randn(3, 50, 6, generator=g)).to("cuda", dtype)
  want = em.decompress(em.compress(y), (50,))
  for S in (2, 64):
    s = em.compress(y, substreams=S)
    assert torch.equal(em.decompress(s, (50,), substreams=S), want)
    items = em.compress_ragged([y[0], y[1, :3]], substreams=S)
    got = em.decompress_ragged(items, [(50,), (3,)], substreams=S)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1, :3])
  scale_fn = models.BMSHJ2018Model(num_filters=8).scale_fn
  ls16 = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3, compression=True,
                                            bottleneck_dtype=dtype).to("cuda")
  yb = (4 * torch.randn(2, 3, 5, 4, generator=g)).to("cuda", dtype)
  idx = torch.randint(0, NUM_SCALES, (2, 3, 5, 4), generator=g).float().cuda()
  loc = torch.randn(2, 3, 5, 4, generator=g).to("cuda", dtype)
  want = ls16.decompress(ls16.compress(yb, idx, loc), idx, loc)
  assert torch.equal(ls16.decompress(ls16.compress(yb, idx, loc, substreams=7), idx, loc, substreams=7), want)
  with pytest.raises(ValueError, match="fused=False"):
    ls16.compress(yb, idx, loc, fused=False, substreams=2)


def test_empty_substreams_decode_and_finalize_ok():
  em = _em()
  y = torch.full((1, 1, 1, 3), 2.5, device="cuda")
  idx = torch.full((1, 1, 1, 3), 10.0, device="cuda")
  s = em.compress(y, idx, substreams=16)
  parts = _split_bytes(s, 16)
  assert sum(len(p) == 0 for p in parts) == 15
  assert torch.equal(em.decompress(s, idx, substreams=16), em.decompress(em.compress(y, idx), idx))


# ---------------------------------------------------------------------------------------------------------------
# launches and synchronisation
# ---------------------------------------------------------------------------------------------------------------
def _launches(fn, sync_free=True):
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  if sync_free:
    torch.cuda.set_sync_debug_mode("error")
  try:
    out = fn()
  finally:
    torch.cuda.set_sync_debug_mode(0)
  return _lib.launch_count() - n0, out


@pytest.mark.parametrize("groups", [(12,), (2, 4, 6)])
def test_context_decoders_make_the_launches_of_s1_without_sync(groups):
  M = sum(groups)
  em = _em()
  packed = _pack(groups, M)
  B, H, W = 2, 5, 7
  y, psi = _latents(B, H, W, M, 4)
  ctx = lambda k, y_hat: torch.zeros(y_hat.shape[:3] + (2 * groups[k],), device=y_hat.device)
  counts, y_hats, enc = {}, {}, {}
  def encode(S):
    y_hat, y_g, loc, index = _encode(groups, packed, y, psi, S)
    if S == 1:
      return y_hat, F.compress_f32((B,), em._lookup_host(), y_g, loc, em.cdf_offset, index=index)
    lengths = F.context_substreams(groups, [H] * B, [W] * B, S)[0]
    return y_hat, F.compress_ragged(em._lookup_host(), lengths, y_g, loc, em.cdf_offset, index=index)

  for S in (1, 7):
    enc[S], (y_hat_enc, parts) = _launches(lambda: encode(S), sync_free=False)
    handle = gen_ops.create_range_decoder(parts, em._lookup_host())
    if len(groups) == 1:
      dec = lambda: F.cb_decode(handle, packed[0], psi, NUM_SCALES, em.cdf_offset, substreams=S)
    else:
      dec = lambda: F.scc_decode(handle, packed, groups, psi, ctx, NUM_SCALES, em.cdf_offset, substreams=S)
    counts[S], y_hats[S] = _launches(dec)
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert torch.equal(y_hats[S], y_hat_enc)
  assert counts[7] == counts[1] == 11 * len(groups)
  assert enc[7] == enc[1] + 1  # the gather
  assert torch.equal(y_hats[7], y_hats[1])


def test_single_phase_encodes_make_no_more_launches():
  em = _em()
  g = torch.Generator().manual_seed(3)
  y = (3 * torch.randn(2, 4, 6, 8, generator=g)).cuda()
  idx = torch.randint(0, NUM_SCALES, (2, 4, 6, 8), generator=g).float().cuda()
  counts = [_launches(lambda: em.compress(y, idx, substreams=S), sync_free=False)[0] for S in (1, 8)]
  assert counts[0] == counts[1]


# ---------------------------------------------------------------------------------------------------------------
# damage
# ---------------------------------------------------------------------------------------------------------------
def test_damage_is_confined_to_its_image():
  groups, M, S = (12,), 12, 5
  em = _em()
  packed = _pack(groups, M)
  shapes = [(3, 4), (5, 7), (2, 6)]
  lat = [_latents(1, h, w, M, h) for h, w in shapes]
  ys, psis = [y[0] for y, _ in lat], [p[0] for _, p in lat]
  _, y_g, loc, index, lengths = F.cb_encode_ragged(packed[0], ys, psis, NUM_SCALES, substreams=S)
  parts = F.compress_ragged(em._lookup_host(), lengths, y_g, loc, em.cdf_offset, index=index)
  good = gen_ops.join_substreams(parts, S, (3,)).tolist()
  subs = [gen_ops.parse_substreams(s, S) for s in good]
  padded = [list(p) for p in subs]
  padded[1][2] += bytes(range(40))  # image 1, substream 2: bytes the decoder does not consume
  truncated = [list(p) for p in subs]
  truncated[1][4] = truncated[1][4][:len(truncated[1][4]) // 2]
  for damaged, must_fail in ((padded, True), (truncated, False)):
    strings = [gen_ops.substream_header([len(p) for p in ps]) + b"".join(ps) for ps in damaged]
    handle = gen_ops.create_range_decoder(gen_ops.split_substreams(gen_ops.Strings.from_bytes(strings, (3,)), S),
                                          em._lookup_host())
    F.cb_decode_ragged(handle, packed[0], psis, NUM_SCALES, em.cdf_offset, substreams=S)
    ok = gen_ops.entropy_decode_finalize(handle).reshape(3, S).all(dim=1).tolist()
    assert ok[0] and ok[2]
    if must_fail:
      assert not ok[1]
  bad = gen_ops.Strings.from_bytes([good[0], bytes([S, 0x80]), good[2]], (3,))
  n0 = _lib.launch_count()
  with pytest.raises(ValueError, match="string 1: truncated"):
    gen_ops.split_substreams(bad, S)
  m = models.CheckerboardModel(num_filters=8, latent_depth=M, substreams=S)
  m.entropy_model = em
  with pytest.raises(ValueError, match="string 1"):
    m._y_decoder(bad)
  assert _lib.launch_count() == n0
