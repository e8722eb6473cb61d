"""GPU: MBT2018's column tiles (functional.ar_encode_tiles / ar_decode_tiles, DESIGN §3.15).  The tile encoder gives
ar_encode_ragged's ŷ, loc, index and scale_index bit for bit, each tile stream is the reference coder's encoding of
its symbols, the tile decoder reproduces the encoder and the one-stream decoder on every key path and at saturated
escapes, the schedule runs lists with far more items than resident CTAs, launches do not depend on the list or on T
and nothing synchronises with the host, damage stays within its image, and MBT2018Model(tiles=T) codes the latents
and reconstructions of tiles=1."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import oracle
from compression_b200 import _lib
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models
from test_ar_reference_gpu import NUM_SCALES, _model, _weights

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (1, 9), (9, 1), (2, 3), (5, 7), (13, 17), (32, 48)]
_PACKED = {}


@pytest.fixture(scope="module", autouse=True)
def _private_memory_pool():
  """Every allocation of this module comes from a pool of its own, released when the module ends: the caching
  allocator's default pool is left exactly as the module found it.  Later modules' allocation checks count a reused
  cached block at its full size, so the free blocks a module leaves behind would change what they measure."""
  pool = torch.cuda.MemPool()
  with torch.cuda.use_mem_pool(pool):
    yield
    _PACKED.clear()
    gc.collect()
    torch.cuda.synchronize()
  del pool


@pytest.fixture(scope="module")
def em():
  return _model(NUM_SCALES)


def _packed(M, seed=7):
  if (M, seed) not in _PACKED:
    _PACKED[(M, seed)] = F.ar_pack_weights(*[w.cuda() for w in _weights(M, seed)])
  return _PACKED[(M, seed)]


def _latents(shapes, M, seed):
  g = torch.Generator().manual_seed(seed)
  ys = [(3 * torch.randn(H, W, M, generator=g)).cuda() for H, W in shapes]
  psis = [torch.randn(H, W, 2 * M, generator=g).cuda() for H, W in shapes]
  return ys, psis


def _gathered(shapes, M, T, *flat):
  """Raster-order flat tensors of a list in tile order."""
  if T == 1:
    return flat
  pos, wid = F.ar_tile_layout([h for h, _ in shapes], [w for _, w in shapes], T, M)
  return tuple(F.substream_gather(pos, wid, T, loc=t)[1] for t in flat)


def _strings(em, enc):
  _, y, loc, index, lengths = enc[:5]
  return F.compress_ragged(em._lookup_host(), lengths, y, loc, em.cdf_offset, index=index)


def _decode_tiles(em, packed, parts, psis, T):
  handle = gen_ops.create_range_decoder(parts, em._lookup_host())
  y_hats = F.ar_decode_tiles(handle, packed, psis, NUM_SCALES, em.cdf_offset, T)
  return y_hats, gen_ops.entropy_decode_finalize(handle)


def _ts(shapes, extra=()):
  ws = {w for _, w in shapes}
  return sorted({1, 2, 3, 5} | ws | {w + 3 for w in ws} | set(extra))


# ---------------------------------------------------------------------------------------------------------------
# the encoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [6, 12, 192])
def test_encoder_equals_the_ragged_encoder_bit_for_bit(M):
  packed = _packed(M)
  ys, psis = _latents(SHAPES, M, 1)
  ref = F.ar_encode_ragged(packed, ys, psis, NUM_SCALES, scale_index=True)
  for T in _ts(SHAPES) if M < 192 else [1, 2, 5, 17, 48, 51]:
    got = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T, scale_index=True)
    assert all(torch.equal(a, b) for a, b in zip(got[0], ref[0])), T
    want = _gathered(SHAPES, M, T, ref[1], ref[2], ref[3].view(torch.float32), ref[5])
    for name, g, w in zip(("y", "loc", "index", "scale_index"), (got[1], got[2], got[3].view(torch.float32), got[5]),
                          want):
      assert torch.equal(g.view(torch.int32), w.view(torch.int32)), (T, name)
    lengths = F.substream_layout(*F.ar_tile_layout([h for h, _ in SHAPES], [w for _, w in SHAPES], T, M), T)[0]
    assert got[4] == lengths.tolist()


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_encoder_on_one_image_at_t_equal_w(shape):
  packed = _packed(12)
  ys, psis = _latents([shape], 12, 2)
  ref = F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)
  for T in (1, shape[1], shape[1] + 3):
    got = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
    assert torch.equal(got[0][0], ref[0][0])
    assert all(torch.equal(g, w) for g, w in zip(got[1:4], _gathered([shape], 12, T, *ref[1:4])))


def test_tile_streams_are_the_reference_encoding_and_keep_the_rate_bound(em):
  O = oracle.best()
  M, T = 12, 5
  packed = _packed(M)
  ys, psis = _latents(SHAPES, M, 3)
  enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
  parts = _strings(em, enc).tolist()
  _, y, loc, index, lengths = enc
  sym = (torch.round(y - loc).to(torch.int32) - em.cdf_offset[index.long()]).cpu().numpy()
  idx = index.cpu().numpy()
  offs = np.concatenate([[0], np.cumsum(lengths)])
  for k, s in enumerate(parts):
    seg = slice(offs[k], offs[k + 1])
    assert s == (O.encode(em._lookup_host(), sym[seg][None], idx[seg][None])[0] if lengths[k] else b""), k
  joined = gen_ops.join_substreams(_strings(em, enc), T, (len(SHAPES),)).tolist()
  one = _strings(em, F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)).tolist()
  for i, s in enumerate(joined):
    mine = parts[i * T:(i + 1) * T]
    header = gen_ops.substream_header([len(p) for p in mine])
    assert s == header + b"".join(mine)
    assert len(s) <= len(one[i]) + len(header) + 4 * T


# ---------------------------------------------------------------------------------------------------------------
# the decoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,shapes,Ts", [(12, SHAPES, [1, 2, 5, 17, 48, 51]),
                                         (192, [(2, 3), (1, 1), (5, 7), (13, 17)], [3, 17])])
def test_decoder_reproduces_the_encoder_and_the_one_stream_decoder(em, M, shapes, Ts):
  packed = _packed(M)
  ys, psis = _latents(shapes, M, 4)
  ref = F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)
  handle = gen_ops.create_range_decoder(_strings(em, ref), em._lookup_host())
  one = F.ar_decode_ragged(handle, packed, psis, NUM_SCALES, em.cdf_offset)
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  assert all(torch.equal(a, b) for a, b in zip(one, ref[0]))
  for T in Ts:
    enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
    y_hats, ok = _decode_tiles(em, packed, _strings(em, enc), psis, T)
    assert bool(ok.all()), T
    assert all(torch.equal(a, b) for a, b in zip(y_hats, one)), T


def _escape_latents(shape, M, T, seed):
  ys, psis = _latents([shape], M, seed)
  y = ys[0]
  W = shape[1]
  for t in range(T):
    c0, c1 = t * W // T, (t + 1) * W // T
    if c1 > c0:
      y[:, c0, 0::2] = 3e9  # saturates to 2^31 - 1
      y[:, c1 - 1, 1::2] = -3e9  # saturates to -2^31
  y[shape[0] // 2, W // 2, :] = 1e6  # every channel of a position escapes
  return ys, psis


@pytest.mark.parametrize("M,T", [(12, 5), (12, 17), (192, 4)])
def test_saturated_escapes_at_tile_edges(em, M, T):
  shape = (4, 17) if M == 192 else (13, 17)
  packed = _packed(M)
  ys, psis = _escape_latents(shape, M, T, 5)
  ref = F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)
  assert float(ref[0][0].abs().max()) >= 2.0**31
  enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
  assert torch.equal(enc[0][0], ref[0][0])
  y_hats, ok = _decode_tiles(em, packed, _strings(em, enc), psis, T)
  assert bool(ok.all()) and torch.equal(y_hats[0], ref[0][0])


@pytest.mark.parametrize("M", [96, 192])
def test_decoder_with_search_keys_in_global_memory(M):
  em_wide = _model(160)  # 160 tables: the keys do not fit beside the activations
  packed = F.ar_pack_weights(*[w.cuda() for w in _weights(M, 7)])
  shapes = [(3, 5), (1, 1), (2, 4)]
  ys, psis = _latents(shapes, M, 6)
  for T in (2, 5):
    y_hats_ref, _, loc, index, lengths = F.ar_encode_ragged(packed, ys, psis, 160)
    enc = F.ar_encode_tiles(packed, ys, psis, 160, T)
    assert all(torch.equal(a, b) for a, b in zip(enc[0], y_hats_ref))
    parts = F.compress_ragged(em_wide._lookup_host(), enc[4], enc[1], enc[2], em_wide.cdf_offset, index=enc[3])
    handle = gen_ops.create_range_decoder(parts, em_wide._lookup_host())
    y_hats = F.ar_decode_tiles(handle, packed, psis, 160, em_wide.cdf_offset, T)
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert all(torch.equal(a, b) for a, b in zip(y_hats, y_hats_ref))


def test_decoder_at_the_largest_depth_with_shared_keys(em):
  M, T = 384, 2
  packed = _packed(M)
  ys, psis = _latents([(3, 4)], M, 7)
  ys[0][0, 0, :4] = torch.tensor([1e5, -1e5, 3e9, -3e9], device="cuda")
  ref = F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)
  enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
  y_hats, ok = _decode_tiles(em, packed, _strings(em, enc), psis, T)
  assert bool(ok.all()) and torch.equal(y_hats[0], ref[0][0]) and torch.equal(enc[0][0], ref[0][0])


# ---------------------------------------------------------------------------------------------------------------
# the schedule, launches and damage
# ---------------------------------------------------------------------------------------------------------------
def test_schedule_at_scale_and_a_one_item_list(em):
  M, T = 6, 48
  packed = _packed(M)
  shapes = [(32, 48)] * 40  # 61 440 items
  assert len(F.ar_tiles_schedule([32] * 40, [48] * 40, T)) == 61440
  ys, psis = _latents(shapes, M, 8)
  ref = F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)
  enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
  assert all(torch.equal(a, b) for a, b in zip(enc[0], ref[0]))
  y_hats, ok = _decode_tiles(em, packed, _strings(em, enc), psis, T)
  assert bool(ok.all()) and all(torch.equal(a, b) for a, b in zip(y_hats, ref[0]))
  ys, psis = _latents([(1, 1)], M, 9)
  for T in (1, 3):
    enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
    y_hats, ok = _decode_tiles(em, packed, _strings(em, enc), psis, T)
    assert bool(ok.all()) and torch.equal(y_hats[0], F.ar_encode_ragged(packed, ys, psis, NUM_SCALES)[0][0])


def test_launches_do_not_depend_on_the_list_or_t_and_nothing_synchronises(em):
  packed = _packed(12)
  dec_counts, enc_counts = [], []
  for shapes in ([(5, 7)], [(5, 7)] * 4, [(1, 5), (3, 7), (17, 9), (2, 2), (32, 48), (5, 1)]):
    ys, psis = _latents(shapes, 12, 10)
    for T in (1, 3, 48):
      torch.cuda.synchronize()
      n0 = _lib.launch_count()
      torch.cuda.set_sync_debug_mode("error")
      try:
        enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
      finally:
        torch.cuda.set_sync_debug_mode(0)
      enc_counts.append(_lib.launch_count() - n0 - (T > 1))  # (the gather into tile order)
      handle = gen_ops.create_range_decoder(_strings(em, enc), em._lookup_host())
      coff = em.cdf_offset.cuda()
      torch.cuda.synchronize()
      n0 = _lib.launch_count()
      torch.cuda.set_sync_debug_mode("error")
      try:
        y_hats = F.ar_decode_tiles(handle, packed, psis, NUM_SCALES, coff, T)
      finally:
        torch.cuda.set_sync_debug_mode(0)
      dec_counts.append(_lib.launch_count() - n0)
      assert bool(gen_ops.entropy_decode_finalize(handle).all())
      assert all(torch.equal(a, b) for a, b in zip(y_hats, enc[0]))
  assert enc_counts == [1] * 9 and dec_counts == [1] * 9


def test_a_damaged_tile_stream_fails_only_its_image(em):
  M, T = 12, 3
  packed = _packed(M)
  shapes = [(5, 7), (3, 9), (13, 17), (2, 3)]
  ys, psis = _latents(shapes, M, 11)
  enc = F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, T)
  parts = _strings(em, enc).tolist()
  i = 2
  bad = list(parts)
  bad[i * T + 1] = bad[i * T + 1] + bytes(range(64))
  y_hats, ok = _decode_tiles(em, packed, gen_ops.Strings.from_bytes(bad, (len(bad),)), psis, T)
  ok = ok.view(len(shapes), T).all(dim=1).tolist()
  assert ok == [j != i for j in range(len(shapes))]
  assert all(torch.equal(y_hats[j], enc[0][j]) for j in range(len(shapes)) if j != i)
  assert all(bool(torch.isfinite(y).all()) for y in y_hats)


def test_bad_arguments_raise_before_any_launch(em):
  M, T = 12, 3
  packed = _packed(M)
  ys, psis = _latents([(3, 7), (2, 2)], M, 12)
  strings = _strings(em, F.ar_encode_ragged(packed, ys, psis, NUM_SCALES))  # one string per image, not per tile
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a list of 2 in 3 tiles"):
    F.ar_decode_tiles(handle, packed, psis, NUM_SCALES, em.cdf_offset, T)
  hs, ws = np.array([3, 2], np.int64), np.array([7, 2], np.int64)
  hp = lambda a: a.ctypes.data_as(C.c_void_p)
  lib = _lib.lib()
  nw = int(lib.tfcb_ar_tiles_workspace_floats(2, hp(hs), hp(ws), T))
  work = torch.empty(nw, device="cuda")
  psi, out = torch.cat([p.reshape(-1) for p in psis]), torch.empty(34 * M, device="cuda")
  coff = em.cdf_offset.cuda()
  with pytest.raises(_lib.InvalidArgumentError, match="the decoder holds 2 strings for a batch of 6"):
    _lib.check(lib.tfcb_ar_decode_tiles(handle._h, F._p(packed), packed.numel(), M, F._p(psi), 2, hp(hs), hp(ws), T,
                                        NUM_SCALES, F._p(coff), F._p(work), nw, F._p(out), None))
  with pytest.raises(ValueError, match="tiles"):
    F.ar_encode_tiles(packed, ys, psis, NUM_SCALES, 0)
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------
def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  out = []
  for h, w in sizes:
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 60 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None] * np.array([1.0, 0.7, 0.4])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)))
  return out


@pytest.fixture(scope="module")
def base_model():
  torch.manual_seed(0)
  return models.MBT2018Model(num_filters=24, latent_depth=12).build("cuda", patch=(64, 64)).fix_tables()


def _tiled(base, T):
  m = models.MBT2018Model(num_filters=24, latent_depth=12, tiles=T).build("cuda", patch=(64, 64))
  m.load_state_dict({k: v for k, v in base.state_dict().items()  # (the weights; fix_tables rebuilds the tables)
                     if not k.startswith(("entropy_model.", "side_entropy_model."))})
  return m.fix_tables()


@pytest.mark.parametrize("T", [2, 7, 48, 64])
def test_model_tiles_decode_the_one_stream_latents(base_model, T):
  m = _tiled(base_model, T)
  x = _images([(112, 200)], 3)[0]  # latents 7 x 13
  one, tiled = base_model.compress(x), m.compress(x)
  assert tiled[1].tolist() == one[1].tolist()  # z is unchanged
  assert all(torch.equal(a, b) for a, b in zip(one[2:], tiled[2:]))
  assert gen_ops.parse_substreams(tiled[0].tolist()[0], T)  # T tile streams in the substream container
  assert torch.equal(m.decompress(*tiled), base_model.decompress(*one))
  # latents: the decoder's ŷ equals the one-stream encoder's
  y = base_model.analysis_transform(x[None].cuda().float())
  z = base_model.hyper_analysis_transform(y)
  psi = base_model._psi(base_model.side_entropy_model.quantize(z), tuple(y.shape[1:3]))
  _, y_hat1, _, _ = base_model._encode_latents(y, psi)
  strings, y_hat_t, _, _ = m._encode_latents(y, psi)
  assert torch.equal(y_hat_t, y_hat1) and torch.equal(m._decode_latents(strings, psi), y_hat1)
  # batch, list, .tfci and evaluate
  xs = _images([(64, 96)] * 3, 4)
  b1, bt = base_model.compress_batch(torch.stack(xs)), m.compress_batch(torch.stack(xs))
  assert torch.equal(m.decompress_batch(*bt), base_model.decompress_batch(*b1))
  imgs = _images([(80, 48), (48, 80), (16, 16), (112, 65)], 5)
  outs = m.decompress_images(m.compress_images(imgs))
  assert all(torch.equal(a, b) for a, b in zip(outs, base_model.decompress_images(base_model.compress_images(imgs))))
  assert torch.equal(m.decompress_from_tfci(m.compress_to_tfci(x)), base_model.decompress(*one))
  big = _images([(176, 192)], 6)  # (MS-SSIM's five scales need 176 pixels a side)
  e1, et = base_model.evaluate(big[0]), m.evaluate(big[0])
  assert e1["mse"] == et["mse"] and e1["msssim"] == et["msssim"] and et["bpp"] >= e1["bpp"]
  assert [d["msssim"] for d in m.evaluate_images(big)] == [d["msssim"] for d in base_model.evaluate_images(big)]


def test_model_strings_are_rejected_under_another_t(base_model):
  m7, m2 = _tiled(base_model, 7), _tiled(base_model, 2)
  x = _images([(112, 200)], 7)[0]
  item = m7.compress(x)
  with pytest.raises(ValueError, match="written with 7 substreams, decoding expects 2"):
    m2.decompress(*item)
  items = m7.compress_images([x, x])
  with pytest.raises(ValueError, match="string 0"):
    m2.decompress_images(items)
