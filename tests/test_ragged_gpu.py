"""GPU: ragged batches -- streams of different lengths coded in one launch (tfcb_compress_ragged /
tfcb_decode_ragged and the entropy-model and image-model layers above them).

The reference codes one image per call and has no ragged op; the contract is that string i of a ragged call is
byte-identical to what the existing path makes of item i alone, and so to the oracle's string for it.
"""
import numpy as np
import pytest
import torch

import oracle
import util

pytestmark = pytest.mark.gpu

SPECIAL = [0, 1, 31, 32, 33, 255, 256, 257, 4109]


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import gen_ops
  return gen_ops


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


def _lengths(rng, n_streams):
  if n_streams == 1:
    return [200_003]
  if n_streams == 7:
    return [0, 1, 33, 257, 4109, 31, 256]
  lens = list(SPECIAL) + [200_001] + [int(v) for v in rng.integers(0, 3000, n_streams - len(SPECIAL) - 1)]
  rng.shuffle(lens)
  return lens


def _tables(rng, nrows, overflow=True):
  precs = [int(rng.integers(5, 17)) for _ in range(nrows)]
  cdfs = [util.random_cdf(rng, int(rng.integers(2, min(40, 1 << p) + 1)), p, peaky=3) for p in precs]
  ovf = [overflow and bool(rng.random() < 0.6) for _ in range(nrows)]
  return cdfs, precs, ovf


def _symbols(rng, cdfs, ovf, rows):
  nb = np.asarray([len(c) - 1 for c in cdfs])[rows]
  is_ovf = np.asarray(ovf)[rows]
  v = (rng.random(rows.shape) * np.where(is_ovf, np.maximum(nb - 1, 1), nb)).astype(np.int64)
  esc = is_ovf & (rng.random(rows.shape) < 0.05)
  wild = rng.integers(-60, 60, size=rows.shape) + np.where(rng.random(rows.shape) < 0.5, 0, nb)
  big = is_ovf & (rng.random(rows.shape) < 0.002)  # escapes of large magnitude: long Elias-gamma tails
  v = np.where(esc, wild, v)
  v = np.where(big, rng.integers(-(1 << 30), 1 << 30, size=rows.shape), v)
  return v.astype(np.int32)


def _rows(rng, lens, nrows, index_mode):
  """Per stream the lookup row of every symbol: the index (index mode) or j mod nrows from 0 (channel mode)."""
  if index_mode:
    return [rng.integers(0, nrows, n).astype(np.int32) for n in lens]
  return [(np.arange(n) % nrows).astype(np.int32) for n in lens]


def _cat(parts, dtype):
  return torch.from_numpy(np.concatenate(parts).astype(dtype) if parts else np.zeros(0, dtype)).cuda()


@pytest.mark.parametrize("n_streams", [1, 7, 300])
@pytest.mark.parametrize("mode", ["channel", "index"])
def test_int32_streams_match_oracle_and_uniform_path(ops, F, n_streams, mode):
  rng = np.random.default_rng(n_streams * 2 + (mode == "index"))
  O = oracle.best()
  nrows = 5  # stream lengths are mostly not multiples of the row count
  cdfs, precs, ovf = _tables(rng, nrows)
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  lens = _lengths(rng, n_streams)
  rows = _rows(rng, lens, nrows, mode == "index")
  vals = [_symbols(rng, cdfs, ovf, r) for r in rows]
  index = _cat(rows, np.int32) if mode == "index" else None
  got = F.compress_ragged(lookup, lens, _cat(vals, np.int32), index=index)
  assert got.shape == (n_streams,)
  got_l = got.tolist()
  want = []
  for v, r in zip(vals, rows):
    want += O.encode(lookup, v[None], r[None] if mode == "index" else None)
  assert got_l == want
  # the uniform path, stream by stream
  for i in [i for i, n in enumerate(lens) if n in SPECIAL or n > 100_000][:12]:
    h = ops.create_range_encoder([1], lookup)
    if mode == "index":
      ops.entropy_encode_index(h, torch.from_numpy(rows[i][None]).cuda(), torch.from_numpy(vals[i][None]).cuda())
    else:
      ops.entropy_encode_channel(h, torch.from_numpy(vals[i][None]).cuda())
    assert ops.entropy_encode_finalize(h).tolist() == [got_l[i]]
  # decoding: our strings and the oracle's
  for strings in (got, ops.Strings.from_bytes(want, (n_streams,))):
    hd = ops.create_range_decoder(strings, lookup)
    dec = F.decode_ragged(hd, lens, index=index)
    assert bool(ops.entropy_decode_finalize(hd).all())
    assert np.array_equal(dec.cpu().numpy(), np.concatenate(vals))


@pytest.mark.parametrize("mode", ["channel", "index"])
def test_float32_quantisation_matches_uniform_path(ops, F, mode):
  """Quantisation offsets (channel) / loc (index) and cdf offsets, fused into the ragged kernels, against
  compress_f32 / decode_*_f32 of every stream alone."""
  rng = np.random.default_rng(40 + (mode == "index"))
  nrows = 6
  cdfs = [util.laplace_cdf(n, 12, s) for n, s in ((41, 3.0), (31, 2.0), (61, 8.0), (9, 0.7), (21, 1.5), (101, 20.0))]
  lookup = util.make_lookup_1d(cdfs, [12] * nrows, [True] * nrows)
  coff = torch.tensor([-(len(c) - 1) // 2 for c in cdfs], dtype=torch.int32).cuda()
  lens = [0, 1, 33, 4109, 257, 31, 1000, 6 * 50]
  total = sum(lens)
  y = torch.from_numpy((rng.standard_normal(total) * 6).astype(np.float32)).cuda()
  y[torch.from_numpy(rng.random(total) < 0.01).cuda()] *= 500  # escapes
  starts = np.concatenate([[0], np.cumsum(lens)])
  if mode == "channel":
    q = torch.from_numpy(rng.uniform(-0.5, 0.5, nrows).astype(np.float32)).cuda()
    index = None
  else:
    q = torch.from_numpy(rng.uniform(-2, 2, total).astype(np.float32)).cuda()
    index = torch.from_numpy(rng.integers(0, nrows, total).astype(np.int32)).cuda()
  got = F.compress_ragged(lookup, lens, y, q, coff, index=index).tolist()
  hd = ops.create_range_decoder(ops.Strings.from_bytes(got, (len(lens),)), lookup)
  dec = F.decode_ragged(hd, lens, index=index, quant_offset=q, cdf_offset=coff)
  assert bool(ops.entropy_decode_finalize(hd).all())
  for i, n in enumerate(lens):
    sl = slice(int(starts[i]), int(starts[i + 1]))
    yi = y[sl][None]
    if mode == "channel":
      one = F.compress_f32((1,), lookup, yi, q, coff)
    else:
      one = F.compress_f32((1,), lookup, yi, q[sl][None], coff, index=index[sl][None])
    assert one.tolist() == [got[i]], i
    if n == 0:
      continue
    hu = ops.create_range_decoder(one, lookup)
    if mode == "channel":
      ref = F.decode_channel_f32(hu, (1, n), q, coff)
    else:
      ref = F.decode_index_f32(hu, index[sl][None], q[sl][None], coff)
    assert torch.equal(dec[sl], ref.reshape(-1)), i


def test_truncated_strings_verdicts_match_oracle(ops, F):
  rng = np.random.default_rng(5)
  O = oracle.best()
  cdfs, precs, ovf = _tables(rng, 4, overflow=False)
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  lens = [0, 1, 100, 2000, 777, 31, 5000, 64]
  rows = _rows(rng, lens, 4, False)
  vals = [_symbols(rng, cdfs, ovf, r) for r in rows]
  strings = F.compress_ragged(lookup, lens, _cat(vals, np.int32)).tolist()
  # odd streams truncated to half (reads past the end see zeros: the verdict may go either way, the oracle's rules);
  # stream 2 with trailing bytes the decoder never reaches (always False)
  cut = [s[:len(s) // 2] if k % 2 else s for k, s in enumerate(strings)]
  cut[2] = cut[2] + b"\x5a\xa5\x33"
  hd = ops.create_range_decoder(ops.Strings.from_bytes(cut, (len(lens),)), lookup)
  F.decode_ragged(hd, lens)
  ok = ops.entropy_decode_finalize(hd).numpy()
  want = np.asarray([bool(O.decode(lookup, [s], n)[1][0]) for s, n in zip(cut, lens)])
  assert np.array_equal(ok, want)
  assert not want[2] and want[0] and want[4]


@pytest.mark.parametrize("mode", ["channel", "index"])
def test_argument_errors_name_stream_and_position(ops, F, mode):
  cdf = np.asarray([0, 4, 8, 16], np.int32)
  lookup = util.make_lookup_1d([cdf, cdf], [4, 4], [False, False])
  lens = [5, 0, 40, 7]
  value = np.zeros(sum(lens), np.int32)
  index = np.zeros(sum(lens), np.int32)
  k, j = 2, 37
  if mode == "channel":
    value[lens[0] + lens[1] + j] = 3
    with pytest.raises(ops.InvalidArgumentError, match=rf"value=3 not in range \[0, 3\) \(stream {k}, element {j}\)"):
      F.compress_ragged(lookup, lens, torch.from_numpy(value).cuda())
  else:
    index[lens[0] + lens[1] + j] = 2
    with pytest.raises(ops.InvalidArgumentError, match=rf"index=2 not in range \[0, 2\) \(stream {k}, element {j}\)"):
      F.compress_ragged(lookup, lens, torch.from_numpy(value).cuda(), index=torch.from_numpy(index).cuda())
  # the pooled encoder that saw the error is clean for the next call
  ok = F.compress_ragged(lookup, lens, torch.zeros(sum(lens), dtype=torch.int32).cuda())
  assert ok.tolist() == [oracle.best().encode(lookup, np.zeros((1, n), np.int32))[0] for n in lens]


def test_cfg2_tables_on_a_mixed_size_set(ops, F):
  """cfg2's committed tables (128 channel rows) over latents of differently sized images, as bench.py synthesises
  them: each string equals compress_f32 of that image alone, and the ragged decode returns the uniform one's."""
  g = np.load(util_golden("cfg2_tables.npz"))
  lookup, coff = g["lookup"], torch.from_numpy(g["cdf_offset"].astype(np.int32)).cuda()
  qoff = torch.from_numpy(g["quantization_offset"]).cuda() if bool(g["has_qoff"]) else None
  C = coff.numel()
  gen = torch.Generator().manual_seed(9)
  scales = torch.exp(torch.linspace(np.log(0.3), np.log(8.0), C))
  sizes = [(768, 512), (512, 768), (1280, 720), (64, 48), (16, 16), (1024, 768)]
  ys = []
  for h, w in sizes:  # Laplace(0, s_c) latents of a 16x-downsampling transform, as bench.py synthesises them
    u = torch.rand(-(-h // 16), -(-w // 16), C, generator=gen) - 0.5
    ys.append((-scales * torch.sign(u) * torch.log1p(-2 * u.abs()).clamp_min(-17.0)).contiguous().cuda())
  lens = [y.numel() for y in ys]
  got = F.compress_ragged(lookup, lens, torch.cat([y.reshape(-1) for y in ys]), qoff, coff)
  got_l = got.tolist()
  hd = ops.create_range_decoder(got, lookup)
  dec = F.decode_ragged(hd, lens, quant_offset=qoff, cdf_offset=coff)
  assert bool(ops.entropy_decode_finalize(hd).all())
  at = 0
  for i, y in enumerate(ys):
    one = F.compress_f32((1,), lookup, y[None], qoff, coff)
    assert one.tolist() == [got_l[i]]
    hu = ops.create_range_decoder(one, lookup)
    ref = F.decode_channel_f32(hu, (1,) + tuple(y.shape), qoff, coff)
    assert torch.equal(dec[at:at + y.numel()], ref.reshape(-1))
    at += y.numel()


def util_golden(name):
  import os
  return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name)


def test_arena_is_the_sum_of_per_stream_bounds(ops, F):
  """One 20 M-symbol stream on overflow rows plus 4 095 one-symbol streams.  Sized as n_streams times the longest
  stream's worst case the arena would need hundreds of GB; sized as the sum it fits."""
  rng = np.random.default_rng(12)
  cdfs = [util.laplace_cdf(33, 12, 2.0), util.laplace_cdf(17, 10, 1.0)]
  lookup = util.make_lookup_1d(cdfs, [12, 10], [True, True])
  big = 20_000_000
  lens = [big] + [1] * 4095
  n = sum(lens)
  value = torch.randint(0, 15, (n,), dtype=torch.int32, device="cuda")
  value[torch.rand(n, device="cuda") < 0.001] = 400  # escapes
  got = F.compress_ragged(lookup, lens, value)
  hd = ops.create_range_decoder(got, lookup)
  dec = F.decode_ragged(hd, lens)
  assert bool(ops.entropy_decode_finalize(hd).all())
  assert torch.equal(dec, value)
  got_l = got.tolist()
  small = value[big:].cpu().numpy()
  want = [oracle.best().encode(lookup, small[i:i + 1][None])[0] for i in range(0, 4095, 97)]
  assert [got_l[1 + i] for i in range(0, 4095, 97)] == want


# ------------------------------------------------------------------------------------------------
# Entropy models and image models
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
def test_batched_entropy_model_ragged(dtype):
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  torch.manual_seed(0)
  prior = D.NoisyLogistic(loc=torch.linspace(-1, 1, 8), scale=torch.linspace(0.5, 4, 8))
  em = E.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=True, bottleneck_dtype=dtype).cuda()
  xs = [torch.randn(n, 8, device="cuda") * 5 for n in (1, 17, 0, 300, 64)]
  strings = em.compress_ragged(xs)
  # (compress() itself takes no empty item outside float32: that one is the empty string, a fresh encoder's flush)
  assert strings.tolist() == [em.compress(x).tolist()[0] if x.numel() else b"" for x in xs]
  back = em.decompress_ragged(strings, [(x.shape[0],) for x in xs])
  for x, b in zip(xs, back):
    assert b.dtype == dtype and b.shape == x.shape
    if dtype != torch.float16:  # (compress quantises float16 latents in float32, quantize() in float16)
      assert torch.equal(b, em.quantize(x))
    if x.numel():
      assert torch.equal(b, em.decompress(em.compress(x[None]), (x.shape[0],))[0])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_indexed_entropy_models_ragged(dtype):
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  torch.manual_seed(1)
  em = E.ContinuousIndexedEntropyModel(D.NoisyNormal, index_ranges=(4, 5), parameter_fns=dict(
      loc=lambda i: i[..., 0] * 0.5, scale=lambda i: torch.exp(i[..., 1] * 0.5)), coding_rank=2,
      channel_axis=-1, compression=True, bottleneck_dtype=dtype).cuda()
  xs = [torch.randn(h, w, device="cuda") * 4 for h, w in ((3, 5), (1, 1), (40, 7), (0, 3))]
  idx = [torch.rand(x.shape + (2,), device="cuda") * torch.tensor([4., 5.], device="cuda") for x in xs]
  strings = em.compress_ragged(xs, idx)
  assert strings.tolist() == [em.compress(x, i).tolist()[0] for x, i in zip(xs, idx)]
  for x, b in zip(xs, em.decompress_ragged(strings, idx)):
    assert torch.equal(b, em.quantize(x))

  ls = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 16, lambda i: torch.exp(i / 4 - 1), coding_rank=3,
                                          compression=True, bottleneck_dtype=dtype).cuda()
  xs = [torch.randn(h, w, 5, device="cuda") * 6 for h, w in ((4, 4), (5, 3), (1, 9), (17, 2))]
  sc = [torch.rand(x.shape, device="cuda") * 16 for x in xs]
  loc = [torch.randn(x.shape, device="cuda", dtype=dtype) for x in xs]
  strings = ls.compress_ragged(xs, sc, loc)
  assert strings.tolist() == [ls.compress(x, s, l).tolist()[0] for x, s, l in zip(xs, sc, loc)]
  for x, l, b in zip(xs, loc, ls.decompress_ragged(strings, sc, loc)):
    assert torch.equal(b, ls.quantize(x, l))


def test_decompress_ragged_sanity_check():
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  from compression_b200 import gen_ops
  prior = D.NoisyLogistic(loc=torch.zeros(4), scale=torch.ones(4) * 3)
  em = E.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=True).cuda()
  xs = [torch.randn(200, 4, device="cuda") * 3, torch.randn(300, 4, device="cuda") * 3]
  strings = em.compress_ragged(xs).tolist()
  bad = [strings[0], strings[1] + b"\x01\x02\x03"]  # trailing bytes the decoder never reaches
  with pytest.raises(gen_ops.InvalidArgumentError, match="Sanity check failed"):
    em.decompress_ragged(bad, [(200,), (300,)])
  em.decode_sanity_check = False
  em.decompress_ragged(bad, [(200,), (300,)])


SIZES = [(64, 64), (80, 48), (48, 80), (33, 65), (16, 16)]


def _images():
  g = torch.Generator().manual_seed(4)
  return [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8) for h, w in SIZES]


def _same(a, b):
  if hasattr(a, "tolist") and not isinstance(a, torch.Tensor):
    return a.shape == b.shape and a.tolist() == b.tolist()
  return torch.equal(a, b)


@pytest.mark.parametrize("name", ["bls2017", "bmshj2018"])
def test_image_models_compress_images(name):
  from compression_b200 import models
  torch.manual_seed(2)
  model = (models.BLS2017Model(num_filters=32) if name == "bls2017" else
           models.BMSHJ2018Model(num_filters=32, num_scales=16)).build("cuda").fix_tables()
  images = _images()
  got = model.compress_images(images)
  assert len(got) == len(images)
  for g, x in zip(got, images):
    want = model.compress(x)
    assert len(g) == len(want) and all(_same(a, b) for a, b in zip(g, want))
  dec = model.decompress_images(got)
  for d, g, x in zip(dec, got, images):
    assert d.shape == x.shape and d.dtype == torch.uint8
    assert torch.equal(d, model.decompress(*g))
