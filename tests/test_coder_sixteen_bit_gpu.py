"""GPU: float16 / bfloat16 bottlenecks on the 16-bit range-coder entries (quantised in the encoder, dequantised in
the decoder, the decoded items of a ragged encode written by the encoder).

The contract is the unfused path on the same device: strings equal `compress(..., fused=False)` byte for byte, decoded
tensors equal `decompress(..., fused=False)` in dtype, shape and bits, ragged strings equal the per-item `compress`,
and `return_decoded` items equal `decompress_ragged` with no decoder run.  The edge values are the ones where 16-bit
and float32 arithmetic part: signed zeros, subnormals, .5 ties, the largest finite values, infinities, NaN,
bfloat16 values beyond 2^31, escapes both ways, decoded magnitudes beyond 2^24 in bfloat16 and float16 decodes that
overflow to inf.
"""
import os

import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
CFG2 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cfg2_tables.npz")
# exactly representable in both types (3.3554432e7 = 2^25, 1207959552 = 1.125 * 2^30, 2147483648 = 2^31)
SPECIAL = [0.0, -0.0, 0.5, -0.5, 1.5, 2.5, -2.5, 3.5, 65504.0, -65504.0, 2.0**-24, -2.0**-24, 2.0**-14 * 0.75,
           float("inf"), float("-inf"), float("nan"), 33554432.0, -1207959552.0, 2147483648.0, 3e9, -3e9, 1e30,
           -1e38, 1e-40, 2.0**-133]


@pytest.fixture(scope="module")
def E():
  from compression_b200 import entropy_models
  return entropy_models


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


def _bits(t):
  return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _same(a, b):
  return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _latents(shape, dtype, seed, scale=4.0, specials=True):
  g = torch.Generator().manual_seed(seed)
  y = torch.randn(shape, generator=g) * scale
  y[torch.rand(shape, generator=g) < 0.02] *= 300  # escapes, both signs
  y = y.reshape(-1)
  if specials and y.numel():
    at = torch.randperm(y.numel(), generator=g)[:min(y.numel(), 4 * len(SPECIAL))]
    y[at] = torch.tensor(SPECIAL * 4)[:at.numel()]
  return y.reshape(shape).to(dtype).cuda()


def _cfg2_model(E, dtype, with_offsets):
  z = np.load(CFG2)
  q = torch.linspace(-0.45, 0.45, 128) if with_offsets else None
  return E.ContinuousBatchedEntropyModel(
      prior_shape=(128,), coding_rank=3, compression=True, cdf=torch.from_numpy(z["lookup"]),
      cdf_offset=torch.from_numpy(z["cdf_offset"]), bottleneck_dtype=dtype, offset_heuristic=False,
      quantization_offset=q).cuda()


def _small_batched(E, dtype, seed=0):
  from compression_b200 import distributions as D
  torch.manual_seed(seed)
  prior = D.NoisyLogistic(loc=torch.linspace(-1, 1, 8), scale=torch.linspace(0.5, 4, 8))
  return E.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=True, bottleneck_dtype=dtype).cuda()


def _indexed(E, dtype):
  from compression_b200 import distributions as D
  return E.ContinuousIndexedEntropyModel(D.NoisyNormal, index_ranges=(4, 5), parameter_fns=dict(
      loc=lambda i: i[..., 0] * 0.5, scale=lambda i: torch.exp(i[..., 1] * 0.5)), coding_rank=2, channel_axis=-1,
      compression=True, bottleneck_dtype=dtype).cuda()


def _loc_scale(E, dtype):
  from compression_b200 import distributions as D
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 16, lambda i: torch.exp(i / 4 - 1), coding_rank=3,
                                            compression=True, bottleneck_dtype=dtype).cuda()


def _count_routes(monkeypatch, F):
  calls = {}
  for name in ("compress_16bit", "compress_ragged_16bit", "decode_16bit", "decode_ragged_16bit"):
    def counted(*a, _fn=getattr(F, name), _name=name, **k):
      calls[_name] = calls.get(_name, 0) + 1
      return _fn(*a, **k)
    monkeypatch.setattr(F, name, counted)
  return calls


def _loc_of(kind, shape, dtype, seed):
  if kind is None:
    return None
  g = torch.Generator().manual_seed(seed)
  loc = torch.randn(shape, generator=g) * 3
  loc.reshape(-1)[:8] = torch.tensor([0.5, -0.5, 1e-3, 65504.0, -2.5, 0.25, 1e4, -0.0])[:loc.numel()]
  return loc.to(dtype if kind == "same" else torch.float32).cuda()


# ------------------------------------------------------------------------------------------------
# compress / decompress against fused=False
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_offsets", [False, True])
@pytest.mark.parametrize("shape", [(1, 1, 1, 128), (3, 2, 5, 128), (16, 4, 4, 128)])
def test_batched_matches_unfused(E, F, monkeypatch, dtype, with_offsets, shape):
  em = _cfg2_model(E, dtype, with_offsets)
  y = _latents(shape, dtype, 10 + len(shape) + shape[0] + with_offsets)
  calls = _count_routes(monkeypatch, F)
  got = em.compress(y)
  want = em.compress(y, fused=False)
  assert calls == {"compress_16bit": 1}
  assert torch.equal(got.offsets_dev, want.offsets_dev) and got.tolist() == want.tolist()
  back = em.decompress(got, shape[1:3])
  assert calls == {"compress_16bit": 1, "decode_16bit": 1}
  assert back.dtype == dtype and _same(back, em.decompress(got, shape[1:3], fused=False))


@pytest.mark.parametrize("dtype", DTYPES)
def test_batched_one_symbol_and_partial_passes(E, F, dtype):
  em = _small_batched(E, dtype)
  for n in (1, 3, 4, 5, 37):  # 8 to 296 symbols: a partial gather pass at the end of each
    y = _latents((2, n, 8), dtype, 50 + n)
    got = em.compress(y)
    assert got.tolist() == em.compress(y, fused=False).tolist()
    assert _same(em.decompress(got, (n,)), em.decompress(got, (n,), fused=False))


@pytest.mark.parametrize("dtype", DTYPES)
def test_indexed_matches_unfused(E, F, monkeypatch, dtype):
  em = _indexed(E, dtype)
  g = torch.Generator().manual_seed(3)
  for shape in ((1, 1), (3, 5), (40, 7)):
    y = _latents((2,) + shape, dtype, 60 + shape[0])
    idx = (torch.rand((2,) + shape + (2,), generator=g) * torch.tensor([4., 5.])).cuda()
    calls = _count_routes(monkeypatch, F)
    got = em.compress(y, idx)
    assert got.tolist() == em.compress(y, idx, fused=False).tolist()
    back = em.decompress(got, idx)
    assert calls == {"compress_16bit": 1, "decode_16bit": 1}
    assert back.dtype == dtype and _same(back, em.decompress(got, idx, fused=False))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("loc_kind", [None, "same", "float32"])
def test_location_scale_matches_unfused(E, F, monkeypatch, dtype, loc_kind):
  em = _loc_scale(E, dtype)
  g = torch.Generator().manual_seed(4)
  for shape in ((1, 1, 1, 1), (2, 3, 4, 5), (4, 16, 16, 8)):
    y = _latents(shape, dtype, 70 + shape[-1])
    sc = (torch.rand(shape, generator=g) * 16).cuda()
    loc = _loc_of(loc_kind, shape, dtype, 80 + shape[-1])
    calls = _count_routes(monkeypatch, F)
    got = em.compress(y, sc, loc)
    assert got.tolist() == em.compress(y, sc, loc, fused=False).tolist()
    back = em.decompress(got, sc, loc)
    assert calls == {"compress_16bit": 1, "decode_16bit": 1}
    want = em.decompress(got, sc, loc, fused=False)
    assert back.dtype == (torch.float32 if loc_kind == "float32" else dtype) and _same(back, want)


@pytest.mark.parametrize("dtype", DTYPES)
def test_other_operands_keep_the_unfused_path(E, F, monkeypatch, dtype):
  """A float64 loc, a loc broadcast from another shape, and a universal model do not reach the 16-bit entries."""
  from compression_b200 import distributions as D
  em = _loc_scale(E, dtype)
  shape = (2, 3, 4, 5)
  y = _latents(shape, dtype, 90)
  sc = torch.rand(shape, device="cuda") * 16
  calls = _count_routes(monkeypatch, F)
  for loc in (torch.randn(shape, device="cuda", dtype=torch.float64), torch.randn(5, device="cuda").to(dtype)):
    s = em.compress(y, sc, loc)
    assert s.tolist() == em.compress(y, sc, loc, fused=False).tolist()
    assert _same(em.decompress(s, sc, loc), em.decompress(s, sc, loc, fused=False))
  ub = E.UniversalBatchedEntropyModel(D.NoisyLogistic(loc=torch.zeros(8), scale=torch.ones(8)), coding_rank=2,
                                      compression=True, bottleneck_dtype=dtype).cuda()
  yu = _latents((2, 5, 8), dtype, 91, specials=False)
  s = ub.compress(yu)
  assert _same(ub.decompress(s, (5,)), ub.decompress(s, (5,), fused=False))
  assert calls == {}


# ------------------------------------------------------------------------------------------------
# Decoding symbols the quantiser never makes: large escapes in both directions
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_offsets", [False, True])
def test_decode_of_large_escapes(E, F, dtype, with_offsets):
  from compression_b200 import gen_ops
  em = _cfg2_model(E, dtype, with_offsets)
  g = torch.Generator().manual_seed(5)
  sym = torch.randint(-3, 4, (4, 3 * 128), generator=g, dtype=torch.int32)
  big = [65519, 65520, 70000, -65520, (1 << 24) + 3, -(1 << 24) - 5, (1 << 25) + 7, 123456789, -987654321,
         (1 << 30) + 12345, (1 << 31) - 100, -(1 << 31) + 100]
  sym.reshape(-1)[torch.randperm(sym.numel(), generator=g)[:len(big)]] = torch.tensor(big, dtype=torch.int32)
  h = gen_ops.create_range_encoder((4,), em._lookup_host())
  gen_ops.entropy_encode_channel(h, sym.cuda())
  strings = gen_ops.entropy_encode_finalize(h)
  got = em.decompress(strings, (3, 1))
  want = em.decompress(strings, (3, 1), fused=False)
  assert _same(got, want)
  if dtype == torch.float16:
    assert bool(torch.isinf(got).any())
  else:
    assert float(got.float().abs().max()) > 2.0**24


# ------------------------------------------------------------------------------------------------
# Ragged batches
# ------------------------------------------------------------------------------------------------
ENCODERS = [("functional", n) for n in ("compress_f32", "compress_ragged", "encode_channel_f32", "encode_index_f32")] + \
           [("gen_ops", n) for n in ("entropy_encode_channel", "entropy_encode_index")]
DECODERS = [("functional", n) for n in ("decode_ragged", "decode_channel_f32", "decode_index_f32", "decode_16bit",
                                        "decode_ragged_16bit")] + \
           [("gen_ops", n) for n in ("create_range_decoder", "entropy_decode_channel", "entropy_decode_index")]


def _count_coders(monkeypatch):
  from compression_b200 import functional, gen_ops
  mods = {"functional": functional, "gen_ops": gen_ops}
  calls = {"encode": 0, "decode": 0}
  for kind, names in (("encode", ENCODERS), ("decode", DECODERS)):
    for mod, name in names:
      def counted(*a, _fn=getattr(mods[mod], name), _kind=kind, **k):
        calls[_kind] += 1
        return _fn(*a, **k)
      monkeypatch.setattr(mods[mod], name, counted)
  return calls


def _check_ragged(monkeypatch, compress_ragged, decompress_ragged, per_item, items):
  calls = _count_coders(monkeypatch)
  strings, dec = compress_ragged(return_decoded=True)
  assert calls == {"encode": 0, "decode": 0}  # (the 16-bit entries are not in the lists)
  monkeypatch.undo()
  assert strings.tolist() == compress_ragged().tolist() == per_item()
  back = decompress_ragged(strings)
  assert len(dec) == len(back) == len(items)
  for d, b in zip(dec, back):
    assert _same(d, b)
  return dec


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_offsets", [False, True])
def test_ragged_batched(E, monkeypatch, dtype, with_offsets):
  em = _small_batched(E, dtype) if with_offsets else _cfg2_model(E, dtype, False)
  rows = 8 if with_offsets else 128
  ns = [1, 0, 3, 17, 300, 64, 4097 // rows + 1]
  xs = [_latents((n, rows) if with_offsets else (n, 1, rows), dtype, 100 + i) for i, n in enumerate(ns)]
  bshape = lambda x: x.shape[:-1]
  per_item = lambda: [em.compress(x).tolist()[0] if x.numel() else b"" for x in xs]
  dec = _check_ragged(monkeypatch, lambda **k: em.compress_ragged(xs, **k),
                      lambda s: em.decompress_ragged(s, [bshape(x) for x in xs]), per_item, xs)
  for d, x in zip(dec, xs):
    if x.numel():
      assert _same(d, em.decompress(em.compress(x[None]), bshape(x), fused=False)[0])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("loc_kind", [None, "same", "float32"])
def test_ragged_location_scale(E, monkeypatch, dtype, loc_kind):
  em = _loc_scale(E, dtype)
  shapes = [(1, 1, 1), (4, 4, 5), (0, 3, 2), (5, 3, 2), (17, 2, 5), (1, 9, 1), (33, 33, 4)]
  xs = [_latents(s, dtype, 200 + i) for i, s in enumerate(shapes)]
  g = torch.Generator().manual_seed(6)
  sc = [(torch.rand(s, generator=g) * 16).cuda() for s in shapes]
  loc = None if loc_kind is None else [_loc_of(loc_kind, s, dtype, 300 + i) for i, s in enumerate(shapes)]
  li = lambda i: None if loc is None else loc[i]
  per_item = lambda: [em.compress(x, sc[i], li(i)).tolist()[0] if x.numel() else b"" for i, x in enumerate(xs)]
  dec = _check_ragged(monkeypatch, lambda **k: em.compress_ragged(xs, sc, loc, **k),
                      lambda s: em.decompress_ragged(s, sc, loc), per_item, xs)
  for i, (d, x) in enumerate(zip(dec, xs)):
    assert d.dtype == (torch.float32 if loc_kind == "float32" else dtype)
    if x.numel():
      want = em.decompress(em.compress(x[None], sc[i][None], None if li(i) is None else li(i)[None]), sc[i][None],
                           None if li(i) is None else li(i)[None], fused=False)[0]
      assert _same(d, want)


@pytest.mark.parametrize("dtype", DTYPES)
def test_ragged_indexed(E, monkeypatch, dtype):
  em = _indexed(E, dtype)
  shapes = [(3, 5), (1, 1), (40, 7), (0, 3)]
  xs = [_latents(s, dtype, 400 + i) for i, s in enumerate(shapes)]
  g = torch.Generator().manual_seed(7)
  idx = [(torch.rand(s + (2,), generator=g) * torch.tensor([4., 5.])).cuda() for s in shapes]
  per_item = lambda: [em.compress(x, i).tolist()[0] if x.numel() else b"" for x, i in zip(xs, idx)]
  _check_ragged(monkeypatch, lambda **k: em.compress_ragged(xs, idx, **k), lambda s: em.decompress_ragged(s, idx),
                per_item, xs)


# ------------------------------------------------------------------------------------------------
# Full cfg2 size, and the compiled reference coder
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_full_cfg2_size(E, dtype):
  em = _cfg2_model(E, dtype, True)
  y = _latents((256, 16, 16, 128), dtype, 500, scale=3.0)
  got = em.compress(y)
  assert torch.equal(got.offsets_dev, em.compress(y, fused=False).offsets_dev)
  assert got.tolist() == em.compress(y, fused=False).tolist()
  assert _same(em.decompress(got, (16, 16)), em.decompress(got, (16, 16), fused=False))
  items = [y[i] for i in range(256)]
  strings, dec = em.compress_ragged(items, return_decoded=True)
  assert strings.tolist() == got.tolist()
  back = em.decompress(got, (16, 16))
  assert all(_same(d, back[i]) for i, d in enumerate(dec))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["channel", "index"])
def test_strings_match_the_reference_coder(E, dtype, mode):
  """A seeded subset (no saturating values, which the reference's escape loop cannot code) against the compiled
  reference coder on the symbols the unfused path makes."""
  O = oracle.best()
  if mode == "channel":
    em = _cfg2_model(E, dtype, True)
    y = _latents((6, 2, 3, 128), dtype, 600, specials=False)
    strings = em.compress(y)
    coff, qoff = em._flat_tables(y.device)
    sym = em._quantize(y, qoff, coff).reshape(6, -1).cpu().numpy()
    assert strings.tolist() == O.encode(em._lookup_host(), sym)
  else:
    em = _loc_scale(E, dtype)
    shape = (6, 5, 7, 3)
    y = _latents(shape, dtype, 601, specials=False)
    sc = torch.rand(shape, device="cuda") * 16
    loc = _loc_of("same", shape, dtype, 602)
    strings = em.compress(y, sc, loc)
    flat = em._flatten_indexes(em._normalize_indexes(sc.to(em.prior_dtype)))
    sym = em._quantize(y, loc, em.cdf_offset.cuda(), flat).reshape(6, -1).cpu().numpy()
    assert strings.tolist() == O.encode(em._lookup_host(), sym, flat.reshape(6, -1).cpu().numpy())


# ------------------------------------------------------------------------------------------------
# The decode entries' argument checks on a real decoder: no launch
# ------------------------------------------------------------------------------------------------
def test_decode_entries_reject_bad_arguments(E):
  import ctypes as C
  from compression_b200 import _lib, gen_ops
  em = _cfg2_model(E, torch.float16, False)
  strings = em.compress(_latents((2, 1, 1, 128), torch.float16, 700))
  h = gen_ops.create_range_decoder(strings, em._lookup_host())
  L = _lib.lib()
  out = torch.empty(256, dtype=torch.float16, device="cuda")
  coff = em.cdf_offset.cuda()
  loc = torch.zeros(256, dtype=torch.float16, device="cuda")
  idx = torch.zeros(256, dtype=torch.int32, device="cuda")
  offs = np.array([0, 128, 256], dtype=np.int64)
  p = lambda t: C.c_void_p(t.data_ptr())
  n0 = _lib.launch_count()
  bad = [
      lambda: L.tfcb_decode_16bit(h._h, None, p(out), 0, None, 0, p(coff), 128, None),
      lambda: L.tfcb_decode_16bit(h._h, None, p(out), 3, None, 0, p(coff), 128, None),
      lambda: L.tfcb_decode_16bit(h._h, None, p(out), 1, p(loc), 1, p(coff), 128, None),
      lambda: L.tfcb_decode_16bit(h._h, p(idx), p(out), 1, p(loc), 2, p(coff), 128, None),
      lambda: L.tfcb_decode_16bit(h._h, None, p(out), 1, None, 0, None, 128, None),
      lambda: L.tfcb_decode_16bit(h._h, None, None, 1, None, 0, p(coff), 128, None),
      lambda: L.tfcb_decode_16bit(h._h, None, p(out), 1, None, 0, p(coff), -1, None),
      lambda: L.tfcb_decode_ragged_16bit(h._h, offs.ctypes.data_as(C.c_void_p), None, p(out), 2, None, 5, p(coff),
                                         None),
      lambda: L.tfcb_decode_ragged_16bit(h._h, offs.ctypes.data_as(C.c_void_p), None, None, 2, None, 0, p(coff),
                                         None),
      lambda: L.tfcb_decode_ragged_16bit(h._h, np.array([0, 256, 128], dtype=np.int64).ctypes.data_as(C.c_void_p),
                                         None, p(out), 2, None, 0, p(coff), None),
  ]
  for call in bad:
    with pytest.raises(_lib.InvalidArgumentError):
      _lib.check(call())
  assert _lib.launch_count() == n0
  # the handle is untouched: it still decodes
  assert _same(em.decompress(strings, (1, 1)), em.decompress(strings, (1, 1), fused=False))
