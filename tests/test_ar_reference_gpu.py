"""GPU: the autoregressive prior's kernels (functional.ar_*) against the CPU references of oracle/ar_oracle.py.

The parameter network equals an exact float32 emulation of the kernel's documented order bit for bit, at every
depth from 6 to 384 (the uneven slice splits at M = 6, 18, 30 and 42 included) and at every border case of the
causal taps, and stays within the derived bound of a float64 restatement.  The encoder equals the emulated encoder
loop, in one launch or in ranges.  Table indexes follow the entropy model at their edges (negative, past the table,
infinite, NaN, and a num_scales below the tables' rows).  The decoder is checked on the paths the encoder/decoder
round trips of test_mbt2018_gpu do not reach: search keys in global memory, M = 384 in shared memory, escapes of up
to 32 magnitude bits with every channel of a position escaping, and decodes split into short launches."""
import math

import numpy as np
import pytest
import torch

from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from oracle import ar_oracle as A

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
SHAPES = [(1, 1), (1, 4), (4, 1), (2, 2), (3, 5), (6, 9)]
DEPTHS = [6, 12, 18, 30, 42, 96, 192, 384]
SMEM_LIMIT = 200 * 1024  # kArSmemLimit: dynamic shared memory of the decode step beside its ring


def _scale_fn(num_scales, scale_max=256.):
  offset = math.log(.11)
  factor = (math.log(scale_max) - offset) / (num_scales - 1.)
  return lambda i: torch.exp(offset + factor * i)


def _model(num_scales):
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, num_scales, _scale_fn(num_scales), coding_rank=3,
                                            compression=True).to("cuda")


@pytest.fixture(scope="module")
def em():
  return _model(NUM_SCALES)


def _weights(M, seed):
  """test_mbt2018_gpu._weights, on the CPU: loc of a few units and scale indexes spread over the table range."""
  g = torch.Generator().manual_seed(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: torch.randn(*s, generator=g)
  b3 = torch.cat([0.5 * r(M), 24 + 4 * r(M)])
  return [r(5, 5, M, 2 * M) / math.sqrt(12 * M), 0.1 * r(2 * M), r(4 * M, n3) / math.sqrt(4 * M), 0.1 * r(n3),
          r(n3, n4) / math.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * M) / math.sqrt(n4), b3]


def _pack(ws):
  return F.ar_pack_weights(*[w.cuda() for w in ws])


def _forced_scales(ws, scale):
  """The weights with W3's scale columns zeroed and b3's scale half set to `scale` [M]: every position's scale_index
  is then exactly `scale` (b + (+0) + ... + (+0); only -0 becomes +0)."""
  M = ws[0].shape[2]
  ws = [w.clone() for w in ws]
  ws[6][:, M:] = 0
  ws[7][M:] = torch.as_tensor(scale, dtype=torch.float32)
  return ws


def _latents(B, H, W, M, seed):
  g = torch.Generator().manual_seed(seed)
  return 3 * torch.randn(B, H, W, M, generator=g), torch.randn(B, H, W, 2 * M, generator=g)


def _cpu(t):
  return t.detach().cpu().contiguous() if isinstance(t, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(t))


def _assert_bitwise(got, want, what):
  """Equal bits, except that any NaN equals any NaN (the GPU's float arithmetic returns the canonical NaN)."""
  got = _cpu(got)
  want = _cpu(want).reshape(got.shape)
  diff = got.view(torch.int32) != want.view(torch.int32)
  if got.is_floating_point():
    diff &= ~(torch.isnan(got) & torch.isnan(want))
  bad = diff.nonzero()
  assert bad.numel() == 0, (f"{what}: {bad.shape[0]} of {got.numel()} differ; first at {bad[0].tolist()}: "
                            f"{got[tuple(bad[0])].item()!r} vs {want[tuple(bad[0])].item()!r}")


def _key_bytes(em):
  """The decode step's search keys and row records in bytes, with range_coder.cu's arithmetic: every row holds
  max(ncdf - 1, 64) + 1 keys of 8 bytes, the table ends with a 64-key zero window, and each row has a 16-byte record."""
  lk = em._lookup_host()
  ncdf, i = [], 0
  while i < len(lk):
    top = 1 << abs(int(lk[i]))
    j = i + 1
    while lk[j] != top:
      j += 1
    ncdf.append(j - i)
    i = j + 1
  pairs = sum(max(n - 1, 64) + 1 for n in ncdf) + 64
  return ((pairs * 8 + 15) & ~15) + 16 * len(ncdf)


def _act_bytes(M):
  return 608 * M // 3  # ar_act_floats: 152 M / 3 floats of taps, [psi, ctx], h1, h2, out and slice partials


# ---------------------------------------------------------------------------------------------------------------
# a. the parameter network: bitwise to the emulation, within the bound of float64
# ---------------------------------------------------------------------------------------------------------------
def _positions(M, H, W):
  if M <= 96:
    return list(range(H * W))
  if H * W > 15:
    return None
  # deep networks: the first row, first and last columns, and one interior position of each shape
  return sorted({p for p in range(H * W) if p < W or p % W in (0, W - 1)} | {(H // 2) * W + W // 2})


@pytest.mark.parametrize("M", DEPTHS)
def test_params_are_the_float32_emulation_bit_for_bit(M):
  B = 3
  ws = _weights(M, M)
  packed = _pack(ws)
  for k, (H, W) in enumerate(SHAPES):
    pos = _positions(M, H, W)
    if pos is None:
      continue
    y_hat, psi = _latents(B, H, W, M, 10 * M + k)
    yd, pd = y_hat.cuda(), psi.cuda()
    got = [F.ar_params(packed, yd, pd, p, NUM_SCALES) for p in pos]
    got = [torch.stack([g[i] for g in got], 1).cpu() for i in range(3)]  # [B, P, M]
    want = A.params32(ws, y_hat, psi, pos, NUM_SCALES)
    for name, g, w in zip(("loc", "scale_index", "index"), got, want):
      _assert_bitwise(g, w, f"M={M} {H}x{W} {name}")
    for g, e, b in zip(got, A.params64(ws, y_hat, psi, pos), A.bound64(ws, y_hat, psi, pos)):
      assert np.all(np.abs(g.double().numpy() - e) <= b), (M, H, W)


# ---------------------------------------------------------------------------------------------------------------
# b. the encoder loop
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [6, 30, 96])
def test_encoder_is_the_emulated_encoder_loop(M):
  B = 3
  ws = _weights(M, M + 1)
  packed = _pack(ws)
  for k, (H, W) in enumerate([(1, 1), (1, 4), (4, 1), (3, 5)]):
    y, psi = _latents(B, H, W, M, 20 * M + k)
    y[torch.rand(y.shape, generator=torch.Generator().manual_seed(k)) < 0.02] *= 500  # a few escapes
    got = F.ar_encode(packed, y.cuda(), psi.cuda(), NUM_SCALES, scale_index=True)
    want = A.encode32(ws, y, psi, NUM_SCALES)
    for name, g, w in zip(("y_hat", "loc", "index", "scale_index"), got, want):
      _assert_bitwise(g, w, f"M={M} {H}x{W} {name}")


def test_encoder_in_ranges_equals_one_call():
  M, B, H, W = 30, 2, 3, 5
  packed = _pack(_weights(M, 3))
  y, psi = (t.cuda() for t in _latents(B, H, W, M, 4))
  one = F.ar_encode(packed, y, psi, NUM_SCALES, scale_index=True)
  y_hat = torch.zeros_like(y)
  parts = [torch.zeros_like(t).view(B, H * W, M) for t in one[1:]]
  # 1, 2 and 7 positions, empty ranges, ranges starting mid-row (3, 11), y_hat carried from call to call
  for a, b in ((0, 1), (1, 3), (3, 3), (3, 10), (10, 10), (10, 11), (11, 13), (13, 15), (15, 15)):
    out = F.ar_encode(packed, y, psi, NUM_SCALES, y_hat=y_hat, p_begin=a, p_end=b, scale_index=True)
    assert out[0].data_ptr() == y_hat.data_ptr()
    for part, t in zip(parts, out[1:]):
      part[:, a:b] = t.view(B, H * W, M)[:, a:b]
  for name, g, w in zip(("y_hat", "loc", "index", "scale_index"), [y_hat] + parts, one):
    _assert_bitwise(g, w, name)


# ---------------------------------------------------------------------------------------------------------------
# c. table indexes at their edges
# ---------------------------------------------------------------------------------------------------------------
def _edges(ns):
  return [-math.inf, -1e30, -1.5, -0.0, 0.0, 0.49, ns - 1, ns - 0.5, ns, 1e30, math.inf, math.nan]


@pytest.mark.parametrize("num_scales", [64, 17])
def test_table_indexes_at_their_edges_code_and_decode(em, num_scales):
  M, B, H, W = 30, 2, 3, 4
  edges = _edges(NUM_SCALES)  # against the 64-row tables: with num_scales=17 they clamp to 16
  scale = torch.tensor((edges * 3)[:M], dtype=torch.float32)
  ws = _forced_scales(_weights(M, 5), scale)
  packed = _pack(ws)
  y, psi = _latents(B, H, W, M, 6)
  yd, pd = y.cuda(), psi.cuda()
  y_hat, loc, index, sc = F.ar_encode(packed, yd, pd, num_scales, scale_index=True)
  want = A.encode32(ws, y, psi, num_scales)
  for name, g, w in zip(("y_hat", "loc", "index", "scale_index"), (y_hat, loc, index, sc), want):
    _assert_bitwise(g, w, name)
  # scale_index is b3 itself (-0 -> +0), the index the oracle's and, at 64 scales, the entropy model's conversion
  expect = torch.where(scale == 0, torch.zeros_like(scale), scale)
  _assert_bitwise(sc.cpu(), expect.expand(B, H, W, M).contiguous(), "scale_index = b3")
  idx = torch.from_numpy(A.table_index(expect.numpy(), num_scales)).expand(B, H, W, M)
  assert torch.equal(index.cpu(), idx)
  assert int(index.max()) == num_scales - 1 and int(index.min()) == 0
  if num_scales == NUM_SCALES:
    assert torch.equal(em._flatten_indexes(em._normalize_indexes(sc)), index)
  strings = F.compress_f32((B,), em._lookup_host(), yd, loc, em.cdf_offset, index=index)
  _check_decode(em, packed, strings, pd, num_scales, y_hat)


def _check_decode(em, packed, strings, psi, num_scales, want):
  """The device decode loop and the naive host loop both give `want` bit for bit, and every stream ends good."""
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  got = F.ar_decode(handle, packed, psi, num_scales, em.cdf_offset)
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  _assert_bitwise(got, want, "ar_decode")
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  naive = F.ar_decode_naive(handle, packed, psi, num_scales, em.cdf_offset)
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  _assert_bitwise(naive, want, "ar_decode_naive")


def _round_trip(em, packed, y, psi, num_scales):
  y_hat, loc, index = F.ar_encode(packed, y, psi, num_scales)
  strings = F.compress_f32((y.shape[0],), em._lookup_host(), y, loc, em.cdf_offset, index=index)
  _check_decode(em, packed, strings, psi, num_scales, y_hat)
  return y_hat, index


# ---------------------------------------------------------------------------------------------------------------
# d. decoder paths
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def em_wide():
  return _model(160)  # 160 rows over the default scale range: search keys that do not fit beside the activations


@pytest.mark.parametrize("M", [96, 192])
@pytest.mark.parametrize("shape", [(1, 1), (16, 24)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_decoder_with_search_keys_in_global_memory(em_wide, M, shape):
  assert _act_bytes(M) + _key_bytes(em_wide) > SMEM_LIMIT + 32 * 1024, (_act_bytes(M), _key_bytes(em_wide))
  packed = _pack(_weights(M, 7))
  y, psi = (t.cuda() for t in _latents(2, *shape, M, 8))
  _round_trip(em_wide, packed, y, psi, 160)


def test_decoder_at_the_largest_depth_keeps_its_keys_in_shared_memory(em):
  M = 384
  need = _act_bytes(M) + _key_bytes(em)
  assert 190 * 1024 < need <= SMEM_LIMIT, need
  packed = _pack(_weights(M, 9))
  y, psi = (t.cuda() for t in _latents(2, 3, 4, M, 10))
  y[1, 0, 0, :8] = torch.tensor([1e5, -1e5, 65520, -65519, 7e6, 1e9, -2e9, 3e9])
  _round_trip(em, packed, y, psi, NUM_SCALES)


ESCAPES = [65519, 65520, -65520, 70000, (1 << 24) + 4, -(1 << 24) - 4, (1 << 30) + 12288, -(1 << 30) - 12288,
           (1 << 31) - 128, -(1 << 31) + 128, -(1 << 31), 3e9, -3e9]  # float32 latents; ±3e9 saturate q


def test_decoder_with_escapes_of_every_size(em):
  """Image 0 is all zeros (a short string); in image 1 every channel of the first row escapes with |q| from 65 519
  to the saturated 2^31 - 1, hundreds of words per position, so the ring is refilled several times in a row."""
  M, B, H, W = 192, 2, 4, 6
  packed = _pack(_weights(M, 11))
  y, psi = _latents(B, H, W, M, 12)
  y[0] = 0
  g = torch.Generator().manual_seed(13)
  big = torch.tensor(ESCAPES, dtype=torch.float32)
  y[1, 0] = big[torch.randint(0, len(ESCAPES), (W, M), generator=g)]
  some = torch.rand(H - 1, W, M, generator=g) < 0.05
  y[1, 1:][some] = big[torch.randint(0, len(ESCAPES), (int(some.sum()),), generator=g)]
  y, psi = y.cuda(), psi.cuda()
  y_hat, _ = _round_trip(em, packed, y, psi, NUM_SCALES)
  assert float(y_hat[1, 0].abs().min()) >= 65000 and float(y_hat[1, 0].abs().max()) >= 2.0**31
  assert bool((y_hat[0].abs() < 16).all())


def test_decoder_with_32_bit_escape_codes(em):
  """Symbols coded straight into an index-mode stream, with each channel's table forced: every channel of the first
  positions escapes with symbol -2^31 (an Elias-gamma code of 32 magnitude bits, the longest there is), 2^31 - 1
  and -2^31 + 1.  The decoded latent is float(int32(symbol + cdf_offset)) + loc, loc from the decoded latents."""
  M, B, H, W = 192, 2, 3, 4
  rows = torch.arange(M) % NUM_SCALES
  ws = _forced_scales(_weights(M, 14), rows.float() + 0.25)
  packed = _pack(ws)
  _, psi = _latents(B, H, W, M, 15)
  psi = psi.cuda()
  coff = em.cdf_offset.to(torch.int32).cpu()
  index = rows.expand(B, H * W, M).to(torch.int32).contiguous()
  g = torch.Generator().manual_seed(16)
  sym = -coff[index] + torch.randint(-2, 3, index.shape, generator=g, dtype=torch.int32)  # q in [-2, 2]
  sym[0] = -coff[index[0]]  # image 0: all latents zero
  extreme = torch.tensor([-(1 << 31), (1 << 31) - 1, -(1 << 31) + 1], dtype=torch.int32)
  sym[1, :W] = extreme[torch.arange(W * M) % 3].view(W, M)
  h = gen_ops.create_range_encoder((B,), em._lookup_host())
  gen_ops.entropy_encode_index(h, index.cuda(), sym.cuda())
  strings = gen_ops.entropy_encode_finalize(h)
  # the expected latents, position by position: the kernel's parameters at the decoded latents
  want = torch.zeros(B, H, W, M, device="cuda")
  flat = want.view(B, H * W, M)
  q = (sym.to(torch.int64) + coff[index].to(torch.int64) + 2**31) % 2**32 - 2**31  # int32 wrap-around
  for p in range(H * W):
    loc, _, idx = F.ar_params(packed, want, psi, p, NUM_SCALES)
    assert torch.equal(idx.cpu(), index[:, p])
    flat[:, p] = q[:, p].to(torch.int32).float().cuda() + loc
  _check_decode(em, packed, strings, psi, NUM_SCALES, want)


def test_decoder_in_short_launches_mixed_with_naive_steps(em):
  M, B, H, W = 96, 3, 5, 7
  packed = _pack(_weights(M, 17))
  y, psi = (t.cuda() for t in _latents(B, H, W, M, 18))
  y_hat_enc, loc, index = F.ar_encode(packed, y, psi, NUM_SCALES)
  strings = F.compress_f32((B,), em._lookup_host(), y, loc, em.cdf_offset, index=index)
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = torch.zeros_like(y)
  flat = y_hat.view(B, H * W, M)
  # device launches of 1, 2 and 7 positions; naive steps (ar_params + decode_index_f32) at 10, 14, 22 and 23
  steps = [(0, 1), (1, 3), (3, 10), 10, (11, 12), (12, 14), 14, (15, 22), 22, 23, (24, 25), (25, 27), (27, 34),
           (34, 35)]
  for s in steps:
    if isinstance(s, int):
      l, _, i = F.ar_params(packed, y_hat, psi, s, NUM_SCALES)
      flat[:, s] = F.decode_index_f32(handle, i, l, em.cdf_offset)
    else:
      F.ar_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset, y_hat=y_hat, p_begin=s[0], p_end=s[1])
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  _assert_bitwise(y_hat, y_hat_enc, "split decode")
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  _assert_bitwise(F.ar_decode(handle, packed, psi, NUM_SCALES, em.cdf_offset), y_hat_enc, "one launch")
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
