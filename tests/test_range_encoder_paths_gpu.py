"""GPU: the range encoder's less travelled paths against the compiled reference coder (oracle.best()).

The encoder leaves carries unresolved: it writes raw 16-bit words and one carry bit per word, and resolves them only
at the end, in enc_write_kernel's carry-lookahead over 32-word groups (cut into kWriteWarps = 8 segments chained
through shared memory) and, for a stream that ends straddling 2^32, in enc_final_length's walk back over the
trailing raw 0xFFFF words.  The streams of carry_streams.py put runs of raw 0xFFFF words around group and segment
boundaries that a carry then crosses ("above"), that stay as they are ("below"), or that finalize walks back over
("straddle"); test_range_encoder_paths_cpu.py shows that each one reaches its state in the reference's string.
Every case here checks that the GPU strings equal the reference's byte for byte, that each side decodes the other's
strings to the symbols, and that every stream passes the sanity check.  The streams go through every encoder entry,
behind odd-length strings (the write kernel's byte path), over several calls on one handle (arena growth with the
run live), and through the host paths of the pooled compress: other CUDA streams, more tables than the table cache
keeps, reuse after an argument error and between ragged and uniform batches, and 1 025 / 70 000 streams.
"""
import functools

import numpy as np
import pytest
import torch

import carry_streams as cs
import oracle
import util

pytestmark = pytest.mark.gpu

CDF3, CDF768 = cs.table_cdf(3), cs.table_cdf(768)
LOOKUP3 = util.make_lookup_1d([CDF3], [16], [False])
LOOKUP768 = util.make_lookup_1d([CDF768], [16], [False])
OTHER = util.laplace_cdf(41, 12, 3.0)  # index mode's second row (overflow)
LOOKUP_IX = util.make_lookup_1d([CDF3, OTHER], [16, 12], [False, True])


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import gen_ops
  return gen_ops


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


def cuda(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@functools.lru_cache(maxsize=None)
def run_cases(ending, width=3):
  """The symbols of every run of carry_streams.runs_for(ending), with a random tail after the "above" and "below"
  runs of unspecified total (so the run does not always end the stream), each with its model string."""
  cdf = cs.table_cdf(width)
  out = []
  for i, (lead, length, total) in enumerate(cs.runs_for(ending)):
    syms, c, _ = cs.run_stream(cdf, ending, i, lead, length, total, tail=0 if i % 2 else 40)
    out.append((syms, c.string()))
  return out


def decode_check(ops, lookup, got, value, index=None):
  """`got` (a Strings): equal to the reference's strings of `value` [S, N] (index [S, N] or None); the GPU decodes
  the reference's strings and the reference decodes `got`, both to `value`, every stream passing the sanity check."""
  O = oracle.best()
  want = O.encode(lookup, value, index)
  assert got.tolist() == want
  hd = ops.create_range_decoder(want, lookup)
  if index is None:
    hd, dec = ops.entropy_decode_channel(hd, [value.shape[1]])
  else:
    hd, dec = ops.entropy_decode_index(hd, cuda(index), [value.shape[1]])
  assert np.array_equal(dec.cpu().numpy().reshape(value.shape), value)
  assert bool(ops.entropy_decode_finalize(hd).all())
  back, ok = O.decode(lookup, want, value.shape[1], index)
  assert np.array_equal(back, value) and ok.all()
  return want


def ragged_check(ops, F, lookup, got, streams, index=None):
  """The ragged form of decode_check: `streams` a list of 1-D symbol arrays (index: matching row arrays or None)."""
  O = oracle.best()
  want = [O.encode(lookup, s[None], None if index is None else index[i][None])[0] if len(s) else b""
          for i, s in enumerate(streams)]
  assert got.tolist() == want
  L = [len(s) for s in streams]
  flat_index = None if index is None else cuda(np.concatenate(index).astype(np.int32))
  dec = F.decode_ragged(ops.create_range_decoder(want, lookup), L, index=flat_index)
  assert np.array_equal(dec.cpu().numpy(), np.concatenate(streams))
  for i, (s, w) in enumerate(zip(streams, got.tolist())):
    if len(s):
      back, ok = O.decode(lookup, [w], len(s), None if index is None else index[i][None])
      assert np.array_equal(back[0], s) and ok.all()
  return want


def batch_of(rng, syms, width=3):
  """A uniform batch around one crafted stream of n symbols: [it, a straddle stream (the string 80), it again, random
  bins], so the crafted string is written at an even and at an odd offset."""
  n = len(syms)
  cdf = cs.table_cdf(width)
  strad = cs.straddle_symbols(cdf, n) if n >= 2 else syms
  return np.stack([syms, strad, syms, rng.integers(0, len(cdf) - 1, n)]).astype(np.int32)


# ------------------------------------------------------------------------------------------------
# 1.-2. Carry chains at the write kernel's group and segment boundaries, at even and odd output offsets
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["channel", "index"])
@pytest.mark.parametrize("ending", cs.ENDINGS)
def test_carry_chains_at_write_boundaries(ops, ending, mode):
  """Each run of carry_streams.runs_for(ending) -- 31, 32 and 33 words at and across group boundaries in streams of
  fewer than 8 groups, one write segment exactly and +- 1, across all 8 segments -- in a batch behind a one-byte
  straddle string, through entropy_encode_channel / entropy_encode_index (the crafted row and an overflow row)."""
  rng = np.random.default_rng(1)
  for syms, model in run_cases(ending):
    value = batch_of(rng, syms)
    index = None
    if mode == "index":
      index = np.zeros_like(value)
      index[3] = rng.integers(0, 2, value.shape[1])
      value[3] = np.where(index[3] == 1, rng.integers(-3, 44, value.shape[1]), value[3])
    h = ops.create_range_encoder([4], LOOKUP3 if index is None else LOOKUP_IX)
    if index is None:
      ops.entropy_encode_channel(h, cuda(value))
    else:
      ops.entropy_encode_index(h, cuda(index), cuda(value))
    got = ops.entropy_encode_finalize(h)
    want = decode_check(ops, LOOKUP3 if index is None else LOOKUP_IX, got, value, index)
    assert want[0] == want[2] == model and want[1] == b"\x80"


# ------------------------------------------------------------------------------------------------
# 3. Every way in: fused float32 and 16-bit compress, ragged (with kModeDecoded), the legacy op
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ending", cs.ENDINGS)
def test_fused_compress(ops, F, ending):
  """compress_f32 (channel and index) with values = symbol + cdf_offset + offset (exact in float32), and
  compress_16bit in float16 and bfloat16 on the 768-wide table (values below 64 in magnitude, exact in both)."""
  rng = np.random.default_rng(2)
  for (syms, _), (syms768, model768) in zip(run_cases(ending), run_cases(ending, 768)):
    value = batch_of(rng, syms)
    S, N = value.shape
    coff = np.asarray([-(len(CDF3) - 1) // 2], np.int32)
    qoff = np.asarray([0.25], np.float32)
    y = (value + coff[0]).astype(np.float32) + qoff[0]
    decode_check(ops, LOOKUP3, F.compress_f32([S], LOOKUP3, cuda(y), cuda(qoff), cuda(coff)), value)
    loc = rng.choice(np.asarray([-0.25, 0.0, 0.25], np.float32), size=(S, N)).astype(np.float32)
    index = np.zeros((S, N), np.int32)
    coff2 = np.asarray([coff[0], -20], np.int32)
    y = (value + coff[0]).astype(np.float32) + loc
    got = F.compress_f32([S], LOOKUP_IX, cuda(y), cuda(loc), cuda(coff2), index=cuda(index))
    decode_check(ops, LOOKUP_IX, got, value, index)

    value = batch_of(rng, syms768, 768)
    S, N = value.shape
    coff = np.asarray([-43], np.int32)
    y = (value + coff[0]).astype(np.float32) + 0.25
    assert np.abs(y).max() < 64
    for dt in (torch.float16, torch.bfloat16):
      got = F.compress_16bit([S], LOOKUP768, cuda(y).to(dt), cuda(np.full(1, 0.25, np.float32)), cuda(coff))
      assert decode_check(ops, LOOKUP768, got, value)[0] == model768
      loc = rng.choice(np.asarray([-0.25, 0.0, 0.25], np.float32), size=(S, N)).astype(np.float32)
      yl = (value + coff[0]).astype(np.float32) + loc
      index = np.zeros((S, N), np.int32)
      got = F.compress_16bit([S], LOOKUP768, cuda(yl).to(dt), cuda(loc).to(dt), cuda(coff), index=cuda(index))
      decode_check(ops, LOOKUP768, got, value, index)


@pytest.mark.parametrize("ending", cs.ENDINGS)
def test_ragged_compress_and_decoded(ops, F, ending):
  """compress_ragged with every run of the ending in one batch, between empty, one-symbol and one-byte straddle
  streams: int32 in channel and index mode, float32 with decoded=True (kModeDecoded: the decoded values are the
  exact dequantised symbols), and compress_ragged_16bit with decoded=True on the 768-wide table."""
  rng = np.random.default_rng(3)
  for width in (3, 768):
    cdf = cs.table_cdf(width)
    lookup = LOOKUP3 if width == 3 else LOOKUP768
    streams, models = [], []
    for syms, model in run_cases(ending, width):
      streams += [np.zeros(0, np.int32), syms, rng.integers(0, len(cdf) - 1, 1).astype(np.int32),
                  cs.straddle_symbols(cdf, 40), syms]
      models += [b"", model, None, b"\x80", model]
    L = [len(s) for s in streams]
    flat = np.concatenate(streams).astype(np.int32)
    coff = np.asarray([-(len(cdf) - 1) // 2], np.int32)
    y = (flat + coff[0]).astype(np.float32) + 0.25
    if width == 3:
      want = ragged_check(ops, F, lookup, F.compress_ragged(lookup, L, cuda(flat)), streams)
      assert all(m is None or m == w for m, w in zip(models, want))
      index = [np.zeros(len(s), np.int32) for s in streams]  # (the crafted row of the two-row table)
      ragged_check(ops, F, LOOKUP_IX, F.compress_ragged(LOOKUP_IX, L, cuda(flat), index=cuda(np.concatenate(index))),
                   streams, index)
      got, dec = F.compress_ragged(lookup, L, cuda(y), quant_offset=cuda(np.full(1, 0.25, np.float32)),
                                   cdf_offset=cuda(coff), decoded=True)
      assert ragged_check(ops, F, lookup, got, streams) == want
      assert torch.equal(dec.cpu(), torch.from_numpy(y))
    else:
      for dt in (torch.float16, torch.bfloat16):
        got, dec = F.compress_ragged_16bit(lookup, L, cuda(y).to(dt), cuda(np.full(1, 0.25, np.float32)),
                                           cuda(coff), decoded=True)
        want = ragged_check(ops, F, lookup, got, streams)
        assert all(m is None or m == w for m, w in zip(models, want))
        assert torch.equal(dec.cpu(), torch.from_numpy(y).to(dt))


@pytest.mark.parametrize("ending", cs.ENDINGS)
def test_legacy_range_encode(ops, ending):
  """RangeEncode (one warp, legacy_encode_kernel, the same drain and write kernel) on every run: int16 data in the
  crafted 21 846-bin table, against the reference's op and the model; both decoders read the strings back."""
  O = oracle.best()
  cdf = CDF3[None]
  for syms, model in run_cases(ending):
    data = syms.astype(np.int16)
    got = ops.range_encode(cuda(data), cuda(cdf), 16)
    assert got == O.range_encode(data, cdf, 16) == model
    assert np.array_equal(O.range_decode(got, data.shape, cdf, 16), data)
    assert np.array_equal(ops.range_decode(got, list(data.shape), cuda(cdf), 16).cpu().numpy(), data)


# ------------------------------------------------------------------------------------------------
# 4. Multi-call handles: arena growth with runs and carry bits live, a carry across the call boundary
# ------------------------------------------------------------------------------------------------
def test_multi_call_growth_with_live_carries(ops):
  """A stream of several runs split over calls on one handle.  The first cut leaves 288 words (a multiple of 32)
  in the middle of a run that a carry crosses in the next call, which grows the arena (enc_grow_kernel) with those
  288 words and the carry bits of the earlier runs live; the last call grows it again with about 700 words live.  Against the reference
  encoder fed the same chunks, with a straddle stream and a random one beside it."""
  spec = [(3, 40, "above"), (60, 100, "below"), (200, 31, "above"), (260, 64, "above"), (400, 600, "above"),
          (1100, 300, "straddle")]
  syms, c, runs = cs.carry_stream(7, CDF3, spec)
  words = []
  replay = cs.Coder(CDF3)
  for k in syms:
    replay.encode(int(k))
    words.append(replay.words)
  words = np.asarray(words)
  cut1 = int(np.argmax(words == 288)) + 1  # inside the run of words 261..324, at a group boundary
  cut2 = int(np.argmax(words == 700)) + 1  # inside the run of words 401..1000
  cut3 = cut2 + 1
  bounds = [0, cut1, cut2, cut3, len(syms)]
  chunks = [b - a for a, b in zip(bounds, bounds[1:])]
  assert words[cut1 - 1] == 288 and all(n > 0 for n in chunks)
  rng = np.random.default_rng(4)
  value = np.stack([syms, cs.straddle_symbols(CDF3, len(syms)), rng.integers(0, len(CDF3) - 1, len(syms))])
  value = value.astype(np.int32)
  O = oracle.best()
  enc = O.encoder(LOOKUP3, 3)
  h = ops.create_range_encoder([3], LOOKUP3)
  for a, b in zip(bounds, bounds[1:]):
    enc.encode(value[:, a:b])
    ops.entropy_encode_channel(h, cuda(value[:, a:b]))
  want = enc.finalize()
  enc.close()
  got = ops.entropy_encode_finalize(h)
  assert got.tolist() == want and want[0] == c.string() and want[1] == b"\x80"
  hd = ops.create_range_decoder(got, LOOKUP3)
  for a, b in zip(bounds, bounds[1:]):
    hd, dec = ops.entropy_decode_channel(hd, [b - a])
    assert np.array_equal(dec.cpu().numpy(), value[:, a:b])
  assert bool(ops.entropy_decode_finalize(hd).all())


# ------------------------------------------------------------------------------------------------
# 5. Host paths of the pooled compress
# ------------------------------------------------------------------------------------------------
def _crafted_batch(rng, S):
  """[S, n] symbols of the crafted table: the canonical run with each ending, straddle and random streams."""
  n = 700
  rows = [cs.canonical_symbols(CDF3, n, e) for e in cs.ENDINGS]
  rows += [rng.integers(0, len(CDF3) - 1, n).astype(np.int32) for _ in range(S - len(rows))]
  return np.stack(rows[:S]).astype(np.int32)


def test_compress_on_several_cuda_streams(ops, F):
  """Compresses of the same stream count on three torch.cuda.Streams, interleaved without synchronising, so the
  pooled encoders move between streams behind their `done` events; every string is checked after one device
  synchronisation."""
  rng = np.random.default_rng(5)
  streams = [torch.cuda.Stream() for _ in range(3)]
  jobs = []
  for i in range(12):
    value = _crafted_batch(rng, 4)
    value = np.roll(value, i, axis=0)
    jobs.append((value, cuda(value)))
  torch.cuda.synchronize()
  outs = []
  for i, (value, dev) in enumerate(jobs):
    with torch.cuda.stream(streams[i % 3]):
      if i % 2:
        outs.append(F.compress_ragged(LOOKUP3, [value.shape[1]] * 4, dev.reshape(-1)))
      else:
        y = dev.to(torch.float32) - 10922.0
        outs.append(F.compress_f32([4], LOOKUP3, y, torch.zeros(1, device="cuda"),
                                   torch.full((1,), -10922, dtype=torch.int32, device="cuda")))
  torch.cuda.synchronize()
  for (value, _), got in zip(jobs, outs):
    decode_check(ops, LOOKUP3, got, value)


def test_more_tables_than_the_cache_keeps(ops, F):
  """20 distinct tables (the crafted row and an overflow row of 10 to 29 bins) in turn, at stream counts 2, 3, 5 and
  6 so that pooled encoders still pin some tables, then the first ones again (evicted and uploaded anew); decoders
  share the cache."""
  rng = np.random.default_rng(6)
  for rnd in range(2):
    for t in list(range(20)) + [0, 1, 2, 3]:
      lookup = util.make_lookup_1d([CDF3, util.laplace_cdf(10 + t, 12, 2.0)], [16, 12], [False, True])
      S = (2, 3, 5, 6)[t % 4]
      value = _crafted_batch(rng, max(S, 3))[:S]
      index = np.zeros_like(value)
      index[-1] = rng.integers(0, 2, value.shape[1])
      value[-1] = np.where(index[-1] == 1, rng.integers(-2, 12 + t, value.shape[1]), value[-1])
      got = F.compress_ragged(lookup, [value.shape[1]] * S, cuda(value).reshape(-1), index=cuda(index).reshape(-1))
      if rnd == 0 or t < 4:
        decode_check(ops, lookup, got, value, index)
      else:
        assert got.tolist() == oracle.best().encode(lookup, value, index)


def test_pooled_encoder_after_an_argument_error(ops, F):
  """A compress that fails with an argument error leaves its pooled encoder clean for the next compress of the same
  stream count: a symbol out of range found by the kernel (after a crafted run was coded), and a missing cdf_offset
  found on the host."""
  rng = np.random.default_rng(7)
  S = 5
  for bad in ("value", "cdf_offset"):
    value = _crafted_batch(rng, S)
    if bad == "value":
      v = value.copy()
      v[2, -3] = len(CDF3) - 1 + 5
      with pytest.raises(ops.InvalidArgumentError, match="not in range"):
        F.compress_ragged(LOOKUP3, [v.shape[1]] * S, cuda(v).reshape(-1))
    else:
      with pytest.raises(ops.InvalidArgumentError, match="cdf_offset"):
        F.compress_ragged(LOOKUP3, [value.shape[1]] * S, cuda(value).reshape(-1).to(torch.float32))
    for _ in range(2):
      decode_check(ops, LOOKUP3, F.compress_ragged(LOOKUP3, [value.shape[1]] * S, cuda(value).reshape(-1)), value)
      decode_check(ops, LOOKUP3, F.compress_f32([S], LOOKUP3, cuda(value).to(torch.float32) - 10922.0,
                                                torch.zeros(1, device="cuda"),
                                                torch.full((1,), -10922, dtype=torch.int32, device="cuda")), value)


def test_pooled_encoder_between_ragged_and_uniform(ops, F):
  """One stream count (7) used ragged, then uniform with longer streams, then ragged with a larger arena, then
  uniform again: prepare_ragged reallocates the arena and sets the uniform capacity it leaves behind."""
  rng = np.random.default_rng(8)
  S = 7
  for n_r, n_u in ((60, 900), (2500, 300), (5, 3000)):
    streams = [cs.canonical_symbols(CDF3, max(2, int(rng.integers(1, n_r + 1))), e)
               for e in (cs.ENDINGS * 3)[:S]]
    streams[3] = np.zeros(0, np.int32)
    ragged_check(ops, F, LOOKUP3, F.compress_ragged(LOOKUP3, [len(s) for s in streams],
                                                    cuda(np.concatenate(streams))), streams)
    value = np.stack([cs.canonical_symbols(CDF3, n_u, e) for e in (cs.ENDINGS * 3)[:S]])
    decode_check(ops, LOOKUP3, F.compress_ragged(LOOKUP3, [n_u] * S, cuda(value).reshape(-1)), value)
    decode_check(ops, LOOKUP3, F.compress_f32([S], LOOKUP3, cuda(value).to(torch.float32),
                                              torch.zeros(1, device="cuda"), torch.zeros(1, dtype=torch.int32,
                                                                                         device="cuda")), value)


# ------------------------------------------------------------------------------------------------
# 6. Stream counts beyond one offsets block and one CTA per stream
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1025, 70000])
def test_many_streams(ops, F, S):
  """Ragged batches of 1 025 and 70 000 streams, most of 0 to 24 random symbols, with crafted streams (every
  ending, long and short, and one-byte straddle strings) at the ends and around the offsets kernel's 1 024-stream
  blocks; and a uniform batch (one encoder handle) of S streams of 24 symbols whose crafted ones are canonical
  runs."""
  rng = np.random.default_rng(S)
  O = oracle.best()
  lengths = rng.integers(0, 25, S)
  streams = [rng.integers(0, len(CDF3) - 1, n).astype(np.int32) for n in lengths]
  crafted = [0, 1, 1023, 1024, S // 2, S - 2, S - 1]
  for j, at in enumerate(crafted):
    e = cs.ENDINGS[j % 3]
    streams[at] = cs.canonical_symbols(CDF3, 1500 if j % 2 else 24, e)
  strings = F.compress_ragged(LOOKUP3, [len(s) for s in streams], cuda(np.concatenate(streams))).tolist()
  want = [b""] * S
  by_len = {}
  for i, s in enumerate(streams):
    by_len.setdefault(len(s), []).append(i)
  for n, ids in by_len.items():
    if n:
      for i, w in zip(ids, O.encode(LOOKUP3, np.stack([streams[i] for i in ids]), threads=8)):
        want[i] = w
  assert strings == want
  dec = F.decode_ragged(ops.create_range_decoder(want, LOOKUP3), [len(s) for s in streams])
  assert np.array_equal(dec.cpu().numpy(), np.concatenate(streams))

  N = 24
  value = rng.integers(0, len(CDF3) - 1, (S, N)).astype(np.int32)
  for j, at in enumerate(crafted):
    value[at] = cs.canonical_symbols(CDF3, N, cs.ENDINGS[j % 3])
  h = ops.create_range_encoder([S], LOOKUP3)
  ops.entropy_encode_channel(h, cuda(value))
  got = ops.entropy_encode_finalize(h)
  want = O.encode(LOOKUP3, value, threads=8)
  assert got.tolist() == want
  assert [want[i][:1] for i in crafted] == [b"\x80", b"\x7f", b"\x80"] * 2 + [b"\x80"]
  hd = ops.create_range_decoder(want, LOOKUP3)
  hd, dec = ops.entropy_decode_channel(hd, [N])
  assert np.array_equal(dec.cpu().numpy(), value) and bool(ops.entropy_decode_finalize(hd).all())
  back, ok = O.decode(LOOKUP3, got.tolist(), N, threads=8)
  assert np.array_equal(back, value) and ok.all()
