"""GPU: decode_kernel's less travelled paths against the compiled reference coder (oracle.best()).

The fused decoder (DESIGN §3.2) relies on invariants of the key table `DeviceLookup::upload` builds: a 64-key window
around each row's median, rows with zero-width bins at either end marked irregular and sent to the slow path,
`search_row` treating a c' = 0 key as below, and a word ring kept kRingAhead words ahead of the chain warp.  The
cases here build the table shapes that reach those paths -- search keys in global memory (the 10 `SMEM = false`
instantiations), zero-width and one-bin rows, precisions 1 to 16, escape-saturated streams, channel mode at odd row
counts and out-of-range indexes -- and check, per case, that the GPU strings equal the reference's byte for byte,
that each side decodes the other's strings to the input symbols, and that every stream passes the sanity check.

Only symbols inside the reference encoder's domain are coded: bins of nonzero width, and escape payloads (the
Elias-gamma value) below 2^30.
"""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
import util

pytestmark = pytest.mark.gpu

SMEM_LIMIT = 200 * 1024  # launch_decode keeps keys and row records in shared memory up to this many bytes
# decode_kernel's modes (range_coder.cu: kModeIndex 1, kModeF32 2, kModeH16 8, kModeB16 16, kModeLocF32 32), the 10
# that `with_mode<false>` compiles
DECODE_MODES = {0, 1, 2, 3, 8, 9, 8 | 1 | 32, 16, 17, 16 | 1 | 32}


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import gen_ops
  return gen_ops


@pytest.fixture(scope="module")
def F():
  from compression_b200 import functional
  return functional


# ------------------------------------------------------------------------------------------------
# Helpers: tables with zero-width bins, key-table sizes, launched kernels
# ------------------------------------------------------------------------------------------------
def cdf_with_empty_bins(rng, n_bins, precision, empty=(), peaky=1.0):
  """CDF of `n_bins` bins at `precision` whose bins listed in `empty` have zero width; every other bin is >= 1.
  `empty` may name leading, interior (single or runs), trailing, or all but one of the bins."""
  empty = np.unique(np.asarray(list(empty), dtype=np.int64))
  keep = np.setdiff1d(np.arange(n_bins), empty)
  assert keep.size >= 1
  pmf = np.zeros(n_bins, np.int64)
  pmf[keep] = np.diff(util.random_cdf(rng, keep.size, precision, peaky=peaky))
  return np.concatenate([[0], np.cumsum(pmf)]).astype(np.int32)


def window_start(cdf, precision):
  """First key index of the row's 64-key search window, as DeviceLookup::upload places it (median - 31, clamped to
  [1, n - 63])."""
  n = len(cdf) - 1
  median = next((e for e in range(1, n + 1) if cdf[e] >= (1 << precision) // 2), n)
  return max(1, min(median - 31, n - 63))


def as_parsed(cdf):
  """The row as the lookup grammar reads it: it ends at its first 2^p, so zero-width bins at the end of a CDF are
  padding (an overflow row's last nonzero bin is then its escape bin)."""
  return cdf[:int(np.argmax(cdf == cdf[-1])) + 1]


def key_table_bytes(cdfs):
  """What launch_decode compares with its shared-memory limit: per row max(ncdf - 1, 64) + 1 keys of 8 B, a 64-key
  all-zero window, the key block rounded up to 16 B, and a 16 B record per row."""
  keys = sum(max(len(as_parsed(c)) - 1, 64) + 1 for c in cdfs) + 64
  return (8 * keys + 15) // 16 * 16 + 16 * len(cdfs)


FILLER_LIVE = 48  # the filler row's bins that are coded


def filler_cdf(seed, n_bins):
  """A regular p = 16 row of `n_bins` bins whose first FILLER_LIVE bins (the only ones coded) are the same for every
  `n_bins`: they hold 2^15, the other bins are one wide except the last.  Two tables that differ only in this row's
  width code the same symbols into the same strings.  The median is the last live bin's upper end, so the search
  window covers the upper part of the live bins and the lower ones take the slow path."""
  head = util.random_cdf(np.random.default_rng(seed), FILLER_LIVE, 15)
  t = n_bins - FILLER_LIVE
  assert 1 <= t <= 1 << 15
  tail = (1 << 15) + np.concatenate([np.arange(1, t), [1 << 15]])
  cdf = np.concatenate([head, tail])
  assert np.all(np.diff(cdf) >= 1) and cdf[-1] == 1 << 16
  return cdf.astype(np.int32)


def pad_to_key_bytes(cdfs, precs, ovf, target, seed=0):
  """Appends one filler row (filler_cdf) so that the decoder's key table takes exactly `target` bytes."""
  n_rows = len(cdfs) + 1
  keys = (target - 16 * n_rows) // 8
  assert (target - 16 * n_rows) % 16 == 0
  n = keys - 64 - sum(max(len(as_parsed(c)) - 1, 64) + 1 for c in cdfs) - 1
  assert 64 <= n <= 30000, n
  out = list(cdfs) + [filler_cdf(seed, n)]
  assert key_table_bytes(out) == target
  return out, list(precs) + [16], list(ovf) + [False]


def decode_kernels(fn):
  """Runs `fn` under torch.profiler; returns (its result, the set of (MODE, SMEM) of the decode_kernel launches).
  Called in a fresh process (fresh_kernels).  A session of a process that has profiled before can miss device
  events, so one that recorded no decode_kernel launch is taken again, at most twice: `fn` must be repeatable."""
  from torch.profiler import ProfilerActivity, profile
  seen = set()
  for _ in range(3):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      out = fn()
      torch.cuda.synchronize()
    for e in prof.events():
      m = re.search(r"\bdecode_kernel<(?:\(\w+\))?(\d+),\s*(true|false)>", e.name)
      if m:
        seen.add((int(m.group(1)), m.group(2) == "true"))
    if seen:
      break
  return out, seen


def rows_of(n_rows, S, N, index, chunks=None):
  """Each position's row: `index`, or in channel mode j % n_rows with j counted from 0 in each call of `chunks`."""
  if index is not None:
    return index
  return np.concatenate([np.broadcast_to(np.arange(n) % n_rows, (S, n)) for n in (chunks or [N])], axis=1)


def uniform_symbols(rng, cdfs, ovf, rows, esc_prob=0.25, esc_lo=-20, esc_hi=10):
  """Per position a symbol drawn uniformly over its row's nonzero bins (the escape bin excluded); on overflow rows
  with a nonzero escape bin, an escape with probability `esc_prob`: a value in [esc_lo, -1] or [n - 1, n - 1 +
  esc_hi].  Rows are taken as parsed (as_parsed)."""
  out = np.empty(rows.shape, np.int32)
  for r, c in enumerate(cdfs):
    c = as_parsed(c)
    at = rows == r
    k = int(at.sum())
    if not k:
      continue
    n = len(c) - 1
    width = np.diff(c)
    live = np.flatnonzero(width[:n - 1] if ovf[r] else width)
    v = rng.choice(live, size=k) if live.size else np.zeros(k, np.int64)
    if ovf[r] and width[-1] > 0:
      esc = rng.random(k) < (esc_prob if live.size else 1.0)
      big = np.where(rng.random(k) < 0.5, rng.integers(esc_lo, 0, size=k), rng.integers(n - 1, n + esc_hi, size=k))
      v = np.where(esc, big, v)
    out[at] = v
  return out


def check_round_trip(ops, lookup, value, index=None, chunks=None):
  """The case's four checks: GPU strings == reference strings, GPU decode of the reference strings and reference
  decode of the GPU strings give `value`, every stream passes the sanity check.  `chunks`: the calls' symbol counts
  on one handle (default one call).  Returns the strings."""
  O = oracle.best()
  S, N = value.shape
  chunks = [N] if chunks is None else chunks
  assert sum(chunks) == N
  enc = O.encoder(lookup, S)
  h = ops.create_range_encoder([S], lookup)
  at = 0
  for n in chunks:
    v = np.ascontiguousarray(value[:, at:at + n])
    i = None if index is None else np.ascontiguousarray(index[:, at:at + n])
    enc.encode(v, i)
    if i is None:
      ops.entropy_encode_channel(h, torch.from_numpy(v).cuda())
    else:
      ops.entropy_encode_index(h, torch.from_numpy(i).cuda(), torch.from_numpy(v).cuda())
    at += n
  want = enc.finalize()
  enc.close()
  got = ops.entropy_encode_finalize(h)
  assert got.tolist() == want
  hd = ops.create_range_decoder(want, lookup)
  dec_o = O.decoder(got.tolist(), lookup)
  at = 0
  for n in chunks:
    i = None if index is None else np.ascontiguousarray(index[:, at:at + n])
    if i is None:
      hd, dec = ops.entropy_decode_channel(hd, [n])
    else:
      hd, dec = ops.entropy_decode_index(hd, torch.from_numpy(i).cuda(), [n])
    assert np.array_equal(dec.cpu().numpy(), value[:, at:at + n]), f"GPU decode of call at {at} ({n} symbols)"
    assert np.array_equal(dec_o.decode(n, i), value[:, at:at + n]), f"reference decode of call at {at}"
    at += n
  assert bool(ops.entropy_decode_finalize(hd).all())
  assert dec_o.finalize().all()
  dec_o.close()
  return want


# ------------------------------------------------------------------------------------------------
# 1. Both sides of the 200 KB shared-memory choice, every decode mode
# ------------------------------------------------------------------------------------------------
def _smem_case():
  """Narrow rows (every |symbol + cdf_offset| < 64, so the float and 16-bit values below are exact in float16 and
  bfloat16) and the symbols of a 4 x 777 batch in channel and index mode."""
  rng = np.random.default_rng(2024)
  sizes = [1, 2, 3, 7, 17, 33, 40, 60, 12, 5]
  precs = [int(rng.integers(max(1, int(np.ceil(np.log2(max(n, 1))))), 17)) for n in sizes]
  cdfs = [util.random_cdf(rng, n, p, peaky=3.0) for n, p in zip(sizes, precs)]
  ovf = [i % 2 == 1 or sizes[i] == 1 for i in range(len(sizes))]
  return rng, cdfs, precs, ovf


def _smem_operands(target):
  """The 200 KB case at key-table size `target`: (lookup, operands, the reference's strings, exact values)."""
  _, cdfs0, precs0, ovf0 = _smem_case()
  O = oracle.best()
  S, N = 4, 777
  cdfs, precs, ovf = pad_to_key_bytes(cdfs0, precs0, ovf0, target, seed=5)
  R = len(cdfs)
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  drng = np.random.default_rng(31)  # the same symbols for both tables
  index = drng.integers(0, R, size=(S, N)).astype(np.int32)
  coded = cdfs[:-1] + [cdfs[-1][:FILLER_LIVE + 1]]  # symbols only in the filler's live bins
  sym_ch = uniform_symbols(drng, coded, ovf, rows_of(R, S, N, None))
  sym_ix = uniform_symbols(drng, coded, ovf, index)
  coff = np.asarray([-((len(c) - 1) // 2) for c in coded], np.int32)
  qoff = drng.choice(np.asarray([-0.25, 0.0, 0.25], np.float32), size=R).astype(np.float32)
  loc = drng.choice(np.asarray([-0.25, 0.0, 0.25], np.float32), size=(S, N)).astype(np.float32)
  rows_ch = rows_of(R, S, N, None)
  assert np.abs(sym_ch + coff[rows_ch]).max() < 64 and np.abs(sym_ix + coff[index]).max() < 64
  y_ch = ((sym_ch + coff[rows_ch]).astype(np.float32) + qoff[rows_ch]).astype(np.float32)
  y_ix = ((sym_ix + coff[index]).astype(np.float32) + loc).astype(np.float32)
  # ragged: prefixes of streams 0..2 with empty streams between them
  L = [N, 0, N // 3, 0, N - 5]
  src = [0, None, 1, None, 2]

  def ragged(a):
    return np.concatenate([a[s, :n] for s, n in zip(src, L) if n])

  d = dict(sym_ch=sym_ch, sym_ix=sym_ix, index=index, coff=coff, qoff=qoff, loc=loc, y_ch=y_ch, y_ix=y_ix, lengths=L,
           r_ch=ragged(sym_ch), r_ix=ragged(sym_ix), r_index=ragged(index), r_loc=ragged(loc), r_y_ch=ragged(y_ch),
           r_y_ix=ragged(y_ix), s_ch=O.encode(lookup, sym_ch), s_ix=O.encode(lookup, sym_ix, index),
           ref_r_ch=[O.encode(lookup, sym_ch[s:s + 1, :n])[0] if n else b"" for s, n in zip(src, L)],
           ref_r_ix=[O.encode(lookup, sym_ix[s:s + 1, :n], index[s:s + 1, :n])[0] if n else b""
                     for s, n in zip(src, L)])
  return lookup, d


def _decode_every_mode(ops, F, lookup, d, profile=False):
  """Every public decode entry on the strings in `d`; returns ({entry: output on the host}, {entry: kernels} when
  `profile`)."""
  outs, kernels = {}, {}

  def run(name, fn):
    if profile:
      outs[name], kernels[name] = decode_kernels(fn)
    else:
      outs[name] = fn()
    outs[name] = outs[name].cpu()

  dev = "cuda"
  S, N = d["sym_ch"].shape
  idx = torch.from_numpy(d["index"]).to(dev)
  coff = torch.from_numpy(d["coff"]).to(dev)
  qoff = torch.from_numpy(d["qoff"]).to(dev)
  loc = torch.from_numpy(d["loc"]).to(dev)
  ridx = torch.from_numpy(d["r_index"]).to(dev)
  rloc = torch.from_numpy(d["r_loc"]).to(dev)
  L = d["lengths"]

  def fresh(key):
    return ops.create_range_decoder(d[{"r_ch": "ref_r_ch", "r_ix": "ref_r_ix"}.get(key, key)], lookup)

  run("int32 channel", lambda: ops.entropy_decode_channel(fresh("s_ch"), [N])[1])
  run("int32 index", lambda: ops.entropy_decode_index(fresh("s_ix"), idx, [N])[1])
  run("int32 ragged channel", lambda: F.decode_ragged(fresh("r_ch"), L))
  run("int32 ragged index", lambda: F.decode_ragged(fresh("r_ix"), L, index=ridx))
  run("f32 channel", lambda: F.decode_channel_f32(fresh("s_ch"), (S, N), qoff, coff))
  run("f32 index", lambda: F.decode_index_f32(fresh("s_ix"), idx, loc, coff))
  run("f32 ragged channel", lambda: F.decode_ragged(fresh("r_ch"), L, quant_offset=qoff, cdf_offset=coff))
  run("f32 ragged index", lambda: F.decode_ragged(fresh("r_ix"), L, index=ridx, quant_offset=rloc, cdf_offset=coff))
  for dt in (torch.float16, torch.bfloat16):
    t = str(dt).split(".")[1]
    run(f"{t} channel", lambda dt=dt: F.decode_16bit(fresh("s_ch"), (S, N), dt, qoff, coff))
    run(f"{t} index", lambda dt=dt: F.decode_16bit(fresh("s_ix"), None, dt, loc.to(dt), coff, index=idx))
    run(f"{t} index f32 loc", lambda dt=dt: F.decode_16bit(fresh("s_ix"), None, dt, loc, coff, index=idx))
    run(f"{t} ragged channel", lambda dt=dt: F.decode_ragged_16bit(fresh("r_ch"), L, dt, qoff, coff))
    run(f"{t} ragged index", lambda dt=dt: F.decode_ragged_16bit(fresh("r_ix"), L, dt, rloc.to(dt), coff, index=ridx))
    run(f"{t} ragged index f32 loc",
        lambda dt=dt: F.decode_ragged_16bit(fresh("r_ix"), L, dt, rloc, coff, index=ridx))
  return outs, kernels


# the mode each entry must launch (H16 / B16 added per type below)
ENTRY_MODES = {"int32 channel": 0, "int32 index": 1, "int32 ragged channel": 0, "int32 ragged index": 1,
               "f32 channel": 2, "f32 index": 3, "f32 ragged channel": 2, "f32 ragged index": 3,
               "channel": 0, "index": 1, "index f32 loc": 1 | 32, "ragged channel": 0, "ragged index": 1,
               "ragged index f32 loc": 1 | 32}


def _entry_mode(name):
  t, rest = name.split(" ", 1)
  if t in ("float16", "bfloat16"):
    return ENTRY_MODES[rest] | (8 if t == "float16" else 16)
  return ENTRY_MODES[name]


def profile_cases():
  """The decode_kernel instantiations each profiled case launches: {case: {entry: [[MODE, SMEM], ...]}}, for the
  200 KB case at both sizes and test_zero_width_bins' four decodes.  Run in a fresh process (fresh_kernels)."""
  from compression_b200 import functional, gen_ops
  out = {}
  for target in (SMEM_LIMIT, SMEM_LIMIT + 16):
    lookup, d = _smem_operands(target)
    out[f"smem {target}"] = _decode_every_mode(gen_ops, functional, lookup, d, profile=True)[1]
  for mode in ("channel", "index"):
    for smem in (True, False):
      lookup, value, index = _zero_width_case(mode, smem)
      strings = oracle.best().encode(lookup, value, index)

      def dec(strings=strings, lookup=lookup, index=index, n=[value.shape[1]]):
        hd = gen_ops.create_range_decoder(strings, lookup)
        if index is None:
          return gen_ops.entropy_decode_channel(hd, n)
        return gen_ops.entropy_decode_index(hd, torch.from_numpy(index).cuda(), n)

      out[f"zero {mode} {smem}"] = {"decode": decode_kernels(dec)[1]}
  return {case: {k: sorted(v) for k, v in kernels.items()} for case, kernels in out.items()}


@pytest.fixture(scope="module")
def fresh_kernels():
  """profile_cases() in a fresh Python process.  In a process that has profiled before (a whole-suite run), a
  torch.profiler session can come back without device events; a fresh process records them."""
  import json
  here = os.path.dirname(os.path.abspath(__file__))
  env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
  code = "import json, test_range_decoder_paths_gpu as T; print(json.dumps(T.profile_cases()))"
  r = subprocess.run([sys.executable, "-s", "-B", "-c", code], env=env, cwd=here, capture_output=True, text=True,
                     timeout=900)
  assert r.returncode == 0, r.stderr[-4000:]
  cases = json.loads(r.stdout.strip().splitlines()[-1])
  return {case: {k: {(int(m), bool(t)) for m, t in v} for k, v in kernels.items()} for case, kernels in cases.items()}


def test_search_keys_in_shared_and_global_memory_every_mode(ops, F, fresh_kernels):
  """Tables of exactly 200 KB (the largest shared-memory launch) and 200 KB + 16 B (keys read from global memory):
  the profiler shows `decode_kernel<M, true>` for the first and `<M, false>` for the second, for each of the 10
  decode modes, through int32 channel / index, float32, ragged (with zero-length streams) and float16 / bfloat16
  entries (float32 loc included).  Both tables code the same symbols into the same strings (the reference's); every
  decoded value is the exact one (the values are exact in every type), the same at both sizes, and equal to what the
  ragged encoders return as their decoded output."""
  results = {}
  for target in (SMEM_LIMIT, SMEM_LIMIT + 16):
    lookup, d = _smem_operands(target)
    L = d["lengths"]
    assert check_round_trip(ops, lookup, d["sym_ch"]) == d["s_ch"]
    assert check_round_trip(ops, lookup, d["sym_ix"], d["index"]) == d["s_ix"]
    assert F.compress_ragged(lookup, L, torch.from_numpy(d["r_ch"]).cuda()).tolist() == d["ref_r_ch"]
    assert F.compress_ragged(lookup, L, torch.from_numpy(d["r_ix"]).cuda(),
                             index=torch.from_numpy(d["r_index"]).cuda()).tolist() == d["ref_r_ix"]
    outs, _ = _decode_every_mode(ops, F, lookup, d)
    kernels = fresh_kernels[f"smem {target}"]
    assert kernels.keys() == outs.keys()
    smem = target <= SMEM_LIMIT
    for name, k in kernels.items():
      assert k == {(_entry_mode(name), smem)}, (target, name, k)
    assert {m for k in kernels.values() for m, _ in k} == DECODE_MODES
    sym_ch, sym_ix, y_ch, y_ix = d["sym_ch"], d["sym_ix"], d["y_ch"], d["y_ix"]
    r_y_ch, r_y_ix = d["r_y_ch"], d["r_y_ix"]
    r_ch, r_ix, ref_r_ch, ref_r_ix = d["r_ch"], d["r_ix"], d["ref_r_ch"], d["ref_r_ix"]
    coff, qoff, r_loc, r_index, s_ch, s_ix = (d[k] for k in ("coff", "qoff", "r_loc", "r_index", "s_ch", "s_ix"))

    # exact expected values
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))  # noqa: E731
    want = {"int32 channel": t(sym_ch), "int32 index": t(sym_ix), "int32 ragged channel": t(r_ch),
            "int32 ragged index": t(r_ix), "f32 channel": t(y_ch), "f32 index": t(y_ix),
            "f32 ragged channel": t(r_y_ch), "f32 ragged index": t(r_y_ix)}
    for dt in (torch.float16, torch.bfloat16):
      n = str(dt).split(".")[1]
      want.update({f"{n} channel": t(y_ch).to(dt), f"{n} index": t(y_ix).to(dt), f"{n} index f32 loc": t(y_ix),
                   f"{n} ragged channel": t(r_y_ch).to(dt), f"{n} ragged index": t(r_y_ix).to(dt),
                   f"{n} ragged index f32 loc": t(r_y_ix)})
    assert want.keys() == outs.keys()
    for name, w in want.items():
      assert outs[name].dtype == w.dtype and torch.equal(outs[name], w), (target, name)

    # the encoders' decoded outputs (float32 and 16-bit ragged encodes of the same values)
    coff_d = t(coff).cuda()
    qoff_d, r_loc_d, r_index_d = t(qoff).cuda(), t(r_loc).cuda(), t(r_index).cuda()
    s, dec = F.compress_ragged(lookup, L, t(r_y_ch).cuda(), quant_offset=qoff_d, cdf_offset=coff_d, decoded=True)
    assert s.tolist() == ref_r_ch and torch.equal(dec.cpu(), outs["f32 ragged channel"])
    s, dec = F.compress_ragged(lookup, L, t(r_y_ix).cuda(), quant_offset=r_loc_d, cdf_offset=coff_d,
                               index=r_index_d, decoded=True)
    assert s.tolist() == ref_r_ix and torch.equal(dec.cpu(), outs["f32 ragged index"])
    for dt in (torch.float16, torch.bfloat16):
      n = str(dt).split(".")[1]
      s, dec = F.compress_ragged_16bit(lookup, L, t(r_y_ch).to(dt).cuda(), qoff_d, coff_d, decoded=True)
      assert s.tolist() == ref_r_ch and torch.equal(dec.cpu(), outs[f"{n} ragged channel"])
      for key, lo in ((f"{n} ragged index", r_loc_d.to(dt)), (f"{n} ragged index f32 loc", r_loc_d)):
        s, dec = F.compress_ragged_16bit(lookup, L, t(r_y_ix).to(dt).cuda(), lo, coff_d, index=r_index_d,
                                         decoded=True)
        assert s.tolist() == ref_r_ix and torch.equal(dec.cpu(), outs[key]), key
    results[target] = (s_ch, s_ix, outs)

  (a_ch, a_ix, a_out), (b_ch, b_ix, b_out) = results[SMEM_LIMIT], results[SMEM_LIMIT + 16]
  assert a_ch == b_ch and a_ix == b_ix
  for name in a_out:
    assert torch.equal(a_out[name], b_out[name]), name


# ------------------------------------------------------------------------------------------------
# 2. Zero-width bins (irregular rows and interior ties); 3. one-bin rows
# ------------------------------------------------------------------------------------------------
def _settle(build, place):
  """Builds a row whose empty bins `place(wfirst)` sit at fixed offsets of its own search window (the window moves
  with the empty bins): iterates to a fixed point."""
  wfirst = None
  for _ in range(20):
    cdf = build(place(wfirst))
    w = window_start(cdf[0], cdf[1])
    if w == wfirst:
      return cdf
    wfirst = w
  raise AssertionError("window placement did not settle")


def zero_width_rows(seed):
  """(cdfs, precisions, overflow, description) of rows with zero-width bins: leading (1, 2, many), interior (at the
  median, at both edges of the 64-key window, runs across its edges), trailing, all bins but one; narrow (< 64
  bins) and wide (up to 4000 bins) rows.  Trailing zero-width bins cannot be written in a lookup: the grammar ends a
  row at its first 2^p and reads the rest as padding (range_coder_kernels.cc:130-134, range_coder.cu's scan_row), so
  such a row codes as the shorter row (as_parsed), and an overflow row's last nonzero bin becomes its escape bin;
  the reference and the GPU must read them alike."""
  rng = np.random.default_rng(seed)
  rows = []

  def add(n, p, empty, o, what, peaky=1.0):
    rows.append((cdf_with_empty_bins(rng, n, p, empty, peaky), p, o, what))

  for o in (False, True):
    add(40, 12, [0], o, "leading 1")
    add(40, 12, [0, 1], o, "leading 2")
    add(40, 12, range(25), o, "leading 25")
    add(40, 12, [19, 20], o, "interior at the median")
    add(40, 12, [5, 17, 18, 30], o, "interior")
    add(40, 12, [38] if o else [39], o, "trailing 1")
    add(40, 12, range(33, 39) if o else range(33, 40), o, "trailing run")
    add(40, 12, [i for i in range(40) if i != 11], o, "all but one")
    add(300, 16, range(3), o, "leading, wide", peaky=4.0)
    add(4000, 16, range(150), o, "leading many, wide (several search rounds)", peaky=4.0)
    add(4000, 16, range(3990, 3999) if o else range(3990, 4000), o, "trailing, wide", peaky=4.0)
  add(40, 12, [39], True, "overflow row with an empty escape bin (read as 39 bins)")
  add(40, 12, [10, 39], True, "the same with an interior empty bin")
  add(3, 4, [0, 2], True, "one live bin after an empty one, escape empty (read as an all-escape row)")
  # interior empty bins at the window's edges (keys wfirst and wfirst + 63 are bins wfirst - 1 / wfirst and
  # wfirst + 62 / wfirst + 63), and runs across them
  for n, p, off in ((200, 14, lambda w: [w - 1, w, w + 62, w + 63]),
                    (200, 14, lambda w: list(range(w - 3, w + 3)) + list(range(w + 60, w + 66))),
                    (1500, 16, lambda w: [w - 1, w + 31, w + 63]),
                    (1500, 16, lambda w: list(range(w - 4, w + 2)))):
    for o in (False, True):
      def build(empty, n=n, p=p, o=o):
        return cdf_with_empty_bins(np.random.default_rng(seed + n + len(rows)), n, p, empty, 2.0), p

      cdf, _ = _settle(build, lambda w, off=off: [] if w is None else off(w))
      w = window_start(cdf, p)
      assert np.diff(cdf)[w - 1] == 0  # the key just left of the window equals the window's first key
      rows.append((cdf, p, o, f"interior at the window edges (wfirst {w})"))
  return [r[0] for r in rows], [r[1] for r in rows], [r[2] for r in rows], [r[3] for r in rows]


def _zero_width_case(mode, smem):
  """(lookup, value, index) of test_zero_width_bins."""
  cdfs, precs, ovf, _ = zero_width_rows(40)
  if not smem:
    cdfs, precs, ovf = pad_to_key_bytes(cdfs, precs, ovf, SMEM_LIMIT + 16)
  assert (key_table_bytes(cdfs) <= SMEM_LIMIT) == smem
  rng = np.random.default_rng(41 if mode == "channel" else 42)
  R = len(cdfs)
  S, N = 6, 60 * R + 17
  index = rng.integers(0, R, (S, N)).astype(np.int32) if mode == "index" else None
  rows = rows_of(R, S, N, index)
  value = uniform_symbols(rng, cdfs, ovf, rows, esc_prob=0.05, esc_lo=-3000, esc_hi=3000)
  # wide rows cannot have every bin hit: half their symbols go to the nonzero bins next to an empty one
  for r, c in enumerate(cdfs):
    c = as_parsed(c)
    width = np.diff(c)[:len(c) - 1 - ovf[r]]
    empty = np.flatnonzero(width == 0)
    near = np.unique(np.clip(empty[:, None] + np.arange(-2, 3), 0, width.size - 1))
    near = near[width[near] > 0]
    at = np.flatnonzero((rows == r).reshape(-1) & (rng.random(S * N) < 0.5))
    if len(c) > 65 and near.size:
      value.reshape(-1)[at] = rng.choice(near, size=at.size)
  return util.make_lookup_1d(cdfs, precs, ovf), value, index


@pytest.mark.parametrize("smem", [True, False], ids=["shared", "global"])
@pytest.mark.parametrize("mode", ["channel", "index"])
def test_zero_width_bins(ops, fresh_kernels, mode, smem):
  """Rows with leading / interior / trailing / all-but-one zero-width bins, narrow and wide, regular and overflow,
  with the keys in shared and in global memory: uniform symbols over the nonzero bins (every bin of the narrow rows
  is hit; on the wide rows half the symbols are next to an empty bin), and escapes."""
  lookup, value, index = _zero_width_case(mode, smem)
  check_round_trip(ops, lookup, value, index)
  assert fresh_kernels[f"zero {mode} {smem}"]["decode"] == {(1 if mode == "index" else 0, smem)}


def test_one_bin_rows(ops):
  """[p, 0, 2^p]: a regular one-bin row codes its symbol in zero bits (a stream made of it alone is empty); an
  overflow one-bin row escapes every value (max_value = 0), here 0, -1, 1 and the largest payloads below 2^30
  (2^30 - 2 and -(2^30 - 1)); both mixed with ordinary rows in channel and index mode."""
  big = (1 << 30) - 1
  for p in (1, 5, 16):
    lookup = util.make_lookup_1d([np.asarray([0, 1 << p], np.int32)], [p], [False])
    strings = check_round_trip(ops, lookup, np.zeros((3, 500), np.int32), chunks=[1, 128, 371])
    assert all(len(s) == 0 for s in strings)
    lookup = util.make_lookup_1d([np.asarray([0, 1 << p], np.int32)], [p], [True])
    v = np.asarray([0, -1, 1, big - 1, -big, 2, -2, 77], np.int32)
    check_round_trip(ops, lookup, np.tile(v, (2, 40)))
  rng = np.random.default_rng(43)
  cdfs = [np.asarray([0, 1 << 16], np.int32), np.asarray([0, 1 << 3], np.int32), util.random_cdf(rng, 20, 12),
          np.asarray([0, 2], np.int32), util.laplace_cdf(41, 15, 5.0), np.asarray([0, 1 << 16], np.int32)]
  precs = [16, 3, 12, 1, 15, 16]
  ovf = [False, True, True, True, False, True]
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  for mode in ("channel", "index"):
    S, N = 5, 1500
    chunks = [N - 129, 129]
    index = rng.integers(0, len(cdfs), (S, N)).astype(np.int32) if mode == "index" else None
    rows = rows_of(len(cdfs), S, N, index, chunks)
    value = uniform_symbols(rng, cdfs, ovf, rows, esc_prob=0.3)
    one = np.asarray([len(c) == 2 and o for c, o in zip(cdfs, ovf)])[rows]
    value[one] = rng.choice(np.asarray([0, -1, 1, big - 1, -big], np.int32), size=int(one.sum()))
    check_round_trip(ops, lookup, value, index, chunks)


# ------------------------------------------------------------------------------------------------
# 4. Every precision 1..16, regular and overflow, in one mixed-precision table
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["channel", "index"])
def test_every_precision_in_one_table(ops, mode):
  """Rows at p = 1..16, once regular and once overflow, with as many bins as the precision allows up to 40 (p = 1:
  one or two bins), in one table; the keys are c << (32 - p) and c = 2^p is {0xFFFFFFFF, 0}."""
  rng = np.random.default_rng(44 if mode == "channel" else 45)
  cdfs, precs, ovf = [], [], []
  for p in range(1, 17):
    for o in (True, False):  # (a regular row's 2^p before the next row's +p' would read as its padding)
      n = min(40, 1 << p) if p > 1 else 1 + int(o)
      cdfs.append(util.random_cdf(rng, n, p, peaky=2.0))
      precs.append(p)
      ovf.append(o)
  assert not util.ambiguous_1d(precs, ovf)
  R = len(cdfs)
  S, N = 7, 40 * R + 3
  index = rng.integers(0, R, (S, N)).astype(np.int32) if mode == "index" else None
  chunks = [N - 300, 300]
  value = uniform_symbols(rng, cdfs, ovf, rows_of(R, S, N, index, chunks), esc_prob=0.2, esc_lo=-500, esc_hi=500)
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  check_round_trip(ops, lookup, value, index, chunks)


# ------------------------------------------------------------------------------------------------
# 5. Escape-saturated streams at the ring bound
# ------------------------------------------------------------------------------------------------
ESC_LOOKUP = util.make_lookup_1d([np.asarray([0, (1 << 16) - 1, 1 << 16], np.int32)], [16], [True])
CALLS = [1, 127, 128, 129, 255, 257, 1151]  # 2048 symbols per stream


def _densest_words(strings, n):
  """Words (16 bit) per 256 symbols of the densest stream, from the string lengths of streams of `n` uniformly
  costly symbols."""
  return max(len(s) for s in strings) / 2 * 256 / n


def test_escape_saturated_streams_at_the_ring_bound(ops):
  """Every symbol escapes through a width-1 escape bin at p = 16 (16 bits) with an Elias-gamma payload in
  [2^29, 2^30) (29 zeros, 30 bits, a sign: 60 bits): 76 bits = 4.75 words per symbol, 1 216 words per 256 symbols
  (two groups), the most any code the reference can write reaches (its payloads stay below 2^30).  kRingAhead =
  1 536 has to cover two groups.  Decoded in one call (16 groups, the ring refilled inside the kernel) and in calls
  of 1, 127, 128, 129, 255, 257 and 1 151 symbols on one handle (refilled from the saved position).  Then the int32
  extremes, an extension the reference cannot code (round trip and sanity only): INT32_MIN's payload 2^31 takes 80
  bits, 1 280 words per 256 symbols."""
  rng = np.random.default_rng(46)
  S, N = 4, sum(CALLS)
  mag = rng.integers(1 << 29, 1 << 30, size=(S, N))  # the payload: v - 1 + 1 for v >= 1, -v for v < 0
  value = np.where(rng.random((S, N)) < 0.5, mag, -mag).astype(np.int32)
  strings = check_round_trip(ops, ESC_LOOKUP, value)
  words = _densest_words(strings, N)
  assert words >= 1200, words
  assert check_round_trip(ops, ESC_LOOKUP, value, chunks=CALLS) == strings

  # special symbols at group positions 0, 1, 126, 127, 128 of every call and in a run, ordinary ones elsewhere
  value2 = np.zeros((S, N), np.int32)
  at = 0
  for n in CALLS:
    for k in [0, 1, 126, 127, 128] + list(range(40, 80)) + list(range(250, 260)):
      if k < n:
        value2[:, at + k] = value[:, at + k]
    at += n
  check_round_trip(ops, ESC_LOOKUP, value2, chunks=CALLS)

  # INT32_MIN / INT32_MAX: the GPU coder only
  ext = np.where(rng.random((S, N)) < 0.5, np.iinfo(np.int32).min, np.iinfo(np.int32).max).astype(np.int32)
  ext[0] = np.iinfo(np.int32).min
  h = ops.create_range_encoder([S], ESC_LOOKUP)
  ops.entropy_encode_channel(h, torch.from_numpy(ext).cuda())
  s = ops.entropy_encode_finalize(h)
  ext_words = _densest_words(s.tolist(), N)
  assert ext_words >= 1279, ext_words
  for chunks in ([N], CALLS):
    hd = ops.create_range_decoder(s, ESC_LOOKUP)
    at = 0
    for n in chunks:
      hd, dec = ops.entropy_decode_channel(hd, [n])
      assert np.array_equal(dec.cpu().numpy(), ext[:, at:at + n])
      at += n
    assert bool(ops.entropy_decode_finalize(hd).all())


# ------------------------------------------------------------------------------------------------
# 6. Channel mode at other row counts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_rows", [31, 32, 33, 100, 129, 1000])
def test_channel_mode_row_counts(ops, n_rows):
  """The prepare warp walks rows as (lane + 32 k) % n_rows, the resolve warp as j % n_rows: row counts around the
  warp width and beyond a group, N a multiple of neither n_rows nor 128, several calls per handle (the row restarts
  at 0 in every call)."""
  rng = np.random.default_rng(47 + n_rows)
  precs = [int(rng.integers(5, 17)) for _ in range(n_rows)]
  cdfs = [util.random_cdf(rng, int(rng.integers(1, 24)), p, peaky=2.0) for p in precs]
  ovf = [bool(rng.random() < 0.4) for _ in range(n_rows)]
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  N = 3 * n_rows + 211
  assert N % n_rows and N % 128
  S = 3
  chunks = [n_rows + 5, 129, N - n_rows - 134]
  value = np.concatenate([uniform_symbols(rng, cdfs, ovf, rows_of(n_rows, S, n, None), esc_prob=0.1)
                          for n in chunks], axis=1)
  check_round_trip(ops, lookup, value, chunks=chunks)


# ------------------------------------------------------------------------------------------------
# 7. The decoder's index check
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("second_call", [False, True], ids=["first_call", "second_call"])
@pytest.mark.parametrize("pos", [0, 127, 128, -1], ids=["at0", "at127", "at128", "last"])
@pytest.mark.parametrize("bad", ["minus_one", "n_rows"])
def test_decoder_index_out_of_range(ops, bad, pos, second_call):
  """An index of -1 or n_rows on the decoder side is an argument error: entropy_decode_finalize raises it with the
  stream and the call-relative element; the next decode on a fresh handle is correct."""
  rng = np.random.default_rng(48)
  cdfs, precs, ovf = [util.random_cdf(rng, 9, 10), util.laplace_cdf(21, 12, 3.0), util.random_cdf(rng, 3, 6)], \
      [10, 12, 6], [False, True, False]
  lookup = util.make_lookup_1d(cdfs, precs, ovf)
  S, N = 3, 300
  index = rng.integers(0, 3, (S, N)).astype(np.int32)
  value = uniform_symbols(rng, cdfs, ovf, index)
  first = 100
  strings = check_round_trip(ops, lookup, value, index, chunks=[first, N - first])
  if second_call:
    bad_index, j = index[:, first:].copy(), pos % (N - first)
  else:
    bad_index, j = index.copy(), pos % N
  stream, v = 1, -1 if bad == "minus_one" else 3
  bad_index[stream, j] = v
  hd = ops.create_range_decoder(strings, lookup)
  if second_call:
    hd, _ = ops.entropy_decode_index(hd, torch.from_numpy(np.ascontiguousarray(index[:, :first])).cuda(), [first])
    hd, _ = ops.entropy_decode_index(hd, torch.from_numpy(bad_index).cuda(), [N - first])
  else:
    hd, _ = ops.entropy_decode_index(hd, torch.from_numpy(bad_index).cuda(), [N])
  msg = re.escape(f"index={v} not in range [0, 3) (stream {stream}, element {j})")
  with pytest.raises(ops.InvalidArgumentError, match=msg):
    ops.entropy_decode_finalize(hd)
  hd = ops.create_range_decoder(strings, lookup)
  hd, dec = ops.entropy_decode_index(hd, torch.from_numpy(index).cuda(), [N])
  assert np.array_equal(dec.cpu().numpy(), value) and bool(ops.entropy_decode_finalize(hd).all())
