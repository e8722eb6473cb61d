"""The carry-chain streams of test_range_encoder_paths_gpu.py (carry_streams.py) against the reference coder
(oracle.best()): the big-integer model codes them into the reference's strings, and each stream reaches the state
it is built for -- the run of raw 0xFFFF words, resolved to 0x0000 by a carry ("above"), left as 0xFFFF ("below"),
or walked back over by finalize ("straddle").  So the GPU tests are known to hit what they claim."""
import numpy as np
import pytest

import carry_streams as cs
import oracle
import util

ENDINGS = cs.ENDINGS


def lookup_of(width):
  return util.make_lookup_1d([cs.table_cdf(width)], [16], [False])


def check_runs(s, c, runs):
  """The stream's string `s` (the reference's) and the model's coder `c` after it: every run is a run of raw 0xFFFF
  words that ends as its ending says."""
  raw, res = c.raw, c.resolved()
  for r in runs:
    assert r.length >= 1 and all(raw[w] == 0xFFFF for w in r.words), (r.lead, r.length)
    assert raw[r.lead] != 0xFFFF
    body = s[2 * (r.lead + 1):2 * (r.lead + 1 + r.length)]
    if r.ending == "above":  # the carry crosses the whole run into the lead word
      assert all(res[w] == 0 for w in r.words) and res[r.lead] == raw[r.lead] + 1
      assert body == bytes(2 * r.length)
      assert s[2 * r.lead:2 * r.lead + 2] == res[r.lead].to_bytes(2, "big")
    elif r.ending == "below":
      assert all(res[w] == raw[w] for w in r.words) and res[r.lead] == raw[r.lead]
      assert body == b"\xff" * (2 * r.length)
    else:  # finalize walks back over the whole run and ends the string in the lead word
      assert c.straddles() and c.words == r.lead + 1 + r.length
      assert len(s) in (2 * r.lead + 1, 2 * r.lead + 2)
      assert s[2 * r.lead:] == ((raw[r.lead] + 1) << 16 >> 16).to_bytes(2, "big")[:len(s) - 2 * r.lead]


@pytest.mark.parametrize("width", [3, 768])
@pytest.mark.parametrize("ending", ENDINGS)
def test_reference_strings_from_the_initial_state(width, ending):
  """From the initial state the point is 2^31: `80 00 ...` (a carry through 1 800 words, 3 600 bytes), `7f ff ...`,
  and the single byte `80`."""
  syms, c, runs = cs.carry_stream(0, cs.table_cdf(width), [(0, 1800, ending)])
  s = oracle.best().encode(lookup_of(width), syms[None])[0]
  assert s == c.string()
  check_runs(s, c, runs)
  if ending == "above":
    assert s[:3602] == b"\x80" + bytes(3601)
  elif ending == "below":
    assert s[:3602] == b"\x7f" + b"\xff" * 3601
  else:
    assert s == b"\x80"
  assert oracle.best().encode(lookup_of(width), cs.straddle_symbols(cs.table_cdf(width), 2000)[None])[0] == b"\x80"


@pytest.mark.parametrize("width", [3, 768])
@pytest.mark.parametrize("ending", ENDINGS)
def test_runs_reach_their_state(width, ending):
  """Every run of carry_streams.runs_for(ending), with and without a tail of random words after the "above" and
  "below" runs; the model's strings are the reference's, and the 768-word streams have 768 words."""
  O = oracle.best()
  cdf = cs.table_cdf(width)
  for i, (lead, length, total) in enumerate(cs.runs_for(ending)):
    for tail in ((0,) if ending == "straddle" or total else (0, 40)):
      syms, c, runs = cs.run_stream(cdf, ending, i, lead, length, total, tail)
      assert [(r.lead, r.length) for r in runs] == [(lead, length)]
      assert total is None or c.words == total
      s = O.encode(lookup_of(width), syms[None])[0]
      assert s == c.string(), (lead, length, tail)
      check_runs(s, c, runs)


def test_canonical_symbols():
  """canonical_symbols at every length 2..60: the strings start 80 00, 7f ff, or are the byte 80."""
  O = oracle.best()
  for width in (3, 768):
    cdf = cs.table_cdf(width)
    for n in range(2, 61):
      for ending, head in (("above", b"\x80"), ("below", b"\x7f"), ("straddle", b"\x80")):
        syms = cs.canonical_symbols(cdf, n, ending)
        s = O.encode(lookup_of(width), syms[None])[0]
        assert len(syms) == n and s == cs.model_string(cdf, syms) and s[:1] == head, (width, n, ending)
        if ending == "straddle":
          assert s == b"\x80"


def test_several_runs_in_one_stream():
  """Runs one after another in a stream (the multi-call test cuts such a stream between calls): each reaches its
  state, and the carries of the earlier ones stay resolved in the string."""
  cdf = cs.table_cdf(3)
  spec = [(3, 40, "above"), (60, 100, "below"), (200, 31, "above"), (260, 64, "above"), (400, 300, "straddle")]
  syms, c, runs = cs.carry_stream(7, cdf, spec)
  s = oracle.best().encode(lookup_of(3), syms[None])[0]
  assert s == c.string()
  check_runs(s, c, runs)


def test_model_matches_reference_on_random_streams():
  """The model against the reference on random symbols of both tables and on short crafted streams cut at every
  length (the straddle case at each cut)."""
  O = oracle.best()
  rng = np.random.default_rng(5)
  for width in (3, 768):
    cdf = cs.table_cdf(width)
    n_bins = len(cdf) - 1
    value = rng.integers(0, n_bins, size=(16, 300)).astype(np.int32)
    for v, s in zip(value, O.encode(lookup_of(width), value)):
      assert cs.model_string(cdf, v) == s
    syms, _, _ = cs.carry_stream(9, cdf, [(2, 20, "above")], tail_words=5)
    for n in range(len(syms) + 1):
      assert cs.model_string(cdf, syms[:n]) == O.encode(lookup_of(width), syms[None, :n])[0]
