"""Symbol sequences that drive the range encoder into long carry chains, and an exact big-integer model of the
strings they code into.

The row is one p = 16 table of equal bins of `width` (not a power of two) and a narrower last bin.  Pick a point P
inside the current interval that is a multiple of 2^16 (in the units of the encoder's 32-bit window) and code, symbol
after symbol, the bin that contains P: the interval keeps straddling P, every renormalisation emits one more raw
0xFFFF word, and nothing is resolved.  How the run ends decides what finalize and the write kernel see:

  "above"     the last symbol is the bin above P: a carry ripples through every raw 0xFFFF word of the run (they
              become 0x0000) into the word before it;
  "below"     the last symbol is the bin below P: the run stays 0xFFFF, no carry;
  "straddle"  no ending symbol: the stream ends straddling P, and finalize walks back over every 0xFFFF word.

From the initial state the first point is 2^31 and the strings are `80 00 ...`, `7f ff ...` and the single byte `80`.
Bins of width 2 do not work: P lands on a bin edge and the interval stops straddling it.

Coder is the arithmetic of RangeEncoder::Encode / Finalize on exact integers: `low` is the whole code value so far
(carries included, because it is one Python integer), so its words are the resolved words, and `raw` records each
word as it was emitted, before later carries.
"""
import bisect

import numpy as np

P = 16


def table_cdf(width):
  """[0, width, 2 width, ..., 2^16]: equal bins of `width` and a last bin of 2^16 mod width (or `width`)."""
  assert width & (width - 1)  # not a power of two
  return np.concatenate([np.arange(0, 1 << P, width), [1 << P]]).astype(np.int32)


class Coder:
  """RangeEncoder on exact integers: `low` and `size` of the current interval (2^16 < size <= 2^32 between symbols),
  in units of 2^-(32 + 16 words)."""

  def __init__(self, cdf):
    self.cdf = [int(c) for c in cdf]
    self.low, self.size, self.words = 0, 1 << 32, 0
    self.raw = []  # each word as emitted, before carries that arrive later

  @property
  def n_bins(self):
    return len(self.cdf) - 1

  def encode(self, k):
    a = (self.size * self.cdf[k]) >> P
    self.size = ((self.size * self.cdf[k + 1]) >> P) - a
    self.low += a
    if self.size <= 1 << 16:  # size - 1 < 2^16: emit the window's top half
      self.raw.append((self.low >> 16) & 0xFFFF)
      self.low <<= 16
      self.size <<= 16
      self.words += 1

  def bin_of(self, point):
    """The bin whose part of the interval holds `point` (which must lie inside the interval)."""
    t = point - self.low
    assert 0 <= t < self.size
    k = min(self.n_bins - 1, bisect.bisect_right(self.cdf, (t << P) // self.size) - 1)
    while (self.size * self.cdf[k]) >> P > t:
      k -= 1
    while (self.size * self.cdf[k + 1]) >> P <= t:
      k += 1
    return k, ((self.size * self.cdf[k]) >> P) == t

  def resolved(self):
    """The emitted words with every carry applied."""
    R = self.words
    return [(self.low >> (32 + 16 * (R - 1 - i))) & 0xFFFF for i in range(R)]

  def straddles(self):
    return (self.low & 0xFFFFFFFF) + self.size - 1 >= 1 << 32

  def string(self):
    """RangeEncoder::Finalize.  Straddling 2^32 ("state 1"): the value is the next multiple of 2^32, +1 into the
    words, whose trailing zero bytes are dropped.  Otherwise the words, then the shortest one- or two-byte tail that
    lands inside the interval (none if the window's low end is 0)."""
    R = self.words
    if self.straddles():
      return ((self.low >> 32) + 1).to_bytes(2 * R, "big").rstrip(b"\0")
    body = (self.low >> 32).to_bytes(2 * R, "big")
    base = self.low & 0xFFFFFFFF
    if base == 0:
      return body
    top = base + self.size - 1
    r24 = ((base - 1) >> 24) + 1
    if r24 <= top >> 24:
      return body + bytes([r24])
    r16 = ((base - 1) >> 16) + 1
    return body + (bytes([r16 >> 8, r16 & 0xFF]) if r16 & 0xFF else bytes([r16 >> 8]))


class Run:
  """Where one crafted run sits in its stream: the word `lead` before the run (the one a carry ends in), and the
  run's raw 0xFFFF words [lead + 1, lead + 1 + length)."""

  def __init__(self, lead, length, ending):
    self.lead, self.length, self.ending = lead, length, ending

  @property
  def words(self):
    return range(self.lead + 1, self.lead + 1 + self.length)


def _random_until(rng, c, syms, words):
  """Random bins until exactly `words` words have been emitted (one symbol emits at most one)."""
  while c.words < words:
    k = int(rng.integers(c.n_bins))
    c.encode(k)
    syms.append(k)


def _crafted_run(c, syms, run_words, ending):
  """Codes a run that straddles a multiple of 2^16 from the current state: the lead word and `run_words` raw 0xFFFF
  words after it, then the ending symbol (none for "straddle").
  The point is the multiple of 2^16 next to the interval's middle (2^31 from the initial state), else the lowest one
  whose run never puts it on a bin edge (which ends the straddle): after a random prefix the interval's size has lost
  the factors of 3 that keep the canonical run off the edges, and most points fail within a few words."""
  saved = (c.low, c.size, c.words, len(c.raw), len(syms))
  mid = (c.low + c.size // 2) >> 16
  first = (c.low >> 16) + 1
  for j in [mid] + list(range(first, min(first + 4096, (c.low + c.size - 1 >> 16) + 1))):
    point = j << 16
    c.low, c.size, c.words = saved[:3]
    del c.raw[saved[3]:], syms[saved[4]:]
    if not c.low < point < c.low + c.size:
      continue
    run = _run_at(c, syms, point, run_words, ending, None)
    if run is not None:
      return run
  raise AssertionError("no point of the interval gives a run")


def _run_at(c, syms, point, run_words, ending, max_syms):
  """The run at `point` (None if the point falls on a bin edge); with `max_syms`, `max_syms` symbols of it instead."""
  lead, n0 = c.words, len(syms)
  while max_syms is None or len(syms) - n0 < max_syms:
    k, on_edge = c.bin_of(point)
    if on_edge:
      return None
    if max_syms is None and c.words - lead - 1 == run_words:
      if ending != "straddle":  # (it may emit one more word: not part of the run)
        end = k + 1 if ending == "above" else k - 1
        c.encode(end)
        syms.append(end)
      break
    before = c.words
    c.encode(k)
    syms.append(k)
    point <<= 16 * (c.words - before)  # the point moves with the interval's units
  return Run(lead, run_words, ending)


def carry_stream(seed, cdf, runs, tail_words=0, total_words=None):
  """Symbols of one stream: for each (lead_word, run_words, ending) in `runs`, random symbols until `lead_word`
  words have been emitted, then a crafted run whose lead word is word `lead_word`; then random symbols until
  `tail_words` more words, or until `total_words` in all.  A "straddle" run must be the last, without a tail.
  Returns (symbols, coder, runs)."""
  rng = np.random.default_rng(seed)
  c = Coder(cdf)
  syms, out = [], []
  for i, (lead, length, ending) in enumerate(runs):
    assert ending != "straddle" or (i == len(runs) - 1 and tail_words == 0)
    _random_until(rng, c, syms, lead)
    assert c.words == lead, (c.words, lead)
    out.append(_crafted_run(c, syms, length, ending))
  _random_until(rng, c, syms, c.words + tail_words if total_words is None else total_words)
  assert total_words is None or c.words == total_words
  return np.asarray(syms, np.int32), c, out


def canonical_symbols(cdf, n, ending):
  """`n` symbols of the run from the initial state (point 2^31), the last one the ending ("straddle": none)."""
  c = Coder(cdf)
  syms = []
  _run_at(c, syms, 1 << 31, None, "straddle", n - (ending != "straddle"))
  if ending != "straddle":
    k, _ = c.bin_of((1 << 31) << 16 * c.words)
    syms.append(k + 1 if ending == "above" else k - 1)
  return np.asarray(syms, np.int32)


def straddle_symbols(cdf, n):
  """A stream of `n` symbols (n >= 2) that ends straddling from the initial state: its string is the single byte
  0x80, so the strings after it start at odd offsets."""
  return canonical_symbols(cdf, n, "straddle")


ENDINGS = ("above", "below", "straddle")
# (lead word, run words, total words or None) of test_range_encoder_paths_*: runs around one 32-word group and at
# group boundaries in streams of fewer than 8 groups (some write-kernel warps get no group); in 768-word streams
# (24 groups: 8 segments of 3 groups, words [96 j, 96 j + 96)) a run of exactly segment 2 and one word less or more
# (a straddle run ends the stream, so its run is the last segment); runs across every segment
RUNS = [(0, 31, None), (0, 32, None), (0, 33, None), (31, 32, None), (32, 31, None), (63, 33, None), (5, 96, None),
        (191, 96, 768), (192, 95, 768), (190, 97, 768), (0, 1800, None), (57, 1800, None)]
STRADDLE_SEGMENT_RUNS = [(671, 96, None), (672, 95, None), (670, 97, None)]


def runs_for(ending):
  return [r for r in RUNS if ending != "straddle" or r[2] is None] + (
      STRADDLE_SEGMENT_RUNS if ending == "straddle" else [])


def run_stream(cdf, ending, i, lead, length, total, tail=0):
  """carry_stream of one run of RUNS / STRADDLE_SEGMENT_RUNS (entry i)."""
  if ending == "straddle":
    tail = 0
  return carry_stream(100 + i, cdf, [(lead, length, ending)], tail_words=tail, total_words=total)


def model_string(cdf, symbols):
  c = Coder(cdf)
  for k in symbols:
    c.encode(int(k))
  return c.string()
