"""GPU: the coding tables themselves.  `pmf_rows_kernel` (csrc/pmf_to_cdf.cu) builds every table the range coder
codes with, and the byte-equality tests elsewhere code with those same tables on both sides, so a wrong count there
would still round-trip.  Here the tables are compared exactly, row by row, with independent expected values:

* the dense op `pmf_to_quantized_cdf` (pmf_to_cdf_kernels.cc:58-208) against the C port on every row, and on rows
  without exact ties also against the compiled reference (`oracle.ref()` when built, else its outputs stored in
  tests/golden/reference_outputs.npz by oracle/make_reference_outputs.py from the generators below);
* `functional.build_lookup` against the per-row loop of continuous_base.py:282-294 restated with the port;
* the entropy models' `cdf` / `cdf_offset` against continuous_base.py:239-294 restated here.

Rows at the edges: n = 2^precision, rows spanning several 256-thread strides, tens of thousands of adjustment steps,
all-zero rows (only the FIFO rule decides), subnormal masses, counts above 2^16 (past the shared log2 table)."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import golden_util
import oracle

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------------------------------
# Case generators (shared with oracle/make_reference_outputs.py)
# ------------------------------------------------------------------------------------------------
PRECISIONS = (1, 2, 7, 8, 12, 15, 16)
NS = (2, 3, 31, 32, 33, 255, 256, 257, 1023, 4097)
DENSE_CASES = sorted({(p, n) for p in PRECISIONS for n in NS if n <= 1 << p} |
                     {(p, (1 << p) + d) for p in (8, 12, 16) for d in (-1, 0)})

ROW_KINDS = ("random", "x0.2", "x0.85", "x1.3", "peaky", "subnormal_mix", "subnormal_all",   # no exact ties
             "upper_half_zero", "all_zero", "spike", "symmetric")
TIE_FREE = ROW_KINDS[:7]
# At n >= 2^16 - 1 bins the port's O(steps * n) greedy takes seconds per row, so those cases use nearly uniform
# rows and the kinds that need few steps.
FULL_WIDTH_KINDS = ("random", "x0.2", "subnormal_all", "all_zero")


def row_kinds(p, n):
  return FULL_WIDTH_KINDS if p == 16 and n >= (1 << p) - 1 else ROW_KINDS


def _distinct(rng, n):
  """n positive float64 values that stay pairwise distinct (relative gaps >= 2^-17) after scaling to float32."""
  return rng.permutation(n) + 1 + 0.5 * rng.random(n)


def _flat_distinct(rng, n):
  """n distinct values in [1, 2): rows of about 2^p / n counts per bin."""
  return 1 + (rng.permutation(n) + 0.5 * rng.random(n)) / n


def _normalised(x, scale=1.0):
  return (x / x.sum() * scale).astype(np.float32)


def dense_rows(p, n):
  """One row of every kind in row_kinds(p, n) for n bins at precision p: float32 [len(kinds), n]."""
  rng = np.random.default_rng(1000 * p + n)
  kinds = row_kinds(p, n)
  rows = []
  for kind in kinds:
    base = _distinct(rng, n) if kinds is ROW_KINDS else _flat_distinct(rng, n)
    if kind == "random":
      row = _normalised(base)
    elif kind.startswith("x"):
      row = _normalised(base, float(kind[1:]))
    elif kind == "peaky":
      row = _normalised((base / base.max())**8)
    elif kind == "subnormal_mix":   # normal masses with about 1e-40 in every third bin
      row = _normalised(base)
      row[::3] = (1e-40 * (1 + base[::3] / n)).astype(np.float32)
    elif kind == "subnormal_all":   # every key is subnormal-sized: a flush to zero would turn them into ties
      t = (base - base.min()) / max(np.ptp(base), 1e-300)
      row = np.exp(np.log(1e-40) + np.log(100.) * t).astype(np.float32)
    elif kind == "upper_half_zero":   # pmf_to_cdf_kernels_test.cc:123-143
      base[n // 2:] = 0
      row = _normalised(base) if n > 1 else base.astype(np.float32)
    elif kind == "all_zero":
      row = np.zeros(n, np.float32)
    elif kind == "spike":
      row = np.zeros(n, np.float32)
      row[0] = 1
    else:   # symmetric: mirror-image bins have equal masses (exact ties)
      k = np.arange(n) - (n - 1) / 2
      row = _normalised(np.exp(-0.5 * (k / max(n / 8, 0.5))**2))
    assert row.shape == (n,) and row.dtype == np.float32
    rows.append(row)
  return np.stack(rows)


def tie_free_dense_rows(p, n):
  kinds = row_kinds(p, n)
  return dense_rows(p, n)[[i for i, k in enumerate(kinds) if k in TIE_FREE]]


def large_count_cases():
  """(precision, pmf) whose counts pass 65 537, the last count the shared log2 table covers.  Every count and row
  sum stays below 2^31 (the reference's int32) and every row below about 2e5 adjustment steps."""
  rng = np.random.default_rng(21)
  mixed = np.stack([_normalised(_distinct(rng, 64)) for _ in range(4)])
  mixed[0, 17] = 40.0                 # 163 840 counts at precision 12
  mixed[2, 63] = 9.5                  # 38 912: under the shared table, in the same launch as a row over it
  mixed[3] *= 1.7
  wide = _normalised(_distinct(rng, 300), 1.5)
  wide[[5, 250]] = [1.25, 1.5]        # two bins over the table at precision 16 (81 920 and 98 304 counts)
  return [(16, np.asarray([[3.0, 1.0]], np.float32)),
          (12, np.asarray([[20.0, 1.0]], np.float32)),
          (12, mixed),
          (16, wide[None])]


def many_rows_case():
  """One call of 3000 rows of 100 bins at precision 12 whose adjustment runs from none to thousands of steps."""
  rng = np.random.default_rng(3000)
  scale = np.exp(rng.uniform(np.log(0.05), np.log(2.0), 3000))
  return np.stack([_normalised(_distinct(rng, 100), s) for s in scale])


def tie_free_reference_rows():
  """The rows compared with the compiled reference, in the order they are stored: (precision, pmf) pairs."""
  for p, n in DENSE_CASES:
    yield p, tie_free_dense_rows(p, n)
  yield from large_count_cases()
  yield 12, many_rows_case()


# ------------------------------------------------------------------------------------------------
# Expected values
# ------------------------------------------------------------------------------------------------
def port_cdf(pmf, precision):
  """oracle.port().pmf_to_cdf row by row on every core (the port releases the GIL)."""
  P = oracle.port()
  pmf = np.ascontiguousarray(pmf, np.float32)
  with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
    return np.stack(list(ex.map(lambda row: P.pmf_to_cdf(row[None], precision)[0], pmf)))


def kernel_order_sum(p):
  """float32 sum of a row in the order pmf_rows_kernel documents: 256 strided per-thread partial sums in index
  order, an xor butterfly within each warp, then the 8 warp sums added in order.  The reference's tf.reduce_sum
  leaves its order unspecified; this order is the one detail the expected tables share with the kernel, and only
  the arbitrary-float rows depend on it (the other rows' partial sums are exact in any order)."""
  p = np.asarray(p, np.float32)
  padded = np.zeros(-(-len(p) // 256) * 256, np.float32)
  padded[:len(p)] = p
  part = np.zeros(256, np.float32)
  for chunk in padded.reshape(-1, 256):
    part = (part + chunk).astype(np.float32)
  lanes = part.reshape(8, 32)
  for d in (16, 8, 4, 2, 1):
    lanes = (lanes + lanes[:, np.arange(32) ^ d]).astype(np.float32)
  total = np.float32(0)
  for w in range(8):
    total = np.float32(total + lanes[w, 0])
  return total


def reference_lookup_row(p, precision, overflow):
  """[-precision, cdf...] of continuous_base.py:284-288 for one sliced row p and its overflow mass."""
  row = np.concatenate([np.asarray(p, np.float32), np.asarray([overflow], np.float32)])
  return np.concatenate([[-precision], oracle.port().pmf_to_cdf(row, precision)]).astype(np.int32)


def _reference_lookup_rows(rows, precision):
  """reference_lookup_row over (p, overflow) pairs on every core."""
  with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
    return list(ex.map(lambda a: reference_lookup_row(a[0], precision, a[1]), rows))


def restated_tables(prior, tail_mass, precision, offset=None):
  """continuous_base.py:239-294 restated: tails, ranges, PMF samples, then per row slice, append
  max(1 - sum(p), 0) summed in the prior's dtype, cast to float32, quantise with the port, prepend -precision."""
  from compression_b200 import distributions as D
  dtype = prior.dtype
  offset = torch.zeros((), dtype=dtype) if offset is None else torch.as_tensor(offset).to("cpu", dtype)
  lower = D.lower_tail(prior, tail_mass).to("cpu")
  upper = D.upper_tail(prior, tail_mass).to("cpu")
  minima = torch.floor(lower - offset).to(torch.int32)
  maxima = torch.ceil(upper - offset).to(torch.int32)
  pmf_start = minima.to(dtype) + offset
  pmf_length = maxima - minima + 1
  max_length = int(pmf_length.max())
  samples = torch.arange(max_length, dtype=dtype).reshape([-1] + pmf_length.dim() * [1]) + pmf_start
  with torch.no_grad():
    pmf = prior.prob(samples.to(getattr(prior, "device", torch.device("cpu")))).detach().cpu()
  pmf_shape = tuple(pmf.shape[1:])
  num_pmfs = int(np.prod(pmf_shape)) if pmf_shape else 1
  pmf = pmf.reshape(max_length, num_pmfs).t().numpy()
  lengths = torch.broadcast_to(pmf_length, pmf_shape).reshape(num_pmfs).numpy()
  cdf_offset = torch.broadcast_to(minima, pmf_shape).reshape(num_pmfs).numpy()
  rows = []
  for i in range(num_pmfs):
    p = pmf[i, :lengths[i]]
    if p.dtype == np.float64:
      overflow = max(1. - p.sum(), 0.)
    else:
      overflow = max(np.float32(1) - kernel_order_sum(p), np.float32(0))
    rows.append((p.astype(np.float32), overflow))
  return np.concatenate(_reference_lookup_rows(rows, precision)), cdf_offset.astype(np.int32)


# ------------------------------------------------------------------------------------------------
# Dense op
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ops():
  from compression_b200 import gen_ops
  return gen_ops


@pytest.fixture(scope="module")
def reference_rows():
  """Compiled-reference tables of tie_free_reference_rows(), live when oracle/_ref is built, else stored."""
  if oracle.have_ref():
    return [oracle.ref().pmf_to_cdf(pmf, p) for p, pmf in tie_free_reference_rows()]
  return stored_reference_rows()


def stored_reference_rows():
  """The compiled reference's tables of tie_free_reference_rows() from tests/golden/reference_outputs.npz (stored as
  bin counts)."""
  counts = golden_util.split_rows(golden_util.load_reference(), "pmf_edge_counts")
  return [np.concatenate([np.zeros(c.shape[:-1] + (1,), np.int32), np.cumsum(c, axis=-1, dtype=np.int32)], -1)
          for c in counts]


def _reference_index(p, pmf):
  for i, (q, x) in enumerate(tie_free_reference_rows()):
    if q == p and x.shape == pmf.shape and np.array_equal(x, pmf):
      return i
  raise KeyError((p, pmf.shape))


def _gpu_cdf(ops, pmf, p):
  return ops.pmf_to_quantized_cdf(torch.from_numpy(np.ascontiguousarray(pmf)).cuda(), p).cpu().numpy()


def _assert_rows_equal(got, want, what):
  bad = [r for r in range(len(want)) if not np.array_equal(got[r], want[r])]
  assert not bad, f"{what}: rows {bad} differ, first at bins {np.flatnonzero(got[bad[0]] != want[bad[0]])[:8]}"


@pytest.mark.parametrize("p,n", DENSE_CASES)
def test_dense_rows_equal_port_and_reference(ops, reference_rows, p, n):
  pmf, kinds = dense_rows(p, n), row_kinds(p, n)
  got = _gpu_cdf(ops, pmf, p)
  assert got.shape == (len(kinds), n + 1)
  assert (got[:, 0] == 0).all() and (got[:, -1] == 1 << p).all() and (np.diff(got, axis=-1) >= 1).all()
  if n == 1 << p:
    assert (got == np.arange(n + 1)).all()
  _assert_rows_equal(got, port_cdf(pmf, p), f"port, kinds {kinds}")
  tie_free = [i for i, k in enumerate(kinds) if k in TIE_FREE]
  ref = reference_rows[DENSE_CASES.index((p, n))]
  _assert_rows_equal(got[tie_free], ref, f"compiled reference, kinds {[kinds[i] for i in tie_free]}")


def test_all_zero_rows_are_pure_round_robin(ops):
  """All keys tie, so only the FIFO rule decides: every bin gets (2^p - n) // n extra counts, the lowest-index bins
  one more."""
  for p, n in ((7, 3), (12, 257), (16, 4097)):
    got = np.diff(_gpu_cdf(ops, np.zeros((2, n), np.float32), p), axis=-1)
    extra = (1 << p) - n
    want = 1 + extra // n + (np.arange(n) < extra % n)
    assert (got == want).all(), (p, n)


def test_large_counts_past_the_shared_log2_table(ops, reference_rows):
  """Counts above 65 537 make the DOWN adjustment read log2 beyond the shared table: the call reruns with a table
  sized for it (one extra launch) and still equals the port and the compiled reference."""
  from compression_b200 import _lib
  n_dense = len(DENSE_CASES)
  for k, (p, pmf) in enumerate(large_count_cases()):
    c0 = _lib.launch_count()
    got = _gpu_cdf(ops, pmf, p)
    assert _lib.launch_count() - c0 == 2
    assert (np.diff(got, axis=-1) >= 1).all() and (got[:, -1] == 1 << p).all()
    _assert_rows_equal(got, port_cdf(pmf, p), f"port, case {k}")
    _assert_rows_equal(got, reference_rows[n_dense + k], f"compiled reference, case {k}")
  # normalised rows keep one launch
  c0 = _lib.launch_count()
  _gpu_cdf(ops, dense_rows(12, 257), 12)
  assert _lib.launch_count() - c0 == 1


def test_counts_beyond_the_largest_table_are_refused(ops):
  """Above 2^24 - 1 counts per bin (a 128 MiB log2 table) the op refuses the input and names the first such bin."""
  pmf = np.asarray([[0.5, 0.5], [0.25, 300.0], [500.0, 0.5]], np.float32)
  with pytest.raises(ops.InvalidArgumentError, match=r"row 1, bin 1 .*16777216"):
    _gpu_cdf(ops, pmf, 16)
  # the op stays usable, and a value error still comes first
  assert np.array_equal(_gpu_cdf(ops, pmf[:1], 16), oracle.port().pmf_to_cdf(pmf[:1], 16))
  pmf[0, 0] = np.nan
  with pytest.raises(ops.InvalidArgumentError, match="non-finite"):
    _gpu_cdf(ops, pmf, 16)


def test_many_rows_of_different_step_counts(ops, reference_rows):
  pmf = many_rows_case()
  got = _gpu_cdf(ops, pmf, 12)
  _assert_rows_equal(got, port_cdf(pmf, 12), "port")
  _assert_rows_equal(got, reference_rows[-1], "compiled reference")


# ------------------------------------------------------------------------------------------------
# functional.build_lookup (the ragged builder every entropy model uses)
# ------------------------------------------------------------------------------------------------
LENGTHS = (1, 2, 31, 32, 33, 255, 256, 257, 2047, 2048)
MASS_KINDS = ("sum_one", "sum_small", "sum_over_one", "arbitrary")


def _exact_masses(rng, length, total):
  """Multiples of 2^-24 adding up to total * 2^-24 <= 1: every partial sum is exact in float32, in any order."""
  w = rng.multinomial(total, rng.dirichlet(np.ones(length)))
  return (w * 2.0**-24).astype(np.float32)


def ragged_case(p, rows):
  """(pmf [rows, max_len] float32 with junk padding, lengths, mass kind per row) at precision p."""
  rng = np.random.default_rng(50 + p)
  allowed = [l for l in LENGTHS if l <= (1 << p) - 1]
  # the first row of each mass kind has the longest length, 2^p - 1; the others cycle through the short ones
  lens = np.asarray([(1 << p) - 1 if r < len(MASS_KINDS) else allowed[r % len(allowed)] for r in range(rows)],
                    np.int32)
  max_len = (1 << p) + 40
  pad = np.asarray([np.nan, -1.0, 1e30, np.inf, -np.inf], np.float32)
  pmf = np.resize(pad, (rows, max_len)).astype(np.float32)   # beyond len: ignored, the reference slices first
  kinds = []
  for r, L in enumerate(lens):
    kind = MASS_KINDS[r % len(MASS_KINDS)]
    base = _flat_distinct(rng, L) if L > 4096 else _distinct(rng, L)
    if kind == "sum_one":
      row = _exact_masses(rng, L, 1 << 24)
    elif kind == "sum_small":
      row = _exact_masses(rng, L, int(rng.integers(1, 1 << 18)))
    elif kind == "sum_over_one":
      row = _normalised(base, 1.3)
    else:
      row = _normalised(base, rng.uniform(0.95, 1.0))
    pmf[r, :L] = row
    kinds.append(kind)
  return pmf, lens, kinds


def expected_lookup(pmf, lens, kinds, p):
  rows = []
  for r, L in enumerate(lens):
    row = pmf[r, :L]
    if kinds[r].startswith("sum_") and kinds[r] != "sum_over_one":
      s = row.astype(np.float64).sum()
      assert np.float32(s) == s <= 1      # exact: independent of the summation order
      overflow = np.float32(1 - s)
    else:
      overflow = max(np.float32(1) - kernel_order_sum(row), np.float32(0))
      if kinds[r] == "sum_over_one":
        assert overflow == 0
    rows.append((row, overflow))
  return np.concatenate(_reference_lookup_rows(rows, p))


def _split_lookup(lookup, lens):
  out, at = [], 0
  for L in lens:
    out.append(lookup[at:at + L + 3])
    at += L + 3
  assert at == len(lookup)
  return out


@pytest.mark.parametrize("p", range(1, 17))
def test_build_lookup_equals_the_reference_loop(p):
  from compression_b200 import functional as F
  pmf, lens, kinds = ragged_case(p, 4096 if p == 12 else 300 if p < 15 else 100)
  got = F.build_lookup(torch.from_numpy(pmf).cuda(), lens, p).cpu().numpy()
  want = expected_lookup(pmf, lens, kinds, p)
  assert got.shape == want.shape
  bad = [r for r, (a, b) in enumerate(zip(_split_lookup(got, lens), _split_lookup(want, lens))) if not np.array_equal(a, b)]
  assert not bad, f"rows {bad[:10]} differ (lengths {lens[bad[:10]]}, kinds {[kinds[r] for r in bad[:10]]})"


def test_build_lookup_names_a_bad_mass_inside_the_length():
  from compression_b200 import functional as F, gen_ops
  pmf, lens, _ = ragged_case(8, 20)
  pmf[3, 5] = np.nan
  with pytest.raises(gen_ops.InvalidArgumentError, match=r"row 3, bin 5"):
    F.build_lookup(torch.from_numpy(pmf).cuda(), lens, 8)


# ------------------------------------------------------------------------------------------------
# Entropy models
# ------------------------------------------------------------------------------------------------
def _assert_model_tables(em, prior, offset=None):
  cdf, cdf_offset = restated_tables(prior, em.tail_mass, int(-em.cdf[0]), offset)
  got = em.cdf.cpu().numpy()
  assert got.shape == cdf.shape and np.array_equal(got, cdf)
  assert np.array_equal(em.cdf_offset.cpu().numpy(), cdf_offset)
  return cdf, cdf_offset


@pytest.mark.parametrize("precision", [12, 16])
def test_batched_deep_factorized_tables(precision):
  import compression_b200 as tfc
  torch.manual_seed(3)
  prior = tfc.NoisyDeepFactorized(batch_shape=(24,))
  em = tfc.ContinuousBatchedEntropyModel(prior, coding_rank=1, compression=True, range_coder_precision=precision)
  _assert_model_tables(em, prior, em.quantization_offset)


@pytest.mark.parametrize("prior_kind", ["laplace", "deep"])
def test_cfg2_tables_and_the_committed_fixture(prior_kind):
  """cfg2's tables (bench.build_model) equal the restatement; the Laplace ones are also the committed fixture that
  `bench.py --impl reference` codes with."""
  import bench
  import compression_b200 as tfc
  scales, _ = bench.synth_latents(0, 0)
  em = bench.build_model(scales, torch.device("cuda", 0), prior_kind)
  if prior_kind == "laplace":
    prior = tfc.NoisyLaplace(loc=torch.zeros_like(scales), scale=scales)
  else:
    torch.manual_seed(11)
    prior = tfc.NoisyDeepFactorized(batch_shape=(len(scales),))
  q = em.quantization_offset
  cdf, cdf_offset = _assert_model_tables(em, prior, None if q is None else q.cpu())
  if prior_kind == "laplace":
    g = np.load(golden_util.PATH.replace("range_coder_golden.npz", "cfg2_tables.npz"))
    assert np.array_equal(g["lookup"], cdf) and np.array_equal(g["cdf_offset"], cdf_offset)


@pytest.mark.parametrize("prior_dtype", [torch.float32, torch.float64])
def test_cfg3_indexed_tables(prior_dtype):
  """64 NoisyNormal scales up to sigma = 256 (more than 1000 bins).  With float64 priors the reference sums the
  overflow mass in float64 and casts afterwards (continuous_base.py:285-286)."""
  import compression_b200 as tfc
  off, fac = np.log(.11), (np.log(256.) - np.log(.11)) / 63
  em = tfc.LocationScaleIndexedEntropyModel(lambda loc, scale: tfc.NoisyNormal(loc, scale, dtype=prior_dtype), 64,
                                            lambda i: torch.exp(off + fac * i), coding_rank=3, compression=True,
                                            prior_dtype=prior_dtype)
  assert em.prior.dtype == prior_dtype
  assert int(np.diff(np.flatnonzero(em.cdf.cpu().numpy() < 0)).max()) > 1000
  _assert_model_tables(em, em.prior)


def test_universal_tables():
  import compression_b200 as tfc
  from compression_b200 import entropy_models as E
  prior = tfc.NoisyLogistic(loc=torch.zeros(3), scale=torch.tensor([.7, 4., 20.]))
  em = tfc.UniversalBatchedEntropyModel(prior, coding_rank=2, compression=True, num_noise_levels=15)
  _assert_model_tables(em, prior, E._range_coding_offsets(15, 1, torch.float32))
  em = tfc.UniversalIndexedEntropyModel(tfc.NoisyLogistic, (5, 3), dict(loc=lambda i: i[..., 0], scale=lambda i: 1. + i[..., 1]),
                                        coding_rank=1, compression=True, num_noise_levels=7)
  _assert_model_tables(em, em.prior, E._range_coding_offsets(7, len(em.prior.batch_shape), torch.float32))


def test_gpu_strings_decode_with_the_restated_tables():
  """The strings a model writes decode, with the compiled reference (or the port), under tables built the
  reference's way."""
  import compression_b200 as tfc
  torch.manual_seed(4)
  prior = tfc.NoisyDeepFactorized(batch_shape=(8,))
  em = tfc.ContinuousBatchedEntropyModel(prior, coding_rank=2, compression=True)
  q = em.quantization_offset
  lookup, cdf_offset = restated_tables(prior, em.tail_mass, 12, q)
  x = torch.randn(5, 300, 8) * 6
  strings = em.compress(x.cuda()).tolist()
  sym = (torch.round(x - q) if q is not None else torch.round(x)).to(torch.int32) - torch.from_numpy(cdf_offset)
  sym = sym.reshape(5, -1).numpy()
  back, ok = oracle.best().decode(lookup, strings, sym.shape[1])
  assert ok.all() and np.array_equal(back, sym)
