"""Ragged RunLengthEncode / RunLengthDecode on the GPU: many strings in one launch, each byte-identical to the
sequential C restatement (oracle port) and to the one-string op, decoded back with the reference's error messages,
and the run-length entropy models' compress_ragged / decompress_ragged on top."""
import os
import re

import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu
CONFIGS = [(-1, -1, False), (-1, -1, True), (0, 0, False), (2, 3, True), (5, -1, False), (-1, 4, True), (3, 0, True)]
KINDS = ["dense", "sparse", "leading", "trailing", "zeros", "nonzeros"]
I32 = np.iinfo(np.int32)


@pytest.fixture(scope="module")
def ops():
  from compression_b200 import functional as F
  from compression_b200 import gen_ops
  return F, gen_ops


def _unit(rng, kind, n, mg):
  d = rng.integers(-40, 41, n).astype(np.int32)
  if kind == "sparse":
    d *= rng.random(n) < 0.07
  if kind == "leading":
    d[:n // 3 + 1] = 0
  if kind == "trailing":
    d[n - n // 3 - 1:] = 0
  if kind == "zeros":
    d[:] = 0
  if kind == "nonzeros":
    d[d == 0] = 5
  if kind == "dense":
    d[::97] = I32.min if mg < 0 else 100000   # gamma codes int32 minimum as its neighbour
    d[1::97] = I32.max if mg < 0 else -100000
  return d


def _mixed_units(rng, mg):
  specs = [(0, "dense"), (1, "dense"), (1, "zeros"), (7001, "dense"), (300_000, "sparse"), (0, "zeros")]
  specs += [(7001, k) for k in KINDS[1:]]
  specs += [(int(rng.integers(0, 40)), KINDS[i % len(KINDS)]) for i in range(300)]
  order = rng.permutation(len(specs))
  return [_unit(rng, specs[i][1], specs[i][0], mg) for i in order]


def _encode(F, units, params):
  flat = np.concatenate(units).astype(np.int32) if units else np.zeros(0, np.int32)
  return F.run_length_encode_ragged(torch.from_numpy(flat).cuda(), [u.size for u in units], *params), flat


@pytest.mark.parametrize("params", CONFIGS)
def test_mixed_units_equal_the_oracle_and_the_one_string_op_and_round_trip(ops, params):
  F, gen_ops = ops
  O = oracle.port()
  rng = np.random.default_rng(abs(hash(params)) % (2**31))
  units = _mixed_units(rng, params[1])
  strings, flat = _encode(F, units, params)
  assert strings.shape == (len(units),)
  got = strings.tolist()
  want = [O.run_length_encode(u, *params) for u in units]
  for i, u in enumerate(units):
    assert got[i] == want[i], f"unit {i} ({u.size} elements)"
    assert got[i] == gen_ops.run_length_encode(torch.from_numpy(u), *params), f"unit {i}"
  lengths = [u.size for u in units]
  back = F.run_length_decode_ragged(strings, lengths, *params).cpu().numpy()
  assert np.array_equal(back, np.concatenate([O.run_length_decode(w, (u.size,), *params).reshape(-1)
                                              for w, u in zip(want, units)]))
  keep = flat != I32.min if params[1] < 0 else np.ones(flat.size, bool)
  assert np.array_equal(back[keep], flat[keep])
  # the same strings as host bytes decode the same way
  assert np.array_equal(F.run_length_decode_ragged(got, lengths, *params).cpu().numpy(), back)


@pytest.mark.parametrize("params", [(-1, -1, False), (2, 3, True), (0, 0, False)])
def test_many_short_units_share_words(ops, params):
  """100 000 units of 1 to 9 elements: most strings are a few bits long and share 32-bit words with neighbours."""
  F, _ = ops
  O = oracle.port()
  rng = np.random.default_rng(3)
  lengths = rng.integers(1, 10, 100_000)
  flat = (rng.integers(-9, 10, int(lengths.sum())) * (rng.random(int(lengths.sum())) < 0.5)).astype(np.int32)
  strings = F.run_length_encode_ragged(torch.from_numpy(flat).cuda(), lengths, *params)
  got = strings.tolist()
  at = 0
  for i, n in enumerate(lengths):
    assert got[i] == O.run_length_encode(flat[at:at + n], *params), f"unit {i}"
    at += n
  assert np.array_equal(F.run_length_decode_ragged(strings, lengths, *params).cpu().numpy(), flat)


def test_golden_vectors_in_one_call_per_parameter_set(ops):
  F, _ = ops
  g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "run_length_golden.npz"))
  groups = {}
  at_d = at_c = 0
  for (rl, mg, nz), nd, nc in zip(g["params"], g["data_len"], g["code_len"]):
    d = np.ascontiguousarray(g["data"][at_d:at_d + nd]).astype(np.int32)
    code = bytes(g["code"][at_c:at_c + nc])
    at_d, at_c = at_d + nd, at_c + nc
    groups.setdefault((int(rl), int(mg), bool(nz)), []).append((d, code))
  assert groups
  for params, vecs in groups.items():
    strings, flat = _encode(F, [d for d, _ in vecs], params)
    assert strings.tolist() == [c for _, c in vecs], params
    back = F.run_length_decode_ragged([c for _, c in vecs], [d.size for d, _ in vecs], *params)
    assert np.array_equal(back.cpu().numpy(), flat), params


def test_a_unit_longer_than_2_to_the_32_bits_beside_tiny_units(ops):
  """~70 M elements of magnitude near 2^30 under gamma: 63 bits each, so the unit's code passes 2^32 bits and its
  bit offsets need all 64 bits of the scan."""
  F, _ = ops
  O = oracle.port()
  params = (-1, -1, False)
  rng = np.random.default_rng(11)
  n_big = 70_000_000
  big = ((2**30 + rng.integers(0, 2**20, n_big)) * np.where(rng.random(n_big) < 0.5, -1, 1)).astype(np.int32)
  tiny = [_unit(rng, KINDS[i % len(KINDS)], int(rng.integers(0, 4)), -1) for i in range(4000)]
  units = tiny[:2000] + [big] + tiny[2000:]
  strings, flat = _encode(F, units, params)
  got = strings.tolist()
  want_big = O.run_length_encode(big, *params)
  assert len(want_big) * 8 > 2**32
  assert got[2000] == want_big
  del want_big
  for i, u in enumerate(units):
    if i != 2000:
      assert got[i] == O.run_length_encode(u, *params), f"unit {i}"
  del got
  back = F.run_length_decode_ragged(strings, [u.size for u in units], *params).cpu().numpy()
  keep = flat != I32.min
  assert np.array_equal(back[keep], flat[keep])


def _oracle_message(code, n, params):
  with pytest.raises(oracle.OracleError) as e:
    oracle.port().run_length_decode(code, (n,), *params)
  return str(e.value)


@pytest.mark.parametrize("params", [(-1, -1, False), (2, 3, True)])
def test_damaged_strings_name_the_lowest_failing_unit(ops, params):
  F, _ = ops
  from compression_b200._lib import InvalidArgumentError
  rng = np.random.default_rng(5)
  units = [_unit(rng, "sparse", int(rng.integers(50, 200)), params[1]) for _ in range(20)]
  units[9] = np.asarray([0, 0, 7, -2, 0, 1], np.int32)
  strings, _ = _encode(F, units, params)
  good = strings.tolist()
  lengths = [u.size for u in units]
  # truncated strings at units 7 and 12: unit 7 is reported
  bad = list(good)
  bad[7] = good[7][:len(good[7]) // 2]
  bad[12] = good[12][:1]
  msg = _oracle_message(bad[7], lengths[7], params)
  with pytest.raises(InvalidArgumentError, match=r"unit 7: " + re.escape(msg)):
    F.run_length_decode_ragged(bad, lengths, *params)
  # past end: unit 9 starts with a run of two zeros, decoded into one element
  short = list(lengths)
  short[9] = 1
  msg = _oracle_message(good[9], 1, params)
  assert msg == "Decoded past end of tensor."
  with pytest.raises(InvalidArgumentError, match=r"unit 9: Decoded past end of tensor\."):
    F.run_length_decode_ragged(good, short, *params)
  # the good strings still decode
  F.run_length_decode_ragged(good, lengths, *params)


def test_gamma_width_error_names_its_unit(ops):
  F, _ = ops
  from compression_b200._lib import InvalidArgumentError
  params = (-1, -1, False)
  codes = [F.run_length_encode_ragged(torch.tensor([0, 3, 0], dtype=torch.int32), [3], *params).tolist()[0]] * 5
  codes[3] = bytes([0, 0, 0, 0, 1])   # 32 zeros, then a one: width 33
  assert _oracle_message(codes[3], 4, params) == "Exceeded maximum gamma bit width."
  with pytest.raises(InvalidArgumentError, match=r"unit 3: Exceeded maximum gamma bit width\."):
    F.run_length_decode_ragged(codes, [3, 3, 3, 4, 3], *params)
  codes[3] = bytes([0, 0, 0, 0])      # no terminating one: out of bits, not too wide
  with pytest.raises(InvalidArgumentError, match=r"unit 3: Out of bits to read\."):
    F.run_length_decode_ragged(codes, [3, 3, 3, 4, 3], *params)


def test_launch_count_does_not_depend_on_the_number_of_units(ops):
  F, _ = ops
  from compression_b200 import _lib
  params = (2, 3, True)
  counts = []
  for k in (10, 100_000):
    lengths = [5] * k
    x = torch.randint(-3, 4, (5 * k,), dtype=torch.int32, device="cuda")
    c0 = _lib.launch_count()
    s = F.run_length_encode_ragged(x, lengths, *params)
    c1 = _lib.launch_count()
    back = F.run_length_decode_ragged(s, lengths, *params)
    c2 = _lib.launch_count()
    assert torch.equal(back, x)
    counts.append((c1 - c0, c2 - c1))
  assert counts[0] == counts[1], counts
  assert counts[0][1] == 1


def _models():
  from compression_b200 import run_length_models as M
  return [M.PowerLawEntropyModel(coding_rank=2), M.LaplaceEntropyModel(coding_rank=2),
          M.LaplaceEntropyModel(coding_rank=2, run_length_code=2, magnitude_code=3, use_run_length_for_non_zeros=True),
          M.PowerLawEntropyModel(coding_rank=2, bottleneck_dtype=torch.float16)]


@pytest.mark.parametrize("em", _models(), ids=["power_law", "laplace", "laplace_rice_nz", "power_law_f16"])
def test_models_ragged_equal_the_per_item_path(em):
  g = torch.Generator().manual_seed(4)
  shapes = [(3, 5), (0, 4), (17, 33), (1, 1), (64, 40)]
  items = [(torch.randn(s, generator=g) * 4 * (torch.rand(s, generator=g) < 0.3)).to(em.bottleneck_dtype)
           for s in shapes]
  strings = em.compress_ragged(items)
  assert strings.shape == (len(items),)
  got = strings.tolist()
  for i, x in enumerate(items):
    assert got[i] == em.compress(x)[()], f"item {i}"
  back = em.decompress_ragged(strings, shapes)
  for i, x in enumerate(items):
    assert back[i].dtype == em.bottleneck_dtype and tuple(back[i].shape) == shapes[i]
    assert torch.equal(back[i].cpu(), em.quantize(x).cpu()), f"item {i}"
    assert torch.equal(back[i].cpu(), em.decompress(got[i], shapes[i]).cpu()), f"item {i}"


def test_models_uniform_batch_and_coding_rank_zero():
  from compression_b200 import run_length_models as M
  g = torch.Generator().manual_seed(6)
  x = torch.randn(4, 3, 50, generator=g) * 3 * (torch.rand(4, 3, 50, generator=g) < 0.4)
  em = M.LaplaceEntropyModel(coding_rank=1)
  assert em.compress_ragged(list(x.reshape(-1, 50))).tolist() == list(em.compress(x).reshape(-1))
  em0 = M.PowerLawEntropyModel(coding_rank=0)
  items = [torch.tensor(3.2), torch.tensor(0.0), torch.tensor(-7.6)]
  strings = em0.compress_ragged(items)
  assert strings.tolist() == [em0.compress(t)[()] for t in items]
  assert [float(t) for t in em0.decompress_ragged(strings, [()] * 3)] == [3.0, 0.0, -8.0]
