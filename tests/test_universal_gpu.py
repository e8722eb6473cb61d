"""GPU: universal quantisation's coding tensors from one kernel (csrc/universal.cu) and the ragged forms of the two
universal entropy models.

The CPU path (entropy_models._philox4x32 and the torch operations of universal.py:30-62,147-170,446-466) is the
checker: on a CUDA device the noise levels, table indexes and offsets must equal it bit for bit."""
import numpy as np
import pytest
import torch

import oracle

pytestmark = pytest.mark.gpu

M32 = 0xFFFFFFFF


@pytest.fixture(scope="module")
def E():
  from compression_b200 import entropy_models
  return entropy_models


@pytest.fixture(scope="module")
def D():
  from compression_b200 import distributions
  return distributions


def _batched(E, D, levels=15, dtype=None, compression=True):
  prior = D.NoisyLogistic(loc=torch.zeros(6), scale=torch.linspace(1., 8., 6))
  return E.UniversalBatchedEntropyModel(prior, coding_rank=2, compression=compression, num_noise_levels=levels,
                                        bottleneck_dtype=dtype)


def _indexed(E, D, levels=7, dtype=None, prior_dtype=torch.float32, coding_rank=2):
  return E.UniversalIndexedEntropyModel(
      D.NoisyLogistic, (5, 3), dict(loc=lambda i: i[..., 0] - 2., scale=lambda i: 1. + i[..., 1]),
      coding_rank=coding_rank, compression=True, num_noise_levels=levels, bottleneck_dtype=dtype,
      prior_dtype=prior_dtype)


# ------------------------------------------------------------------------------------------------
# The noise draw
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("maxval", [1, 2, 7, 15, 255, 65537])
def test_kernel_draws_equal_the_cpu_philox(E, maxval):
  for seed, n in (((0, 0), 1), ((1234, 1234), 4_099), ((M32, M32), 33), ((7, M32), 2_500_003), ((M32, 0), 6)):
    got = E.stateless_uniform_int((n,), seed, maxval, "cuda")
    assert got.dtype == torch.int32 and got.is_cuda
    assert torch.equal(got.cpu(), E.stateless_uniform_int((n,), seed, maxval)), (seed, n)


def test_kernel_draw_keeps_the_shape_and_large_moduli(E):
  got = E.stateless_uniform_int((3, 0, 5), (1, 2), 15, torch.device("cuda"))
  assert got.shape == (3, 0, 5)
  for maxval in (1 << 31, (1 << 32) - 1, 1 << 32, 1 << 40):  # > 2^32: the raw word, wrapped to int32 like torch's cast
    assert torch.equal(E.stateless_uniform_int((2, 7), (9, 9), maxval, "cuda").cpu(),
                       E.stateless_uniform_int((2, 7), (9, 9), maxval))


# ------------------------------------------------------------------------------------------------
# Coding tensors: CUDA against the CPU path, bit for bit
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16])
@pytest.mark.parametrize("levels", [1, 7, 15, 65537])
def test_batched_coding_tensors_equal_the_cpu_path(E, D, dtype, levels):
  em = _batched(E, D, levels, dtype, compression=False)
  for shape in ((), (1,), (333,), (17, 5)):
    flat, off = em._compute_indexes_and_offset(shape, torch.device("cuda"))
    want_flat, want_off = em._compute_indexes_and_offset(shape, torch.device("cpu"))
    assert flat.dtype == torch.int32 and off.dtype == dtype and flat.shape == shape + (6,)
    assert torch.equal(flat.cpu(), want_flat) and torch.equal(off.cpu(), want_off), shape


def _cpu_coding_tensors(em, indexes):
  return em._coding_tensors(indexes.cpu(), torch.device("cpu"))


def _torch_coding_tensors(em, indexes, E):
  """The torch operations of _coding_tensors on the indexes' own device."""
  idx = em._normalize_indexes(E._add_offset_indexes(indexes.to(em.prior_dtype), em._num_noise_levels))
  return em._flatten_indexes(idx), em._offset_from_indexes(idx)


@pytest.mark.parametrize("prior_dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16])
def test_indexed_coding_tensors_equal_the_cpu_path(E, D, prior_dtype, dtype):
  em = _indexed(E, D, 7, dtype, prior_dtype)
  g = torch.Generator().manual_seed(3)
  for shape in ((1,), (4, 9), (3, 50, 11)):
    idx = torch.rand(shape + (2,), generator=g, dtype=torch.float64) * 12 - 4  # negative, fractional, out of range
    idx.view(-1, 2)[::7, 0] = 4.9999
    idx.view(-1, 2)[::5, 1] = -0.5
    for indexes in (idx, idx.to(torch.int64)):
      flat, off = em._coding_tensors(indexes.cuda(), torch.device("cuda"))
      want_flat, want_off = _cpu_coding_tensors(em, indexes)
      assert flat.shape == shape and off.dtype == dtype
      assert torch.equal(flat.cpu(), want_flat) and torch.equal(off.cpu(), want_off), shape
  # NaN: clipping keeps it and the cast gives what torch's cast gives on the same device
  nan_idx = torch.tensor([[[float("nan"), 1.], [2., float("nan")], [-1., 9.]]], dtype=prior_dtype, device="cuda")
  flat, off = em._coding_tensors(nan_idx, torch.device("cuda"))
  want_flat, want_off = _torch_coding_tensors(em, nan_idx, E)
  assert torch.equal(flat, want_flat) and torch.equal(off, want_off)


def test_large_level_counts_and_many_index_dimensions(E, D):
  """Levels beyond float32's integers are rounded in prior_dtype before clipping and flattening, as the torch path
  does; three index dimensions use the strides of (levels,) + index_ranges."""
  em = E.UniversalIndexedEntropyModel(D.NoisyLogistic, (3, 2, 4), dict(loc=lambda i: i[..., 0], scale=lambda i: 1.),
                                      coding_rank=1, compression=False, num_noise_levels=(1 << 25) + 3)
  idx = torch.rand(5000, 3, generator=torch.Generator().manual_seed(1)) * 6 - 1
  flat, off = em._coding_tensors(idx.cuda(), torch.device("cuda"))
  want_flat, want_off = _cpu_coding_tensors(em, idx)
  assert torch.equal(flat.cpu(), want_flat) and torch.equal(off.cpu(), want_off)


def test_forward_at_inference_uses_the_same_offsets(E, D):
  em = _batched(E, D)
  x = torch.randn(3, 500, 6) * 4
  got, bits = em(x.cuda(), training=False)
  want, want_bits = em(x, training=False)
  assert torch.equal(got.cpu(), want)
  emi = _indexed(E, D)
  idx = torch.rand(2, 40, 9, 2) * torch.tensor([5., 3.])
  xi = torch.randn(2, 40, 9) * 3
  got, _ = emi(xi.cuda(), idx.cuda(), training=False)
  want, _ = emi(xi, idx, training=False)
  assert torch.equal(got.cpu(), want)


# ------------------------------------------------------------------------------------------------
# No torch Philox on the device, and one launch per call
# ------------------------------------------------------------------------------------------------
def test_cuda_paths_never_call_the_torch_philox(E, D, monkeypatch):
  from compression_b200 import _lib
  from compression_b200 import functional as F
  em, emi = _batched(E, D), _indexed(E, D)
  x = (torch.randn(4, 300, 6) * 5).cuda()
  xi = (torch.randn(3, 20, 7) * 3).cuda()
  ind = (torch.rand(3, 20, 7, 2) * torch.tensor([5., 3.])).cuda()
  idx_full, off_full = em._unit_coding_tensors(4, (300,), x.device)

  def boom(*_):
    raise AssertionError("torch Philox called on a CUDA path")
  monkeypatch.setattr(E, "_philox4x32", boom)
  strings = em.compress(x)
  em.decompress(strings, (300,))
  em(x, training=False)
  emi.decompress(emi.compress(xi, ind), ind)
  emi(xi, ind, training=False)
  em.decompress_ragged(em.compress_ragged([x[0], x[1, :7]]), [(300,), (7,)])
  emi.decompress_ragged(emi.compress_ragged([xi[0], xi[1, :3]], [ind[0], ind[1, :3]]), [ind[0], ind[1, :3]])

  # compress = the coder's launches + exactly one
  def launches(fn):
    n0 = _lib.launch_count()
    out = fn()
    return _lib.launch_count() - n0, out
  flat_i, off_i = emi._coding_tensors(ind, xi.device)
  coder, _ = launches(lambda: F.compress_f32((4,), em._lookup_host(), x, off_full, em.cdf_offset.cuda(),
                                             index=idx_full))
  n, again = launches(lambda: em.compress(x))
  assert n == coder + 1 and again.tolist() == strings.tolist()
  coder, want = launches(lambda: F.compress_f32((3,), emi._lookup_host(), xi, off_i, emi.cdf_offset.cuda(),
                                                index=flat_i))
  n, got = launches(lambda: emi.compress(xi, ind))
  assert n == coder + 1 and got.tolist() == want.tolist()


def test_batch_units_are_written_directly(E, D):
  """A batch of B units: B equal items from the kernel, equal to the broadcast of one unit."""
  em = _batched(E, D)
  for units, shape in ((1, (5,)), (3, (300,)), (7, (2, 9))):
    flat, off = em._unit_coding_tensors(units, shape, torch.device("cuda"))
    one_flat, one_off = em._compute_indexes_and_offset(shape, torch.device("cpu"))
    assert flat.shape == (units,) + shape + (6,)
    assert torch.equal(flat.cpu(), one_flat.expand_as(flat.cpu()))
    assert torch.equal(off.cpu(), one_off.expand_as(off.cpu()))


# ------------------------------------------------------------------------------------------------
# Ragged batches
# ------------------------------------------------------------------------------------------------
def _oracle_item(em, x, flat, off):
  sym = (torch.round(x.cpu() - off.cpu()).to(torch.int32) - em.cdf_offset.cpu()[flat.cpu().long()]).reshape(1, -1)
  return oracle.best().encode(em.cdf.cpu().numpy(), sym.numpy(), flat.cpu().reshape(1, -1).numpy().astype(np.int32))[0]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_batched_ragged_equals_per_item_calls(E, D, dtype):
  torch.manual_seed(0)
  em = _batched(E, D, 15, dtype)
  lens = (1, 17, 0, 300, 64, 3)
  xs = [(torch.randn(n, 6, device="cuda") * 6).to(dtype) for n in lens]
  strings = em.compress_ragged(xs)
  per_item = [em.compress(x).tolist()[0] if x.numel() else b"" for x in xs]
  assert strings.shape == (len(xs),) and strings.tolist() == per_item
  back = em.decompress_ragged(strings, [(n,) for n in lens])
  for x, b, s in zip(xs, back, per_item):
    assert b.dtype == dtype and b.shape == x.shape
    assert float((b - x).abs().max()) <= 0.5 + 1e-5 if x.numel() else True
    if x.numel():
      assert torch.equal(b, em.decompress([s], (x.shape[0],))[0])
  strings2, decoded = em.compress_ragged(xs, return_decoded=True)
  assert strings2.tolist() == strings.tolist()
  for a, b in zip(decoded, back):
    assert torch.equal(a, b)
  if dtype == torch.float32:  # the oracle's bytes for the symbols the model derives, item by item
    for x, s in zip(xs, per_item):
      if x.numel():
        flat, off = em._compute_indexes_and_offset((x.shape[0],), x.device)
        assert s == _oracle_item(em, x, flat, off)


@pytest.mark.parametrize("dtype, prior_dtype", [(torch.float32, torch.float32), (torch.float64, torch.float64),
                                                (torch.float32, torch.float16)])
def test_indexed_ragged_equals_per_item_calls(E, D, dtype, prior_dtype):
  """float16 indexes take the torch operations (their draw is the kernel's); the tables are built in float32."""
  torch.manual_seed(1)
  em = _indexed(E, D, 7, dtype, torch.float64 if prior_dtype == torch.float64 else torch.float32)
  em._prior_dtype = prior_dtype
  shapes = [(3, 5), (1, 1), (40, 7), (0, 3), (17, 2)]
  xs = [(torch.randn(s, device="cuda") * 4).to(dtype) for s in shapes]
  idx = [torch.rand(s + (2,), device="cuda") * torch.tensor([7., 5.], device="cuda") - 1 for s in shapes]
  strings = em.compress_ragged(xs, idx)
  per_item = [em.compress(x, i).tolist()[0] for x, i in zip(xs, idx)]
  assert strings.tolist() == per_item
  back = em.decompress_ragged(strings, idx)
  for x, i, b, s in zip(xs, idx, back, per_item):
    assert b.shape == x.shape and b.dtype == dtype
    assert torch.equal(b, em.decompress([s], i[None])[0] if x.numel() else b)
  strings2, decoded = em.compress_ragged(xs, idx, return_decoded=True)
  assert strings2.tolist() == per_item
  for a, b in zip(decoded, back):
    assert torch.equal(a, b)
  if dtype == torch.float32 and prior_dtype == torch.float32:
    for x, i, s in zip(xs, idx, per_item):
      if x.numel():
        flat, off = em._coding_tensors(i, x.device)
        assert s == _oracle_item(em, x, flat, off)


def test_ragged_items_are_not_a_stacked_batch(E, D):
  """compress of a stacked [B, ...] batch draws the indexed model's noise over the batch dimension too; a ragged list
  draws it per item."""
  em = _indexed(E, D, 7, coding_rank=1)
  x = torch.randn(4, 500, device="cuda") * 3
  ind = torch.rand(4, 500, 2, device="cuda") * 4
  stacked = em.compress(x, ind).tolist()
  ragged = em.compress_ragged(list(x), list(ind)).tolist()
  assert ragged == [em.compress(x[b], ind[b]).tolist()[0] for b in range(4)]
  assert ragged[0] == stacked[0] and ragged[1:] != stacked[1:]


def test_ragged_argument_errors(E, D):
  from compression_b200 import gen_ops
  em, emi = _batched(E, D), _indexed(E, D)
  with pytest.raises(ValueError, match="`bottlenecks` is empty"):
    em.compress_ragged([])
  with pytest.raises(ValueError, match=r"each item needs 2 dimensions ending in \(6,\): received shape \(4, 5\)"):
    em.compress_ragged([torch.zeros(3, 6), torch.zeros(4, 5)])
  with pytest.raises(ValueError, match=r"each item needs 2 dimensions ending in \(6,\): received shape \(6,\)"):
    em.compress_ragged([torch.zeros(6)])
  good = em.compress_ragged([torch.zeros(3, 6), torch.zeros(5, 6)])
  with pytest.raises(ValueError, match="2 strings for 3 items"):
    em.decompress_ragged(good, [(3,), (5,), (1,)])
  with pytest.raises(ValueError, match="`indexes` is empty"):
    emi.compress_ragged([], [])
  with pytest.raises(ValueError, match=r"each item needs 2 dimensions: received indexes for shape \(4,\)"):
    emi.compress_ragged([torch.zeros(4)], [torch.zeros(4, 2)])
  with pytest.raises(ValueError, match="do not match the indexes'"):
    emi.compress_ragged([torch.zeros(3, 4)], [torch.zeros(3, 5, 2)])
  with pytest.raises(ValueError, match="do not match the indexes'"):
    emi.compress_ragged([torch.zeros(3, 4), torch.zeros(1, 1)], [torch.zeros(3, 4, 2)])
  with pytest.raises(ValueError, match="needs a last dimension of 2"):
    emi.compress_ragged([torch.zeros(3, 4)], [torch.zeros(3, 4, 3)])
  goodi = emi.compress_ragged([torch.zeros(3, 4)], [torch.zeros(3, 4, 2)])
  with pytest.raises(ValueError, match="1 strings for 2 items"):
    emi.decompress_ragged(goodi, [torch.zeros(3, 4, 2), torch.zeros(1, 1, 2)])
  bad = [good.tolist()[0], good.tolist()[1] + b"\x01\x02\x03"]
  with pytest.raises(gen_ops.InvalidArgumentError, match="Sanity check failed"):
    em.decompress_ragged(bad, [(3,), (5,)])
  uncompressed = E.UniversalBatchedEntropyModel(D.NoisyLogistic(loc=torch.zeros(6), scale=torch.ones(6)), coding_rank=2)
  with pytest.raises(RuntimeError, match="compression=True"):
    uncompressed.compress_ragged([torch.zeros(3, 6)])
