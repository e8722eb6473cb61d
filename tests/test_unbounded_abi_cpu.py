"""CPU: the UnboundedIndexRange entries check their host-side arguments before any device work, with the
reference op's messages, so these run without a GPU.  The calls run on a worker thread: the library's last-error
message is per thread, and these tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

from compression_b200 import _lib, gen_ops

_P = C.c_void_p(256)  # never dereferenced: every call below is rejected first


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _arr(a):
  return a.ctypes.data_as(C.c_void_p)


def _args(p=5, w=2, debug=1, cdf_shape=(1, 4), cdf_rank=2, size_len=1, offset_len=1, items=(0, 3), null=None):
  cs = np.asarray(cdf_shape, np.int64)
  it = np.asarray(items, np.int64)
  ptrs = [None if i == null else _P for i in range(6)]  # data or bytes, index, cdf, cdf_size, offset, out
  keep = (cs, it)
  return ptrs, cs, it, keep, (p, w, debug, cdf_rank, size_len, offset_len)


def _encode(**kw):
  ptrs, cs, it, _, (p, w, debug, rank, sl, ol) = _args(**kw)
  h, total = C.c_void_p(), C.c_int64(0)
  return _lib.lib().tfcb_unbounded_index_range_encode_ragged(
      ptrs[0], ptrs[1], it.size - 1, _arr(it), ptrs[2], _arr(cs), rank, ptrs[3], sl, ptrs[4], ol, p, w, debug,
      ptrs[5], None, C.byref(h), C.byref(total))


def _decode(**kw):
  ptrs, cs, it, _, (p, w, debug, rank, sl, ol) = _args(**kw)
  return _lib.lib().tfcb_unbounded_index_range_decode_ragged(
      ptrs[0], _P, it.size - 1, _arr(it), ptrs[1], ptrs[2], _arr(cs), rank, ptrs[3], sl, ptrs[4], ol, p, w, debug,
      ptrs[5], None)


CASES = [
    (dict(p=0), "`precision` must be in [1, 16]"),
    (dict(p=17), "`precision` must be in [1, 16]"),
    (dict(w=0), "`overflow_width` must be in [1, 16]"),
    (dict(w=17), "`overflow_width` must be in [1, 16]"),
    (dict(debug=2), "`debug_level` must be 0 or 1"),
    (dict(cdf_rank=1, cdf_shape=(4,)), "'cdf' should be 2-D"),
    (dict(cdf_shape=(1, 2)), "cdf.dim_size(1) >= 3"),
    (dict(size_len=2), "'cdf_size' should be 1-D and its length should match the number of rows"),
    (dict(offset_len=2), "'offset' should be 1-D and its length should match the number of rows"),
    (dict(items=(1, 3)), "symbol_offsets[0] must be 0"),
    (dict(items=(0, 3, 2)), "symbol_offsets must be non-decreasing"),
    (dict(items=(0,)), "`n_streams` must be positive"),
]


@pytest.mark.parametrize("op", [_encode, _decode])
@pytest.mark.parametrize("kw,msg", CASES)
def test_rejects_bad_arguments_without_a_device(op, kw, msg):
  with pytest.raises(_lib.InvalidArgumentError) as e:
    _on_worker(lambda: _lib.check(op(**kw)))
  assert msg in str(e.value)


@pytest.mark.parametrize("op", [_encode, _decode])
@pytest.mark.parametrize("null", range(6))
def test_rejects_null_pointers_without_a_device(op, null):
  with pytest.raises(_lib.InvalidArgumentError, match="null"):
    _on_worker(lambda: _lib.check(op(null=null)))


def test_empty_items_need_no_tables():
  # no element, so no table is read: only the output pointers matter (still no device work before the check)
  with pytest.raises(_lib.InvalidArgumentError, match="null"):
    _on_worker(lambda: _lib.check(_encode(items=(0, 0), null=5)))


_CDF = np.array([[0, 16, 18, 32]], np.int32)


@pytest.mark.parametrize("kw,msg", [
    (dict(data=np.zeros((2, 3), np.int32), index=np.zeros((3, 2), np.int32)),
     "`data` and `index` should have the same shape"),
    (dict(cdf=np.zeros(4, np.int32)), "'cdf' should be 2-D"),
    (dict(cdf=np.zeros((1, 2), np.int32)), "cdf.dim_size(1) >= 3"),
    (dict(cdf_size=np.zeros((1, 1), np.int32)), "'cdf_size' should be 1-D"),
    (dict(cdf_size=np.zeros(2, np.int32)), "should match the number of rows"),
    (dict(offset=np.zeros((1, 1), np.int32)), "'offset' should be 1-D"),
    (dict(offset=np.zeros(2, np.int32)), "should match the number of rows"),
    (dict(precision=0), "`precision` must be in [1, 16]"),
    (dict(overflow_width=17), "`overflow_width` must be in [1, 16]"),
    (dict(debug_level=2), "`debug_level` must be 0 or 1"),
])
def test_op_shape_checks_come_first(kw, msg):
  args = dict(data=np.zeros(3, np.int32), index=np.zeros(3, np.int32), cdf=_CDF, cdf_size=np.array([4], np.int32),
              offset=np.array([1], np.int32), precision=5, overflow_width=2, debug_level=1)
  args.update(kw)
  with pytest.raises(_lib.InvalidArgumentError) as e:
    gen_ops.unbounded_index_range_encode(**args)
  assert msg in str(e.value)
  if "data" not in kw:
    del args["data"]
    with pytest.raises(_lib.InvalidArgumentError) as e:
      gen_ops.unbounded_index_range_decode(b"", **args)
    assert msg in str(e.value)


def test_encoded_must_be_a_scalar():
  with pytest.raises(_lib.InvalidArgumentError, match="`encoded` should be a scalar"):
    gen_ops.unbounded_index_range_decode([b"", b""], np.zeros(3, np.int32), _CDF, [4], [1], 5, 2)
