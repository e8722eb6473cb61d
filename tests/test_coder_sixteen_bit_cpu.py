"""CPU: which 16-bit bottleneck calls run on the 16-bit range-coder entries (functional._coder16), and the host-side
argument checks of those entries (tfcb_compress_16bit, tfcb_compress_ragged_16bit, tfcb_decode_16bit,
tfcb_decode_ragged_16bit), which reject bad arguments before any device work.  The routing function reads dtypes,
shapes and devices only, so stand-ins with those three attributes take the place of CUDA tensors.  The library calls
run on a worker thread: its last-error message is per thread, and these tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C
import types

import numpy as np
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import functional as F

CUDA = torch.device("cuda", 0)
_P = C.c_void_p(256)  # never dereferenced: every call below is rejected first


def _t(shape, dtype, device=CUDA):
  return types.SimpleNamespace(shape=torch.Size(shape), dtype=dtype, device=device)


# ------------------------------------------------------------------------------------------------
# Routing
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_routing_accepts(dtype):
  shape = (2, 5, 7)
  idx = _t(shape, torch.int32)
  assert F._coder16(dtype, CUDA, None, None, shape)                          # channel, no offsets
  assert F._coder16(dtype, CUDA, _t((7,), torch.float32), None, shape)       # channel, quantisation offsets
  assert F._coder16(dtype, "cuda:0", _t((7,), torch.float32), None, None)    # (shape unused in channel mode)
  assert F._coder16(dtype, CUDA, None, idx, shape)                           # index, no loc
  assert F._coder16(dtype, CUDA, _t(shape, dtype), idx, shape)               # loc in the bottleneck's type
  assert F._coder16(dtype, CUDA, _t(shape, torch.float32), idx, shape)       # float32 loc


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_routing_rejects(dtype):
  shape = (2, 5, 7)
  idx = _t(shape, torch.int32)
  other = torch.bfloat16 if dtype == torch.float16 else torch.float16
  cpu = torch.device("cpu")
  for bad in (torch.float32, torch.float64, torch.int32):                    # not a 16-bit bottleneck
    assert not F._coder16(bad, CUDA, None, None, shape)
  assert not F._coder16(dtype, cpu, None, None, shape)                       # host tensors
  assert not F._coder16(dtype, CUDA, _t((7,), torch.float32, cpu), None, shape)
  assert not F._coder16(dtype, CUDA, None, _t(shape, torch.int32, cpu), shape)
  assert not F._coder16(dtype, CUDA, _t(shape, dtype, torch.device("cuda", 1)), idx, shape)
  assert not F._coder16(dtype, CUDA, _t((7,), dtype), None, shape)           # channel offsets not float32
  assert not F._coder16(dtype, CUDA, _t((7,), torch.float64), None, shape)
  assert not F._coder16(dtype, CUDA, _t((1, 7), torch.float32), None, shape)
  assert not F._coder16(dtype, CUDA, _t(shape, torch.float64), idx, shape)   # loc of another type
  assert not F._coder16(dtype, CUDA, _t(shape, other), idx, shape)
  assert not F._coder16(dtype, CUDA, _t((5, 7), dtype), idx, shape)          # loc broadcast from another shape
  assert not F._coder16(dtype, CUDA, _t((), torch.float32), idx, shape)
  assert not F._coder16(dtype, CUDA, None, _t((2, 35), torch.int32), shape)  # index not shaped like the bottleneck


def test_universal_models_keep_the_unfused_path():
  from compression_b200 import entropy_models as E
  assert E.ContinuousBatchedEntropyModel._coder16_models
  assert E.ContinuousIndexedEntropyModel._coder16_models
  assert E.LocationScaleIndexedEntropyModel._coder16_models
  assert not E.UniversalBatchedEntropyModel._coder16_models
  assert not E.UniversalIndexedEntropyModel._coder16_models


# ------------------------------------------------------------------------------------------------
# Host-side argument checks of the entries: no launch, TFCB_INVALID_ARGUMENT
# ------------------------------------------------------------------------------------------------
_LOOKUP = np.array([-12, 0, 2048, 4096], dtype=np.int32)


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _rejects(call, match):
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _on_worker(lambda: _lib.check(call()))
  assert _lib.launch_count() == n0


def _compress(index=None, value=_P, dtype=1, loc=None, loc_dtype=0, coff=_P, n=4, offsets=_P, out=True):
  h, total = C.c_void_p(), C.c_int64()
  return _lib.lib().tfcb_compress_16bit(
      _LOOKUP.ctypes.data_as(C.c_void_p), _LOOKUP.size, 0, 2, index, value, dtype, loc, loc_dtype, coff, n, offsets,
      None, C.byref(h) if out else None, C.byref(total))


_OFFS = np.array([0, 3, 3, 8], dtype=np.int64)


def _compress_ragged(index=None, value=_P, dtype=1, loc=None, loc_dtype=0, coff=_P, offs=_OFFS, offsets=_P,
                     decoded=None, n_streams=3):
  h, total = C.c_void_p(), C.c_int64()
  return _lib.lib().tfcb_compress_ragged_16bit(
      _LOOKUP.ctypes.data_as(C.c_void_p), _LOOKUP.size, 0, n_streams,
      None if offs is None else offs.ctypes.data_as(C.c_void_p), index, value, dtype, loc, loc_dtype, coff, decoded,
      offsets, None, C.byref(h), C.byref(total))


@pytest.mark.parametrize("entry", [_compress, _compress_ragged])
@pytest.mark.parametrize("dtype", [0, 3, -1])
def test_rejects_unknown_dtypes(entry, dtype):
  _rejects(lambda: entry(dtype=dtype), "`dtype` must be 1")


@pytest.mark.parametrize("entry", [_compress, _compress_ragged])
def test_rejects_unsupported_loc_dtypes(entry):
  _rejects(lambda: entry(loc=_P, loc_dtype=1), "in channel mode")            # channel offsets are float32
  _rejects(lambda: entry(loc=_P, loc_dtype=2, dtype=2), "in channel mode")
  _rejects(lambda: entry(index=_P, loc=_P, loc_dtype=2, dtype=1), "loc_dtype")  # another 16-bit type
  _rejects(lambda: entry(index=_P, loc=_P, loc_dtype=3, dtype=1), "loc_dtype")
  _rejects(lambda: entry(index=_P, loc=_P, loc_dtype=-1, dtype=2), "loc_dtype")


@pytest.mark.parametrize("entry", [_compress, _compress_ragged])
def test_rejects_null_pointers(entry):
  _rejects(lambda: entry(coff=None), "cdf_offset")
  _rejects(lambda: entry(index=_P, coff=None), "cdf_offset")
  _rejects(lambda: entry(value=None), "`value` is null")
  _rejects(lambda: entry(offsets=None), "offsets")


def test_compress_rejects_bad_sizes_and_outputs():
  _rejects(lambda: _compress(n=-1), "negative element count")
  _rejects(lambda: _compress(out=False), "null output")


def test_ragged_rejects_bad_symbol_offsets():
  _rejects(lambda: _compress_ragged(offs=None), "symbol_offsets")
  _rejects(lambda: _compress_ragged(offs=np.array([1, 3, 3, 8], dtype=np.int64)), r"symbol_offsets\[0\]")
  _rejects(lambda: _compress_ragged(offs=np.array([0, 3, 2, 8], dtype=np.int64)), "non-decreasing")
  _rejects(lambda: _compress_ragged(n_streams=0), "n_streams")


def test_decode_entries_reject_a_null_handle():
  L = _lib.lib()
  _rejects(lambda: L.tfcb_decode_16bit(None, None, _P, 1, None, 0, _P, 4, None), "not a decoder")
  _rejects(lambda: L.tfcb_decode_ragged_16bit(None, _OFFS.ctypes.data_as(C.c_void_p), None, _P, 1, None, 0, _P,
                                              None), "not a decoder")


def test_functional_checks_lengths_before_the_library():
  """Operand lengths that do not match the symbols are refused in Python, before any library call."""
  n0 = _lib.launch_count()
  v = torch.zeros(8, dtype=torch.float16)
  coff = torch.zeros(2, dtype=torch.int32)
  with pytest.raises(_lib.InvalidArgumentError, match="`index` has 7"):
    F.compress_16bit((2,), _LOOKUP, v, None, coff, index=torch.zeros(7, dtype=torch.int32))
  with pytest.raises(_lib.InvalidArgumentError, match="`loc` has 9"):
    F.compress_16bit((2,), _LOOKUP, v, torch.zeros(9, dtype=torch.float16), coff, index=torch.zeros(8, dtype=torch.int32))
  with pytest.raises(_lib.InvalidArgumentError, match="`loc` has 3"):
    F.compress_16bit((2,), _LOOKUP, v, torch.zeros(3), coff)
  with pytest.raises(_lib.InvalidArgumentError, match="`value` has 8"):
    F.compress_ragged_16bit(_LOOKUP, [3, 4], v, None, coff)
  with pytest.raises(_lib.InvalidArgumentError, match="`index` has 6"):
    F.compress_ragged_16bit(_LOOKUP, [3, 5], v, None, coff, index=torch.zeros(6, dtype=torch.int32))
  assert _lib.launch_count() == n0
