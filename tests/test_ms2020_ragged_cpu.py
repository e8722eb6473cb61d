"""CPU: tfcb_compress_ragged_decoded (a ragged compress that also writes the decoded values) checks its host-side
arguments before any device work, so these run without a GPU.  The calls run on a worker thread: the library's
last-error message is per thread, and these tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

from compression_b200 import _lib


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


LOOKUP = np.asarray([-12, 0, 1000, 3096, 4096, 4, 0, 4, 12, 16], np.int32)  # overflow row at precision 12, one at 4
DEV = C.c_void_p(8)  # never dereferenced: every case fails before device work


def _compress_ragged_decoded(offsets, n_streams=None, value_is_f32=1, cdf_offset=DEV, decoded=DEV):
  offs = np.ascontiguousarray(offsets, dtype=np.int64)
  h, total = C.c_void_p(), C.c_int64(0)
  n = len(offs) - 1 if n_streams is None else n_streams
  return _lib.lib().tfcb_compress_ragged_decoded(LOOKUP.ctypes.data_as(C.c_void_p), LOOKUP.size, 0, n,
                                                 offs.ctypes.data_as(C.c_void_p) if offs.size else None, None, DEV,
                                                 value_is_f32, None, cdf_offset, DEV, None, C.byref(h),
                                                 C.byref(total), decoded)


@pytest.mark.parametrize("kwargs, message", [
    (dict(value_is_f32=0), r"decoded values need float32 values \(`value_is_f32` is 0\)"),
    (dict(decoded=None), "`decoded` is null"),
    (dict(cdf_offset=None), "`cdf_offset` is null"),
])
def test_rejects_what_cannot_be_decoded_without_a_device(kwargs, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(_compress_ragged_decoded([0, 4, 9], **kwargs)))


@pytest.mark.parametrize("offsets, n_streams, message", [
    ([0], 0, "`n_streams` must be positive"),
    ([], 2, "`symbol_offsets` is null"),
    ([1, 4], None, r"symbol_offsets\[0\] must be 0"),
    ([0, 4, 3, 9], None, r"non-decreasing: symbol_offsets\[1\]=4 > symbol_offsets\[2\]=3"),
    ([0, 10, 10 + 450_000_000], None, r"may not exceed 2\^31 16-bit words \(stream 1\)"),
])
def test_rejects_bad_offsets_like_compress_ragged(offsets, n_streams, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(_compress_ragged_decoded(offsets, n_streams)))
