"""CPU: the ragged entry points of the C ABI check their host-side arguments before any device work, so these
run without a GPU.  The calls run on a worker thread: the library's last-error message is per thread, and these
tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

from compression_b200 import _lib


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


LOOKUP = np.asarray([-12, 0, 1000, 3096, 4096, 4, 0, 4, 12, 16], np.int32)  # overflow row at precision 12, one at 4


def _compress_ragged(offsets, n_streams=None, lookup=LOOKUP, out=True):
  offs = np.ascontiguousarray(offsets, dtype=np.int64)
  h, total = C.c_void_p(), C.c_int64(0)
  n = len(offs) - 1 if n_streams is None else n_streams
  return _lib.lib().tfcb_compress_ragged(lookup.ctypes.data_as(C.c_void_p), lookup.size, 0, n,
                                         offs.ctypes.data_as(C.c_void_p) if offs.size else None, None, None, 0,
                                         None, None, C.c_void_p(8), None, C.byref(h) if out else None,
                                         C.byref(total))


@pytest.mark.parametrize("offsets, n_streams, message", [
    ([0], 0, "`n_streams` must be positive"),
    ([0, 4], -1, "`n_streams` must be positive"),
    ([], 2, "`symbol_offsets` is null"),
    ([1, 4], None, r"symbol_offsets\[0\] must be 0"),
    ([0, 4, 3, 9], None, r"non-decreasing: symbol_offsets\[1\]=4 > symbol_offsets\[2\]=3"),
    # 12 + 65 bits per symbol at most: 2^31 words hold fewer than 446 M symbols of this table
    ([0, 10, 10 + 450_000_000], None, r"may not exceed 2\^31 16-bit words \(stream 1\)"),
])
def test_compress_ragged_rejects_bad_offsets_without_a_device(offsets, n_streams, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(_compress_ragged(offsets, n_streams)))


def test_compress_ragged_checks_outputs_and_table_first():
  with pytest.raises(_lib.InvalidArgumentError, match="null output pointer"):
    _on_worker(lambda: _lib.check(_compress_ragged([0, 4], out=False)))
  with pytest.raises(_lib.InvalidArgumentError, match="CDF must start with 0"):
    _on_worker(lambda: _lib.check(_compress_ragged([0, 4], lookup=np.asarray([4, 1, 16], np.int32))))


def test_decode_ragged_needs_a_decoder():
  offs = np.asarray([0, 3], np.int64)
  with pytest.raises(_lib.InvalidArgumentError, match="not a decoder"):
    _on_worker(lambda: _lib.check(_lib.lib().tfcb_decode_ragged(None, offs.ctypes.data_as(C.c_void_p), None, None, 0,
                                                                None, None, None)))


def test_python_layer_rejects_an_empty_batch():
  import torch
  from compression_b200 import functional as F
  with pytest.raises(_lib.InvalidArgumentError, match="at least one stream"):
    F.compress_ragged(LOOKUP, [], torch.zeros(0, dtype=torch.int32))
