"""CPU: the universal-quantisation entry points of the C ABI check their host-side arguments before any device work,
so these run without a GPU.  The calls run on a worker thread: the library's last-error message is per thread, and
these tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

from compression_b200 import _lib


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _coding_tensors(offsets, n_items=None, levels=15, prior_size=4, ranges=None, n_ranges=None, out=C.c_void_p(8),
                    indexes=None):
  offs = np.ascontiguousarray(offsets, dtype=np.int64)
  rng = None if ranges is None else np.ascontiguousarray(ranges, dtype=np.int64)
  n = len(offs) - 1 if n_items is None else n_items
  nr = (0 if rng is None else rng.size) if n_ranges is None else n_ranges
  return _lib.lib().tfcb_universal_coding_tensors(
      n, offs.ctypes.data_as(C.c_void_p) if offs.size else None, 1234, 1234, levels, prior_size, indexes, 0,
      None if rng is None else rng.ctypes.data_as(C.c_void_p), nr, out, out, 0, None)


@pytest.mark.parametrize("offsets, n_items, message", [
    ([0], 0, "`n_items` must be positive"),
    ([0, 4], -1, "`n_items` must be positive"),
    ([], 2, "`item_offsets` is null"),
    ([1, 4], None, r"item_offsets\[0\] must be 0"),
    ([0, 4, 3, 9], None, r"non-decreasing: item_offsets\[1\]=4 > item_offsets\[2\]=3"),
])
def test_coding_tensors_reject_bad_item_offsets_without_a_device(offsets, n_items, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(_coding_tensors(offsets, n_items)))


@pytest.mark.parametrize("kwargs, message", [
    (dict(levels=0), r"`num_noise_levels` must be in \[1, 2\^31\): 0"),
    (dict(levels=1 << 31), r"`num_noise_levels` must be in \[1, 2\^31\)"),
    (dict(prior_size=0), "`prior_size` must be positive: 0"),
    (dict(ranges=[4] * 9), r"`n_ranges` must be in \[1, 8\]: 9"),
    (dict(ranges=[4, 0, 3]), r"index_ranges\[1\] must be positive: 0"),
    (dict(n_ranges=2), "`index_ranges` is null"),
    (dict(out=None), "null pointer"),
    (dict(ranges=[4, 3]), "null pointer"),  # indexed mode without indexes
])
def test_coding_tensors_reject_bad_models_without_a_device(kwargs, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(_coding_tensors([0, 4, 9], **kwargs)))


def test_empty_items_need_no_device_or_buffers():
  assert _on_worker(lambda: _coding_tensors([0, 0, 0], out=None)) == _lib.OK
  assert _on_worker(lambda: _lib.lib().tfcb_stateless_uniform_int(None, 0, 0, 0, 15, None)) == _lib.OK


@pytest.mark.parametrize("n, maxval, message", [
    (-1, 15, "`n` must be non-negative: -1"),
    (4, 0, "`maxval` must be positive: 0"),
    (4, -3, "`maxval` must be positive: -3"),
    (4, 15, "null pointer"),
])
def test_stateless_uniform_int_rejects_bad_arguments_without_a_device(n, maxval, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(_lib.lib().tfcb_stateless_uniform_int(None, n, 0, 0, maxval, None)))


def test_python_layer_rejects_an_empty_batch_and_bad_maxval():
  import torch
  from compression_b200 import functional as F
  with pytest.raises(_lib.InvalidArgumentError, match="at least one stream"):
    F.universal_coding_tensors([], 15, torch.float32, "cpu", prior_size=4)
  with pytest.raises(_lib.InvalidArgumentError, match="`maxval` must be positive"):
    F.stateless_uniform_int(4, (0, 0), 0, "cpu")
  with pytest.raises(_lib.InvalidArgumentError, match="the kernel reads float32 or float64"):
    F.universal_coding_tensors([2], 15, torch.float32, "cpu", indexes=torch.zeros(2, 1, dtype=torch.float16),
                               index_ranges=(3,))
