"""CPU: the ragged run-length entry points of the C ABI check their host-side arguments before any device work, so
these run without a GPU.  The calls run on a worker thread: the library's last-error message is per thread, and these
tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest

from compression_b200 import _lib

FAKE = C.c_void_p(8)  # never dereferenced: every call below fails its host-side checks first


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _offs(offsets):
  offs = np.ascontiguousarray(offsets, dtype=np.int64)
  return offs, (offs.ctypes.data_as(C.c_void_p) if offs.size else None)


def _encode(offsets, n_units=None, rl=-1, mg=-1, data=FAKE, out=True):
  offs, p = _offs(offsets)
  n = len(offs) - 1 if n_units is None else n_units
  h, total = C.c_void_p(), C.c_int64(0)
  return _lib.lib().tfcb_run_length_encode_ragged(data, n, p, rl, mg, 0, FAKE, None, C.byref(h) if out else None,
                                                  C.byref(total))


def _decode(offsets, n_units=None, rl=-1, mg=-1, data=FAKE, code=FAKE):
  offs, p = _offs(offsets)
  n = len(offs) - 1 if n_units is None else n_units
  return _lib.lib().tfcb_run_length_decode_ragged(code, FAKE, n, p, rl, mg, 0, data, None)


BAD_OFFSETS = [
    ([0], 0, "`n_units` must be positive"),
    ([0, 4], -3, "`n_units` must be positive"),
    ([], 2, "`unit_offsets` is null"),
    ([2, 4], None, r"unit_offsets\[0\] must be 0: 2"),
    ([0, 4, 3, 9], None, r"non-decreasing: unit_offsets\[1\]=4 > unit_offsets\[2\]=3"),
    ([0, 2**30, 2**31], None, r"2147483648 elements; at most 2\^31 - 1"),
]


@pytest.mark.parametrize("offsets, n_units, message", BAD_OFFSETS)
@pytest.mark.parametrize("call", [_encode, _decode], ids=["encode", "decode"])
def test_ragged_run_length_rejects_bad_unit_offsets_without_a_device(call, offsets, n_units, message):
  with pytest.raises(_lib.InvalidArgumentError, match=message):
    _on_worker(lambda: _lib.check(call(offsets, n_units)))


@pytest.mark.parametrize("rl, mg", [(32, 0), (0, 32), (40, -1)])
@pytest.mark.parametrize("call", [_encode, _decode], ids=["encode", "decode"])
def test_ragged_run_length_rejects_wide_rice_parameters(call, rl, mg):
  with pytest.raises(_lib.InvalidArgumentError, match=r"Rice parameter > 31"):
    _on_worker(lambda: _lib.check(call([0, 3, 5], rl=rl, mg=mg)))


def test_ragged_run_length_rejects_null_pointers():
  for fn in (lambda: _encode([0, 3], data=None), lambda: _encode([0, 3], out=False),
             lambda: _decode([0, 3], data=None), lambda: _decode([0, 3], code=None)):
    with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
      _on_worker(lambda: _lib.check(fn()))


def test_write_and_destroy_need_an_encoder():
  with pytest.raises(_lib.InvalidArgumentError, match="not a run-length encoder"):
    _on_worker(lambda: _lib.check(_lib.lib().tfcb_run_length_write(None, FAKE, None)))
  _lib.lib().tfcb_run_length_encoder_destroy(None)


def test_python_layer_rejects_an_empty_batch_and_a_length_mismatch():
  import torch
  from compression_b200 import functional as F
  with pytest.raises(_lib.InvalidArgumentError, match="at least one stream"):
    F.run_length_encode_ragged(torch.zeros(0, dtype=torch.int32), [], -1, -1, False)
  with pytest.raises(_lib.InvalidArgumentError, match="at least one stream"):
    F.run_length_decode_ragged([], [], -1, -1, False)


def test_models_check_item_ranks_before_coding():
  import torch
  from compression_b200 import run_length_models as M
  em = M.LaplaceEntropyModel(coding_rank=2)
  with pytest.raises(ValueError, match="exactly 2 dimensions"):
    em.compress_ragged([torch.zeros(3, 4), torch.zeros(5)])
  with pytest.raises(ValueError, match="`bottlenecks` is empty"):
    em.compress_ragged([])
  with pytest.raises(ValueError, match="exactly 2 dimensions"):
    em.decompress_ragged([b"", b""], [(3, 4), (2, 2, 2)])
