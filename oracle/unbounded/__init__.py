"""ORACLE -- test infrastructure, NOT product code.

UnboundedIndexRangeEncode / UnboundedIndexRangeDecode (``cc/kernels/unbounded_index_range_coding_kernels.cc``) on the
CPU, in the two flavours of the parent package:

* ``port()`` -- ``oracle/unbounded/port.c`` over the C port's range coder (always available).
* ``ref()``  -- ``oracle/unbounded/ref_driver.cc`` around the reference's own ``RangeEncoder`` / ``RangeDecoder``,
  compiled in place into ``oracle/_ref/libubi_ref.so`` where the reference tree exists; the built ``.so`` travels
  with the tree.

Both restate the op loop and refuse, with :class:`oracle.OracleError`, every input on which the reference's loop is
undefined (DESIGN.md §3.8) instead of running it.  Only ``tests/``, ``oracle/make_unbounded_golden.py`` and
``tools/unbounded_bench.py`` use this package; ``compression_b200`` never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import List, Sequence

import numpy as np

from oracle import REFERENCE_ROOT, OracleError

_HERE = os.path.dirname(os.path.abspath(__file__))
_PORT_SO = os.path.join(_HERE, "libubi_port.so")
_REF_SO = os.path.join(os.path.dirname(_HERE), "_ref", "libubi_ref.so")


def build(want_ref: bool = True) -> None:
  """Compiles the port flavour and, when the reference tree is present, the reference flavour."""
  subprocess.run(["make", "-s", "-C", _HERE, "port"], check=True)
  if want_ref and os.path.exists(os.path.join(REFERENCE_ROOT, "tensorflow_compression/cc/lib/range_coder.cc")):
    subprocess.run(["make", "-s", "-C", _HERE, "ref", f"REFERENCE={REFERENCE_ROOT}"], check=True)


def _i32(a) -> np.ndarray:
  return np.ascontiguousarray(a, dtype=np.int32)


class UnboundedOracle:
  """ctypes front-end shared by both flavours (same entry points, other prefix)."""

  def __init__(self, path: str, prefix: str, kind: str):
    self.kind = kind
    self.path = path
    self._lib = C.CDLL(path)
    self._px = prefix
    self._fn("last_error", C.c_char_p, [])
    self._fn("hardware_threads", C.c_int, [])
    self._fn("unbounded_encode", C.c_int, [C.c_void_p] * 3 + [C.c_int64, C.c_void_p, C.c_int64, C.c_int64] +
             [C.c_void_p] * 2 + [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.c_int64])
    self._fn("unbounded_decode", C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int64, C.c_int64, C.c_void_p, C.c_void_p] + [C.c_int] * 4 +
             [C.c_void_p])

  def _fn(self, name, restype, argtypes):
    fn = getattr(self._lib, self._px + name)
    fn.restype = restype
    fn.argtypes = argtypes
    setattr(self, "_" + name, fn)

  def _err(self) -> str:
    return (self._last_error() or b"").decode()

  def hardware_threads(self) -> int:
    return int(self._hardware_threads())

  @staticmethod
  def _tables(cdf, cdf_size, offset):
    cdf, cdf_size, offset = _i32(cdf), _i32(cdf_size).reshape(-1), _i32(offset).reshape(-1)
    assert cdf.ndim == 2 and cdf.shape[1] >= 3 and cdf_size.size == offset.size == cdf.shape[0]
    return cdf, cdf_size, offset

  def encode_batch(self, data, index, lengths, cdf, cdf_size, offset, precision: int, overflow_width: int,
                   debug_level: int = 1, threads: int = 1) -> List[bytes]:
    """String u codes the next lengths[u] elements of the flat `data` / `index` (the reference flavour spreads the
    strings over its persistent thread pool).  Raises OracleError where the reference is undefined or its checks
    fail."""
    data, index = _i32(data).reshape(-1), _i32(index).reshape(-1)
    cdf, cdf_size, offset = self._tables(cdf, cdf_size, offset)
    item = np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))]).astype(np.int64)
    assert data.size == index.size == item[-1]
    k = item.size - 1
    w = int(overflow_width)
    K = (32 + w - 1) // w
    bits = int(precision) + w * (K // ((1 << w) - 1) + 1 + K)
    cap = int(item[-1]) * bits // 8 + 8 * k + 16
    so = np.zeros(k + 1, np.int64)
    out = np.empty(cap, np.uint8)
    rc = self._unbounded_encode(data.ctypes.data, index.ctypes.data, item.ctypes.data, k, cdf.ctypes.data,
                                cdf.shape[0], cdf.shape[1], cdf_size.ctypes.data, offset.ctypes.data, int(precision), w,
                                int(debug_level), int(threads), so.ctypes.data, out.ctypes.data, cap)
    if rc == 1:
      raise OracleError(self._err())
    assert rc == 0, "output bound exceeded"
    return [out[so[u]:so[u + 1]].tobytes() for u in range(k)]

  def decode_batch(self, strings: Sequence[bytes], index, lengths, cdf, cdf_size, offset, precision: int,
                   overflow_width: int, debug_level: int = 1, threads: int = 1) -> np.ndarray:
    """Flat int32 [sum(lengths)]: string u decoded into the next lengths[u] elements."""
    index = _i32(index).reshape(-1)
    cdf, cdf_size, offset = self._tables(cdf, cdf_size, offset)
    item = np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))]).astype(np.int64)
    assert index.size == item[-1] and len(strings) == item.size - 1
    so = np.concatenate([[0], np.cumsum([len(s) for s in strings])]).astype(np.int64)
    buf = np.frombuffer(b"".join(bytes(s) for s in strings) + b"\0", np.uint8).copy()
    out = np.zeros(max(int(item[-1]), 1), np.int32)
    rc = self._unbounded_decode(buf.ctypes.data, so.ctypes.data, len(strings), index.ctypes.data, item.ctypes.data,
                                cdf.ctypes.data, cdf.shape[0], cdf.shape[1], cdf_size.ctypes.data, offset.ctypes.data,
                                int(precision), int(overflow_width), int(debug_level), int(threads), out.ctypes.data)
    if rc != 0:
      raise OracleError(self._err())
    return out[:int(item[-1])]

  def encode(self, data, index, cdf, cdf_size, offset, precision: int, overflow_width: int,
             debug_level: int = 1) -> bytes:
    """UnboundedIndexRangeEncode: the whole `data` as one string."""
    if np.shape(data) != np.shape(index):
      raise OracleError("`data` and `index` should have the same shape")
    return self.encode_batch(data, index, [np.size(data)], cdf, cdf_size, offset, precision, overflow_width,
                             debug_level)[0]

  def decode(self, encoded: bytes, index, cdf, cdf_size, offset, precision: int, overflow_width: int,
             debug_level: int = 1) -> np.ndarray:
    """UnboundedIndexRangeDecode: int32 shaped like `index`."""
    out = self.decode_batch([encoded], index, [np.size(index)], cdf, cdf_size, offset, precision, overflow_width,
                            debug_level)
    return out.reshape(np.shape(index))


_cache = {}


def port() -> UnboundedOracle:
  if "port" not in _cache:
    if not os.path.exists(_PORT_SO):
      build(want_ref=False)
    _cache["port"] = UnboundedOracle(_PORT_SO, "tfcport_", "port")
  return _cache["port"]


def have_ref() -> bool:
  return os.path.exists(_REF_SO)


def ref() -> UnboundedOracle:
  if "ref" not in _cache:
    if not have_ref():
      raise FileNotFoundError(f"{_REF_SO} missing: run `make -C oracle/unbounded ref` where the reference tree exists")
    _cache["ref"] = UnboundedOracle(_REF_SO, "tfcref_", "reference")
  return _cache["ref"]


def best() -> UnboundedOracle:
  """The compiled reference when present, else the C port."""
  return ref() if have_ref() else port()
