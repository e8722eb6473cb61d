"""Operator surface of the reference's ``gen_ops`` module, backed by libtfcb200.so.

Mirrors ``tensorflow_compression/python/ops/gen_ops.py:25-40`` (same function names and argument
order; op contracts in ``cc/ops/range_coder_ops.cc:28-247``, ``cc/ops/range_coding_ops.cc:30-124``,
``cc/ops/pmf_to_cdf_ops.cc:28-57``).  Tensors are CUDA ``torch.Tensor``s; ``tf.string`` tensors
become :class:`Strings` (device bytes + offsets, convertible to a list of ``bytes``); DT_VARIANT
handles become :class:`EncoderHandle` / :class:`DecoderHandle`.  Argument errors raise
:class:`InvalidArgumentError` (a ``ValueError``), the analogue of ``tf.errors.InvalidArgumentError``.

Everything computes on the GPU through the C ABI; there is no CPU path.
"""
import ctypes as C
from typing import List, Optional, Sequence, Union

import numpy as np
import torch

from compression_b200 import _lib
from compression_b200._lib import InvalidArgumentError, check

__all__ = [
    "stochastic_round",
    "run_length_encode",
    "run_length_decode",
    "run_length_gamma_encode",
    "run_length_gamma_decode",
    "create_range_encoder",
    "create_range_decoder",
    "entropy_decode_channel",
    "entropy_decode_finalize",
    "entropy_decode_index",
    "entropy_encode_channel",
    "entropy_encode_finalize",
    "entropy_encode_index",
    "pmf_to_quantized_cdf",
    "range_encode",
    "range_decode",
    "unbounded_index_range_encode",
    "unbounded_index_range_decode",
    "Strings",
    "InvalidArgumentError",
]


def _stream() -> int:
  return torch.cuda.current_stream().cuda_stream


def _device() -> torch.device:
  if not torch.cuda.is_available():
    raise RuntimeError("compression_b200 needs a CUDA device (no CPU fallback)")
  return torch.device("cuda", torch.cuda.current_device())


def _ptr(t: Optional[torch.Tensor]):
  return None if t is None else C.c_void_p(t.data_ptr())


def _host_i32(x) -> np.ndarray:
  if isinstance(x, torch.Tensor):
    x = x.detach().cpu().numpy()
  return np.ascontiguousarray(np.asarray(x), dtype=np.int32)


def _dev(x, dtype) -> torch.Tensor:
  """Contiguous CUDA tensor of the given dtype (moves / casts host data if needed)."""
  if not isinstance(x, torch.Tensor):
    x = torch.as_tensor(np.asarray(x))
  return x.to(device=_device(), dtype=dtype).contiguous()


def _prod(shape) -> int:
  n = 1
  for d in shape:
    n *= int(d)
  return n


def _split_items(flat: torch.Tensor, shapes) -> List[torch.Tensor]:
  """Views of a flat tensor holding items of the given shapes back to back."""
  out, at = [], 0
  for shape in shapes:
    n = _prod(shape)
    out.append(flat[at:at + n].reshape(shape))
    at += n
  return out


class Strings:
  """A tensor of byte strings (stand-in for a ``tf.string`` tensor).

  ``bytes_dev`` (uint8) holds all strings back to back, ``offsets_dev`` (int64, numel + 1) delimits
  them.  ``tolist()`` / ``numpy()`` copy to the host lazily.
  """

  def __init__(self, bytes_dev: torch.Tensor, offsets_dev: torch.Tensor, shape):
    self.bytes_dev = bytes_dev
    self.offsets_dev = offsets_dev
    self.shape = tuple(int(d) for d in shape)
    self._host = None

  @classmethod
  def from_bytes(cls, strings, shape=None) -> "Strings":
    if isinstance(strings, (bytes, bytearray)):
      strings, shape = [bytes(strings)], ()
    arr = np.asarray(strings, dtype=object)
    if shape is None:
      shape = arr.shape
    flat = [bytes(s) for s in arr.reshape(-1)]
    offs = np.zeros(len(flat) + 1, dtype=np.int64)
    for i, s in enumerate(flat):
      offs[i + 1] = offs[i] + len(s)
    buf = np.frombuffer(b"".join(flat) + b"\0", dtype=np.uint8).copy()
    dev = _device()
    out = cls(torch.from_numpy(buf).to(dev), torch.from_numpy(offs).to(dev), shape)
    out._host = flat
    return out

  def numel(self) -> int:
    return _prod(self.shape)

  def tolist(self) -> List[bytes]:
    if self._host is None:
      offs = self.offsets_dev.cpu().numpy()
      raw = self.bytes_dev[:int(offs[-1])].cpu().numpy().tobytes()
      self._host = [raw[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]
    return list(self._host)

  def numpy(self) -> np.ndarray:
    out = np.empty(len(self.tolist()), dtype=object)
    for i, s in enumerate(self._host):
      out[i] = s
    return out.reshape(self.shape)

  def nbytes(self) -> int:
    return int(self.offsets_dev[-1].item())

  def split(self) -> List["Strings"]:
    """Every string on its own, as a Strings of shape (1,) that views this one's bytes (one host synchronisation)."""
    offs = self.offsets_dev.cpu().tolist()
    ends = self.offsets_dev[1:] - self.offsets_dev[:-1]
    local = torch.stack([torch.zeros_like(ends), ends], dim=1)  # row i: offsets of string i in its own view
    return [Strings(self.bytes_dev[offs[i]:offs[i + 1]], local[i], (1,)) for i in range(len(offs) - 1)]

  @classmethod
  def concat(cls, parts: Sequence["Strings"]) -> "Strings":
    """The strings of `parts`, in order, as one Strings of shape (total,) (one host synchronisation)."""
    parts = list(parts)
    if not parts:
      raise InvalidArgumentError("nothing to concatenate")
    counts = [p.numel() for p in parts]
    offs = torch.cat([p.offsets_dev for p in parts]).cpu().numpy()
    out_offs, chunks, base, at = [0], [], 0, 0
    for p, n in zip(parts, counts):
      o = offs[at:at + n + 1]
      at += n + 1
      out_offs.extend(int(base + v - o[0]) for v in o[1:])
      chunks.append(p.bytes_dev[int(o[0]):int(o[-1])])
      base += int(o[-1] - o[0])
    dev = parts[0].bytes_dev.device
    data = torch.cat(chunks + [torch.zeros(1, dtype=torch.uint8, device=dev)])
    return cls(data, torch.tensor(out_offs, dtype=torch.int64).to(dev), (len(out_offs) - 1,))

  def __len__(self):
    return self.shape[0] if self.shape else 1


# ------------------------------------------------------------------------------------------------
# Substream strings (DESIGN §3.14).  With S > 1 substreams a coding unit's string is varint(S), varint(len_0) ...
# varint(len_{S-2}), then the S substreams back to back, the last one running to the end of the string; varints are
# unsigned LEB128 in minimal form.  S = 1 is the plain range-coded string, with no header.
# ------------------------------------------------------------------------------------------------
MAX_SUBSTREAMS = 1024


def check_substreams(substreams, name="substreams") -> int:
  """`substreams` as an int in [1, MAX_SUBSTREAMS]; anything else raises InvalidArgumentError (a ValueError).  `name`
  is the argument's name in the message (MBT2018Model's `tiles` are the substreams of its y strings)."""
  if isinstance(substreams, (bool, np.bool_)) or not isinstance(substreams, (int, np.integer)):
    raise InvalidArgumentError(f"`{name}` must be an integer: {substreams!r}")
  if not 1 <= int(substreams) <= MAX_SUBSTREAMS:
    raise InvalidArgumentError(f"`{name}` must be in [1, {MAX_SUBSTREAMS}]: {int(substreams)}")
  return int(substreams)


def _varint(v: int) -> bytes:
  out = bytearray()
  while True:
    b = v & 0x7F
    v >>= 7
    if not v:
      out.append(b)
      return bytes(out)
    out.append(b | 0x80)


def substream_header(lengths) -> bytes:
  """The header of a unit whose S = len(lengths) substreams have these byte lengths (b"" for S = 1)."""
  lengths = [int(n) for n in lengths]
  if len(lengths) == 1:
    return b""
  return _varint(len(lengths)) + b"".join(_varint(n) for n in lengths[:-1])


def _read_varint(s: bytes, at: int, i: int):
  v, shift, start = 0, 0, at
  while True:
    if at >= len(s):
      raise InvalidArgumentError(f"string {i}: truncated substream header")
    b = s[at]
    at += 1
    v |= (b & 0x7F) << shift
    if not b & 0x80:
      break
    shift += 7
    if shift > 63:
      raise InvalidArgumentError(f"string {i}: substream header varint longer than 64 bits")
  if at - start > 1 and b == 0:
    raise InvalidArgumentError(f"string {i}: substream header varint not in minimal form")
  return v, at


def parse_substreams(s: bytes, substreams: int, i: int = 0) -> List[bytes]:
  """The S substreams of string number `i`, `s`, written with `substreams` = S > 1.  A truncated or non-minimal
  varint, another S, or lengths past the end raise InvalidArgumentError naming the string."""
  n, at = _read_varint(s, 0, i)
  if n != substreams:
    raise InvalidArgumentError(f"string {i}: written with {n} substreams, decoding expects {substreams}")
  lengths = []
  for _ in range(substreams - 1):
    v, at = _read_varint(s, at, i)
    lengths.append(v)
  out = []
  for v in lengths:
    if at + v > len(s):
      raise InvalidArgumentError(f"string {i}: substream lengths run past the end of its {len(s)} bytes")
    out.append(s[at:at + v])
    at += v
  return out + [s[at:]]


def join_substreams(parts: Strings, substreams: int, shape) -> Strings:
  """Strings of `shape` from the unit x S substreams `parts` (unit u's substream s at u S + s): each unit's header
  and its substreams.  One device-to-host copy (the offsets); the bytes stay on the device."""
  S = substreams
  n = parts.numel() // S
  offs = parts.offsets_dev.cpu().numpy()
  heads = [substream_header(np.diff(offs[u * S:(u + 1) * S + 1])) for u in range(n)]
  dev = parts.bytes_dev.device
  hbuf = torch.from_numpy(np.frombuffer(b"".join(heads) + b"\0", dtype=np.uint8).copy()).to(dev)
  chunks, out_offs, at = [], [0], 0
  for u, h in enumerate(heads):
    lo, hi = int(offs[u * S]), int(offs[(u + 1) * S])
    chunks += [hbuf[at:at + len(h)], parts.bytes_dev[lo:hi]]
    at += len(h)
    out_offs.append(out_offs[-1] + len(h) + hi - lo)
  data = torch.cat(chunks + [torch.zeros(1, dtype=torch.uint8, device=dev)])
  return Strings(data, torch.tensor(out_offs, dtype=torch.int64).to(dev), shape)


def split_substreams(strings: Strings, substreams: int) -> Strings:
  """The payloads of strings written with `substreams` = S > 1, without their headers, as a Strings of shape
  (numel S,) (string i's substream s at i S + s): what a decoder handle takes.  Parsed on the host before any device
  work."""
  payload = []
  for i, s in enumerate(strings.tolist()):
    payload += parse_substreams(s, substreams, i)
  return Strings.from_bytes(payload, (len(payload),))


class EncoderHandle:
  """Stand-in for the DT_VARIANT encoder handle (cc/kernels/range_coder_kernels.cc:62-66)."""

  def __init__(self, shape, lookup):
    self.shape = tuple(int(d) for d in shape)
    if any(d < 0 for d in self.shape):
      raise InvalidArgumentError(f"invalid handle shape {self.shape}")
    lookup = _host_i32(lookup)
    if lookup.ndim not in (1, 2):
      raise InvalidArgumentError(f"`lookup` must be rank 1 or 2: {lookup.shape}")
    self._lookup = lookup
    cols = 0 if lookup.ndim == 1 else lookup.shape[1]
    self.n_streams = _prod(self.shape)
    h = C.c_void_p()
    _device()
    check(_lib.lib().tfcb_encoder_create(
        lookup.ctypes.data_as(C.c_void_p), lookup.size, cols, self.n_streams, _stream(), C.byref(h)))
    self._h = h
    self._finalized = False

  def _require(self):
    if self._h is None:
      raise InvalidArgumentError("'handle' is not an encoder")
    if self.n_streams == 0:
      raise InvalidArgumentError(f"`handle` is empty: handle.shape={self.shape}")

  def close(self):
    if getattr(self, "_h", None) is not None:
      _lib.lib().tfcb_encoder_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint:disable=broad-except
      pass


class DecoderHandle:
  """Stand-in for the DT_VARIANT decoder handle."""

  def __init__(self, encoded: Strings, lookup):
    self.shape = encoded.shape
    self.n_streams = encoded.numel()
    if self.n_streams == 0:
      raise InvalidArgumentError(f"`encoded` is empty: {self.shape}")
    lookup = _host_i32(lookup)
    if lookup.ndim not in (1, 2):
      raise InvalidArgumentError(f"`lookup` must be rank 1 or 2: {lookup.shape}")
    cols = 0 if lookup.ndim == 1 else lookup.shape[1]
    self._encoded = encoded  # borrowed by the C handle
    h = C.c_void_p()
    check(_lib.lib().tfcb_decoder_create(
        _ptr(encoded.bytes_dev), _ptr(encoded.offsets_dev), self.n_streams,
        lookup.ctypes.data_as(C.c_void_p), lookup.size, cols, _stream(), C.byref(h)))
    self._h = h

  def close(self):
    if getattr(self, "_h", None) is not None:
      _lib.lib().tfcb_decoder_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint:disable=broad-except
      pass


# ------------------------------------------------------------------------------------------------
# Encoder ops
# ------------------------------------------------------------------------------------------------
def create_range_encoder(shape, lookup) -> EncoderHandle:
  """CreateRangeEncoder (cc/ops/range_coder_ops.cc:28-63)."""
  shape = [int(d) for d in np.asarray(shape.cpu() if isinstance(shape, torch.Tensor) else shape).reshape(-1)]
  return EncoderHandle(shape, lookup)


def _check_prefix(handle_shape, value_shape, what="value"):
  hs, vs = tuple(handle_shape), tuple(int(d) for d in value_shape)
  if vs[:len(hs)] != hs:
    raise InvalidArgumentError(
        f"'{what}' shape should start with 'handle' shape: {what}.shape={list(vs)} does not start with "
        f"handle.shape={list(hs)}")


def entropy_encode_channel(handle: EncoderHandle, value) -> EncoderHandle:
  """EntropyEncodeChannel (cc/ops/range_coder_ops.cc:65-101)."""
  handle._require()
  value = _dev(value, torch.int32)
  _check_prefix(handle.shape, value.shape)
  n = value.numel() // handle.n_streams
  check(_lib.lib().tfcb_encode_channel(handle._h, _ptr(value), n, _stream()))
  return handle


def entropy_encode_index(handle: EncoderHandle, index, value) -> EncoderHandle:
  """EntropyEncodeIndex (cc/ops/range_coder_ops.cc:103-121)."""
  handle._require()
  value = _dev(value, torch.int32)
  index = _dev(index, torch.int32)
  _check_prefix(handle.shape, value.shape)
  if tuple(index.shape) != tuple(value.shape):
    raise InvalidArgumentError(
        f"'index' shape should match 'value' shape: index.shape={list(index.shape)} != "
        f"value.shape={list(value.shape)}")
  n = value.numel() // handle.n_streams
  check(_lib.lib().tfcb_encode_index(handle._h, _ptr(index), _ptr(value), n, _stream()))
  return handle


def entropy_encode_finalize(handle: EncoderHandle) -> Strings:
  """EntropyEncodeFinalize (cc/ops/range_coder_ops.cc:123-135): one string per handle element."""
  handle._require()
  dev = _device()
  offsets = torch.empty(handle.n_streams + 1, dtype=torch.int64, device=dev)
  total = C.c_int64(0)
  check(_lib.lib().tfcb_encode_finalize(handle._h, _ptr(offsets), _stream(), C.byref(total)))
  out = torch.empty(max(int(total.value), 1), dtype=torch.uint8, device=dev)
  check(_lib.lib().tfcb_encode_write(handle._h, _ptr(offsets), _ptr(out), _stream()))
  return Strings(out, offsets, handle.shape)


# ------------------------------------------------------------------------------------------------
# Decoder ops
# ------------------------------------------------------------------------------------------------
def create_range_decoder(encoded, lookup) -> DecoderHandle:
  """CreateRangeDecoder (cc/ops/range_coder_ops.cc:137-170)."""
  if not isinstance(encoded, Strings):
    encoded = Strings.from_bytes(encoded)
  return DecoderHandle(encoded, lookup)


def _suffix(shape) -> List[int]:
  if isinstance(shape, torch.Tensor):
    shape = shape.cpu().numpy()
  return [int(d) for d in np.asarray(shape).reshape(-1)]


def entropy_decode_channel(handle: DecoderHandle, shape, Tdecoded=torch.int32):
  """EntropyDecodeChannel (cc/ops/range_coder_ops.cc:172-207) -> (handle, int32[handle.shape+shape])."""
  if Tdecoded not in (torch.int32,):
    raise InvalidArgumentError("Tdecoded must be int32")
  suffix = _suffix(shape)
  n = _prod(suffix)
  out = torch.empty(tuple(handle.shape) + tuple(suffix), dtype=torch.int32, device=_device())
  check(_lib.lib().tfcb_decode_channel(handle._h, _ptr(out), n, _stream()))
  return handle, out


def entropy_decode_index(handle: DecoderHandle, index, shape, Tdecoded=torch.int32):
  """EntropyDecodeIndex (cc/ops/range_coder_ops.cc:209-231)."""
  if Tdecoded not in (torch.int32,):
    raise InvalidArgumentError("Tdecoded must be int32")
  suffix = _suffix(shape)
  index = _dev(index, torch.int32)
  out_shape = tuple(handle.shape) + tuple(suffix)
  if tuple(index.shape) != out_shape:
    raise InvalidArgumentError(
        "'index' shape should match 'handle' shape + 'shape': "
        f"index.shape={list(index.shape)}, handle.shape={list(handle.shape)}, shape={suffix}")
  n = _prod(suffix)
  out = torch.empty(out_shape, dtype=torch.int32, device=_device())
  check(_lib.lib().tfcb_decode_index(handle._h, _ptr(index), _ptr(out), n, _stream()))
  return handle, out


def entropy_decode_finalize(handle: DecoderHandle) -> torch.Tensor:
  """EntropyDecodeFinalize (cc/ops/range_coder_ops.cc:233-247) -> bool[handle.shape] (on the host)."""
  ok = np.zeros(handle.n_streams, dtype=np.uint8)
  check(_lib.lib().tfcb_decode_finalize(handle._h, ok.ctypes.data_as(C.c_void_p), _stream()))
  return torch.from_numpy(ok.astype(bool)).reshape(handle.shape)


# ------------------------------------------------------------------------------------------------
# PmfToQuantizedCdf
# ------------------------------------------------------------------------------------------------
def pmf_to_quantized_cdf(pmf, precision: int) -> torch.Tensor:
  """PmfToQuantizedCdf (cc/ops/pmf_to_cdf_ops.cc:28-57): float32 [..., n] -> int32 [..., n + 1]."""
  precision = int(precision)
  pmf = _dev(pmf, torch.float32)
  if pmf.dim() < 1:
    raise InvalidArgumentError("`pmf` should be at least 1-D.")
  n = pmf.shape[-1]
  rows = pmf.numel() // max(n, 1)
  cdf = torch.empty(tuple(pmf.shape[:-1]) + (n + 1,), dtype=torch.int32, device=pmf.device)
  check(_lib.lib().tfcb_pmf_to_quantized_cdf(_ptr(pmf), rows, n, precision, _ptr(cdf), _stream()))
  return cdf


# ------------------------------------------------------------------------------------------------
# Legacy single-stream ops
# ------------------------------------------------------------------------------------------------
def _shape_arr(shape) -> np.ndarray:
  return np.ascontiguousarray(np.asarray([int(d) for d in shape], dtype=np.int64))


def range_encode(data, cdf, precision: int, debug_level: int = 1) -> bytes:
  """RangeEncode (cc/ops/range_coding_ops.cc:30-90): int16 data, int32 cdf -> one byte string."""
  data = _dev(data, torch.int16)
  cdf = _dev(cdf, torch.int32)
  ds, cs = _shape_arr(data.shape), _shape_arr(cdf.shape)
  cap = 2 * data.numel() + 64
  out = np.empty(cap, dtype=np.uint8)
  n = C.c_int64(0)
  check(_lib.lib().tfcb_range_encode(
      _ptr(data), ds.ctypes.data_as(C.c_void_p), data.dim(), _ptr(cdf), cs.ctypes.data_as(C.c_void_p),
      cdf.dim(), int(precision), int(debug_level), out.ctypes.data_as(C.c_void_p), cap, C.byref(n),
      _stream()))
  return out[:n.value].tobytes()


def range_decode(encoded, shape, cdf, precision: int, debug_level: int = 1) -> torch.Tensor:
  """RangeDecode (cc/ops/range_coding_ops.cc:92-124): byte string + shape + cdf -> int16 tensor."""
  if isinstance(encoded, Strings):
    if encoded.shape != ():
      raise InvalidArgumentError(f"Invalid `encoded` shape: {list(encoded.shape)}")
    encoded = encoded.tolist()[0]
  if not isinstance(encoded, (bytes, bytearray)):
    raise InvalidArgumentError("Invalid `encoded` shape: expected a scalar string")
  shape_np = np.asarray(shape.cpu() if isinstance(shape, torch.Tensor) else shape)
  if shape_np.ndim != 1:
    raise InvalidArgumentError(f"Invalid `shape` shape: {list(shape_np.shape)}")
  cdf = _dev(cdf, torch.int32)
  ds, cs = _shape_arr(shape_np), _shape_arr(cdf.shape)
  out = torch.empty(tuple(int(d) for d in ds), dtype=torch.int16, device=cdf.device)
  buf = np.frombuffer(bytes(encoded) + b"\0", dtype=np.uint8)
  check(_lib.lib().tfcb_range_decode(
      buf.ctypes.data_as(C.c_void_p), len(encoded), ds.ctypes.data_as(C.c_void_p), len(ds), _ptr(cdf),
      cs.ctypes.data_as(C.c_void_p), cdf.dim(), int(precision), int(debug_level), _ptr(out), _stream()))
  return out


# ------------------------------------------------------------------------------------------------
# Quantisation ops
# ------------------------------------------------------------------------------------------------
_SR_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def stochastic_round(inputs, step_size, seed) -> torch.Tensor:
  """StochasticRound (cc/ops/quantization_ops.cc:28-53, cc/kernels/quantization_kernels.cc:48-95):
  int32 floor(inputs / step_size) + Bernoulli(fractional part).  `seed`: int32 tensor / sequence of any shape; the
  same seed gives the same integers as the reference CPU op; an empty seed seeds from the clock."""
  if not isinstance(inputs, torch.Tensor):
    inputs = torch.as_tensor(inputs, dtype=torch.float32)
  if inputs.dtype not in _SR_DTYPES:
    raise InvalidArgumentError(f"StochasticRound: unsupported dtype {inputs.dtype} (bfloat16, float16, float32)")
  step = np.asarray(step_size.cpu() if isinstance(step_size, torch.Tensor) else step_size, dtype=np.float32)
  if step.ndim != 0:
    raise InvalidArgumentError("step_size must be a scalar.")
  inputs = inputs.to(_device()).contiguous()
  sd = np.ascontiguousarray(np.asarray(seed.cpu() if isinstance(seed, torch.Tensor) else seed, dtype=np.int32).reshape(-1))
  out = torch.empty(inputs.shape, dtype=torch.int32, device=inputs.device)
  check(_lib.lib().tfcb_stochastic_round(_ptr(inputs), _SR_DTYPES[inputs.dtype], inputs.numel(), float(step),
                                         sd.ctypes.data_as(C.c_void_p) if sd.size else None, sd.size, _ptr(out),
                                         _stream()))
  return out


# ------------------------------------------------------------------------------------------------
# Run-length / Rice / gamma bit coding (cc/ops/run_length_ops.cc:28-84, run_length_gamma_ops.cc)
# ------------------------------------------------------------------------------------------------
def run_length_encode(data, run_length_code: int, magnitude_code: int, use_run_length_for_non_zeros: bool) -> bytes:
  """RunLengthEncode: int32 tensor of any shape -> one bit string (zeros as run lengths, non-zeros as sign +
  magnitude; Rice codes for parameters >= 0, Elias gamma otherwise)."""
  data = _dev(data, torch.int32).reshape(-1)
  n = data.numel()
  if n == 0:
    return b""
  cap = 4 * ((2 * n + 64 + 3) // 4)
  while True:
    code = torch.empty(cap, dtype=torch.uint8, device=data.device)
    nb = C.c_int64(0)
    rc = _lib.lib().tfcb_run_length_encode(_ptr(data), n, int(run_length_code), int(magnitude_code),
                                           int(bool(use_run_length_for_non_zeros)), _ptr(code), cap, C.byref(nb),
                                           _stream())
    if rc == _lib.INVALID_ARGUMENT and nb.value > cap - 4:   # the code is longer than the first guess: once more
      cap = 4 * ((nb.value + 3) // 4) + 4
      continue
    check(rc)
    return code[:nb.value].cpu().numpy().tobytes()


def run_length_decode(code, shape, run_length_code: int, magnitude_code: int, use_run_length_for_non_zeros: bool):
  """RunLengthDecode: the inverse; `shape` of the encoded tensor must be known (cc/ops/run_length_ops.cc:50-84)."""
  if isinstance(code, Strings):
    if code.shape != ():
      raise InvalidArgumentError(f"Invalid `code` shape: {list(code.shape)}")
    code = code.tolist()[0]
  if not isinstance(code, (bytes, bytearray)):
    raise InvalidArgumentError("Invalid `code` shape: expected a scalar string")
  shape_np = np.asarray(shape.cpu() if isinstance(shape, torch.Tensor) else shape)
  if shape_np.ndim != 1:
    raise InvalidArgumentError(f"Invalid `shape` shape: {list(shape_np.shape)}")
  dims = tuple(int(d) for d in shape_np)
  out = torch.empty(dims, dtype=torch.int32, device=_device())
  buf = torch.from_numpy(np.frombuffer(bytes(code) + b"\0\0\0\0", dtype=np.uint8).copy()).to(out.device)
  check(_lib.lib().tfcb_run_length_decode(_ptr(buf), len(code), int(run_length_code), int(magnitude_code),
                                          int(bool(use_run_length_for_non_zeros)), _ptr(out), out.numel(), _stream()))
  return out


def run_length_gamma_encode(data) -> bytes:
  """RunLengthGammaEncode = RunLengthEncode(-1, -1, False) (cc/ops/run_length_ops.cc:34-37)."""
  return run_length_encode(data, -1, -1, False)


def run_length_gamma_decode(code, shape):
  return run_length_decode(code, shape, -1, -1, False)


# ------------------------------------------------------------------------------------------------
# UnboundedIndexRangeEncode / UnboundedIndexRangeDecode (cc/ops/range_coding_ops.cc:126-247)
# ------------------------------------------------------------------------------------------------
def _shape_of(x):
  return tuple(int(d) for d in (x.shape if hasattr(x, "shape") else np.shape(x)))


def _ubi_check(precision, overflow_width, debug_level, index_shape, cdf, cdf_size, offset, data_shape=None):
  """The op's attribute and shape checks, in the reference's order, before anything reaches the device."""
  if not 0 < int(precision) <= 16:
    raise InvalidArgumentError(f"`precision` must be in [1, 16]: {precision}")
  if not 0 < int(overflow_width) <= 16:
    raise InvalidArgumentError(f"`overflow_width` must be in [1, 16]: {overflow_width}")
  if int(debug_level) not in (0, 1):
    raise InvalidArgumentError(f"`debug_level` must be 0 or 1: {debug_level}")
  if data_shape is not None and tuple(data_shape) != tuple(index_shape):
    raise InvalidArgumentError(f"`data` and `index` should have the same shape: data.shape={list(data_shape)}, "
                               f"index.shape={list(index_shape)}")
  cs, ss, os_ = _shape_of(cdf), _shape_of(cdf_size), _shape_of(offset)
  if len(cs) != 2 or cs[1] < 3:
    raise InvalidArgumentError(f"'cdf' should be 2-D and cdf.dim_size(1) >= 3: {list(cs)}")
  if len(ss) != 1 or ss[0] != cs[0]:
    raise InvalidArgumentError("'cdf_size' should be 1-D and its length should match the number of rows in "
                               f"'cdf': {list(ss)}")
  if len(os_) != 1 or os_[0] != cs[0]:
    raise InvalidArgumentError("'offset' should be 1-D and its length should match the number of rows in 'cdf': "
                               f"offset.shape={list(os_)}, cdf.shape={list(cs)}")


def _ubi_encode(data, index, item_offsets, cdf, cdf_size, offset, precision, overflow_width, debug_level) -> Strings:
  """Strings [k]: item u is data[item_offsets[u]:item_offsets[u + 1]] (flat int32 on the device)."""
  dev = _device()
  data, index = _dev(data, torch.int32).reshape(-1), _dev(index, torch.int32).reshape(-1)
  cdf, cdf_size, offset = _dev(cdf, torch.int32), _dev(cdf_size, torch.int32), _dev(offset, torch.int32)
  k = item_offsets.size - 1
  cs = _shape_arr(cdf.shape)
  offsets = torch.empty(k + 1, dtype=torch.int64, device=dev)
  h, total = C.c_void_p(), C.c_int64(0)
  L = _lib.lib()
  check(L.tfcb_unbounded_index_range_encode_ragged(
      _ptr(data), _ptr(index), k, item_offsets.ctypes.data_as(C.c_void_p), _ptr(cdf), cs.ctypes.data_as(C.c_void_p),
      cdf.dim(), _ptr(cdf_size), cdf_size.numel(), _ptr(offset), offset.numel(), int(precision), int(overflow_width),
      int(debug_level), _ptr(offsets), _stream(), C.byref(h), C.byref(total)))
  try:
    out = torch.empty(max(int(total.value), 1), dtype=torch.uint8, device=dev)
  except BaseException:
    L.tfcb_unbounded_index_range_encoder_destroy(h)
    raise
  check(L.tfcb_unbounded_index_range_write(h, _ptr(out), _stream()))
  return Strings(out, offsets, (k,))


def _ubi_decode(strings: Strings, index, item_offsets, cdf, cdf_size, offset, precision, overflow_width,
                debug_level) -> torch.Tensor:
  """Flat int32 [item_offsets[-1]]: string u decoded into elements item_offsets[u]:item_offsets[u + 1]."""
  index = _dev(index, torch.int32).reshape(-1)
  cdf, cdf_size, offset = _dev(cdf, torch.int32), _dev(cdf_size, torch.int32), _dev(offset, torch.int32)
  k = item_offsets.size - 1
  cs = _shape_arr(cdf.shape)
  out = torch.empty(int(item_offsets[-1]), dtype=torch.int32, device=index.device)
  check(_lib.lib().tfcb_unbounded_index_range_decode_ragged(
      _ptr(strings.bytes_dev), _ptr(strings.offsets_dev), k, item_offsets.ctypes.data_as(C.c_void_p), _ptr(index),
      _ptr(cdf), cs.ctypes.data_as(C.c_void_p), cdf.dim(), _ptr(cdf_size), cdf_size.numel(), _ptr(offset),
      offset.numel(), int(precision), int(overflow_width), int(debug_level), _ptr(out), _stream()))
  return out


def unbounded_index_range_encode(data, index, cdf, cdf_size, offset, precision: int, overflow_width: int,
                                 debug_level: int = 1) -> bytes:
  """UnboundedIndexRangeEncode: int32 `data` coded with row index[i] of `cdf` (first cdf_size[r] entries, the last
  bin the escape) into one byte string; values outside [offset[r], offset[r] + cdf_size[r] - 2) escape into
  overflow_width-bit digits."""
  _ubi_check(precision, overflow_width, debug_level, _shape_of(index), cdf, cdf_size, offset, _shape_of(data))
  n = _prod(_shape_of(data))
  s = _ubi_encode(data, index, np.array([0, n], np.int64), cdf, cdf_size, offset, precision, overflow_width,
                  debug_level)
  return s.tolist()[0]


def unbounded_index_range_decode(encoded, index, cdf, cdf_size, offset, precision: int, overflow_width: int,
                                 debug_level: int = 1) -> torch.Tensor:
  """UnboundedIndexRangeDecode: the inverse; returns int32 shaped like `index`."""
  if isinstance(encoded, Strings):
    if encoded.shape != ():
      raise InvalidArgumentError(f"`encoded` should be a scalar: {list(encoded.shape)}")
  elif not isinstance(encoded, (bytes, bytearray)):
    raise InvalidArgumentError(f"`encoded` should be a scalar: {list(np.shape(encoded))}")
  shape = _shape_of(index)
  _ubi_check(precision, overflow_width, debug_level, shape, cdf, cdf_size, offset)
  if not isinstance(encoded, Strings):
    encoded = Strings.from_bytes(bytes(encoded))
  out = _ubi_decode(encoded, index, np.array([0, _prod(shape)], np.int64), cdf, cdf_size, offset, precision,
                    overflow_width, debug_level)
  return out.reshape(shape)
