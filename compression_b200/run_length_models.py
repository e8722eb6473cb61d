"""Entropy models over the run-length bit coder: ``PowerLawEntropyModel`` and ``LaplaceEntropyModel``.

Host-side mirror of the reference's two callers of ``RunLength{Gamma}Encode/Decode``
(python/entropy_models/power_law.py:27-209, python/entropy_models/laplace.py:25-233): no tables, no prior --
rounding, one bit string per coding unit through ``gen_ops.run_length_encode`` (the CUDA coder of
csrc/run_length.cu), and a differentiable penalty standing in for the code length during training.
``compress_ragged`` / ``decompress_ragged`` code a list of differently shaped coding units in one launch each.
"""
from typing import List, Sequence

import numpy as np
import torch

from compression_b200 import functional
from compression_b200 import gen_ops
from compression_b200 import math_ops


class _RunLengthEntropyModel(torch.nn.Module):
  """What power_law.py and laplace.py share: quantise with a straight-through round, code every coding unit
  (the innermost ``coding_rank`` axes) as its own string, decode back to ``bottleneck_dtype``."""

  def __init__(self, coding_rank, bottleneck_dtype=None):
    super().__init__()
    self._coding_rank = int(coding_rank)
    if self._coding_rank < 0:
      raise ValueError("`coding_rank` must be at least 0.")
    # the reference falls back to the Keras policy's compute dtype, then floatx (power_law.py:80-84)
    self._bottleneck_dtype = torch.get_default_dtype() if bottleneck_dtype is None else bottleneck_dtype

  @property
  def coding_rank(self):
    """Number of innermost dimensions considered a coding unit."""
    return self._coding_rank

  @property
  def bottleneck_dtype(self):
    """Data type of the bottleneck tensor."""
    return self._bottleneck_dtype

  # the three code parameters of RunLengthEncode (cc/ops/run_length_ops.cc:28-48); gamma / gamma / False is
  # RunLengthGammaEncode
  run_length_code = -1
  magnitude_code = -1
  use_run_length_for_non_zeros = False

  def encode_fn(self, symbols) -> bytes:
    return gen_ops.run_length_encode(symbols, self.run_length_code, self.magnitude_code,
                                     self.use_run_length_for_non_zeros)

  def decode_fn(self, code, shape):
    return gen_ops.run_length_decode(code, shape, self.run_length_code, self.magnitude_code,
                                     self.use_run_length_for_non_zeros)

  def _as_bottleneck(self, bottleneck):
    return torch.as_tensor(bottleneck).to(self.bottleneck_dtype)

  def _reduce(self, per_element):
    if self.coding_rank == 0:
      return per_element
    return per_element.sum(dim=tuple(range(-self.coding_rank, 0)))

  def penalty(self, bottleneck):
    raise NotImplementedError

  def forward(self, bottleneck):
    """-> ``(self.quantize(bottleneck), self.penalty(bottleneck))`` (power_law.py:101-113)."""
    bottleneck = self._as_bottleneck(bottleneck)
    return self.quantize(bottleneck), self.penalty(bottleneck)

  def quantize(self, bottleneck):
    """Rounds to integers; the gradient is the identity (power_law.py:131-146)."""
    return math_ops.round_st(self._as_bottleneck(bottleneck))

  def compress(self, bottleneck) -> np.ndarray:
    """One bit string per coding unit (power_law.py:148-184): object array of ``bytes`` shaped like
    ``bottleneck`` without its ``coding_rank`` innermost axes."""
    bottleneck = self._as_bottleneck(bottleneck)
    if bottleneck.dim() < self.coding_rank:
      raise ValueError(f"`bottleneck` must have at least {self.coding_rank} dimensions.")
    shape = tuple(bottleneck.shape)
    strings_shape = shape if self.coding_rank == 0 else shape[:len(shape) - self.coding_rank]
    unit = gen_ops._prod(shape[len(strings_shape):])
    symbols = torch.round(bottleneck).to(torch.int32).reshape(gen_ops._prod(strings_shape), unit)
    strings = np.empty(symbols.shape[0], dtype=object)
    for i in range(symbols.shape[0]):
      strings[i] = self.encode_fn(symbols[i])
    return strings.reshape(strings_shape)

  def decompress(self, strings, code_shape: Sequence[int]) -> torch.Tensor:
    """-> tensor of shape ``strings.shape + code_shape`` in ``bottleneck_dtype`` (power_law.py:186-209)."""
    if isinstance(strings, gen_ops.Strings):
      strings = strings.numpy()
    if isinstance(strings, (bytes, bytearray)):
      arr = np.empty((), dtype=object)
      arr[()] = bytes(strings)
    else:
      arr = np.asarray(strings, dtype=object)
    code_shape = tuple(int(d) for d in code_shape)
    units = [torch.as_tensor(self.decode_fn(s, code_shape)) for s in arr.reshape(-1)]
    if not units:
      return torch.zeros(arr.shape + code_shape, dtype=self.bottleneck_dtype)
    return torch.stack(units).reshape(arr.shape + code_shape).to(self.bottleneck_dtype)

  def _code(self):
    return self.run_length_code, self.magnitude_code, self.use_run_length_for_non_zeros

  def compress_ragged(self, bottlenecks) -> gen_ops.Strings:
    """Compresses a list of coding units of different shapes in one coder launch.  Each item has exactly
    `coding_rank` dimensions.  Returns a Strings of shape (k,) whose string i equals `compress(bottlenecks[i])[()]`;
    a uniform batch ``x`` is ``compress_ragged(list(x.reshape(-1, *code_shape)))``."""
    items = [self._as_bottleneck(b) for b in bottlenecks]
    if not items:
      raise ValueError("`bottlenecks` is empty")
    for b in items:
      if b.dim() != self.coding_rank:
        raise ValueError(f"each item needs exactly {self.coding_rank} dimensions: received shape {tuple(b.shape)}")
    dev = gen_ops._device()
    symbols = torch.cat([torch.round(b.to(dev)).to(torch.int32).reshape(-1) for b in items])
    return functional.run_length_encode_ragged(symbols, [b.numel() for b in items], *self._code())

  def decompress_ragged(self, strings, code_shapes) -> List[torch.Tensor]:
    """Inverse of compress_ragged in one coder launch: item i has shape `code_shapes[i]` (exactly `coding_rank`
    dimensions), equals `decompress(strings[i], code_shapes[i])` and is in `bottleneck_dtype`.  The items are views
    into one allocation."""
    shapes = [tuple(int(d) for d in s) for s in code_shapes]
    for s in shapes:
      if len(s) != self.coding_rank:
        raise ValueError(f"each code shape needs exactly {self.coding_rank} dimensions: received {s}")
    lengths = [gen_ops._prod(s) for s in shapes]
    flat = functional.run_length_decode_ragged(strings, lengths, *self._code()).to(self.bottleneck_dtype)
    return gen_ops._split_items(flat, shapes)


class PowerLawEntropyModel(_RunLengthEntropyModel):
  """Entropy model for power-law distributed variables (power_law.py:27-209): the Elias-gamma run-length code, and
  the penalty ``log((abs(x) + alpha) / alpha)`` that follows its code length ``1 + 2 floor(log2 abs(x))``."""

  def __init__(self, coding_rank, alpha=1e-2, bottleneck_dtype=None):
    super().__init__(coding_rank, bottleneck_dtype)
    self._alpha = float(alpha)
    if self._alpha <= 0:
      raise ValueError("`alpha` must be greater than 0.")

  @property
  def alpha(self):
    return self._alpha

  def penalty(self, bottleneck):
    """power_law.py:115-129."""
    bottleneck = self._as_bottleneck(bottleneck)
    return self._reduce(torch.log((bottleneck.abs() + self.alpha) / self.alpha))


class LaplaceEntropyModel(_RunLengthEntropyModel):
  """Entropy model for Laplace distributed variables (laplace.py:25-233): Rice (or gamma) codes for run lengths and
  magnitudes, penalty ``l1 * sum(abs(x))``."""

  def __init__(self, coding_rank, l1=0.01, run_length_code=-1, magnitude_code=0, use_run_length_for_non_zeros=False,
               bottleneck_dtype=None):
    super().__init__(coding_rank, bottleneck_dtype)
    self._l1 = float(l1)
    if self._l1 <= 0:
      raise ValueError("`l1` must be greater than 0.")
    self.run_length_code = int(run_length_code)
    self.magnitude_code = int(magnitude_code)
    self.use_run_length_for_non_zeros = bool(use_run_length_for_non_zeros)

  @property
  def l1(self):
    return self._l1

  def penalty(self, bottleneck):
    """laplace.py:140-153."""
    return self.l1 * self._reduce(self._as_bottleneck(bottleneck).abs())
