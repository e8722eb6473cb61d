"""Entropy models of the reference on the CUDA range coder.

Mirrors tensorflow_compression/python/entropy_models:
  continuous_base.py:36-370     ContinuousEntropyModelBase (table build, storage, config)
  continuous_batched.py:30-436  ContinuousBatchedEntropyModel
  continuous_indexed.py:30-633  ContinuousIndexedEntropyModel, LocationScaleIndexedEntropyModel
Same constructor keywords, properties and method semantics; tensors are CUDA torch tensors,
`tf.string` results are `gen_ops.Strings`.  `EntropyBottleneck` (the TFC-1.x name used by the task
statement) is provided as a thin alias, see the bottom of the file.
"""
import functools
import math
import warnings

import numpy as np
import torch
from torch import nn

from compression_b200 import distributions as D
from compression_b200 import functional as F
from compression_b200 import gen_ops, math_ops

__all__ = [
    "ContinuousEntropyModelBase", "ContinuousBatchedEntropyModel", "ContinuousIndexedEntropyModel",
    "LocationScaleIndexedEntropyModel", "UniversalBatchedEntropyModel", "UniversalIndexedEntropyModel",
    "EntropyBottleneck", "MixtureEntropyModel",
]


def _cuda():
  return torch.device("cuda", torch.cuda.current_device())


class ContinuousEntropyModelBase(nn.Module):
  """continuous_base.py:36-370.

  The range-coding plumbing every model's compress / decompress and their ragged forms share lives here (`_encode`,
  `_decode`, `_encode_ragged`, `_decode_ragged`); a model derives only its batch shape or item shapes, and the
  table index and offset of every element.  Two coding modes:
    channel mode (`index` None, ContinuousBatchedEntropyModel): element j of a coding unit uses table row
      j % rows, where `coff` / `off` hold one value per row (float32 offsets);
    index mode: element j uses row `index[j]`, and `off` (or None) has the bottleneck's shape.
  """

  decode_sanity_check = True

  def __init__(self, coding_rank=None, compression=False, stateless=False, expected_grads=False,
               tail_mass=2**-8, bottleneck_dtype=None, laplace_tail_mass=0):
    super().__init__()
    self._prior = None  # set by the subclasses; an nn.Module prior registers as a submodule (see _set_prior)
    self._coding_rank = int(coding_rank)
    self._compression = bool(compression)
    self._stateless = bool(stateless)
    self._expected_grads = bool(expected_grads)
    self._tail_mass = float(tail_mass)
    self._bottleneck_dtype = bottleneck_dtype or torch.float32
    self._laplace_tail_mass = laplace_tail_mass
    if self.coding_rank < 0:
      raise ValueError("`coding_rank` must be at least 0.")
    if not 0 < self.tail_mass < 1:
      raise ValueError("`tail_mass` must be between 0 and 1.")

  def _check_compression(self):
    if not self.compression:
      raise RuntimeError(
          "For range coding, the entropy model must be instantiated with `compression=True`.")

  @property
  def prior(self):
    if self._prior is None:
      raise RuntimeError(
          "This entropy model doesn't hold a reference to its prior distribution. This can happen "
          "depending on how it is instantiated, (e.g., if it is unserialized).")
    return self._prior

  @prior.deleter
  def prior(self):
    self._prior = None

  def _set_prior(self, prior, register=True):
    """A prior the caller hands in is part of the model exactly as in the reference, where assigning it on the
    tf.Module makes its variables trainable_variables / checkpoint state (continuous_batched.py:205): an
    nn.Module prior becomes a registered submodule (parameters(), state_dict(), .to()).  Priors the model
    derives itself from `indexes` (continuous_indexed.py:226-232) hold no variables and stay plain attributes."""
    if register or not isinstance(prior, nn.Module):
      self._prior = prior
    else:
      self._modules.pop("_prior", None)
      object.__setattr__(self, "_prior", prior)

  @property
  def cdf(self):
    self._check_compression()
    return self._cdf

  @property
  def cdf_offset(self):
    self._check_compression()
    return self._cdf_offset

  bottleneck_dtype = property(lambda self: self._bottleneck_dtype)
  expected_grads = property(lambda self: self._expected_grads)
  laplace_tail_mass = property(lambda self: self._laplace_tail_mass)
  coding_rank = property(lambda self: self._coding_rank)
  compression = property(lambda self: self._compression)
  stateless = property(lambda self: self._stateless)
  tail_mass = property(lambda self: self._tail_mass)

  @property
  def range_coder_precision(self):
    return -int(self.cdf[0])

  def _init_compression(self, cdf, cdf_offset, cdf_shapes):
    """continuous_base.py:167-215: tables are stored (buffers), never rebuilt on the receiving side."""
    if not ((cdf is None) == (cdf_offset is None) == (cdf_shapes is not None)):
      raise ValueError("Either both `cdf` and `cdf_offset`, or `cdf_shapes` must be provided.")
    if cdf_shapes is not None:
      if self.stateless:
        raise ValueError("With `stateless=True`, can't provide `cdf_shapes`.")
      cdf_shapes = tuple(map(int, cdf_shapes))
      if len(cdf_shapes) != 2:
        raise ValueError("`cdf_shapes` must have two elements.")
      cdf = torch.zeros(cdf_shapes[0], dtype=torch.int32)
      cdf_offset = torch.zeros(cdf_shapes[1], dtype=torch.int32)
    cdf = torch.as_tensor(cdf).to(torch.int32)
    cdf_offset = torch.as_tensor(cdf_offset).to(torch.int32)
    if self.stateless:
      self._cdf, self._cdf_offset = cdf, cdf_offset
    else:
      self.register_buffer("_cdf", cdf)
      self.register_buffer("_cdf_offset", cdf_offset)
    self._cdf_host = None

  def _lookup_host(self):
    """Host copy of the table for handle creation (cached; tables are immutable once built)."""
    if self._cdf_host is None or self._cdf_host[0] is not self._cdf:
      self._cdf_host = (self._cdf, np.ascontiguousarray(self._cdf.detach().cpu().numpy(), dtype=np.int32))
    return self._cdf_host[1]

  def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
    # table buffers are restored with whatever shape was saved (validate_shape=False in the reference)
    for name in ("_cdf", "_cdf_offset", "_quantization_offset"):
      key = prefix + name
      if key in state_dict and getattr(self, name, None) is not None:
        setattr(self, name, state_dict[key].clone())
    self._cdf_host = None
    super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
    if self._prior is None:
      # a model rebuilt from its config holds tables, not a prior (continuous_base.py:336-360): prior weights
      # saved next to the tables are ignored instead of being reported as unexpected keys
      unexpected = args[3] if len(args) > 3 else kwargs.get("unexpected_keys")
      if unexpected is not None:
        unexpected[:] = [k for k in unexpected if not k.startswith(prefix + "_prior.")]

  @torch.no_grad()
  def _build_tables(self, prior, precision, offset=None):
    """continuous_base.py:217-296.  Returns (cdf 1-D int32 [-p, cdf...]*, cdf_offset int32)."""
    precision = int(precision)
    dev = _cuda()
    dtype = prior.dtype
    offset = torch.zeros((), dtype=dtype) if offset is None else torch.as_tensor(offset, dtype=dtype)
    lower = D.lower_tail(prior, self.tail_mass).to("cpu")
    upper = D.upper_tail(prior, self.tail_mass).to("cpu")
    offset = offset.to("cpu")
    minima = torch.floor(lower - offset).to(torch.int32)
    maxima = torch.ceil(upper - offset).to(torch.int32)
    pmf_start = minima.to(dtype) + offset
    pmf_length = maxima - minima + 1
    max_length = int(pmf_length.max())
    if max_length > 2048:
      warnings.warn(f"Very wide PMF with {max_length} elements may lead to out of memory issues. Consider "
                    "priors with smaller variance, or increasing `tail_mass` parameter.")
    prior_dev = getattr(prior, "device", torch.device("cpu"))
    samples = torch.arange(max_length, dtype=dtype).reshape([-1] + pmf_length.dim() * [1]) + pmf_start
    pmf = prior.prob(samples.to(prior_dev))
    pmf_shape = tuple(pmf.shape[1:])
    num_pmfs = gen_ops._prod(pmf_shape)
    pmf = pmf.reshape(max_length, num_pmfs).t().contiguous()
    pmf_length = torch.broadcast_to(pmf_length, pmf_shape).reshape(num_pmfs)
    cdf_offset = torch.broadcast_to(minima, pmf_shape).reshape(num_pmfs)
    cdf = F.build_lookup(pmf.to(dev, torch.float32), pmf_length, precision)
    return cdf, cdf_offset.to(dev)

  def _log_prob(self, prior, bottleneck_perturbed):
    """continuous_base.py:298-334."""
    x = bottleneck_perturbed.to(prior.dtype)
    ltm = float(self.laplace_tail_mass)
    if ltm > 0:
      if not ltm < 1:
        raise ValueError("`laplace_tail_mass` must be less than 1.")
      lap = D.NoisyLaplace(loc=torch.zeros((), device=x.device), scale=torch.ones((), device=x.device))
      probs = (1 - ltm) * prior.prob(x) + ltm * lap.prob(x)
      too_small = probs < 1e-10
      return torch.where(too_small, math.log(ltm) + lap.log_prob(x), torch.log(torch.clamp(probs, min=1e-10)))
    return prior.log_prob(x)

  def get_config(self):
    """continuous_base.py:336-360."""
    if self.stateless or not self.compression:
      raise RuntimeError(
          "Serializing entropy models with `compression=False` or `stateless=True` is not supported.")
    return dict(
        coding_rank=self.coding_rank,
        compression=True,
        stateless=False,
        expected_grads=self.expected_grads,
        tail_mass=self.tail_mass,
        cdf_shapes=(int(self.cdf.shape[0]), int(self.cdf_offset.shape[0])),
        bottleneck_dtype=str(self.bottleneck_dtype).replace("torch.", ""),
        laplace_tail_mass=float(self.laplace_tail_mass),
    )

  def get_weights(self):
    return [b.detach().cpu().numpy() for _, b in self.named_buffers()]

  def set_weights(self, weights):
    names = [n for n, _ in self.named_buffers()]
    if len(weights) != len(names):
      raise ValueError(f"`set_weights` expects a list of {len(names)} arrays, received {len(weights)}.")
    for n, w in zip(names, weights):
      old = getattr(self, n)
      setattr(self, n, torch.as_tensor(w).to(device=old.device, dtype=old.dtype))
    self._cdf_host = None

  # -- range coding --
  @staticmethod
  def _strings(strings, k=None):
    """`strings` as a Strings; with `k`, a list of the k strings of a ragged batch."""
    if not isinstance(strings, gen_ops.Strings):
      if k is not None:
        strings = list(strings)
      strings = gen_ops.Strings.from_bytes(strings, None if k is None else (len(strings),))
    if k is not None and strings.numel() != k:
      raise ValueError(f"{strings.numel()} strings for {k} items")
    return strings

  def _finish_decode(self, handle):
    sanity = gen_ops.entropy_decode_finalize(handle)
    if self.decode_sanity_check and not bool(sanity.all()):
      raise gen_ops.InvalidArgumentError("Sanity check failed.")

  def _quantize(self, b, off, coff, index=None):
    """The unfused quantisation to the symbols the coder takes.  Channel mode: rint(float32(b) - off[row]) -> int32 -
    coff[row], as [elements / rows, rows].  Index mode: rint(b - off) -> int32 - coff[index] in b's dtype, shaped like
    b.  (continuous_batched.py casts to float32 first, continuous_indexed.py and universal.py do not: the two differ
    for float16 and float64 bottlenecks.)"""
    if index is None:
      b = b.to(torch.float32).reshape(-1, coff.numel())
      return torch.round(b if off is None else b - off).to(torch.int32) - coff
    return torch.round(b if off is None else b - off).to(torch.int32) - coff[index.long()]

  def _dequantize(self, symbols, off, coff, index=None):
    """Inverse of _quantize, in bottleneck_dtype: float(sym + coff[row]) + off[row], as [elements / rows, rows]
    (channel mode), or float(sym + coff[index]) + off shaped like `symbols` (index mode)."""
    if index is None:
      out = (symbols.reshape(-1, coff.numel()) + coff).to(self.bottleneck_dtype)
      return out if off is None else out + off.to(out.dtype)
    out = (symbols + coff[index.long()]).to(self.bottleneck_dtype)
    return out if off is None else out + off

  # float16 / bfloat16 bottlenecks are quantised in the encoder and dequantised in the decoder where
  # functional._coder16 accepts the operands; the universal models keep the unfused path
  _coder16_models = True

  def _coder16(self, dtype, device, off, index, shape):
    return self._coder16_models and F._coder16(dtype, device, off, index, shape)

  # substreams (DESIGN §3.14): with S > 1 each coding unit's string holds S independently decodable streams, and every
  # call runs on the ragged entries over units x S streams.  A unit is one phase of positions: rows of the tables
  # (channel mode) or of the innermost axis (index mode), so every stream starts at a position.
  @staticmethod
  def _substreams(substreams, fused=True):
    S = gen_ops.check_substreams(substreams)
    if S > 1 and not fused:
      raise ValueError("`fused=False` issues the reference's op sequence, which writes one stream per string: "
                       "substreams must be 1")
    return S

  @staticmethod
  def _substream_layout(shapes, coff, index, substreams):
    """F.substream_layout of single-phase units of the given shapes."""
    if index is None:
      widths = [coff.numel()] * len(shapes)
    else:
      widths = [max(int(s[-1]), 1) if len(s) else 1 for s in shapes]
    return F.substream_layout([[gen_ops._prod(s) // w] for s, w in zip(shapes, widths)], [[w] for w in widths],
                              substreams)

  @staticmethod
  def _flat_unit_operands(off, index):
    """off and index flat for the ragged entries (off stays per row in channel mode)."""
    if index is not None:
      if off is not None and off.numel() == index.numel():
        off = off.reshape(-1)
      index = index.reshape(-1)
    return off, index

  def _encode(self, batch_shape, b, off, coff, index=None, fused=True, substreams=1):
    """One string per element of `batch_shape` for `b` (in bottleneck_dtype, coding units innermost).  A float32
    bottleneck, and a 16-bit one with the operands _coder16 accepts, is quantised inside the encoder unless
    `fused=False`, which issues the reference's op sequence."""
    S = self._substreams(substreams, fused)
    if S > 1:
      unit = tuple((b if index is None else index).shape[len(batch_shape):])
      off, index = self._flat_unit_operands(off, index)
      strings = self._encode_ragged([unit] * gen_ops._prod(batch_shape), b.reshape(-1), off, coff, index,
                                    substreams=S)
      return gen_ops.Strings(strings.bytes_dev, strings.offsets_dev, batch_shape)
    if fused and b.dtype == torch.float32:
      return F.compress_f32(batch_shape, self._lookup_host(), b, off, coff, index=index)
    if fused and self._coder16(b.dtype, b.device, off, index, b.shape):
      return F.compress_16bit(batch_shape, self._lookup_host(), b, off, coff, index=index)
    handle = gen_ops.create_range_encoder(batch_shape, self._lookup_host())
    symbols = self._quantize(b, off, coff, index)
    if index is None:  # the reference's iid_shape + [-1]: every axis left of prior_shape, then the table rows
      gen_ops.entropy_encode_channel(handle, symbols.reshape(b.shape[:b.dim() - len(self.prior_shape)] + (-1,)))
    else:
      gen_ops.entropy_encode_index(handle, index, symbols)
    return gen_ops.entropy_encode_finalize(handle)

  def _decode(self, strings, shape, off, coff, index=None, fused=True, substreams=1):
    """Inverse of _encode: a tensor of shape strings.shape + `shape` (the coding unit's) in bottleneck_dtype."""
    S = self._substreams(substreams, fused)
    if S > 1:
      off, index = self._flat_unit_operands(off, index)
      out = self._decode_flat(strings, [tuple(shape)] * strings.numel(), off, coff, index, S)
      return out.reshape(tuple(strings.shape) + tuple(shape))
    handle = gen_ops.create_range_decoder(strings, self._lookup_host())
    if fused and self.bottleneck_dtype == torch.float32:
      if index is None:
        out = F.decode_channel_f32(handle, strings.shape + shape, off, coff)
      else:
        out = F.decode_index_f32(handle, index, off, coff)
      self._finish_decode(handle)
      return out
    dev = strings.bytes_dev.device
    if fused and self._coder16(self.bottleneck_dtype, dev, off, index, None if index is None else index.shape):
      out = F.decode_16bit(handle, strings.shape + shape, self.bottleneck_dtype, off, coff, index=index)
      self._finish_decode(handle)
      return out
    if index is None:  # the reference decodes shape[:-rank(prior_shape)] + [rows]
      lead = shape[:len(shape) - len(self.prior_shape)]
      handle, symbols = gen_ops.entropy_decode_channel(handle, lead + (gen_ops._prod(self.prior_shape),))
    else:
      handle, symbols = gen_ops.entropy_decode_index(handle, index, shape)
    self._finish_decode(handle)
    return self._dequantize(symbols, off, coff, index).reshape(strings.shape + shape)

  # ragged batches: items of different shapes, one range-coder launch (an extension; the reference has none)
  def _encode_ragged(self, shapes, b, off, coff, index=None, return_decoded=False, substreams=1):
    """Strings of shape (k,) for the k items of the given shapes that `b` (in bottleneck_dtype) holds back to back;
    with `return_decoded`, also what _decode_ragged makes of them.  A float32 bottleneck, and a 16-bit one with the
    operands _coder16 accepts, is quantised inside the encoder, which then also writes the decoded items.  With
    `substreams` = S > 1 the encode runs over items x S streams, in item order, and the strings are joined."""
    S = self._substreams(substreams)
    lengths = [gen_ops._prod(s) for s in shapes] if S == 1 else self._substream_layout(shapes, coff, index, S)[0]
    fused = b.dtype == torch.float32 or self._coder16(b.dtype, b.device, off, index, b.shape)
    if b.dtype == torch.float32:
      out = F.compress_ragged(self._lookup_host(), lengths, b, off, coff, index=index, decoded=return_decoded)
    elif fused:
      out = F.compress_ragged_16bit(self._lookup_host(), lengths, b, off, coff, index=index, decoded=return_decoded)
    else:
      out = F.compress_ragged(self._lookup_host(), lengths, self._quantize(b, off, coff, index), index=index)
    strings, decoded = out if fused and return_decoded else (out, None)
    if S > 1:
      strings = gen_ops.join_substreams(strings, S, (len(shapes),))
    if not return_decoded:
      return strings
    if decoded is None:
      return strings, self._decode_ragged(strings, shapes, off, coff, index, S)
    return strings, gen_ops._split_items(decoded, shapes)

  def _decode_ragged(self, strings, shapes, off, coff, index=None, substreams=1):
    """Inverse of _encode_ragged: the items, views into one allocation."""
    S = self._substreams(substreams)
    return gen_ops._split_items(self._decode_flat(strings, shapes, off, coff, index, S), shapes)

  def _decode_flat(self, strings, shapes, off, coff, index, substreams):
    """The items of _decode_ragged back to back in one flat tensor.  With substreams the headers are parsed on the
    host before any device work, and the sanity check of an item is that of all its streams."""
    lengths = [gen_ops._prod(s) for s in shapes]
    if substreams > 1:
      lengths = self._substream_layout(shapes, coff, index, substreams)[0]
      strings = gen_ops.split_substreams(strings, substreams)
    handle = gen_ops.create_range_decoder(strings, self._lookup_host())
    dtype, dev = self.bottleneck_dtype, strings.bytes_dev.device
    unfused = False
    if dtype == torch.float32:
      out = F.decode_ragged(handle, lengths, index=index, quant_offset=off, cdf_offset=coff)
    elif self._coder16(dtype, dev, off, index, None if index is None else index.shape):
      out = F.decode_ragged_16bit(handle, lengths, dtype, off, coff, index=index)
    else:
      out = F.decode_ragged(handle, lengths, index=index)
      unfused = True
    self._finish_decode(handle)
    if unfused:
      out = self._dequantize(out, off, coff, index).reshape(-1)
    return out


class ContinuousBatchedEntropyModel(ContinuousEntropyModelBase):
  """continuous_batched.py:30-436: one table per element of `prior.batch_shape` (channel mode)."""

  def __init__(self, prior=None, coding_rank=None, compression=False, stateless=False, expected_grads=False,
               tail_mass=2**-8, range_coder_precision=12, bottleneck_dtype=None, prior_shape=None, cdf=None,
               cdf_offset=None, cdf_shapes=None, offset_heuristic=True, quantization_offset=None,
               decode_sanity_check=True, laplace_tail_mass=0):
    if (prior is None) == (prior_shape is None):
      raise ValueError("Either `prior` or `prior_shape` must be provided.")
    if (prior is None) + (cdf_shapes is None) + (cdf is None) != 2:
      raise ValueError("Must provide exactly one of `prior`, `cdf`, or `cdf_shapes`.")
    if not compression and not (cdf is None and cdf_offset is None and cdf_shapes is None):
      raise ValueError("CDFs can't be provided with `compression=False`")
    super().__init__(coding_rank=coding_rank, compression=compression, stateless=stateless,
                     expected_grads=expected_grads, tail_mass=tail_mass, bottleneck_dtype=bottleneck_dtype,
                     laplace_tail_mass=laplace_tail_mass)
    self._set_prior(prior)
    self._offset_heuristic = bool(offset_heuristic)
    self._prior_shape = tuple(int(s) for s in (prior_shape if prior is None else prior.batch_shape))
    if self.coding_rank < len(self.prior_shape):
      raise ValueError("`coding_rank` can't be smaller than `prior_shape`.")
    self.decode_sanity_check = decode_sanity_check

    if cdf_shapes is not None:
      assert isinstance(quantization_offset, bool)
      assert self.compression
      quantization_offset = torch.zeros(self.prior_shape) if quantization_offset else None
    elif quantization_offset is not None:
      pass
    elif self.offset_heuristic and self.compression:
      if self._prior is None:
        raise ValueError("To use the offset heuristic, a `prior` needs to be provided.")
      quantization_offset = D.quantization_offset(self.prior)
      if bool(torch.all(quantization_offset == 0.)):
        quantization_offset = None
      else:
        quantization_offset = torch.broadcast_to(quantization_offset, self.prior_shape).clone()
    else:
      quantization_offset = None
    if quantization_offset is None:
      self._quantization_offset = None
    else:
      q = torch.as_tensor(quantization_offset).detach().to(self.bottleneck_dtype)
      if self.compression and not self.stateless:
        self.register_buffer("_quantization_offset", q)
      else:
        self._quantization_offset = q
    if self.compression:
      if cdf is None and cdf_shapes is None:
        cdf, cdf_offset = self._build_tables(self.prior, range_coder_precision, offset=quantization_offset)
      self._init_compression(cdf, cdf_offset, cdf_shapes)

  prior_shape = property(lambda self: self._prior_shape)
  offset_heuristic = property(lambda self: self._offset_heuristic)

  @property
  def prior_shape_tensor(self):
    return torch.tensor(self.prior_shape, dtype=torch.int32)

  @property
  def quantization_offset(self):
    """continuous_batched.py:272-289."""
    if self._quantization_offset is not None:
      return self._quantization_offset
    if self.offset_heuristic and not self.compression:
      if self._prior is None:
        raise RuntimeError("To use the offset heuristic, a `prior` needs to be provided.")
      return D.quantization_offset(self.prior).to(self.bottleneck_dtype)
    return None

  def forward(self, bottleneck, training=True):
    """continuous_batched.py:291-322 -> (bottleneck_perturbed, bits)."""
    bottleneck = torch.as_tensor(bottleneck).to(self.bottleneck_dtype)
    log_prob_fn = functools.partial(self._log_prob, self.prior)
    if training:
      log_probs, perturbed = math_ops.perturb_and_apply(log_prob_fn, bottleneck,
                                                        expected_grads=self.expected_grads)
    else:
      perturbed = self.quantize(bottleneck)
      log_probs = log_prob_fn(perturbed)
    axes = tuple(range(-self.coding_rank, 0))
    bits = (log_probs.sum(dim=axes) if axes else log_probs) / -math.log(2.)
    return perturbed, bits

  def quantize(self, bottleneck):
    """continuous_batched.py:324-345."""
    bottleneck = torch.as_tensor(bottleneck).to(self.bottleneck_dtype)
    off = self.quantization_offset
    return math_ops.round_st(bottleneck, None if off is None else off.to(bottleneck.device))

  def _flat_tables(self, device):
    coff = self.cdf_offset.to(device).reshape(-1)
    qoff = self.quantization_offset
    return coff, (None if qoff is None else qoff.to(device, torch.float32).reshape(-1))

  def compress(self, bottleneck, fused=True, *, substreams=1):
    """continuous_batched.py:347-383.  `fused=True` quantises inside the encode kernel (same arithmetic);
    `fused=False` issues the reference's op sequence literally.  `substreams` = S > 1 writes each string as S
    independently decodable streams behind a small header (DESIGN §3.14; S = 1 is the reference's string), to be
    decompressed with the same S."""
    self._check_compression()
    bottleneck = torch.as_tensor(bottleneck).to(device=_cuda(), dtype=self.bottleneck_dtype)
    shape = tuple(bottleneck.shape)
    if len(shape) < self.coding_rank:
      raise ValueError("`bottleneck` has fewer dimensions than `coding_rank`.")
    batch_shape = shape[:len(shape) - self.coding_rank]
    rank_p = len(self.prior_shape)
    if rank_p and shape[-rank_p:] != self.prior_shape:
      bottleneck = torch.broadcast_to(bottleneck, shape[:-rank_p] + self.prior_shape)
    coff, qoff = self._flat_tables(bottleneck.device)
    return self._encode(batch_shape, bottleneck, qoff, coff, fused=fused, substreams=substreams)

  def decompress(self, strings, broadcast_shape, fused=True, *, substreams=1):
    """continuous_batched.py:385-422."""
    self._check_compression()
    strings = self._strings(strings)
    broadcast_shape = tuple(int(d) for d in np.asarray(broadcast_shape).reshape(-1))
    coff, qoff = self._flat_tables(strings.bytes_dev.device)
    return self._decode(strings, broadcast_shape + self.prior_shape, qoff, coff, fused=fused, substreams=substreams)

  # -- ragged batches: items of different shapes, one range-coder launch (an extension; the reference has none) --
  def compress_ragged(self, bottlenecks, return_decoded=False, *, substreams=1):
    """Compresses a list of coding units of different shapes in one range-coder launch.  Each item has exactly
    `coding_rank` dimensions ending in `prior_shape` (no broadcasting).  Returns a Strings of shape (k,) whose string
    i equals `compress(bottlenecks[i], substreams=substreams)`.

    `return_decoded=True` returns `(strings, items)` with `items` equal, bit for bit, to
    `decompress_ragged(strings, ...)`: written by the encoder itself for a float32 bottleneck, decoded from the
    fresh strings otherwise."""
    self._check_compression()
    dev = _cuda()
    items = [torch.as_tensor(b).to(device=dev, dtype=self.bottleneck_dtype) for b in bottlenecks]
    rank_p = len(self.prior_shape)
    for b in items:
      if b.dim() != self.coding_rank or (rank_p and tuple(b.shape[-rank_p:]) != self.prior_shape):
        raise ValueError(f"each item needs {self.coding_rank} dimensions ending in {self.prior_shape}: "
                         f"received shape {tuple(b.shape)}")
    if not items:
      raise ValueError("`bottlenecks` is empty")
    coff, qoff = self._flat_tables(dev)
    # every item holds whole rows of prior_shape, so channel mode's rows line up across items
    return self._encode_ragged([tuple(b.shape) for b in items], torch.cat([b.reshape(-1) for b in items]), qoff,
                               coff, return_decoded=return_decoded, substreams=substreams)

  def decompress_ragged(self, strings, broadcast_shapes, *, substreams=1):
    """Inverse of compress_ragged: item i has shape `broadcast_shapes[i] + prior_shape` and equals
    `decompress(strings[i:i+1], broadcast_shapes[i])[0]`.  The items are views into one allocation."""
    self._check_compression()
    shapes = [tuple(int(d) for d in np.asarray(s).reshape(-1)) + self.prior_shape for s in broadcast_shapes]
    strings = self._strings(strings, len(shapes))
    coff, qoff = self._flat_tables(strings.bytes_dev.device)
    return self._decode_ragged(strings, shapes, qoff, coff, substreams=substreams)

  def get_config(self):
    """continuous_batched.py:424-436."""
    config = super().get_config()
    config.update(prior_shape=tuple(map(int, self.prior_shape)), offset_heuristic=self.offset_heuristic,
                  quantization_offset=self.quantization_offset is not None)
    return config

  @classmethod
  def from_config(cls, config):
    config = dict(config)
    dt = config.pop("bottleneck_dtype", "float32")
    return cls(bottleneck_dtype=getattr(torch, dt) if isinstance(dt, str) else dt, **config)


class ContinuousIndexedEntropyModel(ContinuousEntropyModelBase):
  """continuous_indexed.py:30-428: the table of every element is selected by an index tensor."""

  def __init__(self, prior_fn, index_ranges, parameter_fns, coding_rank, channel_axis=-1, compression=False,
               stateless=False, expected_grads=False, tail_mass=2**-8, range_coder_precision=12,
               bottleneck_dtype=None, prior_dtype=torch.float32, decode_sanity_check=True, laplace_tail_mass=0):
    if not callable(prior_fn):
      raise TypeError("`prior_fn` must be a class or factory function.")
    for name, fn in parameter_fns.items():
      if not isinstance(name, str):
        raise TypeError("`parameter_fns` must have string keys.")
      if not callable(fn):
        raise TypeError(f"`parameter_fns['{name}']` must be callable.")
    super().__init__(coding_rank=coding_rank, compression=compression, stateless=stateless,
                     expected_grads=expected_grads, tail_mass=tail_mass, bottleneck_dtype=bottleneck_dtype,
                     laplace_tail_mass=laplace_tail_mass)
    self._index_ranges = tuple(int(r) for r in index_ranges)
    if not self.index_ranges:
      raise ValueError("`index_ranges` must have at least one element.")
    self._channel_axis = None if channel_axis is None else int(channel_axis)
    if self.channel_axis is None and len(self.index_ranges) > 1:
      raise ValueError("`channel_axis` can't be `None` for `len(index_ranges) > 1`.")
    self._prior_fn = prior_fn
    self._parameter_fns = dict(parameter_fns)
    self._prior_dtype = prior_dtype
    self.decode_sanity_check = decode_sanity_check
    if self.compression:
      if self.channel_axis is None:
        indexes = torch.arange(self.index_ranges[0], dtype=torch.int32)
      else:
        grids = torch.meshgrid(*[torch.arange(r, dtype=torch.int32) for r in self.index_ranges], indexing="ij")
        indexes = torch.stack(grids, dim=self.channel_axis)
      self._set_prior(self._make_prior(indexes), register=False)
      cdf, cdf_offset = self._build_tables(self.prior, range_coder_precision)
      self._init_compression(cdf, cdf_offset, None)

  index_ranges = property(lambda self: self._index_ranges)
  parameter_fns = property(lambda self: self._parameter_fns)
  prior_dtype = property(lambda self: self._prior_dtype)
  prior_fn = property(lambda self: self._prior_fn)
  channel_axis = property(lambda self: self._channel_axis)

  def _make_prior(self, indexes):
    indexes = indexes.to(self.prior_dtype)
    parameters = {k: f(indexes) for k, f in self.parameter_fns.items()}
    prior = self.prior_fn(**parameters)
    assert prior.dtype == self.prior_dtype
    return prior

  def _normalize_indexes(self, indexes):
    """continuous_indexed.py:272-281."""
    indexes = math_ops.lower_bound(indexes, 0.)
    if self.channel_axis is None:
      bounds = torch.tensor(self.index_ranges[0] - 1, dtype=indexes.dtype, device=indexes.device)
    else:
      axes = [1] * indexes.dim()
      axes[self.channel_axis] = len(self.index_ranges)
      bounds = torch.tensor([s - 1 for s in self.index_ranges], dtype=indexes.dtype,
                            device=indexes.device).reshape(axes)
    return math_ops.upper_bound(indexes, bounds)

  def _flatten_indexes(self, indexes):
    """continuous_indexed.py:283-289."""
    indexes = indexes.to(torch.int32)
    if self.channel_axis is None:
      return indexes
    strides = np.cumprod((self.index_ranges + (1,))[::-1])[::-1][1:]
    strides = torch.tensor(strides.copy(), dtype=torch.int32, device=indexes.device)
    return (indexes.movedim(self.channel_axis, -1) * strides).sum(dim=-1, dtype=torch.int32)  # integer matmul does not exist on CUDA

  def forward(self, bottleneck, indexes, training=True):
    """continuous_indexed.py:291-334."""
    bottleneck = torch.as_tensor(bottleneck).to(self.bottleneck_dtype)
    indexes = self._normalize_indexes(torch.as_tensor(indexes, dtype=self.prior_dtype, device=bottleneck.device))
    if training:
      def log_prob_fn(x, idx):
        return self._log_prob(self._make_prior(idx), x)
      log_probs, perturbed = math_ops.perturb_and_apply(log_prob_fn, bottleneck, indexes,
                                                        expected_grads=self.expected_grads)
    else:
      prior = self._make_prior(indexes)
      perturbed = self.quantize(bottleneck)
      log_probs = self._log_prob(prior, perturbed)
    axes = tuple(range(-self.coding_rank, 0))
    bits = (log_probs.sum(dim=axes) if axes else log_probs) / -math.log(2.)
    return perturbed, bits

  def quantize(self, bottleneck):
    return math_ops.round_st(torch.as_tensor(bottleneck).to(self.bottleneck_dtype))

  def compress(self, bottleneck, indexes, fused=True, _loc=None, *, substreams=1):
    """continuous_indexed.py:354-386.  `substreams` as in ContinuousBatchedEntropyModel.compress."""
    self._check_compression()
    dev = _cuda()
    bottleneck = torch.as_tensor(bottleneck).to(device=dev, dtype=self.bottleneck_dtype)
    indexes = self._normalize_indexes(torch.as_tensor(indexes).to(device=dev, dtype=self.prior_dtype))
    flat = self._flatten_indexes(indexes)
    fshape = tuple(flat.shape)
    return self._encode(fshape[:len(fshape) - self.coding_rank], bottleneck, _loc, self.cdf_offset.to(dev), flat,
                        fused, substreams)

  def decompress(self, strings, indexes, fused=True, _loc=None, *, substreams=1):
    """continuous_indexed.py:388-417."""
    self._check_compression()
    strings = self._strings(strings)
    dev = strings.bytes_dev.device
    indexes = self._normalize_indexes(torch.as_tensor(indexes).to(device=dev, dtype=self.prior_dtype))
    flat = self._flatten_indexes(indexes)
    fshape = tuple(flat.shape)
    return self._decode(strings, fshape[len(fshape) - self.coding_rank:], _loc, self.cdf_offset.to(dev), flat, fused,
                        substreams)

  # -- ragged batches: items of different shapes, one range-coder launch (an extension; the reference has none) --
  def _ragged_indexes(self, indexes, dev):
    """Normalised, flattened table indexes of every item, concatenated, and the items' coding shapes."""
    indexes = [torch.as_tensor(i).to(device=dev, dtype=self.prior_dtype) for i in indexes]
    if not indexes:
      raise ValueError("`indexes` is empty")
    if self.channel_axis is None:  # elementwise: normalise all items at once
      flat = self._flatten_indexes(self._normalize_indexes(torch.cat([i.reshape(-1) for i in indexes])))
      shapes = [tuple(i.shape) for i in indexes]
    else:
      per_item = [self._flatten_indexes(self._normalize_indexes(i)) for i in indexes]
      flat = torch.cat([f.reshape(-1) for f in per_item])
      shapes = [tuple(f.shape) for f in per_item]
    for s in shapes:
      if len(s) != self.coding_rank:
        raise ValueError(f"each item needs {self.coding_rank} dimensions: received indexes for shape {s}")
    return flat, shapes

  def compress_ragged(self, bottlenecks, indexes, _loc=None, return_decoded=False, *, substreams=1):
    """Compresses a list of coding units of different shapes (each with exactly `coding_rank` dimensions) in one
    range-coder launch.  Returns a Strings of shape (k,) whose string i equals `compress(bottlenecks[i],
    indexes[i])`.

    `return_decoded=True` returns `(strings, items)` with `items` equal, bit for bit, to
    `decompress_ragged(strings, indexes)`: written by the encoder itself for a float32 bottleneck, decoded from the
    fresh strings otherwise."""
    self._check_compression()
    dev = _cuda()
    items = [torch.as_tensor(b).to(device=dev, dtype=self.bottleneck_dtype) for b in bottlenecks]
    flat, shapes = self._ragged_indexes(indexes, dev)
    if len(items) != len(shapes) or any(tuple(b.shape) != s for b, s in zip(items, shapes)):
      raise ValueError(f"bottleneck shapes {[tuple(b.shape) for b in items]} do not match the indexes' {shapes}")
    loc = None if _loc is None else torch.cat([torch.as_tensor(l).to(dev).reshape(-1) for l in _loc])
    b = torch.cat([b.reshape(-1) for b in items])
    if loc is not None and loc.numel() != b.numel():
      raise ValueError("each `loc` item must have the shape of its bottleneck")
    return self._encode_ragged(shapes, b, loc, self.cdf_offset.to(dev), flat, return_decoded, substreams)

  def decompress_ragged(self, strings, indexes, _loc=None, *, substreams=1):
    """Inverse of compress_ragged: item i has the coding shape of `indexes[i]`.  The items are views into one
    allocation."""
    self._check_compression()
    strings = self._strings(strings, len(indexes))
    dev = strings.bytes_dev.device
    flat, shapes = self._ragged_indexes(indexes, dev)
    loc = None if _loc is None else torch.cat([torch.as_tensor(l).to(dev).reshape(-1) for l in _loc])
    return self._decode_ragged(strings, shapes, loc, self.cdf_offset.to(dev), flat, substreams)

  def get_config(self):
    raise NotImplementedError("Serializing indexed entropy models is not yet implemented.")

  @classmethod
  def from_config(cls, config):
    raise NotImplementedError("Serializing indexed entropy models is not yet implemented.")


class LocationScaleIndexedEntropyModel(ContinuousIndexedEntropyModel):
  """continuous_indexed.py:431-633."""

  def __init__(self, prior_fn, num_scales, scale_fn, coding_rank, compression=False, stateless=False,
               expected_grads=False, tail_mass=2**-8, range_coder_precision=12, bottleneck_dtype=None,
               prior_dtype=torch.float32, laplace_tail_mass=0):
    num_scales = int(num_scales)
    super().__init__(prior_fn=prior_fn, index_ranges=(num_scales,),
                     parameter_fns=dict(loc=lambda _: 0., scale=scale_fn), coding_rank=coding_rank,
                     channel_axis=None, compression=compression, stateless=stateless,
                     expected_grads=expected_grads, tail_mass=tail_mass,
                     range_coder_precision=range_coder_precision, bottleneck_dtype=bottleneck_dtype,
                     prior_dtype=prior_dtype, laplace_tail_mass=laplace_tail_mass)

  def forward(self, bottleneck, scale_indexes, loc=None, training=True):
    if loc is None:
      return super().forward(bottleneck, scale_indexes, training=training)
    perturbed, bits = super().forward(bottleneck - loc, scale_indexes, training=training)
    return perturbed + loc, bits

  def quantize(self, bottleneck, loc=None):
    return math_ops.round_st(torch.as_tensor(bottleneck).to(self.bottleneck_dtype), loc)

  def compress(self, bottleneck, scale_indexes, loc=None, fused=True, *, substreams=1):
    return super().compress(bottleneck, scale_indexes, fused=fused, _loc=loc, substreams=substreams)

  def decompress(self, strings, scale_indexes, loc=None, fused=True, *, substreams=1):
    return super().decompress(strings, scale_indexes, fused=fused, _loc=loc, substreams=substreams)

  def compress_ragged(self, bottlenecks, scale_indexes, loc=None, return_decoded=False, *, substreams=1):
    """`loc`: None or a list with one tensor per item."""
    return super().compress_ragged(bottlenecks, scale_indexes, _loc=loc, return_decoded=return_decoded,
                                   substreams=substreams)

  def decompress_ragged(self, strings, scale_indexes, loc=None, *, substreams=1):
    return super().decompress_ragged(strings, scale_indexes, _loc=loc, substreams=substreams)


# ------------------------------------------------------------------------------------------------
# Universal quantisation (universal.py:30-603): "quantisation" is additive uniform noise whose value is shared by
# sender and receiver through a stateless pseudo-random stream; coding runs in index mode with one extra leading
# index, the noise level.
# ------------------------------------------------------------------------------------------------
_M32 = 0xFFFFFFFF


def _philox4x32(counter, key, rounds=10):
  """Philox-4x32-10 (Salmon et al., SC'11) on int64 tensors holding uint32 words: counter [n, 4] -> [n, 4]."""
  c = [counter[:, i].clone() for i in range(4)]
  k0, k1 = int(key[0]) & _M32, int(key[1]) & _M32
  for _ in range(rounds):
    p0, p1 = c[0] * 0xD2511F53, c[2] * 0xCD9E8D57          # < 2^64 as unsigned: split the products by hand
    hi0 = ((c[0] >> 16) * 0xD2511F53 + (((c[0] & 0xFFFF) * 0xD2511F53) >> 16)) >> 16
    hi1 = ((c[2] >> 16) * 0xCD9E8D57 + (((c[2] & 0xFFFF) * 0xCD9E8D57) >> 16)) >> 16
    lo0, lo1 = p0 & _M32, p1 & _M32
    c = [(hi1 ^ c[1] ^ k0) & _M32, lo1, (hi0 ^ c[3] ^ k1) & _M32, lo0]
    k0, k1 = (k0 + 0x9E3779B9) & _M32, (k1 + 0xBB67AE85) & _M32
  return torch.stack(c, dim=1)


def stateless_uniform_int(shape, seed, maxval, device=None):
  """Counter-based stand-in for `tf.random.stateless_uniform(shape, seed, 0, maxval, int32)` (universal.py:33-39):
  element i is word i % 4 of Philox-4x32-10(counter = i // 4, key = seed), reduced modulo `maxval`.  It depends on
  nothing but (seed, i), so sender and receiver -- on any device -- draw the same noise levels.  TensorFlow's own
  key / counter conventions are not reproduced (there is no TF here to pin them against): strings written with
  universal quantisation decode with THIS implementation, not with the reference's.  On a CUDA device the draw is one
  kernel (functional.stateless_uniform_int); on the CPU it is the int64 torch arithmetic of _philox4x32."""
  shape = tuple(int(d) for d in shape)
  n = gen_ops._prod(shape)
  if device is not None and torch.device(device).type == "cuda":
    return F.stateless_uniform_int(n, seed, maxval, device).reshape(shape)
  blocks = (n + 3) // 4
  counter = torch.zeros(blocks, 4, dtype=torch.int64, device=device)
  idx = torch.arange(blocks, dtype=torch.int64, device=device)
  counter[:, 0] = idx & _M32
  counter[:, 1] = idx >> 32
  words = _philox4x32(counter, seed).reshape(-1)[:n]
  return (words % int(maxval)).to(torch.int32).reshape(shape)


_NOISE_SEED = (1234, 1234)  # universal.py:33-39


def _add_offset_indexes(indexes, num_noise_levels):
  """universal.py:30-42: prepends the shared pseudo-random noise-level index to the last axis of `indexes`."""
  offset_indexes = stateless_uniform_int(indexes.shape[:-1], _NOISE_SEED, num_noise_levels, indexes.device)
  return torch.cat((offset_indexes.to(indexes.dtype)[..., None], indexes), dim=-1)


def _offset_indexes_to_offset(offset_indexes, num_noise_levels, dtype):
  """universal.py:45-47: level k of n -> (k + 1) / (n + 1) - 0.5."""
  return ((offset_indexes.to(torch.float64) + 1) / (num_noise_levels + 1) - 0.5).to(dtype)


def _range_coding_offsets(num_noise_levels, prior_rank, dtype):
  """universal.py:55-62."""
  offset_indexes = torch.arange(num_noise_levels, dtype=dtype).reshape([-1] + [1] * prior_rank)
  return _offset_indexes_to_offset(offset_indexes, num_noise_levels, dtype)


def _on_cuda(device):
  return torch.device(device).type == "cuda"


def _kernel_offset_dtype(bottleneck_dtype):
  """The coding-tensor kernel writes float32 offsets for float32 bottlenecks (the fused coder's type) and float64
  for every other type, which torch then casts as _offset_indexes_to_offset does."""
  return torch.float32 if bottleneck_dtype == torch.float32 else torch.float64


class UniversalBatchedEntropyModel(ContinuousEntropyModelBase):
  """universal.py:65-330."""

  _coder16_models = False  # (offsets follow a float64 rule, see _kernel_offset_dtype)

  def __init__(self, prior, coding_rank, compression=False, laplace_tail_mass=0.0, expected_grads=False,
               tail_mass=2**-8, range_coder_precision=12, bottleneck_dtype=None, num_noise_levels=15, stateless=False,
               decode_sanity_check=True):
    super().__init__(coding_rank=coding_rank, compression=compression, stateless=stateless,
                     expected_grads=expected_grads, tail_mass=tail_mass, bottleneck_dtype=bottleneck_dtype,
                     laplace_tail_mass=laplace_tail_mass)
    self._set_prior(prior)
    self._num_noise_levels = int(num_noise_levels)
    self._prior_shape = tuple(int(s) for s in prior.batch_shape)
    if self.coding_rank < len(self.prior_shape):
      raise ValueError("`coding_rank` can't be smaller than `prior_shape`.")
    self.decode_sanity_check = decode_sanity_check
    if self.compression:
      offset = _range_coding_offsets(self._num_noise_levels, len(self.prior_shape), self.bottleneck_dtype)
      cdf, cdf_offset = self._build_tables(self.prior, range_coder_precision, offset=offset)
      self._init_compression(cdf, cdf_offset, None)

  prior_shape = property(lambda self: self._prior_shape)

  @property
  def prior_shape_tensor(self):
    return torch.tensor(self.prior_shape, dtype=torch.int32)

  def _item_coding_tensors(self, lengths, device):
    """Flat table index and offset (in bottleneck_dtype) of items of `lengths` elements, one after the other, from
    one kernel launch; the noise position restarts in every item, as in a compress of that item alone."""
    flat, offset = F.universal_coding_tensors(lengths, self._num_noise_levels,
                                              _kernel_offset_dtype(self.bottleneck_dtype), device,
                                              prior_size=gen_ops._prod(self.prior_shape), seed=_NOISE_SEED)
    return flat, offset.to(self.bottleneck_dtype)

  def _unit_coding_tensors(self, units, broadcast_shape, device):
    """Table index and offset of `units` coding units of shape broadcast_shape + prior_shape, shaped
    (units,) + that shape.  A CUDA device writes every unit directly; the CPU broadcasts one unit."""
    full_shape = tuple(broadcast_shape) + self.prior_shape
    if units > 0 and _on_cuda(device):
      flat, offset = self._item_coding_tensors([gen_ops._prod(full_shape)] * units, device)
      return flat.reshape((units,) + full_shape), offset.reshape((units,) + full_shape)
    indexes, offset = self._compute_indexes_and_offset(broadcast_shape, device)
    return (torch.broadcast_to(indexes, (units,) + full_shape).contiguous(),
            torch.broadcast_to(offset, (units,) + full_shape).contiguous())

  def _compute_indexes_and_offset(self, broadcast_shape, device):
    """universal.py:147-170 -> (flat table index, quantisation offset), both of shape broadcast_shape + prior_shape.
    One kernel launch on a CUDA device, torch operations on the CPU."""
    broadcast_shape = tuple(int(d) for d in broadcast_shape)
    if _on_cuda(device):
      flat, offset = self._item_coding_tensors([gen_ops._prod(broadcast_shape + self.prior_shape)], device)
      return flat.reshape(broadcast_shape + self.prior_shape), offset.reshape(broadcast_shape + self.prior_shape)
    prior_size = gen_ops._prod(self.prior_shape)
    indexes = torch.arange(prior_size, dtype=torch.int32, device=device)
    indexes = torch.broadcast_to(indexes, broadcast_shape + (prior_size,))[..., None]
    indexes = _add_offset_indexes(indexes, self._num_noise_levels)
    offset = _offset_indexes_to_offset(indexes[..., 0], self._num_noise_levels, self.bottleneck_dtype)
    flat = indexes[..., 0] * prior_size + indexes[..., 1]          # strides of index_ranges [levels, prior_size]
    full_shape = broadcast_shape + self.prior_shape
    return flat.reshape(full_shape).to(torch.int32), offset.reshape(full_shape)

  def forward(self, bottleneck, training=True):
    """universal.py:172-211."""
    bottleneck = torch.as_tensor(bottleneck).to(self.bottleneck_dtype)
    log_prob_fn = functools.partial(self._log_prob, self.prior)
    if training:
      log_probs, perturbed = math_ops.perturb_and_apply(log_prob_fn, bottleneck, expected_grads=self.expected_grads)
    else:
      coding_shape = tuple(bottleneck.shape[bottleneck.dim() - self.coding_rank:])
      broadcast_shape = coding_shape[:self.coding_rank - len(self.prior_shape)]
      _, offset = self._compute_indexes_and_offset(broadcast_shape, bottleneck.device)
      perturbed = torch.round(bottleneck - offset) + offset
      log_probs = log_prob_fn(perturbed)
    axes = tuple(range(-self.coding_rank, 0))
    return perturbed, log_probs.sum(dim=axes) / -math.log(2.)

  def compress(self, bottleneck, fused=True):
    """universal.py:213-251."""
    self._check_compression()
    dev = _cuda()
    bottleneck = torch.as_tensor(bottleneck).to(device=dev, dtype=self.bottleneck_dtype)
    shape = tuple(bottleneck.shape)
    batch_shape, coding_shape = shape[:len(shape) - self.coding_rank], shape[len(shape) - self.coding_rank:]
    broadcast_shape = coding_shape[:self.coding_rank - len(self.prior_shape)]
    if coding_shape == broadcast_shape + self.prior_shape:  # (else prior dimensions of size 1 are broadcast)
      indexes, offset = self._unit_coding_tensors(gen_ops._prod(batch_shape), broadcast_shape, dev)
      indexes, offset = indexes.reshape(shape), offset.reshape(shape)
    else:
      indexes, offset = self._compute_indexes_and_offset(broadcast_shape, dev)
      indexes = torch.broadcast_to(indexes, shape).contiguous()
      offset = torch.broadcast_to(offset, shape).contiguous()
    return self._encode(batch_shape, bottleneck, offset, self.cdf_offset.to(dev), indexes, fused)

  def decompress(self, strings, broadcast_shape, fused=True):
    """universal.py:253-289."""
    self._check_compression()
    strings = self._strings(strings)
    dev = strings.bytes_dev.device
    broadcast_shape = tuple(int(d) for d in np.asarray(broadcast_shape).reshape(-1))
    decode_shape = broadcast_shape + self.prior_shape
    output_shape = tuple(strings.shape) + decode_shape
    indexes, offset = self._unit_coding_tensors(gen_ops._prod(strings.shape), broadcast_shape, dev)
    indexes, offset = indexes.reshape(output_shape), offset.reshape(output_shape)
    return self._decode(strings, decode_shape, offset, self.cdf_offset.to(dev), indexes, fused)

  # -- ragged batches: items of different shapes, one range-coder launch (an extension; the reference has none) --
  def compress_ragged(self, bottlenecks, return_decoded=False):
    """Compresses a list of coding units of different shapes in one range-coder launch.  Each item has exactly
    `coding_rank` dimensions ending in `prior_shape` (no broadcasting).  Returns a Strings of shape (k,) whose string
    i equals `compress(bottlenecks[i])`: the noise levels of item i are drawn over its own positions.

    `return_decoded=True` returns `(strings, items)` with `items` equal, bit for bit, to
    `decompress_ragged(strings, ...)`: written by the encoder itself for a float32 bottleneck, decoded from the
    fresh strings otherwise."""
    self._check_compression()
    dev = _cuda()
    items = [torch.as_tensor(b).to(device=dev, dtype=self.bottleneck_dtype) for b in bottlenecks]
    rank_p = len(self.prior_shape)
    for b in items:
      if b.dim() != self.coding_rank or (rank_p and tuple(b.shape[-rank_p:]) != self.prior_shape):
        raise ValueError(f"each item needs {self.coding_rank} dimensions ending in {self.prior_shape}: "
                         f"received shape {tuple(b.shape)}")
    if not items:
      raise ValueError("`bottlenecks` is empty")
    indexes, offset = self._item_coding_tensors([b.numel() for b in items], dev)
    return self._encode_ragged([tuple(b.shape) for b in items], torch.cat([b.reshape(-1) for b in items]), offset,
                               self.cdf_offset.to(dev), indexes, return_decoded)

  def decompress_ragged(self, strings, broadcast_shapes):
    """Inverse of compress_ragged: item i has shape `broadcast_shapes[i] + prior_shape` and equals
    `decompress(strings[i:i+1], broadcast_shapes[i])[0]`.  The items are views into one allocation."""
    self._check_compression()
    shapes = [tuple(int(d) for d in np.asarray(s).reshape(-1)) + self.prior_shape for s in broadcast_shapes]
    strings = self._strings(strings, len(shapes))
    dev = strings.bytes_dev.device
    indexes, offset = self._item_coding_tensors([gen_ops._prod(s) for s in shapes], dev)
    return self._decode_ragged(strings, shapes, offset, self.cdf_offset.to(dev), indexes)

  def get_config(self):
    raise NotImplementedError()


class UniversalIndexedEntropyModel(ContinuousEntropyModelBase):
  """universal.py:292-603."""

  _coder16_models = False  # (offsets follow a float64 rule, see _kernel_offset_dtype)

  def __init__(self, prior_fn, index_ranges, parameter_fns, coding_rank, compression=False, laplace_tail_mass=0.0,
               expected_grads=False, tail_mass=2**-8, range_coder_precision=12, bottleneck_dtype=None,
               prior_dtype=torch.float32, stateless=False, num_noise_levels=15, decode_sanity_check=True):
    if coding_rank <= 0:
      raise ValueError("`coding_rank` must be larger than 0.")
    if not callable(prior_fn):
      raise TypeError("`prior_fn` must be a class or factory function.")
    for name, fn in parameter_fns.items():
      if not isinstance(name, str):
        raise TypeError("`parameter_fns` must have string keys.")
      if not callable(fn):
        raise TypeError(f"`parameter_fns['{name}']` must be callable.")
    super().__init__(coding_rank=coding_rank, compression=compression, stateless=stateless,
                     expected_grads=expected_grads, tail_mass=tail_mass, bottleneck_dtype=bottleneck_dtype,
                     laplace_tail_mass=laplace_tail_mass)
    self._index_ranges = tuple([int(num_noise_levels)] + [int(r) for r in index_ranges])  # extra index: noise level
    if len(self._index_ranges) < 2:
      raise ValueError("`index_ranges` must have at least one element.")
    self._prior_fn = prior_fn
    self._parameter_fns = dict(parameter_fns)
    self._prior_dtype = prior_dtype
    self._num_noise_levels = int(num_noise_levels)
    self.decode_sanity_check = decode_sanity_check
    if self.compression:
      grids = torch.meshgrid(*[torch.arange(r, dtype=torch.int32) for r in self.index_ranges_without_offsets], indexing="ij")
      indexes = torch.stack(grids, dim=-1)
      self._set_prior(self._make_prior(indexes), register=False)
      offset = _range_coding_offsets(self._num_noise_levels, len(self.prior.batch_shape), self.bottleneck_dtype)
      cdf, cdf_offset = self._build_tables(self.prior, range_coder_precision, offset=offset)
      self._init_compression(cdf, cdf_offset, None)

  index_ranges = property(lambda self: self._index_ranges)
  parameter_fns = property(lambda self: self._parameter_fns)
  prior_dtype = property(lambda self: self._prior_dtype)
  prior_fn = property(lambda self: self._prior_fn)
  index_ranges_without_offsets = property(lambda self: self._index_ranges[1:])

  def _make_prior(self, indexes):
    indexes = indexes.to(self.prior_dtype)
    return self.prior_fn(**{k: f(indexes) for k, f in self.parameter_fns.items()})

  def _flatten_indexes(self, indexes):
    """universal.py:446-449."""
    strides = np.cumprod((self.index_ranges + (1,))[::-1])[::-1][1:]
    strides = torch.tensor(strides.copy(), dtype=torch.int32, device=indexes.device)
    return (indexes.to(torch.int32) * strides).sum(dim=-1, dtype=torch.int32)  # integer matmul does not exist on CUDA

  def _normalize_indexes(self, indexes):
    """universal.py:451-466: clips every index to its range (with or without the leading noise-level index)."""
    num = indexes.shape[-1]
    ranges = self.index_ranges if num == len(self.index_ranges) else self.index_ranges_without_offsets
    assert num == len(ranges)
    indexes = math_ops.lower_bound(indexes, 0.)
    bounds = torch.tensor([s - 1 for s in ranges], dtype=indexes.dtype, device=indexes.device)
    return math_ops.upper_bound(indexes, bounds.reshape([1] * (indexes.dim() - 1) + [num]))

  def _offset_from_indexes(self, indexes_with_offsets):
    return _offset_indexes_to_offset(indexes_with_offsets[..., 0], self._num_noise_levels, self.bottleneck_dtype)

  def forward(self, bottleneck, indexes, training=True):
    """universal.py:473-528."""
    bottleneck = torch.as_tensor(bottleneck).to(self.bottleneck_dtype)
    indexes = self._normalize_indexes(torch.as_tensor(indexes, dtype=self.prior_dtype, device=bottleneck.device))
    if training:
      def log_prob_fn(x, idx):
        return self._log_prob(self._make_prior(idx), x)
      log_probs, perturbed = math_ops.perturb_and_apply(log_prob_fn, bottleneck, indexes,
                                                        expected_grads=self.expected_grads)
    else:
      prior = self._make_prior(indexes)
      if self._kernel_path(indexes.device):
        offset = self._coding_tensors(indexes.detach(), indexes.device)[1]
      else:
        offset = self._offset_from_indexes(_add_offset_indexes(indexes, self._num_noise_levels))
      perturbed = torch.round(bottleneck - offset) + offset
      log_probs = self._log_prob(prior, perturbed)
    axes = tuple(range(-self.coding_rank, 0))
    return perturbed, log_probs.sum(dim=axes) / -math.log(2.)

  def _kernel_path(self, device):
    """Whether the coding tensors come from the CUDA kernel: on a CUDA device with a float32 / float64 `prior_dtype`.
    16-bit index types keep the torch operations (whose noise draw is still the kernel's on a CUDA device)."""
    return _on_cuda(device) and self.prior_dtype in F.UNIVERSAL_INDEX_DTYPES

  def _check_index_shape(self, indexes):
    num = len(self.index_ranges_without_offsets)
    if indexes.dim() == 0 or indexes.shape[-1] != num:
      raise ValueError(f"`indexes` needs a last dimension of {num} (one per index range): received shape "
                       f"{tuple(indexes.shape)}")

  def _kernel_coding_tensors(self, lengths, indexes, dev):
    flat, offset = F.universal_coding_tensors(lengths, self._num_noise_levels,
                                              _kernel_offset_dtype(self.bottleneck_dtype), dev, indexes=indexes,
                                              index_ranges=self.index_ranges_without_offsets, seed=_NOISE_SEED)
    return flat, offset.to(self.bottleneck_dtype)

  def _coding_tensors(self, indexes, dev):
    """universal.py:530-598: (flat table index, offset in bottleneck_dtype), both of shape indexes.shape[:-1].  The
    noise is drawn over every position of that shape, batch dimensions included."""
    indexes = torch.as_tensor(indexes).to(device=dev, dtype=self.prior_dtype)
    if self._kernel_path(dev):
      self._check_index_shape(indexes)
      shape = tuple(indexes.shape[:-1])
      flat, offset = self._kernel_coding_tensors([gen_ops._prod(shape)], indexes, dev)
      return flat.reshape(shape), offset.reshape(shape)
    indexes = self._normalize_indexes(_add_offset_indexes(indexes, self._num_noise_levels))
    return self._flatten_indexes(indexes).contiguous(), self._offset_from_indexes(indexes).contiguous()

  def _ragged_coding_tensors(self, indexes, dev):
    """Flat table indexes and offsets of every item, concatenated (the noise position restarting in every item), and
    the items' coding shapes."""
    indexes = [torch.as_tensor(i).to(device=dev, dtype=self.prior_dtype) for i in indexes]
    if not indexes:
      raise ValueError("`indexes` is empty")
    for i in indexes:
      self._check_index_shape(i)
    shapes = [tuple(i.shape[:-1]) for i in indexes]
    for s in shapes:
      if len(s) != self.coding_rank:
        raise ValueError(f"each item needs {self.coding_rank} dimensions: received indexes for shape {s}")
    if self._kernel_path(dev):
      flat, offset = self._kernel_coding_tensors([gen_ops._prod(s) for s in shapes],
                                                 torch.cat([i.reshape(-1) for i in indexes]), dev)
    else:
      parts = [self._coding_tensors(i, dev) for i in indexes]
      flat = torch.cat([p[0].reshape(-1) for p in parts])
      offset = torch.cat([p[1].reshape(-1) for p in parts])
    return flat, offset, shapes

  def compress(self, bottleneck, indexes, fused=True):
    """universal.py:530-566."""
    self._check_compression()
    dev = _cuda()
    bottleneck = torch.as_tensor(bottleneck).to(device=dev, dtype=self.bottleneck_dtype)
    flat, offset = self._coding_tensors(indexes, dev)
    fshape = tuple(flat.shape)
    return self._encode(fshape[:len(fshape) - self.coding_rank], bottleneck, offset, self.cdf_offset.to(dev), flat,
                        fused)

  def decompress(self, strings, indexes, fused=True):
    """universal.py:568-598."""
    self._check_compression()
    strings = self._strings(strings)
    dev = strings.bytes_dev.device
    flat, offset = self._coding_tensors(indexes, dev)
    fshape = tuple(flat.shape)
    return self._decode(strings, fshape[len(fshape) - self.coding_rank:], offset, self.cdf_offset.to(dev), flat,
                        fused)

  # -- ragged batches: items of different shapes, one range-coder launch (an extension; the reference has none) --
  def compress_ragged(self, bottlenecks, indexes, return_decoded=False):
    """Compresses a list of coding units of different shapes (each with exactly `coding_rank` dimensions) in one
    range-coder launch.  Returns a Strings of shape (k,) whose string i equals `compress(bottlenecks[i],
    indexes[i])`.  The noise levels of item i are drawn over its own positions, so the strings differ from those of
    one `compress` of the items stacked into a batch, which draws them over the batch dimensions too.

    `return_decoded=True` returns `(strings, items)` with `items` equal, bit for bit, to
    `decompress_ragged(strings, indexes)`: written by the encoder itself for a float32 bottleneck, decoded from the
    fresh strings otherwise."""
    self._check_compression()
    dev = _cuda()
    items = [torch.as_tensor(b).to(device=dev, dtype=self.bottleneck_dtype) for b in bottlenecks]
    flat, offset, shapes = self._ragged_coding_tensors(indexes, dev)
    if len(items) != len(shapes) or any(tuple(b.shape) != s for b, s in zip(items, shapes)):
      raise ValueError(f"bottleneck shapes {[tuple(b.shape) for b in items]} do not match the indexes' {shapes}")
    return self._encode_ragged(shapes, torch.cat([b.reshape(-1) for b in items]), offset, self.cdf_offset.to(dev),
                               flat, return_decoded)

  def decompress_ragged(self, strings, indexes):
    """Inverse of compress_ragged: item i has the coding shape of `indexes[i]` (without its last dimension).  The
    items are views into one allocation."""
    self._check_compression()
    strings = self._strings(strings, len(indexes))
    dev = strings.bytes_dev.device
    flat, offset, shapes = self._ragged_coding_tensors(indexes, dev)
    return self._decode_ragged(strings, shapes, offset, self.cdf_offset.to(dev), flat)

  def get_config(self):
    raise NotImplementedError()


class MixtureEntropyModel(nn.Module):
  """Every element coded under its own mixture of K Normal or Logistic components (Cheng et al. 2020), with its CDF
  built on the device from (weight, loc, scale) (DESIGN §3.18).  There are no tables: `weight`, `loc` and `scale`
  have the bottleneck's shape plus a last axis of K components; the weights need not sum to 1 and are normalised.
  The string of a coding unit (the last `coding_rank` axes) is one range-coded stream, or S independently decodable
  ones with `substreams` = S (DESIGN §3.14).  float32 only."""

  decode_sanity_check = True

  def __init__(self, family="normal", coding_rank=0, tail_mass=2**-8, range_coder_precision=16, max_support=256):
    super().__init__()
    if family not in F.MIXTURE_FAMILIES:
      raise ValueError(f"`family` must be one of {sorted(F.MIXTURE_FAMILIES)}: {family!r}")
    if int(coding_rank) < 0:
      raise ValueError("`coding_rank` must be at least 0.")
    if not 0 < tail_mass < 1:
      raise ValueError("`tail_mass` must be between 0 and 1.")
    if not 1 <= int(max_support) <= 256:
      raise ValueError(f"`max_support` must be in [1, 256]: {max_support}")
    if not 1 <= int(range_coder_precision) <= 16 or (1 << int(range_coder_precision)) <= int(max_support):
      raise ValueError(f"`range_coder_precision` must be in [1, 16] with 2^precision > max_support: "
                       f"{range_coder_precision}")
    self.family = family
    self.coding_rank = int(coding_rank)
    self.tail_mass = float(tail_mass)
    self.range_coder_precision = int(range_coder_precision)
    self.max_support = int(max_support)

  def _prior(self, weight, loc, scale):
    cls = D.NoisyNormalMixture if self.family == "normal" else D.NoisyLogisticMixture
    return cls(loc, scale, weight / weight.sum(-1, keepdim=True))

  def _check(self, bottleneck, weight, loc, scale):
    for name, t in (("bottleneck", bottleneck), ("weight", weight), ("loc", loc), ("scale", scale)):
      if t is None and name == "bottleneck":  # (decompress: the parameters alone give the shape)
        continue
      if not isinstance(t, torch.Tensor) or t.dtype != torch.float32:
        raise ValueError(f"MixtureEntropyModel codes float32 only: `{name}` is "
                         f"{getattr(t, 'dtype', type(t).__name__)}")
    if weight.dim() < 1 or weight.shape != loc.shape or weight.shape != scale.shape:
      raise ValueError(f"weight, loc and scale must share one shape: {tuple(weight.shape)}, {tuple(loc.shape)}, "
                       f"{tuple(scale.shape)}")
    if bottleneck is not None and tuple(bottleneck.shape) != tuple(weight.shape[:-1]):
      raise ValueError(f"the parameters' shape {tuple(weight.shape)} must be the bottleneck's "
                       f"{tuple(bottleneck.shape)} plus the components")
    if weight.dim() - 1 < self.coding_rank:
      raise ValueError(f"coding_rank {self.coding_rank} exceeds the bottleneck's rank {weight.dim() - 1}")

  @staticmethod
  def _components(weights):
    """The one component count K of a list of items' parameters; items with different K are rejected."""
    ks = {int(w.shape[-1]) for w in weights}
    if len(ks) != 1:
      raise ValueError(f"every item must have the same number of components: {sorted(ks)}")
    return ks.pop()

  def forward(self, bottleneck, weight, loc, scale, training=True):
    """(perturbed or rounded bottleneck, bits per coding unit) through the NoisyNormalMixture /
    NoisyLogisticMixture graph: the rate term training already uses."""
    self._check(bottleneck, weight, loc, scale)
    prior = self._prior(weight, loc, scale)
    if training:
      log_probs, perturbed = math_ops.perturb_and_apply(lambda x: prior.log_prob(x), bottleneck,
                                                        expected_grads=False)
    else:
      perturbed = math_ops.round_st(bottleneck)
      log_probs = prior.log_prob(perturbed)
    axes = tuple(range(-self.coding_rank, 0))
    bits = (log_probs.sum(dim=axes) if axes else log_probs) / -math.log(2.)
    return perturbed, bits

  def _coder_args(self):
    return dict(family=self.family, precision=self.range_coder_precision, tail_mass=self.tail_mass,
                max_support=self.max_support)

  @staticmethod
  def _lengths(shapes, substreams):
    """Stream lengths of coding units of these shapes: one stream each, or substream_layout's split of the unit's
    positions along its last axis."""
    if substreams == 1:
      return [gen_ops._prod(s) for s in shapes]
    widths = [max(int(s[-1]), 1) if len(s) else 1 for s in shapes]
    return F.substream_layout([[gen_ops._prod(s) // w] for s, w in zip(shapes, widths)], [[w] for w in widths],
                              substreams)[0]

  def _encode(self, shapes, y, weight, loc, scale, substreams):
    S = gen_ops.check_substreams(substreams)
    strings = F.mixture_encode_ragged(y.reshape(-1), weight, loc, scale, self._lengths(shapes, S),
                                      **self._coder_args())
    return gen_ops.join_substreams(strings, S, (len(shapes),)) if S > 1 else strings

  def _decode(self, strings, shapes, weight, loc, scale, substreams):
    S = gen_ops.check_substreams(substreams)
    if S > 1:
      strings = gen_ops.split_substreams(strings, S)
    return F.mixture_decode_ragged(strings, weight, loc, scale, self._lengths(shapes, S), **self._coder_args())

  def compress(self, bottleneck, weight, loc, scale, *, substreams=1):
    """One string per coding unit: Strings of shape bottleneck.shape[:-coding_rank]."""
    self._check(bottleneck, weight, loc, scale)
    r = self.coding_rank
    batch = tuple(bottleneck.shape[:bottleneck.dim() - r])
    unit = tuple(bottleneck.shape[bottleneck.dim() - r:])
    s = self._encode([unit] * gen_ops._prod(batch), bottleneck, weight, loc, scale, substreams)
    return gen_ops.Strings(s.bytes_dev, s.offsets_dev, batch)

  def decompress(self, strings, weight, loc, scale, *, substreams=1):
    """Inverse of compress: float32 of weight.shape[:-1]."""
    self._check(None, weight, loc, scale)
    r = self.coding_rank
    shape = tuple(weight.shape[:-1])
    batch, unit = shape[:len(shape) - r], shape[len(shape) - r:]
    n = gen_ops._prod(batch)
    if not isinstance(strings, gen_ops.Strings):
      strings = gen_ops.Strings.from_bytes(strings)
    if strings.numel() != n:
      raise ValueError(f"{strings.numel()} strings for a batch of {n} coding units")
    flat = gen_ops.Strings(strings.bytes_dev, strings.offsets_dev, (n,))
    return self._decode(flat, [unit] * n, weight, loc, scale, substreams).reshape(shape)

  def compress_ragged(self, bottlenecks, weights, locs, scales, *, substreams=1):
    """One string per item of a list of differently shaped bottlenecks (each item one coding unit), in one launch
    sequence; string i equals the string of item i alone."""
    items = list(zip(bottlenecks, weights, locs, scales))
    if not items or len({len(bottlenecks), len(weights), len(locs), len(scales)}) != 1:
      raise ValueError("compress_ragged needs at least one item, and as many parameters as bottlenecks")
    for b, w, l, s in items:
      self._check(b, w, l, s)
    K = self._components(weights)
    cat = lambda ts: torch.cat([t.reshape(-1) for t in ts])
    w, l, s = (cat(ts).reshape(-1, K) for ts in (weights, locs, scales))
    return self._encode([tuple(b.shape) for b in bottlenecks], cat(bottlenecks), w, l, s, substreams)

  def decompress_ragged(self, strings, weights, locs, scales, *, substreams=1):
    """Inverse of compress_ragged: a list of float32 items shaped weights[i].shape[:-1]."""
    items = list(zip(weights, locs, scales))
    if not items or len({len(weights), len(locs), len(scales)}) != 1:
      raise ValueError("decompress_ragged needs at least one item, and as many locs and scales as weights")
    for w, l, s in items:
      self._check(None, w, l, s)
    K = self._components(weights)
    shapes = [tuple(w.shape[:-1]) for w in weights]
    if not isinstance(strings, gen_ops.Strings):
      strings = gen_ops.Strings.from_bytes(list(strings), (len(strings),))
    if strings.numel() != len(items):
      raise ValueError(f"{strings.numel()} strings for {len(items)} items")
    cat = lambda ts: torch.cat([t.reshape(-1) for t in ts]).reshape(-1, K)
    out = self._decode(strings, shapes, cat(weights), cat(locs), cat(scales), substreams)
    return gen_ops._split_items(out, shapes)


def EntropyBottleneck(num_channels=None, prior=None, coding_rank=3, compression=True, **kwargs):
  """TFC-1.x name.  In this snapshot of the reference its role is played by
  `ContinuousBatchedEntropyModel(NoisyDeepFactorized(batch_shape=(C,)), coding_rank=3)`
  (models/bls2017.py:103,160-161); this adaptor builds exactly that."""
  if prior is None:
    if num_channels is None:
      raise ValueError("Either `num_channels` or `prior` must be given.")
    prior = D.NoisyDeepFactorized(batch_shape=(int(num_channels),))
  return ContinuousBatchedEntropyModel(prior, coding_rank=coding_rank, compression=compression, **kwargs)
