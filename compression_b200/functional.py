"""Functional CUDA entry points that have no op in the reference because the reference composes them from
TF primitives: GDN/IGDN forward + backward (``python/layers/gdn.py:371-421`` + TF autodiff) and the fused
quantise+encode / decode+dequantise paths of the entropy models."""
import ctypes as C
import math
import os

import numpy as np
import torch

from compression_b200 import _lib, gen_ops
from compression_b200._lib import check

GDN_INVERSE = 1
GDN_RECTIFY = 2


def _stream() -> int:
  return torch.cuda.current_stream().cuda_stream


def _p(t):
  return None if t is None else C.c_void_p(t.data_ptr())


GDN_POW_ALPHA = 4      # trainable alpha: literal u ** alpha (no |u| / u^2 shortcut), gdn.py:380-388
GDN_POW_EPSILON = 8    # trainable epsilon: literal n ** epsilon, gdn.py:406-411


def _flags(inverse, rectify, pow_alpha=False, pow_epsilon=False):
  return ((GDN_INVERSE if inverse else 0) | (GDN_RECTIFY if rectify else 0) | (GDN_POW_ALPHA if pow_alpha else 0) |
          (GDN_POW_EPSILON if pow_epsilon else 0))


_IO16 = {torch.float16: 1, torch.bfloat16: 2}


def _gdn_args(x, gamma, beta):
  assert x.is_cuda and x.dtype in (torch.float32, torch.float16, torch.bfloat16)
  x = x.contiguous()
  C_ = x.shape[-1]
  gamma = gamma.to(device=x.device, dtype=torch.float32).contiguous()
  beta = beta.to(device=x.device, dtype=torch.float32).contiguous()
  assert gamma.shape == (C_, C_) and beta.shape == (C_,)
  return x, gamma, beta, C_, x.numel() // C_


def _gdn_native16(x, C_, n_pix, alpha, epsilon, pow_alpha, pow_epsilon, dy=None):
  """Whether a 16-bit GDN call (forward, or backward with `dy`) runs on the kernels that read and write the 16-bit
  elements themselves: C = 128 or 192 with the fixed exponents' shortcuts, 16-byte aligned tensors, and for the
  backward dy in the activations' type.  Everything else, and everything under TFCB_GDN_FP32=1 (which keeps GDN off
  the tensor cores), converts to float32 and back; both give the same bits."""
  if os.environ.get("TFCB_GDN_FP32", "").startswith("1"):
    return False
  # dy.contiguous() keeps a contiguous dy's pointer and copies any other dy to a fresh (aligned) allocation
  if dy is not None and (dy.dtype != x.dtype or dy.shape != x.shape or dy.data_ptr() % 16 != 0):
    return False
  return (x.dtype in _IO16 and C_ in (128, 192) and not pow_alpha and not pow_epsilon and
          float(alpha) in (1.0, 2.0) and float(epsilon) in (1.0, 0.5) and n_pix > 0 and x.data_ptr() % 16 == 0)


_CF_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _gdn_native_cf(x, alpha, epsilon, pow_alpha, pow_epsilon, dy=None, exponent_grads=False):
  """Whether a channels-first GDN call (x [N, C, *spatial]; the backward with `dy`, and with `exponent_grads` the
  one that also returns dalpha / depsilon) runs on the kernels that read and write that layout in place
  (tfcb_gdn_*_cf).  That is exactly where the channels-last path runs on the tensor cores: float32 at C in
  {128, 192, 256, 320} with any exponents, float16 / bfloat16 at C in {128, 192} with alpha in {1, 2}, epsilon in
  {1, 1/2} and neither exponent trainable.  x has rank >= 3, is contiguous in the default memory format and 16-byte
  aligned; dy has x's type, shape and layout and is 16-byte aligned; the exponent gradients need the float32 literal-pow
  kernels (a trainable exponent, or a fixed one outside the shortcuts).  Never under TFCB_GDN_FP32=1.  Every other
  call takes the channels-last path on x.movedim(1, -1), which gives the same values; in particular a
  torch.channels_last tensor, whose movedim(1, -1) is already contiguous.  The device is not looked at here: every
  channels-first call checks it first (_check_cf_devices), so a host tensor is refused on either path."""
  if os.environ.get("TFCB_GDN_FP32", "").startswith("1"):
    return False
  if x.dim() < 3 or x.dtype not in _CF_DTYPES or not x.is_contiguous() or x.data_ptr() % 16 != 0:
    return False
  if dy is not None and (dy.dtype != x.dtype or dy.shape != x.shape or not dy.is_contiguous() or
                         dy.data_ptr() % 16 != 0):
    return False
  C_ = x.shape[1]
  shortcuts = (not pow_alpha and not pow_epsilon and float(alpha) in (1.0, 2.0) and float(epsilon) in (1.0, 0.5))
  if x.dtype == torch.float32:
    return C_ in (128, 192, 256, 320) and not (exponent_grads and shortcuts)
  return C_ in (128, 192) and shortcuts and not exponent_grads


def _check_cf_devices(x, dy=None):
  """Channels-first calls take CUDA tensors, dy on x's device: anything else is refused before it can reach the
  library (whose kernels would be handed host pointers), on the native and the movedim path alike."""
  if not x.is_cuda:
    raise _lib.InvalidArgumentError(f"GDN takes CUDA tensors, got x on {x.device}")
  if dy is not None and dy.device != x.device:
    raise _lib.InvalidArgumentError(f"GDN: dy is on {dy.device}, x on {x.device}")


def _gdn_cf_args(x, gamma, beta, dy=None):
  _check_cf_devices(x, dy)
  C_ = x.shape[1]
  gamma = gamma.to(device=x.device, dtype=torch.float32).contiguous()
  beta = beta.to(device=x.device, dtype=torch.float32).contiguous()
  assert gamma.shape == (C_, C_) and beta.shape == (C_,)
  if beta.data_ptr() % 16 != 0:  # the kernels read beta in pairs and the library checks its alignment
    beta = beta.clone()
  return gamma, beta, C_, x.shape[0], math.prod(x.shape[2:])


def _gdn_backward_cf(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pow_alpha, pow_epsilon, exponent_grads):
  """One tfcb_gdn_backward_cf call for inputs _gdn_native_cf accepts: (dx, dgamma, dbeta, dalpha_depsilon or None)."""
  gamma, beta, C_, n_items, spatial = _gdn_cf_args(x, gamma, beta, dy)
  dx = torch.empty_like(x)
  dgamma = torch.empty_like(gamma)
  dbeta = torch.empty_like(beta)
  # the library fills the exponent gradients whenever an exponent is trainable
  dae = torch.empty(2, dtype=torch.float32, device=x.device) if exponent_grads or pow_alpha or pow_epsilon else None
  L = _lib.lib()
  dtype = _CF_DTYPES[x.dtype]
  ws = torch.empty(int(L.tfcb_gdn_backward_cf_workspace_bytes(n_items, spatial, C_, dtype)), dtype=torch.uint8,
                   device=x.device)
  check(L.tfcb_gdn_backward_cf(_p(x), _p(gamma), _p(beta), _p(dy), _p(dx), _p(dgamma), _p(dbeta), _p(dae), _p(ws),
                               n_items, spatial, C_, dtype, _flags(inverse, rectify, pow_alpha, pow_epsilon),
                               float(alpha), float(epsilon), _stream()))
  return dx, dgamma, dbeta, dae


def gdn_forward(x, gamma, beta, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, pow_alpha=False,
                pow_epsilon=False, channels_first=False):
  """x: float32 CUDA [..., C] (channels-last, contiguous) -> y of the same shape.  With `channels_first`, x is
  [N, C, *spatial]: inputs _gdn_native_cf accepts give a contiguous y from one library call, any other the
  movedim(-1, 1) view of the channels-last result on x.movedim(1, -1); the values are the same."""
  if channels_first:
    _check_cf_devices(x)
    if not _gdn_native_cf(x, alpha, epsilon, pow_alpha, pow_epsilon):
      return gdn_forward(x.movedim(1, -1), gamma, beta, inverse, rectify, alpha, epsilon, pow_alpha,
                         pow_epsilon).movedim(-1, 1)
    gamma, beta, C_, n_items, spatial = _gdn_cf_args(x, gamma, beta)
    y = torch.empty_like(x)
    check(_lib.lib().tfcb_gdn_forward_cf(_p(x), _p(gamma), _p(beta), _p(y), n_items, spatial, C_,
                                         _CF_DTYPES[x.dtype], _flags(inverse, rectify, pow_alpha, pow_epsilon),
                                         float(alpha), float(epsilon), _stream()))
    return y
  x, gamma, beta, C_, n_pix = _gdn_args(x, gamma, beta)
  if x.dtype in _IO16:
    # mixed precision (gdn_test.py:200-210): 16-bit activations, float32 parameters and arithmetic.  The result is the
    # float32 kernel's on the widened x, rounded once, on either path.
    if _gdn_native16(x, C_, n_pix, alpha, epsilon, pow_alpha, pow_epsilon):
      y = torch.empty_like(x)
      check(_lib.lib().tfcb_gdn_forward_16bit(_p(x), _p(gamma), _p(beta), _p(y), n_pix, C_, _IO16[x.dtype],
                                              _flags(inverse, rectify), float(alpha), float(epsilon), _stream()))
      return y
    return gdn_forward(x.float(), gamma, beta, inverse, rectify, alpha, epsilon, pow_alpha, pow_epsilon).to(x.dtype)
  y = torch.empty_like(x)
  check(_lib.lib().tfcb_gdn_forward(_p(x), _p(gamma), _p(beta), _p(y), n_pix, C_,
                                    _flags(inverse, rectify, pow_alpha, pow_epsilon), float(alpha), float(epsilon),
                                    _stream()))
  return y


def gdn_backward(x, gamma, beta, dy, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, pow_alpha=False,
                 pow_epsilon=False, channels_first=False):
  """Returns (dx, dgamma, dbeta) for upstream gradient dy.  With `channels_first` (x, dy [N, C, *spatial]) dx is
  contiguous when _gdn_native_cf accepts x and dy, else the movedim(-1, 1) view of the channels-last dx."""
  if channels_first:
    _check_cf_devices(x, dy)
    if not _gdn_native_cf(x, alpha, epsilon, pow_alpha, pow_epsilon, dy):
      dx, dgamma, dbeta = gdn_backward(x.movedim(1, -1), gamma, beta, dy.movedim(1, -1), inverse, rectify, alpha,
                                       epsilon, pow_alpha, pow_epsilon)
      return dx.movedim(-1, 1), dgamma, dbeta
    return _gdn_backward_cf(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pow_alpha, pow_epsilon, False)[:3]
  x, gamma, beta, C_, n_pix = _gdn_args(x, gamma, beta)
  if x.dtype in _IO16:
    # dx in the activations' type: the float32 backward's dx of the widened x and dy, rounded once, on either path
    if _gdn_native16(x, C_, n_pix, alpha, epsilon, pow_alpha, pow_epsilon, dy):
      dy = dy.contiguous()
      dx = torch.empty_like(x)
      dgamma = torch.empty_like(gamma)
      dbeta = torch.empty_like(beta)
      L = _lib.lib()
      ws = torch.empty(int(L.tfcb_gdn_backward_16bit_workspace_bytes(n_pix, C_)), dtype=torch.uint8, device=x.device)
      check(L.tfcb_gdn_backward_16bit(_p(x), _p(gamma), _p(beta), _p(dy), _p(dx), _p(dgamma), _p(dbeta), _p(ws), n_pix,
                                      C_, _IO16[x.dtype], _flags(inverse, rectify), float(alpha), float(epsilon),
                                      _stream()))
      return dx, dgamma, dbeta
    dx, dgamma, dbeta = gdn_backward(x.float(), gamma, beta, dy, inverse, rectify, alpha, epsilon, pow_alpha, pow_epsilon)
    return dx.to(x.dtype), dgamma, dbeta
  dy = dy.to(dtype=torch.float32).contiguous()
  dx = torch.empty_like(x)
  dgamma = torch.empty_like(gamma)
  dbeta = torch.empty_like(beta)
  ws_bytes = int(_lib.lib().tfcb_gdn_backward_workspace_bytes(n_pix, C_))
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device=x.device)
  check(_lib.lib().tfcb_gdn_backward(_p(x), _p(gamma), _p(beta), _p(dy), _p(dx), _p(dgamma), _p(dbeta), _p(ws),
                                     n_pix, C_, _flags(inverse, rectify, pow_alpha, pow_epsilon), float(alpha),
                                     float(epsilon), _stream()))
  return dx, dgamma, dbeta


def gdn_exponent_grads(x, gamma, beta, dy, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, pow_alpha=True,
                       pow_epsilon=True):
  """(dL/dalpha, dL/depsilon) as a float32 [2] tensor: the gradients TF autodiff produces through `inputs ** alpha`
  and `norm_pool ** epsilon` when the exponents are trainable GDNParameters (gdn.py:345-367,388,411)."""
  x, gamma, beta, C_, n_pix = _gdn_args(x.float(), gamma, beta)
  dy = dy.to(dtype=torch.float32).contiguous()
  out = torch.empty(2, dtype=torch.float32, device=x.device)
  ws = torch.empty(int(_lib.lib().tfcb_gdn_exponent_grads_workspace_bytes()), dtype=torch.uint8, device=x.device)
  check(_lib.lib().tfcb_gdn_exponent_grads(_p(x), _p(gamma), _p(beta), _p(dy), _p(out), _p(ws), n_pix, C_,
                                           _flags(inverse, rectify, pow_alpha, pow_epsilon), float(alpha),
                                           float(epsilon), _stream()))
  return out


def gdn_backward_exponents(x, gamma, beta, dy, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, pow_alpha=True,
                           pow_epsilon=True, channels_first=False):
  """(dx, dgamma, dbeta, dalpha_depsilon) in one library call: gdn_backward's three gradients and gdn_exponent_grads'
  [2] tensor.  With a trainable exponent at C = 128, 192, 256 or 320 the exponent sums are fused into the tensor-core
  backward.  16-bit activations go through float32 (dx is rounded once to their type).  `channels_first` as for
  gdn_backward."""
  if channels_first:
    _check_cf_devices(x, dy)
    if not _gdn_native_cf(x, alpha, epsilon, pow_alpha, pow_epsilon, dy, exponent_grads=True):
      dx, dgamma, dbeta, dae = gdn_backward_exponents(x.movedim(1, -1), gamma, beta, dy.movedim(1, -1), inverse,
                                                      rectify, alpha, epsilon, pow_alpha, pow_epsilon)
      return dx.movedim(-1, 1), dgamma, dbeta, dae
    return _gdn_backward_cf(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pow_alpha, pow_epsilon, True)
  if x.dtype in _IO16:
    dx, dgamma, dbeta, dae = gdn_backward_exponents(x.float(), gamma, beta, dy, inverse, rectify, alpha, epsilon,
                                                    pow_alpha, pow_epsilon)
    return dx.to(x.dtype), dgamma, dbeta, dae
  x, gamma, beta, C_, n_pix = _gdn_args(x, gamma, beta)
  dy = dy.to(dtype=torch.float32).contiguous()
  dx = torch.empty_like(x)
  dgamma = torch.empty_like(gamma)
  dbeta = torch.empty_like(beta)
  dae = torch.empty(2, dtype=torch.float32, device=x.device)
  L = _lib.lib()
  ws = torch.empty(int(L.tfcb_gdn_backward_exponents_workspace_bytes(n_pix, C_)), dtype=torch.uint8, device=x.device)
  check(L.tfcb_gdn_backward_exponents(_p(x), _p(gamma), _p(beta), _p(dy), _p(dx), _p(dgamma), _p(dbeta), _p(dae),
                                      _p(ws), n_pix, C_, _flags(inverse, rectify, pow_alpha, pow_epsilon),
                                      float(alpha), float(epsilon), _stream()))
  return dx, dgamma, dbeta, dae


class _GDNFunction(torch.autograd.Function):
  """alpha_t / epsilon_t: 0-d tensors when the exponent is trainable (their value is read on the host: the kernels
  take the exponents as scalars), else None and the fixed value travels in `alpha` / `epsilon`."""

  @staticmethod
  def forward(ctx, x, gamma, beta, alpha_t, epsilon_t, inverse, rectify, alpha, epsilon, channels_first):
    pa, pe = alpha_t is not None, epsilon_t is not None
    if pa:
      alpha = float(alpha_t)
    if pe:
      epsilon = float(epsilon_t)
    ctx.save_for_backward(x, gamma, beta)
    ctx.cfg = (inverse, rectify, alpha, epsilon, pa, pe, channels_first)
    return gdn_forward(x, gamma, beta, inverse, rectify, alpha, epsilon, pa, pe, channels_first=channels_first)

  @staticmethod
  def backward(ctx, dy):
    x, gamma, beta = ctx.saved_tensors
    inverse, rectify, alpha, epsilon, pa, pe, cf = ctx.cfg
    dalpha = depsilon = None
    if (pa and ctx.needs_input_grad[3]) or (pe and ctx.needs_input_grad[4]):
      dx, dgamma, dbeta, g2 = gdn_backward_exponents(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe,
                                                     channels_first=cf)
      dalpha = g2[0] if pa else None
      depsilon = g2[1] if pe else None
    else:
      dx, dgamma, dbeta = gdn_backward(x, gamma, beta, dy, inverse, rectify, alpha, epsilon, pa, pe, channels_first=cf)
    return dx, dgamma, dbeta, dalpha, depsilon, None, None, None, None, None


def gdn(x, gamma, beta, inverse=False, rectify=False, alpha=1.0, epsilon=1.0, channels_first=False):
  """Differentiable GDN/IGDN on channels-last float32 / float16 / bfloat16 CUDA tensors (float32 parameters).  `alpha` / `epsilon`: Python numbers (fixed
  exponents: |u|, u^2, sqrt shortcuts and the tensor-core kernels apply) or 0-d tensors (trainable: literal pow, with
  gradients).  `channels_first`: x is [N, C, *spatial] (gdn_forward / gdn_backward describe the layouts returned)."""
  at = alpha if isinstance(alpha, torch.Tensor) else None
  et = epsilon if isinstance(epsilon, torch.Tensor) else None
  return _GDNFunction.apply(x, gamma, beta, at, et, bool(inverse), bool(rectify),
                            1.0 if at is not None else float(alpha), 1.0 if et is not None else float(epsilon),
                            bool(channels_first))


# ------------------------------------------------------------------------------------------------
# Rate term: log p(y) under uniform noise (UniformNoiseAdapter.log_prob, uniform_noise.py:128-151), fused
# ------------------------------------------------------------------------------------------------
DEEP_FACTORIZED_PARAMS = 28  # per channel of num_filters (3, 3); layout in include/tfcb200.h
LOC_SCALE_BASES = {"normal": 0, "logistic": 1, "laplace": 2}


def _contiguous_f32(t):
  assert t.is_cuda and t.dtype == torch.float32, "the fused log-likelihood takes float32 CUDA tensors"
  return t.contiguous()


class _NoisyDeepFactorizedLogProb(torch.autograd.Function):

  @staticmethod
  def forward(ctx, y, packed):
    y, packed = _contiguous_f32(y), _contiguous_f32(packed)
    ctx.save_for_backward(y, packed)
    out = torch.empty_like(y)
    check(_lib.lib().tfcb_noisy_deep_factorized_log_prob(_p(y), _p(packed), _p(out), y.numel(), packed.shape[0],
                                                         _stream()))
    return out

  @staticmethod
  @torch.autograd.function.once_differentiable
  def backward(ctx, dout):
    y, packed = ctx.saved_tensors
    dout = dout.to(torch.float32).contiguous()
    n, C_ = y.numel(), packed.shape[0]
    dy = torch.empty_like(y)
    dpacked = torch.empty_like(packed)
    L = _lib.lib()
    ws = torch.empty(max(int(L.tfcb_noisy_deep_factorized_workspace_bytes(n, C_)), 1), dtype=torch.uint8,
                     device=y.device)
    check(L.tfcb_noisy_deep_factorized_log_prob_backward(_p(y), _p(packed), _p(dout), _p(dy), _p(dpacked), _p(ws), n,
                                                         C_, _stream()))
    return dy, dpacked


def noisy_deep_factorized_log_prob(y, packed):
  """log p(y) of NoisyDeepFactorized with num_filters (3, 3), differentiable in `y` and `packed`.  y: float32 CUDA,
  channel of element i = i mod C (trailing dimensions = the prior's batch shape); packed: float32 [C, 28], the
  transformed parameters (DeepFactorized._packed_parameters)."""
  assert packed.dim() == 2 and packed.shape[1] == DEEP_FACTORIZED_PARAMS
  return _NoisyDeepFactorizedLogProb.apply(y, packed)


class _NoisyLocScaleLogProb(torch.autograd.Function):
  """loc / scale are either y-shaped or 0-d (one value for every element)."""

  @staticmethod
  def forward(ctx, base, y, loc, scale):
    y, loc, scale = _contiguous_f32(y), _contiguous_f32(loc), _contiguous_f32(scale)
    ctx.save_for_backward(y, loc, scale)
    ctx.base = base
    out = torch.empty_like(y)
    check(_lib.lib().tfcb_noisy_loc_scale_log_prob(base, _p(y), _p(loc), int(loc.dim() == 0), _p(scale),
                                                   int(scale.dim() == 0), _p(out), y.numel(), _stream()))
    return out

  @staticmethod
  @torch.autograd.function.once_differentiable
  def backward(ctx, dout):
    y, loc, scale = ctx.saved_tensors
    dout = dout.to(torch.float32).contiguous()
    dy = torch.empty_like(y)
    want_loc, want_scale = ctx.needs_input_grad[2], ctx.needs_input_grad[3]
    dloc = torch.empty_like(y) if want_loc else None
    dscale = torch.empty_like(y) if want_scale else None
    check(_lib.lib().tfcb_noisy_loc_scale_log_prob_backward(
        ctx.base, _p(y), _p(loc), int(loc.dim() == 0), _p(scale), int(scale.dim() == 0), _p(dout), _p(dy), _p(dloc),
        _p(dscale), y.numel(), _stream()))

    def reduce(d, operand):  # a 0-d operand of a larger y: the elementwise terms summed in double
      if d is None or operand.dim() == y.dim():
        return d
      return d.double().sum().to(torch.float32)

    return None, dy, reduce(dloc, loc), reduce(dscale, scale)


def _scalar_or_full(t, shape):
  """A y-shaped operand as the fused kernel takes it: the 0-d value behind a broadcast scalar (every stride 0; its
  gradient reaches the original through the indexing), else the tensor itself."""
  if t.dim() and t.numel() and all(s == 0 for s in t.stride()):
    return t[(0,) * t.dim()]
  assert tuple(t.shape) == tuple(shape)
  return t


def noisy_loc_scale_log_prob(base, y, loc, scale):
  """log p(y) of NoisyNormal / NoisyLogistic / NoisyLaplace (`base` "normal" / "logistic" / "laplace"),
  differentiable in y, loc and scale.  y float32 CUDA; loc / scale y-shaped, or broadcast scalars."""
  return _NoisyLocScaleLogProb.apply(LOC_SCALE_BASES[base], y, _scalar_or_full(loc, y.shape),
                                     _scalar_or_full(scale, y.shape))


# ------------------------------------------------------------------------------------------------
# Fused quantise + encode / decode + dequantise (K3 fused into K4/K5 and K6)
# ------------------------------------------------------------------------------------------------
def _f32(t, device):
  return None if t is None else t.to(device=device, dtype=torch.float32).contiguous()


def _i32(t, device):
  return None if t is None else t.to(device=device, dtype=torch.int32).contiguous()


def encode_channel_f32(handle, y, quant_offset, cdf_offset):
  """symbols = int32(rint(y - quant_offset[c])) - cdf_offset[c] range-coded in channel mode, without
  materialising the int32 tensor (continuous_batched.py:375-382)."""
  handle._require()
  y = _f32(y, y.device)
  n = y.numel() // handle.n_streams
  check(_lib.lib().tfcb_encode_channel_f32(handle._h, _p(y), _p(_f32(quant_offset, y.device)),
                                           _p(_i32(cdf_offset, y.device)), n, _stream()))
  return handle


def encode_index_f32(handle, index, y, loc, cdf_offset):
  """symbols = int32(rint(y - loc)) - cdf_offset[index], index mode (continuous_indexed.py:378-385)."""
  handle._require()
  y = _f32(y, y.device)
  n = y.numel() // handle.n_streams
  check(_lib.lib().tfcb_encode_index_f32(handle._h, _p(_i32(index, y.device)), _p(y), _p(_f32(loc, y.device)),
                                         _p(_i32(cdf_offset, y.device)), n, _stream()))
  return handle


def _host_lookup(lookup):
  lookup = gen_ops._host_i32(lookup)
  if lookup.ndim not in (1, 2):
    raise _lib.InvalidArgumentError(f"`lookup` must be rank 1 or 2: {lookup.shape}")
  return lookup


def _compress(entry, lookup, shape, dev, *args, decoded=None):
  """What compress_f32 and compress_ragged share: calls the library's `entry` with the table, the stream count,
  `args`, the strings' offsets and (if given) the `decoded` buffer, then allocates the strings' bytes (releasing
  the encoder if that fails) and writes the strings into them."""
  n_streams = gen_ops._prod(shape)
  offsets = torch.empty(n_streams + 1, dtype=torch.int64, device=dev)
  h, total = C.c_void_p(), C.c_int64(0)
  stream = _stream()
  tail = () if decoded is None else (_p(decoded),)
  check(entry(lookup.ctypes.data_as(C.c_void_p), lookup.size, 0 if lookup.ndim == 1 else lookup.shape[1], n_streams,
              *args, _p(offsets), stream, C.byref(h), C.byref(total), *tail))
  L = _lib.lib()
  try:
    out = torch.empty(max(int(total.value), 1), dtype=torch.uint8, device=dev)
  except BaseException:
    L.tfcb_encoder_destroy(h)
    raise
  check(L.tfcb_compress_write(h, _p(offsets), _p(out), stream))
  return gen_ops.Strings(out, offsets, shape)


def compress_f32(batch_shape, lookup, y, quant_offset, cdf_offset, index=None):
  """create_range_encoder + encode_channel_f32 (index None) or encode_index_f32 (`quant_offset` is then the loc
  tensor) + entropy_encode_finalize, as two library calls with one host synchronisation.  The strings are
  written into tensors this call allocates, so each result owns its memory."""
  shape = tuple(int(d) for d in batch_shape)
  lookup = _host_lookup(lookup)
  n_streams = gen_ops._prod(shape)
  if n_streams == 0:
    raise _lib.InvalidArgumentError(f"`handle` is empty: handle.shape={shape}")
  y = _f32(y, y.device)
  dev = y.device
  index, qoff, coff = _i32(index, dev), _f32(quant_offset, dev), _i32(cdf_offset, dev)
  return _compress(_lib.lib().tfcb_compress, lookup, shape, dev, _p(index), _p(y), 1, _p(qoff), _p(coff),
                   y.numel() // n_streams)


def _symbol_offsets(lengths):
  import numpy as np
  lengths = np.asarray([int(n) for n in lengths], dtype=np.int64)
  if lengths.size == 0:
    raise _lib.InvalidArgumentError("a ragged batch needs at least one stream")
  return np.ascontiguousarray(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64))


def compress_ragged(lookup, lengths, value, quant_offset=None, cdf_offset=None, index=None, decoded=False):
  """One compress over streams of different lengths: stream i is the next `lengths[i]` elements of the flat
  `value`.  `value` int32 holds symbols; float32 is quantised in the kernel like compress_f32 (`quant_offset` per
  row in channel mode, the loc tensor in index mode; `cdf_offset` required).  Channel mode (index None) restarts
  at row 0 in every stream.  Returns a Strings of shape (len(lengths),) whose string i equals what compress_f32 /
  entropy_encode_* give for stream i alone.

  `decoded=True` (float values only) returns `(strings, decoded_flat)`: the encoder also writes, per symbol, what
  decode_ragged with the same `quant_offset` / `cdf_offset` returns for these strings, bit for bit, so an encoder
  that conditions on its own reconstruction needs no decode."""
  offs = _symbol_offsets(lengths)
  lookup = _host_lookup(lookup)
  k = offs.size - 1
  dev = value.device
  is_f32 = value.dtype != torch.int32
  value = (_f32 if is_f32 else _i32)(value, dev).reshape(-1)
  index = _i32(index, dev)
  if value.numel() != offs[-1] or (index is not None and index.numel() != offs[-1]):
    raise _lib.InvalidArgumentError(f"ragged batch of {int(offs[-1])} symbols, but `value` has {value.numel()}"
                                    + ("" if index is None else f" and `index` {index.numel()}"))
  qoff, coff = _f32(quant_offset, dev), _i32(cdf_offset, dev)  # (kept alive until the call has returned)
  args = (offs.ctypes.data_as(C.c_void_p), _p(index), _p(value), int(is_f32), _p(qoff), _p(coff))
  if not decoded:
    return _compress(_lib.lib().tfcb_compress_ragged, lookup, (k,), dev, *args)
  buf = torch.empty(max(int(offs[-1]), 1), dtype=torch.float32, device=dev)  # (never null, even with no symbols)
  strings = _compress(_lib.lib().tfcb_compress_ragged_decoded, lookup, (k,), dev, *args, decoded=buf)
  return strings, buf[:int(offs[-1])]


def decode_ragged(handle, lengths, index=None, quant_offset=None, cdf_offset=None):
  """Decodes `lengths[i]` more symbols of stream i of a decoder handle into one flat tensor, stream after stream.
  With `cdf_offset` the symbols are dequantised as decode_channel_f32 / decode_index_f32 do (float32), without it
  they are returned as int32.  Channel mode (index None) restarts at row 0 in every stream."""
  offs = _symbol_offsets(lengths)
  if offs.size - 1 != handle.n_streams:
    raise _lib.InvalidArgumentError(f"{offs.size - 1} lengths for {handle.n_streams} strings")
  dev = handle._encoded.bytes_dev.device
  index = _i32(index, dev)
  if index is not None and index.numel() != offs[-1]:
    raise _lib.InvalidArgumentError(f"ragged batch of {int(offs[-1])} symbols, but `index` has {index.numel()}")
  f32 = cdf_offset is not None
  out = torch.empty(int(offs[-1]), dtype=torch.float32 if f32 else torch.int32, device=dev)
  check(_lib.lib().tfcb_decode_ragged(handle._h, offs.ctypes.data_as(C.c_void_p), _p(index), _p(out), int(f32),
                                      _p(_f32(quant_offset, dev)), _p(_i32(cdf_offset, dev)), _stream()))
  return out


# ------------------------------------------------------------------------------------------------
# Substreams (DESIGN §3.14): the library's split of coding units into S streams, and the encoder's gather
# ------------------------------------------------------------------------------------------------
def _phase_table(positions, widths):
  import numpy as np
  pos = np.ascontiguousarray(np.asarray(positions, dtype=np.int64))
  wid = np.ascontiguousarray(np.broadcast_to(np.asarray(widths, dtype=np.int64), pos.shape))
  if pos.ndim != 2 or pos.shape[0] == 0 or pos.shape[1] == 0:
    raise _lib.InvalidArgumentError(f"`positions` must be [units, phases]: shape {pos.shape}")
  return pos, wid


def substream_layout(positions, widths, substreams):
  """The split of units into `substreams` = S streams: `positions` [units, phases] (phase p of unit u has that many
  positions of widths[u, p] symbols; `widths` broadcasts).  Returns (stream_lengths [units S], phase_lengths
  [phases, units S]) as int64 numpy arrays: stream u S + s's symbols in all (for compress_ragged) and in phase p (for
  one decode_ragged per phase)."""
  import numpy as np
  pos, wid = _phase_table(positions, widths)
  U, P = pos.shape
  S = int(substreams)
  offs = np.zeros(U * S + 1, dtype=np.int64)
  phase = np.zeros((P, U * S), dtype=np.int64)
  check(_lib.lib().tfcb_substream_layout(U, P, _host(pos), _host(wid), S, _host(offs), _host(phase)))
  return np.diff(offs), phase


def substream_gather(positions, widths, substreams, y=None, loc=None, index=None):
  """Units held back to back in coding order -> substream order, in one launch: y and loc (float32) and index
  (int32), flat, each rewritten as substream_layout splits `positions` / `widths`.  Returns the new (y, loc, index),
  None where the operand is None."""
  pos, wid = _phase_table(positions, widths)
  U, P = pos.shape
  S = int(substreams)
  lib = _lib.lib()
  given = [t for t in (y, loc, index) if t is not None]
  if not given:
    raise _lib.InvalidArgumentError("substream_gather needs y, loc or index")
  dev = given[0].device
  ins = (_f32(y, dev), _f32(loc, dev), _i32(index, dev))
  outs = tuple(None if t is None else torch.empty_like(t) for t in ins)
  nw = int(lib.tfcb_substream_gather_workspace_bytes(U, P, S))
  work = torch.empty(max(nw // 8, 1), dtype=torch.int64, device=dev)
  check(lib.tfcb_substream_gather(U, P, _host(pos), _host(wid), S, *[_p(t) for t in ins], *[_p(t) for t in outs],
                                  _p(work), work.numel() * 8, _stream()))
  return outs


def context_phases(groups, hs, ws, multistage=False):
  """positions and widths [images, 2K] of the context models' coding order: per group c_k, its anchors, then its
  non-anchors (the checkerboard model is the one group (M,)).  With `multistage`, [images, 4K]: per group its
  stages 0 to 3 of the 2x2 schedule (the multistage model is the one group (M,))."""
  import numpy as np
  hs = np.asarray(hs, dtype=np.int64).reshape(-1)
  ws = np.asarray(ws, dtype=np.int64).reshape(-1)
  if multistage:
    passes = [((hs - a + 1) // 2) * ((ws - b + 1) // 2) for a, b in MSC_PHASES]
  else:
    passes = [(hs * ws + 1) // 2, hs * ws // 2]
  pos = np.stack([n for _ in groups for n in passes], axis=1)
  wid = np.broadcast_to(np.asarray([int(c) for c in groups for _ in passes], dtype=np.int64), pos.shape)
  return pos, wid


# ------------------------------------------------------------------------------------------------
# Universal quantisation: shared noise levels and coding tensors (universal.py:30-62,147-170,446-466)
# ------------------------------------------------------------------------------------------------
def _seed_words(seed):
  return int(seed[0]) & 0xFFFFFFFF, int(seed[1]) & 0xFFFFFFFF


def stateless_uniform_int(n, seed, maxval, device):
  """int32 [n]: element i is word i % 4 of Philox-4x32-10(counter = i // 4, key = seed) modulo `maxval`, drawn on
  the CUDA `device` in one launch (entropy_models.stateless_uniform_int on the CPU gives the same integers)."""
  maxval = int(maxval)
  if maxval < 1:
    raise _lib.InvalidArgumentError(f"`maxval` must be positive: {maxval}")
  out = torch.empty(int(n), dtype=torch.int32, device=device)
  check(_lib.lib().tfcb_stateless_uniform_int(_p(out), out.numel(), *_seed_words(seed), min(maxval, 1 << 62),
                                              _stream()))
  return out


UNIVERSAL_INDEX_DTYPES = (torch.float32, torch.float64)  # index types the coding-tensor kernel reads


def universal_coding_tensors(lengths, num_noise_levels, offset_dtype, device, prior_size=None, indexes=None,
                             index_ranges=None, seed=(1234, 1234)):
  """Flat int32 table indexes and offsets of items of `lengths` elements, one after the other, in one launch; the
  noise position restarts in every item.  Batched (`prior_size`): level * prior_size + i % prior_size.  Indexed
  (`indexes` float32 / float64 [sum(lengths), len(index_ranges)]): the level and the indexes clipped to their ranges
  and flattened with the strides of (num_noise_levels,) + index_ranges.  The offset (level + 1) / (levels + 1) - 1/2
  is computed in double and returned as float32 when `offset_dtype` is float32, else as float64."""
  import numpy as np
  offs = _symbol_offsets(lengths)
  n = int(offs[-1])
  table = torch.empty(n, dtype=torch.int32, device=device)
  off64 = offset_dtype != torch.float32
  offset = torch.empty(n, dtype=torch.float64 if off64 else torch.float32, device=device)
  if indexes is None:
    idx, is_f64, ranges, n_ranges, prior_size = None, 0, None, 0, int(prior_size)
  else:
    if indexes.dtype not in UNIVERSAL_INDEX_DTYPES:
      raise _lib.InvalidArgumentError(f"indexes of type {indexes.dtype}: the kernel reads float32 or float64")
    ranges = np.ascontiguousarray(np.asarray(index_ranges, dtype=np.int64).reshape(-1))
    idx = indexes.to(device).contiguous()
    if idx.numel() != n * ranges.size:
      raise _lib.InvalidArgumentError(f"{n} elements of {ranges.size} indexes each, but `indexes` has {idx.numel()}")
    is_f64, n_ranges, prior_size = int(idx.dtype == torch.float64), ranges.size, 0
  check(_lib.lib().tfcb_universal_coding_tensors(
      offs.size - 1, offs.ctypes.data_as(C.c_void_p), *_seed_words(seed), int(num_noise_levels), prior_size, _p(idx),
      is_f64, None if ranges is None else ranges.ctypes.data_as(C.c_void_p), n_ranges, _p(table), _p(offset),
      int(off64), _stream()))
  return table, offset


def run_length_encode_ragged(values, lengths, run_length_code, magnitude_code, use_run_length_for_non_zeros):
  """RunLengthEncode of many strings in one launch: string i codes the next `lengths[i]` elements of the flat int32
  `values`.  Returns a Strings of shape (len(lengths),) whose string i equals gen_ops.run_length_encode of those
  elements alone (the empty string for a length of 0)."""
  offs = _symbol_offsets(lengths)
  k = offs.size - 1
  dev = gen_ops._device()
  values = _i32(values, dev).reshape(-1)
  if values.numel() != offs[-1]:
    raise _lib.InvalidArgumentError(f"ragged batch of {int(offs[-1])} elements, but `values` has {values.numel()}")
  offsets = torch.empty(k + 1, dtype=torch.int64, device=dev)
  h, total = C.c_void_p(), C.c_int64(0)
  stream = _stream()
  L = _lib.lib()
  check(L.tfcb_run_length_encode_ragged(_p(values), k, offs.ctypes.data_as(C.c_void_p), int(run_length_code),
                                        int(magnitude_code), int(bool(use_run_length_for_non_zeros)), _p(offsets),
                                        stream, C.byref(h), C.byref(total)))
  try:
    out = torch.empty(max(int(total.value), 1), dtype=torch.uint8, device=dev)
  except BaseException:
    L.tfcb_run_length_encoder_destroy(h)
    raise
  check(L.tfcb_run_length_write(h, _p(out), stream))
  return gen_ops.Strings(out, offsets, (k,))


def run_length_decode_ragged(strings, lengths, run_length_code, magnitude_code, use_run_length_for_non_zeros):
  """Inverse of run_length_encode_ragged, one thread per string in one launch: `strings` (a Strings or a list of
  bytes) holds len(lengths) strings; returns int32 [sum(lengths)], string after string.  A damaged string raises
  InvalidArgumentError naming the lowest-numbered failing string and the message gen_ops.run_length_decode gives."""
  offs = _symbol_offsets(lengths)
  k = offs.size - 1
  if not isinstance(strings, gen_ops.Strings):
    strings = gen_ops.Strings.from_bytes(list(strings), (len(strings),))
  if strings.numel() != k:
    raise _lib.InvalidArgumentError(f"{strings.numel()} strings for {k} lengths")
  dev = strings.bytes_dev.device
  out = torch.empty(int(offs[-1]), dtype=torch.int32, device=dev)
  check(_lib.lib().tfcb_run_length_decode_ragged(
      _p(strings.bytes_dev), _p(strings.offsets_dev), k, offs.ctypes.data_as(C.c_void_p), int(run_length_code),
      int(magnitude_code), int(bool(use_run_length_for_non_zeros)), _p(out), _stream()))
  return out


def decode_channel_f32(handle, out_shape, quant_offset, cdf_offset):
  """Decodes and dequantises: float(sym + cdf_offset[c]) + quant_offset[c] (continuous_batched.py:416-421)."""
  dev = handle._encoded.bytes_dev.device
  out = torch.empty(tuple(out_shape), dtype=torch.float32, device=dev)
  n = out.numel() // handle.n_streams
  check(_lib.lib().tfcb_decode_channel_f32(handle._h, _p(out), _p(_f32(quant_offset, dev)),
                                           _p(_i32(cdf_offset, dev)), n, _stream()))
  return out


def decode_index_f32(handle, index, loc, cdf_offset):
  """Decodes and dequantises in index mode (continuous_indexed.py:409-416)."""
  dev = handle._encoded.bytes_dev.device
  index = _i32(index, dev)
  out = torch.empty(tuple(index.shape), dtype=torch.float32, device=dev)
  n = out.numel() // handle.n_streams
  check(_lib.lib().tfcb_decode_index_f32(handle._h, _p(index), _p(out), _p(_f32(loc, dev)),
                                         _p(_i32(cdf_offset, dev)), n, _stream()))
  return out


# ------------------------------------------------------------------------------------------------
# 16-bit bottlenecks: quantised in the encoder, dequantised in the decoder (tfcb_*_16bit), with the arithmetic of
# the entropy models' unfused path (ContinuousEntropyModelBase._quantize / _dequantize)
# ------------------------------------------------------------------------------------------------
_LOC_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _coder16(dtype, device, off=None, index=None, shape=None):
  """Whether range coding of a `dtype` bottleneck on `device` runs on the 16-bit entries below, which give the bytes
  and bits of the unfused path: `dtype` float16 or bfloat16 on a CUDA device; channel mode (`index` None): `off` None
  or float32 with one value per table row (the models' quantisation offsets); index mode: `index` of shape `shape`,
  and `off` None or of that shape in `dtype` or float32.  Every operand is on `device`.  Reads dtypes, shapes and
  devices only.  Everything else (e.g. a float64 loc, or a loc broadcast from another shape) keeps the unfused
  path."""
  device = torch.device(device)
  if dtype not in _IO16 or device.type != "cuda":
    return False
  if any(t is not None and t.device != device for t in (off, index)):
    return False
  if index is None:
    return off is None or (off.dtype == torch.float32 and len(off.shape) == 1)
  shape = tuple(shape)
  return tuple(index.shape) == shape and (off is None or (off.dtype in (dtype, torch.float32) and
                                                          tuple(off.shape) == shape))


def _loc16(loc, dev):
  """A 16-bit call's loc operand as the library takes it: (contiguous flat tensor or None, loc_dtype code)."""
  if loc is None:
    return None, 0
  loc = loc.to(dev).contiguous().reshape(-1)
  return loc, _LOC_DTYPES.get(loc.dtype, -1)


def _out16_dtype(dtype, loc, index):
  """The decoded values' type: the bottleneck's, or float32 in index mode with a float32 loc (torch's promotion of
  the unfused path's `out + loc`)."""
  return torch.float32 if index is not None and loc is not None and loc.dtype == torch.float32 else dtype


def _check16_lengths(n, loc, index, cdf_offset, value=None):
  """A 16-bit call's operands against its `n` symbols, before the library is called: value and index have n
  elements, loc n (index mode) or one per cdf_offset row (channel mode)."""
  if value is not None and value.numel() != n:
    raise _lib.InvalidArgumentError(f"{n} symbols, but `value` has {value.numel()}")
  if index is not None and index.numel() != n:
    raise _lib.InvalidArgumentError(f"{n} symbols, but `index` has {index.numel()}")
  if loc is not None:
    want = n if index is not None else (loc.numel() if cdf_offset is None else cdf_offset.numel())
    if loc.numel() != want:
      raise _lib.InvalidArgumentError(f"`loc` has {loc.numel()} elements, expected {want}")


def compress_16bit(batch_shape, lookup, value, loc, cdf_offset, index=None):
  """compress_f32 for a float16 / bfloat16 `value`, quantised in the encoder as the entropy models' unfused path
  does: channel mode (index None) rint(float32(value) - loc[row]) with `loc` the float32 quantisation offsets (or
  None); index mode rint(value - loc) in torch's promoted type (`loc` None, in value's dtype, or float32).  The
  strings are those of the unfused path, byte for byte."""
  shape = tuple(int(d) for d in batch_shape)
  lookup = _host_lookup(lookup)
  n_streams = gen_ops._prod(shape)
  if n_streams == 0:
    raise _lib.InvalidArgumentError(f"`handle` is empty: handle.shape={shape}")
  dev = value.device
  value = value.contiguous()
  index, coff = _i32(index, dev), _i32(cdf_offset, dev)
  loc, loc_dtype = _loc16(loc, dev)
  _check16_lengths(value.numel(), loc, index, coff)
  return _compress(_lib.lib().tfcb_compress_16bit, lookup, shape, dev, _p(index), _p(value), _IO16.get(value.dtype, 0),
                   _p(loc), loc_dtype, _p(coff), value.numel() // n_streams)


def compress_ragged_16bit(lookup, lengths, value, loc=None, cdf_offset=None, index=None, decoded=False):
  """compress_ragged for a float16 / bfloat16 `value` (quantised as compress_16bit).  `decoded=True` returns
  `(strings, decoded_flat)`: per symbol, exactly what decode_ragged_16bit returns for these strings, written by the
  encoder (in value's dtype, or float32 in index mode with a float32 loc)."""
  offs = _symbol_offsets(lengths)
  lookup = _host_lookup(lookup)
  k, n = offs.size - 1, int(offs[-1])
  dev = value.device
  value = value.contiguous().reshape(-1)
  index, coff = _i32(index, dev), _i32(cdf_offset, dev)
  loc, loc_dtype = _loc16(loc, dev)
  _check16_lengths(n, loc, index, coff, value)
  buf = torch.empty(max(n, 1), dtype=_out16_dtype(value.dtype, loc, index), device=dev) if decoded else None
  strings = _compress(_lib.lib().tfcb_compress_ragged_16bit, lookup, (k,), dev, offs.ctypes.data_as(C.c_void_p),
                      _p(index), _p(value), _IO16.get(value.dtype, 0), _p(loc), loc_dtype, _p(coff), _p(buf))
  return (strings, buf[:n]) if decoded else strings


def decode_16bit(handle, out_shape, dtype, loc, cdf_offset, index=None):
  """Decodes and dequantises float16 / bfloat16 values as the entropy models' unfused path: h = dtype(float(sym +
  cdf_offset[row])), then h + loc computed in float32 and rounded to dtype -- or returned as float32 in index mode
  with a float32 loc.  Shape `out_shape` in channel mode, index's shape in index mode."""
  dev = handle._encoded.bytes_dev.device
  index, coff = _i32(index, dev), _i32(cdf_offset, dev)
  loc, loc_dtype = _loc16(loc, dev)
  shape = tuple(out_shape) if index is None else tuple(index.shape)
  out = torch.empty(shape, dtype=_out16_dtype(dtype, loc, index), device=dev)
  _check16_lengths(out.numel(), loc, index, coff)
  check(_lib.lib().tfcb_decode_16bit(handle._h, _p(index), _p(out), _IO16.get(dtype, 0), _p(loc), loc_dtype, _p(coff),
                                     out.numel() // handle.n_streams, _stream()))
  return out


def decode_ragged_16bit(handle, lengths, dtype, loc=None, cdf_offset=None, index=None):
  """decode_ragged of float16 / bfloat16 values, dequantised as decode_16bit: one flat tensor, stream after
  stream."""
  offs = _symbol_offsets(lengths)
  if offs.size - 1 != handle.n_streams:
    raise _lib.InvalidArgumentError(f"{offs.size - 1} lengths for {handle.n_streams} strings")
  dev = handle._encoded.bytes_dev.device
  index, coff = _i32(index, dev), _i32(cdf_offset, dev)
  loc, loc_dtype = _loc16(loc, dev)
  _check16_lengths(int(offs[-1]), loc, index, coff)
  out = torch.empty(int(offs[-1]), dtype=_out16_dtype(dtype, loc, index), device=dev)
  check(_lib.lib().tfcb_decode_ragged_16bit(handle._h, offs.ctypes.data_as(C.c_void_p), _p(index), _p(out),
                                            _IO16.get(dtype, 0), _p(loc), loc_dtype, _p(coff), _stream()))
  return out


def build_lookup(pmf, pmf_length, precision):
  """The per-row PMF -> CDF loop of _build_tables in one launch (continuous_base.py:282-294):
  pmf float32 [rows, max_len] (CUDA), pmf_length int [rows] -> 1-D int32 lookup [-p, cdf...]*rows."""
  import numpy as np
  pmf = pmf.to(dtype=torch.float32).contiguous()
  assert pmf.is_cuda and pmf.dim() == 2
  lens = np.ascontiguousarray(np.asarray(pmf_length.cpu() if isinstance(pmf_length, torch.Tensor) else pmf_length,
                                         dtype=np.int32).reshape(-1))
  assert lens.shape[0] == pmf.shape[0]
  total = int(lens.astype(np.int64).sum() + 3 * lens.shape[0])
  lookup = torch.empty(total, dtype=torch.int32, device=pmf.device)
  check(_lib.lib().tfcb_build_lookup(_p(pmf), pmf.shape[0], pmf.shape[1], lens.ctypes.data_as(C.c_void_p),
                                     int(precision), _p(lookup), _stream()))
  return lookup


def unbounded_index_range_encode_ragged(data, index, lengths, cdf, cdf_size, offset, precision, overflow_width,
                                        debug_level=1):
  """UnboundedIndexRangeEncode of many strings in one launch, one warp per string: string i codes the next
  `lengths[i]` elements of the flat int32 `data` with the same elements of `index`.  Returns a Strings of shape
  (len(lengths),) whose string i equals gen_ops.unbounded_index_range_encode of those elements alone (the empty
  string for a length of 0).  Errors name the lowest failing string and element."""
  offs = _symbol_offsets(lengths)
  gen_ops._ubi_check(precision, overflow_width, debug_level, (int(offs[-1]),), cdf, cdf_size, offset)
  n_data, n_index = (int(np.prod(gen_ops._shape_of(x))) for x in (data, index))
  if n_data != offs[-1] or n_index != offs[-1]:
    raise _lib.InvalidArgumentError(f"ragged batch of {int(offs[-1])} elements, but `data` has {n_data} and "
                                    f"`index` {n_index}")
  return gen_ops._ubi_encode(data, index, offs, cdf, cdf_size, offset, precision, overflow_width, debug_level)


def unbounded_index_range_decode_ragged(strings, index, lengths, cdf, cdf_size, offset, precision, overflow_width,
                                        debug_level=1):
  """Inverse of unbounded_index_range_encode_ragged: `strings` (a Strings or a list of bytes) holds len(lengths)
  strings; returns int32 [sum(lengths)], string after string.  A width prefix longer than any encoder writes raises
  InvalidArgumentError naming the lowest failing string and element."""
  offs = _symbol_offsets(lengths)
  gen_ops._ubi_check(precision, overflow_width, debug_level, (int(offs[-1]),), cdf, cdf_size, offset)
  if not isinstance(strings, gen_ops.Strings):
    strings = gen_ops.Strings.from_bytes(list(strings), (len(strings),))
  if strings.numel() != offs.size - 1:
    raise _lib.InvalidArgumentError(f"{strings.numel()} strings for {offs.size - 1} lengths")
  n_index = int(np.prod(gen_ops._shape_of(index)))
  if n_index != offs[-1]:
    raise _lib.InvalidArgumentError(f"ragged batch of {int(offs[-1])} elements, but `index` has {n_index}")
  return gen_ops._ubi_decode(strings, index, offs, cdf, cdf_size, offset, precision, overflow_width, debug_level)


# ------------------------------------------------------------------------------------------------
# Mixture priors (DESIGN §3.18): every element coded under its own Normal or Logistic mixture, its row built on the
# device (tfcb_mixture_*).  weight / loc / scale are float32 [elements, K], components innermost.
# ------------------------------------------------------------------------------------------------
MIXTURE_FAMILIES = {"normal": 0, "logistic": 1}


def _mixture_args(weight, loc, scale, family, n=None):
  """(weight, loc, scale, K, family code) as contiguous float32 CUDA tensors [elements, K], checked on the host."""
  if family not in MIXTURE_FAMILIES:
    raise _lib.InvalidArgumentError(f"`family` must be one of {sorted(MIXTURE_FAMILIES)}: {family!r}")
  ts = (weight, loc, scale)
  for name, t in zip(("weight", "loc", "scale"), ts):
    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda:
      raise _lib.InvalidArgumentError(f"`{name}` must be a float32 CUDA tensor")
    if t.dim() < 1 or t.shape != weight.shape:
      raise _lib.InvalidArgumentError(f"weight, loc and scale must share one shape [..., K]: {tuple(t.shape)}")
  K = int(weight.shape[-1])
  m = weight.numel() // K if K else 0
  if n is not None and m != n:
    raise _lib.InvalidArgumentError(f"{n} elements, but the parameters hold {m} mixtures")
  return (*(t.reshape(-1, K).contiguous() for t in ts), K, MIXTURE_FAMILIES[family])


def mixture_tables(weight, loc, scale, family="normal", precision=16, tail_mass=2**-8, max_support=256):
  """The rows the mixture coder builds, for tests and for the reference coder: (start int32 [n], size int32 [n], mass
  int64 [n, max_support + 1], rows int32 [n, max_support + 3]).  Row e is [-precision, c_0, .., c_{L+1}] padded with
  2^precision; mass[e] holds m_0 .. m_{L-1}, the escape mass m_L, then zeros."""
  w, l, s, K, fam = _mixture_args(weight, loc, scale, family)
  n = w.shape[0]
  dev = w.device
  start = torch.empty(n, dtype=torch.int32, device=dev)
  size = torch.empty(n, dtype=torch.int32, device=dev)
  mass = torch.empty((n, int(max_support) + 1), dtype=torch.int64, device=dev)
  rows = torch.empty((n, int(max_support) + 3), dtype=torch.int32, device=dev)
  check(_lib.lib().tfcb_mixture_tables(_p(w), _p(l), _p(s), n, K, fam, int(precision), float(tail_mass),
                                       int(max_support), _p(start), _p(size), _p(mass), _p(rows), _stream()))
  return start, size, mass, rows


def mixture_encode_ragged(y, weight, loc, scale, lengths, family="normal", precision=16, tail_mass=2**-8,
                          max_support=256):
  """String i codes the next `lengths[i]` elements of the flat float32 `y` (CUDA), each quantised to int32(rint(y))
  and coded under its own mixture.  Returns a Strings of shape (len(lengths),); one host synchronisation."""
  offs = _symbol_offsets(lengths)
  n = int(offs[-1])
  if not isinstance(y, torch.Tensor) or y.dtype != torch.float32 or not y.is_cuda:
    raise _lib.InvalidArgumentError("`y` must be a float32 CUDA tensor")
  if y.numel() != n:
    raise _lib.InvalidArgumentError(f"ragged batch of {n} elements, but `y` has {y.numel()}")
  w, l, s, K, fam = _mixture_args(weight, loc, scale, family, n)
  y = y.reshape(-1).contiguous()
  k = offs.size - 1
  offsets = torch.empty(k + 1, dtype=torch.int64, device=y.device)
  h, total = C.c_void_p(), C.c_int64(0)
  L = _lib.lib()
  check(L.tfcb_mixture_encode_ragged(_p(y), _p(w), _p(l), _p(s), K, fam, int(precision), float(tail_mass),
                                     int(max_support), k, offs.ctypes.data_as(C.c_void_p), _p(offsets), _stream(),
                                     C.byref(h), C.byref(total)))
  try:
    out = torch.empty(max(int(total.value), 1), dtype=torch.uint8, device=y.device)
  except BaseException:
    L.tfcb_mixture_encoder_destroy(h)
    raise
  check(L.tfcb_mixture_write(h, _p(out), _stream()))
  return gen_ops.Strings(out, offsets, (k,))


def mixture_decode_ragged(strings, weight, loc, scale, lengths, family="normal", precision=16, tail_mass=2**-8,
                          max_support=256):
  """Inverse of mixture_encode_ragged: float32 [sum(lengths)] on the parameters' device, string after string."""
  offs = _symbol_offsets(lengths)
  n = int(offs[-1])
  w, l, s, K, fam = _mixture_args(weight, loc, scale, family, n)
  if not isinstance(strings, gen_ops.Strings):
    strings = gen_ops.Strings.from_bytes(list(strings), (len(strings),))
  if strings.numel() != offs.size - 1:
    raise _lib.InvalidArgumentError(f"{strings.numel()} strings for {offs.size - 1} lengths")
  out = torch.empty(n, dtype=torch.float32, device=w.device)
  check(_lib.lib().tfcb_mixture_decode_ragged(_p(strings.bytes_dev), _p(strings.offsets_dev), offs.size - 1,
                                              offs.ctypes.data_as(C.c_void_p), _p(w), _p(l), _p(s), K, fam,
                                              int(precision), float(tail_mass), int(max_support), _p(out), _stream()))
  return out


# ------------------------------------------------------------------------------------------------
# Joint autoregressive + hierarchical prior (Minnen 2018): the packed parameter network and the parameter, encoder and
# decoder steps over latent positions in raster order (tfcb_ar_*).  Latents are float32 CUDA [B, H, W, M], the hyper
# feature psi [B, H, W, 2M].
# ------------------------------------------------------------------------------------------------
def ar_packed_floats(M):
  """Floats of the packed parameter buffer for latent depth M (a multiple of 6 in [6, 384])."""
  n = int(_lib.lib().tfcb_ar_packed_floats(int(M)))
  if n < 0:
    raise _lib.InvalidArgumentError(f"latent depth M={M} must be a positive multiple of 6 and at most 384")
  return n


def ar_pack_weights(ctx_kernel, ctx_bias, w1, b1, w2, b2, w3, b3):
  """The device layout the parameter kernel reads: the context kernel [5, 5, M, 2M] (masked or not: only its 12
  causal taps are read), then each 1x1 layer as [inputs, outputs] and its bias.  Returns float32 [packed floats] on
  the context kernel's device; the values are copied unchanged."""
  return _pack_weights(ctx_kernel.detach(), None, ctx_bias, w1, b1, w2, b2, w3, b3)


def _pack_weights(ctx_kernel, taps, ctx_bias, w1, b1, w2, b2, w3, b3):
  """tfcb_ar_pack_weights of a [5, 5, M, 2M] context kernel, whose first 12 * M * 2M floats the library reads:
  unchanged (`taps` None) or its taps [(dy + 2, dx + 2), ...] gathered into a contiguous [12, M, 2M]."""
  if ctx_kernel.dim() != 4 or ctx_kernel.shape[:2] != (5, 5) or ctx_kernel.shape[3] != 2 * ctx_kernel.shape[2]:
    raise _lib.InvalidArgumentError(f"context kernel must be [5, 5, M, 2M]: {tuple(ctx_kernel.shape)}")
  M = int(ctx_kernel.shape[2])
  n = ar_packed_floats(M)
  n3, n4 = 10 * M // 3, 8 * M // 3
  dev = ctx_kernel.device
  if dev.type != "cuda":
    raise _lib.InvalidArgumentError(f"the parameters must be on a CUDA device, not {dev}")
  want = ((ctx_bias, (2 * M,)), (w1, (4 * M, n3)), (b1, (n3,)), (w2, (n3, n4)), (b2, (n4,)), (w3, (n4, 2 * M)),
          (b3, (2 * M,)))
  if taps is not None:
    ctx_kernel = ctx_kernel[[y for y, _ in taps], [x for _, x in taps]]
  ops = [_f32(ctx_kernel, dev)]
  for t, shape in want:
    t = t.detach()
    if tuple(t.shape) != shape:
      raise _lib.InvalidArgumentError(f"parameter of shape {tuple(t.shape)} where M={M} needs {shape}")
    ops.append(_f32(t, dev))
  packed = torch.empty(n, dtype=torch.float32, device=dev)
  check(_lib.lib().tfcb_ar_pack_weights(M, *[_p(t) for t in ops], _p(packed), n, _stream()))
  return packed


def _ar_tensor(t, name, shape, dev, dtype=torch.float32):
  if not isinstance(t, torch.Tensor) or t.device != dev or t.dtype != dtype:
    raise _lib.InvalidArgumentError(f"`{name}` must be a {dtype} tensor on {dev}")
  if tuple(t.shape) != tuple(shape):
    raise _lib.InvalidArgumentError(f"`{name}` has shape {tuple(t.shape)}, expected {tuple(shape)}")
  return t.contiguous()


def _ar_dims(packed, psi):
  """(B, H, W, M, packed floats) from psi [B, H, W, 2M], checked against the packed buffer."""
  if not isinstance(psi, torch.Tensor) or psi.dim() != 4 or psi.shape[-1] % 2:
    raise _lib.InvalidArgumentError("`psi` must be [B, H, W, 2M]")
  B, H, W, M = int(psi.shape[0]), int(psi.shape[1]), int(psi.shape[2]), int(psi.shape[3]) // 2
  if B == 0 or H == 0 or W == 0:
    raise _lib.InvalidArgumentError(f"empty latents: psi has shape {tuple(psi.shape)}")
  if not isinstance(packed, torch.Tensor) or packed.dim() != 1 or packed.dtype != torch.float32:
    raise _lib.InvalidArgumentError("`packed` must be a float32 vector from ar_pack_weights")
  n = ar_packed_floats(M)
  if packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, M={M} needs {n}")
  if packed.device.type != "cuda" or psi.device != packed.device:
    raise _lib.InvalidArgumentError(f"`packed` ({packed.device}) and `psi` ({psi.device}) must share a CUDA device")
  return B, H, W, M, n


def ar_params(packed, y_hat, psi, p, num_scales):
  """The parameter step at position p (0 <= p < H * W) of every image: (loc, scale_index, index) [B, M], float32,
  float32 and int32, from y_hat [B, H, W, M] at earlier positions.  Row b depends only on image b."""
  B, H, W, M, n = _ar_dims(packed, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  if not 0 <= int(p) < H * W:
    raise _lib.InvalidArgumentError(f"position {p} outside [0, {H * W})")
  loc = torch.empty((B, M), dtype=torch.float32, device=dev)
  scale = torch.empty_like(loc)
  index = torch.empty((B, M), dtype=torch.int32, device=dev)
  check(_lib.lib().tfcb_ar_params(_p(packed), n, M, _p(y_hat), _p(psi), B, H, W, int(p), int(num_scales), _p(loc),
                                  _p(scale), _p(index), _stream()))
  return loc, scale, index


def _ar_range(p_begin, p_end, H, W):
  p_end = H * W if p_end is None else int(p_end)
  if not 0 <= int(p_begin) <= p_end <= H * W:
    raise _lib.InvalidArgumentError(f"positions [{p_begin}, {p_end}) outside [0, {H * W})")
  return int(p_begin), p_end


def ar_encode(packed, y, psi, num_scales, y_hat=None, p_begin=0, p_end=None, scale_index=False):
  """Encoder steps p_begin <= p < p_end (default: all) in one launch: returns (y_hat, loc, index) [B, H, W, M], and
  scale_index last with `scale_index=True`.  y_hat = float(int32(rint(y - loc))) + loc; a given `y_hat` holds the
  earlier positions and is written in place.  The strings are one index-mode encode of y with `index` and `loc`."""
  B, H, W, M, n = _ar_dims(packed, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  y = _ar_tensor(y, "y", (B, H, W, M), dev)
  p_begin, p_end = _ar_range(p_begin, p_end, H, W)
  if y_hat is None:
    y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  elif not (isinstance(y_hat, torch.Tensor) and y_hat.is_contiguous()):
    raise _lib.InvalidArgumentError("`y_hat` must be a contiguous tensor (it is written in place)")
  y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  loc = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  index = torch.zeros((B, H, W, M), dtype=torch.int32, device=dev)
  scale = torch.zeros_like(loc) if scale_index else None
  check(_lib.lib().tfcb_ar_encode(_p(packed), n, M, _p(y), _p(psi), B, H, W, p_begin, p_end, int(num_scales),
                                  _p(y_hat), _p(loc), _p(index), _p(scale), _stream()))
  return (y_hat, loc, index) + ((scale,) if scale_index else ())


def ar_decode(handle, packed, psi, num_scales, cdf_offset, y_hat=None, p_begin=0, p_end=None):
  """Decoder steps p_begin <= p < p_end (default: all) in one launch, continuing `handle` (a DecoderHandle of B
  index-mode strings): returns y_hat [B, H, W, M], written in place into a given `y_hat` that holds the earlier
  positions.  Stream errors surface at entropy_decode_finalize, as for the other decode calls."""
  B, H, W, M, n = _ar_dims(packed, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  if handle.n_streams != B:
    raise _lib.InvalidArgumentError(f"the decoder holds {handle.n_streams} strings for a batch of {B}")
  p_begin, p_end = _ar_range(p_begin, p_end, H, W)
  if y_hat is None:
    y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  elif not (isinstance(y_hat, torch.Tensor) and y_hat.is_contiguous()):
    raise _lib.InvalidArgumentError("`y_hat` must be a contiguous tensor (it is written in place)")
  y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  coff = _i32(cdf_offset, dev)
  check(_lib.lib().tfcb_ar_decode(handle._h, _p(packed), n, M, _p(psi), B, H, W, p_begin, p_end, int(num_scales),
                                  _p(coff), _p(y_hat), _stream()))
  return y_hat


def ar_decode_naive(handle, packed, psi, num_scales, cdf_offset):
  """The decoder as a host loop, for comparison: per position one tfcb_ar_params launch and one
  tfcb_decode_index_f32 of M symbols per stream, written into y_hat by torch.  Gives ar_decode's y_hat bit for bit;
  2 H W library launches and H W torch copies."""
  B, H, W, M, _ = _ar_dims(packed, psi)
  dev = packed.device
  y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  flat = y_hat.view(B, H * W, M)
  coff = _i32(cdf_offset, dev)
  for p in range(H * W):
    loc, _, index = ar_params(packed, y_hat, psi, p, num_scales)
    flat[:, p] = decode_index_f32(handle, index, loc, coff)
  return y_hat


# ------------------------------------------------------------------------------------------------
# Checkerboard context model (He et al. 2021): two parameter passes over the positions of one colour (tfcb_cb_*) on
# the packed network of ar_pack_weights.  Anchors are the positions (r, c) with r + c even; coding order is the
# anchors in raster order, then the non-anchors in raster order.  Latents are float32 CUDA [B, H, W, M], psi
# [B, H, W, 2M]; coding-order tensors are [B, n, M] for one colour and [B, H * W, M] for both.
# ------------------------------------------------------------------------------------------------
CB_TAPS = tuple((dy, dx) for dy in range(-2, 3) for dx in range(-2, 3) if (dy + dx) % 2)  # raster order, 12 taps


def cb_pack_weights(ctx_kernel, ctx_bias, w1, b1, w2, b2, w3, b3):
  """ar_pack_weights for the checkerboard parameter passes: the 12 checkerboard taps of the context kernel
  [5, 5, M, 2M] (masked or not: no other tap is read) are packed in raster order where ar_pack_weights puts the
  causal ones."""
  return _pack_weights(ctx_kernel.detach(), [(dy + 2, dx + 2) for dy, dx in CB_TAPS], ctx_bias, w1, b1, w2, b2, w3,
                       b3)


def cb_counts(H, W):
  """(anchors, non-anchors) of an H x W latent: (ceil(H W / 2), floor(H W / 2))."""
  return (H * W + 1) // 2, H * W // 2


def _cb_pass(packed, y_hat, psi, anchors, num_scales, whole, loc, scale, index, y=None, y_cb=None, y_hat_out=None):
  B, H, W, M, n = _ar_dims(packed, psi)
  dev = packed.device
  lib = _lib.lib()
  nw = int(lib.tfcb_cb_workspace_floats(M, B, H, W, int(bool(anchors))))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=dev)
  check(lib.tfcb_cb_params(_p(packed), n, M, _p(y_hat), _p(psi), B, H, W, int(bool(anchors)), int(num_scales),
                           _p(work), nw, int(whole), _p(loc), _p(scale), _p(index), _p(y), _p(y_cb), _p(y_hat_out),
                           _stream()))


def cb_params(packed, y_hat, psi, anchors, num_scales):
  """One parameter pass: (loc, scale_index, index) [B, n, M] (float32, float32, int32) of the n positions of one
  colour of every image, in coding order.  The non-anchor pass reads the anchors of y_hat [B, H, W, M]; the anchor
  pass reads no latent (y_hat may be None).  Row b depends only on image b."""
  B, H, W, M, _ = _ar_dims(packed, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  if y_hat is not None or not anchors:
    y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  n = cb_counts(H, W)[0 if anchors else 1]
  loc = torch.empty((B, n, M), dtype=torch.float32, device=dev)
  scale = torch.empty_like(loc)
  index = torch.empty((B, n, M), dtype=torch.int32, device=dev)
  _cb_pass(packed, y_hat, psi, anchors, num_scales, False, loc, scale, index)
  return loc, scale, index


def cb_encode(packed, y, psi, num_scales, scale_index=False, substreams=1):
  """The two-pass encoder: returns y_hat [B, H, W, M] and y, loc, index in coding order [B, H * W, M] (and
  scale_index last with `scale_index=True`).  y_hat = float(int32(rint(y - loc))) + loc, the anchors' before the
  non-anchor pass reads them.  The strings are one index-mode encode of the coding-order y with index and loc.  With
  `substreams` = S > 1 the coding-order tensors are rewritten into substream order by one gather (a second one for
  scale_index), ready for compress_ragged with the stream lengths of context_substreams."""
  B, H, W, M, _ = _ar_dims(packed, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  y = _ar_tensor(y, "y", (B, H, W, M), dev)
  y_hat = torch.empty((B, H, W, M), dtype=torch.float32, device=dev)
  y_cb, loc = (torch.empty((B, H * W, M), dtype=torch.float32, device=dev) for _ in range(2))
  index = torch.empty((B, H * W, M), dtype=torch.int32, device=dev)
  scale = torch.empty_like(loc) if scale_index else None
  for anchors in (True, False):
    _cb_pass(packed, y_hat, psi, anchors, num_scales, True, loc, scale, index, y, y_cb, y_hat)
  return (y_hat,) + _to_substreams((M,), [H] * B, [W] * B, substreams, y_cb, loc, index, scale)


def cb_decode(handle, packed, psi, num_scales, cdf_offset, substreams=1):
  """The two-pass decoder, continuing `handle` (a DecoderHandle of B index-mode strings in coding order): anchor
  parameters, decode_index_f32 of the anchors, their latents to [B, H, W, M], non-anchor parameters, decode of the
  non-anchors, to [B, H, W, M].  Returns y_hat [B, H, W, M].  A fixed number of library launches whatever B, H and W
  (fewer at H W = 1, where the non-anchor pass is empty) and no host synchronisation; stream errors surface at
  entropy_decode_finalize.  With `substreams` = S > 1 the handle holds B S substreams (gen_ops.split_substreams) and
  each pass decodes with one decode_ragged in place of decode_index_f32: the same launches."""
  B, H, W, M, _ = _ar_dims(packed, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  phases = _substream_phases(handle, (M,), [H] * B, [W] * B, substreams)
  coff = _i32(cdf_offset, dev)
  y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  lib = _lib.lib()
  for p, anchors in enumerate((True, False)):
    loc, _, index = cb_params(packed, y_hat, psi, anchors, num_scales)
    part = _decode_phase(handle, phases, p, index, loc, coff)
    check(lib.tfcb_cb_scatter(_p(part), B, H, W, M, int(anchors), _p(y_hat), _stream()))
  return y_hat


def context_substreams(groups, hs, ws, substreams, multistage=False):
  """(stream_lengths, phase_lengths) of substream_layout for the context models' coding order of images of latent
  shapes hs[i] x ws[i] with channel groups `groups` (`multistage` as in context_phases)."""
  return substream_layout(*context_phases(groups, hs, ws, multistage), substreams)


def _to_substreams(groups, hs, ws, substreams, y, loc, index, scale=None, multistage=False):
  """An encoder's coding-order outputs, rewritten into substream order when `substreams` > 1 (shapes kept)."""
  out = (y, loc, index) + (() if scale is None else (scale,))
  if substreams == 1:
    return out
  pos, wid = context_phases(groups, hs, ws, multistage)
  moved = substream_gather(pos, wid, substreams, y.reshape(-1), loc.reshape(-1), index.reshape(-1))
  if scale is not None:
    moved += (substream_gather(pos, wid, substreams, loc=scale.reshape(-1))[1],)
  return tuple(m.view(t.shape) for m, t in zip(moved, out))


def _substream_phases(handle, groups, hs, ws, substreams, what="batch", multistage=False):
  """A context decoder's per-pass decode lengths (None for S = 1), after checking the handle's stream count."""
  units = len(hs)
  if handle.n_streams != units * substreams:
    raise _lib.InvalidArgumentError(f"the decoder holds {handle.n_streams} strings for a {what} of {units}" +
                                    ("" if substreams == 1 else f" in {substreams} substreams"))
  return None if substreams == 1 else context_substreams(groups, hs, ws, substreams, multistage)[1]


def _decode_phase(handle, phases, p, index, loc, coff):
  """Pass p's symbols of every image in coding order: one decode_index_f32, or with substreams one decode_ragged."""
  if phases is None:
    return decode_index_f32(handle, index, loc, coff)
  return decode_ragged(handle, phases[p], index=index, quant_offset=loc, cdf_offset=coff)


# ------------------------------------------------------------------------------------------------
# Space-channel context model (He et al. 2022): the checkerboard passes per channel group (tfcb_scc_*).  The groups
# (c_0, ..., c_{K-1}) split y's M channels; group k is the span (o_k, c_k), channels [o_k, o_k + c_k).  Each group
# has its own packed network (scc_pack_weights), whose layer 1 reads [psi, the channel context of group k (none for
# k = 0), its spatial context].  Coding order: per image, group 0's anchors, group 0's non-anchors, group 1's
# anchors, ..., each in raster order with c_k channels per position; the coding-order tensors are [B, H * W * M].
# ------------------------------------------------------------------------------------------------
def scc_spans(groups):
  """[(offset, channels), ...] of the channel counts `groups`."""
  spans, o = [], 0
  for c in groups:
    spans.append((o, int(c)))
    o += int(c)
  return spans


def scc_layout(M, group):
  """The library's packed layout of group (offset, channels) of a depth-M latent: a dict of the widths K1, N3, N4,
  the offsets of wc, bc, w1, b1, w2, b2, w3, b3 and the `total` floats."""
  o, c = (int(v) for v in group)
  out = (C.c_int64 * 11)()
  n = int(_lib.lib().tfcb_scc_packed_floats(int(M), o, c, out))
  if n < 0:
    raise _lib.InvalidArgumentError(f"group of {c} channels at offset {o} of a latent of depth M={M}: M must be a "
                                    "positive even number at most 1024, with every channel inside it")
  keys = ("K1", "N3", "N4", "wc", "bc", "w1", "b1", "w2", "b2", "w3", "b3")
  return dict(zip(keys, (int(v) for v in out)), total=n)


def scc_pack_weights(M, group, ctx_kernel, ctx_bias, w1, b1, w2, b2, w3, b3):
  """The device layout of group (offset, channels)'s parameter passes: the 12 checkerboard taps of its context
  kernel [5, 5, c, 2c] (masked or not: no other tap is read), then each 1x1 layer as [inputs, outputs] and its bias,
  with the widths scc_layout gives.  Returns float32 [total] on the context kernel's device."""
  o, c = (int(v) for v in group)
  lay = scc_layout(M, group)
  ctx_kernel = ctx_kernel.detach()
  if tuple(ctx_kernel.shape) != (5, 5, c, 2 * c):
    raise _lib.InvalidArgumentError(f"context kernel must be [5, 5, {c}, {2 * c}]: {tuple(ctx_kernel.shape)}")
  dev = ctx_kernel.device
  if dev.type != "cuda":
    raise _lib.InvalidArgumentError(f"the parameters must be on a CUDA device, not {dev}")
  k1, n3, n4 = lay["K1"], lay["N3"], lay["N4"]
  want = ((ctx_bias, (2 * c,)), (w1, (k1, n3)), (b1, (n3,)), (w2, (n3, n4)), (b2, (n4,)), (w3, (n4, 2 * c)),
          (b3, (2 * c,)))
  ops = [_f32(ctx_kernel[[dy + 2 for dy, _ in CB_TAPS], [dx + 2 for _, dx in CB_TAPS]], dev)]
  for t, shape in want:
    t = t.detach()
    if tuple(t.shape) != shape:
      raise _lib.InvalidArgumentError(f"parameter of shape {tuple(t.shape)} where group ({o}, {c}) of M={M} needs "
                                      f"{shape}")
    ops.append(_f32(t, dev))
  packed = torch.empty(lay["total"], dtype=torch.float32, device=dev)
  check(_lib.lib().tfcb_scc_pack_weights(int(M), o, c, *[_p(t) for t in ops], _p(packed), lay["total"], _stream()))
  return packed


def _scc_dims(packed, group, psi, layout=scc_layout):
  """(B, H, W, M, offset, channels, packed floats) from psi [B, H, W, 2M], checked against the group's packed
  buffer (of scc_layout, or mscc_layout for the space-channel multistage model)."""
  if not isinstance(psi, torch.Tensor) or psi.dim() != 4 or psi.shape[-1] % 2:
    raise _lib.InvalidArgumentError("`psi` must be [B, H, W, 2M]")
  B, H, W, M = int(psi.shape[0]), int(psi.shape[1]), int(psi.shape[2]), int(psi.shape[3]) // 2
  if B == 0 or H == 0 or W == 0:
    raise _lib.InvalidArgumentError(f"empty latents: psi has shape {tuple(psi.shape)}")
  o, c = (int(v) for v in group)
  n = layout(M, group)["total"]
  if not isinstance(packed, torch.Tensor) or packed.dim() != 1 or packed.dtype != torch.float32:
    raise _lib.InvalidArgumentError(f"`packed` must be a float32 vector from {_PACKERS[layout]}")
  if packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, group ({o}, {c}) of M={M} needs {n}")
  if packed.device.type != "cuda" or psi.device != packed.device:
    raise _lib.InvalidArgumentError(f"`packed` ({packed.device}) and `psi` ({psi.device}) must share a CUDA device")
  return B, H, W, M, o, c, n


def _scc_pass(packed, group, y_hat, psi, ch_ctx, anchors, num_scales, whole, loc, scale, index, y=None, y_cc=None,
              y_hat_out=None):
  B, H, W, M, o, c, n = _scc_dims(packed, group, psi)
  lib = _lib.lib()
  nw = int(lib.tfcb_scc_workspace_floats(M, o, c, B, H, W, int(bool(anchors))))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=packed.device)
  check(lib.tfcb_scc_params(_p(packed), n, M, o, c, _p(y_hat), _p(psi), _p(ch_ctx), B, H, W, int(bool(anchors)),
                            int(num_scales), _p(work), nw, int(whole), _p(loc), _p(scale), _p(index), _p(y), _p(y_cc),
                            _p(y_hat_out), _stream()))


def _scc_ch_ctx(ch_ctx, group, shape, dev):
  """The channel context [B, H, W, 2c] of a group at a positive offset; None at offset 0."""
  o, c = (int(v) for v in group)
  if o == 0:
    if ch_ctx is not None:
      raise _lib.InvalidArgumentError("the group at offset 0 has no channel context: pass None")
    return None
  return _ar_tensor(ch_ctx, "ch_ctx", tuple(shape) + (2 * c,), dev)


def scc_params(packed, group, y_hat, psi, ch_ctx, anchors, num_scales):
  """One parameter pass of group (offset, channels): (loc, scale_index, index) [B, n, c] (float32, float32, int32)
  of the n positions of one colour of every image, in coding order.  ch_ctx [B, H, W, 2c] is the group's channel
  context (None at offset 0); the non-anchor pass reads the group's channels of the anchors of y_hat [B, H, W, M]
  (y_hat may be None for the anchor pass).  Row b depends only on image b."""
  B, H, W, M, o, c, _ = _scc_dims(packed, group, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  ch_ctx = _scc_ch_ctx(ch_ctx, group, (B, H, W), dev)
  if y_hat is not None or not anchors:
    y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  n = cb_counts(H, W)[0 if anchors else 1]
  loc = torch.empty((B, n, c), dtype=torch.float32, device=dev)
  scale = torch.empty_like(loc)
  index = torch.empty((B, n, c), dtype=torch.int32, device=dev)
  _scc_pass(packed, group, y_hat, psi, ch_ctx, anchors, num_scales, False, loc, scale, index)
  return loc, scale, index


def _scc_batch(packed, groups, psi, layout=scc_layout):
  """(B, H, W, M, spans, psi) of a whole-latent call, with every group's packed buffer checked."""
  if not isinstance(psi, torch.Tensor) or psi.dim() != 4 or psi.shape[-1] % 2:
    raise _lib.InvalidArgumentError("`psi` must be [B, H, W, 2M]")
  M = int(psi.shape[3]) // 2
  spans = scc_spans(groups)
  if sum(c for _, c in spans) != M or len(packed) != len(spans):
    raise _lib.InvalidArgumentError(f"{len(packed)} packed networks and groups {tuple(groups)} for a latent of depth "
                                    f"{M}: one network per group, and the groups must sum to M")
  for p, g in zip(packed, spans):
    B, H, W = _scc_dims(p, g, psi, layout)[:3]
  return B, H, W, M, spans, _ar_tensor(psi, "psi", (B, H, W, 2 * M), psi.device)


def scc_encode(packed, groups, y, psi, channel_context, num_scales, scale_index=False, substreams=1):
  """The group-by-group encoder: `packed` holds one scc_pack_weights buffer per group.  Per group k, its channel
  context `channel_context(k, y_hat)` [B, H, W, 2c_k] (called for k >= 1, once y_hat holds groups 0 to k - 1), the
  anchor pass, then the non-anchor pass.  Returns y_hat [B, H, W, M] and y, loc, index in coding order
  [B, H * W * M] (and scale_index last with `scale_index=True`).  y_hat = float(int32(rint(y - loc))) + loc.  The
  strings are one index-mode encode of the coding-order y with index and loc.  `substreams` as in cb_encode."""
  B, H, W, M, spans, psi = _scc_batch(packed, groups, psi)
  dev = psi.device
  y = _ar_tensor(y, "y", (B, H, W, M), dev)
  y_hat = torch.empty((B, H, W, M), dtype=torch.float32, device=dev)
  y_cc, loc = (torch.empty((B, H * W * M), dtype=torch.float32, device=dev) for _ in range(2))
  index = torch.empty((B, H * W * M), dtype=torch.int32, device=dev)
  scale = torch.empty_like(loc) if scale_index else None
  for k, (p, g) in enumerate(zip(packed, spans)):
    ch = _scc_ch_ctx(channel_context(k, y_hat) if k else None, g, (B, H, W), dev)
    for anchors in (True, False):
      _scc_pass(p, g, y_hat, psi, ch, anchors, num_scales, True, loc, scale, index, y, y_cc, y_hat)
  return (y_hat,) + _to_substreams(groups, [H] * B, [W] * B, substreams, y_cc, loc, index, scale)


def scc_decode(handle, packed, groups, psi, channel_context, num_scales, cdf_offset, substreams=1):
  """The group-by-group decoder, continuing `handle` (a DecoderHandle of B index-mode strings in coding order): per
  group its channel context (as in scc_encode), then per colour the parameter pass, decode_index_f32 and the scatter
  into y_hat [B, H, W, M], which it returns.  2K decode calls on the handle; per group a fixed number of library
  launches whatever B, H and W (fewer at H W = 1, where the non-anchor passes are empty), and no host
  synchronisation; stream errors surface at entropy_decode_finalize.  `substreams` as in cb_decode."""
  B, H, W, M, spans, psi = _scc_batch(packed, groups, psi)
  dev = psi.device
  phases = _substream_phases(handle, groups, [H] * B, [W] * B, substreams)
  coff = _i32(cdf_offset, dev)
  y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  lib = _lib.lib()
  for k, (p, (o, c)) in enumerate(zip(packed, spans)):
    ch = channel_context(k, y_hat) if k else None
    for anchors in (True, False):
      loc, _, index = scc_params(p, (o, c), y_hat, psi, ch, anchors, num_scales)
      part = _decode_phase(handle, phases, 2 * k + (0 if anchors else 1), index, loc, coff)
      check(lib.tfcb_scc_scatter(_p(part), B, H, W, M, o, c, int(anchors), _p(y_hat), _stream()))
  return y_hat


# ------------------------------------------------------------------------------------------------
# Ragged lists of latents (§3.13): the context models over images of their own latent shapes in one launch sequence.
# A list holds n images with latents [H_i, W_i, M] and psi [H_i, W_i, 2M] (float32 CUDA tensors); inside the calls
# they are flat, image after image.  Coding-order tensors are flat too: image i's H_i W_i M values follow image
# i - 1's, so `compress_ragged(lookup, lengths, y, loc, cdf_offset, index=index)` with the returned lengths makes each
# image's string, byte for byte the string of the fixed-shape call on that image alone.  Decoded latents are returned
# as a list of views of one flat buffer.
# ------------------------------------------------------------------------------------------------
def _ragged_list(psis):
  """(heights, widths, M) of a list of psi [H_i, W_i, 2M]; heights and widths are int64 numpy arrays."""
  import numpy as np
  if not isinstance(psis, (list, tuple)) or not psis:
    raise _lib.InvalidArgumentError("a ragged call needs a non-empty list of latents")
  for psi in psis:
    if not isinstance(psi, torch.Tensor) or psi.dim() != 3 or psi.shape[-1] % 2 or psi.shape[-1] != psis[0].shape[-1]:
      raise _lib.InvalidArgumentError("every `psi` must be [H_i, W_i, 2M] with one M")
    if psi.shape[0] == 0 or psi.shape[1] == 0:
      raise _lib.InvalidArgumentError(f"empty latents: psi has shape {tuple(psi.shape)}")
  hs = np.ascontiguousarray([int(p.shape[0]) for p in psis], dtype=np.int64)
  ws = np.ascontiguousarray([int(p.shape[1]) for p in psis], dtype=np.int64)
  return hs, ws, int(psis[0].shape[-1]) // 2


def _ragged_cat(ts, name, hs, ws, ch, dev):
  """The flat concatenation of the list `ts` of [H_i, W_i, ch] tensors."""
  if not isinstance(ts, (list, tuple)) or len(ts) != hs.size:
    raise _lib.InvalidArgumentError(f"`{name}` must be a list of {hs.size} tensors, one per image")
  return torch.cat([_ar_tensor(t, name, (int(h), int(w), ch), dev).reshape(-1) for t, h, w in zip(ts, hs, ws)])


def _ragged_views(flat, hs, ws, ch):
  """Image i's [H_i, W_i, ch] view of a flat list."""
  out, at = [], 0
  for h, w in zip(hs.tolist(), ws.tolist()):
    out.append(flat[at:at + h * w * ch].view(h, w, ch))
    at += h * w * ch
  return out


def _host(a):
  return a.ctypes.data_as(C.c_void_p)


def _ar_ragged(packed, psis):
  """(heights, widths, M, packed floats, flat psi) of a ragged call of the autoregressive model."""
  hs, ws, M = _ragged_list(psis)
  if not isinstance(packed, torch.Tensor) or packed.dim() != 1 or packed.dtype != torch.float32:
    raise _lib.InvalidArgumentError("`packed` must be a float32 vector from ar_pack_weights")
  n = ar_packed_floats(M)
  if packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, M={M} needs {n}")
  if packed.device.type != "cuda":
    raise _lib.InvalidArgumentError(f"`packed` must be on a CUDA device, not {packed.device}")
  return hs, ws, M, n, _ragged_cat(psis, "psi", hs, ws, 2 * M, packed.device)


def _ar_work(k, dev):
  nw = int(_lib.lib().tfcb_ar_ragged_workspace_floats(k))
  return torch.empty(max(nw, 1), dtype=torch.float32, device=dev), nw


def ar_encode_ragged(packed, ys, psis, num_scales, scale_index=False):
  """ar_encode of every position of a list of images of their own shapes, one CTA per image in one launch: returns
  (y_hats, y, loc, index, lengths), and scale_index last with `scale_index=True`.  y_hats is the list of [H_i, W_i, M];
  y, loc and index are flat in coding order (raster order, image after image), `lengths` the images' H_i W_i M."""
  hs, ws, M, n, psi = _ar_ragged(packed, psis)
  dev = packed.device
  y = _ragged_cat(ys, "y", hs, ws, M, dev)
  y_hat, loc = torch.empty_like(y), torch.empty_like(y)
  index = torch.empty(y.shape, dtype=torch.int32, device=dev)
  scale = torch.empty_like(y) if scale_index else None
  work, nw = _ar_work(hs.size, dev)
  check(_lib.lib().tfcb_ar_encode_ragged(_p(packed), n, M, _p(y), _p(psi), hs.size, _host(hs), _host(ws),
                                         int(num_scales), _p(work), nw, _p(y_hat), _p(loc), _p(index), _p(scale),
                                         _stream()))
  return (_ragged_views(y_hat, hs, ws, M), y, loc, index, (hs * ws * M).tolist()) + ((scale,) if scale_index else ())


def ar_decode_ragged(handle, packed, psis, num_scales, cdf_offset):
  """ar_decode of every position of a list of images, continuing `handle` (a DecoderHandle of one index-mode string per
  image): returns the list of y_hat [H_i, W_i, M].  One launch, one CTA per image, no host synchronisation; stream
  errors surface at entropy_decode_finalize."""
  hs, ws, M, n, psi = _ar_ragged(packed, psis)
  dev = packed.device
  if handle.n_streams != hs.size:
    raise _lib.InvalidArgumentError(f"the decoder holds {handle.n_streams} strings for a list of {hs.size}")
  y_hat = torch.zeros(int((hs * ws).sum()) * M, dtype=torch.float32, device=dev)
  work, nw = _ar_work(hs.size, dev)
  coff = _i32(cdf_offset, dev)
  check(_lib.lib().tfcb_ar_decode_ragged(handle._h, _p(packed), n, M, _p(psi), hs.size, _host(hs), _host(ws),
                                         int(num_scales), _p(coff), _p(work), nw, _p(y_hat), _stream()))
  return _ragged_views(y_hat, hs, ws, M)


# ------------------------------------------------------------------------------------------------
# Column tiles (DESIGN §3.15): the autoregressive model's latents as T independent streams per image, tile t holding
# columns [floor(t W / T), floor((t + 1) W / T)) of every row, encoded and decoded as a wavefront over many CTAs.
# ------------------------------------------------------------------------------------------------
def ar_tile_layout(hs, ws, tiles, depth=1):
  """(positions, widths) [images, max H_i] for substream_layout / substream_gather with S = `tiles`: one phase per
  latent row of W_i positions of `depth` symbols (M for the y strings); rows past H_i have no positions."""
  import numpy as np
  gen_ops.check_substreams(tiles, "tiles")
  hs = np.asarray(hs, dtype=np.int64).reshape(-1)
  ws = np.asarray(ws, dtype=np.int64).reshape(-1)
  if hs.size == 0 or hs.size != ws.size or (hs <= 0).any() or (ws <= 0).any():
    raise _lib.InvalidArgumentError(f"latent shapes {hs.tolist()} x {ws.tolist()}: one positive pair per image")
  pos = np.where(np.arange(int(hs.max()))[None, :] < hs[:, None], ws[:, None], 0).astype(np.int64)
  return pos, np.full(pos.shape, int(depth), dtype=np.int64)


def ar_tiles_schedule(hs, ws, tiles):
  """The library's ticket order of a list: int64 [items, 5] rows (image, row, tile, first column, end column)."""
  import numpy as np
  hs = np.ascontiguousarray(hs, dtype=np.int64).reshape(-1)
  ws = np.ascontiguousarray(ws, dtype=np.int64).reshape(-1)
  if hs.size != ws.size:
    raise _lib.InvalidArgumentError(f"{hs.size} heights and {ws.size} widths")
  n = C.c_int64(0)
  lib = _lib.lib()
  check(lib.tfcb_ar_tiles_schedule(hs.size, _host(hs), _host(ws), int(tiles), C.byref(n), None))
  out = np.zeros((n.value, 5), dtype=np.int64)
  check(lib.tfcb_ar_tiles_schedule(hs.size, _host(hs), _host(ws), int(tiles), C.byref(n), _host(out)))
  return out


def _ar_tiles_work(hs, ws, tiles, dev):
  nw = int(_lib.lib().tfcb_ar_tiles_workspace_floats(hs.size, _host(hs), _host(ws), int(tiles)))
  if nw < 0:
    raise _lib.InvalidArgumentError(f"tiles={tiles} is not supported for this list (1 <= tiles <= 1024)")
  return torch.empty((nw + 1) // 2, dtype=torch.float64, device=dev), nw  # (8-byte aligned)


def ar_encode_tiles(packed, ys, psis, num_scales, tiles, scale_index=False):
  """ar_encode_ragged over `tiles` = T column tiles per image, in one launch on many CTAs: returns (y_hats, y, loc,
  index, lengths), and scale_index last with `scale_index=True`.  y_hats are ar_encode_ragged's bit for bit; y, loc,
  index (and scale_index) are in tile order (image i's tile t at stream i T + t, as substream_gather makes them from
  ar_tile_layout) and `lengths` holds the n T stream lengths, ready for compress_ragged.  At T > 1 one gather (two
  with scale_index) follows the launch.  A schedule that could not finish leaves index -1 at the positions it skipped,
  which compress_ragged rejects."""
  T = gen_ops.check_substreams(tiles, "tiles")
  hs, ws, M, n, psi = _ar_ragged(packed, psis)
  dev = packed.device
  y = _ragged_cat(ys, "y", hs, ws, M, dev)
  y_hat, loc = torch.empty_like(y), torch.empty_like(y)
  index = torch.empty(y.shape, dtype=torch.int32, device=dev)
  scale = torch.empty_like(y) if scale_index else None
  work, nw = _ar_tiles_work(hs, ws, T, dev)
  check(_lib.lib().tfcb_ar_encode_tiles(_p(packed), n, M, _p(y), _p(psi), hs.size, _host(hs), _host(ws), T,
                                        int(num_scales), _p(work), nw, _p(y_hat), _p(loc), _p(index), _p(scale),
                                        _stream()))
  out = (y, loc, index) + ((scale,) if scale_index else ())
  lengths = (hs * ws * M).tolist()
  if T > 1:
    pos, wid = ar_tile_layout(hs, ws, T, M)
    out = substream_gather(pos, wid, T, y, loc, index)
    if scale_index:
      out += (substream_gather(pos, wid, T, loc=scale)[1],)
    lengths = substream_layout(pos, wid, T)[0].tolist()
  return (_ragged_views(y_hat, hs, ws, M),) + out[:3] + (lengths,) + out[3:]


def ar_decode_tiles(handle, packed, psis, num_scales, cdf_offset, tiles):
  """ar_decode_ragged of strings written in `tiles` = T column tiles: `handle` holds n T streams (image i's tile t at
  i T + t, gen_ops.split_substreams of the strings).  Returns the list of y_hat [H_i, W_i, M], ar_decode_ragged's bit
  for bit.  One launch, no host synchronisation; stream errors, including a schedule that could not finish, surface at
  entropy_decode_finalize."""
  T = gen_ops.check_substreams(tiles, "tiles")
  hs, ws, M, n, psi = _ar_ragged(packed, psis)
  dev = packed.device
  if handle.n_streams != hs.size * T:
    raise _lib.InvalidArgumentError(f"the decoder holds {handle.n_streams} strings for a list of {hs.size}"
                                    f" in {T} tiles")
  y_hat = torch.zeros(int((hs * ws).sum()) * M, dtype=torch.float32, device=dev)
  work, nw = _ar_tiles_work(hs, ws, T, dev)
  coff = _i32(cdf_offset, dev)
  check(_lib.lib().tfcb_ar_decode_tiles(handle._h, _p(packed), n, M, _p(psi), hs.size, _host(hs), _host(ws), T,
                                        int(num_scales), _p(coff), _p(work), nw, _p(y_hat), _stream()))
  return _ragged_views(y_hat, hs, ws, M)


def _scc_ragged(packed, groups, psis, layout=scc_layout):
  """(heights, widths, M, spans, flat psi) of a whole-latent ragged call, with every group's packed buffer checked."""
  hs, ws, M = _ragged_list(psis)
  spans = scc_spans(groups)
  if sum(c for _, c in spans) != M or len(packed) != len(spans):
    raise _lib.InvalidArgumentError(f"{len(packed)} packed networks and groups {tuple(groups)} for a latent of depth "
                                    f"{M}: one network per group, and the groups must sum to M")
  for p, g in zip(packed, spans):
    _scc_check_packed(p, M, g, layout)
  return hs, ws, M, spans, _ragged_cat(psis, "psi", hs, ws, 2 * M, packed[0].device)


def _scc_check_packed(packed, M, group, layout=scc_layout):
  o, c = (int(v) for v in group)
  n = layout(M, group)["total"]
  if not isinstance(packed, torch.Tensor) or packed.dim() != 1 or packed.dtype != torch.float32:
    raise _lib.InvalidArgumentError(f"`packed` must be a float32 vector from {_PACKERS[layout]}")
  if packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, group ({o}, {c}) of M={M} needs {n}")
  if packed.device.type != "cuda":
    raise _lib.InvalidArgumentError(f"`packed` must be on a CUDA device, not {packed.device}")
  return n


def _scc_pass_ragged(packed, group, M, hs, ws, y_hat, psi, ch_ctx, anchors, num_scales, whole=False, loc=None,
                     scale=None, index=None, y=None, y_cc=None, y_hat_out=None):
  """One pass of group (offset, channels) over the flat list.  Per-pass outputs (whole False, loc None) are allocated:
  returns (loc, scale_index, index, lengths, work) with image i's n_k,i c values at c Q_i; the workspace holds the
  image table for the scatter."""
  o, c = (int(v) for v in group)
  n = _scc_check_packed(packed, M, group)
  dev = packed.device
  lib = _lib.lib()
  k = hs.size
  counts = (hs * ws + 1) // 2 if anchors else hs * ws // 2
  if loc is None:
    total = int(counts.sum()) * c
    loc, scale = (torch.empty(total, dtype=torch.float32, device=dev) for _ in range(2))
    index = torch.empty(total, dtype=torch.int32, device=dev)
  nw = int(lib.tfcb_scc_ragged_workspace_floats(M, o, c, k, _host(hs), _host(ws), int(bool(anchors))))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=dev)
  check(lib.tfcb_scc_params_ragged(_p(packed), n, M, o, c, _p(y_hat), _p(psi), _p(ch_ctx), k, _host(hs), _host(ws),
                                   int(bool(anchors)), int(num_scales), _p(work), nw, int(whole), _p(loc), _p(scale),
                                   _p(index), _p(y), _p(y_cc), _p(y_hat_out), _stream()))
  return loc, scale, index, (counts * c).tolist(), work


def _scc_ch_ctx_ragged(ch_ctx, group, hs, ws, dev):
  """The flat channel context of a group at a positive offset (a list of [H_i, W_i, 2c]); None at offset 0."""
  o, c = (int(v) for v in group)
  if o == 0:
    if ch_ctx is not None:
      raise _lib.InvalidArgumentError("the group at offset 0 has no channel context: pass None")
    return None
  return _ragged_cat(ch_ctx, "ch_ctx", hs, ws, 2 * c, dev)


def scc_params_ragged(packed, group, y_hats, psis, ch_ctx, anchors, num_scales):
  """scc_params over a list of images of their own shapes in one pass: returns (loc, scale_index, index, lengths),
  flat, image i's n_i c values (n_i its positions of this colour) after image i - 1's; `lengths` are the n_i c.
  ch_ctx is a list of [H_i, W_i, 2c] (None at offset 0); y_hats a list of [H_i, W_i, M] (may be None for the anchor
  pass).  Image i's values equal scc_params on that image alone, bit for bit."""
  hs, ws, M = _ragged_list(psis)
  _scc_check_packed(packed, M, group)
  dev = packed.device
  psi = _ragged_cat(psis, "psi", hs, ws, 2 * M, dev)
  ch = _scc_ch_ctx_ragged(ch_ctx, group, hs, ws, dev)
  y_hat = None if y_hats is None and anchors else _ragged_cat(y_hats, "y_hat", hs, ws, M, dev)
  return _scc_pass_ragged(packed, group, M, hs, ws, y_hat, psi, ch, anchors, num_scales)[:4]


def scc_encode_ragged(packed, groups, ys, psis, channel_context, num_scales, scale_index=False, substreams=1):
  """scc_encode of a list of images of their own shapes, one pass sequence for the whole list: returns (y_hats, y,
  loc, index, lengths), and scale_index last with `scale_index=True`.  `channel_context(k, y_hats)` takes and returns
  lists ([H_i, W_i, 2c_k] per image).  y, loc and index are flat in coding order, image i's H_i W_i M values (its
  `lengths` entry) after image i - 1's.  With `substreams` = S > 1 they are in substream order (one gather, a second
  one for scale_index) and `lengths` holds the n S stream lengths, image i's substream s at i S + s."""
  hs, ws, M, spans, psi = _scc_ragged(packed, groups, psis)
  dev = psi.device
  y = _ragged_cat(ys, "y", hs, ws, M, dev)
  y_hat, y_cc, loc = (torch.empty_like(y) for _ in range(3))
  index = torch.empty(y.shape, dtype=torch.int32, device=dev)
  scale = torch.empty_like(y) if scale_index else None
  views = _ragged_views(y_hat, hs, ws, M)
  for k, (p, g) in enumerate(zip(packed, spans)):
    ch = _scc_ch_ctx_ragged(channel_context(k, views) if k else None, g, hs, ws, dev)
    for anchors in (True, False):
      _scc_pass_ragged(p, g, M, hs, ws, y_hat, psi, ch, anchors, num_scales, True, loc, scale, index, y, y_cc, y_hat)
  out = _to_substreams(groups, hs, ws, substreams, y_cc, loc, index, scale)
  lengths = (hs * ws * M).tolist() if substreams == 1 else context_substreams(groups, hs, ws, substreams)[0].tolist()
  return (views,) + out[:3] + (lengths,) + out[3:]


def scc_decode_ragged(handle, packed, groups, psis, channel_context, num_scales, cdf_offset, substreams=1):
  """scc_decode of a list of images of their own shapes, continuing `handle` (one index-mode string per image): per
  group its channel context (as in scc_encode_ragged), then per colour one ragged parameter pass, one decode_ragged
  and one scatter for the whole list.  Returns the list of y_hat [H_i, W_i, M].  The library launches depend on the
  groups, not on the images' number or shapes (fewer when every image is 1x1); no host synchronisation.  With
  `substreams` = S > 1 the handle holds n S substreams and each decode_ragged takes that pass's substream lengths."""
  hs, ws, M, spans, psi = _scc_ragged(packed, groups, psis)
  dev = psi.device
  phases = _substream_phases(handle, groups, hs, ws, substreams, "list")
  coff = _i32(cdf_offset, dev)
  y_hat = torch.zeros(int((hs * ws).sum()) * M, dtype=torch.float32, device=dev)
  views = _ragged_views(y_hat, hs, ws, M)
  lib = _lib.lib()
  for k, (p, (o, c)) in enumerate(zip(packed, spans)):
    ch = _scc_ch_ctx_ragged(channel_context(k, views) if k else None, (o, c), hs, ws, dev)
    for anchors in (True, False):
      loc, _, index, lengths, work = _scc_pass_ragged(p, (o, c), M, hs, ws, y_hat, psi, ch, anchors, num_scales)
      if phases is not None:
        lengths = phases[2 * k + (0 if anchors else 1)]
      part = decode_ragged(handle, lengths, index=index, quant_offset=loc, cdf_offset=coff)
      check(lib.tfcb_scc_scatter_ragged(_p(part), hs.size, _host(hs), _host(ws), M, o, c, int(anchors), _p(work),
                                        work.numel(), _p(y_hat), _stream()))
  return views


def _cb_ragged_check(packed, psis):
  """The checkerboard model's packed size (M a multiple of 6) before the group (0, M) calls."""
  M = _ragged_list(psis)[2]
  n = ar_packed_floats(M)
  if isinstance(packed, torch.Tensor) and packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, M={M} needs {n}")
  return M


def cb_params_ragged(packed, y_hats, psis, anchors, num_scales):
  """cb_params over a list of images of their own shapes in one pass: (loc, scale_index, index, lengths) as
  scc_params_ragged gives them for the group (0, M), which is the checkerboard pass bit for bit."""
  M = _cb_ragged_check(packed, psis)
  return scc_params_ragged(packed, (0, M), y_hats, psis, None, anchors, num_scales)


def cb_encode_ragged(packed, ys, psis, num_scales, scale_index=False, substreams=1):
  """cb_encode of a list of images of their own shapes: (y_hats, y, loc, index, lengths) as scc_encode_ragged."""
  M = _cb_ragged_check(packed, psis)
  return scc_encode_ragged([packed], (M,), ys, psis, None, num_scales, scale_index, substreams)


def cb_decode_ragged(handle, packed, psis, num_scales, cdf_offset, substreams=1):
  """cb_decode of a list of images of their own shapes: two parameter passes, two decode_ragged calls and two
  scatters for the whole list.  Returns the list of y_hat [H_i, W_i, M]."""
  M = _cb_ragged_check(packed, psis)
  return scc_decode_ragged(handle, [packed], (M,), psis, None, num_scales, cdf_offset, substreams)


# ------------------------------------------------------------------------------------------------
# Checkerboard context model with mixture priors (DESIGN §3.19): the checkerboard's two parameter passes on a network
# whose last layer has 3KM outputs, each ending in the per-latent mixtures of the mixture coder (tfcb_cbm_*).  Coding
# order is the checkerboard's.  One image's y string is varint(len A) ‖ A ‖ N, A and N the strings
# mixture_encode_ragged writes for its anchors' and its non-anchors' coding-order latents (with S substreams each
# when substreams = S > 1).  Latents are float32 CUDA [B, H, W, M], psi [B, H, W, 2M]; mixture parameters are
# [..., M, K], components innermost.
# ------------------------------------------------------------------------------------------------
CBM_LAYOUT_KEYS = ("K1", "N3", "N4", "NO", "wc", "bc", "w1", "b1", "w2", "b2", "w3", "b3")


def cbm_layout(M, K):
  """The packed network of latent depth M (a multiple of 6 in [6, 384]) with K components (in [1, 64]): widths K1,
  N3, N4, NO = 3KM, the offsets of its eight operands and `total`, in floats."""
  lay = np.zeros(len(CBM_LAYOUT_KEYS), dtype=np.int64)
  n = int(_lib.lib().tfcb_cbm_packed_floats(int(M), int(K), lay.ctypes.data_as(C.POINTER(C.c_int64))))
  if n < 0:
    raise _lib.InvalidArgumentError(f"latent depth M={M} must be a positive multiple of 6 and at most 384, and K={K} "
                                    f"in [1, 64]")
  return dict(zip(CBM_LAYOUT_KEYS, (int(v) for v in lay)), total=n)


def cbm_pack_weights(ctx_kernel, ctx_bias, w1, b1, w2, b2, w3, b3):
  """cb_pack_weights for the mixture network: the 12 checkerboard taps of the context kernel [5, 5, M, 2M], then the
  1x1 layers [4M, 10M/3], [10M/3, 8M/3], [8M/3, 3KM] and their biases; K is read from W3's width.  Returns float32
  [total] on the context kernel's device, the values copied unchanged."""
  ctx_kernel = ctx_kernel.detach()
  if ctx_kernel.dim() != 4 or ctx_kernel.shape[:2] != (5, 5) or ctx_kernel.shape[3] != 2 * ctx_kernel.shape[2]:
    raise _lib.InvalidArgumentError(f"context kernel must be [5, 5, M, 2M]: {tuple(ctx_kernel.shape)}")
  M = int(ctx_kernel.shape[2])
  if w3.dim() != 2 or M <= 0 or w3.shape[1] % (3 * M):
    raise _lib.InvalidArgumentError(f"W3 of shape {tuple(w3.shape)} must be [8M/3, 3KM] for M={M}")
  K = int(w3.shape[1]) // (3 * M)
  lay = cbm_layout(M, K)
  dev = ctx_kernel.device
  if dev.type != "cuda":
    raise _lib.InvalidArgumentError(f"the parameters must be on a CUDA device, not {dev}")
  n3, n4, no = lay["N3"], lay["N4"], lay["NO"]
  want = ((ctx_bias, (2 * M,)), (w1, (4 * M, n3)), (b1, (n3,)), (w2, (n3, n4)), (b2, (n4,)), (w3, (n4, no)),
          (b3, (no,)))
  ops = [_f32(ctx_kernel[[dy + 2 for dy, _ in CB_TAPS], [dx + 2 for _, dx in CB_TAPS]], dev)]
  for t, shape in want:
    t = t.detach()
    if tuple(t.shape) != shape:
      raise _lib.InvalidArgumentError(f"parameter of shape {tuple(t.shape)} where M={M}, K={K} needs {shape}")
    ops.append(_f32(t, dev))
  packed = torch.empty(lay["total"], dtype=torch.float32, device=dev)
  check(_lib.lib().tfcb_cbm_pack_weights(M, K, *[_p(t) for t in ops], _p(packed), lay["total"], _stream()))
  return packed


def _cbm_check_packed(packed, M, K):
  n = cbm_layout(M, K)["total"]
  if not isinstance(packed, torch.Tensor) or packed.dim() != 1 or packed.dtype != torch.float32:
    raise _lib.InvalidArgumentError("`packed` must be a float32 vector from cbm_pack_weights")
  if packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, M={M} with K={K} needs {n}")
  if packed.device.type != "cuda":
    raise _lib.InvalidArgumentError(f"`packed` must be on a CUDA device, not {packed.device}")
  return n


def _cbm_dims(packed, K, psi):
  """(B, H, W, M, packed floats) from psi [B, H, W, 2M], checked against the packed buffer."""
  if not isinstance(psi, torch.Tensor) or psi.dim() != 4 or psi.shape[-1] % 2:
    raise _lib.InvalidArgumentError("`psi` must be [B, H, W, 2M]")
  B, H, W, M = int(psi.shape[0]), int(psi.shape[1]), int(psi.shape[2]), int(psi.shape[3]) // 2
  if B == 0 or H == 0 or W == 0:
    raise _lib.InvalidArgumentError(f"empty latents: psi has shape {tuple(psi.shape)}")
  n = _cbm_check_packed(packed, M, K)
  if psi.device != packed.device:
    raise _lib.InvalidArgumentError(f"`packed` ({packed.device}) and `psi` ({psi.device}) must share a CUDA device")
  return B, H, W, M, n


def _cbm_coder(family, precision, tail_mass, max_support):
  if family not in MIXTURE_FAMILIES:
    raise _lib.InvalidArgumentError(f"`family` must be one of {sorted(MIXTURE_FAMILIES)}: {family!r}")
  return dict(family=family, precision=precision, tail_mass=tail_mass, max_support=max_support)


def _cbm_lengths(counts, M, substreams):
  """The stream lengths of items of counts[u] positions of M latents: one stream each, or S substreams each as
  MixtureEntropyModel splits a [positions, M] coding unit."""
  if substreams == 1:
    return [int(c) * M for c in counts]
  return substream_layout([[int(c)] for c in counts], M, substreams)[0].tolist()


def cbm_join(parts):
  """The y strings of B images from the 2B strings `parts` (image b's anchors at 2b, its non-anchors at 2b + 1):
  varint(len A) ‖ A ‖ N each.  One device-to-host copy (the offsets); the bytes stay on the device."""
  offs = parts.offsets_dev.cpu().numpy()
  n = parts.numel() // 2
  heads = [gen_ops._varint(int(offs[2 * b + 1] - offs[2 * b])) for b in range(n)]
  dev = parts.bytes_dev.device
  hbuf = torch.from_numpy(np.frombuffer(b"".join(heads) + b"\0", dtype=np.uint8).copy()).to(dev)
  chunks, out_offs, at = [], [0], 0
  for b, h in enumerate(heads):
    lo, hi = int(offs[2 * b]), int(offs[2 * b + 2])
    chunks += [hbuf[at:at + len(h)], parts.bytes_dev[lo:hi]]
    at += len(h)
    out_offs.append(out_offs[-1] + len(h) + hi - lo)
  data = torch.cat(chunks + [torch.zeros(1, dtype=torch.uint8, device=dev)])
  return gen_ops.Strings(data, torch.tensor(out_offs, dtype=torch.int64).to(dev), (n,))


def cbm_split(s, i=0):
  """(A, N) of string number `i`, `s` (bytes).  A truncated or non-minimal varint, or an anchor part that runs past
  the end of the string, raises InvalidArgumentError naming the string."""
  s = bytes(s)
  v, shift, at = 0, 0, 0
  while True:
    if at >= len(s):
      raise _lib.InvalidArgumentError(f"string {i}: truncated length of its anchor part")
    b = s[at]
    at += 1
    v |= (b & 0x7F) << shift
    if not b & 0x80:
      break
    shift += 7
    if shift > 63:
      raise _lib.InvalidArgumentError(f"string {i}: anchor length varint longer than 64 bits")
  if at > 1 and b == 0:
    raise _lib.InvalidArgumentError(f"string {i}: anchor length varint not in minimal form")
  if v > len(s) - at:
    raise _lib.InvalidArgumentError(f"string {i}: an anchor part of {v} bytes runs past the end of its {len(s)} bytes")
  return s[at:at + v], s[at + v:]


def _cbm_parts(strings, n, substreams):
  """Both colours' strings of n y strings, split on the host before any device work: (anchors, non-anchors), each a
  Strings of their payloads (n S substreams with S > 1)."""
  if not isinstance(strings, gen_ops.Strings):
    strings = gen_ops.Strings.from_bytes(list(strings), (len(strings),))
  if strings.numel() != n:
    raise _lib.InvalidArgumentError(f"{strings.numel()} strings for {n} images")
  split = [cbm_split(s, i) for i, s in enumerate(strings.tolist())]
  out = []
  for c in range(2):
    part = gen_ops.Strings.from_bytes([p[c] for p in split], (n,))
    out.append(gen_ops.split_substreams(part, substreams) if substreams > 1 else part)
  return out


def _cbm_pass(packed, K, y_hat, psi, anchors, whole, weight, loc, scale, y=None, y_cb=None, y_hat_out=None):
  B, H, W, M, n = _cbm_dims(packed, K, psi)
  lib = _lib.lib()
  nw = int(lib.tfcb_cbm_workspace_floats(M, int(K), B, H, W, int(bool(anchors))))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=packed.device)
  check(lib.tfcb_cbm_params(_p(packed), n, M, int(K), _p(y_hat), _p(psi), B, H, W, int(bool(anchors)), _p(work), nw,
                            int(whole), _p(weight), _p(loc), _p(scale), _p(y), _p(y_cb), _p(y_hat_out), _stream()))


def cbm_params(packed, K, y_hat, psi, anchors):
  """One parameter pass: (weight, loc, scale) [B, n, M, K] of the n positions of one colour of every image, in coding
  order, as the mixture coder takes them (weights unnormalised, the largest 1).  The non-anchor pass reads the
  anchors of y_hat [B, H, W, M]; the anchor pass reads no latent (y_hat may be None)."""
  B, H, W, M, _ = _cbm_dims(packed, K, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  if y_hat is not None or not anchors:
    y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  n = cb_counts(H, W)[0 if anchors else 1]
  weight, loc, scale = (torch.empty((B, n, M, int(K)), dtype=torch.float32, device=dev) for _ in range(3))
  _cbm_pass(packed, K, y_hat, psi, anchors, False, weight, loc, scale)
  return weight, loc, scale


def cbm_encode(packed, K, y, psi, family="normal", substreams=1, precision=16, tail_mass=2**-8, max_support=256):
  """The two-pass encoder: returns (y_hat [B, H, W, M], strings of shape (B,)).  y_hat = float(int32(rint(y)))
  (saturating, NaN -> 0), the anchors' before the non-anchor pass reads them; then one mixture_encode_ragged of the
  coding-order y over the 2B items (image, colour) and one join."""
  coder = _cbm_coder(family, precision, tail_mass, max_support)
  S = gen_ops.check_substreams(substreams)
  B, H, W, M, _ = _cbm_dims(packed, K, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  y = _ar_tensor(y, "y", (B, H, W, M), dev)
  y_hat = torch.empty((B, H, W, M), dtype=torch.float32, device=dev)
  y_cb = torch.empty((B, H * W, M), dtype=torch.float32, device=dev)
  weight, loc, scale = (torch.empty((B, H * W, M, int(K)), dtype=torch.float32, device=dev) for _ in range(3))
  for anchors in (True, False):
    _cbm_pass(packed, K, y_hat, psi, anchors, True, weight, loc, scale, y, y_cb, y_hat)
  parts = mixture_encode_ragged(y_cb, weight, loc, scale, _cbm_lengths(cb_counts(H, W) * B, M, S), **coder)
  if S > 1:
    parts = gen_ops.join_substreams(parts, S, (2 * B,))
  return y_hat, cbm_join(parts)


def cbm_decode(strings, packed, K, psi, family="normal", substreams=1, precision=16, tail_mass=2**-8,
               max_support=256):
  """Inverse of cbm_encode: anchor parameters, one mixture decode of every image's anchors, their latents to
  [B, H, W, M], non-anchor parameters, one decode of the non-anchors, to [B, H, W, M].  Returns y_hat [B, H, W, M].
  The strings are split on the host first; a length that overruns its string or a wrong `substreams` raises
  InvalidArgumentError before any device work."""
  coder = _cbm_coder(family, precision, tail_mass, max_support)
  S = gen_ops.check_substreams(substreams)
  B, H, W, M, _ = _cbm_dims(packed, K, psi)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  parts = _cbm_parts(strings, B, S)
  y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  lib = _lib.lib()
  for c, anchors in enumerate((True, False)):
    n = cb_counts(H, W)[c]
    if n == 0:
      continue
    weight, loc, scale = cbm_params(packed, K, y_hat, psi, anchors)
    part = mixture_decode_ragged(parts[c], weight, loc, scale, _cbm_lengths([n] * B, M, S), **coder)
    check(lib.tfcb_cb_scatter(_p(part), B, H, W, M, int(anchors), _p(y_hat), _stream()))
  return y_hat


def _cbm_ragged(packed, K, psis):
  """(heights, widths, M, packed floats, flat psi) of a ragged call."""
  hs, ws, M = _ragged_list(psis)
  n = _cbm_check_packed(packed, M, K)
  return hs, ws, M, n, _ragged_cat(psis, "psi", hs, ws, 2 * M, packed.device)


def _cbm_pass_ragged(packed, K, M, n, hs, ws, y_hat, psi, anchors, whole=False, weight=None, loc=None, scale=None,
                     y=None, y_cb=None, y_hat_out=None):
  """One pass over the flat list.  Per-pass outputs (weight None) are allocated: returns (weight, loc, scale, counts,
  work) with image i's n_k,i M rows at M Q_i; the workspace holds the image table for the scatter."""
  dev = packed.device
  lib = _lib.lib()
  k = hs.size
  counts = (hs * ws + 1) // 2 if anchors else hs * ws // 2
  if weight is None:
    weight, loc, scale = (torch.empty((int(counts.sum()) * M, int(K)), dtype=torch.float32, device=dev)
                          for _ in range(3))
  nw = int(lib.tfcb_cbm_ragged_workspace_floats(M, int(K), k, _host(hs), _host(ws), int(bool(anchors))))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=dev)
  check(lib.tfcb_cbm_params_ragged(_p(packed), n, M, int(K), _p(y_hat), _p(psi), k, _host(hs), _host(ws),
                                   int(bool(anchors)), _p(work), nw, int(whole), _p(weight), _p(loc), _p(scale), _p(y),
                                   _p(y_cb), _p(y_hat_out), _stream()))
  return weight, loc, scale, counts, work


def cbm_params_ragged(packed, K, y_hats, psis, anchors):
  """cbm_params over a list of images of their own shapes in one pass: (weight, loc, scale, lengths), the first three
  [sum n_i M, K] with image i's n_i M rows (n_i its positions of this colour) after image i - 1's; `lengths` are the
  n_i M.  y_hats is a list of [H_i, W_i, M] (may be None for the anchor pass).  Image i's values equal cbm_params on
  that image alone, bit for bit."""
  hs, ws, M, n, psi = _cbm_ragged(packed, K, psis)
  dev = packed.device
  y_hat = None if y_hats is None and anchors else _ragged_cat(y_hats, "y_hat", hs, ws, M, dev)
  weight, loc, scale, counts, _ = _cbm_pass_ragged(packed, K, M, n, hs, ws, y_hat, psi, anchors)
  return weight, loc, scale, (counts * M).tolist()


def cbm_encode_ragged(packed, K, ys, psis, family="normal", substreams=1, precision=16, tail_mass=2**-8,
                      max_support=256):
  """cbm_encode of a list of images of their own shapes, one pass sequence and one mixture encode for the whole list:
  returns (y_hats, strings of shape (n,)), y_hats the list of [H_i, W_i, M].  String i equals cbm_encode's string of
  image i alone."""
  coder = _cbm_coder(family, precision, tail_mass, max_support)
  S = gen_ops.check_substreams(substreams)
  hs, ws, M, n, psi = _cbm_ragged(packed, K, psis)
  dev = packed.device
  y = _ragged_cat(ys, "y", hs, ws, M, dev)
  y_hat, y_cb = torch.empty_like(y), torch.empty_like(y)
  weight, loc, scale = (torch.empty((y.numel(), int(K)), dtype=torch.float32, device=dev) for _ in range(3))
  for anchors in (True, False):
    _cbm_pass_ragged(packed, K, M, n, hs, ws, y_hat, psi, anchors, True, weight, loc, scale, y, y_cb, y_hat)
  counts = np.stack([(hs * ws + 1) // 2, hs * ws // 2], 1).reshape(-1)
  parts = mixture_encode_ragged(y_cb, weight, loc, scale, _cbm_lengths(counts, M, S), **coder)
  if S > 1:
    parts = gen_ops.join_substreams(parts, S, (2 * hs.size,))
  return _ragged_views(y_hat, hs, ws, M), cbm_join(parts)


def cbm_decode_ragged(strings, packed, K, psis, family="normal", substreams=1, precision=16, tail_mass=2**-8,
                      max_support=256):
  """cbm_decode of a list of images of their own shapes, one string per image: per colour one ragged parameter pass,
  one mixture decode and one scatter for the whole list.  Returns the list of y_hat [H_i, W_i, M]."""
  coder = _cbm_coder(family, precision, tail_mass, max_support)
  S = gen_ops.check_substreams(substreams)
  hs, ws, M, n, psi = _cbm_ragged(packed, K, psis)
  dev = packed.device
  parts = _cbm_parts(strings, hs.size, S)
  y_hat = torch.zeros(int((hs * ws).sum()) * M, dtype=torch.float32, device=dev)
  lib = _lib.lib()
  for c, anchors in enumerate((True, False)):
    weight, loc, scale, counts, work = _cbm_pass_ragged(packed, K, M, n, hs, ws, y_hat, psi, anchors)
    if not counts.any():
      continue
    part = mixture_decode_ragged(parts[c], weight, loc, scale, _cbm_lengths(counts, M, S), **coder)
    check(lib.tfcb_scc_scatter_ragged(_p(part), hs.size, _host(hs), _host(ws), M, 0, M, int(anchors), _p(work),
                                      work.numel(), _p(y_hat), _stream()))
  return _ragged_views(y_hat, hs, ws, M)


# ------------------------------------------------------------------------------------------------
# Multistage context model (Lin et al. 2023): four parameter passes over the stages of a 2x2 schedule (tfcb_msc_*).
# Position (r, c) has phase (r mod 2, c mod 2); the phases (0, 0), (1, 1), (0, 1), (1, 0) are stages 0 to 3.  Stage
# s >= 1 reads the decoded latents at its taps (the offsets whose neighbour is in an earlier stage) through its own
# context kernel; the three 1x1 entropy-parameter layers are shared.  Coding order: per image, stage 0, 1, 2, 3, each
# in raster order with M channels per position.  Latents are float32 CUDA [B, H, W, M], psi [B, H, W, 2M];
# coding-order tensors are [B, n_s, M] for one stage and [B, H * W, M] for all four.
# ------------------------------------------------------------------------------------------------
MSC_PHASES = ((0, 0), (1, 1), (0, 1), (1, 0))


def msc_stage(r, c):
  """The stage of latent position (r, c)."""
  return MSC_PHASES.index((r % 2, c % 2))


MSC_TAPS = tuple(tuple((dy, dx) for dy in range(-2, 3) for dx in range(-2, 3)
                       if (dy, dx) != (0, 0) and msc_stage(a + dy, b + dx) < s)
                 for s, (a, b) in enumerate(MSC_PHASES))  # per stage, raster order: 0, 4, 12 and 16 taps


def msc_packed_floats(M):
  """Floats of the packed parameter buffer for latent depth M (a multiple of 6 in [6, 384])."""
  n = int(_lib.lib().tfcb_msc_packed_floats(int(M)))
  if n < 0:
    raise _lib.InvalidArgumentError(f"latent depth M={M} must be a positive multiple of 6 and at most 384")
  return n


def msc_pack_weights(ctx_kernels, ctx_biases, w1, b1, w2, b2, w3, b3):
  """The device layout of the four passes: for stages 1, 2 and 3 the taps of its context kernel [5, 5, M, 2M]
  (masked or not: no other tap is read), gathered as [T_s, M, 2M], and its bias [2M]; then the shared 1x1 layers
  as [inputs, outputs] and their biases.  Returns float32 [msc_packed_floats(M)] on the kernels' device."""
  ctx_kernels, ctx_biases = list(ctx_kernels), list(ctx_biases)
  if len(ctx_kernels) != 3 or len(ctx_biases) != 3:
    raise _lib.InvalidArgumentError("one context kernel and one bias for each of stages 1, 2 and 3")
  k = ctx_kernels[0]
  if k.dim() != 4 or k.shape[:2] != (5, 5) or k.shape[3] != 2 * k.shape[2]:
    raise _lib.InvalidArgumentError(f"context kernels must be [5, 5, M, 2M]: {tuple(k.shape)}")
  M = int(k.shape[2])
  n = msc_packed_floats(M)
  ops = _ms_operands(M, 4 * M, ctx_kernels, ctx_biases, (w1, b1, w2, b2, w3, b3), f"M={M}")
  packed = torch.empty(n, dtype=torch.float32, device=ops[0].device)
  check(_lib.lib().tfcb_msc_pack_weights(M, *[_p(t) for t in ops], _p(packed), n, _stream()))
  return packed


def _ms_operands(c, k1, ctx_kernels, ctx_biases, dense, where):
  """The twelve operands of a multistage network of c channels whose layer 1 is k1 wide, in the library's order:
  per stage 1-3 the taps of its context kernel [5, 5, c, 2c] gathered as [T_s, c, 2c] and its bias [2c]; then the
  1x1 layers (W1, b1, W2, b2, W3, b3) as [inputs, outputs] and their biases, K1 -> 5 K1 / 6 -> 2 K1 / 3 -> 2c."""
  dev = ctx_kernels[0].device
  if dev.type != "cuda":
    raise _lib.InvalidArgumentError(f"the parameters must be on a CUDA device, not {dev}")
  n3, n4 = 5 * k1 // 6, 2 * k1 // 3

  def operand(t, shape):
    t = t.detach()
    if tuple(t.shape) != shape:
      raise _lib.InvalidArgumentError(f"parameter of shape {tuple(t.shape)} where {where} needs {shape}")
    return _f32(t, dev)

  ops = []
  for s, (kernel, bias) in enumerate(zip(ctx_kernels, ctx_biases), 1):
    kernel = operand(kernel, (5, 5, c, 2 * c))
    taps = MSC_TAPS[s]
    ops += [kernel[[dy + 2 for dy, _ in taps], [dx + 2 for _, dx in taps]].contiguous(), operand(bias, (2 * c,))]
  for t, shape in zip(dense, ((k1, n3), (n3,), (n3, n4), (n4,), (n4, 2 * c), (2 * c,))):
    ops.append(operand(t, shape))
  return ops


def msc_counts(H, W):
  """Positions of stages 0 to 3 of an H x W latent: ceil((H - a) / 2) * ceil((W - b) / 2) at phase (a, b)."""
  return tuple(((H - a + 1) // 2) * ((W - b + 1) // 2) for a, b in MSC_PHASES)


def _msc_dims(packed, psi):
  """(B, H, W, M, packed floats) from psi [B, H, W, 2M], checked against the packed buffer."""
  if not isinstance(psi, torch.Tensor) or psi.dim() != 4 or psi.shape[-1] % 2:
    raise _lib.InvalidArgumentError("`psi` must be [B, H, W, 2M]")
  B, H, W, M = int(psi.shape[0]), int(psi.shape[1]), int(psi.shape[2]), int(psi.shape[3]) // 2
  if B == 0 or H == 0 or W == 0:
    raise _lib.InvalidArgumentError(f"empty latents: psi has shape {tuple(psi.shape)}")
  _msc_check_packed(packed, M)
  if psi.device != packed.device:
    raise _lib.InvalidArgumentError(f"`packed` ({packed.device}) and `psi` ({psi.device}) must share a CUDA device")
  return B, H, W, M, packed.numel()


def _msc_check_packed(packed, M):
  if not isinstance(packed, torch.Tensor) or packed.dim() != 1 or packed.dtype != torch.float32:
    raise _lib.InvalidArgumentError("`packed` must be a float32 vector from msc_pack_weights")
  n = msc_packed_floats(M)
  if packed.numel() != n:
    raise _lib.InvalidArgumentError(f"packed weights hold {packed.numel()} floats, M={M} needs {n}")
  if packed.device.type != "cuda":
    raise _lib.InvalidArgumentError(f"`packed` must be on a CUDA device, not {packed.device}")
  return n


def _msc_stage_arg(stage):
  if int(stage) not in range(4):
    raise _lib.InvalidArgumentError(f"stage {stage} outside [0, 4)")
  return int(stage)


def msc_params(packed, y_hat, psi, stage, num_scales):
  """One parameter pass: (loc, scale_index, index) [B, n_s, M] (float32, float32, int32) of the n_s positions of
  stage `stage` of every image, in coding order.  Stages 1-3 read the earlier stages' positions of y_hat
  [B, H, W, M]; stage 0 reads no latent (y_hat may be None).  Row b depends only on image b.  (mscc_params of the
  one group (0, M), bit for bit.)"""
  stage = _msc_stage_arg(stage)
  M = _msc_dims(packed, psi)[3]
  return mscc_params(packed, (0, M), y_hat, psi, None, stage, num_scales)


def msc_phases(hs, ws, M):
  """positions and widths [images, 4] of the multistage coding order for substream_layout: per image its positions
  of stages 0 to 3, M symbols each."""
  return context_phases((M,), hs, ws, multistage=True)


def msc_substreams(hs, ws, M, substreams):
  """(stream_lengths, phase_lengths) of substream_layout for the multistage coding order of images of latent shapes
  hs[i] x ws[i] and depth M, four phases per image."""
  return context_substreams((M,), hs, ws, substreams, multistage=True)


def msc_encode(packed, y, psi, num_scales, scale_index=False, substreams=1):
  """The four-pass encoder: returns y_hat [B, H, W, M] and y, loc, index in coding order [B, H * W, M] (and
  scale_index last with `scale_index=True`).  y_hat = float(int32(rint(y - loc))) + loc, each stage's before the
  next stage reads it.  The strings are one index-mode encode of the coding-order y with index and loc.  With
  `substreams` = S > 1 the coding-order tensors are rewritten into substream order by one gather (a second one for
  scale_index), ready for compress_ragged with the stream lengths of msc_substreams."""
  S = gen_ops.check_substreams(substreams)
  B, H, W, M, _ = _msc_dims(packed, psi)
  out = mscc_encode([packed], (M,), y, psi, None, num_scales, scale_index, S)
  return out[:1] + tuple(t.view(B, H * W, M) for t in out[1:])


def msc_decode(handle, packed, psi, num_scales, cdf_offset, substreams=1):
  """The four-pass decoder, continuing `handle` (a DecoderHandle of B index-mode strings in coding order): per stage
  its parameters, decode_index_f32 of its positions and their latents to y_hat [B, H, W, M], which it returns.  A
  fixed number of library launches whatever B, H and W (fewer when a stage is empty, at H = 1 or W = 1) and no host
  synchronisation; stream errors surface at entropy_decode_finalize.  With `substreams` = S > 1 the handle holds B S
  substreams (gen_ops.split_substreams) and each stage decodes with one decode_ragged: the same launches."""
  M = _msc_dims(packed, psi)[3]
  return mscc_decode(handle, [packed], (M,), psi, None, num_scales, cdf_offset, gen_ops.check_substreams(substreams))


def _msc_ragged_check(packed, psis):
  """M of a ragged multistage call, with the packed buffer checked."""
  M = _ragged_list(psis)[2]
  _msc_check_packed(packed, M)
  return M


def msc_params_ragged(packed, y_hats, psis, stage, num_scales):
  """msc_params over a list of images of their own shapes in one pass: returns (loc, scale_index, index, lengths),
  flat, image i's n_s,i M values after image i - 1's; `lengths` are the n_s,i M.  y_hats is a list of [H_i, W_i, M]
  (may be None at stage 0).  Image i's values equal msc_params on that image alone, bit for bit."""
  stage = _msc_stage_arg(stage)
  M = _msc_ragged_check(packed, psis)
  return mscc_params_ragged(packed, (0, M), y_hats, psis, None, stage, num_scales)


def msc_encode_ragged(packed, ys, psis, num_scales, scale_index=False, substreams=1):
  """msc_encode of a list of images of their own shapes, one four-pass sequence for the whole list: returns (y_hats,
  y, loc, index, lengths), and scale_index last with `scale_index=True`.  y, loc and index are flat in coding order,
  image i's H_i W_i M values (its `lengths` entry) after image i - 1's.  With `substreams` = S > 1 they are in
  substream order (one gather, a second one for scale_index) and `lengths` holds the n S stream lengths, image i's
  substream s at i S + s."""
  S = gen_ops.check_substreams(substreams)
  M = _msc_ragged_check(packed, psis)
  return mscc_encode_ragged([packed], (M,), ys, psis, None, num_scales, scale_index, S)


def msc_decode_ragged(handle, packed, psis, num_scales, cdf_offset, substreams=1):
  """msc_decode of a list of images of their own shapes, continuing `handle` (one index-mode string per image, or S
  substreams per image): per stage one ragged parameter pass, one decode_ragged and one scatter for the whole list.
  Returns the list of y_hat [H_i, W_i, M].  The library launches do not depend on the images' number or shapes
  (fewer when a stage is empty in every image); no host synchronisation."""
  M = _msc_ragged_check(packed, psis)
  return mscc_decode_ragged(handle, [packed], (M,), psis, None, num_scales, cdf_offset,
                            gen_ops.check_substreams(substreams))


# ------------------------------------------------------------------------------------------------
# Space-channel multistage context model (DESIGN §3.17): the space-channel model's channel groups (scc_spans), each
# coded in the four stages of the multistage schedule (tfcb_mscc_*).  Group k has its own packed network
# (mscc_pack_weights): a context kernel per stage 1-3 over its own c_k channels, and three 1x1 layers shared by its
# stages whose layer 1 reads [psi, the channel context of group k (none for k = 0), its spatial context].  Coding
# order: per image, group 0's stages 0, 1, 2, 3, then group 1's, ..., each stage in raster order with c_k channels
# per position; the coding-order tensors are [B, H * W * M].  The multistage model (msc_*) is the one group (M,).
# ------------------------------------------------------------------------------------------------
def mscc_layout(M, group):
  """The library's packed layout of group (offset, channels) of a depth-M latent: a dict of the widths K1, N3, N4,
  the offsets of wc1, bc1, wc2, bc2, wc3, bc3, w1, b1, w2, b2, w3, b3 and the `total` floats."""
  o, c = (int(v) for v in group)
  out = (C.c_int64 * 15)()
  n = int(_lib.lib().tfcb_mscc_packed_floats(int(M), o, c, out))
  if n < 0:
    raise _lib.InvalidArgumentError(f"group of {c} channels at offset {o} of a latent of depth M={M}: M must be a "
                                    "positive even number at most 1024, with every channel inside it")
  keys = ("K1", "N3", "N4", "wc1", "bc1", "wc2", "bc2", "wc3", "bc3", "w1", "b1", "w2", "b2", "w3", "b3")
  return dict(zip(keys, (int(v) for v in out)), total=n)


_PACKERS = {scc_layout: "scc_pack_weights", mscc_layout: "mscc_pack_weights"}


def mscc_pack_weights(M, group, ctx_kernels, ctx_biases, w1, b1, w2, b2, w3, b3):
  """The device layout of group (offset, channels)'s four passes: for stages 1, 2 and 3 the taps of its context
  kernel [5, 5, c, 2c] (masked or not: no other tap is read), gathered as [T_s, c, 2c], and its bias [2c]; then the
  group's 1x1 layers as [inputs, outputs] and their biases, with the widths mscc_layout gives.  Returns float32
  [total] on the kernels' device."""
  o, c = (int(v) for v in group)
  lay = mscc_layout(M, group)
  ctx_kernels, ctx_biases = list(ctx_kernels), list(ctx_biases)
  if len(ctx_kernels) != 3 or len(ctx_biases) != 3:
    raise _lib.InvalidArgumentError("one context kernel and one bias for each of stages 1, 2 and 3")
  ops = _ms_operands(c, lay["K1"], ctx_kernels, ctx_biases, (w1, b1, w2, b2, w3, b3), f"group ({o}, {c}) of M={M}")
  packed = torch.empty(lay["total"], dtype=torch.float32, device=ops[0].device)
  check(_lib.lib().tfcb_mscc_pack_weights(int(M), o, c, *[_p(t) for t in ops], _p(packed), lay["total"], _stream()))
  return packed


def _mscc_pass(packed, group, y_hat, psi, ch_ctx, stage, num_scales, whole, loc, scale, index, y=None, y_cc=None,
               y_hat_out=None):
  B, H, W, M, o, c, n = _scc_dims(packed, group, psi, mscc_layout)
  lib = _lib.lib()
  nw = int(lib.tfcb_mscc_workspace_floats(M, o, c, B, H, W, int(stage)))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=packed.device)
  check(lib.tfcb_mscc_params(_p(packed), n, M, o, c, _p(y_hat), _p(psi), _p(ch_ctx), B, H, W, int(stage),
                             int(num_scales), _p(work), nw, int(whole), _p(loc), _p(scale), _p(index), _p(y), _p(y_cc),
                             _p(y_hat_out), _stream()))


def mscc_params(packed, group, y_hat, psi, ch_ctx, stage, num_scales):
  """One parameter pass of group (offset, channels): (loc, scale_index, index) [B, n_s, c] (float32, float32, int32)
  of the n_s positions of stage `stage` of every image, in coding order.  ch_ctx [B, H, W, 2c] is the group's
  channel context (None at offset 0); stages 1-3 read the group's channels of the earlier stages' positions of y_hat
  [B, H, W, M] (y_hat may be None at stage 0).  Row b depends only on image b."""
  stage = _msc_stage_arg(stage)
  B, H, W, M, o, c, _ = _scc_dims(packed, group, psi, mscc_layout)
  dev = packed.device
  psi = _ar_tensor(psi, "psi", (B, H, W, 2 * M), dev)
  ch_ctx = _scc_ch_ctx(ch_ctx, group, (B, H, W), dev)
  if y_hat is not None or stage:
    y_hat = _ar_tensor(y_hat, "y_hat", (B, H, W, M), dev)
  n = msc_counts(H, W)[stage]
  loc = torch.empty((B, n, c), dtype=torch.float32, device=dev)
  scale = torch.empty_like(loc)
  index = torch.empty((B, n, c), dtype=torch.int32, device=dev)
  _mscc_pass(packed, group, y_hat, psi, ch_ctx, stage, num_scales, False, loc, scale, index)
  return loc, scale, index


def mscc_encode(packed, groups, y, psi, channel_context, num_scales, scale_index=False, substreams=1):
  """The group-by-group, stage-by-stage encoder: `packed` holds one mscc_pack_weights buffer per group.  Per group k,
  its channel context `channel_context(k, y_hat)` [B, H, W, 2c_k] (called for k >= 1, once y_hat holds groups 0 to
  k - 1), then its stages 0 to 3.  Returns y_hat [B, H, W, M] and y, loc, index in coding order [B, H * W * M] (and
  scale_index last with `scale_index=True`).  y_hat = float(int32(rint(y - loc))) + loc.  The strings are one
  index-mode encode of the coding-order y with index and loc.  With `substreams` = S > 1 the coding-order tensors
  are rewritten into substream order (4K phases per image), ready for compress_ragged with the stream lengths of
  context_substreams(groups, ..., multistage=True)."""
  S = gen_ops.check_substreams(substreams)
  B, H, W, M, spans, psi = _scc_batch(packed, groups, psi, mscc_layout)
  dev = psi.device
  y = _ar_tensor(y, "y", (B, H, W, M), dev)
  y_hat = torch.empty((B, H, W, M), dtype=torch.float32, device=dev)
  y_cc, loc = (torch.empty((B, H * W * M), dtype=torch.float32, device=dev) for _ in range(2))
  index = torch.empty((B, H * W * M), dtype=torch.int32, device=dev)
  scale = torch.empty_like(loc) if scale_index else None
  for k, (p, g) in enumerate(zip(packed, spans)):
    ch = _scc_ch_ctx(channel_context(k, y_hat) if k else None, g, (B, H, W), dev)
    for stage in range(4):
      _mscc_pass(p, g, y_hat, psi, ch, stage, num_scales, True, loc, scale, index, y, y_cc, y_hat)
  return (y_hat,) + _to_substreams(groups, [H] * B, [W] * B, S, y_cc, loc, index, scale, multistage=True)


def mscc_decode(handle, packed, groups, psi, channel_context, num_scales, cdf_offset, substreams=1):
  """The group-by-group, stage-by-stage decoder, continuing `handle` (a DecoderHandle of B index-mode strings in
  coding order, or B S substreams): per group its channel context (as in mscc_encode), then per stage the parameter
  pass, one decode call and the scatter into y_hat [B, H, W, M], which it returns.  4K decode calls on the handle;
  per group a fixed number of library launches whatever B, H and W (fewer when a stage is empty, at H = 1 or W = 1),
  and no host synchronisation; stream errors surface at entropy_decode_finalize."""
  B, H, W, M, spans, psi = _scc_batch(packed, groups, psi, mscc_layout)
  dev = psi.device
  phases = _substream_phases(handle, groups, [H] * B, [W] * B, substreams, multistage=True)
  coff = _i32(cdf_offset, dev)
  y_hat = torch.zeros((B, H, W, M), dtype=torch.float32, device=dev)
  lib = _lib.lib()
  for k, (p, (o, c)) in enumerate(zip(packed, spans)):
    ch = channel_context(k, y_hat) if k else None
    for stage in range(4):
      loc, _, index = mscc_params(p, (o, c), y_hat, psi, ch, stage, num_scales)
      part = _decode_phase(handle, phases, 4 * k + stage, index, loc, coff)
      check(lib.tfcb_mscc_scatter(_p(part), B, H, W, M, o, c, stage, _p(y_hat), _stream()))
  return y_hat


def _mscc_pass_ragged(packed, group, M, hs, ws, y_hat, psi, ch_ctx, stage, num_scales, whole=False, loc=None,
                      scale=None, index=None, y=None, y_cc=None, y_hat_out=None):
  """One stage of group (offset, channels) over the flat list.  Per-stage outputs (whole False, loc None) are
  allocated: returns (loc, scale_index, index, lengths, work) with image i's n_s,i c values at c Q_i; the workspace
  holds the image table for the scatter."""
  o, c = (int(v) for v in group)
  n = _scc_check_packed(packed, M, group, mscc_layout)
  dev = packed.device
  lib = _lib.lib()
  k = hs.size
  a, b = MSC_PHASES[stage]
  counts = ((hs - a + 1) // 2) * ((ws - b + 1) // 2)
  if loc is None:
    total = int(counts.sum()) * c
    loc, scale = (torch.empty(total, dtype=torch.float32, device=dev) for _ in range(2))
    index = torch.empty(total, dtype=torch.int32, device=dev)
  nw = int(lib.tfcb_mscc_ragged_workspace_floats(M, o, c, k, _host(hs), _host(ws), int(stage)))
  work = torch.empty(max(nw, 1), dtype=torch.float32, device=dev)
  check(lib.tfcb_mscc_params_ragged(_p(packed), n, M, o, c, _p(y_hat), _p(psi), _p(ch_ctx), k, _host(hs), _host(ws),
                                    int(stage), int(num_scales), _p(work), nw, int(whole), _p(loc), _p(scale),
                                    _p(index), _p(y), _p(y_cc), _p(y_hat_out), _stream()))
  return loc, scale, index, (counts * c).tolist(), work


def mscc_params_ragged(packed, group, y_hats, psis, ch_ctx, stage, num_scales):
  """mscc_params over a list of images of their own shapes in one pass: returns (loc, scale_index, index, lengths),
  flat, image i's n_s,i c values after image i - 1's; `lengths` are the n_s,i c.  ch_ctx is a list of [H_i, W_i, 2c]
  (None at offset 0); y_hats a list of [H_i, W_i, M] (may be None at stage 0).  Image i's values equal mscc_params
  on that image alone, bit for bit."""
  stage = _msc_stage_arg(stage)
  hs, ws, M = _ragged_list(psis)
  _scc_check_packed(packed, M, group, mscc_layout)
  dev = packed.device
  psi = _ragged_cat(psis, "psi", hs, ws, 2 * M, dev)
  ch = _scc_ch_ctx_ragged(ch_ctx, group, hs, ws, dev)
  y_hat = None if y_hats is None and not stage else _ragged_cat(y_hats, "y_hat", hs, ws, M, dev)
  return _mscc_pass_ragged(packed, group, M, hs, ws, y_hat, psi, ch, stage, num_scales)[:4]


def mscc_encode_ragged(packed, groups, ys, psis, channel_context, num_scales, scale_index=False, substreams=1):
  """mscc_encode of a list of images of their own shapes, one pass sequence for the whole list: returns (y_hats, y,
  loc, index, lengths), and scale_index last with `scale_index=True`.  `channel_context(k, y_hats)` takes and
  returns lists ([H_i, W_i, 2c_k] per image).  y, loc and index are flat in coding order, image i's H_i W_i M values
  (its `lengths` entry) after image i - 1's.  With `substreams` = S > 1 they are in substream order and `lengths`
  holds the n S stream lengths, image i's substream s at i S + s."""
  S = gen_ops.check_substreams(substreams)
  hs, ws, M, spans, psi = _scc_ragged(packed, groups, psis, mscc_layout)
  dev = psi.device
  y = _ragged_cat(ys, "y", hs, ws, M, dev)
  y_hat, y_cc, loc = (torch.empty_like(y) for _ in range(3))
  index = torch.empty(y.shape, dtype=torch.int32, device=dev)
  scale = torch.empty_like(y) if scale_index else None
  views = _ragged_views(y_hat, hs, ws, M)
  for k, (p, g) in enumerate(zip(packed, spans)):
    ch = _scc_ch_ctx_ragged(channel_context(k, views) if k else None, g, hs, ws, dev)
    for stage in range(4):
      _mscc_pass_ragged(p, g, M, hs, ws, y_hat, psi, ch, stage, num_scales, True, loc, scale, index, y, y_cc, y_hat)
  out = _to_substreams(groups, hs, ws, S, y_cc, loc, index, scale, multistage=True)
  lengths = (hs * ws * M).tolist() if S == 1 else context_substreams(groups, hs, ws, S, multistage=True)[0].tolist()
  return (views,) + out[:3] + (lengths,) + out[3:]


def mscc_decode_ragged(handle, packed, groups, psis, channel_context, num_scales, cdf_offset, substreams=1):
  """mscc_decode of a list of images of their own shapes, continuing `handle` (one index-mode string per image, or S
  substreams per image): per group its channel context (as in mscc_encode_ragged), then per stage one ragged
  parameter pass, one decode_ragged and one scatter for the whole list.  Returns the list of y_hat [H_i, W_i, M].
  The library launches depend on the groups, not on the images' number or shapes (fewer when a stage is empty in
  every image); no host synchronisation."""
  hs, ws, M, spans, psi = _scc_ragged(packed, groups, psis, mscc_layout)
  dev = psi.device
  phases = _substream_phases(handle, groups, hs, ws, substreams, "list", multistage=True)
  coff = _i32(cdf_offset, dev)
  y_hat = torch.zeros(int((hs * ws).sum()) * M, dtype=torch.float32, device=dev)
  views = _ragged_views(y_hat, hs, ws, M)
  lib = _lib.lib()
  for k, (p, (o, c)) in enumerate(zip(packed, spans)):
    ch = _scc_ch_ctx_ragged(channel_context(k, views) if k else None, (o, c), hs, ws, dev)
    for stage in range(4):
      loc, _, index, lengths, work = _mscc_pass_ragged(p, (o, c), M, hs, ws, y_hat, psi, ch, stage, num_scales)
      if phases is not None:
        lengths = phases[4 * k + stage]
      part = decode_ragged(handle, lengths, index=index, quant_offset=loc, cdf_offset=coff)
      check(lib.tfcb_mscc_scatter_ragged(_p(part), hs.size, _host(hs), _host(ws), M, o, c, stage, _p(work),
                                         work.numel(), _p(y_hat), _stream()))
  return views
