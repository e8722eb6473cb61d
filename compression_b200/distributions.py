"""Priors used to derive range-coding tables, mirroring tensorflow_compression/python/distributions:
helpers.py:29-219 (tail / offset estimation), deep_factorized.py:50-267, uniform_noise.py:50-262 and
round_adapters.py:36-288.
TensorFlow Probability is replaced by a minimal scalar-distribution protocol on PyTorch:
``cdf / survival_function / log_cdf / log_survival_function / quantile / batch_shape / dtype``."""
import math

import torch
from torch import nn

__all__ = [
    "estimate_tails", "quantization_offset", "lower_tail", "upper_tail", "DeepFactorized",
    "NoisyDeepFactorized", "UniformNoiseAdapter", "Normal", "Laplace", "Logistic", "NoisyNormal",
    "NoisyLaplace", "NoisyLogistic", "MonotonicAdapter", "RoundAdapter", "NoisyRoundAdapter",
    "NoisyRoundedNormal", "NoisyRoundedDeepFactorized", "SoftRoundAdapter", "NoisySoftRoundAdapter",
    "NoisySoftRoundedNormal", "NoisySoftRoundedDeepFactorized", "MixtureSameFamily", "NoisyMixtureSameFamily",
    "NoisyNormalMixture", "NoisyLogisticMixture",
]


# ------------------------------------------------------------------------------------------------
# helpers.py
# ------------------------------------------------------------------------------------------------
def estimate_tails(func, target, shape, dtype=torch.float32, device=None, check_every=16):
  """Adam-style root finding of func(x) == target (helpers.py:29-102), vectorised over `shape`.

  The reference's `tf.while_loop` condition (max loss > 1e-8 and min count < 100) is evaluated on the device: the
  loop state is frozen by a 0-d `active` flag once the condition turns false, and the host looks at that flag only
  every `check_every` iterations -- the result is the one of the sequential loop, without two host round trips
  per iteration (the loop runs 100-300 iterations per table build)."""
  shape = tuple(int(s) for s in shape)
  target = torch.as_tensor(target, dtype=dtype, device=device)
  tails = torch.zeros(shape, dtype=dtype, device=device)
  if tails.numel() == 0:
    return tails
  m = torch.zeros_like(tails)
  v = torch.ones_like(tails)
  loss = torch.full_like(tails, torch.finfo(dtype).max)
  count = torch.zeros(shape, dtype=torch.int32, device=tails.device)
  best_tails, best_loss = tails.clone(), loss.clone()
  active = torch.ones((), dtype=torch.bool, device=tails.device)
  keep = lambda new, old: torch.where(active, new, old)
  while True:
    for _ in range(check_every):
      active = active & (loss.max() > 1e-8) & (count.min() < 100)  # loop_cond, helpers.py:61-66
      t = tails.detach().requires_grad_(True)
      with torch.enable_grad():
        new_loss = (func(t) - target).abs()
        grad, = torch.autograd.grad(new_loss.sum(), t)
      new_loss = new_loss.detach()
      better = active & (new_loss < best_loss)
      best_tails = torch.where(better, tails, best_tails)
      best_loss = torch.where(better, new_loss, best_loss)
      new_m = (m + grad) / 2
      new_v = (v + grad.square()) / 2
      k = torch.sqrt((count + 1).to(dtype))
      new_tails = tails - 0.1 * new_m / (k * torch.sqrt(new_v) + 1e-20)
      new_count = torch.where((count > 0) | (m * grad < 0), count + 1, count)
      tails, m, v, loss, count = (keep(new_tails, tails), keep(new_m, m), keep(new_v, v), keep(new_loss, loss),
                                  keep(new_count, count))
    if not bool(active):  # the only host synchronisation
      break
  return best_tails


def quantization_offset(distribution):
  """helpers.py:104-147: offset - round(offset) of the best available location statistic."""
  offset = None
  for name in ("_quantization_offset", "mode", "median", "mean"):
    fn = getattr(distribution, name, None)
    if fn is None:
      continue
    try:
      offset = fn()
      break
    except NotImplementedError:
      continue
  if offset is None:
    offset = torch.zeros((), dtype=distribution.dtype)
  offset = torch.as_tensor(offset).detach()
  return offset - torch.round(offset)


def _tail(distribution, tail_mass, lower):
  own = getattr(distribution, "_lower_tail" if lower else "_upper_tail", None)
  if own is not None:
    try:
      return own(tail_mass).detach()
    except NotImplementedError:
      pass
  try:
    q = tail_mass / 2 if lower else 1 - tail_mass / 2
    return distribution.quantile(q).detach()
  except NotImplementedError:
    pass
  fn = getattr(distribution, "log_cdf" if lower else "log_survival_function", None)
  if fn is None:
    raise NotImplementedError(
        "`distribution` must implement `_lower_tail()`/`_upper_tail()`, `quantile()`, or "
        "`log_cdf()`/`log_survival_function()` so that the tails can be located.")
  target = math.log(tail_mass / 2)
  return estimate_tails(fn, target, distribution.batch_shape, distribution.dtype,
                        getattr(distribution, "device", None)).detach()


def lower_tail(distribution, tail_mass):
  """helpers.py:150-183."""
  return _tail(distribution, tail_mass, True)


def upper_tail(distribution, tail_mass):
  """helpers.py:186-219."""
  return _tail(distribution, tail_mass, False)


# ------------------------------------------------------------------------------------------------
# deep_factorized.py
# ------------------------------------------------------------------------------------------------
def _log_expm1(x):
  x = torch.as_tensor(x, dtype=torch.float64)
  return torch.where(x < 15.0, torch.log(torch.expm1(torch.clamp(x, max=15.0))), x)


class DeepFactorized(nn.Module):
  """Fully factorized density with a small monotone MLP per channel as CDF logits
  (deep_factorized.py:50-260)."""

  def __init__(self, batch_shape=(), num_filters=(3, 3), init_scale=10, dtype=torch.float32, device=None):
    super().__init__()
    self._batch_shape = tuple(int(s) for s in batch_shape)
    self.num_filters = tuple(int(f) for f in num_filters)
    self.init_scale = float(init_scale)
    self.dtype = dtype
    channels = 1
    for s in self._batch_shape:
      channels *= s
    self._channels = channels
    filters = (1,) + self.num_filters + (1,)
    scale = self.init_scale**(1 / (len(self.num_filters) + 1))
    self.matrices = nn.ParameterList()
    self.biases = nn.ParameterList()
    self.factors = nn.ParameterList()
    for i in range(len(self.num_filters) + 1):
      init = float(_log_expm1(1 / scale / filters[i + 1]))
      self.matrices.append(nn.Parameter(
          torch.full((channels, filters[i + 1], filters[i]), init, dtype=dtype, device=device)))
      self.biases.append(nn.Parameter(
          torch.rand((channels, filters[i + 1], 1), dtype=dtype, device=device) - 0.5))
      if i < len(self.num_filters):
        self.factors.append(nn.Parameter(torch.zeros((channels, filters[i + 1], 1), dtype=dtype, device=device)))

  @property
  def batch_shape(self):
    return self._batch_shape

  @property
  def device(self):
    return self.matrices[0].device

  def _broadcast(self, inputs):
    inputs = torch.as_tensor(inputs, dtype=self.dtype, device=self.device)
    shape = torch.broadcast_shapes(tuple(inputs.shape), self._batch_shape)
    return inputs.expand(shape)

  def _logits_cumulative(self, inputs):
    """deep_factorized.py:166-193."""
    inputs = self._broadcast(inputs)
    shape = inputs.shape
    x = inputs.reshape(-1, 1, self._channels).permute(2, 1, 0)  # (channels, 1, batch)
    logits = x
    for i in range(len(self.num_filters) + 1):
      logits = torch.matmul(torch.nn.functional.softplus(self.matrices[i]), logits) + self.biases[i]
      if i < len(self.num_filters):
        logits = logits + torch.tanh(self.factors[i]) * torch.tanh(logits)
    return logits.permute(2, 1, 0).reshape(shape)

  def _packed_parameters(self):
    """[channels, P]: softplus(matrices), biases, tanh(factors), each flattened row-major per channel, in that
    order -- the layout of the fused log-likelihood kernels (P = 28 for num_filters (3, 3)).  Built with torch
    operations, so gradients reach the raw parameters through autograd."""
    C = self._channels
    return torch.cat([torch.nn.functional.softplus(m).reshape(C, -1) for m in self.matrices] +
                     [b.reshape(C, -1) for b in self.biases] + [torch.tanh(f).reshape(C, -1) for f in self.factors],
                     dim=1)

  def log_cdf(self, x):
    return torch.nn.functional.logsigmoid(self._logits_cumulative(x))

  def log_survival_function(self, x):
    return torch.nn.functional.logsigmoid(-self._logits_cumulative(x))

  def cdf(self, x):
    return torch.sigmoid(self._logits_cumulative(x))

  def survival_function(self, x):
    return torch.sigmoid(-self._logits_cumulative(x))

  def _live(self, x):
    """The point the density is differentiated at: x itself when it is already part of a graph (so the density
    stays differentiable in x, deep_factorized.py:195-230), else a fresh leaf."""
    x = self._broadcast(x)
    return x if (torch.is_grad_enabled() and x.requires_grad) else x.detach().requires_grad_(True)

  def prob(self, x):
    keep = torch.is_grad_enabled()
    x = self._live(x)
    with torch.enable_grad():
      c = self.cdf(x)
      p, = torch.autograd.grad(c.sum(), x, create_graph=keep)
    return p

  def log_prob(self, x):
    keep = torch.is_grad_enabled()
    x = self._live(x)
    with torch.enable_grad():
      logits = self._logits_cumulative(x)
      dlogits, = torch.autograd.grad(logits.sum(), x, create_graph=keep)
      out = torch.nn.functional.logsigmoid(logits) + torch.nn.functional.logsigmoid(-logits) + torch.log(dlogits)
    return out if keep else out.detach()

  def quantile(self, q):
    raise NotImplementedError

  # no closed forms for these either (deep_factorized.py leaves the tfp defaults, which raise)
  def mean(self):
    raise NotImplementedError

  def mode(self):
    raise NotImplementedError

  def sample(self, sample_shape=(), generator=None):
    raise NotImplementedError

  def _quantization_offset(self):
    return estimate_tails(self._logits_cumulative, 0., self._batch_shape, self.dtype, self.device)

  def _lower_tail(self, tail_mass):
    logits = math.log(tail_mass / 2 / (1. - tail_mass / 2))
    return estimate_tails(self._logits_cumulative, logits, self._batch_shape, self.dtype, self.device)

  def _upper_tail(self, tail_mass):
    logits = -math.log(tail_mass / 2 / (1. - tail_mass / 2))
    return estimate_tails(self._logits_cumulative, logits, self._batch_shape, self.dtype, self.device)


# ------------------------------------------------------------------------------------------------
# Closed-form location-scale bases (stand-ins for tfp.distributions.{Normal,Laplace,Logistic})
# ------------------------------------------------------------------------------------------------
class _LocScale:

  def __init__(self, loc, scale, dtype=torch.float32):
    loc = torch.as_tensor(loc, dtype=dtype)
    scale = torch.as_tensor(scale, dtype=dtype, device=loc.device if loc.dim() else None)
    if scale.device != loc.device:
      loc = loc.to(scale.device)
    self.loc, self.scale = torch.broadcast_tensors(loc, scale)
    self.dtype = self.loc.dtype

  @property
  def batch_shape(self):
    return tuple(self.loc.shape)

  @property
  def device(self):
    return self.loc.device

  def _z(self, x):
    x = torch.as_tensor(x, dtype=self.dtype, device=self.device)
    return (x - self.loc) / self.scale

  def mean(self):
    return self.loc

  def mode(self):
    return self.loc

  def survival_function(self, x):
    return self._std_cdf(-self._z(x))

  def cdf(self, x):
    return self._std_cdf(self._z(x))

  def log_cdf(self, x):
    return self._std_log_cdf(self._z(x))

  def log_survival_function(self, x):
    return self._std_log_cdf(-self._z(x))

  def quantile(self, q):
    q = torch.as_tensor(q, dtype=self.dtype, device=self.device)
    return self.loc + self.scale * self._std_quantile(q)

  def sample(self, sample_shape=(), generator=None):
    """Inverse-CDF sampling; shape sample_shape + batch_shape."""
    shape = tuple(sample_shape) + self.batch_shape
    u = torch.rand(shape, dtype=self.dtype, device=self.device, generator=generator)
    tiny = torch.finfo(self.dtype).tiny
    return self.quantile(u.clamp(tiny, 1 - torch.finfo(self.dtype).eps / 2))


def _float32_on_cpu(fn):
  """torch's CPU kernels of the ndtr family have no float16 / bfloat16 variants (the CUDA ones do): 16-bit inputs on
  the CPU go through float32 and come back in their own dtype."""

  def wrapped(z):
    if z.device.type == "cpu" and z.dtype in (torch.float16, torch.bfloat16):
      return fn(z.float()).to(z.dtype)
    return fn(z)

  return staticmethod(wrapped)


class Normal(_LocScale):
  _std_cdf = _float32_on_cpu(torch.special.ndtr)
  _std_log_cdf = _float32_on_cpu(torch.special.log_ndtr)
  _std_quantile = _float32_on_cpu(torch.special.ndtri)


class Logistic(_LocScale):
  _std_cdf = staticmethod(torch.sigmoid)
  _std_log_cdf = staticmethod(torch.nn.functional.logsigmoid)
  _std_quantile = staticmethod(torch.logit)


class Laplace(_LocScale):

  @staticmethod
  def _std_cdf(z):
    return 0.5 - 0.5 * torch.sign(z) * torch.expm1(-z.abs())

  @staticmethod
  def _std_log_cdf(z):
    return torch.where(z < 0, math.log(0.5) + z, torch.log1p(-0.5 * torch.exp(-z.abs())))

  @staticmethod
  def _std_quantile(q):
    return torch.where(q < 0.5, torch.log(2 * q), -torch.log(2 * (1 - q)))


# ------------------------------------------------------------------------------------------------
# uniform_noise.py
# ------------------------------------------------------------------------------------------------
def _logsum_expbig_minus_expsmall(big, small):
  return torch.where(torch.isinf(big), big, torch.log1p(-torch.exp(small - big)) + big)


_LOC_SCALE_KINDS = {Normal: "normal", Logistic: "logistic", Laplace: "laplace"}


def _fused_log_prob_form(base, y):
  """Which fused kernel computes UniformNoiseAdapter(base).log_prob(y), judged from dtypes and shapes alone:
  "deep_factorized", "normal", "logistic", "laplace" or None (the graph).
    * DeepFactorized with num_filters (3, 3): y contiguous with trailing dimensions equal to the batch shape, so the
      channel of element i is i mod prod(batch_shape);
    * Normal / Logistic / Laplace: loc and scale each y-shaped and contiguous, or a broadcast scalar (every stride
      0, as `_LocScale`'s broadcast_tensors hands over a scalar);
  everything float32."""
  if not isinstance(y, torch.Tensor) or y.dtype != torch.float32:
    return None
  if type(base) is DeepFactorized:
    k = len(base.batch_shape)
    params = list(base.matrices) + list(base.biases) + list(base.factors)
    if (base.num_filters != (3, 3) or any(p.dtype != torch.float32 for p in params) or not y.is_contiguous() or
        y.dim() < k or tuple(y.shape[y.dim() - k:]) != base.batch_shape):
      return None
    return "deep_factorized"
  kind = _LOC_SCALE_KINDS.get(type(base))
  if kind is None:
    return None
  for t in (base.loc, base.scale):
    if (t.dtype != torch.float32 or tuple(t.shape) != tuple(y.shape) or
        not (t.is_contiguous() or all(s == 0 for s in t.stride()))):
      return None
  return kind


def _fused_log_prob_kind(base, y):
  """The routing of UniformNoiseAdapter.log_prob: `_fused_log_prob_form` on CUDA tensors of one device, else None."""
  kind = _fused_log_prob_form(base, y)
  if kind is None or y.device.type != "cuda":
    return None
  tensors = ((base.loc, base.scale) if kind != "deep_factorized" else
             list(base.matrices) + list(base.biases) + list(base.factors))
  return kind if all(t.device == y.device for t in tensors) else None


class UniformNoiseAdapter(nn.Module):
  """p(y) = c(y + .5) - c(y - .5) of a base density (uniform_noise.py:50-191)."""

  def __init__(self, base):
    super().__init__()
    self.base = base

  @property
  def dtype(self):
    return self.base.dtype

  @property
  def batch_shape(self):
    return self.base.batch_shape

  @property
  def device(self):
    return self.base.device

  def log_prob(self, y):
    """uniform_noise.py:128-151.  float32 CUDA priors of the forms `_fused_log_prob_kind` accepts run the fused
    kernels (forward and backward, `functional.noisy_*_log_prob`); everything else runs the graph."""
    kind = _fused_log_prob_kind(self.base, y)
    if kind is None:
      return self._log_prob_graph(y)
    from compression_b200 import functional
    if kind == "deep_factorized":
      return functional.noisy_deep_factorized_log_prob(y, self.base._packed_parameters())
    return functional.noisy_loc_scale_log_prob(kind, y, self.base.loc, self.base.scale)

  def _log_prob_graph(self, y):
    """The log-sf / log-cdf select as a graph of torch operations (any device and dtype)."""
    b = self.base
    logsf_p, logsf_m = b.log_survival_function(y + .5), b.log_survival_function(y - .5)
    logcdf_p, logcdf_m = b.log_cdf(y + .5), b.log_cdf(y - .5)
    right = logsf_p < logcdf_p
    big = torch.where(right, logsf_m, logcdf_p)
    small = torch.where(right, logsf_p, logcdf_m)
    return _logsum_expbig_minus_expsmall(big, small)

  def prob(self, y):
    """uniform_noise.py:171-183."""
    b = self.base
    sf_p, sf_m = b.survival_function(y + .5), b.survival_function(y - .5)
    cdf_p, cdf_m = b.cdf(y + .5), b.cdf(y - .5)
    return torch.where(sf_p < cdf_p, sf_m - sf_p, cdf_p - cdf_m)

  def mean(self):
    return self.base.mean()

  def sample(self, sample_shape=(), generator=None):
    """base sample + U(-.5, .5) (uniform_noise.py:103-112)."""
    x = self.base.sample(sample_shape, generator=generator)
    return x + torch.rand(x.shape, dtype=x.dtype, device=x.device, generator=generator) - .5

  # the noisy density has no closed-form mode / quantile / survival function (uniform_noise.py leaves the tfp
  # defaults, which raise)
  def mode(self):
    raise NotImplementedError("mode is not implemented for UniformNoiseAdapter")

  def quantile(self, value):
    raise NotImplementedError("quantile is not implemented for UniformNoiseAdapter")

  def survival_function(self, y):
    raise NotImplementedError("survival_function is not implemented for UniformNoiseAdapter")

  def _quantization_offset(self):
    return quantization_offset(self.base)

  def _lower_tail(self, tail_mass):
    return lower_tail(self.base, tail_mass)

  def _upper_tail(self, tail_mass):
    return upper_tail(self.base, tail_mass)


class NoisyDeepFactorized(UniformNoiseAdapter):
  """deep_factorized.py:263-267."""

  def __init__(self, **kwargs):
    super().__init__(DeepFactorized(**kwargs))


class NoisyNormal(UniformNoiseAdapter):
  """uniform_noise.py:257-262."""

  def __init__(self, loc, scale, dtype=torch.float32):
    super().__init__(Normal(loc, scale, dtype))


class NoisyLogistic(UniformNoiseAdapter):

  def __init__(self, loc, scale, dtype=torch.float32):
    super().__init__(Logistic(loc, scale, dtype))


class NoisyLaplace(UniformNoiseAdapter):

  def __init__(self, loc, scale, dtype=torch.float32):
    super().__init__(Laplace(loc, scale, dtype))


class MixtureSameFamily:
  """Stand-in for `tfp.distributions.MixtureSameFamily` over a scalar family: `probs[..., K]` weights the K
  components held in the last batch axis of `components`; that axis is summed out."""

  def __init__(self, probs, components):
    self.components = components
    self.dtype = components.dtype
    self.probs = torch.as_tensor(probs, dtype=self.dtype, device=components.device)
    full = torch.broadcast_shapes(tuple(self.probs.shape), tuple(components.batch_shape))
    self._batch_shape = tuple(full[:-1])

  @property
  def batch_shape(self):
    return self._batch_shape

  @property
  def device(self):
    return self.components.device

  def _x(self, x):
    return torch.as_tensor(x, dtype=self.dtype, device=self.device).unsqueeze(-1)

  def cdf(self, x):
    return (self.probs * self.components.cdf(self._x(x))).sum(-1)

  def survival_function(self, x):
    return (self.probs * self.components.survival_function(self._x(x))).sum(-1)

  def log_cdf(self, x):
    return torch.logsumexp(torch.log(self.probs) + self.components.log_cdf(self._x(x)), -1)

  def log_survival_function(self, x):
    return torch.logsumexp(torch.log(self.probs) + self.components.log_survival_function(self._x(x)), -1)

  def mean(self):
    return (self.probs * self.components.mean()).sum(-1)

  def mode(self):
    raise NotImplementedError("mode is not implemented for MixtureSameFamily")

  def quantile(self, value):
    raise NotImplementedError("quantile is not implemented for MixtureSameFamily")

  def sample(self, sample_shape=(), generator=None):
    x = self.components.sample(sample_shape, generator=generator)            # sample_shape + component batch
    comp = tuple(self.components.batch_shape)
    full = self.batch_shape + (max(comp[-1], self.probs.shape[-1]),)
    x = x.reshape(tuple(sample_shape) + (1,) * (len(full) - len(comp)) + comp)
    x = x.expand(tuple(sample_shape) + full)                                 # sample_shape + batch + [K]
    w = self.probs.expand(x.shape).reshape(-1, x.shape[-1])
    k = torch.multinomial(w, 1, generator=generator).reshape(x.shape[:-1] + (1,))
    return torch.gather(x, -1, k).squeeze(-1)


class NoisyMixtureSameFamily(nn.Module):
  """Mixture of distributions with additive uniform noise (uniform_noise.py:200-244): the noise is added to every
  component, tails come from the noiseless mixture, the quantisation offset is that of the component under which
  its own offset is most probable."""

  def __init__(self, mixture_probs, components_distribution):
    super().__init__()
    self.components_distribution = UniformNoiseAdapter(components_distribution)
    self.base = MixtureSameFamily(mixture_probs, components_distribution)

  @property
  def mixture_probs(self):
    return self.base.probs

  @property
  def dtype(self):
    return self.base.dtype

  @property
  def batch_shape(self):
    return self.base.batch_shape

  @property
  def device(self):
    return self.base.device

  def log_prob(self, y):
    y = torch.as_tensor(y, dtype=self.dtype, device=self.device).unsqueeze(-1)
    return torch.logsumexp(torch.log(self.mixture_probs) + self.components_distribution._log_prob_graph(y), -1)

  def prob(self, y):
    y = torch.as_tensor(y, dtype=self.dtype, device=self.device).unsqueeze(-1)
    return (self.mixture_probs * self.components_distribution.prob(y)).sum(-1)

  def mean(self):
    return self.base.mean()

  def sample(self, sample_shape=(), generator=None):
    x = self.base.sample(sample_shape, generator=generator)
    return x + torch.rand(x.shape, dtype=x.dtype, device=x.device, generator=generator) - .5

  def mode(self):
    raise NotImplementedError("mode is not implemented for NoisyMixtureSameFamily")

  def quantile(self, value):
    raise NotImplementedError("quantile is not implemented for NoisyMixtureSameFamily")

  def survival_function(self, y):
    raise NotImplementedError("survival_function is not implemented for NoisyMixtureSameFamily")

  def _quantization_offset(self):
    """uniform_noise.py:231-237."""
    offsets = quantization_offset(self.components_distribution)
    offsets = offsets.expand(self.batch_shape + offsets.shape[-1:])
    at = offsets.movedim(-1, 0)                                # [K] + batch: every component's offset as a point
    component = torch.argmax(self.log_prob(at), dim=0)          # batch
    return torch.gather(offsets, -1, component.unsqueeze(-1)).squeeze(-1)

  def _lower_tail(self, tail_mass):
    return lower_tail(self.base, tail_mass)

  def _upper_tail(self, tail_mass):
    return upper_tail(self.base, tail_mass)


class NoisyNormalMixture(NoisyMixtureSameFamily):
  """uniform_noise.py:268-285."""

  def __init__(self, loc, scale, weight, dtype=torch.float32):
    super().__init__(weight, Normal(loc, scale, dtype))


class NoisyLogisticMixture(NoisyMixtureSameFamily):
  """uniform_noise.py:288-305."""

  def __init__(self, loc, scale, weight, dtype=torch.float32):
    super().__init__(weight, Logistic(loc, scale, dtype))


# ------------------------------------------------------------------------------------------------
# round_adapters.py
# ------------------------------------------------------------------------------------------------
class MonotonicAdapter(nn.Module):
  """A continuous distribution seen through an ascending monotonic function (round_adapters.py:36-147;
  Agustsson & Theis 2020, appendix E): cdf_Y(y) = cdf_X(inverse_transform(y))."""
  invertible = True  # False: quantile / mode / tails of the base cannot be pushed through `transform`

  def __init__(self, base):
    super().__init__()
    self.base = base

  @property
  def dtype(self):
    return self.base.dtype

  @property
  def batch_shape(self):
    return self.base.batch_shape

  @property
  def device(self):
    return self.base.device

  def transform(self, x):
    raise NotImplementedError()

  def inverse_transform(self, y):
    raise NotImplementedError()

  def sample(self, sample_shape=(), generator=None):
    return self.transform(self.base.sample(sample_shape, generator=generator))

  def prob(self, *args, **kwargs):
    raise NotImplementedError

  def log_prob(self, *args, **kwargs):
    raise NotImplementedError

  def _y(self, y):
    return torch.as_tensor(y, dtype=self.dtype, device=self.device)

  def cdf(self, y):
    return self.base.cdf(self.inverse_transform(self._y(y)))

  def log_cdf(self, y):
    return self.base.log_cdf(self.inverse_transform(self._y(y)))

  def survival_function(self, y):
    return self.base.survival_function(self.inverse_transform(self._y(y)))

  def log_survival_function(self, y):
    return self.base.log_survival_function(self.inverse_transform(self._y(y)))

  def _require_invertible(self):
    if not self.invertible:
      raise NotImplementedError()

  def quantile(self, value):
    self._require_invertible()
    return self.transform(self.base.quantile(value))

  def mode(self):
    self._require_invertible()
    return self.transform(self.base.mode())

  def _quantization_offset(self):
    self._require_invertible()
    return self.transform(quantization_offset(self.base))

  def _lower_tail(self, tail_mass):
    self._require_invertible()
    return self.transform(lower_tail(self.base, tail_mass))

  def _upper_tail(self, tail_mass):
    self._require_invertible()
    return self.transform(upper_tail(self.base, tail_mass))


class RoundAdapter(MonotonicAdapter):
  """Continuous density + round (round_adapters.py:150-169): cdf_Y(y) = cdf_X(ceil(y) - 1/2)."""
  invertible = False

  def transform(self, x):
    return torch.round(x)

  def inverse_transform(self, y):
    return torch.ceil(y) - .5

  def _quantization_offset(self):
    return torch.zeros((), dtype=self.dtype)

  def _lower_tail(self, tail_mass):
    return torch.floor(lower_tail(self.base, tail_mass))

  def _upper_tail(self, tail_mass):
    return torch.ceil(upper_tail(self.base, tail_mass))


class NoisyRoundAdapter(UniformNoiseAdapter):
  """Uniform noise + round (round_adapters.py:172-183)."""

  def __init__(self, base):
    super().__init__(RoundAdapter(base))


class NoisyRoundedDeepFactorized(NoisyRoundAdapter):
  """round_adapters.py:186-191."""

  def __init__(self, **kwargs):
    super().__init__(DeepFactorized(**kwargs))


class NoisyRoundedNormal(NoisyRoundAdapter):
  """round_adapters.py:194-198."""

  def __init__(self, loc, scale, dtype=torch.float32):
    super().__init__(Normal(loc, scale, dtype))


class SoftRoundAdapter(MonotonicAdapter):
  """Differentiable approximation of round (round_adapters.py:201-221)."""

  def __init__(self, base, alpha):
    super().__init__(base)
    self._alpha = alpha

  @property
  def alpha(self):
    return self._alpha

  def transform(self, x):
    from compression_b200 import math_ops
    return math_ops.soft_round(x, self._alpha)

  def inverse_transform(self, y):
    from compression_b200 import math_ops
    return math_ops.soft_round_inverse(y, self._alpha)


class NoisySoftRoundAdapter(UniformNoiseAdapter):
  """Uniform noise + soft round (round_adapters.py:224-236)."""

  def __init__(self, base, alpha):
    super().__init__(SoftRoundAdapter(base, alpha))


class NoisySoftRoundedNormal(NoisySoftRoundAdapter):
  """round_adapters.py:239-247."""

  def __init__(self, alpha=5.0, loc=0., scale=1., dtype=torch.float32):
    super().__init__(Normal(loc, scale, dtype), alpha)


class NoisySoftRoundedDeepFactorized(NoisySoftRoundAdapter):
  """round_adapters.py:250-260."""

  def __init__(self, alpha=5.0, **kwargs):
    super().__init__(DeepFactorized(**kwargs), alpha)
