"""GDN layer and its non-negative parameterisation, mirroring tensorflow_compression/python/layers/gdn.py
(:127-175 ctor, :308-334 properties, :336-369 build, :371-421 call, :426-470 config) and
layers/parameters.py:186-269 (GDNParameter).  The normalisation itself runs in the CUDA kernels of
csrc/gdn*.cu through `functional.gdn`."""
import torch
from torch import nn

from compression_b200 import functional as F
from compression_b200.parameters import Parameter
from compression_b200 import math_ops

__all__ = ["GDN", "GDNParameter"]


class GDNParameter(Parameter):
  """theta = max(v, sqrt(minimum + offset^2))^2 - offset^2 (parameters.py:186-269)."""

  def __init__(self, initial_value, name=None, minimum=0., offset=2**-18, shape=None, dtype=None):
    super().__init__()
    self._minimum = float(minimum)
    self._offset = float(offset)
    self.name = name
    if initial_value is None:
      if shape is None:
        raise ValueError("If initial_value is None, shape must be specified.")
      initial_value = torch.zeros(tuple(shape), dtype=dtype or torch.float32)
    else:
      initial_value = torch.as_tensor(initial_value, dtype=dtype)
    pedestal = self.offset**2
    self.variable = nn.Parameter(torch.sqrt(torch.clamp(initial_value + pedestal, min=pedestal)))

  minimum = property(lambda self: self._minimum)
  offset = property(lambda self: self._offset)

  def forward(self, compute_dtype=None):
    variable = self.variable if compute_dtype is None else self.variable.to(compute_dtype)
    pedestal = self.offset**2
    bound = (self.minimum + self.offset**2)**.5
    return math_ops.lower_bound(variable, bound).square() - pedestal

  def get_config(self):
    return dict(name=self.name, initial_value=None, minimum=self.minimum, offset=self.offset,
                shape=tuple(map(int, self.variable.shape)), dtype=str(self.variable.dtype).replace("torch.", ""))


def _convert(parameter, dtype, device):
  value = parameter() if callable(parameter) else parameter
  return torch.as_tensor(value, dtype=dtype, device=device)


class GDN(nn.Module):
  """Generalized divisive normalization: y_i = x_i / (beta_i + sum_j gamma_ji |x_j|^alpha)^epsilon
  (or `*` when `inverse`).  Same constructor keywords and attribute semantics as `tfc.GDN`."""

  _SETTABLE = ("inverse", "rectify", "data_format", "alpha_parameter", "beta_parameter", "gamma_parameter",
               "epsilon_parameter", "alpha_initializer", "beta_initializer", "gamma_initializer",
               "epsilon_initializer")

  def __init__(self, inverse=False, rectify=False, data_format="channels_last", alpha_parameter=1,
               beta_parameter=None, gamma_parameter=None, epsilon_parameter=1, alpha_initializer="ones",
               beta_initializer="ones", gamma_initializer=None, epsilon_initializer="ones", name=None):
    super().__init__()
    object.__setattr__(self, "built", False)
    self.name = name
    self.inverse = inverse
    self.rectify = rectify
    self.data_format = data_format
    self.alpha_parameter = alpha_parameter
    self.beta_parameter = beta_parameter
    self.gamma_parameter = gamma_parameter
    self.epsilon_parameter = epsilon_parameter
    self.alpha_initializer = alpha_initializer
    self.beta_initializer = beta_initializer
    self.gamma_initializer = gamma_initializer  # None -> 0.1 * identity (gdn.py:137)
    self.epsilon_initializer = epsilon_initializer

  def __setattr__(self, name, value):
    if name in GDN._SETTABLE and getattr(self, "built", False):
      raise RuntimeError("Can't modify layer attributes after it has been built.")
    if name in ("inverse", "rectify"):
      value = bool(value)
    if name == "data_format" and value not in ("channels_first", "channels_last"):
      raise ValueError(f"Unknown data format: '{value}'.")
    super().__setattr__(name, value)

  @staticmethod
  def _initial(initializer, shape):
    if callable(initializer):
      return torch.as_tensor(initializer(shape), dtype=torch.float32)
    if initializer in ("ones", None) and len(shape) < 2:
      return torch.ones(shape)
    if initializer == "zeros":
      return torch.zeros(shape)
    if initializer is None:  # gamma default
      return 0.1 * torch.eye(shape[0])
    if initializer == "ones":
      return torch.ones(shape)
    raise ValueError(f"Unknown initializer {initializer!r}")

  @property
  def _channel_axis(self):
    return {"channels_first": 1, "channels_last": -1}[self.data_format]

  def build(self, input_shape, device=None):
    """gdn.py:336-369."""
    input_shape = tuple(input_shape)
    if len(input_shape) < 2:
      raise ValueError(f"Input tensor must have at least rank 2, received shape {input_shape}.")
    C = input_shape[self._channel_axis]
    if C is None:
      raise ValueError("The channel dimension of the inputs must be defined.")
    C = int(C)
    if self.alpha_parameter is None:
      self.alpha_parameter = GDNParameter(self._initial(self.alpha_initializer, ()), name="alpha", minimum=1)
    if self.beta_parameter is None:
      self.beta_parameter = GDNParameter(self._initial(self.beta_initializer, (C,)), name="beta", minimum=1e-6)
    if self.gamma_parameter is None:
      self.gamma_parameter = GDNParameter(self._initial(self.gamma_initializer, (C, C)), name="gamma", minimum=0)
    if self.epsilon_parameter is None:
      self.epsilon_parameter = GDNParameter(self._initial(self.epsilon_initializer, ()), name="epsilon",
                                            minimum=1e-6)
    if device is not None:
      self.to(device)
    object.__setattr__(self, "built", True)

  def _param(self, name, dtype=torch.float32, device=None):
    p = getattr(self, name + "_parameter")
    if p is None:
      raise RuntimeError(f"{name} is not initialized yet. Call build().")
    return _convert(p, dtype, device)

  alpha = property(lambda self: self._param("alpha"))
  beta = property(lambda self: self._param("beta"))
  gamma = property(lambda self: self._param("gamma"))
  epsilon = property(lambda self: self._param("epsilon"))

  def forward(self, inputs):
    """gdn.py:371-421."""
    if inputs.dim() < 2:
      raise ValueError(f"Input tensor must have at least rank 2, received shape {tuple(inputs.shape)}.")
    if not self.built:
      self.build(inputs.shape, device=inputs.device)
    dev = inputs.device
    alpha, epsilon = self.alpha_parameter, self.epsilon_parameter
    # trainable exponents travel as 0-d tensors: literal pow in the kernels plus the two scalar gradients
    # (gdn.py:345-367,388,411); fixed ones as Python numbers (|u| / u^2 / sqrt shortcuts, tensor-core kernels)
    a = self._param("alpha", device=dev) if callable(alpha) else float(alpha)
    e = self._param("epsilon", device=dev) if callable(epsilon) else float(epsilon)
    if self.data_format == "channels_first" and F._gdn_native_cf(inputs, a, e, callable(alpha), callable(epsilon)):
      # contiguous [N, C, *spatial] read and written in place: y and, in the backward, dx come back contiguous
      return F.gdn(inputs, self._param("gamma", device=dev), self._param("beta", device=dev), self.inverse,
                   self.rectify, a, e, channels_first=True)
    x = inputs.movedim(1, -1) if self.data_format == "channels_first" else inputs
    out_dtype = x.dtype
    # float16 / bfloat16 activations go to the kernels as they are (mixed precision, gdn_test.py:200-210)
    x32 = (x if x.dtype in (torch.float32, torch.float16, torch.bfloat16) else x.to(torch.float32)).contiguous()
    y = F.gdn(x32, self._param("gamma", device=dev), self._param("beta", device=dev), self.inverse, self.rectify, a, e)
    y = y.to(out_dtype)
    return y.movedim(-1, 1) if self.data_format == "channels_first" else y

  def _torch_graph(self, x, dev):
    """NOT on the product path (forward() runs the CUDA kernels for every exponent configuration): the reference's
    graph, kept as the checker of the trainable-exponent kernels in the tests.  gdn.py:377-415 literally: the fixed-exponent special cases are kept even when the OTHER exponent is
    trainable (|x| for alpha == 1 without rectify, square for alpha == 2, sqrt for epsilon == .5)."""
    u = torch.relu(x) if self.rectify else x
    alpha, epsilon = self.alpha_parameter, self.epsilon_parameter
    if not callable(alpha) and alpha == 1 and self.rectify:
      pool = u
    elif not callable(alpha) and alpha == 1:
      pool = u.abs()
    elif not callable(alpha) and alpha == 2:
      pool = u.square()
    else:
      pool = u**self._param("alpha", device=dev)
    n = pool @ self._param("gamma", device=dev) + self._param("beta", device=dev)
    if not callable(epsilon) and epsilon == 1:
      pass
    elif not callable(epsilon) and epsilon == .5:
      n = n.sqrt()
    else:
      n = n**self._param("epsilon", device=dev)
    return u * n if self.inverse else u / n

  def compute_output_shape(self, input_shape):
    return tuple(input_shape)

  def get_config(self):
    def ser(p):
      if p is None:
        return None
      if isinstance(p, GDNParameter):
        return dict(class_name="GDNParameter", config=p.get_config())
      return float(p)
    return dict(name=self.name, inverse=self.inverse, rectify=self.rectify, data_format=self.data_format,
                alpha_parameter=ser(self.alpha_parameter), beta_parameter=ser(self.beta_parameter),
                gamma_parameter=ser(self.gamma_parameter), epsilon_parameter=ser(self.epsilon_parameter))
