"""The two models the hot path serves, driven end to end: `BLS2017Model` (models/bls2017.py:55-190) and
`BMSHJ2018Model` (models/bmshj2018.py:53-264) -- analysis / synthesis (and hyper) transforms built from
`SignalConv2D` glue + the CUDA `GDN`, the entropy models on the CUDA range coder, `compress` / `decompress`
with the reference's signatures and the `.tfci` container (`PackedTensors`) around them.

The convolutions are cuDNN through torch (glue, no kernel claim); GDN/IGDN, quantisation, table build and range
coding are this repo's kernels.  There is no TF here, so weights are the layers' own initialisers (or a
state_dict); what is reproduced is the data path: shapes, cropping, casts, the order of the coded tensors and the
bytes of the container.

Batches: the reference's `compress` takes ONE image `[H, W, 3]` uint8 (it adds the batch dimension itself);
`compress_batch` / `decompress_batch` take `[B, H, W, 3]` and code B streams in one launch -- what
BASELINE.json configs[1]/[2] ("batch=256 / 128") time.  `compress_images` / `decompress_images` take a list of
images of different sizes: the transforms run per image (grouping equal shapes into one conv batch could let cuDNN
pick another algorithm and change the strings), the range coder once for all of them (ragged batches).
"""
import math

import numpy as np
import torch
from torch import nn

from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops, math_ops
from compression_b200.gdn import GDN
from compression_b200.packed_tensors import PackedTensors
from compression_b200.signal_conv import SignalConv2D

__all__ = ["BLS2017Model", "BMSHJ2018Model", "MS2020Model", "MBT2018Model", "CheckerboardModel", "SpaceChannelModel", "MultistageModel", "MixtureHyperpriorModel", "CheckerboardMixtureModel", "MaskedConv2D", "AnalysisTransform", "SynthesisTransform", "HyperAnalysisTransform",
           "HyperSynthesisTransform", "bench_model_paths", "mean_metrics"]


class _Scale(nn.Module):
  """tf.keras.layers.Lambda(lambda x: x / 255.) and its inverse."""

  def __init__(self, factor):
    super().__init__()
    self.factor = factor

  def forward(self, x):
    return x * self.factor


def _conv(filters, k, name, down=1, up=1, corr=True, use_bias=True, activation=None, **kw):
  return SignalConv2D(filters, (k, k), name=name, corr=corr, strides_down=down, strides_up=up, padding="same_zeros",
                      use_bias=use_bias, activation=activation, **kw)


class AnalysisTransform(nn.Sequential):
  """bls2017.py:55-72 (three layers, 9x9/4 then 5x5/2 twice) or bmshj2018.py:53-74 (`hyperprior=True`: four 5x5/2)."""

  def __init__(self, num_filters, hyperprior=False):
    if hyperprior:
      layers = [_conv(num_filters, 5, f"layer_{i}", down=2, activation=GDN(name=f"gdn_{i}")) for i in range(3)]
      layers.append(_conv(num_filters, 5, "layer_3", down=2))
    else:
      layers = [_conv(num_filters, 9, "layer_0", down=4, activation=GDN(name="gdn_0")),
                _conv(num_filters, 5, "layer_1", down=2, activation=GDN(name="gdn_1")),
                _conv(num_filters, 5, "layer_2", down=2, use_bias=False)]
    super().__init__(_Scale(1 / 255.), *layers)


class SynthesisTransform(nn.Sequential):
  """bls2017.py:75-92 / bmshj2018.py:77-98."""

  def __init__(self, num_filters, hyperprior=False):
    if hyperprior:
      layers = [_conv(num_filters, 5, f"layer_{i}", up=2, corr=False, activation=GDN(name=f"igdn_{i}", inverse=True))
                for i in range(3)]
      layers.append(_conv(3, 5, "layer_3", up=2, corr=False))
    else:
      layers = [_conv(num_filters, 5, "layer_0", up=2, corr=False, activation=GDN(name="igdn_0", inverse=True)),
                _conv(num_filters, 5, "layer_1", up=2, corr=False, activation=GDN(name="igdn_1", inverse=True)),
                _conv(3, 9, "layer_2", up=4, corr=False)]
    super().__init__(*layers, _Scale(255.))


class HyperAnalysisTransform(nn.Sequential):
  """bmshj2018.py:101-118."""

  def __init__(self, num_filters):
    super().__init__(_conv(num_filters, 3, "layer_0", activation=torch.relu),
                     _conv(num_filters, 5, "layer_1", down=2, activation=torch.relu),
                     _conv(num_filters, 5, "layer_2", down=2, use_bias=False))


class HyperSynthesisTransform(nn.Sequential):
  """bmshj2018.py:121-138 (plain-variable kernels)."""

  def __init__(self, num_filters):
    super().__init__(_conv(num_filters, 5, "layer_0", up=2, corr=False, kernel_parameter="variable", activation=torch.relu),
                     _conv(num_filters, 5, "layer_1", up=2, corr=False, kernel_parameter="variable", activation=torch.relu),
                     _conv(num_filters, 3, "layer_2", corr=False, kernel_parameter="variable"))


def _to_uint8(x_hat):
  """tf.saturate_cast(tf.round(x_hat), tf.uint8)."""
  return torch.clamp(torch.round(x_hat), 0, 255).to(torch.uint8)


def _as_batch(x):
  x = torch.as_tensor(x)
  if x.dim() != 4 or x.shape[-1] != 3:
    raise ValueError(f"expected images [B, H, W, 3], received shape {tuple(x.shape)}")
  return x


def _as_image(x):
  x = torch.as_tensor(x)
  if x.dim() != 3 or x.shape[-1] != 3:
    raise ValueError(f"expected one image [H, W, 3], received shape {tuple(x.shape)}")
  return x


def mean_metrics(per_image):
  """The mean of each key over a list of `evaluate` / `evaluate_images` dicts: a rate-distortion point as the
  reference's results report it, per-image values averaged at one lambda."""
  per_image = list(per_image)
  if not per_image:
    raise ValueError("no metrics to average")
  return {k: math.fsum(d[k] for d in per_image) / len(per_image) for k in per_image[0]}


class _Model(nn.Module):

  # whether the model's decoders can use substreams (DESIGN §3.14); MBT2018Model's decodes positions serially
  _substream_decoder = True

  def _device(self):
    return next(self.parameters()).device

  def _set_substreams(self, substreams):
    """`substreams` = S: every string the model writes (y, z, each MS2020 slice) holds S independently decodable
    streams behind a small header, so that one image decodes on S SMs; S = 1 writes the reference's strings."""
    S = gen_ops.check_substreams(substreams)
    if S > 1 and not self._substream_decoder:
      raise ValueError(f"{type(self).__name__} decodes its positions one after another, so substreams cannot help "
                       f"it: substreams must be 1, not {S}")
    self.substreams = S

  def build(self, device="cuda", patch=(64, 64)):
    """Keras `self.build((None, None, None, 3))`: creates every variable (the layers build lazily on a first pass)."""
    self.to(device)
    with torch.no_grad():
      self(torch.zeros((1,) + tuple(patch) + (3,), device=device), training=False)
    return self

  def rate_distortion(self, x, bits):
    num_pixels = float(np.prod(x.shape[:-1]))
    bpp = bits / num_pixels
    mse = torch.mean((x - self._last_x_hat)**2)
    return bpp + self.lmbda * mse, bpp, mse

  @torch.no_grad()
  def evaluate(self, x):
    """The verbose block of the reference's `compress` (bls2017.py:287-305) for one uint8 image [H, W, 3]: codes it
    to `.tfci`, decodes that, and returns the metrics of the float32 pair as Python floats: `mse`, `psnr` and `msssim`
    (tf.image's, max_val 255), `msssim_db` = -10 log10(1 - msssim), and `bpp`, the container's bits per pixel."""
    from compression_b200 import image
    x = _as_image(x)
    tfci = self.compress_to_tfci(x)
    x_hat = self.decompress_from_tfci(tfci)
    x = x.to(device=x_hat.device, dtype=torch.float32)
    x_hat = x_hat.to(torch.float32)
    mse = torch.mean((x - x_hat)**2)
    psnr = image.psnr(x, x_hat, 255)
    msssim = image.ssim_multiscale(x, x_hat, 255)
    msssim_db = -10. * torch.log(1 - msssim) / math.log(10.)
    bpp = len(tfci) * 8 / (x.shape[0] * x.shape[1])
    return {"mse": float(mse), "psnr": float(psnr), "msssim": float(msssim), "msssim_db": float(msssim_db),
            "bpp": float(bpp)}

  @torch.no_grad()
  def evaluate_images(self, images):
    """`evaluate` for a list of uint8 images [H_i, W_i, 3] of their own sizes, one dict of Python floats per image.

    Runs `compress_images` once, packs each image's items into its own `.tfci` (for `bpp`), runs `decompress_images`
    once, then one `image.metrics_ragged` call per colour space on the float32 pairs (max_val 255).  The keys of
    `evaluate` have its meaning, with the same `bpp` and `msssim` bit for bit (`mse` and `psnr` are summed in another
    order).  Added: `psnr_y`, `msssim_y`, `msssim_db_y` on Y', and `psnr_ycbcr`, `msssim_ycbcr`, `msssim_db_ycbcr`, the
    6:1:1 average over Y'CbCr that the reference's results recommend.  `mean_metrics` averages the list."""
    from compression_b200 import image
    images = [_as_image(x) for x in images]
    if not images:
      return []
    items = self.compress_images(images)
    n_bytes = []
    for item in items:
      packed = PackedTensors()
      packed.pack(item)
      n_bytes.append(len(packed.string))
    x_hats = [x.to(torch.float32) for x in self.decompress_images(items)]
    xs = [x.to(device=x_hat.device, dtype=torch.float32) for x, x_hat in zip(images, x_hats)]
    out = [{"bpp": n * 8 / (x.shape[0] * x.shape[1])} for n, x in zip(n_bytes, images)]
    for color, suffix in (("rgb", ""), ("y", "_y"), ("ycbcr", "_ycbcr")):
      metrics = image.metrics_ragged(xs, x_hats, 255, color)
      for key in ("mse", "psnr", "msssim", "msssim_db") if color == "rgb" else ("psnr", "msssim", "msssim_db"):
        for d, v in zip(out, metrics[key].tolist()):
          d[key + suffix] = v
    return out

  def compress_to_tfci(self, x):
    """The .tfci container (bls2017.py:262-282): `compress(x)` packed into one byte string."""
    packed = PackedTensors()
    packed.pack(self.compress(x))
    return packed.string


class BLS2017Model(_Model):
  """models/bls2017.py:95-190."""

  def __init__(self, lmbda=0.01, num_filters=128, substreams=1):
    super().__init__()
    self._set_substreams(substreams)
    self.lmbda = lmbda
    self.num_filters = int(num_filters)
    self.analysis_transform = AnalysisTransform(num_filters)
    self.synthesis_transform = SynthesisTransform(num_filters)
    self.prior = D.NoisyDeepFactorized(batch_shape=(num_filters,))
    self.entropy_model = None

  def forward(self, x, training=True):
    """bls2017.py:106-124 -> (loss, bpp, mse)."""
    entropy_model = E.ContinuousBatchedEntropyModel(self.prior, coding_rank=3, compression=False)
    x = x.to(torch.float32)
    y = self.analysis_transform(x)
    y_hat, bits = entropy_model(y, training=training)
    self._last_x_hat = self.synthesis_transform(y_hat)
    return self.rate_distortion(x, bits.sum())

  def fix_tables(self):
    """bls2017.py:156-161 (end of `fit`): fixes the range-coding tables from the trained prior."""
    self.entropy_model = E.ContinuousBatchedEntropyModel(self.prior, coding_rank=3, compression=True).to(self._device())
    return self

  # -- one image, the reference's signatures (bls2017.py:163-190) --
  def compress(self, x):
    """x: uint8 [H, W, 3] -> (string [1], x_shape [2], y_shape [2])."""
    return self.compress_batch(_as_image(x)[None])

  def decompress(self, string, x_shape, y_shape):
    """-> uint8 [H, W, 3]."""
    return self.decompress_batch(string, x_shape, y_shape)[0]

  # -- batches --
  @torch.no_grad()
  def compress_batch(self, x):
    x = _as_batch(x).to(device=self._device(), dtype=torch.float32)
    y = self.analysis_transform(x)
    x_shape = torch.tensor(x.shape[1:-1], dtype=torch.int32)
    y_shape = torch.tensor(y.shape[1:-1], dtype=torch.int32)
    return self.entropy_model.compress(y, substreams=self.substreams), x_shape, y_shape

  @torch.no_grad()
  def decompress_batch(self, strings, x_shape, y_shape):
    y_hat = self.entropy_model.decompress(strings, tuple(int(v) for v in y_shape), substreams=self.substreams)
    x_hat = self.synthesis_transform(y_hat)
    x_hat = x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :]
    return _to_uint8(x_hat)

  # -- lists of differently sized images: transforms per image, one range-coder launch for all --
  @torch.no_grad()
  def compress_images(self, images):
    """images: list of uint8 [H_i, W_i, 3] -> the list of what `compress(image)` returns, element for element."""
    ys, shapes = [], []
    for x in images:
      x = _as_image(x)[None].to(device=self._device(), dtype=torch.float32)
      y = self.analysis_transform(x)
      ys.append(y[0])
      shapes.append((torch.tensor(x.shape[1:-1], dtype=torch.int32), torch.tensor(y.shape[1:-1], dtype=torch.int32)))
    strings = self.entropy_model.compress_ragged(ys, substreams=self.substreams).split()
    return [(s,) + sh for s, sh in zip(strings, shapes)]

  @torch.no_grad()
  def decompress_images(self, items):
    """items: tuples as `compress_images` returns them -> list of uint8 [H_i, W_i, 3]."""
    items = list(items)
    y_hats = self.entropy_model.decompress_ragged(gen_ops.Strings.concat([it[0] for it in items]),
                                                  [tuple(int(v) for v in it[2]) for it in items],
                                                  substreams=self.substreams)
    out = []
    for y_hat, (_, x_shape, _) in zip(y_hats, items):
      x_hat = self.synthesis_transform(y_hat[None])
      out.append(_to_uint8(x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :])[0])
    return out

  # -- .tfci container (bls2017.py:308-321 `decompress`) --
  def decompress_from_tfci(self, data):
    string, x_shape, y_shape = PackedTensors(data).unpack([bytes, torch.int32, torch.int32])
    return self.decompress(string, x_shape, y_shape)


class BMSHJ2018Model(_Model):
  """models/bmshj2018.py:141-264 (scale hyperprior)."""

  def __init__(self, lmbda=0.01, num_filters=192, num_scales=64, scale_min=.11, scale_max=256., substreams=1):
    super().__init__()
    self._set_substreams(substreams)
    self.lmbda = lmbda
    self.num_scales = int(num_scales)
    offset = math.log(scale_min)
    factor = (math.log(scale_max) - math.log(scale_min)) / (num_scales - 1.)
    self.scale_fn = lambda i: torch.exp(offset + factor * i)
    self.analysis_transform = AnalysisTransform(num_filters, hyperprior=True)
    self.synthesis_transform = SynthesisTransform(num_filters, hyperprior=True)
    self.hyper_analysis_transform = HyperAnalysisTransform(num_filters)
    self.hyper_synthesis_transform = HyperSynthesisTransform(num_filters)
    self.hyperprior = D.NoisyDeepFactorized(batch_shape=(num_filters,))
    self.entropy_model = None
    self.side_entropy_model = None

  def forward(self, x, training=True):
    """bmshj2018.py:159-184."""
    entropy_model = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, self.num_scales, self.scale_fn, coding_rank=3,
                                                       compression=False)
    side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=False)
    x = x.to(torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y.abs())
    z_hat, side_bits = side_entropy_model(z, training=training)
    indexes = self.hyper_synthesis_transform(z_hat)
    indexes = indexes[:, :y.shape[1], :y.shape[2], :]
    y_hat, bits = entropy_model(y, indexes, training=training)
    self._last_x_hat = self.synthesis_transform(y_hat)[:, :x.shape[1], :x.shape[2], :]
    return self.rate_distortion(x, bits.sum() + side_bits.sum())

  def fix_tables(self):
    """bmshj2018.py:216-223."""
    self.entropy_model = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, self.num_scales, self.scale_fn,
                                                            coding_rank=3, compression=True)
    self.side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=True)
    self.entropy_model.to(self._device())
    self.side_entropy_model.to(self._device())
    return self

  def compress(self, x):
    """bmshj2018.py:225-245: uint8 [H, W, 3] -> (string, side_string, x_shape, y_shape, z_shape)."""
    return self.compress_batch(_as_image(x)[None])

  def decompress(self, string, side_string, x_shape, y_shape, z_shape):
    """bmshj2018.py:247-264."""
    return self.decompress_batch(string, side_string, x_shape, y_shape, z_shape)[0]

  @torch.no_grad()
  def compress_batch(self, x):
    x = _as_batch(x).to(device=self._device(), dtype=torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y.abs())
    x_shape = torch.tensor(x.shape[1:-1], dtype=torch.int32)
    y_shape = torch.tensor(y.shape[1:-1], dtype=torch.int32)
    z_shape = torch.tensor(z.shape[1:-1], dtype=torch.int32)
    z_hat = self.side_entropy_model.quantize(z)
    indexes = self.hyper_synthesis_transform(z_hat)
    indexes = indexes[:, :y.shape[1], :y.shape[2], :]
    side_string = self.side_entropy_model.compress(z, substreams=self.substreams)
    string = self.entropy_model.compress(y, indexes, substreams=self.substreams)
    return string, side_string, x_shape, y_shape, z_shape

  @torch.no_grad()
  def decompress_batch(self, string, side_string, x_shape, y_shape, z_shape):
    z_hat = self.side_entropy_model.decompress(side_string, tuple(int(v) for v in z_shape), substreams=self.substreams)
    indexes = self.hyper_synthesis_transform(z_hat)
    indexes = indexes[:, :int(y_shape[0]), :int(y_shape[1]), :]
    y_hat = self.entropy_model.decompress(string, indexes, substreams=self.substreams)
    x_hat = self.synthesis_transform(y_hat)
    x_hat = x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :]
    return _to_uint8(x_hat)

  # -- lists of differently sized images: transforms per image, one range-coder launch for z and one for y --
  @torch.no_grad()
  def compress_images(self, images):
    """images: list of uint8 [H_i, W_i, 3] -> the list of what `compress(image)` returns, element for element."""
    ys, zs, idxs, shapes = [], [], [], []
    for x in images:
      x = _as_image(x)[None].to(device=self._device(), dtype=torch.float32)
      y = self.analysis_transform(x)
      z = self.hyper_analysis_transform(y.abs())
      indexes = self.hyper_synthesis_transform(self.side_entropy_model.quantize(z))
      ys.append(y[0])
      zs.append(z[0])
      idxs.append(indexes[0, :y.shape[1], :y.shape[2], :])
      shapes.append(tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z)))
    side_strings = self.side_entropy_model.compress_ragged(zs, substreams=self.substreams).split()
    strings = self.entropy_model.compress_ragged(ys, idxs, substreams=self.substreams).split()
    return [(s, side) + sh for s, side, sh in zip(strings, side_strings, shapes)]

  @torch.no_grad()
  def decompress_images(self, items):
    """items: tuples as `compress_images` returns them -> list of uint8 [H_i, W_i, 3]."""
    items = list(items)
    z_hats = self.side_entropy_model.decompress_ragged(gen_ops.Strings.concat([it[1] for it in items]),
                                                       [tuple(int(v) for v in it[4]) for it in items],
                                                       substreams=self.substreams)
    idxs = []
    for z_hat, (_, _, _, y_shape, _) in zip(z_hats, items):
      idxs.append(self.hyper_synthesis_transform(z_hat[None])[0, :int(y_shape[0]), :int(y_shape[1]), :])
    y_hats = self.entropy_model.decompress_ragged(gen_ops.Strings.concat([it[0] for it in items]), idxs,
                                                  substreams=self.substreams)
    out = []
    for y_hat, (_, _, x_shape, _, _) in zip(y_hats, items):
      x_hat = self.synthesis_transform(y_hat[None])
      out.append(_to_uint8(x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :])[0])
    return out

  def decompress_from_tfci(self, data):
    dtypes = [bytes, bytes, torch.int32, torch.int32, torch.int32]
    return self.decompress(*PackedTensors(data).unpack(dtypes))


class _MS2020SliceTransform(nn.Sequential):
  """ms2020.py:139-166: channel-conditional parameter / latent-residual-prediction transform of one slice."""

  def __init__(self, slice_depth):
    conv = lambda f, k, name, act: _conv(f, k, name, corr=False, kernel_parameter="variable", activation=act)
    super().__init__(conv(224, 5, "layer_0", torch.relu), conv(128, 5, "layer_1", torch.relu),
                     conv(slice_depth, 3, "layer_2", None))


class MS2020Model(_Model):
  """models/ms2020.py:169-440 (channel-wise autoregressive entropy model with latent residual prediction): the
  callers' side of the index-mode coder -- every slice of y is coded by one `LocationScaleIndexedEntropyModel`
  call conditioned on the hyperprior and on the slices decoded before it, so compress() issues num_slices + 1
  encodes AND the matching decodes (ms2020.py:334-389)."""

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=320, hyperprior_depth=192, num_slices=10,
               max_support_slices=5, num_scales=64, scale_min=.11, scale_max=256., substreams=1):
    super().__init__()
    self._set_substreams(substreams)
    if latent_depth % num_slices:
      raise ValueError("Slices do not evenly divide latent depth (%d / %d)" % (latent_depth, num_slices))
    self.lmbda = lmbda
    self.num_scales, self.num_slices, self.max_support_slices = int(num_scales), int(num_slices), int(max_support_slices)
    offset = math.log(scale_min)
    factor = (math.log(scale_max) - math.log(scale_min)) / (num_scales - 1.)
    self.scale_fn = lambda i: torch.exp(offset + factor * i)
    f = num_filters
    self.analysis_transform = nn.Sequential(                                       # ms2020.py:53-71
        _Scale(1 / 255.), *[_conv(f, 5, f"layer_{i}", down=2, activation=GDN(name=f"gdn_{i}")) for i in range(3)],
        _conv(latent_depth, 5, "layer_3", down=2))
    self.synthesis_transform = nn.Sequential(                                      # ms2020.py:74-95
        *[_conv(f, 5, f"layer_{i}", up=2, corr=False, activation=GDN(name=f"igdn_{i}", inverse=True)) for i in range(3)],
        _conv(3, 5, "layer_3", up=2, corr=False), _Scale(255.))
    self.hyper_analysis_transform = nn.Sequential(                                 # ms2020.py:98-115
        _conv(320, 3, "layer_0", activation=torch.relu), _conv(256, 5, "layer_1", down=2, activation=torch.relu),
        _conv(hyperprior_depth, 5, "layer_2", down=2, use_bias=False))
    hs = lambda: nn.Sequential(                                                    # ms2020.py:118-136
        _conv(192, 5, "layer_0", up=2, corr=False, kernel_parameter="variable", activation=torch.relu),
        _conv(256, 5, "layer_1", up=2, corr=False, kernel_parameter="variable", activation=torch.relu),
        _conv(320, 3, "layer_2", corr=False, kernel_parameter="variable", activation=torch.relu))
    self.hyper_synthesis_mean_transform, self.hyper_synthesis_scale_transform = hs(), hs()
    sd = latent_depth // num_slices
    self.cc_mean_transforms = nn.ModuleList([_MS2020SliceTransform(sd) for _ in range(num_slices)])
    self.cc_scale_transforms = nn.ModuleList([_MS2020SliceTransform(sd) for _ in range(num_slices)])
    self.lrp_transforms = nn.ModuleList([_MS2020SliceTransform(sd) for _ in range(num_slices)])
    self.hyperprior = D.NoisyDeepFactorized(batch_shape=(hyperprior_depth,))
    self.em_z = self.em_y = None

  def _slice_params(self, i, latent_means, latent_scales, y_hat_slices, y_hw):
    """mu, scale indexes and the LRP support of slice i (ms2020.py:241-253)."""
    support = y_hat_slices if self.max_support_slices < 0 else y_hat_slices[:self.max_support_slices]
    mean_support = torch.cat([latent_means] + support, dim=-1)
    mu = self.cc_mean_transforms[i](mean_support)[:, :y_hw[0], :y_hw[1], :]
    scale_support = torch.cat([latent_scales] + support, dim=-1)
    sigma = self.cc_scale_transforms[i](scale_support)[:, :y_hw[0], :y_hw[1], :]
    return mu, sigma, mean_support

  def _lrp(self, i, mean_support, y_hat_slice):
    return y_hat_slice + 0.5 * torch.tanh(self.lrp_transforms[i](torch.cat([mean_support, y_hat_slice], dim=-1)))

  def forward(self, x, training=True):
    """ms2020.py:200-286 -> (loss, bpp, mse)."""
    x = x.to(torch.float32)
    y = self.analysis_transform(x)
    y_hw = tuple(y.shape[1:-1])
    z = self.hyper_analysis_transform(y)
    num_pixels = float(np.prod(x.shape[1:-1]))
    em_z = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=False, offset_heuristic=False)
    _, z_bits = em_z(z, training=training)
    z_hat = em_z.quantize(z)
    latent_scales = self.hyper_synthesis_scale_transform(z_hat)
    latent_means = self.hyper_synthesis_mean_transform(z_hat)
    em_y = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, self.num_scales, self.scale_fn, coding_rank=3,
                                              compression=False)
    y_hat_slices, bpp = [], z_bits.mean() / num_pixels
    for i, y_slice in enumerate(torch.chunk(y, self.num_slices, dim=-1)):
      mu, sigma, mean_support = self._slice_params(i, latent_means, latent_scales, y_hat_slices, y_hw)
      _, slice_bits = em_y(y_slice, sigma, loc=mu, training=training)
      bpp = bpp + slice_bits.mean() / num_pixels
      y_hat_slices.append(self._lrp(i, mean_support, em_y.quantize(y_slice, loc=mu)))
    x_hat = self.synthesis_transform(torch.cat(y_hat_slices, dim=-1))
    mse = torch.mean((x - x_hat[:, :x.shape[1], :x.shape[2], :])**2)
    return bpp + self.lmbda * mse, bpp, mse

  def fix_tables(self):
    """ms2020.py:321-329."""
    dev = self._device()
    self.em_z = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=True,
                                                offset_heuristic=False).to(dev)
    self.em_y = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, self.num_scales, self.scale_fn, coding_rank=3,
                                                   compression=True).to(dev)
    return self

  @torch.no_grad()
  def compress_batch(self, x):
    """ms2020.py:331-389 for B images: (x_shape, y_shape, z_shape, z_strings, y_strings[0], ..., y_strings[S - 1])."""
    x = _as_batch(x).to(device=self._device(), dtype=torch.float32)
    y = self.analysis_transform(x)
    y_hw = tuple(y.shape[1:-1])
    z = self.hyper_analysis_transform(y)
    S = self.substreams
    z_string = self.em_z.compress(z, substreams=S)
    z_hat = self.em_z.decompress(z_string, tuple(z.shape[1:-1]), substreams=S)
    latent_scales = self.hyper_synthesis_scale_transform(z_hat)
    latent_means = self.hyper_synthesis_mean_transform(z_hat)
    y_strings, y_hat_slices = [], []
    for i, y_slice in enumerate(torch.chunk(y, self.num_slices, dim=-1)):
      mu, sigma, mean_support = self._slice_params(i, latent_means, latent_scales, y_hat_slices, y_hw)
      y_strings.append(self.em_y.compress(y_slice.contiguous(), sigma, mu, substreams=S))
      y_hat_slices.append(self._lrp(i, mean_support, self.em_y.decompress(y_strings[-1], sigma, mu, substreams=S)))
    shapes = [torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z)]
    return tuple(shapes) + (z_string,) + tuple(y_strings)

  @torch.no_grad()
  def decompress_batch(self, x_shape, y_shape, z_shape, z_string, *y_strings):
    """ms2020.py:391-433."""
    assert len(y_strings) == self.num_slices
    y_hw = (int(y_shape[0]), int(y_shape[1]))
    S = self.substreams
    z_hat = self.em_z.decompress(z_string, tuple(int(v) for v in z_shape), substreams=S)
    latent_scales = self.hyper_synthesis_scale_transform(z_hat)
    latent_means = self.hyper_synthesis_mean_transform(z_hat)
    y_hat_slices = []
    for i, y_string in enumerate(y_strings):
      mu, sigma, mean_support = self._slice_params(i, latent_means, latent_scales, y_hat_slices, y_hw)
      y_hat_slices.append(self._lrp(i, mean_support, self.em_y.decompress(y_string, sigma, loc=mu, substreams=S)))
    x_hat = self.synthesis_transform(torch.cat(y_hat_slices, dim=-1))
    return _to_uint8(x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :])

  def compress(self, x):
    """One image uint8 [H, W, 3], the reference's signature (ms2020.py:331-389)."""
    return self.compress_batch(_as_image(x)[None])

  def decompress(self, x_shape, y_shape, z_shape, z_string, *y_strings):
    return self.decompress_batch(x_shape, y_shape, z_shape, z_string, *y_strings)[0]

  # -- lists of differently sized images: transforms per image; one range-coder launch for z and one per slice, each
  # encode handing back the latents it coded, so the encoder decodes nothing --
  @torch.no_grad()
  def compress_images(self, images):
    """images: list of uint8 [H_i, W_i, 3] -> the list of what `compress(image)` returns, element for element.
    num_slices + 1 encode launches in all, whatever the number of images, and no decode."""
    xs = [_as_image(x)[None].to(device=self._device(), dtype=torch.float32) for x in images]
    if not xs:
      raise ValueError("`images` is empty")
    ys = [self.analysis_transform(x) for x in xs]
    zs = [self.hyper_analysis_transform(y) for y in ys]
    y_hws = [tuple(y.shape[1:-1]) for y in ys]
    z_strings, z_hats = self.em_z.compress_ragged([z[0] for z in zs], return_decoded=True, substreams=self.substreams)
    z_strings = z_strings.split()
    latents = [(self.hyper_synthesis_mean_transform(z_hat[None]), self.hyper_synthesis_scale_transform(z_hat[None]))
               for z_hat in z_hats]
    y_hat_slices = [[] for _ in xs]
    y_strings = []
    y_slices = [torch.chunk(y, self.num_slices, dim=-1) for y in ys]
    for i in range(self.num_slices):
      params = [self._slice_params(i, lm, ls, sl, hw) for (lm, ls), sl, hw in zip(latents, y_hat_slices, y_hws)]
      strings, y_hats = self.em_y.compress_ragged([s[i][0] for s in y_slices], [p[1][0] for p in params],
                                                  loc=[p[0][0] for p in params], return_decoded=True,
                                                  substreams=self.substreams)
      y_strings.append(strings.split())
      for sl, p, y_hat in zip(y_hat_slices, params, y_hats):
        sl.append(self._lrp(i, p[2], y_hat[None]))
    out = []
    for k, (x, y, z) in enumerate(zip(xs, ys, zs)):
      shapes = tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
      out.append(shapes + (z_strings[k],) + tuple(s[k] for s in y_strings))
    return out

  @torch.no_grad()
  def decompress_images(self, items):
    """items: tuples as `compress_images` returns them -> list of uint8 [H_i, W_i, 3].  num_slices + 1 decode
    launches in all, whatever the number of images."""
    items = list(items)
    if not items:
      raise ValueError("`items` is empty")
    for it in items:
      if len(it) != 4 + self.num_slices:
        raise ValueError(f"each item needs 3 shapes and {self.num_slices + 1} strings: received {len(it)} elements")
    y_hws = [(int(it[1][0]), int(it[1][1])) for it in items]
    z_hats = self.em_z.decompress_ragged(gen_ops.Strings.concat([it[3] for it in items]),
                                         [tuple(int(v) for v in it[2]) for it in items], substreams=self.substreams)
    latents = [(self.hyper_synthesis_mean_transform(z_hat[None]), self.hyper_synthesis_scale_transform(z_hat[None]))
               for z_hat in z_hats]
    y_hat_slices = [[] for _ in items]
    for i in range(self.num_slices):
      params = [self._slice_params(i, lm, ls, sl, hw) for (lm, ls), sl, hw in zip(latents, y_hat_slices, y_hws)]
      y_hats = self.em_y.decompress_ragged(gen_ops.Strings.concat([it[4 + i] for it in items]),
                                           [p[1][0] for p in params], loc=[p[0][0] for p in params],
                                           substreams=self.substreams)
      for sl, p, y_hat in zip(y_hat_slices, params, y_hats):
        sl.append(self._lrp(i, p[2], y_hat[None]))
    out = []
    for sl, it in zip(y_hat_slices, items):
      x_hat = self.synthesis_transform(torch.cat(sl, dim=-1))
      out.append(_to_uint8(x_hat[:, :int(it[0][0]), :int(it[0][1]), :])[0])
    return out

  def decompress_from_tfci(self, data):
    dtypes = [torch.int32] * 3 + [bytes] * (self.num_slices + 1)
    return self.decompress(*PackedTensors(data).unpack(dtypes))


def _leaky(x):
  """The LeakyReLU of the joint-prior model's hyper transforms and entropy-parameter layers (slope 0.01, as in the
  parameter kernel: x > 0 ? x : 0.01 x)."""
  return torch.nn.functional.leaky_relu(x, 0.01)


def causal_mask(kernel_size=5):
  """Type-A mask [k, k]: 1 at the taps strictly before the centre in raster order (12 for k = 5), 0 elsewhere."""
  m = torch.zeros(kernel_size * kernel_size)
  m[:kernel_size * kernel_size // 2] = 1
  return m.reshape(kernel_size, kernel_size)


class MaskedConv2D(nn.Module):
  """The context model of Minnen et al. 2018: a 5x5 correlation with a type-A mask, channels-last, zero padded to
  the input's size.  `kernel` is [5, 5, in, out] like SignalConv2D's; the training path multiplies it by the fixed
  mask and runs one conv2d, the coding path reads the 12 causal taps from the packed parameters."""

  def __init__(self, in_channels, filters):
    super().__init__()
    std = math.sqrt(1.0 / (12 * in_channels))
    self.kernel = nn.Parameter(torch.randn(5, 5, in_channels, filters) * std)
    self.bias = nn.Parameter(torch.zeros(filters))
    self.register_buffer("mask", causal_mask(5)[:, :, None, None], persistent=False)

  def forward(self, x):
    w = (self.kernel * self.mask).permute(3, 2, 0, 1)
    y = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), w.to(x.dtype), self.bias.to(x.dtype), padding=2)
    return y.permute(0, 2, 3, 1).contiguous()


class MBT2018Model(_Model):
  """Joint autoregressive and hierarchical priors (Minnen, Ballé & Toderici, NeurIPS 2018, Fig. 4 / Table 1).
  N = num_filters, M = latent_depth (a multiple of 6).  bmshj2018's analysis / synthesis with GDN; hyper analysis
  of y (3x3 N, 5x5/2 N, 5x5/2 N); hyper synthesis to psi (5x5 x2 M, 5x5 x2 3M/2, 3x3 2M); a 5x5 type-A masked
  context model M -> 2M; entropy parameters 1x1 4M -> 10M/3 -> 8M/3 -> 2M on [psi, ctx] = [loc, scale_index], with
  LeakyReLU between layers.  z is coded with a NoisyDeepFactorized prior, y by a LocationScaleIndexedEntropyModel
  (NoisyNormal, 64 scales from 0.11 to 256) with `loc`.

  Coding runs on the parameter kernel (functional.ar_*): the encoder visits positions in raster order, then ONE
  index-mode encode of y with the kernel's table indexes and loc makes the strings (the bytes of
  `LocationScaleIndexedEntropyModel.compress(y, scale_index, loc)`); the decoder runs the parameter step and the
  M symbols of each position in one launch.  The hyper synthesis runs per image, so psi, and with it the decoded
  latents, do not depend on how images were batched.

  `tiles` = T > 1 (keyword only, at most 1024) writes every y string as T column tiles (DESIGN §3.15): tile t holds
  columns [floor(t W / T), floor((t + 1) W / T)) of every latent row, coded as its own stream inside the substream
  container (gen_ops.join_substreams with S = T), and the encoder and decoder run the positions of one image as a
  wavefront over many SMs (functional.ar_encode_tiles / ar_decode_tiles).  The latents and reconstructions are those
  of T = 1 bit for bit; only the y strings change, and they must be decoded with the same T.  The z strings are
  unchanged.  T = 1 is the one-stream model."""

  _substream_decoder = False
  tiles = 1  # (the subclasses' y strings are never tiled)

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=192, num_scales=64, scale_min=.11, scale_max=256.,
               substreams=1, *, tiles=1):
    super().__init__()
    self._set_substreams(substreams)
    self.tiles = gen_ops.check_substreams(tiles, "tiles")
    N, M = int(num_filters), int(latent_depth)
    if M <= 0 or M % 6:
      raise ValueError(f"latent_depth must be a positive multiple of 6 (3M/2, 10M/3 and 8M/3 are layer widths): {M}")
    self._init_transforms(lmbda, N, M, num_scales, scale_min, scale_max)
    self.context_model = MaskedConv2D(M, 2 * M)
    ep = lambda f, name, act: _conv(f, 1, name, kernel_parameter="variable", activation=act)
    self.entropy_parameters = nn.Sequential(
        ep(10 * M // 3, "layer_0", _leaky), ep(8 * M // 3, "layer_1", _leaky), ep(2 * M, "layer_2", None))
    self._init_entropy_models(N)

  def _init_transforms(self, lmbda, N, M, num_scales, scale_min, scale_max, psi_width=None):
    """The analysis, synthesis and hyper transforms and the scale table; the hyper synthesis ends in `psi_width`
    channels (2M by default)."""
    self.lmbda = lmbda
    self.num_filters, self.latent_depth, self.num_scales = N, M, int(num_scales)
    offset = math.log(scale_min)
    factor = (math.log(scale_max) - math.log(scale_min)) / (num_scales - 1.)
    self.scale_fn = lambda i: torch.exp(offset + factor * i)
    self.analysis_transform = nn.Sequential(
        _Scale(1 / 255.), *[_conv(N, 5, f"layer_{i}", down=2, activation=GDN(name=f"gdn_{i}")) for i in range(3)],
        _conv(M, 5, "layer_3", down=2))
    self.synthesis_transform = SynthesisTransform(N, hyperprior=True)
    self.hyper_analysis_transform = nn.Sequential(
        _conv(N, 3, "layer_0", activation=_leaky), _conv(N, 5, "layer_1", down=2, activation=_leaky),
        _conv(N, 5, "layer_2", down=2, use_bias=False))
    hs = lambda f, k, name, up, act: _conv(f, k, name, up=up, corr=False, kernel_parameter="variable", activation=act)
    self.hyper_synthesis_transform = nn.Sequential(
        hs(M, 5, "layer_0", 2, _leaky), hs(3 * M // 2, 5, "layer_1", 2, _leaky),
        hs(psi_width or 2 * M, 3, "layer_2", 1, None))

  def _init_entropy_models(self, N):
    self.hyperprior = D.NoisyDeepFactorized(batch_shape=(N,))
    self.entropy_model = None
    self.side_entropy_model = None
    self._packed = None

  def _psi(self, z_hat, y_hw):
    """The hyper feature of each image, computed one image at a time, cropped to y's size: [B, H, W, 2M]."""
    return torch.cat([self.hyper_synthesis_transform(z_hat[i:i + 1])[:, :y_hw[0], :y_hw[1], :]
                      for i in range(z_hat.shape[0])]).contiguous()

  def entropy_parameters_of(self, y_ctx, psi):
    """The parallel (training) form of the parameter network: (loc, scale_index) of every position from the latents
    the context model sees and psi."""
    ctx = self._context(y_ctx)
    params = self.entropy_parameters(torch.cat([psi, ctx], dim=-1))
    return params[..., :self.latent_depth], params[..., self.latent_depth:]

  def _context(self, y_ctx):
    return self.context_model(y_ctx)

  def forward(self, x, training=True):
    """-> (loss, bpp, mse).  The context model sees y plus uniform noise when training, round(y) otherwise."""
    entropy_model = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, self.num_scales, self.scale_fn, coding_rank=3,
                                                       compression=False)
    side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=False)
    x = x.to(torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y)
    z_hat, side_bits = side_entropy_model(z, training=training)
    psi = self.hyper_synthesis_transform(z_hat)[:, :y.shape[1], :y.shape[2], :]
    y_ctx = y + torch.empty_like(y).uniform_(-.5, .5) if training else torch.round(y)
    loc, scale_index = self.entropy_parameters_of(y_ctx, psi)
    y_hat, bits = entropy_model(y, scale_index, loc=loc, training=training)
    self._last_x_hat = self.synthesis_transform(y_hat)[:, :x.shape[1], :x.shape[2], :]
    return self.rate_distortion(x, bits.sum() + side_bits.sum())

  def fix_tables(self):
    """Builds the coding tables and packs the parameter network for the coding kernels (call again after the
    weights change)."""
    dev = self._device()
    self.entropy_model = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, self.num_scales, self.scale_fn,
                                                            coding_rank=3, compression=True).to(dev)
    self.side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=True).to(dev)
    self._packed = self._pack()
    return self

  def _pack(self):
    return self._pack_weights(self.context_model.kernel, self.context_model.bias,
                              *_dense_weights(self.entropy_parameters))

  _pack_weights = staticmethod(F.ar_pack_weights)

  # -- coding: one latent shape per call --
  def _encode_latents(self, y, psi):
    """(strings, y_hat, loc, index) of latents y [B, H, W, M] with hyper feature psi (loc and index flat in tile order
    with tiles > 1)."""
    em = self.entropy_model
    y = y.contiguous()
    if self.tiles > 1:
      y_hats, y_t, loc, index, lengths = F.ar_encode_tiles(self._packed, list(y), list(psi), self.num_scales,
                                                           self.tiles)
      return self._compress_coding_order(y_t, loc, index, lengths, len(y_hats)), torch.stack(y_hats), loc, index
    y_hat, loc, index = F.ar_encode(self._packed, y, psi, self.num_scales)
    strings = F.compress_f32((y.shape[0],), em._lookup_host(), y, loc, em.cdf_offset.to(y.device), index=index)
    return strings, y_hat, loc, index

  def _decode_latents(self, strings, psi):
    em = self.entropy_model
    if self.tiles > 1:
      handle = self._y_decoder(strings)
      y_hats = F.ar_decode_tiles(handle, self._packed, list(psi), self.num_scales, em.cdf_offset.to(psi.device),
                                 self.tiles)
      em._finish_decode(handle)
      return torch.stack(y_hats)
    handle = gen_ops.create_range_decoder(em._strings(strings), em._lookup_host())
    y_hat = F.ar_decode(handle, self._packed, psi, self.num_scales, em.cdf_offset.to(psi.device))
    em._finish_decode(handle)
    return y_hat

  def _y_streams(self):
    """Streams per y string: the substreams, or MBT2018Model's column tiles (at most one of them is above 1)."""
    return self.substreams * self.tiles

  def _y_decoder(self, strings):
    """A decoder handle of y strings (their substreams or tiles when there are several)."""
    em = self.entropy_model
    strings = em._strings(strings)
    if self._y_streams() > 1:
      strings = gen_ops.split_substreams(strings, self._y_streams())
    return gen_ops.create_range_decoder(strings, em._lookup_host())

  def _compress_coding_order(self, y, loc, index, lengths, units):
    """The y strings of `units` images from an encoder's coding-order tensors (substream order, and `lengths` the
    stream lengths, with substreams or tiles > 1)."""
    em = self.entropy_model
    coff = em.cdf_offset.to(y.device)
    S = self._y_streams()
    if S == 1 and lengths is None:
      return F.compress_f32((units,), em._lookup_host(), y, loc, coff, index=index)
    strings = F.compress_ragged(em._lookup_host(), lengths, y, loc, coff, index=index)
    return strings if S == 1 else gen_ops.join_substreams(strings, S, (units,))

  def _coded(self, y, loc, index, B, H, W):
    """The y strings of a batch of B latents of H x W from the context models' coding-order tensors (`_groups()` are
    their channel groups)."""
    lengths = None
    if self.substreams > 1:
      lengths = F.context_substreams(self._groups(), [H] * B, [W] * B, self.substreams)[0]
    return self._compress_coding_order(y, loc, index, lengths, B)

  def compress(self, x):
    """uint8 [H, W, 3] -> (string, side_string, x_shape, y_shape, z_shape), bmshj2018's signature."""
    return self.compress_batch(_as_image(x)[None])

  def decompress(self, string, side_string, x_shape, y_shape, z_shape):
    return self.decompress_batch(string, side_string, x_shape, y_shape, z_shape)[0]

  @torch.no_grad()
  def compress_batch(self, x):
    x = _as_batch(x).to(device=self._device(), dtype=torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y)
    shapes = tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
    side_string = self.side_entropy_model.compress(z, substreams=self.substreams)
    psi = self._psi(self.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
    string = self._encode_latents(y, psi)[0]
    return (string, side_string) + shapes

  @torch.no_grad()
  def decompress_batch(self, string, side_string, x_shape, y_shape, z_shape):
    z_hat = self.side_entropy_model.decompress(side_string, tuple(int(v) for v in z_shape), substreams=self.substreams)
    psi = self._psi(z_hat, (int(y_shape[0]), int(y_shape[1])))
    y_hat = self._decode_latents(string, psi)
    x_hat = self.synthesis_transform(y_hat)
    return _to_uint8(x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :])

  # -- lists of differently sized images: transforms per image, one ragged coding call for the whole list --
  def _encode_ragged(self, ys, psis):
    """(y, loc, index, lengths) in coding order of latents ys [H_i, W_i, M] with hyper features psis (tile order and
    the stream lengths with tiles > 1)."""
    if self.tiles > 1:
      return F.ar_encode_tiles(self._packed, ys, psis, self.num_scales, self.tiles)[1:]
    return F.ar_encode_ragged(self._packed, ys, psis, self.num_scales)[1:]

  def _decode_ragged(self, handle, psis, cdf_offset):
    """The list of y_hat [H_i, W_i, M], continuing `handle` (one string per image, or one per tile)."""
    if self.tiles > 1:
      return F.ar_decode_tiles(handle, self._packed, psis, self.num_scales, cdf_offset, self.tiles)
    return F.ar_decode_ragged(handle, self._packed, psis, self.num_scales, cdf_offset)

  @torch.no_grad()
  def compress_images(self, images):
    """images: list of uint8 [H_i, W_i, 3] -> the list of what `compress(image)` returns, element for element.
    The transforms run per image; the latents of the whole list, whatever their shapes, share one ragged encoder
    launch sequence and one range encode."""
    xs = [_as_image(x)[None].to(device=self._device(), dtype=torch.float32) for x in images]
    if not xs:
      raise ValueError("`images` is empty")
    ys = [self.analysis_transform(x) for x in xs]
    zs = [self.hyper_analysis_transform(y) for y in ys]
    side_strings = self.side_entropy_model.compress_ragged([z[0] for z in zs], substreams=self.substreams).split()
    psis = [self._psi(self.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))[0] for y, z in zip(ys, zs)]
    y_cc, loc, index, lengths = self._encode_ragged([y[0] for y in ys], psis)
    strings = self._compress_coding_order(y_cc, loc, index, lengths, len(xs)).split()
    return [(strings[i], side_strings[i]) + tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
            for i, (x, y, z) in enumerate(zip(xs, ys, zs))]

  @torch.no_grad()
  def decompress_images(self, items):
    """items: tuples as `compress_images` returns them -> list of uint8 [H_i, W_i, 3]."""
    items = list(items)
    if not items:
      raise ValueError("`items` is empty")
    z_hats = self.side_entropy_model.decompress_ragged(gen_ops.Strings.concat([it[1] for it in items]),
                                                       [tuple(int(v) for v in it[4]) for it in items],
                                                       substreams=self.substreams)
    psis = [self._psi(z_hat[None], (int(it[3][0]), int(it[3][1])))[0] for z_hat, it in zip(z_hats, items)]
    em = self.entropy_model
    handle = self._y_decoder(gen_ops.Strings.concat([it[0] for it in items]))
    y_hats = self._decode_ragged(handle, psis, em.cdf_offset.to(psis[0].device))
    em._finish_decode(handle)
    out = []
    for y_hat, it in zip(y_hats, items):
      x_hat = self.synthesis_transform(y_hat[None])
      out.append(_to_uint8(x_hat[:, :int(it[2][0]), :int(it[2][1]), :])[0])
    return out

  def decompress_from_tfci(self, data):
    dtypes = [bytes, bytes, torch.int32, torch.int32, torch.int32]
    return self.decompress(*PackedTensors(data).unpack(dtypes))


class MixtureHyperpriorModel(_Model):
  """Hyperprior with a discretized mixture prior on y (Cheng et al., CVPR 2020, without the attention modules and the
  context model).  N = num_filters, M = latent_depth, K = num_components.  MBT2018Model's analysis, synthesis and
  hyper transforms, the hyper synthesis widened to 3KM channels: channel c of y reads its K logits, K locs and K
  scales, in that order, from channels 3Kc .. 3Kc + 3K - 1; weights = softmax(logits), scales bounded below at 0.11.
  z is coded with a NoisyDeepFactorized prior as in MBT2018Model, y by entropy_models.MixtureEntropyModel
  (coding_rank 3), whose rows are built on the device (DESIGN §3.18).  The hyper synthesis runs per image, so the
  strings of an image do not depend on its batch or list."""

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=192, num_components=3, family="normal", substreams=1):
    super().__init__()
    self._set_substreams(substreams)
    N, M, K = int(num_filters), int(latent_depth), int(num_components)
    if M <= 0 or M % 2:
      raise ValueError(f"latent_depth must be a positive even number (3M/2 is a layer width): {M}")
    if K < 1 or K > 64:
      raise ValueError(f"num_components must be in [1, 64]: {K}")
    if family not in F.MIXTURE_FAMILIES:
      raise ValueError(f"`family` must be one of {sorted(F.MIXTURE_FAMILIES)}: {family!r}")
    self.num_components, self.family = K, family
    MBT2018Model._init_transforms(self, lmbda, N, M, 64, .11, 256., psi_width=3 * K * M)
    self.hyperprior = D.NoisyDeepFactorized(batch_shape=(N,))
    self.entropy_model = E.MixtureEntropyModel(family, coding_rank=3)
    self.side_entropy_model = None

  def mixture_parameters(self, psi):
    """(weight, loc, scale), each [B, H, W, M, K], from the hyper feature psi [B, H, W, 3KM]."""
    K = self.num_components
    p = psi.reshape(psi.shape[:-1] + (self.latent_depth, 3, K))
    weight = torch.softmax(p[..., 0, :], dim=-1)
    scale = math_ops.lower_bound(p[..., 2, :], .11)
    return weight.contiguous(), p[..., 1, :].contiguous(), scale.contiguous()

  def _params(self, z_hat, y_hw):
    """The mixture parameters of each image, the hyper synthesis run one image at a time and cropped to y's size."""
    psi = torch.cat([self.hyper_synthesis_transform(z_hat[i:i + 1])[:, :y_hw[0], :y_hw[1], :]
                     for i in range(z_hat.shape[0])])
    return self.mixture_parameters(psi)

  def forward(self, x, training=True):
    """-> (loss, bpp, mse), with the rate of y through the NoisyNormalMixture / NoisyLogisticMixture graph."""
    side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=False)
    x = x.to(torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y)
    z_hat, side_bits = side_entropy_model(z, training=training)
    psi = self.hyper_synthesis_transform(z_hat)[:, :y.shape[1], :y.shape[2], :]
    y_hat, bits = self.entropy_model(y, *self.mixture_parameters(psi), training=training)
    self._last_x_hat = self.synthesis_transform(y_hat)[:, :x.shape[1], :x.shape[2], :]
    return self.rate_distortion(x, bits.sum() + side_bits.sum())

  def fix_tables(self):
    """Builds z's coding tables from the trained hyperprior (y needs none)."""
    self.side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3,
                                                              compression=True).to(self._device())
    return self

  def compress(self, x):
    """uint8 [H, W, 3] -> (string, side_string, x_shape, y_shape, z_shape), bmshj2018's signature."""
    return self.compress_batch(_as_image(x)[None])

  def decompress(self, string, side_string, x_shape, y_shape, z_shape):
    return self.decompress_batch(string, side_string, x_shape, y_shape, z_shape)[0]

  @torch.no_grad()
  def compress_batch(self, x):
    x = _as_batch(x).to(device=self._device(), dtype=torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y)
    shapes = tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
    side_string = self.side_entropy_model.compress(z, substreams=self.substreams)
    params = self._params(self.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
    string = self.entropy_model.compress(y.contiguous(), *params, substreams=self.substreams)
    return (string, side_string) + shapes

  @torch.no_grad()
  def decompress_batch(self, string, side_string, x_shape, y_shape, z_shape):
    z_hat = self.side_entropy_model.decompress(side_string, tuple(int(v) for v in z_shape), substreams=self.substreams)
    params = self._params(z_hat, (int(y_shape[0]), int(y_shape[1])))
    y_hat = self.entropy_model.decompress(string, *params, substreams=self.substreams)
    x_hat = self.synthesis_transform(y_hat)
    return _to_uint8(x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :])

  @torch.no_grad()
  def compress_images(self, images):
    """images: list of uint8 [H_i, W_i, 3] -> the list of what `compress(image)` returns, element for element.  The
    transforms run per image; z and y of the whole list are each coded in one ragged launch sequence."""
    xs = [_as_image(x)[None].to(device=self._device(), dtype=torch.float32) for x in images]
    if not xs:
      raise ValueError("`images` is empty")
    ys = [self.analysis_transform(x) for x in xs]
    zs = [self.hyper_analysis_transform(y) for y in ys]
    side_strings = self.side_entropy_model.compress_ragged([z[0] for z in zs], substreams=self.substreams).split()
    params = [self._params(self.side_entropy_model.quantize(z), tuple(y.shape[1:-1])) for y, z in zip(ys, zs)]
    ws, ls, ss = ([p[j][0] for p in params] for j in range(3))
    strings = self.entropy_model.compress_ragged([y[0] for y in ys], ws, ls, ss, substreams=self.substreams).split()
    return [(strings[i], side_strings[i]) + tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
            for i, (x, y, z) in enumerate(zip(xs, ys, zs))]

  @torch.no_grad()
  def decompress_images(self, items):
    """items: tuples as `compress_images` returns them -> list of uint8 [H_i, W_i, 3]."""
    items = list(items)
    if not items:
      raise ValueError("`items` is empty")
    z_hats = self.side_entropy_model.decompress_ragged(gen_ops.Strings.concat([it[1] for it in items]),
                                                       [tuple(int(v) for v in it[4]) for it in items],
                                                       substreams=self.substreams)
    params = [self._params(z_hat[None], (int(it[3][0]), int(it[3][1]))) for z_hat, it in zip(z_hats, items)]
    ws, ls, ss = ([p[j][0] for p in params] for j in range(3))
    y_hats = self.entropy_model.decompress_ragged(gen_ops.Strings.concat([it[0] for it in items]), ws, ls, ss,
                                                  substreams=self.substreams)
    out = []
    for y_hat, it in zip(y_hats, items):
      x_hat = self.synthesis_transform(y_hat[None])
      out.append(_to_uint8(x_hat[:, :int(it[2][0]), :int(it[2][1]), :])[0])
    return out

  def decompress_from_tfci(self, data):
    dtypes = [bytes, bytes, torch.int32, torch.int32, torch.int32]
    return self.decompress(*PackedTensors(data).unpack(dtypes))


def _dense_weights(layers):
  """[W1, b1, W2, b2, ...] ([inputs, outputs] and [outputs]) of a stack of built 1x1 convolutions."""
  layers = list(layers)
  if any(not layer.built for layer in layers):
    raise RuntimeError("the entropy-parameter layers are not built: call build() first")
  return [t for layer in layers for t in (layer.kernel.reshape(layer.kernel.shape[-2:]), layer.bias)]


def checkerboard_mask(kernel_size=5):
  """[k, k]: 1 at the offsets (dy, dx) from the centre with dy + dx odd (12 for k = 5), 0 elsewhere.  Centred on a
  non-anchor, every such tap is an anchor."""
  r = torch.arange(kernel_size)
  return ((r[:, None] + r[None, :]) % 2 == 1).to(torch.float32)


def anchor_mask(H, W, device=None, dtype=torch.float32):
  """[1, H, W, 1]: 1 at the anchors (r + c even), 0 at the non-anchors."""
  r, c = torch.arange(H, device=device), torch.arange(W, device=device)
  return ((r[:, None] + c[None, :]) % 2 == 0).to(dtype)[None, :, :, None]


class CheckerboardConv2D(MaskedConv2D):
  """MaskedConv2D with the checkerboard mask: 12 taps of odd parity around the centre."""

  def __init__(self, in_channels, filters):
    super().__init__(in_channels, filters)
    self.mask.copy_(checkerboard_mask(5)[:, :, None, None])


def checkerboard_context(context_model, y):
  """The context feature of the training path: nonanchor * context_model(anchor * y).  Anchors get 0 (bias
  included); a non-anchor gets its context model's output over the anchors around it."""
  a = anchor_mask(y.shape[1], y.shape[2], y.device, y.dtype)
  return (1 - a) * context_model(a * y)


class CheckerboardModel(MBT2018Model):
  """MBT2018Model with the checkerboard context model of He, Zheng, Sun, Wang & Qin (CVPR 2021): the same
  transforms, hyper prior, widths and entropy models; the 5x5 context model sees only the anchors (positions with
  r + c even), and anchors take a context feature of zero.  So coding is two passes in which every position is
  independent: the anchors' parameters from psi alone, then the non-anchors' from psi and the decoded anchors.

  Coding runs on the parameter passes (functional.cb_*): the strings are one index-mode encode of y in coding order
  (each image's anchors in raster order, then its non-anchors), the bytes of
  `LocationScaleIndexedEntropyModel.compress(y_cb, scale_index_cb, loc_cb)` of the coding-order tensors; the decoder
  makes two decode_index_f32 calls on one decoder handle."""

  _substream_decoder = True

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=192, num_scales=64, scale_min=.11, scale_max=256.,
               substreams=1):
    super().__init__(lmbda, num_filters, latent_depth, num_scales, scale_min, scale_max, substreams)
    self.context_model = CheckerboardConv2D(self.latent_depth, 2 * self.latent_depth)

  def _context(self, y_ctx):
    return checkerboard_context(self.context_model, y_ctx)

  _pack_weights = staticmethod(F.cb_pack_weights)

  def _groups(self):
    return (self.latent_depth,)

  def _encode_latents(self, y, psi):
    """(strings, y_hat, loc, index): y_hat [B, H, W, M]; loc and index in coding order [B, H * W, M] (substream
    order with substreams > 1)."""
    B, H, W = (int(d) for d in y.shape[:3])
    y_hat, y_cb, loc, index = F.cb_encode(self._packed, y.contiguous(), psi, self.num_scales,
                                          substreams=self.substreams)
    return self._coded(y_cb, loc, index, B, H, W), y_hat, loc, index

  def _decode_latents(self, strings, psi):
    handle = self._y_decoder(strings)
    y_hat = F.cb_decode(handle, self._packed, psi, self.num_scales, self.entropy_model.cdf_offset.to(psi.device),
                        substreams=self.substreams)
    self.entropy_model._finish_decode(handle)
    return y_hat

  def _encode_ragged(self, ys, psis):
    return F.cb_encode_ragged(self._packed, ys, psis, self.num_scales, substreams=self.substreams)[1:]

  def _decode_ragged(self, handle, psis, cdf_offset):
    return F.cb_decode_ragged(handle, self._packed, psis, self.num_scales, cdf_offset, substreams=self.substreams)


class CheckerboardMixtureModel(_Model):
  """The checkerboard context model with a discretized mixture prior on y (Cheng et al., CVPR 2020, without the
  attention modules).  N = num_filters, M = latent_depth (a multiple of 6), K = num_components (in [1, 64]).
  CheckerboardModel's transforms, psi of width 2M and CheckerboardConv2D(M, 2M) context model; the entropy-parameter
  layers are 1x1 4M -> 10M/3 -> 8M/3 -> 3KM with LeakyReLU between them, channel c reading its K logits, K locs and K
  scales from outputs 3Kc .. 3Kc + 3K - 1 as MixtureHyperpriorModel reads its hyper synthesis.  z is coded as in
  MixtureHyperpriorModel, y by entropy_models.MixtureEntropyModel's coder.

  Coding runs on the checkerboard's two parameter passes (functional.cbm_*, DESIGN §3.19): every latent is coded as
  int32(rint(y)), so y_hat does not depend on the parameters; the anchors' mixtures come from psi alone, the
  non-anchors' from psi and the decoded anchors.  An image's y string is varint(len A) ‖ A ‖ N, A and N the
  MixtureEntropyModel strings of its anchors' and its non-anchors' coding-order latents (each with `substreams`
  substreams).  The hyper synthesis runs per image, so an image's strings do not depend on its batch or list."""

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=192, num_components=3, family="normal", substreams=1):
    super().__init__()
    self._set_substreams(substreams)
    N, M, K = int(num_filters), int(latent_depth), int(num_components)
    if M <= 0 or M % 6:
      raise ValueError(f"latent_depth must be a positive multiple of 6 (3M/2, 10M/3 and 8M/3 are layer widths): {M}")
    if K < 1 or K > 64:
      raise ValueError(f"num_components must be in [1, 64]: {K}")
    if family not in F.MIXTURE_FAMILIES:
      raise ValueError(f"`family` must be one of {sorted(F.MIXTURE_FAMILIES)}: {family!r}")
    self.num_components, self.family = K, family
    MBT2018Model._init_transforms(self, lmbda, N, M, 64, .11, 256.)
    self.context_model = CheckerboardConv2D(M, 2 * M)
    ep = lambda f, name, act: _conv(f, 1, name, kernel_parameter="variable", activation=act)
    self.entropy_parameters = nn.Sequential(
        ep(10 * M // 3, "layer_0", _leaky), ep(8 * M // 3, "layer_1", _leaky), ep(3 * K * M, "layer_2", None))
    self.hyperprior = D.NoisyDeepFactorized(batch_shape=(N,))
    self.entropy_model = E.MixtureEntropyModel(family, coding_rank=3)
    self.side_entropy_model = None
    self._packed = None

  _psi = MBT2018Model._psi

  def mixture_parameters(self, y_ctx, psi):
    """The parallel (training) form of the parameter network: (weight, loc, scale), each [B, H, W, M, K], from the
    latents the context model sees and psi [B, H, W, 2M]; weights are a softmax, scales bounded below at 0.11."""
    params = self.entropy_parameters(torch.cat([psi, checkerboard_context(self.context_model, y_ctx)], dim=-1))
    return MixtureHyperpriorModel.mixture_parameters(self, params)

  def forward(self, x, training=True):
    """-> (loss, bpp, mse).  The context model sees y plus uniform noise when training, round(y) otherwise; the rate
    of y goes through the NoisyNormalMixture / NoisyLogisticMixture graph."""
    side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3, compression=False)
    x = x.to(torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y)
    z_hat, side_bits = side_entropy_model(z, training=training)
    psi = self.hyper_synthesis_transform(z_hat)[:, :y.shape[1], :y.shape[2], :]
    y_ctx = y + torch.empty_like(y).uniform_(-.5, .5) if training else torch.round(y)
    y_hat, bits = self.entropy_model(y, *self.mixture_parameters(y_ctx, psi), training=training)
    self._last_x_hat = self.synthesis_transform(y_hat)[:, :x.shape[1], :x.shape[2], :]
    return self.rate_distortion(x, bits.sum() + side_bits.sum())

  def fix_tables(self):
    """Builds z's coding tables and packs the parameter network for the coding kernels (call again after the weights
    change)."""
    self.side_entropy_model = E.ContinuousBatchedEntropyModel(self.hyperprior, coding_rank=3,
                                                              compression=True).to(self._device())
    self._packed = F.cbm_pack_weights(self.context_model.kernel, self.context_model.bias,
                                      *_dense_weights(self.entropy_parameters))
    return self

  def _coder(self):
    return dict(substreams=self.substreams, **self.entropy_model._coder_args())

  def compress(self, x):
    """uint8 [H, W, 3] -> (string, side_string, x_shape, y_shape, z_shape), bmshj2018's signature."""
    return self.compress_batch(_as_image(x)[None])

  def decompress(self, string, side_string, x_shape, y_shape, z_shape):
    return self.decompress_batch(string, side_string, x_shape, y_shape, z_shape)[0]

  @torch.no_grad()
  def compress_batch(self, x):
    x = _as_batch(x).to(device=self._device(), dtype=torch.float32)
    y = self.analysis_transform(x)
    z = self.hyper_analysis_transform(y)
    shapes = tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
    side_string = self.side_entropy_model.compress(z, substreams=self.substreams)
    psi = self._psi(self.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
    string = F.cbm_encode(self._packed, self.num_components, y.contiguous(), psi, **self._coder())[1]
    return (string, side_string) + shapes

  @torch.no_grad()
  def decompress_batch(self, string, side_string, x_shape, y_shape, z_shape):
    z_hat = self.side_entropy_model.decompress(side_string, tuple(int(v) for v in z_shape), substreams=self.substreams)
    psi = self._psi(z_hat, (int(y_shape[0]), int(y_shape[1])))
    if not isinstance(string, gen_ops.Strings):
      string = gen_ops.Strings.from_bytes(string)
    y_hat = F.cbm_decode(gen_ops.Strings(string.bytes_dev, string.offsets_dev, (string.numel(),)), self._packed,
                         self.num_components, psi, **self._coder())
    x_hat = self.synthesis_transform(y_hat)
    return _to_uint8(x_hat[:, :int(x_shape[0]), :int(x_shape[1]), :])

  @torch.no_grad()
  def compress_images(self, images):
    """images: list of uint8 [H_i, W_i, 3] -> the list of what `compress(image)` returns, element for element.  The
    transforms run per image; z and y of the whole list are each coded in one ragged launch sequence."""
    xs = [_as_image(x)[None].to(device=self._device(), dtype=torch.float32) for x in images]
    if not xs:
      raise ValueError("`images` is empty")
    ys = [self.analysis_transform(x) for x in xs]
    zs = [self.hyper_analysis_transform(y) for y in ys]
    side_strings = self.side_entropy_model.compress_ragged([z[0] for z in zs], substreams=self.substreams).split()
    psis = [self._psi(self.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))[0] for y, z in zip(ys, zs)]
    strings = F.cbm_encode_ragged(self._packed, self.num_components, [y[0] for y in ys], psis,
                                  **self._coder())[1].split()
    return [(strings[i], side_strings[i]) + tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
            for i, (x, y, z) in enumerate(zip(xs, ys, zs))]

  @torch.no_grad()
  def decompress_images(self, items):
    """items: tuples as `compress_images` returns them -> list of uint8 [H_i, W_i, 3]."""
    items = list(items)
    if not items:
      raise ValueError("`items` is empty")
    z_hats = self.side_entropy_model.decompress_ragged(gen_ops.Strings.concat([it[1] for it in items]),
                                                       [tuple(int(v) for v in it[4]) for it in items],
                                                       substreams=self.substreams)
    psis = [self._psi(z_hat[None], (int(it[3][0]), int(it[3][1])))[0] for z_hat, it in zip(z_hats, items)]
    y_hats = F.cbm_decode_ragged(gen_ops.Strings.concat([it[0] for it in items]), self._packed, self.num_components,
                                 psis, **self._coder())
    out = []
    for y_hat, it in zip(y_hats, items):
      x_hat = self.synthesis_transform(y_hat[None])
      out.append(_to_uint8(x_hat[:, :int(it[2][0]), :int(it[2][1]), :])[0])
    return out

  def decompress_from_tfci(self, data):
    dtypes = [bytes, bytes, torch.int32, torch.int32, torch.int32]
    return self.decompress(*PackedTensors(data).unpack(dtypes))


class SpaceChannelModel(MBT2018Model):
  """The space-channel context model (SCCTX) of ELIC (He, Yang, Peng, Ma, Qin & Wang, CVPR 2022) on MBT2018Model's
  analysis, synthesis and hyper transforms (psi of 2M) and entropy models.  y is split into the uneven channel
  groups `groups` (c_0, ..., c_{K-1}), summing to M; group k holds channels [o_k, o_k + c_k).  Each group is coded
  in two checkerboard passes (CheckerboardModel's anchors and taps), conditioned on psi, on the groups before it
  (the channel context g_ch^k(y_hat[..., :o_k]), 2c_k wide, none for k = 0) and on its own decoded anchors (the
  spatial context, a CheckerboardConv2D(c_k, 2c_k)).  The group's entropy parameters are three 1x1 layers with
  LeakyReLU, K1 -> 5 K1 / 6 -> 2 K1 / 3 -> 2c_k on [psi, channel ctx, spatial ctx] of width K1 (MBT2018's ratios,
  so with one group the widths are MBT2018's).  g_ch^k is MS2020's slice transform stack (5x5 -> 224, 5x5 -> 128,
  3x3 -> 2c_k); in coding it runs one image at a time, so nothing depends on the batch.

  Coding runs on the group passes (functional.scc_*): one string per image, the bytes of
  `LocationScaleIndexedEntropyModel.compress(y_cc, scale_index_cc, loc_cc)` of the coding-order tensors [B, H W M]
  (group 0's anchors, group 0's non-anchors, group 1's anchors, ..., each in raster order); the decoder makes 2K
  decode_index_f32 calls on one decoder handle."""

  _substream_decoder = True

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=320, groups=(16, 16, 32, 64, 192), num_scales=64,
               scale_min=.11, scale_max=256., substreams=1):
    _Model.__init__(self)
    self._set_substreams(substreams)
    N, M = int(num_filters), int(latent_depth)
    groups = tuple(int(c) for c in groups)
    if M <= 0 or M % 2:
      raise ValueError(f"latent_depth must be a positive even number (3M/2 is a layer width): {M}")
    if not groups or min(groups) < 1:
      raise ValueError(f"every group needs at least one channel: {groups}")
    if sum(groups) != M:
      raise ValueError(f"the groups {groups} hold {sum(groups)} channels, but latent_depth is {M}")
    self.groups = groups
    self.spans = F.scc_spans(groups)
    self._init_transforms(lmbda, N, M, num_scales, scale_min, scale_max)
    self.context_models = nn.ModuleList([self._spatial_context_model(c) for c in groups])
    self.channel_context_transforms = nn.ModuleList([_MS2020SliceTransform(2 * c) for c in groups[1:]])
    ep = lambda f, name, act: _conv(f, 1, name, kernel_parameter="variable", activation=act)
    stacks = []
    for k, c in enumerate(groups):
      k1 = 2 * M + (2 * c if k else 0) + 2 * c
      stacks.append(nn.Sequential(ep(5 * k1 // 6, "layer_0", _leaky), ep(2 * k1 // 3, "layer_1", _leaky),
                                  ep(2 * c, "layer_2", None)))
    self.entropy_parameters = nn.ModuleList(stacks)
    self._init_entropy_models(N)

  def entropy_parameters_of(self, y_ctx, psi):
    """The parallel (training) form: (loc, scale_index) [B, H, W, M] of every position from the latents both
    contexts see and psi."""
    locs, scales = [], []
    for k, (o, c) in enumerate(self.spans):
      parts = [psi]
      if k:
        parts.append(self.channel_context_transforms[k - 1](y_ctx[..., :o]))
      parts.append(self._spatial_context(k, y_ctx[..., o:o + c]))
      params = self.entropy_parameters[k](torch.cat(parts, dim=-1))
      locs.append(params[..., :c])
      scales.append(params[..., c:])
    return torch.cat(locs, dim=-1), torch.cat(scales, dim=-1)

  @staticmethod
  def _spatial_context_model(c):
    """The spatial context model of a group of c channels."""
    return CheckerboardConv2D(c, 2 * c)

  def _spatial_context(self, k, y):
    """The training form's spatial context [B, H, W, 2c_k] of group k from its channels y [B, H, W, c_k]."""
    return checkerboard_context(self.context_models[k], y)

  def _channel_context(self, k, y_hat):
    """g_ch^k of y_hat[..., :o_k] [B, H, W, 2c_k], one image at a time."""
    o = self.spans[k][0]
    g = self.channel_context_transforms[k - 1]
    return torch.cat([g(y_hat[i:i + 1, ..., :o]) for i in range(y_hat.shape[0])]).contiguous()

  def _channel_contexts(self, k, y_hats):
    """g_ch^k of each y_hat[..., :o_k] of a list of [H_i, W_i, M]: a list of [H_i, W_i, 2c_k]."""
    o = self.spans[k][0]
    g = self.channel_context_transforms[k - 1]
    return [g(y_hat[None, ..., :o])[0] for y_hat in y_hats]

  def _pack(self):
    M = self.latent_depth
    return [F.scc_pack_weights(M, span, cm.kernel, cm.bias, *_dense_weights(ep))
            for span, cm, ep in zip(self.spans, self.context_models, self.entropy_parameters)]

  def _groups(self):
    return self.groups

  def _encode_latents(self, y, psi):
    """(strings, y_hat, loc, index): y_hat [B, H, W, M]; loc and index in coding order [B, H W M] (substream order
    with substreams > 1)."""
    B, H, W = (int(d) for d in y.shape[:3])
    y_hat, y_cc, loc, index = F.scc_encode(self._packed, self.groups, y.contiguous(), psi, self._channel_context,
                                           self.num_scales, substreams=self.substreams)
    return self._coded(y_cc, loc, index, B, H, W), y_hat, loc, index

  def _decode_latents(self, strings, psi):
    handle = self._y_decoder(strings)
    y_hat = F.scc_decode(handle, self._packed, self.groups, psi, self._channel_context, self.num_scales,
                         self.entropy_model.cdf_offset.to(psi.device), substreams=self.substreams)
    self.entropy_model._finish_decode(handle)
    return y_hat

  def _encode_ragged(self, ys, psis):
    return F.scc_encode_ragged(self._packed, self.groups, ys, psis, self._channel_contexts, self.num_scales,
                               substreams=self.substreams)[1:]

  def _decode_ragged(self, handle, psis, cdf_offset):
    return F.scc_decode_ragged(handle, self._packed, self.groups, psis, self._channel_contexts, self.num_scales,
                               cdf_offset, substreams=self.substreams)


def multistage_mask(stage, kernel_size=5):
  """[k, k]: 1 at the offsets (dy, dx) from the centre whose neighbour lies in a stage before `stage` of the 2x2
  schedule (functional.MSC_TAPS: 0, 4, 12 and 16 taps at k = 5), 0 elsewhere.  The mask is the same at every
  position of the stage."""
  h = kernel_size // 2
  m = torch.zeros(kernel_size, kernel_size)
  for dy, dx in F.MSC_TAPS[stage]:
    if abs(dy) <= h and abs(dx) <= h:
      m[dy + h, dx + h] = 1
  return m


def multistage_stage_map(H, W, device=None):
  """[H, W] int64: the stage of each position, (0,0) -> 0, (1,1) -> 1, (0,1) -> 2, (1,0) -> 3 on (r mod 2, c mod 2)."""
  r, c = torch.arange(H, device=device) % 2, torch.arange(W, device=device) % 2
  table = torch.tensor([[0, 2], [3, 1]], device=device)
  return table[r[:, None], c[None, :]]


class MultistageConv2D(MaskedConv2D):
  """MaskedConv2D with the mask of one stage s >= 1 of the 2x2 schedule (multistage_mask(s))."""

  def __init__(self, in_channels, filters, stage):
    super().__init__(in_channels, filters)
    self.stage = int(stage)
    self.mask.copy_(multistage_mask(self.stage)[:, :, None, None])


def multistage_context(context_models, y):
  """The context feature of the training path: sum over s of [stage(p) = s] * context_models[s - 1](y)(p) for the
  stages s = 1, 2, 3.  Stage 0 gets 0 (bias included); a position of stage s gets its stage's masked convolution,
  which reads only positions of earlier stages."""
  stage = multistage_stage_map(y.shape[1], y.shape[2], y.device)[None, :, :, None]
  out = torch.zeros(y.shape[:3] + (2 * y.shape[3],), device=y.device, dtype=y.dtype)
  for s, cm in enumerate(context_models, 1):
    out = out + (stage == s).to(y.dtype) * cm(y)
  return out


class MultistageModel(MBT2018Model):
  """MBT2018Model with a multistage spatial context (after Lin et al., ICASSP 2023): the same transforms, hyper
  prior, widths and entropy models.  Each 2x2 patch of the latent is coded in four stages, (0,0), (1,1), (0,1),
  (1,0) by (r mod 2, c mod 2); stage 0 takes a context feature of zero, and stage s >= 1 has its own 5x5 context
  model M -> 2M (a MultistageConv2D) that sees the stages before it: 4, 12 and 16 taps.  The three 1x1 entropy-
  parameter layers are shared by the stages.  All positions of a stage are independent, so coding is four parallel
  passes, and only a quarter of the positions code without spatial context (half with CheckerboardModel).

  Coding runs on the parameter passes (functional.msc_*): the strings are one index-mode encode of y in coding order
  (each image's stage 0 in raster order, then stages 1, 2 and 3), the bytes of
  `LocationScaleIndexedEntropyModel.compress(y_ms, scale_index_ms, loc_ms)` of the coding-order tensors; the decoder
  makes four decode_index_f32 calls on one decoder handle."""

  _substream_decoder = True

  def __init__(self, lmbda=0.01, num_filters=192, latent_depth=192, num_scales=64, scale_min=.11, scale_max=256.,
               substreams=1):
    _Model.__init__(self)
    self._set_substreams(substreams)
    N, M = int(num_filters), int(latent_depth)
    if M <= 0 or M % 6:
      raise ValueError(f"latent_depth must be a positive multiple of 6 (3M/2, 10M/3 and 8M/3 are layer widths): {M}")
    self._init_transforms(lmbda, N, M, num_scales, scale_min, scale_max)
    self.context_models = nn.ModuleList([MultistageConv2D(M, 2 * M, s) for s in (1, 2, 3)])
    ep = lambda f, name, act: _conv(f, 1, name, kernel_parameter="variable", activation=act)
    self.entropy_parameters = nn.Sequential(
        ep(10 * M // 3, "layer_0", _leaky), ep(8 * M // 3, "layer_1", _leaky), ep(2 * M, "layer_2", None))
    self._init_entropy_models(N)

  def _context(self, y_ctx):
    return multistage_context(self.context_models, y_ctx)

  def _pack(self):
    return F.msc_pack_weights([cm.kernel for cm in self.context_models], [cm.bias for cm in self.context_models],
                              *_dense_weights(self.entropy_parameters))

  def _coded(self, y, loc, index, B, H, W):
    lengths = None
    if self.substreams > 1:
      lengths = F.msc_substreams([H] * B, [W] * B, self.latent_depth, self.substreams)[0]
    return self._compress_coding_order(y, loc, index, lengths, B)

  def _encode_latents(self, y, psi):
    """(strings, y_hat, loc, index): y_hat [B, H, W, M]; loc and index in coding order [B, H * W, M] (substream
    order with substreams > 1)."""
    B, H, W = (int(d) for d in y.shape[:3])
    y_hat, y_ms, loc, index = F.msc_encode(self._packed, y.contiguous(), psi, self.num_scales,
                                           substreams=self.substreams)
    return self._coded(y_ms, loc, index, B, H, W), y_hat, loc, index

  def _decode_latents(self, strings, psi):
    handle = self._y_decoder(strings)
    y_hat = F.msc_decode(handle, self._packed, psi, self.num_scales, self.entropy_model.cdf_offset.to(psi.device),
                         substreams=self.substreams)
    self.entropy_model._finish_decode(handle)
    return y_hat

  def _encode_ragged(self, ys, psis):
    return F.msc_encode_ragged(self._packed, ys, psis, self.num_scales, substreams=self.substreams)[1:]

  def _decode_ragged(self, handle, psis, cdf_offset):
    return F.msc_decode_ragged(handle, self._packed, psis, self.num_scales, cdf_offset, substreams=self.substreams)


class SpaceChannelMultistageModel(SpaceChannelModel):
  """SpaceChannelModel with each channel group coded in the four stages of MultistageModel's 2x2 schedule (DESIGN
  §3.17): the same transforms, channel groups, channel-context stacks, entropy-parameter stacks and entropy models.
  Group k's spatial context is 0 at stage 0 and, at stage s >= 1, its own MultistageConv2D(c_k, 2c_k, s) over the
  group's channels at the earlier stages' positions (4, 12 and 16 taps); `context_models[k]` holds the three.  The
  group's entropy-parameter layers are shared by its four stages.  So only a quarter of each group's positions code
  without spatial context (half with SpaceChannelModel), and every stage is position-parallel.

  Coding runs on the group passes (functional.mscc_*): one string per image, the bytes of
  `LocationScaleIndexedEntropyModel.compress(y_cc, scale_index_cc, loc_cc)` of the coding-order tensors [B, H W M]
  (group 0's stages 0, 1, 2, 3, then group 1's, ..., each in raster order); the decoder makes 4K decode_index_f32
  calls on one decoder handle.  With groups = (M,) and M a multiple of 6 the strings are MultistageModel's with the
  same weights."""

  @staticmethod
  def _spatial_context_model(c):
    return nn.ModuleList([MultistageConv2D(c, 2 * c, s) for s in (1, 2, 3)])

  def _spatial_context(self, k, y):
    return multistage_context(self.context_models[k], y)

  def _pack(self):
    M = self.latent_depth
    return [F.mscc_pack_weights(M, span, [cm.kernel for cm in cms], [cm.bias for cm in cms], *_dense_weights(ep))
            for span, cms, ep in zip(self.spans, self.context_models, self.entropy_parameters)]

  def _coded(self, y, loc, index, B, H, W):
    lengths = None
    if self.substreams > 1:
      lengths = F.context_substreams(self.groups, [H] * B, [W] * B, self.substreams, multistage=True)[0]
    return self._compress_coding_order(y, loc, index, lengths, B)

  def _encode_latents(self, y, psi):
    """(strings, y_hat, loc, index): y_hat [B, H, W, M]; loc and index in coding order [B, H W M] (substream order
    with substreams > 1)."""
    B, H, W = (int(d) for d in y.shape[:3])
    y_hat, y_cc, loc, index = F.mscc_encode(self._packed, self.groups, y.contiguous(), psi, self._channel_context,
                                            self.num_scales, substreams=self.substreams)
    return self._coded(y_cc, loc, index, B, H, W), y_hat, loc, index

  def _decode_latents(self, strings, psi):
    handle = self._y_decoder(strings)
    y_hat = F.mscc_decode(handle, self._packed, self.groups, psi, self._channel_context, self.num_scales,
                          self.entropy_model.cdf_offset.to(psi.device), substreams=self.substreams)
    self.entropy_model._finish_decode(handle)
    return y_hat

  def _encode_ragged(self, ys, psis):
    return F.mscc_encode_ragged(self._packed, self.groups, ys, psis, self._channel_contexts, self.num_scales,
                                substreams=self.substreams)[1:]

  def _decode_ragged(self, handle, psis, cdf_offset):
    return F.mscc_decode_ragged(handle, self._packed, self.groups, psis, self._channel_contexts, self.num_scales,
                                cdf_offset, substreams=self.substreams)


# ------------------------------------------------------------------------------------------------
# bench extra: BASELINE.json configs[1] / [2] as the configs name them (images -> strings, strings -> images)
# ------------------------------------------------------------------------------------------------
def _stage_ms(fn, reps=5):
  """Median device time of one call (event between consecutive calls); two warm-up calls that keep the previous
  result alive like the timed loop, so that no cudaMalloc of an output lands inside the timed region."""
  out = None
  for _ in range(2):
    out = fn()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
  torch.cuda.synchronize()
  ev[0].record()
  for i in range(reps):
    out = fn()
    ev[i + 1].record()
  torch.cuda.synchronize()
  ts = sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
  return ts[len(ts) // 2], out


def bench_model_paths(dev, batch2=256, batch3=128, hw=256):
  """Times image batch -> strings and strings -> image batch for both models with a per-stage breakdown.  The conv
  stages are cuDNN glue and are reported only so that the coder / GDN share of the path is visible."""
  out = {}
  g = torch.Generator().manual_seed(1)
  for name, model, batch in (("cfg2_bls2017", BLS2017Model(num_filters=128), batch2),
                             ("cfg3_bmshj2018", BMSHJ2018Model(num_filters=192), batch3)):
    torch.manual_seed(3)
    model.build(dev).fix_tables()
    x = torch.randint(0, 256, (batch, hw, hw, 3), generator=g, dtype=torch.uint8).to(dev)
    enc_ms, packed = _stage_ms(lambda: model.compress_batch(x))
    dec_ms, x_hat = _stage_ms(lambda: model.decompress_batch(*packed))
    xf = x.float()
    ana_ms, y = _stage_ms(lambda: model.analysis_transform(xf))
    if name == "cfg2_bls2017":
      code_ms, strings = _stage_ms(lambda: model.entropy_model.compress(y))
      n_sym = y.numel()
      nbytes = strings.nbytes()
      decode_ms, y_hat = _stage_ms(lambda: model.entropy_model.decompress(strings, tuple(y.shape[1:-1])))
    else:
      z = model.hyper_analysis_transform(y.abs())
      idx = model.hyper_synthesis_transform(model.side_entropy_model.quantize(z))[:, :y.shape[1], :y.shape[2], :]
      code_ms, (s_y, s_z) = _stage_ms(lambda: (model.entropy_model.compress(y, idx), model.side_entropy_model.compress(z)))
      n_sym = y.numel() + z.numel()
      nbytes = s_y.nbytes() + s_z.nbytes()
      decode_ms, y_hat = _stage_ms(lambda: (model.side_entropy_model.decompress(s_z, tuple(z.shape[1:-1])),
                                            model.entropy_model.decompress(s_y, idx))[1])
    syn_ms, _ = _stage_ms(lambda: model.synthesis_transform(y_hat))
    gdn_ms = 0.0
    h = xf * (1 / 255.)
    for layer in list(model.analysis_transform)[1:]:
      act, layer.activation = layer.activation, None
      pre = layer(h)
      layer.activation = act
      if isinstance(act, GDN):
        ms, h = _stage_ms(lambda: act(pre))
        gdn_ms += ms
      else:
        h = pre if act is None else act(pre)
    out[name] = {
        "images": f"[{batch},{hw},{hw},3] uint8 (synthetic, seed 1), random-init weights",
        "compress_ms": enc_ms, "decompress_ms": dec_ms,
        "images_per_s_compress": batch / (enc_ms * 1e-3), "images_per_s_decompress": batch / (dec_ms * 1e-3),
        "stages_ms": {"analysis_transform (cuDNN convs + GDN kernels)": ana_ms, "of which GDN kernels": gdn_ms,
                      "entropy models compress (quantise + range encode + pack)": code_ms,
                      "entropy models decompress": decode_ms,
                      "synthesis_transform (cuDNN transposed convs + IGDN kernels)": syn_ms},
        "symbols": int(n_sym), "bits_per_pixel": 8.0 * nbytes / (batch * hw * hw),
        "coder_msym_s": n_sym / (code_ms * 1e-3) / 1e6,
        "reconstruction_shape": list(x_hat.shape), "round_trip_is_uint8": bool(x_hat.dtype == torch.uint8),
    }
    del model, x, xf, y, y_hat, x_hat, packed
    torch.cuda.empty_cache()
  return out
