"""CPU: the joint autoregressive + hierarchical prior model (MBT2018Model) without a device -- the type-A mask, the
training path's causality on the CPU, construction and the width rule, and the tfcb_ar_* entries' bindings and the
argument checks they make before any device work."""
import ctypes as C

import pytest
import torch

from compression_b200 import _lib
from compression_b200 import functional as F
from compression_b200 import models

AR_SYMBOLS = ("tfcb_ar_packed_floats", "tfcb_ar_pack_weights", "tfcb_ar_params", "tfcb_ar_encode", "tfcb_ar_decode")


def test_mask_is_type_a_with_twelve_taps_in_raster_order():
  m = models.causal_mask(5)
  assert m.shape == (5, 5)
  flat = m.reshape(-1)
  assert int(flat.sum()) == 12
  assert flat[:12].eq(1).all() and flat[12:].eq(0).all()  # the centre (12) and everything after it are masked
  assert m[2, 2] == 0


def test_masked_conv_is_causal_on_the_cpu():
  torch.manual_seed(0)
  conv = models.MaskedConv2D(6, 12)
  x = torch.randn(1, 5, 7, 6)
  base = conv(x)
  for p in (0, 9, 17, 34):
    py, px = divmod(p, 7)
    x2 = x.clone()
    x2.view(1, 35, 6)[:, p:] += torch.randn(1, 35 - p, 6)  # change position p and everything after it
    out = conv(x2).view(1, 35, 12)
    assert torch.equal(out[:, :p + 1], base.view(1, 35, 12)[:, :p + 1]), p  # position p sees only earlier ones


@pytest.mark.parametrize("M", [6, 96, 192, 384])
def test_model_widths(M):
  m = models.MBT2018Model(num_filters=32, latent_depth=M)
  assert m.analysis_transform[-1].filters == M
  assert [l.filters for l in m.hyper_synthesis_transform] == [M, 3 * M // 2, 2 * M]
  assert [l.filters for l in m.entropy_parameters] == [10 * M // 3, 8 * M // 3, 2 * M]
  assert tuple(m.context_model.kernel.shape) == (5, 5, M, 2 * M)
  assert F.ar_packed_floats(M) == (12 * M * 2 * M + 2 * M + 4 * M * (10 * M // 3) + 10 * M // 3 +
                                   (10 * M // 3) * (8 * M // 3) + 8 * M // 3 + (8 * M // 3) * 2 * M + 2 * M)


@pytest.mark.parametrize("M", [0, 4, 128, 190, -6])
def test_width_rule_rejects_depths_that_are_not_multiples_of_six(M):
  with pytest.raises(ValueError, match="multiple of 6"):
    models.MBT2018Model(latent_depth=M)


def test_every_ar_symbol_is_declared_exported_and_bound():
  with open(_lib.HEADER_PATH) as f:
    header = f.read()
  raw = C.CDLL(_lib.LIB_PATH)
  for name in AR_SYMBOLS:
    assert f" {name}(" in header, name
    assert hasattr(raw, name), name
    assert name in _lib.SIGNATURES, name


def test_packed_size_query():
  lib = _lib.lib()
  assert lib.tfcb_ar_packed_floats(192) == F.ar_packed_floats(192)
  for M in (0, 128, 390, -6):
    assert lib.tfcb_ar_packed_floats(M) == -1
  with pytest.raises(_lib.InvalidArgumentError, match="multiple of 6"):
    F.ar_packed_floats(128)


_FAKE = C.c_void_p(0x1000)  # never dereferenced: every call below fails its checks first


def _params(**kw):
  a = dict(packed=_FAKE, n=F.ar_packed_floats(12), M=12, yhat=_FAKE, psi=_FAKE, B=2, H=3, W=4, p=0, ns=64,
           loc=None, scale=None, index=None)
  a.update(kw)
  return _lib.lib().tfcb_ar_params(a["packed"], a["n"], a["M"], a["yhat"], a["psi"], a["B"], a["H"], a["W"], a["p"],
                                   a["ns"], a["loc"], a["scale"], a["index"], None)


@pytest.mark.parametrize("kw, match", [
    (dict(M=128), "multiple of 6"), (dict(M=390), "multiple of 6"), (dict(n=7), "packed weights hold 7"),
    (dict(packed=None), "`packed` is null"), (dict(B=0), "batch size"), (dict(H=0), "latent shape"),
    (dict(W=-1), "latent shape"), (dict(p=12), r"positions \[12, 13\)"), (dict(p=-1), "positions"),
    (dict(ns=0), "num_scales"), (dict(yhat=None), "null"), (dict(psi=None), "null")])
def test_params_rejections(kw, match):
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_params(**kw))
  assert _lib.launch_count() == n0


def test_encode_and_decode_rejections():
  lib = _lib.lib()
  n = F.ar_packed_floats(12)
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="null"):
    _lib.check(lib.tfcb_ar_encode(_FAKE, n, 12, _FAKE, _FAKE, 1, 2, 2, 0, 4, 64, _FAKE, None, _FAKE, None, None))
  with pytest.raises(_lib.InvalidArgumentError, match=r"positions \[3, 2\)"):
    _lib.check(lib.tfcb_ar_encode(_FAKE, n, 12, _FAKE, _FAKE, 1, 2, 2, 3, 2, 64, _FAKE, _FAKE, _FAKE, None, None))
  with pytest.raises(_lib.InvalidArgumentError, match=r"positions \[0, 5\)"):
    _lib.check(lib.tfcb_ar_encode(_FAKE, n, 12, _FAKE, _FAKE, 1, 2, 2, 0, 5, 64, _FAKE, _FAKE, _FAKE, None, None))
  with pytest.raises(_lib.InvalidArgumentError, match="not a decoder"):
    _lib.check(lib.tfcb_ar_decode(None, _FAKE, n, 12, _FAKE, 1, 2, 2, 0, 4, 64, _FAKE, _FAKE, None))
  with pytest.raises(_lib.InvalidArgumentError, match="null"):
    _lib.check(lib.tfcb_ar_pack_weights(12, _FAKE, None, _FAKE, _FAKE, _FAKE, _FAKE, _FAKE, _FAKE, _FAKE, n, None))
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    _lib.check(lib.tfcb_ar_pack_weights(12, *([_FAKE] * 9), n + 1, None))
  assert _lib.launch_count() == n0


def test_python_wrappers_reject_before_the_library():
  M = 12
  with pytest.raises(_lib.InvalidArgumentError, match=r"\[5, 5, M, 2M\]"):
    F.ar_pack_weights(torch.zeros(3, 3, M, 2 * M), *([None] * 7))
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.ar_pack_weights(torch.zeros(5, 5, M, 2 * M), *([None] * 7))
  packed = torch.zeros(F.ar_packed_floats(M))
  psi = torch.zeros(1, 2, 2, 2 * M)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.ar_params(torch.zeros(5), torch.zeros(1, 2, 2, M), psi, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.ar_params(packed, torch.zeros(1, 2, 2, M), psi, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match=r"\[B, H, W, 2M\]"):
    F.ar_encode(packed, torch.zeros(1, 2, 2, M), torch.zeros(1, 2, 2, 2 * M + 1), 64)
  with pytest.raises(_lib.InvalidArgumentError, match="empty"):
    F.ar_encode(packed, torch.zeros(0, 2, 2, M), torch.zeros(0, 2, 2, 2 * M), 64)
