"""CPU: the checkerboard context model without a device -- the mask, the colours and the coding order, the training
path's dependencies in float64, the float32 emulation against float64 and its sensitivity to a wrong gather, the
tfcb_cb_* bindings and the checks they make before any device work, and the compiled kernels."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import functional as F
from compression_b200 import models
from oracle import ar_oracle
from oracle import checkerboard_oracle as cbo

CB_SYMBOLS = ("tfcb_cb_workspace_floats", "tfcb_cb_params", "tfcb_cb_scatter")
SHAPES = [(1, 1), (1, 2), (2, 1), (1, 9), (7, 1), (5, 7), (6, 8)]
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compression_b200", "csrc")


# ---------------------------------------------------------------------------------------------------------------
# definitions
# ---------------------------------------------------------------------------------------------------------------
def test_mask_has_twelve_taps_of_odd_parity_in_raster_order():
  m = models.checkerboard_mask(5)
  taps = [(y - 2, x - 2) for y in range(5) for x in range(5) if m[y, x] == 1]
  assert len(taps) == 12 and all((dy + dx) % 2 for dy, dx in taps)
  assert tuple(taps) == F.CB_TAPS == cbo.TAPS
  conv = models.CheckerboardConv2D(6, 12)
  assert torch.equal(conv.mask[:, :, 0, 0], m)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_colours_counts_and_coding_order(shape):
  H, W = shape
  a = models.anchor_mask(H, W)[0, :, :, 0]
  n_a, n_n = F.cb_counts(H, W)
  assert n_a == -(-H * W // 2) == int(a.sum()) and n_a + n_n == H * W
  order = cbo.coding_order(H, W)
  assert sorted(order.tolist()) == list(range(H * W))  # a permutation ...
  inverse = np.empty_like(order)
  inverse[order] = np.arange(H * W)
  assert np.array_equal(order[inverse], np.arange(H * W))  # ... with an inverse
  flat = a.reshape(-1)
  assert flat[order[:n_a]].eq(1).all() and flat[order[n_a:]].eq(0).all()
  assert np.all(np.diff(order[:n_a]) > 0) and np.all(np.diff(order[n_a:]) > 0)  # raster order within a colour
  for p in order[n_a:]:  # every tap of a non-anchor is an anchor
    py, px = divmod(int(p), W)
    for dy, dx in cbo.TAPS:
      if 0 <= py + dy < H and 0 <= px + dx < W:
        assert a[py + dy, px + dx] == 1


def test_training_path_dependencies_in_float64():
  torch.manual_seed(0)
  M, H, W = 6, 6, 7
  conv = models.CheckerboardConv2D(M, 2 * M).double()
  with torch.no_grad():
    conv.bias.normal_()
  y = torch.randn(1, H, W, M, dtype=torch.float64)
  base = models.checkerboard_context(conv, y)
  a = models.anchor_mask(H, W, dtype=torch.float64)[0, :, :, 0]
  assert base[0][a == 1].eq(0).all()  # anchors: zero, bias included
  with torch.no_grad():
    for p in range(H * W):
      py, px = divmod(p, W)
      y2 = y.clone()
      y2[0, py, px] += 1.0
      changed = (models.checkerboard_context(conv, y2) != base).any(-1)[0]
      if a[py, px] == 0:  # a non-anchor's latent changes no context
        assert not changed.any(), p
        continue
      want = torch.zeros(H, W, dtype=torch.bool)  # an anchor's changes exactly the non-anchors it is a tap of
      for dy, dx in cbo.TAPS:
        if 0 <= py - dy < H and 0 <= px - dx < W:
          want[py - dy, px - dx] = True
      assert torch.equal(changed, want), p


# ---------------------------------------------------------------------------------------------------------------
# the float32 emulation against float64
# ---------------------------------------------------------------------------------------------------------------
def _weights(M, seed):
  rng = np.random.default_rng(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: rng.standard_normal(s).astype(np.float32)
  return [r(5, 5, M, 2 * M) / np.sqrt(12 * M), 0.1 * r(2 * M), r(4 * M, n3) / np.sqrt(4 * M), 0.1 * r(n3),
          r(n3, n4) / np.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * M) / np.sqrt(n4),
          np.concatenate([0.5 * r(M), 24 + 4 * r(M)])]


def _inputs(B, H, W, M, seed):
  rng = np.random.default_rng(100 + seed)
  return (np.round(3 * rng.standard_normal((B, H, W, M))).astype(np.float32),
          rng.standard_normal((B, H, W, 2 * M)).astype(np.float32))


@pytest.mark.parametrize("M", [6, 18, 30, 96])
def test_emulation_holds_to_the_rounding_bound_layer_by_layer(M):
  ws = _weights(M, M)
  for H, W in ((5, 7), (1, 9), (6, 8)):
    y_hat, psi = _inputs(2, H, W, M, H)
    for anchors in (True, False):
      errs = cbo.layer_errors(ws, y_hat, psi, anchors)
      assert len(errs) == (3 if anchors else 4)
      for err, bound, mag in errs:
        assert np.all(err <= bound)
        assert np.all(bound <= 1e-4 * (1 + mag.max()))
      loc, scale, _ = cbo.params32(ws, y_hat, psi, anchors, 64)
      (l64, s64), (lb, sb) = cbo.params64(ws, y_hat, psi, anchors), cbo.bound64(ws, y_hat, psi, anchors)
      assert np.all(np.abs(loc - l64) <= lb) and np.all(np.abs(scale - s64) <= sb)


def test_a_wrong_gather_changes_the_bits():
  M, H, W = 6, 6, 7
  ws = _weights(M, 1)
  y_hat, psi = _inputs(1, H, W, M, 1)
  y_hat += 0.25 * np.arange(H * W, dtype=np.float32).reshape(1, H, W, 1)  # every position distinct
  want = cbo.params32(ws, y_hat, psi, False, 64)[0]
  type_a = tuple((t // 5 - 2, t % 5 - 2) for t in range(12))  # the causal taps of a type-A mask
  wrong = {
      "type-A taps": lambda y, pos: cbo.gather(y, pos, taps=type_a),
      "rows wrap": lambda y, pos: cbo.gather(y, pos, wrap=True),
  }
  for name, g in wrong.items():
    got = cbo.params32(ws, y_hat, psi, False, 64, gather_fn=g)[0]
    assert not np.array_equal(got.view(np.int32), want.view(np.int32)), name
  # the anchors' parameters read no latent at all
  a = cbo.params32(ws, y_hat, psi, True, 64)[0]
  assert np.array_equal(a.view(np.int32), cbo.params32(ws, 0 * y_hat, psi, True, 64)[0].view(np.int32))


def test_anchor_path_is_the_network_on_a_zero_context():
  """Skipping the ctx half at the anchors is the full network on [psi, 0] in float32, bit for bit."""
  M, H, W = 12, 5, 7
  ws = _weights(M, 2)
  y_hat, psi = _inputs(2, H, W, M, 2)
  zero_ctx = [ws[0], np.zeros_like(ws[1])] + ws[2:]
  pos = cbo.positions(H, W, True)
  x = np.zeros((2, len(pos), 12 * M), np.float32)
  out = ar_oracle.network32(cbo.packed_list(zero_ctx), x.reshape(-1, 12 * M),
                            psi.reshape(2, H * W, 2 * M)[:, pos].reshape(-1, 2 * M)).reshape(2, len(pos), -1)
  assert np.array_equal(out[..., :M].view(np.int32), cbo.params32(ws, y_hat, psi, True, 64)[0].view(np.int32))


# ---------------------------------------------------------------------------------------------------------------
# bindings and rejections
# ---------------------------------------------------------------------------------------------------------------
def test_every_cb_symbol_is_declared_exported_and_bound():
  with open(_lib.HEADER_PATH) as f:
    header = f.read()
  raw = C.CDLL(_lib.LIB_PATH)
  for name in CB_SYMBOLS:
    assert f" {name}(" in header, name
    assert hasattr(raw, name), name
    assert name in _lib.SIGNATURES, name


def test_workspace_query():
  lib = _lib.lib()
  M, B, H, W = 12, 3, 5, 7
  n3, n4 = 40, 32
  assert lib.tfcb_cb_workspace_floats(M, B, H, W, 1) == B * 18 * (n3 + n4)
  assert lib.tfcb_cb_workspace_floats(M, B, H, W, 0) == B * 17 * (2 * M + n3 + n4)
  for args in ((128, 1, 2, 2, 1), (12, 0, 2, 2, 1), (12, 1, 0, 2, 0), (12, 1, 2, -1, 0)):
    assert lib.tfcb_cb_workspace_floats(*args) == -1


_FAKE = C.c_void_p(0x1000)  # never dereferenced: every call below fails its checks first


def _params(**kw):
  a = dict(packed=_FAKE, n=F.ar_packed_floats(12), M=12, yhat=_FAKE, psi=_FAKE, B=2, H=3, W=4, anchors=0, ns=64,
           work=_FAKE, nwork=1 << 20, whole=0, loc=None, scale=None, index=None, y=None, y_cb=None, yhat_out=None)
  a.update(kw)
  return _lib.lib().tfcb_cb_params(a["packed"], a["n"], a["M"], a["yhat"], a["psi"], a["B"], a["H"], a["W"],
                                   a["anchors"], a["ns"], a["work"], a["nwork"], a["whole"], a["loc"], a["scale"],
                                   a["index"], a["y"], a["y_cb"], a["yhat_out"], None)


@pytest.mark.parametrize("kw, match", [
    (dict(M=128), "multiple of 6"), (dict(n=7), "packed weights hold 7"), (dict(packed=None), "`packed` is null"),
    (dict(B=0), "batch size"), (dict(H=0), "latent shape"), (dict(W=-1), "latent shape"), (dict(ns=0), "num_scales"),
    (dict(psi=None), "null"), (dict(yhat=None), "null"), (dict(work=None), "workspace"),
    (dict(nwork=100), "workspace of 100 floats"), (dict(y=_FAKE, loc=_FAKE), "the encoder needs")])
def test_params_rejections(kw, match):
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_params(**kw))
  assert _lib.launch_count() == n0


def test_scatter_rejections():
  lib = _lib.lib()
  n0 = _lib.launch_count()
  for args, match in (((_FAKE, 1, 2, 2, 0, 1, _FAKE), "M=0"), ((_FAKE, 0, 2, 2, 6, 1, _FAKE), "batch size"),
                      ((_FAKE, 1, 0, 2, 6, 1, _FAKE), "latent shape"), ((None, 1, 2, 2, 6, 1, _FAKE), "null")):
    with pytest.raises(_lib.InvalidArgumentError, match=match):
      _lib.check(lib.tfcb_cb_scatter(*args, None))
  assert _lib.launch_count() == n0


def test_python_wrappers_reject_before_the_library():
  M = 12
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=r"\[5, 5, M, 2M\]"):
    F.cb_pack_weights(torch.zeros(3, 3, M, 2 * M), *([None] * 7))
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.cb_pack_weights(torch.zeros(5, 5, M, 2 * M), *([None] * 7))
  packed = torch.zeros(F.ar_packed_floats(M))
  psi = torch.zeros(1, 2, 2, 2 * M)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.cb_params(torch.zeros(5), None, psi, True, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.cb_params(packed, None, psi, True, 64)
  with pytest.raises(_lib.InvalidArgumentError, match=r"\[B, H, W, 2M\]"):
    F.cb_encode(packed, torch.zeros(1, 2, 2, M), torch.zeros(1, 2, 2, 2 * M + 1), 64)
  with pytest.raises(_lib.InvalidArgumentError, match="empty"):
    F.cb_encode(packed, torch.zeros(0, 2, 2, M), torch.zeros(0, 2, 2, 2 * M), 64)
  assert _lib.launch_count() == n0


def test_model_widths_and_rule():
  m = models.CheckerboardModel(num_filters=32, latent_depth=12)
  assert isinstance(m.context_model, models.CheckerboardConv2D)
  assert tuple(m.context_model.kernel.shape) == (5, 5, 12, 24)
  assert [l.filters for l in m.entropy_parameters] == [40, 32, 24]
  with pytest.raises(ValueError, match="multiple of 6"):
    models.CheckerboardModel(latent_depth=128)


# ---------------------------------------------------------------------------------------------------------------
# compiled code
# ---------------------------------------------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
needs_nvcc = pytest.mark.skipif(NVCC is None, reason="nvcc is not installed")


def _compile(src, out, extra=()):
  cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(CSRC, "..", "..", "include"), "-I" + CSRC, *extra, "-c", os.path.join(CSRC, src), "-o",
         out]
  return subprocess.run(cmd, capture_output=True, text=True, check=True)


@needs_nvcc
def test_checkerboard_kernels_build_for_sm90a_without_spills(tmp_path):
  r = _compile("checkerboard.cu", str(tmp_path / "cb.o"), ["-Xptxas", "-v"])
  spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
  assert len(spills) == 5  # four dense-layer kernels and the scatter
  assert all(s == ("0", "0") for s in spills), r.stderr


# sha256 of ar_kernel's four instantiations' SASS (instructions only, in template order), as compiled by CUDA 12.9
# before the shared definitions moved to autoregressive.cuh
AR_KERNEL_SASS = ("12.9", "b7ea0ade940e0bed7882ad336f3ec58477cc6bce94e22f6d1892dfcc166927dc")


@needs_nvcc
def test_ar_kernel_sass_is_unchanged(tmp_path):
  version = re.search(r"release (\d+\.\d+)", subprocess.run([NVCC, "--version"], capture_output=True,
                                                             text=True).stdout).group(1)
  if version != AR_KERNEL_SASS[0]:
    pytest.skip(f"the reference hash is CUDA {AR_KERNEL_SASS[0]}'s, this is {version}")
  _compile("autoregressive.cu", str(tmp_path / "ar.o"))
  cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
  sass = subprocess.run([cuobjdump, "-sass", str(tmp_path / "ar.o")], capture_output=True, text=True,
                        check=True).stdout
  funcs, cur = {}, None
  for line in sass.splitlines():
    m = re.match(r"\s+Function : (\S+)", line)
    if m:
      cur = m.group(1)
      funcs[cur] = []
      continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;?\s*(/\*.*\*/)?\s*$", line)
    if cur and m:
      funcs[cur].append(m.group(1))
  names = sorted(n for n in funcs if "ar_kernel" in n)
  assert len(names) == 4
  digest = hashlib.sha256("\n".join("\n".join(funcs[n]) for n in names).encode()).hexdigest()
  assert digest == AR_KERNEL_SASS[1]
