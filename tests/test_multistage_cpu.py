"""CPU: the multistage context model without a device -- the tap sets and masks, the stages' counts and positions
and the coding order, the float32 emulation against its float64 bound, the training form's context against the
oracle's in float64, the tfcb_msc_* bindings and the checks they make before any device work, and the compiled
kernels (no spills; the checkerboard kernels' SASS pinned)."""
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
from oracle import multistage_oracle as mso

MSC_SYMBOLS = ("tfcb_msc_packed_floats", "tfcb_msc_pack_weights", "tfcb_msc_workspace_floats", "tfcb_msc_params",
               "tfcb_msc_scatter", "tfcb_msc_ragged_workspace_floats", "tfcb_msc_params_ragged",
               "tfcb_msc_scatter_ragged")
SHAPES = [(1, 1), (1, 2), (2, 1), (1, 7), (6, 1), (3, 5), (4, 6), (7, 9)]
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compression_b200", "csrc")


# ---------------------------------------------------------------------------------------------------------------
# definitions
# ---------------------------------------------------------------------------------------------------------------
def test_tap_sets_follow_the_schedule():
  assert [len(t) for t in F.MSC_TAPS] == [0, 4, 12, 16]
  assert F.MSC_TAPS == mso.TAPS
  assert F.MSC_TAPS[1] == ((-1, -1), (-1, 1), (1, -1), (1, 1))
  assert F.MSC_TAPS[2] == F.CB_TAPS
  assert set(F.MSC_TAPS[3]) == {(dy, dx) for dy in range(-2, 3) for dx in range(-2, 3) if dy % 2 or dx % 2}
  for s, taps in enumerate(F.MSC_TAPS):
    assert list(taps) == sorted(taps)  # raster order
    a, b = F.MSC_PHASES[s]
    for dy in range(-2, 3):  # exactly the neighbours in an earlier stage, wherever the position lies
      for dx in range(-2, 3):
        if (dy, dx) != (0, 0):
          assert ((dy, dx) in taps) == (F.msc_stage(a + dy, b + dx) < s)


def test_masks_are_the_tap_sets():
  for s in range(4):
    m = models.multistage_mask(s)
    assert [(y - 2, x - 2) for y in range(5) for x in range(5) if m[y, x] == 1] == list(F.MSC_TAPS[s])
  for s in (1, 2, 3):
    conv = models.MultistageConv2D(6, 12, s)
    assert torch.equal(conv.mask[:, :, 0, 0], models.multistage_mask(s))
  stage = models.multistage_stage_map(4, 5)
  for r in range(4):
    for c in range(5):
      assert stage[r, c] == F.msc_stage(r, c) == mso.stage_of(r, c)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_counts_positions_and_coding_order(shape):
  H, W = shape
  n = F.msc_counts(H, W)
  assert n == mso.counts(H, W) and sum(n) == H * W
  if H == 1:
    assert n[1] == n[3] == 0
  if W == 1:
    assert n[1] == n[2] == 0
  for s, (a, b) in enumerate(F.MSC_PHASES):
    ws = (W - b + 1) // 2
    want = [(a + 2 * (j // ws)) * W + b + 2 * (j % ws) for j in range(n[s])]  # the j-th position of the stage
    assert mso.positions(H, W, s) == want
  order = mso.coding_order(H, W)
  assert sorted(order.tolist()) == list(range(H * W))  # a permutation ...
  inverse = np.empty_like(order)
  inverse[order] = np.arange(H * W)
  assert np.array_equal(order[inverse], np.arange(H * W))  # ... with an inverse
  pos, wid = F.msc_phases([H, 2 * H], [W, W + 1], 12)
  assert pos[0].tolist() == list(n) and pos[1].tolist() == list(F.msc_counts(2 * H, W + 1))
  assert (wid == 12).all()


def test_every_tap_of_a_stage_is_decoded_before_it():
  H, W = 7, 9
  order = mso.coding_order(H, W).tolist()
  rank = {p: i for i, p in enumerate(order)}
  for s in range(4):
    first = min(rank[p] for p in mso.positions(H, W, s))
    for p in mso.positions(H, W, s):
      r, c = divmod(p, W)
      for dy, dx in F.MSC_TAPS[s]:
        if 0 <= r + dy < H and 0 <= c + dx < W:
          assert rank[(r + dy) * W + c + dx] < first


# ---------------------------------------------------------------------------------------------------------------
# the float32 emulation against float64, and the training form
# ---------------------------------------------------------------------------------------------------------------
def _weights(M, seed):
  rng = np.random.default_rng(seed)
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: rng.standard_normal(s).astype(np.float32)
  return [[r(5, 5, M, 2 * M) / np.sqrt(12 * M) for _ in range(3)], [0.1 * r(2 * M) for _ in range(3)],
          r(4 * M, n3) / np.sqrt(4 * M), 0.1 * r(n3), r(n3, n4) / np.sqrt(n3), 0.1 * r(n4),
          8 * r(n4, 2 * M) / np.sqrt(n4), np.concatenate([0.5 * r(M), 24 + 4 * r(M)])]


def _inputs(B, H, W, M, seed):
  rng = np.random.default_rng(100 + seed)
  return (np.round(3 * rng.standard_normal((B, H, W, M))).astype(np.float32),
          rng.standard_normal((B, H, W, 2 * M)).astype(np.float32))


@pytest.mark.parametrize("M", [6, 18, 48])
def test_emulation_holds_to_the_float64_bound(M):
  ws = _weights(M, M)
  for H, W in ((5, 7), (1, 9), (6, 1), (4, 4)):
    y_hat, psi = _inputs(2, H, W, M, H + W)
    for s in range(4):
      loc, scale, index = mso.params32(ws, y_hat, psi, s, 64)
      (l64, s64), (lb, sb) = mso.params64(ws, y_hat, psi, s), mso.bound64(ws, y_hat, psi, s)
      assert loc.shape == (2, F.msc_counts(H, W)[s], M)
      assert np.all(np.abs(loc - l64) <= lb) and np.all(np.abs(scale - s64) <= sb)


def test_stage_zero_reads_no_latent_and_other_stages_read_their_taps():
  M, H, W = 6, 6, 7
  ws = _weights(M, 1)
  y_hat, psi = _inputs(1, H, W, M, 1)
  a = mso.params32(ws, y_hat, psi, 0, 64)[0]
  assert np.array_equal(a.view(np.int32), mso.params32(ws, 0 * y_hat, psi, 0, 64)[0].view(np.int32))
  for s in (1, 2, 3):  # changing a latent of stage >= s changes nothing at stage s
    later = y_hat.copy()
    for p in range(H * W):
      if F.msc_stage(*divmod(p, W)) >= s:
        later.reshape(1, H * W, M)[0, p] += 5
    assert np.array_equal(mso.params32(ws, later, psi, s, 64)[0], mso.params32(ws, y_hat, psi, s, 64)[0])
    assert not np.array_equal(mso.params32(ws, y_hat + 1, psi, s, 64)[0], mso.params32(ws, y_hat, psi, s, 64)[0])


def test_training_context_is_the_oracles_per_stage_context_in_float64():
  torch.manual_seed(0)
  M, H, W = 6, 7, 6
  convs = [models.MultistageConv2D(M, 2 * M, s).double() for s in (1, 2, 3)]
  with torch.no_grad():
    for cv in convs:
      cv.bias.normal_()
    y = torch.randn(2, H, W, M, dtype=torch.float64)
    got = models.multistage_context(convs, y).numpy()
  want = mso.context64([cv.kernel.detach().numpy() for cv in convs], [cv.bias.detach().numpy() for cv in convs],
                       y.numpy())
  assert np.abs(got - want).max() <= 1e-12 * (1 + np.abs(want).max())
  stage = models.multistage_stage_map(H, W)
  assert (got[:, stage.numpy() == 0] == 0).all()  # stage 0: zero, bias included


# ---------------------------------------------------------------------------------------------------------------
# bindings and rejections
# ---------------------------------------------------------------------------------------------------------------
def test_every_msc_symbol_is_declared_exported_and_bound():
  with open(_lib.HEADER_PATH) as f:
    header = f.read()
  raw = C.CDLL(_lib.LIB_PATH)
  for name in MSC_SYMBOLS:
    assert f" {name}(" in header, name
    assert hasattr(raw, name), name
    assert name in _lib.SIGNATURES, name


def test_sizes():
  lib = _lib.lib()
  M = 12
  n3, n4 = 40, 32
  assert lib.tfcb_msc_packed_floats(M) == (4 + 12 + 16) * M * 2 * M + 3 * 2 * M + 4 * M * n3 + n3 + n3 * n4 + n4 + \
      n4 * 2 * M + 2 * M
  assert F.msc_packed_floats(M) == lib.tfcb_msc_packed_floats(M)
  for bad in (0, 8, 390):
    assert lib.tfcb_msc_packed_floats(bad) == -1
  B, H, W = 3, 5, 7
  for s, n in enumerate(F.msc_counts(H, W)):
    assert lib.tfcb_msc_workspace_floats(M, B, H, W, s) == B * n * ((2 * M if s else 0) + n3 + n4)
  for args in ((12, 1, 2, 2, 4), (12, 1, 2, 2, -1), (10, 1, 2, 2, 0), (12, 0, 2, 2, 0), (12, 1, 0, 2, 1)):
    assert lib.tfcb_msc_workspace_floats(*args) == -1
  hs, ws = np.array([1, 3], np.int64), np.array([4, 1], np.int64)
  h, w = hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p)
  for s in range(4):
    n = F.msc_counts(1, 4)[s] + F.msc_counts(3, 1)[s]
    assert lib.tfcb_msc_ragged_workspace_floats(M, 2, h, w, s) == 2 * 8 + n * ((2 * M if s else 0) + n3 + n4)
  assert lib.tfcb_msc_ragged_workspace_floats(M, 2, h, w, 4) == -1


_FAKE = C.c_void_p(0x1000)  # never dereferenced: every call below fails its checks first


def _params(**kw):
  a = dict(packed=_FAKE, n=F.msc_packed_floats(12), M=12, yhat=_FAKE, psi=_FAKE, B=2, H=3, W=4, stage=1, ns=64,
           work=_FAKE, nwork=1 << 20, whole=0, loc=None, scale=None, index=None, y=None, y_ms=None, yhat_out=None)
  a.update(kw)
  return _lib.lib().tfcb_msc_params(a["packed"], a["n"], a["M"], a["yhat"], a["psi"], a["B"], a["H"], a["W"],
                                    a["stage"], a["ns"], a["work"], a["nwork"], a["whole"], a["loc"], a["scale"],
                                    a["index"], a["y"], a["y_ms"], a["yhat_out"], None)


@pytest.mark.parametrize("kw, match", [
    (dict(M=128), "multiple of 6"), (dict(stage=4), "stage 4"), (dict(stage=-1), "stage -1"),
    (dict(n=7), "packed weights hold 7"), (dict(packed=None), "`packed` is null"), (dict(B=0), "batch size"),
    (dict(H=0), "latent shape"), (dict(W=-1), "latent shape"), (dict(ns=0), "num_scales"), (dict(psi=None), "null"),
    (dict(yhat=None), "null"), (dict(work=None), "workspace"), (dict(nwork=100), "workspace of 100 floats"),
    (dict(y=_FAKE, loc=_FAKE), "the encoder needs")])
def test_params_rejections(kw, match):
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_params(**kw))
  assert _lib.launch_count() == n0


def test_ragged_and_scatter_rejections():
  lib = _lib.lib()
  n = F.msc_packed_floats(12)
  hs, ws = np.array([2, 0], np.int64), np.array([3, 3], np.int64)
  h, w = hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p)
  n0 = _lib.launch_count()
  cases = [
      (lambda: lib.tfcb_msc_params_ragged(_FAKE, n, 12, _FAKE, _FAKE, 2, h, w, 0, 64, _FAKE, 1 << 20, 0, None, None,
                                          None, None, None, None, None), "image 1: latent shape 0 x 3"),
      (lambda: lib.tfcb_msc_params_ragged(_FAKE, n, 12, _FAKE, _FAKE, 0, h, w, 0, 64, _FAKE, 1 << 20, 0, None, None,
                                          None, None, None, None, None), "a list of 0 images"),
      (lambda: lib.tfcb_msc_params_ragged(_FAKE, n, 12, _FAKE, _FAKE, 1, h, w, 5, 64, _FAKE, 1 << 20, 0, None, None,
                                          None, None, None, None, None), "stage 5"),
      (lambda: lib.tfcb_msc_params_ragged(_FAKE, n, 12, _FAKE, _FAKE, 1, h, w, 1, 64, _FAKE, 10, 0, None, None,
                                          None, None, None, None, None), "workspace of 10 floats"),
      (lambda: lib.tfcb_msc_scatter_ragged(_FAKE, 1, h, w, 12, 0, None, 0, _FAKE, None), "workspace"),
      (lambda: lib.tfcb_msc_scatter_ragged(_FAKE, 2, h, w, 12, 0, _FAKE, 1 << 20, _FAKE, None), "latent shape"),
      (lambda: lib.tfcb_msc_scatter(_FAKE, 1, 2, 2, 0, 1, _FAKE, None), "M=0"),
      (lambda: lib.tfcb_msc_scatter(_FAKE, 1, 2, 2, 12, 4, _FAKE, None), "stage 4"),
      (lambda: lib.tfcb_msc_scatter(_FAKE, 0, 2, 2, 12, 0, _FAKE, None), "batch size"),
      (lambda: lib.tfcb_msc_scatter(_FAKE, 1, 0, 2, 12, 0, _FAKE, None), "latent shape"),
      (lambda: lib.tfcb_msc_scatter(None, 1, 2, 2, 12, 0, _FAKE, None), "null"),
      (lambda: lib.tfcb_msc_pack_weights(12, *([_FAKE] * 12), _FAKE, 7, None), "packed weights hold 7"),
      (lambda: lib.tfcb_msc_pack_weights(12, *([_FAKE] * 11), None, _FAKE, n, None), "operand 11 is null"),
      (lambda: lib.tfcb_msc_pack_weights(9, *([_FAKE] * 12), _FAKE, n, None), "M=9"),
  ]
  for call, match in cases:
    with pytest.raises(_lib.InvalidArgumentError, match=match):
      _lib.check(call())
  assert _lib.launch_count() == n0


def test_python_wrappers_reject_before_the_library():
  M = 12
  n0 = _lib.launch_count()
  k = torch.zeros(5, 5, M, 2 * M)
  with pytest.raises(_lib.InvalidArgumentError, match="each of stages"):
    F.msc_pack_weights([k, k], [None] * 2, *([None] * 6))
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.msc_pack_weights([k] * 3, [None] * 3, *([None] * 6))
  packed = torch.zeros(F.msc_packed_floats(M))
  psi = torch.zeros(1, 2, 2, 2 * M)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.msc_params(torch.zeros(5), None, psi, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.msc_params(packed, None, psi, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="stage 4"):
    F.msc_params(packed, None, psi, 4, 64)
  with pytest.raises(_lib.InvalidArgumentError, match=r"\[B, H, W, 2M\]"):
    F.msc_encode(packed, torch.zeros(1, 2, 2, M), torch.zeros(1, 2, 2, 2 * M + 1), 64)
  with pytest.raises(_lib.InvalidArgumentError, match="empty"):
    F.msc_encode(packed, torch.zeros(0, 2, 2, M), torch.zeros(0, 2, 2, 2 * M), 64)
  assert _lib.launch_count() == n0


def test_model_widths_and_rule():
  m = models.MultistageModel(num_filters=32, latent_depth=12)
  assert not hasattr(m, "context_model")
  assert [cm.stage for cm in m.context_models] == [1, 2, 3]
  assert all(tuple(cm.kernel.shape) == (5, 5, 12, 24) for cm in m.context_models)
  assert [l.filters for l in m.entropy_parameters] == [40, 32, 24]
  assert models.MultistageModel(latent_depth=12, substreams=4).substreams == 4
  with pytest.raises(ValueError, match="multiple of 6"):
    models.MultistageModel(latent_depth=128)


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
def test_multistage_kernels_build_for_sm90a_without_spills(tmp_path):
  r = _compile("multistage.cu", str(tmp_path / "ms.o"), ["-Xptxas", "-v"])
  spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
  assert len(spills) == 5  # four dense-layer kernels and the scatter
  assert all(s == ("0", "0") for s in spills), r.stderr


# sha256 of checkerboard.cu's five kernels' SASS (instructions only, in name order), as compiled by CUDA 12.9 with the
# tile machinery in checkerboard.cuh.  Their PTX is the parent's instruction for instruction; ptxas picks different
# integer instructions in the tap-gathering kernel only because its shared arrays are now named after the shared body.
CB_KERNEL_SASS = ("12.9", "dd014caed9aded5e3953583a3415e97144582074d4c22eeaaddd14db47c90049")


@needs_nvcc
def test_checkerboard_kernel_sass_is_pinned(tmp_path):
  version = re.search(r"release (\d+\.\d+)", subprocess.run([NVCC, "--version"], capture_output=True,
                                                             text=True).stdout).group(1)
  if version != CB_KERNEL_SASS[0]:
    pytest.skip(f"the reference hash is CUDA {CB_KERNEL_SASS[0]}'s, this is {version}")
  _compile("checkerboard.cu", str(tmp_path / "cb.o"))
  cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
  sass = subprocess.run([cuobjdump, "-sass", str(tmp_path / "cb.o")], capture_output=True, text=True,
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
  names = sorted(funcs)
  assert len(names) == 5
  digest = hashlib.sha256("\n".join("\n".join(funcs[n]) for n in names).encode()).hexdigest()
  assert digest == CB_KERNEL_SASS[1]
