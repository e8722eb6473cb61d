"""CPU: the checkerboard context model with mixture priors (DESIGN §3.19) without a GPU: the y string's split at its
varint edges and its rejections, the float32 emulation of both passes and the epilogue against their float64
restatement within its bound, the C ABI's and the model's host checks (nothing launches), and the kernels' build."""
import concurrent.futures
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from compression_b200 import _lib, gen_ops, models
from compression_b200 import functional as F
from oracle import cb_mixture_oracle as cmo
from oracle import checkerboard_oracle as cbo

CSRC = os.path.join(os.path.dirname(__file__), "..", "compression_b200", "csrc")


# ---- the y string: varint(len A) ‖ A ‖ N ----
@pytest.mark.parametrize("na", [0, 1, 127, 128, 16383, 16384, 2**21])
@pytest.mark.parametrize("nn", [0, 5])
def test_split_at_the_varint_edges(na, nn):
  a, n = bytes(range(256)) * (na // 256) + bytes(na % 256), b"\x07" * nn
  s = gen_ops._varint(na) + a + n
  assert len(s) == len(gen_ops._varint(na)) + na + nn
  assert F.cbm_split(s) == (a, n)


@pytest.mark.parametrize("s,msg", [
    (b"", "truncated length"),
    (b"\x80", "truncated length"),
    (b"\xff" * 10 + b"\x01", "longer than 64 bits"),
    (b"\x80\x00", "minimal form"),
    (b"\x05abcd", "runs past the end of its 5 bytes"),
    (b"\x81\x01" + b"x" * 128, "129 bytes runs past"),
])
def test_split_rejects_damaged_lengths(s, msg):
  with pytest.raises(_lib.InvalidArgumentError, match=f"string 3: .*{msg}"):
    F.cbm_split(s, 3)


# ---- the oracle: float32 emulation against the float64 restatement ----
def _weights(rng, M, K):
  n3, n4 = 10 * M // 3, 8 * M // 3
  r = lambda *s: rng.standard_normal(s).astype(np.float32)
  b3 = np.stack([r(M, K), 0.5 * r(M, K), 1.5 + r(M, K)], 1).reshape(-1)
  return [r(5, 5, M, 2 * M) / np.sqrt(12 * M), 0.1 * r(2 * M), r(4 * M, n3) / np.sqrt(4 * M), 0.1 * r(n3),
          r(n3, n4) / np.sqrt(n3), 0.1 * r(n4), 2 * r(n4, 3 * K * M) / np.sqrt(n4), b3]


@pytest.mark.parametrize("M,K,H,W", [(6, 1, 1, 1), (6, 3, 3, 5), (12, 3, 4, 4), (6, 8, 2, 7), (6, 64, 1, 3)])
def test_emulation_lies_within_the_float64_bound(M, K, H, W):
  rng = np.random.default_rng(M * 100 + K)
  ws = [w.astype(np.float32) for w in _weights(rng, M, K)]
  y = (3 * rng.standard_normal((2, H, W, M))).astype(np.float32)
  psi = rng.standard_normal((2, H, W, 2 * M)).astype(np.float32)
  y_hat = np.rint(y)
  for anchors in (True, False):
    raw = cmo.raw32(ws, y_hat, psi, anchors)
    assert raw.shape == (2, cbo.counts(H, W)[0 if anchors else 1], 3 * K * M)
    if raw.shape[1] == 0:
      continue
    exact, bound = cmo.raw64(ws, y_hat, psi, anchors)
    err = np.abs(raw.astype(np.float64) - exact)
    assert (err <= bound).all() and (bound < 1e-2).all()
    got = cmo.epilogue32(raw, K)
    want = cmo.epilogue64(exact, K)
    bounds = cmo.epilogue_bound64(exact, bound, K)
    for g, w, b in zip(got, want, bounds):
      assert (np.abs(g.astype(np.float64) - w) <= b).all()


def test_epilogue_definitions_at_their_edges():
  raw = np.array([[3.0, np.nan, -1.0, 0.5, 0.25, -7.0, 0.01, 0.2, 1e-30]], np.float32)  # one channel, K = 3
  w, mu, s = cmo.epilogue32(raw, 3)
  assert w[0, 0, 0] == 1 and np.isnan(w[0, 0, 1])  # the largest logit ignores NaN; a NaN logit stays NaN
  assert w[0, 0, 2] == np.float32(np.exp(np.float64(np.float32(-4.0))))
  np.testing.assert_array_equal(mu[0, 0], np.float32([0.5, 0.25, -7.0]))
  np.testing.assert_array_equal(s[0, 0], np.float32([0.11, 0.2, 0.11]))
  w1, _, _ = cmo.epilogue32(np.float32([[-1e30, 2.0, 3.0]]), 1)
  assert w1[0, 0, 0] == 1  # K = 1: every weight is 1


# ---- host checks: the C ABI (no pointer dereferenced, nothing launched) and the model ----
_P = C.c_void_p(256)
M, K = 12, 3


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _params_call(ragged, **kw):
  L = _lib.lib()
  n = int(L.tfcb_cbm_packed_floats(M, K, None))
  a = dict(packed=_P, pf=n, M=M, K=K, yhat=_P, psi=_P, B=2, H=4, W=5, anchors=1, work=_P, wf=1 << 40, whole=0,
           w=_P, l=_P, s=_P, y=None, ycb=None, yho=None)
  a.update(kw)
  if not ragged:
    return L.tfcb_cbm_params(*a.values(), None)
  hs, ws = np.int64([4, 1]), np.int64([5, 1])
  if a["H"] == 0:
    hs[1] = 0
  v = list(a.values())
  return L.tfcb_cbm_params_ragged(*v[:6], 2, hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p),
                                  *v[9:], None)


PARAM_CASES = [
    (dict(M=10), "multiple of 6"),
    (dict(M=390), "multiple of 6 and at most 384"),
    (dict(K=0), "`K` must be in \\[1, 64\\]"),
    (dict(K=65), "`K` must be in \\[1, 64\\]"),
    (dict(pf=7), "packed weights hold 7 floats"),
    (dict(packed=None), "`packed` is null"),
    (dict(psi=None), "`psi` or `yhat` is null"),
    (dict(anchors=0, yhat=None), "`psi` or `yhat` is null"),
    (dict(wf=10), "workspace of 10 floats"),
    (dict(work=None), "workspace of 0 floats"),
    (dict(w=None), "`weight`, `loc` or `scale` is null"),
    (dict(s=None), "`weight`, `loc` or `scale` is null"),
    (dict(y=_P), "the encoder needs `y_cb` and `yhat_out`"),
    (dict(H=0), "latent shape|out of range"),
]


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("kw,msg", PARAM_CASES, ids=lambda x: str(x))
def test_abi_rejects_before_any_launch(ragged, kw, msg):
  n0 = _lib.launch_count()

  def run():
    rc = _params_call(ragged, **kw)
    return rc, _lib.lib().tfcb_last_error().decode()
  rc, err = _on_worker(run)
  assert rc == _lib.INVALID_ARGUMENT
  assert re.search(msg, err), err
  assert _lib.launch_count() == n0


def test_abi_sizes_and_pack_rejections():
  L = _lib.lib()
  lay = np.zeros(12, np.int64)
  n = int(L.tfcb_cbm_packed_floats(M, K, lay.ctypes.data_as(C.POINTER(C.c_int64))))
  d = F.cbm_layout(M, K)
  assert n == d["total"] == d["b3"] + 3 * K * M and list(lay) == [d[k] for k in F.CBM_LAYOUT_KEYS]
  assert (d["K1"], d["N3"], d["N4"], d["NO"]) == (4 * M, 10 * M // 3, 8 * M // 3, 3 * K * M)
  assert d["w3"] - d["b2"] == d["N4"] and d["b3"] - d["w3"] == d["N4"] * d["NO"]
  for m, k in ((10, 3), (0, 3), (390, 3), (12, 0), (12, 65)):
    assert L.tfcb_cbm_packed_floats(m, k, None) == -1
    assert L.tfcb_cbm_workspace_floats(m, k, 1, 4, 4, 1) == -1
  assert L.tfcb_cbm_workspace_floats(M, K, 0, 4, 4, 1) == -1
  assert L.tfcb_cbm_workspace_floats(M, K, 1, 4, 4, 1) == 8 * (10 * M // 3 + 8 * M // 3 + 3 * K * M)
  assert L.tfcb_cbm_workspace_floats(M, K, 1, 4, 4, 0) == 8 * (2 * M + 10 * M // 3 + 8 * M // 3 + 3 * K * M)
  hs, ws = np.int64([3, 1]), np.int64([3, 1])
  got = L.tfcb_cbm_ragged_workspace_floats(M, K, 2, hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p), 1)
  assert got == 2 * 8 + 6 * (10 * M // 3 + 8 * M // 3 + 3 * K * M)  # the table (32 bytes an image), 5 + 1 anchors
  with pytest.raises(_lib.InvalidArgumentError, match="multiple of 6"):
    F.cbm_layout(8, 3)
  n0 = _lib.launch_count()

  def run():
    rcs = [L.tfcb_cbm_pack_weights(M, K, *[_P] * 8, _P, n - 1, None),
           L.tfcb_cbm_pack_weights(M, 65, *[_P] * 8, _P, n, None),
           L.tfcb_cbm_pack_weights(M, K, *[_P] * 7, None, _P, n, None)]
    return rcs
  assert _on_worker(run) == [_lib.INVALID_ARGUMENT] * 3
  assert _lib.launch_count() == n0


def test_model_constructor_checks():
  m = models.CheckerboardMixtureModel(num_filters=16, latent_depth=12, num_components=4, family="logistic")
  assert [l.filters for l in m.entropy_parameters] == [40, 32, 3 * 4 * 12]
  assert tuple(m.context_model.kernel.shape) == (5, 5, 12, 24)
  assert m.hyper_synthesis_transform[-1].filters == 24
  assert m.entropy_model.family == "logistic" and m.substreams == 1
  assert models.CheckerboardMixtureModel(latent_depth=12, substreams=8).substreams == 8
  with pytest.raises(ValueError, match="multiple of 6"):
    models.CheckerboardMixtureModel(latent_depth=8)
  for k in (0, 65):
    with pytest.raises(ValueError, match="num_components"):
      models.CheckerboardMixtureModel(latent_depth=12, num_components=k)
  with pytest.raises(ValueError, match="family"):
    models.CheckerboardMixtureModel(latent_depth=12, family="laplace")
  with pytest.raises(ValueError, match="substreams"):
    models.CheckerboardMixtureModel(latent_depth=12, substreams=0)


def test_functional_family_check_comes_first():
  with pytest.raises(_lib.InvalidArgumentError, match="family"):
    F.cbm_encode(None, K, None, None, family="laplace")
  with pytest.raises(_lib.InvalidArgumentError, match="family"):
    F.cbm_decode([b""], None, K, None, family="gaussian")


# ---- compiled code ----
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


@pytest.mark.skipif(NVCC is None, reason="nvcc is not installed")
def test_kernels_build_for_sm90a_without_spills(tmp_path):
  cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(CSRC, "..", "..", "include"), "-I" + CSRC, "-Xptxas", "-v", "-c",
         os.path.join(CSRC, "cb_mixture.cu"), "-o", str(tmp_path / "cbm.o")]
  r = subprocess.run(cmd, capture_output=True, text=True, check=True)
  spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
  assert len(spills) == 4  # three dense-layer kernels and the epilogue
  assert all(s == ("0", "0") for s in spills), r.stderr
