"""CPU: the host side of the context models' ragged-list entries (§3.13).  Their argument checks run before any device
work, the workspace sizes and the list layout follow the formulas of the design, and tools/rd_eval.py takes the
context models and the mixed-size list."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest

from compression_b200 import _lib
from compression_b200 import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(1, 1), (1, 5), (5, 1), (2, 2), (3, 7), (17, 9), (32, 48)]


def _host(a):
  return a.ctypes.data_as(C.c_void_p)


def _list(shapes):
  return (np.ascontiguousarray([h for h, _ in shapes], dtype=np.int64),
          np.ascontiguousarray([w for _, w in shapes], dtype=np.int64))


def _net_widths(M, o, c):
  k1 = 2 * M + (2 * c if o else 0) + 2 * c
  return k1, 5 * k1 // 6, 2 * k1 // 3


def test_workspace_sizes_follow_the_layout():
  lib = _lib.lib()
  hs, ws = _list(SHAPES)
  for M, o, c in ((12, 0, 12), (24, 6, 6), (320, 128, 192)):
    _, n3, n4 = _net_widths(M, o, c)
    for anchors in (1, 0):
      n_k = (hs * ws + 1) // 2 if anchors else hs * ws // 2
      want = 8 * hs.size + int(n_k.sum()) * ((0 if anchors else 2 * c) + n3 + n4)
      assert lib.tfcb_scc_ragged_workspace_floats(M, o, c, hs.size, _host(hs), _host(ws), anchors) == want
  assert lib.tfcb_ar_ragged_workspace_floats(5) == 20
  for n in (0, -1):
    assert lib.tfcb_ar_ragged_workspace_floats(n) == -1
    assert lib.tfcb_scc_ragged_workspace_floats(12, 0, 12, n, _host(hs), _host(ws), 1) == -1
  bad_h = np.array([3, 0], dtype=np.int64)
  assert lib.tfcb_scc_ragged_workspace_floats(12, 0, 12, 2, _host(bad_h), _host(ws), 1) == -1
  big = np.array([1 << 16, 1 << 16], dtype=np.int64)
  assert lib.tfcb_scc_ragged_workspace_floats(12, 0, 12, 2, _host(big), _host(big), 1) == -1
  assert lib.tfcb_scc_ragged_workspace_floats(12, 0, 12, 2, None, _host(ws), 1) == -1
  assert lib.tfcb_scc_ragged_workspace_floats(13, 0, 13, 2, _host(hs), _host(ws), 1) == -1  # odd M


def test_list_views_start_at_the_pixel_prefix():
  import torch
  hs, ws = _list(SHAPES)
  M = 6
  flat = torch.arange(int((hs * ws).sum()) * M, dtype=torch.float32)
  views = F._ragged_views(flat, hs, ws, M)
  P = np.concatenate([[0], np.cumsum(hs * ws)])
  for i, v in enumerate(views):
    assert tuple(v.shape) == (hs[i], ws[i], M)
    assert int(v.reshape(-1)[0]) == M * P[i] and v.data_ptr() == flat.data_ptr() + 4 * M * int(P[i])


def test_pass_lengths_are_the_colour_counts():
  hs, ws = _list(SHAPES)
  for anchors in (True, False):
    counts = (hs * ws + 1) // 2 if anchors else hs * ws // 2
    assert counts.tolist() == [F.cb_counts(h, w)[0 if anchors else 1] for h, w in SHAPES]
  assert F.cb_counts(1, 1) == (1, 0)


def _null_args(lib, **over):
  hs, ws = over.pop("list", _list(SHAPES))
  M, o, c = over.pop("group", (12, 0, 12))
  n = over.pop("n", None)
  if n is None:
    n = lib.tfcb_scc_packed_floats(M, o, c, None)
  a = dict(packed=C.c_void_p(16), n=n, M=M, o=o, c=c, yhat=None,
           psi=C.c_void_p(16), ch=None, k=over.pop("k", hs.size), hs=_host(hs), ws=_host(ws), anchors=1,
           ns=over.pop("ns", 64), work=C.c_void_p(16), nw=over.pop("nw", 1 << 40), whole=0, loc=None, scale=None,
           index=None, y=None, y_cb=None, y_out=None, stream=None)
  return list(a.values())


@pytest.mark.parametrize("case, msg", [
    (dict(group=(12, 0, 13)), "does not fit"), (dict(group=(13, 0, 13)), "even"), (dict(n=7), "packed"),
    (dict(k=0), "list"), (dict(list=_list([(3, 7), (0, 5)])), "image 1"), (dict(list=_list([(70000, 70000)])),
                                                                          "image 0"),
    (dict(ns=0), "num_scales"), (dict(nw=3), "workspace")])
def test_params_ragged_rejects_before_any_launch(case, msg):
  lib = _lib.lib()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=msg):
    _lib.check(lib.tfcb_scc_params_ragged(*_null_args(lib, **case)))
  assert _lib.launch_count() == n0


def test_ar_and_scatter_ragged_reject_before_any_launch():
  lib = _lib.lib()
  hs, ws = _list(SHAPES)
  n0 = _lib.launch_count()
  packed_n = F.ar_packed_floats(12)
  good = dict(packed=C.c_void_p(16), n=packed_n, M=12, y=C.c_void_p(16), psi=C.c_void_p(16), k=hs.size,
              hs=_host(hs), ws=_host(ws), ns=64, work=C.c_void_p(16), nw=4 * hs.size, yhat=C.c_void_p(16),
              loc=C.c_void_p(16), index=C.c_void_p(16), scale=None, stream=None)
  for over, msg in ((dict(M=10), "multiple of 6"), (dict(n=packed_n + 1), "packed"), (dict(k=0), "list"),
                    (dict(hs=None), "null"), (dict(nw=4 * hs.size - 1), "workspace"), (dict(y=None), "null"),
                    (dict(ns=0), "num_scales")):
    with pytest.raises(_lib.InvalidArgumentError, match=msg):
      _lib.check(lib.tfcb_ar_encode_ragged(*{**good, **over}.values()))
  with pytest.raises(_lib.InvalidArgumentError, match="decoder"):
    _lib.check(lib.tfcb_ar_decode_ragged(None, C.c_void_p(16), packed_n, 12, C.c_void_p(16), hs.size, _host(hs),
                                         _host(ws), 64, C.c_void_p(16), C.c_void_p(16), 28, C.c_void_p(16), None))
  with pytest.raises(_lib.InvalidArgumentError, match="workspace"):
    _lib.check(lib.tfcb_scc_scatter_ragged(C.c_void_p(16), hs.size, _host(hs), _host(ws), 12, 0, 12, 1,
                                           C.c_void_p(16), 8 * hs.size - 1, C.c_void_p(16), None))
  with pytest.raises(_lib.InvalidArgumentError, match="list"):
    _lib.check(lib.tfcb_scc_scatter_ragged(C.c_void_p(16), 0, _host(hs), _host(ws), 12, 0, 12, 1, C.c_void_p(16),
                                           1 << 20, C.c_void_p(16), None))
  assert _lib.launch_count() == n0


def test_python_lists_are_checked():
  import torch
  with pytest.raises(_lib.InvalidArgumentError, match="non-empty"):
    F.ar_encode_ragged(torch.zeros(3), [], [], 64)
  with pytest.raises(_lib.InvalidArgumentError, match="one M"):
    F.cb_params_ragged(torch.zeros(3), None, [torch.zeros(2, 2, 24), torch.zeros(2, 2, 12)], True, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="empty latents"):
    F.cb_params_ragged(torch.zeros(3), None, [torch.zeros(0, 2, 24)], True, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="packed"):
    F.cb_params_ragged(torch.zeros(3), None, [torch.zeros(2, 2, 24)], True, 64)


def _rd_eval():
  spec = importlib.util.spec_from_file_location("rd_eval", os.path.join(ROOT, "tools", "rd_eval.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_rd_eval_takes_the_context_models_and_the_mixed_list():
  rd = _rd_eval()
  for name in ("mbt2018", "checkerboard", "space_channel"):
    args = rd.parser().parse_args(["--synthetic", "mixed", "--model", name])
    assert args.model == name and args.synthetic == "mixed"
  shapes = rd.mixed_shapes(0)
  assert len(shapes) == 24 and len({(h // 16, w // 16) for h, w in shapes}) == 24
  assert all(h % 16 == 0 and w % 16 == 0 and 256 <= min(h, w) and max(h, w) <= 1024 for h, w in shapes)
  assert shapes == rd.mixed_shapes(0) != rd.mixed_shapes(1)
  imgs = rd.synthetic(0, shapes[:2])
  assert [tuple(x.shape) for x in imgs] == [shapes[0] + (3,), shapes[1] + (3,)]
