"""CPU: the space-channel context model without a device -- the float32 emulation of each group pass against float64
layer by layer, its one-group case against the checkerboard emulation, its sensitivity to a wrong gather, a
misplaced segment or a swapped group order, the model's arguments and coding-order layout, and the tfcb_scc_*
bindings and the checks they make before any device work."""
import ctypes as C

import numpy as np
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import functional as F
from compression_b200 import models
from oracle import checkerboard_oracle as cbo
from oracle import space_channel_oracle as sco

SCC_SYMBOLS = ("tfcb_scc_packed_floats", "tfcb_scc_pack_weights", "tfcb_scc_workspace_floats", "tfcb_scc_params",
               "tfcb_scc_scatter")


def _group_weights(M, k, c, rng):
  k1, n3, n4 = sco.widths(M, k, c)
  r = lambda *s: rng.standard_normal(s).astype(np.float32)
  return [r(5, 5, c, 2 * c) / np.sqrt(12 * c), 0.1 * r(2 * c), r(k1, n3) / np.sqrt(k1), 0.1 * r(n3),
          r(n3, n4) / np.sqrt(n3), 0.1 * r(n4), 8 * r(n4, 2 * c) / np.sqrt(n4),
          np.concatenate([0.5 * r(c), 24 + 4 * r(c)])]


def _weights(groups, seed):
  rng = np.random.default_rng(seed)
  return [_group_weights(sum(groups), k, c, rng) for k, c in enumerate(groups)]


def _inputs(B, H, W, M, seed):
  rng = np.random.default_rng(100 + seed)
  return (np.round(3 * rng.standard_normal((B, H, W, M))).astype(np.float32),
          rng.standard_normal((B, H, W, 2 * M)).astype(np.float32))


def _ch(B, H, W, c, seed):
  return np.random.default_rng(200 + seed).standard_normal((B, H, W, 2 * c)).astype(np.float32)


def _bits(a):
  return np.asarray(a).view(np.int32)


# ---------------------------------------------------------------------------------------------------------------
# the float32 emulation against float64, and against the checkerboard emulation
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [(6,), (1, 5), (2, 4, 6, 12)], ids=str)
def test_emulation_holds_to_the_rounding_bound_layer_by_layer(groups):
  M = sum(groups)
  ws = _weights(groups, M)
  for H, W in ((5, 7), (1, 9)):
    y_hat, psi = _inputs(2, H, W, M, H)
    for k, (g, w) in enumerate(zip(sco.spans(groups), ws)):
      ch = _ch(2, H, W, g[1], k) if k else None
      for anchors in (True, False):
        errs = sco.layer_errors(w, g, y_hat, psi, ch, anchors)
        assert len(errs) == (3 if anchors else 4)
        for err, bound, mag in errs:
          assert np.all(err <= bound)
          assert np.all(bound <= 1e-4 * (1 + mag.max()))
        loc, scale, _ = sco.params32(w, g, y_hat, psi, ch, anchors, 64)
        (l64, s64), (lb, sb) = sco.params64(w, g, y_hat, psi, ch, anchors), sco.bound64(w, g, y_hat, psi, ch, anchors)
        assert np.all(np.abs(loc - l64) <= lb) and np.all(np.abs(scale - s64) <= sb)


@pytest.mark.parametrize("M", [6, 12, 30])
def test_one_group_is_the_checkerboard_emulation_bit_for_bit(M):
  ws = _weights((M,), M)[0]
  assert sco.widths(M, 0, M) == (4 * M, 10 * M // 3, 8 * M // 3)
  for H, W in ((1, 1), (5, 7), (6, 8)):
    y_hat, psi = _inputs(2, H, W, M, W)
    for anchors in (True, False):
      got = sco.params32(ws, (0, M), y_hat, psi, None, anchors, 64)
      want = cbo.params32(ws, y_hat, psi, anchors, 64)
      for g, w in zip(got, want):
        assert np.array_equal(_bits(g), _bits(w)), (H, W, anchors)
  y = _inputs(2, 5, 7, M, 3)[0] + 0.3
  psi = _inputs(2, 5, 7, M, 4)[1]
  got = sco.encode32([ws], (M,), y, psi, None, 64)
  want = cbo.encode32(ws, y, psi, 64)
  for g, w in zip(got, want):
    assert np.array_equal(_bits(g).reshape(-1), _bits(w).reshape(-1))


def test_a_wrong_layout_changes_the_bits():
  groups = (2, 2, 2)
  M, H, W = 6, 5, 7
  ws = _weights(groups, 1)
  y_hat, psi = _inputs(1, H, W, M, 1)
  y_hat += 0.25 * np.arange(H * W * M, dtype=np.float32).reshape(1, H, W, M)  # every latent distinct
  g, ch = (2, 2), _ch(1, H, W, 2, 1)
  want = sco.params32(ws[1], g, y_hat, psi, ch, False, 64)[0]
  wrong = {
      "another group's channels": sco.params32(ws[1], (4, 2), y_hat, psi, ch, False, 64)[0],
      "rows wrap": sco.params32(ws[1], g, y_hat, psi, ch, False, 64,
                                gather_fn=lambda y, pos: cbo.gather(y, pos, wrap=True))[0],
      "ctx before the channel context": sco.params32(ws[1], g, y_hat, psi, ch, False, 64,
                                                     segments=("psi", "ctx", "ch"))[0],
      "psi last": sco.params32(ws[1], g, y_hat, psi, ch, False, 64, segments=("ch", "ctx", "psi"))[0],
  }
  for name, got in wrong.items():
    assert not np.array_equal(_bits(got), _bits(want)), name
  # at the anchors the spatial context is zero: a misplaced zero segment changes the bits too
  a = sco.params32(ws[1], g, y_hat, psi, ch, True, 64)[0]
  assert not np.array_equal(_bits(a), _bits(sco.params32(ws[1], g, y_hat, psi, ch, True, 64,
                                                         segments=("psi", "ctx", "ch"))[0]))
  # the anchors read no latent
  assert np.array_equal(_bits(a), _bits(sco.params32(ws[1], g, 0 * y_hat, psi, ch, True, 64)[0]))
  # swapping the order of two groups of equal size changes the encoder's bits
  y = y_hat + 0.3
  chf = lambda k, yh: yh[..., [j % (2 * k) for j in range(4)]] * np.float32(0.5)
  base = sco.encode32(ws, groups, y, psi, chf, 64)
  swapped = sco.encode32([ws[0], ws[2], ws[1]], groups, y, psi, chf, 64)
  assert not np.array_equal(_bits(base[2]), _bits(swapped[2]))


def test_coding_order_layout():
  groups, H, W = (1, 2, 3), 3, 5
  M = sum(groups)
  order = sco.coding_order(H, W, groups)
  assert sorted(order.tolist()) == list(range(H * W * M))
  n_a, n_n = F.cb_counts(H, W)
  at = 0
  for o, c in F.scc_spans(groups):
    for anchors, n in ((True, n_a), (False, n_n)):
      block = order[at:at + n * c].reshape(n, c)
      assert np.array_equal(block // M, np.repeat(np.array(cbo.positions(H, W, anchors))[:, None], c, 1))
      assert np.array_equal(block % M, np.tile(np.arange(o, o + c), (n, 1)))
      at += n * c
  y = np.arange(H * W * M, dtype=np.float32).reshape(1, H, W, M)
  ws = _weights(groups, 3)
  y_cc = sco.encode32(ws, groups, y, _inputs(1, H, W, M, 3)[1], lambda k, yh: np.zeros((1, H, W, 2 * groups[k]),
                                                                                      np.float32), 64)[1]
  assert np.array_equal(y_cc[0], y.reshape(-1)[order])


# ---------------------------------------------------------------------------------------------------------------
# the library's layout, bindings and rejections
# ---------------------------------------------------------------------------------------------------------------
def test_every_scc_symbol_is_declared_exported_and_bound():
  with open(_lib.HEADER_PATH) as f:
    header = f.read()
  raw = C.CDLL(_lib.LIB_PATH)
  for name in SCC_SYMBOLS:
    assert f" {name}(" in header, name
    assert hasattr(raw, name), name
    assert name in _lib.SIGNATURES, name


@pytest.mark.parametrize("M", [6, 96, 384])
def test_one_group_layout_is_the_packed_layout_of_the_checkerboard_model(M):
  lay = F.scc_layout(M, (0, M))
  assert lay["total"] == F.ar_packed_floats(M)
  assert (lay["K1"], lay["N3"], lay["N4"]) == (4 * M, 10 * M // 3, 8 * M // 3)
  assert lay["bc"] == 24 * M * M and lay["w1"] == lay["bc"] + 2 * M
  lib = _lib.lib()
  assert lib.tfcb_scc_workspace_floats(M, 0, M, 3, 5, 7, 0) == lib.tfcb_cb_workspace_floats(M, 3, 5, 7, 0)
  assert lib.tfcb_scc_workspace_floats(M, 0, M, 3, 5, 7, 1) == lib.tfcb_cb_workspace_floats(M, 3, 5, 7, 1)


def test_group_layout_and_workspace():
  M = 320
  for k, (o, c) in enumerate(F.scc_spans((16, 16, 32, 64, 192))):
    lay = F.scc_layout(M, (o, c))
    k1, n3, n4 = sco.widths(M, k, c)
    assert (lay["K1"], lay["N3"], lay["N4"]) == (k1, n3, n4)
    assert lay["total"] == 24 * c * c + 2 * c + k1 * n3 + n3 + n3 * n4 + n4 + n4 * 2 * c + 2 * c
    assert _lib.lib().tfcb_scc_workspace_floats(M, o, c, 2, 5, 7, 1) == 2 * 18 * (n3 + n4)
    assert _lib.lib().tfcb_scc_workspace_floats(M, o, c, 2, 5, 7, 0) == 2 * 17 * (2 * c + n3 + n4)
  for args in ((7, 0, 7), (0, 0, 1), (6, 0, 0), (6, -1, 2), (6, 4, 3), (2048, 0, 2048)):
    assert _lib.lib().tfcb_scc_packed_floats(*args, None) == -1
    with pytest.raises(_lib.InvalidArgumentError, match="group of"):
      F.scc_layout(args[0], args[1:])


_FAKE = C.c_void_p(0x1000)  # never dereferenced: every call below fails its checks first


def _params(**kw):
  a = dict(M=24, o=6, C=6, B=2, H=3, W=4, anchors=0, ns=64, yhat=_FAKE, psi=_FAKE, ch=_FAKE, packed=_FAKE,
           work=_FAKE, nwork=1 << 20, whole=0, loc=None, scale=None, index=None, y=None, y_cb=None, yhat_out=None)
  a.update(kw)
  n = a.pop("n", F.scc_layout(24, (6, 6))["total"])
  return _lib.lib().tfcb_scc_params(a["packed"], n, a["M"], a["o"], a["C"], a["yhat"], a["psi"], a["ch"], a["B"],
                                    a["H"], a["W"], a["anchors"], a["ns"], a["work"], a["nwork"], a["whole"], a["loc"],
                                    a["scale"], a["index"], a["y"], a["y_cb"], a["yhat_out"], None)


@pytest.mark.parametrize("kw, match", [
    (dict(M=23), "positive even"), (dict(M=2048), "positive even"), (dict(o=20), "does not fit"),
    (dict(C=0), "does not fit"), (dict(o=-1), "does not fit"), (dict(n=7), "packed weights hold 7"),
    (dict(packed=None), "`packed` is null"), (dict(B=0), "batch size"), (dict(H=0), "latent shape"),
    (dict(W=-1), "latent shape"), (dict(ns=0), "num_scales"), (dict(psi=None), "null"), (dict(yhat=None), "null"),
    (dict(ch=None), "chctx"), (dict(work=None), "workspace"), (dict(nwork=100), "workspace of 100 floats"),
    (dict(y=_FAKE, loc=_FAKE), "the encoder needs")])
def test_params_rejections(kw, match):
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_params(**kw))
  assert _lib.launch_count() == n0


def test_scatter_and_pack_rejections():
  lib = _lib.lib()
  n0 = _lib.launch_count()
  for args, match in (((_FAKE, 1, 2, 2, 6, 4, 3, 1, _FAKE), "does not fit"),
                      ((_FAKE, 1, 2, 2, 5, 0, 5, 1, _FAKE), "positive even"),
                      ((_FAKE, 0, 2, 2, 6, 0, 3, 1, _FAKE), "batch size"),
                      ((_FAKE, 1, 0, 2, 6, 0, 3, 1, _FAKE), "latent shape"),
                      ((None, 1, 2, 2, 6, 0, 3, 1, _FAKE), "null")):
    with pytest.raises(_lib.InvalidArgumentError, match=match):
      _lib.check(lib.tfcb_scc_scatter(*args, None))
  n = F.scc_layout(6, (0, 3))["total"]
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    _lib.check(lib.tfcb_scc_pack_weights(6, 0, 3, *([_FAKE] * 9), n + 1, None))
  with pytest.raises(_lib.InvalidArgumentError, match="weight operand 2 is null"):
    _lib.check(lib.tfcb_scc_pack_weights(6, 0, 3, _FAKE, _FAKE, None, *([_FAKE] * 6), n, None))
  assert _lib.launch_count() == n0


def test_python_wrappers_reject_before_the_library():
  M, g = 12, (4, 8)
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=r"\[5, 5, 8, 16\]"):
    F.scc_pack_weights(M, g, torch.zeros(5, 5, M, 2 * M), *([None] * 7))
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.scc_pack_weights(M, g, torch.zeros(5, 5, 8, 16), *([None] * 7))
  packed = torch.zeros(F.scc_layout(M, g)["total"])
  psi = torch.zeros(1, 2, 2, 2 * M)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.scc_params(torch.zeros(5), g, None, psi, None, True, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.scc_params(packed, g, None, psi, None, True, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="groups must sum to M"):
    F.scc_encode([packed], (4, 8), torch.zeros(1, 2, 2, M), psi, None, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="groups must sum to M"):
    F.scc_encode([packed, packed], (4, 4), torch.zeros(1, 2, 2, M), psi, None, 64)
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------
def test_model_widths_and_argument_errors():
  m = models.SpaceChannelModel(num_filters=32, latent_depth=20, groups=(2, 2, 4, 12))
  assert m.spans == [(0, 2), (2, 2), (4, 4), (8, 12)]
  assert [tuple(cm.kernel.shape) for cm in m.context_models] == [(5, 5, c, 2 * c) for c in (2, 2, 4, 12)]
  assert all(isinstance(cm, models.CheckerboardConv2D) for cm in m.context_models)
  assert len(m.channel_context_transforms) == 3
  assert [list(t)[-1].filters for t in m.channel_context_transforms] == [4, 8, 24]
  for k, (ep, c) in enumerate(zip(m.entropy_parameters, (2, 2, 4, 12))):
    assert [l.filters for l in ep] == list(sco.widths(20, k, c)[1:]) + [2 * c]
  assert models.SpaceChannelModel().groups == (16, 16, 32, 64, 192)
  for kw, match in ((dict(latent_depth=21, groups=(21,)), "even"), (dict(latent_depth=20, groups=(2, 2)), "hold 4"),
                    (dict(latent_depth=4, groups=(4, 0)), "at least one"), (dict(latent_depth=4, groups=()), "at least"),
                    (dict(latent_depth=4, groups=(5, -1)), "at least one")):
    with pytest.raises(ValueError, match=match):
      models.SpaceChannelModel(num_filters=8, **kw)
  with pytest.raises(ValueError, match="multiple of 6"):
    models.MBT2018Model(latent_depth=320)
  with pytest.raises(ValueError, match="multiple of 6"):
    models.CheckerboardModel(latent_depth=320)
