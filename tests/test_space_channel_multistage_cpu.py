"""CPU: the space-channel multistage context model without a device -- the float32 emulation of each group's stages
against float64 layer by layer, its one-group case against the multistage emulation and its stage 0 against the
space-channel model's anchor pass, its sensitivity to a wrong gather, a misplaced segment or a swapped group order,
the coding order and substream phases, the training form's context in float64, the model's arguments, and the
tfcb_mscc_* bindings and the checks they make before any device work."""
import ctypes as C
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
from oracle import checkerboard_oracle as cbo
from oracle import multistage_oracle as mso
from oracle import space_channel_multistage_oracle as scmo
from oracle import space_channel_oracle as sco

MSCC_SYMBOLS = ("tfcb_mscc_packed_floats", "tfcb_mscc_pack_weights", "tfcb_mscc_workspace_floats",
                "tfcb_mscc_params", "tfcb_mscc_scatter", "tfcb_mscc_ragged_workspace_floats",
                "tfcb_mscc_params_ragged", "tfcb_mscc_scatter_ragged")
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compression_b200", "csrc")


def _group_weights(M, k, c, rng):
  k1, n3, n4 = sco.widths(M, k, c)
  r = lambda *s: rng.standard_normal(s).astype(np.float32)
  return [[r(5, 5, c, 2 * c) / np.sqrt(12 * c) for _ in range(3)], [0.1 * r(2 * c) for _ in range(3)],
          r(k1, n3) / np.sqrt(k1), 0.1 * r(n3), r(n3, n4) / np.sqrt(n3), 0.1 * r(n4),
          8 * r(n4, 2 * c) / np.sqrt(n4), np.concatenate([0.5 * r(c), 24 + 4 * r(c)])]


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
# the float32 emulation against float64, the multistage emulation and the space-channel anchor pass
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [(6,), (1, 5), (2, 4, 6, 12)], ids=str)
def test_emulation_holds_to_the_rounding_bound_layer_by_layer(groups):
  M = sum(groups)
  ws = _weights(groups, M)
  for H, W in ((5, 7), (1, 9), (4, 1)):
    y_hat, psi = _inputs(2, H, W, M, H)
    for k, (g, w) in enumerate(zip(scmo.spans(groups), ws)):
      ch = _ch(2, H, W, g[1], k) if k else None
      for stage in range(4):
        loc, scale, _ = scmo.params32(w, g, y_hat, psi, ch, stage, 64)
        assert loc.shape == (2, F.msc_counts(H, W)[stage], g[1])
        if loc.size == 0:
          continue
        errs = scmo.layer_errors(w, g, y_hat, psi, ch, stage)
        assert len(errs) == (3 if stage == 0 else 4)
        for err, bound, mag in errs:
          assert np.all(err <= bound)
          assert np.all(bound <= 1e-4 * (1 + mag.max()))
        (l64, s64) = scmo.params64(w, g, y_hat, psi, ch, stage)
        (lb, sb) = scmo.bound64(w, g, y_hat, psi, ch, stage)
        assert np.all(np.abs(loc - l64) <= lb) and np.all(np.abs(scale - s64) <= sb)


@pytest.mark.parametrize("M", [6, 12, 30])
def test_one_group_is_the_multistage_emulation_bit_for_bit(M):
  ws = _weights((M,), M)[0]
  assert sco.widths(M, 0, M) == (4 * M, 10 * M // 3, 8 * M // 3)
  for H, W in ((1, 1), (1, 6), (5, 7), (6, 8)):
    y_hat, psi = _inputs(2, H, W, M, W)
    for stage in range(4):
      got = scmo.params32(ws, (0, M), y_hat, psi, None, stage, 64)
      want = mso.params32(ws, y_hat, psi, stage, 64)
      for g, w in zip(got, want):
        assert np.array_equal(_bits(g), _bits(w)), (H, W, stage)
  y = _inputs(2, 5, 7, M, 3)[0] + 0.3
  psi = _inputs(2, 5, 7, M, 4)[1]
  got = scmo.encode32([ws], (M,), y, psi, None, 64)
  want = mso.encode32(ws, y, psi, 64)
  for g, w in zip(got, want):
    assert np.array_equal(_bits(g).reshape(-1), _bits(w).reshape(-1))


@pytest.mark.parametrize("groups", [(6,), (1, 5), (2, 4, 6, 12)], ids=str)
def test_stage_zero_is_the_space_channel_anchor_pass_at_its_positions(groups):
  M = sum(groups)
  ws = _weights(groups, 7)
  H, W = 5, 7
  y_hat, psi = _inputs(2, H, W, M, 5)
  anchors = cbo.positions(H, W, True)
  at = [anchors.index(p) for p in mso.positions(H, W, 0)]
  for k, (g, w) in enumerate(zip(scmo.spans(groups), ws)):
    ch = _ch(2, H, W, g[1], k) if k else None
    # the space-channel group's network: the same 1x1 layers, any context kernel (the anchors read none)
    sc_ws = [w[0][1]] + [w[1][1]] + w[2:]
    got = scmo.params32(w, g, y_hat, psi, ch, 0, 64)
    want = sco.params32(sc_ws, g, y_hat, psi, ch, True, 64)
    for a, b in zip(got, want):
      assert np.array_equal(_bits(a), _bits(b[:, at])), (g,)


def test_a_wrong_layout_changes_the_bits():
  groups = (2, 2, 2)
  M, H, W = 6, 5, 7
  ws = _weights(groups, 1)
  y_hat, psi = _inputs(1, H, W, M, 1)
  y_hat += 0.25 * np.arange(H * W * M, dtype=np.float32).reshape(1, H, W, M)  # every latent distinct
  g, ch = (2, 2), _ch(1, H, W, 2, 1)
  for stage in (1, 2, 3):
    want = scmo.params32(ws[1], g, y_hat, psi, ch, stage, 64)[0]
    wrong = {
        "another group's channels": scmo.params32(ws[1], (4, 2), y_hat, psi, ch, stage, 64)[0],
        "taps in reverse order": scmo.params32(ws[1], g, y_hat, psi, ch, stage, 64,
                                               gather_fn=lambda y, pos, taps: mso.gather(y, pos, taps[::-1]))[0],
        "ctx before the channel context": scmo.params32(ws[1], g, y_hat, psi, ch, stage, 64,
                                                        segments=("psi", "ctx", "ch"))[0],
        "psi last": scmo.params32(ws[1], g, y_hat, psi, ch, stage, 64, segments=("ch", "ctx", "psi"))[0],
    }
    for name, got in wrong.items():
      assert not np.array_equal(_bits(got), _bits(want)), (stage, name)
  # at stage 0 the spatial context is zero: a misplaced zero segment changes the bits too
  a = scmo.params32(ws[1], g, y_hat, psi, ch, 0, 64)[0]
  assert not np.array_equal(_bits(a), _bits(scmo.params32(ws[1], g, y_hat, psi, ch, 0, 64,
                                                          segments=("psi", "ctx", "ch"))[0]))
  # stage 0 reads no latent; a later stage reads only its group's channels of earlier stages
  assert np.array_equal(_bits(a), _bits(scmo.params32(ws[1], g, 0 * y_hat, psi, ch, 0, 64)[0]))
  other = y_hat.copy()
  other[..., [0, 1, 4, 5]] += 3
  for stage in (1, 2, 3):
    assert np.array_equal(_bits(scmo.params32(ws[1], g, other, psi, ch, stage, 64)[0]),
                          _bits(scmo.params32(ws[1], g, y_hat, psi, ch, stage, 64)[0]))
  # swapping the order of two groups of equal size changes the encoder's bits
  y = y_hat + 0.3
  chf = lambda k, yh: yh[..., [j % (2 * k) for j in range(4)]] * np.float32(0.5)
  base = scmo.encode32(ws, groups, y, psi, chf, 64)
  swapped = scmo.encode32([ws[0], ws[2], ws[1]], groups, y, psi, chf, 64)
  assert not np.array_equal(_bits(base[2]), _bits(swapped[2]))


# ---------------------------------------------------------------------------------------------------------------
# coding order, substream phases and the training form
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1), (1, 6), (5, 1), (3, 5), (4, 6)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_coding_order_and_substream_phases(shape):
  H, W = shape
  groups = (1, 2, 3)
  M = sum(groups)
  order = scmo.coding_order(H, W, groups)
  assert sorted(order.tolist()) == list(range(H * W * M))  # a permutation
  n = F.msc_counts(H, W)
  at = 0
  for o, c in F.scc_spans(groups):
    for stage in range(4):
      block = order[at:at + n[stage] * c].reshape(n[stage], c)
      assert np.array_equal(block // M, np.repeat(np.array(mso.positions(H, W, stage), np.int64)[:, None], c, 1))
      assert np.array_equal(block % M, np.tile(np.arange(o, o + c), (n[stage], 1)))
      at += n[stage] * c
  ws = _weights(groups, 3)
  y = np.arange(H * W * M, dtype=np.float32).reshape(1, H, W, M)
  y_cc = scmo.encode32(ws, groups, y, _inputs(1, H, W, M, 3)[1],
                       lambda k, yh: np.zeros((1, H, W, 2 * groups[k]), np.float32), 64)[1]
  assert np.array_equal(y_cc[0], y.reshape(-1)[order])
  pos, wid = F.context_phases(groups, [H, 2 * H + 1], [W, W + 2], multistage=True)
  assert pos.shape == (2, 12) and wid.shape == (2, 12)
  assert pos[0].tolist() == list(n) * 3 and pos[1].tolist() == list(F.msc_counts(2 * H + 1, W + 2)) * 3
  assert wid[0].tolist() == [c for c in groups for _ in range(4)]
  assert int((pos[0] * wid[0]).sum()) == H * W * M
  # the one-group phases are the multistage model's, and the checkerboard phases are unchanged
  mp, mw = F.msc_phases([H], [W], M)
  assert np.array_equal(mp, F.context_phases((M,), [H], [W], multistage=True)[0]) and (mw == M).all()
  cp = F.context_phases(groups, [H], [W])[0]
  assert cp[0].tolist() == [(H * W + 1) // 2, H * W // 2] * 3


def test_training_context_is_the_oracles_group_context_in_float64():
  torch.manual_seed(0)
  groups, H, W = (2, 4), 7, 6
  M = sum(groups)
  m = models.SpaceChannelMultistageModel(num_filters=8, latent_depth=M, groups=groups).double()
  with torch.no_grad():
    for cms in m.context_models:
      for cv in cms:
        cv.bias.normal_()
    y = torch.randn(2, H, W, M, dtype=torch.float64)
    for k, (o, c) in enumerate(m.spans):
      got = m._spatial_context(k, y[..., o:o + c]).numpy()
      cms = m.context_models[k]
      want = scmo.context64([cv.kernel.numpy() for cv in cms], [cv.bias.numpy() for cv in cms], y.numpy(), (o, c))
      assert got.shape == (2, H, W, 2 * c)
      assert np.abs(got - want).max() <= 1e-12 * (1 + np.abs(want).max())
      assert (got[:, models.multistage_stage_map(H, W).numpy() == 0] == 0).all()


# ---------------------------------------------------------------------------------------------------------------
# the library's layout, bindings and rejections
# ---------------------------------------------------------------------------------------------------------------
def test_every_mscc_symbol_is_declared_exported_and_bound():
  with open(_lib.HEADER_PATH) as f:
    header = f.read()
  raw = C.CDLL(_lib.LIB_PATH)
  for name in MSCC_SYMBOLS:
    assert f" {name}(" in header, name
    assert hasattr(raw, name), name
    assert name in _lib.SIGNATURES, name


@pytest.mark.parametrize("M", [6, 96, 384])
def test_one_group_layout_is_the_multistage_layout(M):
  lay = F.mscc_layout(M, (0, M))
  assert lay["total"] == F.msc_packed_floats(M)
  assert (lay["K1"], lay["N3"], lay["N4"]) == (4 * M, 10 * M // 3, 8 * M // 3)
  assert lay["bc1"] == 8 * M * M and lay["wc2"] == lay["bc1"] + 2 * M and lay["w1"] == 64 * M * M + 6 * M
  lib = _lib.lib()
  for s in range(4):
    assert lib.tfcb_mscc_workspace_floats(M, 0, M, 3, 5, 7, s) == lib.tfcb_msc_workspace_floats(M, 3, 5, 7, s)


def test_group_layout_and_workspace():
  M = 320
  hs, ws = np.array([1, 3], np.int64), np.array([4, 1], np.int64)
  h, w = hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p)
  lib = _lib.lib()
  for k, (o, c) in enumerate(F.scc_spans((16, 16, 32, 64, 192))):
    lay = F.mscc_layout(M, (o, c))
    k1, n3, n4 = sco.widths(M, k, c)
    assert (lay["K1"], lay["N3"], lay["N4"]) == (k1, n3, n4)
    assert lay["total"] == 64 * c * c + 6 * c + k1 * n3 + n3 + n3 * n4 + n4 + n4 * 2 * c + 2 * c
    assert [lay[key] for key in ("wc1", "bc1", "wc2", "bc2", "wc3", "bc3", "w1")] == [
        0, 8 * c * c, 8 * c * c + 2 * c, 32 * c * c + 2 * c, 32 * c * c + 4 * c, 64 * c * c + 4 * c, 64 * c * c + 6 * c]
    for s, n in enumerate(F.msc_counts(5, 7)):
      assert lib.tfcb_mscc_workspace_floats(M, o, c, 2, 5, 7, s) == 2 * n * ((2 * c if s else 0) + n3 + n4)
      n = F.msc_counts(1, 4)[s] + F.msc_counts(3, 1)[s]
      assert lib.tfcb_mscc_ragged_workspace_floats(M, o, c, 2, h, w, s) == 2 * 8 + n * ((2 * c if s else 0) + n3 + n4)
  for args in ((7, 0, 7), (0, 0, 1), (6, 0, 0), (6, -1, 2), (6, 4, 3), (2048, 0, 2048)):
    assert lib.tfcb_mscc_packed_floats(*args, None) == -1
    with pytest.raises(_lib.InvalidArgumentError, match="group of"):
      F.mscc_layout(args[0], args[1:])
  for args in ((12, 0, 4, 1, 2, 2, 4), (12, 0, 4, 1, 2, 2, -1), (11, 0, 4, 1, 2, 2, 0), (12, 10, 4, 1, 2, 2, 0),
               (12, 0, 4, 0, 2, 2, 0), (12, 0, 4, 1, 0, 2, 1)):
    assert lib.tfcb_mscc_workspace_floats(*args) == -1
  assert lib.tfcb_mscc_ragged_workspace_floats(M, 0, 16, 2, h, w, 4) == -1


_FAKE = C.c_void_p(0x1000)  # never dereferenced: every call below fails its checks first


def _params(**kw):
  a = dict(M=24, o=6, C=6, B=2, H=3, W=4, stage=1, ns=64, yhat=_FAKE, psi=_FAKE, ch=_FAKE, packed=_FAKE,
           work=_FAKE, nwork=1 << 20, whole=0, loc=None, scale=None, index=None, y=None, y_cc=None, yhat_out=None)
  a.update(kw)
  n = a.pop("n", F.mscc_layout(24, (6, 6))["total"])
  return _lib.lib().tfcb_mscc_params(a["packed"], n, a["M"], a["o"], a["C"], a["yhat"], a["psi"], a["ch"], a["B"],
                                     a["H"], a["W"], a["stage"], a["ns"], a["work"], a["nwork"], a["whole"], a["loc"],
                                     a["scale"], a["index"], a["y"], a["y_cc"], a["yhat_out"], None)


@pytest.mark.parametrize("kw, match", [
    (dict(M=23), "positive even"), (dict(M=2048), "positive even"), (dict(o=20), "does not fit"),
    (dict(C=0), "does not fit"), (dict(o=-1), "does not fit"), (dict(stage=4), "stage 4"),
    (dict(stage=-1), "stage -1"), (dict(n=7), "packed weights hold 7"), (dict(packed=None), "`packed` is null"),
    (dict(B=0), "batch size"), (dict(H=0), "latent shape"), (dict(W=-1), "latent shape"), (dict(ns=0), "num_scales"),
    (dict(psi=None), "null"), (dict(yhat=None), "null"), (dict(ch=None), "chctx"), (dict(work=None), "workspace"),
    (dict(nwork=100), "workspace of 100 floats"), (dict(y=_FAKE, loc=_FAKE), "the encoder needs")])
def test_params_rejections(kw, match):
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _lib.check(_params(**kw))
  assert _lib.launch_count() == n0


def test_ragged_scatter_and_pack_rejections():
  lib = _lib.lib()
  n = F.mscc_layout(12, (4, 8))["total"]
  hs, ws = np.array([2, 0], np.int64), np.array([3, 3], np.int64)
  h, w = hs.ctypes.data_as(C.c_void_p), ws.ctypes.data_as(C.c_void_p)
  ragged = lambda nimg, stage, nwork, M=12, o=4, c=8, ch=_FAKE: lib.tfcb_mscc_params_ragged(
      _FAKE, n, M, o, c, _FAKE, _FAKE, ch, nimg, h, w, stage, 64, _FAKE, nwork, 0, None, None, None, None, None, None,
      None)
  n0 = _lib.launch_count()
  cases = [
      (lambda: ragged(2, 0, 1 << 20), "image 1: latent shape 0 x 3"),
      (lambda: ragged(0, 0, 1 << 20), "a list of 0 images"),
      (lambda: ragged(1, 5, 1 << 20), "stage 5"),
      (lambda: ragged(1, 1, 10), "workspace of 10 floats"),
      (lambda: ragged(1, 1, 1 << 20, ch=None), "chctx"),
      (lambda: ragged(1, 1, 1 << 20, o=8), "does not fit"),
      (lambda: lib.tfcb_mscc_scatter_ragged(_FAKE, 1, h, w, 12, 4, 8, 0, None, 0, _FAKE, None), "workspace"),
      (lambda: lib.tfcb_mscc_scatter_ragged(_FAKE, 2, h, w, 12, 4, 8, 0, _FAKE, 1 << 20, _FAKE, None), "latent shape"),
      (lambda: lib.tfcb_mscc_scatter_ragged(_FAKE, 1, h, w, 12, 4, 8, 4, _FAKE, 1 << 20, _FAKE, None), "stage 4"),
      (lambda: lib.tfcb_mscc_scatter(_FAKE, 1, 2, 2, 6, 4, 3, 1, _FAKE, None), "does not fit"),
      (lambda: lib.tfcb_mscc_scatter(_FAKE, 1, 2, 2, 5, 0, 5, 1, _FAKE, None), "positive even"),
      (lambda: lib.tfcb_mscc_scatter(_FAKE, 1, 2, 2, 6, 0, 3, 4, _FAKE, None), "stage 4"),
      (lambda: lib.tfcb_mscc_scatter(_FAKE, 0, 2, 2, 6, 0, 3, 1, _FAKE, None), "batch size"),
      (lambda: lib.tfcb_mscc_scatter(_FAKE, 1, 0, 2, 6, 0, 3, 1, _FAKE, None), "latent shape"),
      (lambda: lib.tfcb_mscc_scatter(None, 1, 2, 2, 6, 0, 3, 1, _FAKE, None), "null"),
      (lambda: lib.tfcb_mscc_pack_weights(12, 4, 8, *([_FAKE] * 12), _FAKE, n + 1, None), "packed weights hold"),
      (lambda: lib.tfcb_mscc_pack_weights(12, 4, 8, *([_FAKE] * 12), None, n, None), "`packed` is null"),
      (lambda: lib.tfcb_mscc_pack_weights(12, 4, 8, *([_FAKE] * 11), None, _FAKE, n, None), "operand 11 is null"),
      (lambda: lib.tfcb_mscc_pack_weights(12, 8, 8, *([_FAKE] * 12), _FAKE, n, None), "does not fit"),
  ]
  for call, match in cases:
    with pytest.raises(_lib.InvalidArgumentError, match=match):
      _lib.check(call())
  assert _lib.launch_count() == n0


def test_python_wrappers_reject_before_the_library():
  M, g = 12, (4, 8)
  n0 = _lib.launch_count()
  k = torch.zeros(5, 5, 8, 16)
  with pytest.raises(_lib.InvalidArgumentError, match="each of stages"):
    F.mscc_pack_weights(M, g, [k, k], [None] * 2, *([None] * 6))
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.mscc_pack_weights(M, g, [k] * 3, [None] * 3, *([None] * 6))
  packed = torch.zeros(F.mscc_layout(M, g)["total"])
  psi = torch.zeros(1, 2, 2, 2 * M)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.mscc_params(torch.zeros(5), g, None, psi, None, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="mscc_pack_weights"):
    F.mscc_params(torch.zeros(5, dtype=torch.int32), g, None, psi, None, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.mscc_params(packed, g, None, psi, None, 0, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="stage 4"):
    F.mscc_params(packed, g, None, psi, None, 4, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="groups must sum to M"):
    F.mscc_encode([packed], (4, 8), torch.zeros(1, 2, 2, M), psi, None, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="groups must sum to M"):
    F.mscc_encode([packed, packed], (4, 4), torch.zeros(1, 2, 2, M), psi, None, 64)
  with pytest.raises(_lib.InvalidArgumentError, match="substreams"):
    F.mscc_encode([packed], (M,), torch.zeros(1, 2, 2, M), psi, None, 64, substreams=0)
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------
def test_model_widths_and_argument_errors():
  m = models.SpaceChannelMultistageModel(num_filters=32, latent_depth=20, groups=(2, 2, 4, 12))
  assert m.spans == [(0, 2), (2, 2), (4, 4), (8, 12)]
  for cms, c in zip(m.context_models, (2, 2, 4, 12)):
    assert isinstance(cms, torch.nn.ModuleList) and [cm.stage for cm in cms] == [1, 2, 3]
    assert all(isinstance(cm, models.MultistageConv2D) for cm in cms)
    assert all(tuple(cm.kernel.shape) == (5, 5, c, 2 * c) for cm in cms)
  assert len(m.channel_context_transforms) == 3
  for k, (ep, c) in enumerate(zip(m.entropy_parameters, (2, 2, 4, 12))):
    assert [l.filters for l in ep] == list(sco.widths(20, k, c)[1:]) + [2 * c]
  d = models.SpaceChannelMultistageModel(substreams=3)
  assert d.groups == (16, 16, 32, 64, 192) and d.latent_depth == 320 and d.substreams == 3
  for kw, match in ((dict(latent_depth=21, groups=(21,)), "even"), (dict(latent_depth=20, groups=(2, 2)), "hold 4"),
                    (dict(latent_depth=4, groups=(4, 0)), "at least one"), (dict(latent_depth=4, groups=()), "at least")):
    with pytest.raises(ValueError, match=match):
      models.SpaceChannelMultistageModel(num_filters=8, **kw)


# ---------------------------------------------------------------------------------------------------------------
# compiled code
# ---------------------------------------------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


@pytest.mark.skipif(NVCC is None, reason="nvcc is not installed")
def test_group_kernels_build_for_sm90a_without_spills(tmp_path):
  cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(CSRC, "..", "..", "include"), "-I" + CSRC, "-Xptxas", "-v", "-c",
         os.path.join(CSRC, "multistage.cu"), "-o", str(tmp_path / "ms.o")]
  r = subprocess.run(cmd, capture_output=True, text=True, check=True)
  spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
  assert len(spills) == 5  # the multistage and space-channel multistage passes share four dense kernels and a scatter
  assert all(s == ("0", "0") for s in spills), r.stderr
