"""CPU: the host side of substreams (DESIGN §3.14).  The library's layout equals a NumPy restatement of the split, the
string header round-trips and rejects malformed strings by number before any launch, bad `substreams` values are
refused, and the new C entries check their arguments before any device work."""
import ctypes as C

import numpy as np
import pytest

from compression_b200 import _lib
from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models


def _host(a):
  return a.ctypes.data_as(C.c_void_p)


def _split_np(pos, wid, S):
  """§3.14 restated: (stream lengths [U S], phase lengths [P, U S], the coding-order index of every symbol in
  substream order)."""
  pos, wid = np.asarray(pos, np.int64), np.broadcast_to(np.asarray(wid, np.int64), np.shape(pos))
  U, P = pos.shape
  streams, phases, perm, base = [], np.zeros((P, U * S), np.int64), [], 0
  for u in range(U):
    starts = base + np.concatenate([[0], np.cumsum(pos[u] * wid[u])[:-1]])
    for s in range(S):
      n_s = 0
      for p in range(P):
        lo, hi = s * pos[u, p] // S, (s + 1) * pos[u, p] // S
        phases[p, u * S + s] = (hi - lo) * wid[u, p]
        perm.extend(range(starts[p] + lo * wid[u, p], starts[p] + hi * wid[u, p]))
        n_s += (hi - lo) * wid[u, p]
      streams.append(n_s)
    base += int((pos[u] * wid[u]).sum())
  return np.asarray(streams, np.int64), phases, np.asarray(perm, np.int64)


def _context(groups, shapes):
  hs = [h for h, _ in shapes]
  ws = [w for _, w in shapes]
  return F.context_phases(groups, hs, ws)


CASES = [
    ("one phase", [[10]], [[7]]),
    ("one phase, units", [[3], [64], [1000]], [[4]]),
    ("two phases", *_context((12,), [(5, 7), (1, 1), (2, 3), (32, 48)])),
    ("scc (2, 4, 6, 12)", *_context((2, 4, 6, 12), [(3, 5), (1, 1), (17, 9)])),
    ("scc default", *_context((16, 16, 32, 64, 192), [(32, 48), (2, 3)])),
]


@pytest.mark.parametrize("name,pos,wid", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("S", [1, 2, 7, 32, 64, 1024])
def test_layout_is_the_numpy_split(name, pos, wid, S):
  lengths, phases = F.substream_layout(pos, wid, S)
  want_lengths, want_phases, perm = _split_np(pos, wid, S)
  assert np.array_equal(lengths, want_lengths)
  assert np.array_equal(phases, want_phases)
  assert np.array_equal(phases.sum(axis=0), lengths)
  assert np.array_equal(np.sort(perm), np.arange(perm.size))  # a permutation of every symbol
  n = np.asarray(pos)
  if S == 1:
    assert np.array_equal(lengths, (n * np.broadcast_to(np.asarray(wid), n.shape)).sum(axis=1))


def test_layout_covers_short_equal_and_long_phases():
  for n in (3, 8, 8000):  # n_p < S, n_p = S, n_p >> S
    lengths, phases = F.substream_layout([[n, n // 2]], [[5, 3]], 8)
    want_lengths, want_phases, _ = _split_np([[n, n // 2]], [[5, 3]], 8)
    assert np.array_equal(lengths, want_lengths) and np.array_equal(phases, want_phases)
    if n < 8:
      assert (lengths == 0).any()  # empty substreams
    assert lengths.max() - lengths.min() <= 5 + 3


def test_context_phases_are_anchors_then_non_anchors_per_group():
  pos, wid = F.context_phases((2, 4), [3, 1], [5, 1])
  assert pos.tolist() == [[8, 7, 8, 7], [1, 0, 1, 0]]
  assert wid.tolist() == [[2, 2, 4, 4], [2, 2, 4, 4]]


# ---------------------------------------------------------------------------------------------------------------
# the string header
# ---------------------------------------------------------------------------------------------------------------
def test_header_round_trips_and_s1_adds_nothing():
  rng = np.random.default_rng(0)
  assert gen_ops.substream_header([123]) == b""
  for S in (2, 3, 127, 128, 1024):
    lens = rng.integers(0, 70000, S)
    lens[0] = 0
    parts = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in lens]
    s = gen_ops.substream_header(lens) + b"".join(parts)
    assert gen_ops.parse_substreams(s, S, 5) == parts
  assert gen_ops.substream_header([127, 128, 1]) == bytes([3, 127, 0x80, 1])
  assert gen_ops.substream_header([0] * 128 + [9]) == bytes([0x81, 1]) + bytes(128)


@pytest.mark.parametrize("string,match", [
    (b"", "truncated"),
    (bytes([0x82]), "truncated"),
    (bytes([2, 0x85]), "truncated"),
    (bytes([0x82, 0]), "minimal"),
    (bytes([2, 0x81, 0x00]) + bytes(3), "minimal"),
    (bytes([3, 1]) + bytes(4), "written with 3 substreams, decoding expects 2"),
    (bytes([1]) + bytes(4), "written with 1 substreams"),
    (bytes([2, 9, 1, 2, 3]), "past the end"),
])
def test_malformed_headers_raise_naming_the_string_before_any_launch(string, match):
  good = gen_ops.substream_header([1, 1]) + b"ab"
  n0 = _lib.launch_count()
  with pytest.raises(ValueError, match=match) as e:
    for i, s in enumerate([good, good, string]):
      gen_ops.parse_substreams(s, 2, i)
  assert "string 2" in str(e.value)
  assert _lib.launch_count() == n0


@pytest.mark.parametrize("bad", [0, -1, 1025, 2.0, "2", True, None])
def test_bad_substream_counts_are_rejected(bad):
  with pytest.raises(ValueError):
    gen_ops.check_substreams(bad)
  with pytest.raises(ValueError):
    models.BLS2017Model(num_filters=8, substreams=bad)
  with pytest.raises(ValueError):
    E.ContinuousBatchedEntropyModel._substreams(bad)


def test_good_substream_counts_are_accepted():
  for S in (1, 2, 1024, np.int64(7)):
    assert gen_ops.check_substreams(S) == int(S)


def test_fused_false_and_mbt2018_reject_substreams():
  with pytest.raises(ValueError, match="fused=False"):
    E.ContinuousBatchedEntropyModel._substreams(2, fused=False)
  assert E.ContinuousBatchedEntropyModel._substreams(1, fused=False) == 1
  with pytest.raises(ValueError, match="MBT2018Model"):
    models.MBT2018Model(num_filters=8, latent_depth=12, substreams=2)
  assert models.MBT2018Model(num_filters=8, latent_depth=12).substreams == 1
  for cls, kw in ((models.BMSHJ2018Model, dict(num_filters=8)), (models.MS2020Model, dict(num_filters=8)),
                  (models.CheckerboardModel, dict(num_filters=8, latent_depth=12)),
                  (models.SpaceChannelModel, dict(num_filters=8, latent_depth=12, groups=(2, 4, 6)))):
    assert cls(substreams=64, **kw).substreams == 64


def test_universal_models_take_no_substreams():
  prior = D.NoisyDeepFactorized(batch_shape=(4,))
  em = E.UniversalBatchedEntropyModel(prior, coding_rank=2, compression=False)
  for call in (lambda: em.compress(np.zeros((2, 4), np.float32), substreams=2),
               lambda: em.decompress([b""], (2,), substreams=2),
               lambda: em.compress_ragged([np.zeros((2, 4), np.float32)], substreams=2)):
    with pytest.raises(TypeError):
      call()


# ---------------------------------------------------------------------------------------------------------------
# the C entries' host checks
# ---------------------------------------------------------------------------------------------------------------
def test_new_entries_reject_bad_arguments_before_device_work():
  lib = _lib.lib()
  pos = np.ascontiguousarray([[4, 3]], dtype=np.int64)
  wid = np.ascontiguousarray([[2, 2]], dtype=np.int64)
  offs = np.zeros(3, np.int64)
  n0 = _lib.launch_count()
  bad_layouts = [
      ((0, 2, _host(pos), _host(wid), 2), "coding units"),
      ((1, 0, _host(pos), _host(wid), 2), "phases"),
      ((1, 2, _host(pos), _host(wid), 0), "substreams=0"),
      ((1, 2, _host(pos), _host(wid), 1025), "substreams=1025"),
      ((1, 2, None, _host(wid), 2), "null"),
      ((1, 2, _host(pos), _host(np.zeros((1, 2), np.int64)), 2), "width 0"),
      ((1, 2, _host(np.full((1, 2), -1, np.int64)), _host(wid), 2), "-1 positions"),
  ]
  for args, match in bad_layouts:
    with pytest.raises(_lib.InvalidArgumentError, match=match):
      _lib.check(lib.tfcb_substream_layout(*args, _host(offs), None))
  assert lib.tfcb_substream_gather_workspace_bytes(1, 2, 2) == 4 * 16
  for args in ((0, 2, 2), (1, 0, 2), (1, 2, 0), (1, 2, 1025), (1 << 30, 2, 1024)):
    assert lib.tfcb_substream_gather_workspace_bytes(*args) == -1
  fake = C.c_void_p(256)  # never dereferenced: every check below fails before device work
  with pytest.raises(_lib.InvalidArgumentError, match="no operand"):
    _lib.check(lib.tfcb_substream_gather(1, 2, _host(pos), _host(wid), 2, None, None, None, None, None, None, fake,
                                         64, None))
  with pytest.raises(_lib.InvalidArgumentError, match="needs its output"):
    _lib.check(lib.tfcb_substream_gather(1, 2, _host(pos), _host(wid), 2, fake, None, None, None, None, None, fake,
                                         64, None))
  with pytest.raises(_lib.InvalidArgumentError, match="workspace of 32 bytes, this call needs 64"):
    _lib.check(lib.tfcb_substream_gather(1, 2, _host(pos), _host(wid), 2, fake, None, None, fake, None, None, fake,
                                         32, None))
  with pytest.raises(_lib.InvalidArgumentError, match="aligned"):
    _lib.check(lib.tfcb_substream_gather(1, 2, _host(pos), _host(wid), 2, fake, None, None, fake, None, None,
                                         C.c_void_p(260), 64, None))
  with pytest.raises(_lib.InvalidArgumentError, match="substreams=0"):
    _lib.check(lib.tfcb_substream_gather(1, 2, _host(pos), _host(wid), 0, fake, None, None, fake, None, None, fake,
                                         64, None))
  assert _lib.launch_count() == n0
