"""CPU: the host side of MBT2018's column tiles (DESIGN §3.15).  The tile layout equals a NumPy restatement, the
library's ticket order puts every item after the items it waits for, a simulation of workers taking tickets in that
order always finishes with the critical path DESIGN quotes, the new C entries check their arguments before any device
work, and the model, the functional wrappers and rd_eval validate `tiles`.  The tile kernels build without spills."""
import ctypes as C
import heapq
import importlib.util
import inspect
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from compression_b200 import _lib
from compression_b200 import functional as F
from compression_b200 import models

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "compression_b200", "csrc")


def _host(a):
  return a.ctypes.data_as(C.c_void_p)


def _list(shapes):
  hs = np.ascontiguousarray([h for h, _ in shapes], dtype=np.int64)
  ws = np.ascontiguousarray([w for _, w in shapes], dtype=np.int64)
  return hs, ws


def _tiles_np(W, T):
  """[(t, c0, c1)] of the non-empty tiles of a row of W positions."""
  return [(t, t * W // T, (t + 1) * W // T) for t in range(T) if (t + 1) * W // T > t * W // T]


# ---------------------------------------------------------------------------------------------------------------
# the layout
# ---------------------------------------------------------------------------------------------------------------
SHAPE_LISTS = [[(1, 1)], [(1, 9)], [(9, 1)], [(2, 3)], [(32, 48)], [(5, 7), (1, 1), (2, 3), (13, 17)],
               [(3, 4), (9, 2), (1, 9), (6, 6)]]


def _t_values(ws):
  W = max(ws)
  return sorted({t for t in (1, 2, 3, W - 1, W, W + 5, 1024) if t >= 1})


@pytest.mark.parametrize("shapes", SHAPE_LISTS, ids=lambda s: "+".join(f"{h}x{w}" for h, w in s))
@pytest.mark.parametrize("M", [1, 12])
def test_tile_layout_is_the_numpy_split(shapes, M):
  hs, ws = _list(shapes)
  for T in _t_values(ws.tolist()):
    pos, wid = F.ar_tile_layout(hs, ws, T, M)
    assert pos.shape == (len(shapes), hs.max()) and (wid == M).all()
    lengths, phases = F.substream_layout(pos, wid, T)
    want_len = np.zeros(len(shapes) * T, np.int64)
    want_phase = np.zeros((hs.max(), len(shapes) * T), np.int64)
    for i, (H, W) in enumerate(shapes):
      for t in range(T):
        cols = (t + 1) * W // T - t * W // T  # tile t: columns [floor(t W / T), floor((t + 1) W / T))
        want_len[i * T + t] = H * cols * M
        want_phase[:H, i * T + t] = cols * M
    assert np.array_equal(lengths, want_len)
    assert np.array_equal(phases, want_phase)
    if T > max(ws):
      assert (lengths == 0).any()  # tiles with no columns are empty streams


def test_tile_layout_is_raster_order_per_tile():
  """The gather order of ar_tile_layout: tile t is its rows in order, its columns within each row."""
  H, W, T = 3, 7, 3
  pos, wid = F.ar_tile_layout([H], [W], T)
  from test_substreams_cpu import _split_np
  _, _, perm = _split_np(pos, wid, T)
  want = [r * W + c for t, c0, c1 in _tiles_np(W, T) for r in range(H) for c in range(c0, c1)]
  assert perm.tolist() == want


@pytest.mark.parametrize("bad", [0, 1025, 2.0, True, None, "2"])
def test_tile_layout_rejects_bad_tiles(bad):
  with pytest.raises(ValueError, match="tiles"):
    F.ar_tile_layout([2], [3], bad)


# ---------------------------------------------------------------------------------------------------------------
# the schedule
# ---------------------------------------------------------------------------------------------------------------
def _deps(item, W, T):
  """The two items (image, row, tile) that item (image, row, tile) waits for under DESIGN §3.15's rule."""
  i, r, t = item[:3]
  tiles = _tiles_np(W, T)
  rank = [x[0] for x in tiles].index(t)
  out = []
  if rank:
    out.append((i, r, tiles[rank - 1][0]))
  if r:
    col = min(W - 1, tiles[rank][2] + 1)  # column c_last + 2
    out.append((i, r - 1, next(tt for tt, c0, c1 in tiles if c0 <= col < c1)))
  return out


def _simulate(order, deps, cost, workers):
  """Finish time of `workers` workers taking tickets in order, each blocking until the item's dependencies are done.
  None when a worker waits for an item that no worker can take (a stall)."""
  finish = {}
  free = [0] * min(workers, len(order))
  heapq.heapify(free)
  for key in order:
    if any(d not in finish for d in deps[key]):
      return None  # (its dependency has a later ticket: with every worker blocked this way, nothing moves)
    start = max([heapq.heappop(free)] + [finish[d] for d in deps[key]])
    finish[key] = start + cost[key]
    heapq.heappush(free, finish[key])
  return max(finish.values())


SCHEDULE_CASES = [([(32, 48)], 8), ([(32, 48)], 16), ([(32, 48)], 24), ([(32, 48)], 48), ([(32, 48)], 64),
                  ([(1, 1)], 1), ([(1, 1)], 7), ([(9, 1)], 3), ([(1, 9)], 4), ([(2, 3)], 2),
                  ([(5, 7), (1, 1), (13, 17), (32, 48), (2, 3)], 5), ([(32, 48)] * 3 + [(48, 32)] * 2, 48)]


@pytest.mark.parametrize("shapes,T", SCHEDULE_CASES, ids=lambda v: str(v))
def test_schedule_orders_every_item_after_its_dependencies(shapes, T):
  hs, ws = _list(shapes)
  sched = F.ar_tiles_schedule(hs, ws, T)
  keys = [tuple(int(v) for v in row[:3]) for row in sched]
  want = {(i, r, t) for i, (H, W) in enumerate(shapes) for r in range(H) for t, _, _ in _tiles_np(W, T)}
  assert len(keys) == len(want) and set(keys) == want
  for row in sched:
    i, r, t, c0, c1 = (int(v) for v in row)
    assert (c0, c1) == (t * ws[i] // T, (t + 1) * ws[i] // T)
  at = {k: n for n, k in enumerate(keys)}
  deps = {k: _deps(k, int(ws[k[0]]), T) for k in keys}
  assert all(at[d] < at[k] for k in keys for d in deps[k])
  # the ticket key: (2 r + rank, r, image), non-decreasing
  ranks = {(i, t): n for i, W in enumerate(ws.tolist()) for n, (t, _, _) in enumerate(_tiles_np(W, T))}
  tk = [(2 * r + ranks[(i, t)], r, i) for i, r, t in keys]
  assert tk == sorted(tk)


@pytest.mark.parametrize("shapes,T", SCHEDULE_CASES, ids=lambda v: str(v))
def test_schedule_always_finishes_for_any_worker_count(shapes, T):
  hs, ws = _list(shapes)
  sched = F.ar_tiles_schedule(hs, ws, T)
  keys = [tuple(int(v) for v in row[:3]) for row in sched]
  deps = {k: _deps(k, int(ws[k[0]]), T) for k in keys}
  cost = {tuple(int(v) for v in row[:3]): int(row[4] - row[3]) for row in sched}
  total = sum(cost.values())
  times = [_simulate(keys, deps, cost, k) for k in (1, 2, 3, 132, 10000)]
  assert None not in times
  assert times[0] == total == int((hs * ws).sum())  # one worker: every position in turn
  assert times == sorted(times, reverse=True)


@pytest.mark.parametrize("T,positions", [(8, 420), (16, 234), (24, 172), (48, 141)])
def test_critical_path_is_the_design_formula(T, positions):
  """DESIGN §3.15: with enough workers a 32 x 48 image takes (2 (H - 1) + U) items of width w >= 2, or
  (3 (H - 1) + U) at w = 1."""
  H, W = 32, 48
  sched = F.ar_tiles_schedule([H], [W], T)
  keys = [tuple(int(v) for v in row[:3]) for row in sched]
  deps = {k: _deps(k, W, T) for k in keys}
  cost = {tuple(int(v) for v in row[:3]): int(row[4] - row[3]) for row in sched}
  w, U = W // T, min(T, W)
  formula = (2 * (H - 1) + U) * w if w >= 2 else 3 * (H - 1) + U
  assert formula == positions
  assert _simulate(keys, deps, cost, 10000) == positions
  assert _simulate(keys, deps, cost, 132) >= positions  # (blocked tickets hold workers: 132 may fall short of it)


def test_row_major_order_would_also_finish_but_serialises():
  """The (2 r + u) key is what runs the diagonal concurrently: row-major tickets also finish, on a longer path."""
  H, W, T = 32, 48, 16
  sched = F.ar_tiles_schedule([H], [W], T)
  keys = [tuple(int(v) for v in row[:3]) for row in sched]
  deps = {k: _deps(k, W, T) for k in keys}
  cost = {k: 3 for k in keys}
  assert _simulate(sorted(keys, key=lambda k: (k[1], k[2])), deps, cost, 4) > _simulate(keys, deps, cost, 4)


# ---------------------------------------------------------------------------------------------------------------
# the C entries' host checks
# ---------------------------------------------------------------------------------------------------------------
def test_workspace_sizes():
  lib = _lib.lib()
  hs, ws = _list([(32, 48), (2, 3)])
  for T in (1, 2, 48, 1024):
    n_items = sum(h * min(T, w) for h, w in zip(hs.tolist(), ws.tolist()))
    counters = sum(min(T, w) for w in ws.tolist())
    want = (2 * 16 + 32 * n_items + 4 * (counters + 3) + 3) // 4  # images, items, counters and three words
    assert lib.tfcb_ar_tiles_workspace_floats(2, _host(hs), _host(ws), T) == want
  for args in ((0, _host(hs), _host(ws), 2), (2, None, _host(ws), 2), (2, _host(hs), _host(ws), 0),
               (2, _host(hs), _host(ws), 1025)):
    assert lib.tfcb_ar_tiles_workspace_floats(*args) == -1
  zero = np.zeros(1, np.int64)
  assert lib.tfcb_ar_tiles_workspace_floats(1, _host(zero), _host(ws), 2) == -1


def test_new_entries_reject_bad_arguments_before_device_work():
  lib = _lib.lib()
  hs, ws = _list([(5, 7), (2, 3)])
  M, T = 12, 3
  packed_n = F.ar_packed_floats(M)
  nw = lib.tfcb_ar_tiles_workspace_floats(2, _host(hs), _host(ws), T)
  fake = C.c_void_p(256)  # never dereferenced: every check below fails before device work
  n0 = _lib.launch_count()
  good = dict(packed=fake, n=packed_n, M=M, y=fake, psi=fake, k=2, hs=_host(hs), ws=_host(ws), T=T, ns=64, work=fake,
              nw=nw, yhat=fake, loc=fake, index=fake, scale=None, stream=None)
  for over, msg in ((dict(T=0), "tiles=0"), (dict(T=1025), "tiles=1025"), (dict(M=10), "multiple of 6"),
                    (dict(n=packed_n + 1), "packed"), (dict(k=0), "list"), (dict(hs=None), "null"),
                    (dict(packed=None), "null"), (dict(y=None), "null"), (dict(index=None), "null"),
                    (dict(nw=nw - 1), f"workspace of {nw - 1} floats, this call needs {nw}"),
                    (dict(work=None), "workspace"), (dict(work=C.c_void_p(260)), "aligned"),
                    (dict(ns=0), "num_scales")):
    with pytest.raises(_lib.InvalidArgumentError, match=msg):
      _lib.check(lib.tfcb_ar_encode_tiles(*{**good, **over}.values()))
  dec = dict(h=None, packed=fake, n=packed_n, M=M, psi=fake, k=2, hs=_host(hs), ws=_host(ws), T=T, ns=64, coff=fake,
             work=fake, nw=nw, yhat=fake, stream=None)
  with pytest.raises(_lib.InvalidArgumentError, match="decoder"):
    _lib.check(lib.tfcb_ar_decode_tiles(*dec.values()))
  n = C.c_int64(-1)
  for args, msg in (((2, _host(hs), _host(ws), 0), "tiles=0"), ((2, _host(hs), _host(ws), 1025), "tiles=1025"),
                    ((0, _host(hs), _host(ws), 2), "list"), ((2, None, _host(ws), 2), "null")):
    with pytest.raises(_lib.InvalidArgumentError, match=msg):
      _lib.check(lib.tfcb_ar_tiles_schedule(*args, C.byref(n), None))
  with pytest.raises(_lib.InvalidArgumentError, match="null"):
    _lib.check(lib.tfcb_ar_tiles_schedule(2, _host(hs), _host(ws), 2, None, None))
  assert _lib.launch_count() == n0


def test_python_wrappers_check_before_the_library():
  import torch
  n0 = _lib.launch_count()
  handle = types.SimpleNamespace(n_streams=2)
  packed = torch.zeros(F.ar_packed_floats(12))
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA"):
    F.ar_decode_tiles(handle, packed, [torch.zeros(2, 3, 24)] * 2, 64, None, 3)
  for bad in (0, 1025, 2.5, True):
    with pytest.raises(ValueError, match="tiles"):
      F.ar_encode_tiles(packed, [torch.zeros(2, 3, 12)], [torch.zeros(2, 3, 24)], 64, bad)
    with pytest.raises(ValueError, match="tiles"):
      F.ar_decode_tiles(handle, packed, [torch.zeros(2, 3, 24)], 64, None, bad)
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# models and tools
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [0, -1, 1025, 2.0, "2", True, None])
def test_mbt2018_rejects_bad_tiles(bad):
  with pytest.raises(ValueError, match="tiles"):
    models.MBT2018Model(num_filters=8, latent_depth=12, tiles=bad)


def test_mbt2018_takes_tiles_as_a_keyword_only():
  for T in (1, 2, 48, 1024, np.int64(7)):
    assert models.MBT2018Model(num_filters=8, latent_depth=12, tiles=T).tiles == int(T)
  assert models.MBT2018Model(num_filters=8, latent_depth=12).tiles == 1
  with pytest.raises(TypeError):
    models.MBT2018Model(0.01, 8, 12, 64, .11, 256., 1, 2)
  with pytest.raises(ValueError, match="MBT2018Model"):  # substreams stay rejected, with or without tiles
    models.MBT2018Model(num_filters=8, latent_depth=12, substreams=2, tiles=2)


def test_checkerboard_and_space_channel_take_no_tiles():
  for cls, kw in ((models.CheckerboardModel, dict(num_filters=8, latent_depth=12)),
                  (models.SpaceChannelModel, dict(num_filters=8, latent_depth=12, groups=(2, 4, 6)))):
    assert "tiles" not in inspect.signature(cls.__init__).parameters
    with pytest.raises(TypeError):
      cls(tiles=2, **kw)
    assert cls(**kw).tiles == 1


def _rd_eval():
  spec = importlib.util.spec_from_file_location("rd_eval", os.path.join(ROOT, "tools", "rd_eval.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_rd_eval_takes_tiles_for_mbt2018():
  rd = _rd_eval()
  args = rd.parser().parse_args(["--synthetic", "kodak", "--model", "mbt2018", "--tiles", "16"])
  assert args.tiles == 16
  assert rd.parser().parse_args(["--synthetic", "kodak"]).tiles == 1
  params = list(inspect.signature(rd.make_model).parameters)
  assert params[:5] == ["name", "num_filters", "state_dict", "seed", "substreams"]
  with pytest.raises(SystemExit, match="mbt2018 only"):
    rd.make_model("checkerboard", 8, None, 0, 1, 2)


# ---------------------------------------------------------------------------------------------------------------
# compiled code
# ---------------------------------------------------------------------------------------------------------------
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


@pytest.mark.skipif(NVCC is None, reason="nvcc is not installed")
def test_tile_kernels_build_for_sm90a_without_spills(tmp_path):
  cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "-I" + os.path.join(ROOT, "include"), "-I" + CSRC, "-Xptxas", "-v", "-c",
         os.path.join(CSRC, "autoregressive.cu"), "-o", str(tmp_path / "ar.o")]
  err = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
  entries = re.findall(r"Compiling entry function '(\S+)'.*?\n(?:.*\n)*?\s*(\d+) bytes stack frame, (\d+) bytes spill "
                       r"stores, (\d+) bytes spill loads\n.*?Used (\d+) registers", err)
  tiles = [e for e in entries if "ar_tile_kernel" in e[0]]
  assert len(tiles) == 3, err  # the encoder, and the decoder with keys in shared and in global memory
  for name, stack, st, ld, regs in tiles:
    assert (st, ld) == ("0", "0") and int(regs) <= 128, (name, err)
