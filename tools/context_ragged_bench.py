"""Times the context models' list calls (one ragged launch sequence per list) against the per-shape path, in one run
with the two paths alternated call by call.

  python tools/context_ragged_bench.py [--reps 3] [--models mbt2018,checkerboard,space_channel] [--out FILE.json]

For each model (torch.manual_seed(0) weights, num_filters 192 and the model's default latent depth) and each of two
lists: (a) the 24 Kodak-shaped images of the other benches (two latent shapes), and (b) 24 seeded images whose latent
shapes all differ (sides multiples of 16 from 256 to 1024, tools/rd_eval.py --synthetic mixed with seed 1), it times
`compress_images` / `decompress_images` against the per-shape path: the transforms per image and one batch encode
or decode (the coding of `compress_batch` / `decompress_batch`) per group of images of one latent shape, as the models
coded lists before.  Medians of --reps host-timed calls ending in a synchronise, after one warm-up call of each; the library launches of one call; the card's name, power limit and SM
clock read before and after.  Both paths must give the same strings and the same decoded latents, bit for bit; the
images they decode from them may differ by one level (the synthesis transform is not bitwise repeatable).  Prints
one JSON object."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from compression_b200 import _lib, gen_ops, models  # noqa: E402
import rd_eval  # noqa: E402

MODELS = {"mbt2018": models.MBT2018Model, "checkerboard": models.CheckerboardModel,
          "space_channel": models.SpaceChannelModel}


def _once(fn):
  """(ms, library launches, result) of one call ending in a synchronisation."""
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) * 1e3, _lib.launch_count() - n0, out


def _shape_groups(shapes):
  """Indexes of the items of each distinct shape, in order of first appearance."""
  groups = {}
  for i, s in enumerate(shapes):
    groups.setdefault(tuple(s), []).append(i)
  return list(groups.values())


def per_shape_compress(m, images):
  """The per-shape path, as the models coded lists before: the transforms per image, then one batch encode
  (`_encode_latents`, what `compress_batch` codes) per group of images of one latent shape."""
  xs = [x[None].to(torch.float32) for x in images]
  ys = [m.analysis_transform(x) for x in xs]
  zs = [m.hyper_analysis_transform(y) for y in ys]
  side_strings = m.side_entropy_model.compress_ragged([z[0] for z in zs]).split()
  psis = [m._psi(m.side_entropy_model.quantize(z), tuple(y.shape[1:-1])) for y, z in zip(ys, zs)]
  strings = [None] * len(xs)
  for members in _shape_groups([tuple(y.shape[1:-1]) for y in ys]):
    group = m._encode_latents(torch.cat([ys[i] for i in members]), torch.cat([psis[i] for i in members]))[0]
    for i, s in zip(members, group.split()):
      strings[i] = s
  return [(strings[i], side_strings[i]) + tuple(torch.tensor(t.shape[1:-1], dtype=torch.int32) for t in (x, y, z))
          for i, (x, y, z) in enumerate(zip(xs, ys, zs))]


def per_shape_decompress(m, items):
  """The per-shape path of `decompress_images`: one batch decode (`_decode_latents`, what `decompress_batch` decodes)
  per group of items of one latent shape."""
  z_hats = m.side_entropy_model.decompress_ragged(gen_ops.Strings.concat([it[1] for it in items]),
                                                  [tuple(int(v) for v in it[4]) for it in items])
  y_hws = [(int(it[3][0]), int(it[3][1])) for it in items]
  psis = [m._psi(z_hat[None], hw) for z_hat, hw in zip(z_hats, y_hws)]
  out = [None] * len(items)
  for members in _shape_groups(y_hws):
    y_hat = m._decode_latents(gen_ops.Strings.concat([items[i][0] for i in members]),
                              torch.cat([psis[i] for i in members]))
    for k, i in enumerate(members):
      x_hat = m.synthesis_transform(y_hat[k:k + 1])
      out[i] = models._to_uint8(x_hat[:, :int(items[i][2][0]), :int(items[i][2][1]), :])[0]
  return out


def _psis(m, items):
  z_hats = m.side_entropy_model.decompress_ragged(gen_ops.Strings.concat([it[1] for it in items]),
                                                  [tuple(int(v) for v in it[4]) for it in items])
  return [m._psi(z_hat[None], (int(it[3][0]), int(it[3][1]))) for z_hat, it in zip(z_hats, items)]


def _latents_ragged(m, items):
  """The decoded latents of the ragged path, as bytes per image."""
  em, psis = m.entropy_model, [p[0] for p in _psis(m, items)]
  handle = gen_ops.create_range_decoder(em._strings(gen_ops.Strings.concat([it[0] for it in items])), em._lookup_host())
  y_hats = m._decode_ragged(handle, psis, em.cdf_offset.cuda())
  em._finish_decode(handle)
  return [y.cpu().numpy().tobytes() for y in y_hats]


def _latents_per_shape(m, items):
  psis = _psis(m, items)
  out = [None] * len(items)
  for members in _shape_groups([tuple(int(v) for v in it[3]) for it in items]):
    y_hat = m._decode_latents(gen_ops.Strings.concat([items[i][0] for i in members]),
                              torch.cat([psis[i] for i in members]))
    for k, i in enumerate(members):
      out[i] = y_hat[k].cpu().numpy().tobytes()
  return out


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--models", default=",".join(MODELS))
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("context_ragged_bench needs a CUDA device")
  lists = {"a_kodak": [x.cuda() for x in rd_eval.synthetic(0)],
           "b_mixed": [x.cuda() for x in rd_eval.synthetic(1, rd_eval.mixed_shapes(1))]}
  res = {"card_before": rd_eval.card(), "num_filters": a.num_filters, "reps": a.reps,
         "lists": {k: [list(x.shape[:2]) for x in v] for k, v in lists.items()}}
  for name in a.models.split(","):
    torch.manual_seed(0)
    m = MODELS[name](num_filters=a.num_filters).build("cuda", patch=(64, 64)).fix_tables()
    res[name] = {"latent_depth": m.latent_depth}
    for lname, imgs in lists.items():
      with torch.no_grad():
        calls = {
            "compress_ragged": lambda: m.compress_images(imgs),
            "compress_per_shape": lambda: per_shape_compress(m, imgs),
        }
        items = calls["compress_ragged"]()
        coded = calls["compress_per_shape"]()
        calls["decompress_ragged"] = lambda: m.decompress_images(items)
        calls["decompress_per_shape"] = lambda: per_shape_decompress(m, coded)
        times = {c: [] for c in calls}
        launches, outs = {}, {}
        for fn in calls.values():  # warm-up
          fn()
        for _ in range(a.reps):
          for c, fn in calls.items():  # the two paths alternate call by call
            t, n, out = _once(fn)
            times[c].append(t)
            launches[c] = n
            outs[c] = out
        for r_item, s_item in zip(outs["compress_ragged"], outs["compress_per_shape"]):
          assert r_item[0].tolist() == s_item[0].tolist() and r_item[1].tolist() == s_item[1].tolist(), (name, lname)
        assert _latents_ragged(m, items) == _latents_per_shape(m, items), (name, lname)
        # (the synthesis transform's transposed convolutions are not bitwise repeatable from call to call, so images
        # decoded from the same latents may differ by one level where a value lies at a rounding boundary)
        diff = max(int((x.int() - y.int()).abs().max()) for x, y in zip(outs["decompress_ragged"],
                                                                         outs["decompress_per_shape"]))
        assert diff <= 1, (name, lname, diff)
      r = {c: {"ms": float(np.median(ts)), "all_ms": ts, "launches": launches[c]} for c, ts in times.items()}
      for op in ("compress", "decompress"):
        r[op + "_speedup"] = r[op + "_per_shape"]["ms"] / r[op + "_ragged"]["ms"]
      r["latent_shapes"] = len(_shape_groups([tuple(it[3].tolist()) for it in items]))
      res[name][lname] = r
      print(json.dumps({name: {lname: {c: v["ms"] if isinstance(v, dict) else v for c, v in r.items()}}}),
            file=sys.stderr, flush=True)
    del m
    torch.cuda.empty_cache()
  res["card_after"] = rd_eval.card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
