"""Times MBT2018Model's column tiles (DESIGN §3.15): one-image coding of a 512x768 and a 768x512 image and the
decoding of two 24-image lists at several tile counts T, alternated call by call in one run.

  python tools/ar_tiles_bench.py [--tiles 1,8,16,24,48] [--reps 5] [--list-reps 3] [--num-filters 192] [--out F]

One model object per T (torch.manual_seed(0) weights, N = M = 192 by default; every object loads the first one's
state).  For each image (tools/rd_eval.py --synthetic kodak, images 0 and 12, latents 32 x 48 and 48 x 32):
`compress`, `decompress`, and the latent decode alone (`_decode_latents`: the range decoder and the tile kernel,
from a precomputed psi).  For the lists of tools/context_ragged_bench.py, (a) the 24 Kodak shapes and (b) 24 seeded
images of 24 different shapes: `decompress_images`.  Each entry is the median and range of host-timed calls ending
in a synchronise (after one warm-up call of every T), the library launches of one call and the bytes (all of an
image's strings, headers included).  Every T must give the latents of T = 1 bit for bit: the tool asserts it for
every image and list.  The card's name, power limit and SM clock are read before and after.  Prints one JSON
object."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from compression_b200 import models  # noqa: E402
import rd_eval  # noqa: E402
from substream_bench import _alternate, _bytes, _capture, _summary  # noqa: E402


def bench(counts, reps, list_reps, num_filters, images, lists):
  ms = {}
  for T in counts:
    torch.manual_seed(0)
    ms[T] = models.MBT2018Model(num_filters=num_filters, latent_depth=num_filters, tiles=T).build("cuda",
                                                                                                   patch=(64, 64))
  state = ms[counts[0]].state_dict()
  for T in counts:
    ms[T].load_state_dict(state)
    ms[T].fix_tables()
  res = {"images": {}, "lists": {}}
  with torch.no_grad():
    for iname, image in images.items():
      items = {T: ms[T].compress(image) for T in counts}
      it = items[counts[0]]
      m0 = ms[counts[0]]
      z_hat = m0.side_entropy_model.decompress(it[1], tuple(int(v) for v in it[4]))
      psi = m0._psi(z_hat, (int(it[3][0]), int(it[3][1])))
      calls = {}
      for T in counts:
        calls[(T, "compress")] = lambda T=T: ms[T].compress(image)
        calls[(T, "decompress")] = lambda T=T: _capture(ms[T], lambda: ms[T].decompress(*items[T]))
        calls[(T, "y_decode")] = lambda T=T: ms[T]._decode_latents(items[T][0], psi)
      out = _alternate(calls, reps)
      base = out[(counts[0], "y_decode")][2]
      res["images"][iname] = {}
      for T in counts:
        assert torch.equal(out[(T, "y_decode")][2], base), (iname, T)
        assert all(torch.equal(a, b) for a, b in zip(out[(T, "decompress")][2][1], [base])), (iname, T)
        r = {op: _summary(out[(T, op)][0], out[(T, op)][1]) for op in ("compress", "decompress", "y_decode")}
        r["bytes"] = _bytes(items[T])
        res["images"][iname][T] = r
      print(json.dumps({iname: {T: {k: (v["ms"] if isinstance(v, dict) else v) for k, v in r.items()}
                                for T, r in res["images"][iname].items()}}), file=sys.stderr, flush=True)
    for lname, imgs in lists.items():
      coded = {T: ms[T].compress_images(imgs) for T in counts}
      calls = {(T, "decompress_images"): (lambda T=T: _capture(ms[T], lambda: ms[T].decompress_images(coded[T])))
               for T in counts}
      out = _alternate(calls, list_reps)
      base = out[(counts[0], "decompress_images")][2][1]
      res["lists"][lname] = {}
      for T in counts:
        assert all(torch.equal(a, b) for a, b in zip(out[(T, "decompress_images")][2][1], base)), (lname, T)
        r = _summary(*out[(T, "decompress_images")][:2])
        r["bytes_per_image"] = sum(_bytes(it) for it in coded[T]) / len(imgs)
        res["lists"][lname][T] = r
      print(json.dumps({lname: {T: r["ms"] for T, r in res["lists"][lname].items()}}), file=sys.stderr, flush=True)
  return res


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--tiles", default="1,8,16,24,48")
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--list-reps", type=int, default=3)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("ar_tiles_bench needs a CUDA device")
  counts = [int(s) for s in a.tiles.split(",")]
  kodak = rd_eval.synthetic(0)
  images = {"512x768": kodak[0].cuda(), "768x512": kodak[12].cuda()}
  lists = {"a_kodak": [x.cuda() for x in kodak],
           "b_mixed": [x.cuda() for x in rd_eval.synthetic(1, rd_eval.mixed_shapes(1))]}
  res = {"card_before": rd_eval.card(), "num_filters": a.num_filters, "tiles": counts, "reps": a.reps,
         "list_reps": a.list_reps}
  res.update(bench(counts, a.reps, a.list_reps, a.num_filters, images, lists))
  res["card_after"] = rd_eval.card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
