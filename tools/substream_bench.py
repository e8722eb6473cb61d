"""Times one-image coding and image-list decoding of the five substream-capable models at several substream counts
(DESIGN §3.14), in one run with the counts alternated call by call.

  python tools/substream_bench.py [--substreams 1,8,32,128] [--reps 5] [--list-reps 3] [--models ...] [--out F]

For each model (torch.manual_seed(0) weights, num_filters 192 and the model's default latent depth; one model object
per S, with the same weights):
  one image   `compress` and `decompress` of one seeded Kodak-shaped 512x768 image (tools/rd_eval.py --synthetic
              kodak, image 0), and for the context models the y decode alone (`_decode_latents`, the parameter
              passes, range decodes and scatters, from a precomputed psi);
  lists       `decompress_images` of the 24-image lists of tools/context_ragged_bench.py: (a) the Kodak shapes,
              (b) 24 seeded images of 24 different shapes (not for MS2020, whose y sides must be multiples of 4).
Each entry is the median and range of host-timed calls ending in a synchronise (after one warm-up call of every S),
with the library launches of one call and the bytes per image (all of an image's strings, headers included).  Every
S must decode the latents of S = 1 bit for bit.  The card's name, power limit and SM clock are read before and after.
Prints one JSON object."""
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

MODELS = {"bls2017": models.BLS2017Model, "bmshj2018": models.BMSHJ2018Model, "ms2020": models.MS2020Model,
          "checkerboard": models.CheckerboardModel, "space_channel": models.SpaceChannelModel}
CONTEXT = ("checkerboard", "space_channel")


def _once(fn):
  """(ms, library launches, result) of one call ending in a synchronisation."""
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) * 1e3, _lib.launch_count() - n0, out


def _bytes(item):
  return sum(s.nbytes() for s in item if isinstance(s, gen_ops.Strings))


def _alternate(calls, reps):
  """{(S, name): (times, launches, last result)}, the S values alternated call by call after one warm-up each."""
  for fn in calls.values():
    fn()
  out = {k: ([], 0, None) for k in calls}
  for _ in range(reps):
    for k, fn in calls.items():
      t, n, r = _once(fn)
      out[k] = (out[k][0] + [t], n, r)
  return out


def _summary(times, launches):
  return {"ms": float(np.median(times)), "min_ms": float(min(times)), "max_ms": float(max(times)),
          "launches": launches}


def _capture(m, fn):
  """fn()'s result and the latents its synthesis transform received."""
  got = []
  hook = m.synthesis_transform.register_forward_pre_hook(lambda _, args: got.append(args[0].clone()))
  try:
    return fn(), got
  finally:
    hook.remove()


def bench_model(name, counts, reps, list_reps, num_filters, image, lists):
  ms = {}
  for S in counts:
    torch.manual_seed(0)
    ms[S] = MODELS[name](num_filters=num_filters, substreams=S).build("cuda", patch=(64, 64)).fix_tables()
  state = ms[counts[0]].state_dict()
  for S in counts:
    ms[S].load_state_dict(state)
    ms[S].fix_tables()
  res = {"one_image": {}, "lists": {}}
  with torch.no_grad():
    items = {S: ms[S].compress(image) for S in counts}
    calls = {}
    for S in counts:
      calls[(S, "compress")] = lambda S=S: ms[S].compress(image)
      calls[(S, "decompress")] = lambda S=S: _capture(ms[S], lambda: ms[S].decompress(*items[S]))
      if name in CONTEXT:
        it = items[S]
        z_hat = ms[S].side_entropy_model.decompress(it[1], tuple(int(v) for v in it[4]), substreams=S)
        psi = ms[S]._psi(z_hat, (int(it[3][0]), int(it[3][1])))
        calls[(S, "y_decode")] = lambda S=S, psi=psi: ms[S]._decode_latents(items[S][0], psi)
    out = _alternate(calls, reps)
    base = out[(counts[0], "decompress")][2][1]
    for S in counts:
      assert all(torch.equal(a, b) for a, b in zip(out[(S, "decompress")][2][1], base)), (name, S)
      r = {op: _summary(out[(S, op)][0], out[(S, op)][1]) for op in ("compress", "decompress", "y_decode")
           if (S, op) in out}
      r["bytes"] = _bytes(items[S])
      res["one_image"][S] = r
    for lname, imgs in lists.items():
      if name == "ms2020" and any(x.shape[0] % 64 or x.shape[1] % 64 for x in imgs):
        continue  # MS2020's slice transforms need y's sides to be multiples of 4 (its hyper transforms downsample by 4)
      coded = {S: ms[S].compress_images(imgs) for S in counts}
      calls = {(S, "decompress_images"): (lambda S=S: _capture(ms[S], lambda: ms[S].decompress_images(coded[S])))
               for S in counts}
      out = _alternate(calls, list_reps)
      base = out[(counts[0], "decompress_images")][2][1]
      res["lists"][lname] = {}
      for S in counts:
        assert all(torch.equal(a, b) for a, b in zip(out[(S, "decompress_images")][2][1], base)), (name, lname, S)
        r = _summary(*out[(S, "decompress_images")][:2])
        r["bytes_per_image"] = sum(_bytes(it) for it in coded[S]) / len(imgs)
        res["lists"][lname][S] = r
  return res


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument("--substreams", default="1,8,32,128")
  ap.add_argument("--reps", type=int, default=5)
  ap.add_argument("--list-reps", type=int, default=3)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--models", default=",".join(MODELS))
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("substream_bench needs a CUDA device")
  counts = [int(s) for s in a.substreams.split(",")]
  image = rd_eval.synthetic(0)[0].cuda()
  lists = {"a_kodak": [x.cuda() for x in rd_eval.synthetic(0)],
           "b_mixed": [x.cuda() for x in rd_eval.synthetic(1, rd_eval.mixed_shapes(1))]}
  res = {"card_before": rd_eval.card(), "num_filters": a.num_filters, "substreams": counts, "reps": a.reps,
         "list_reps": a.list_reps, "image": list(image.shape[:2])}
  for name in a.models.split(","):
    res[name] = bench_model(name, counts, a.reps, a.list_reps, a.num_filters, image, lists)
    print(json.dumps({name: {S: {k: (v["ms"] if isinstance(v, dict) else v) for k, v in r.items()}
                             for S, r in res[name]["one_image"].items()}}), file=sys.stderr, flush=True)
    torch.cuda.empty_cache()
  res["card_after"] = rd_eval.card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
