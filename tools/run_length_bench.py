"""Run-length coding on the H100: one ragged launch against the run-length models' per-unit loop.

Workloads (seeded):
  (A) a cfg2-shaped bottleneck [256, 16, 16, 128] of sparse Laplace-like latents (about 7 % non-zeros) at
      coding_rank=3: 256 coding units of 32 768 elements;
  (B) a ragged set of image latents [ceil(H/16), ceil(W/16), 128], sizes drawn from five image sizes, one coding unit
      per image.
For each it times LaplaceEntropyModel(coding_rank=3)'s per-unit `compress` / `decompress` against one
`compress_ragged` / `decompress_ragged` call and checks that both give the same strings and values.  On (A) it also
times the encode kernels alone and the decode kernel alone (torch.profiler).  With `--parent DIR` (a built checkout
of another version) it times the one-string `gen_ops.run_length_decode` of one 300 000-element unit in both trees,
alternated in fresh processes, and checks that the decoded tensors agree.  The card's name and power limit are read
in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/run_length_bench.py [--images 40] [--seed 0] [--reps 3] [--parent DIR] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(768, 512), (512, 768), (1280, 720), (1024, 768), (2048, 1360)]
C = 128
PARAMS = (-1, 0, False)  # LaplaceEntropyModel's defaults


def sparse_latents(rng, shape):
  """Laplace-like integers, about 7 % non-zero."""
  mag = np.ceil(rng.exponential(2.0, shape)).astype(np.int32)
  return (mag * np.where(rng.random(shape) < 0.5, -1, 1) * (rng.random(shape) < 0.07)).astype(np.float32)


def single_decode(root, reps):
  """Median time of gen_ops.run_length_decode of one 300 000-element unit with the library of the tree at `root`."""
  sys.path.insert(0, root)
  import torch
  from compression_b200 import gen_ops
  d = torch.from_numpy(sparse_latents(np.random.default_rng(7), (300_000,)).astype(np.int32))
  code = gen_ops.run_length_encode(d, *PARAMS)
  out = gen_ops.run_length_decode(code, [d.numel()], *PARAMS)
  torch.cuda.synchronize()
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    out = gen_ops.run_length_decode(code, [d.numel()], *PARAMS)  # synchronises
    ts.append(time.perf_counter() - t0)
  return {"ms": sorted(ts)[len(ts) // 2] * 1e3, "bytes": len(code), "round_trip": bool(torch.equal(out.cpu(), d)),
          "checksum": int(out.long().mul(torch.arange(1, d.numel() + 1, device=out.device)).sum())}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--images", type=int, default=40)
  ap.add_argument("--seed", type=int, default=0)
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--parent", default=None, help="root of another built tree for the one-string decode comparison")
  ap.add_argument("--single-decode", default=None, help=argparse.SUPPRESS)  # child mode: tree root to time
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if args.single_decode:
    print(json.dumps(single_decode(args.single_decode, max(args.reps, 5))))
    return

  import torch
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tools"))
  from ragged_bench import card, kernel_ms, timed
  from compression_b200 import run_length_models as M
  if not torch.cuda.is_available():
    raise SystemExit("run_length_bench needs a CUDA device")
  dev = torch.device("cuda")
  res = {"card_before": card(), "params": PARAMS}
  em = M.LaplaceEntropyModel(coding_rank=3)
  rng = np.random.default_rng(args.seed)

  def compare(name, items):
    shapes = [tuple(x.shape) for x in items]
    r = {"units": len(items), "elements": int(sum(x.numel() for x in items)),
         "longest_unit": int(max(x.numel() for x in items)),
         "nonzero_fraction": float(sum(int((x != 0).sum()) for x in items) / sum(x.numel() for x in items))}
    r["encode_ms_ragged"], strings = timed(lambda: em.compress_ragged(items), args.reps)
    r["encode_ms_per_unit_loop"], loop = timed(lambda: [em.compress(x)[()] for x in items], 1)
    ragged_l = strings.tolist()
    r["strings_identical"] = loop == ragged_l
    r["bytes"] = int(sum(len(s) for s in ragged_l))
    r["decode_ms_ragged"], back = timed(lambda: em.decompress_ragged(strings, shapes), args.reps)
    r["decode_ms_per_unit_loop"], back_loop = timed(lambda: [em.decompress(s, sh) for s, sh in zip(loop, shapes)], 1)
    r["decoded_identical"] = all(torch.equal(a, b) and torch.equal(a.cpu(), x.cpu())
                                 for a, b, x in zip(back, back_loop, items))
    r["speedup"] = {"encode": r["encode_ms_per_unit_loop"] / r["encode_ms_ragged"],
                    "decode": r["decode_ms_per_unit_loop"] / r["decode_ms_ragged"]}
    res[name] = r
    return strings, shapes

  xa = torch.from_numpy(sparse_latents(rng, (256, 16, 16, C))).to(dev)
  items_a = list(xa)
  strings_a, shapes_a = compare("A_cfg2_bottleneck_256x16x16x128", items_a)
  sizes = [SIZES[i] for i in rng.integers(0, len(SIZES), args.images)]
  items_b = [torch.from_numpy(sparse_latents(rng, (-(-h // 16), -(-w // 16), C))).to(dev) for h, w in sizes]
  compare(f"B_{args.images}_images_from_{len(SIZES)}_sizes", items_b)

  def enc_kernels(prof_key):
    return ("rl_" in prof_key and "rl_decode" not in prof_key) or "DeviceScan" in prof_key
  from torch.profiler import ProfilerActivity, profile
  em.compress_ragged(items_a)
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
      em.compress_ragged(items_a)
    torch.cuda.synchronize()
  enc_k = sum(e.device_time_total for e in prof.key_averages() if enc_kernels(e.key)) / 5 / 1e3
  dec_k = kernel_ms(lambda: em.decompress_ragged(strings_a, shapes_a), "rl_decode_kernel")
  res["A_kernels_ms"] = {"encode_kernels": enc_k, "decode_kernel": dec_k,
                         "source": "torch.profiler device time per call, mean of 5 calls"}

  if args.parent:
    runs = {"this": [], "parent": []}
    for _ in range(3):
      for tag, root in (("this", ROOT), ("parent", os.path.abspath(args.parent))):
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--single-decode", root], check=True,
                             capture_output=True, text=True).stdout.strip().splitlines()[-1]
        runs[tag].append(json.loads(out))
    res["single_decode_300k"] = {
        tag: {"ms": [r["ms"] for r in rs], "bytes": rs[0]["bytes"], "round_trip": all(r["round_trip"] for r in rs)}
        for tag, rs in runs.items()}
    res["single_decode_300k"]["same_output"] = len({r["checksum"] for rs in runs.values() for r in rs}) == 1
  else:
    res["single_decode_300k"] = "not measured (no --parent tree)"
  res["card_after"] = card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "run_length_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
