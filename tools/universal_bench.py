"""Universal quantisation on the H100: the per-call cost of the universal entropy models' compress / decompress,
whose coding tensors (noise levels, table indexes, offsets) come from one kernel, against another build.

Workloads (seeded):
  (A) UniversalBatchedEntropyModel, prior batch (128,), 15 noise levels, coding_rank=3, on [256, 16, 16, 128];
  (B) UniversalIndexedEntropyModel with 64 scale indexes, 15 noise levels, coding_rank=3, on [64, 16, 16, 192];
  (C) a ragged list of image latents [ceil(H/16), ceil(W/16), 128] of five image sizes (model A): one
      compress_ragged / decompress_ragged against the per-item compress / decompress loop.
For each call it reports the median of CUDA-event times, the CUDA kernels per call (torch.profiler, in a separate
pass) and the peak of the torch allocator above what was allocated before the call, and a digest of the strings.
With `--parent DIR` (a built checkout of another version) both trees are measured in fresh processes, alternated,
and the strings are compared; a tree without the ragged forms reports only the per-item loop.  The card's name,
power limit and SM clock are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/universal_bench.py [--images 256] [--reps 20] [--rounds 2] [--parent DIR] [--out DIR]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(768, 512), (512, 768), (1280, 720), (1024, 768), (2048, 1360)]


def card():
  import torch
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
  except Exception as e:  # pylint:disable=broad-except
    return {"name": torch.cuda.get_device_name(), "error": str(e)}


def measure(fn, reps, prof_fn=None, prof_scale=1):
  """(median ms of CUDA events, kernels per call, peak torch-allocator bytes above the start, last result).  The
  kernels are counted on `prof_fn` (default `fn`) times `prof_scale`: a per-item loop is profiled on a few items."""
  import torch
  from torch.profiler import ProfilerActivity, profile
  out = fn()
  torch.cuda.synchronize()
  ts = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  fn()
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated() - base
  calls = 3 if reps >= 3 else 1
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(calls):
      (prof_fn or fn)()
    torch.cuda.synchronize()
  kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                and not e.name.startswith(("Memcpy", "Memset")))
  print(f"  {statistics.median(ts):.3f} ms", file=sys.stderr, flush=True)
  return {"ms": statistics.median(ts), "kernels": kernels * prof_scale / calls, "peak_bytes": int(peak)}, out


def digest(strings_lists):
  h = hashlib.sha256()
  for s in strings_lists:
    h.update(len(s).to_bytes(8, "little"))
    h.update(s)
  return h.hexdigest()[:16]


def run_tree(root, images, reps):
  """All workloads with the package of the tree at `root`."""
  sys.path.insert(0, root)
  import numpy as np
  import torch
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  dev = torch.device("cuda")
  res = {}

  scales = torch.exp(torch.linspace(np.log(0.3), np.log(8.0), 128))
  prior = D.NoisyLogistic(loc=torch.zeros(128), scale=scales)
  em = E.UniversalBatchedEntropyModel(prior, coding_rank=3, compression=True, num_noise_levels=15)
  g = torch.Generator(device=dev).manual_seed(0)
  x = torch.randn(256, 16, 16, 128, generator=g, device=dev) * scales.to(dev) * 1.5
  print("A batched", file=sys.stderr, flush=True)
  r, strings = measure(lambda: em.compress(x), reps)
  res["A_batched_compress"] = dict(r, strings=digest(strings.tolist()), bytes=int(sum(map(len, strings.tolist()))))
  r, back = measure(lambda: em.decompress(strings, (16, 16)), reps)
  res["A_batched_decompress"] = dict(r, max_abs_error=float((back - x).abs().max()))

  emi = E.UniversalIndexedEntropyModel(D.NoisyNormal, (64,), dict(loc=lambda i: 0. * i[..., 0],
                                                                    scale=lambda i: torch.exp(i[..., 0] / 8. - 2.)),
                                       coding_rank=3, compression=True, num_noise_levels=15)
  ind = torch.randint(0, 64, (64, 16, 16, 192, 1), generator=g, device=dev).float()
  xi = torch.randn(64, 16, 16, 192, generator=g, device=dev) * torch.exp(ind[..., 0] / 8. - 2.) * 1.5
  print("B indexed", file=sys.stderr, flush=True)
  r, si = measure(lambda: emi.compress(xi, ind), reps)
  res["B_indexed_compress"] = dict(r, strings=digest(si.tolist()), bytes=int(sum(map(len, si.tolist()))))
  r, backi = measure(lambda: emi.decompress(si, ind), reps)
  res["B_indexed_decompress"] = dict(r, max_abs_error=float((backi - xi).abs().max()))

  rng = np.random.default_rng(0)
  sizes = [SIZES[i] for i in rng.integers(0, len(SIZES), images)]
  items = [torch.randn(-(-h // 16), -(-w // 16), 128, generator=g, device=dev) * scales.to(dev) * 1.5
           for h, w in sizes]
  bshapes = [tuple(t.shape[:2]) for t in items]
  print("C ragged", file=sys.stderr, flush=True)
  few = max(1, images // 16)  # the loops' kernels are counted on `few` items and scaled
  r, loop = measure(lambda: [em.compress(t).tolist()[0] for t in items], 1,
                    lambda: [em.compress(t).tolist()[0] for t in items[:few]], images / few)
  res["C_loop_compress"] = dict(r, strings=digest(loop))
  r, _ = measure(lambda: [em.decompress([s], b) for s, b in zip(loop, bshapes)], 1,
                 lambda: [em.decompress([s], b) for s, b in zip(loop[:few], bshapes[:few])], images / few)
  res["C_loop_decompress"] = r
  if hasattr(em, "compress_ragged"):
    r, rs = measure(lambda: em.compress_ragged(items), reps)
    res["C_ragged_compress"] = dict(r, strings=digest(rs.tolist()))
    r, rb = measure(lambda: em.decompress_ragged(rs, bshapes), reps)
    one = [em.decompress([s], b)[0] for s, b in zip(loop, bshapes)]
    res["C_ragged_decompress"] = dict(r, equals_loop=all(torch.equal(a, b) for a, b in zip(rb, one)))
  res["C_images"] = {"count": images, "elements": int(sum(t.numel() for t in items))}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--images", type=int, default=256)
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--rounds", type=int, default=2)
  ap.add_argument("--parent", default=None, help="root of another built tree to compare against")
  ap.add_argument("--tree", default=None, help=argparse.SUPPRESS)  # child mode: tree root to measure
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if args.tree:
    print(json.dumps(run_tree(args.tree, args.images, args.reps)))
    return

  import torch
  if not torch.cuda.is_available():
    raise SystemExit("universal_bench needs a CUDA device")
  trees = [("this", ROOT)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
  res = {"card_before": card(), "images": args.images, "reps": args.reps}
  runs = {tag: [] for tag, _ in trees}
  for _ in range(args.rounds):
    for tag, root in trees:
      print(f"measuring {tag}", file=sys.stderr, flush=True)
      out = subprocess.run([sys.executable, os.path.abspath(__file__), "--tree", root, "--images", str(args.images),
                            "--reps", str(args.reps)], stdout=subprocess.PIPE, text=True)  # (progress on stderr)
      if out.returncode:
        raise SystemExit(f"measuring {root} failed")
      runs[tag].append(json.loads(out.stdout.strip().splitlines()[-1]))
  for tag, rs in runs.items():
    summary = {}
    for name in rs[0]:
      first = rs[0][name]
      entry = {k: v for k, v in first.items() if k not in ("ms",)}
      if "ms" in first:
        entry["ms_per_round"] = [r[name]["ms"] for r in rs]
        entry["ms"] = statistics.median(entry["ms_per_round"])
      summary[name] = entry
    res[tag] = summary
  if args.parent:
    this, parent = res["this"], res["parent"]
    res["strings_identical"] = all(this[k]["strings"] == parent[k]["strings"]
                                   for k in ("A_batched_compress", "B_indexed_compress", "C_loop_compress"))
    res["ragged_strings_equal_loop"] = this["C_ragged_compress"]["strings"] == this["C_loop_compress"]["strings"]
    res["speedup_vs_parent"] = {k: parent[k]["ms"] / this[k]["ms"] for k in parent if "ms" in parent[k]}
    res["ragged_speedup_vs_parent_loop"] = {
        "compress": parent["C_loop_compress"]["ms"] / this["C_ragged_compress"]["ms"],
        "decompress": parent["C_loop_decompress"]["ms"] / this["C_ragged_decompress"]["ms"]}
  res["card_after"] = card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "universal_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
