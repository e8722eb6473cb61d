"""float16 / bfloat16 bottlenecks on the 16-bit range-coder entries against the unfused path they replace.

Workloads (cfg2 tables, tests/golden/cfg2_tables.npz, in a ContinuousBatchedEntropyModel over prior_shape (128,)):
  full     bench.py's cfg2 latents y[256,16,16,128] cast to the type: compress, decompress
  ragged   a list of 256 items (h, w, 128), h and w drawn from [8, 24] (seed 3), from the same latents:
           compress_ragged(return_decoded=True)
The unfused path is `compress(..., fused=False)` / `decompress(..., fused=False)`, and for the ragged encode the
model's previous route (int32 symbols from the torch quantise graph, the int32 ragged encode, then a ragged decode of
the fresh strings and the torch dequantise graph), selected by clearing the model's `_coder16_models`.  The two paths
are timed alternately in one process, each call between host synchronisations; medians of --reps.  The outputs of
both paths are compared bit for bit on the timed inputs.  The card's name, power limit and SM clock are read in the
same run.  Prints one JSON object; --out also writes it to a file.

  python tools/coder16_bench.py [--reps 9] [--warmup 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (cfg2's latents)
from compression_b200 import entropy_models as E  # noqa: E402


def card():
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
  except Exception as e:  # pylint:disable=broad-except
    return {"name": torch.cuda.get_device_name(), "error": str(e)}


def model(dtype):
  z = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_tables.npz"))
  q = torch.from_numpy(z["quantization_offset"]) if z["has_qoff"] else None
  return E.ContinuousBatchedEntropyModel(
      prior_shape=(128,), coding_rank=3, compression=True, cdf=torch.from_numpy(z["lookup"]),
      cdf_offset=torch.from_numpy(z["cdf_offset"]), bottleneck_dtype=dtype, offset_heuristic=False,
      quantization_offset=q).cuda()


def timed(fn):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return time.perf_counter() - t0, out


def same(a, b):
  if isinstance(a, torch.Tensor):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))
  return a.tolist() == b.tolist()


def compare(name, n_sym, new, old, check, reps, warmup):
  """Alternates new / old `reps` times after `warmup` rounds; medians in ms and Gsym/s."""
  for _ in range(warmup):
    new()
    old()
  t_new, t_old = [], []
  out_new = out_old = None
  for _ in range(reps):
    t, out_new = timed(new)
    t_new.append(t)
    t, out_old = timed(old)
    t_old.append(t)
  ok = check(out_new, out_old)
  m_new, m_old = float(np.median(t_new)), float(np.median(t_old))
  return dict(workload=name, symbols=n_sym, new_ms=round(1e3 * m_new, 3), unfused_ms=round(1e3 * m_old, 3),
              new_gsym_s=round(n_sym / m_new / 1e9, 3), unfused_gsym_s=round(n_sym / m_old / 1e9, 3),
              speedup=round(m_old / m_new, 2), new_ms_min_max=[round(1e3 * min(t_new), 3), round(1e3 * max(t_new), 3)],
              unfused_ms_min_max=[round(1e3 * min(t_old), 3), round(1e3 * max(t_old), 3)], bitwise_equal=bool(ok))


def run(dtype, reps, warmup):
  em = model(dtype)
  _, ys = bench.synth_latents(0, 1)
  y = ys[0].to(dtype).cuda()
  n_sym = y.numel()
  res = []
  res.append(compare("compress", n_sym, lambda: em.compress(y), lambda: em.compress(y, fused=False), same, reps,
                     warmup))
  strings = em.compress(y)
  res.append(compare("decompress", n_sym, lambda: em.decompress(strings, (16, 16)),
                     lambda: em.decompress(strings, (16, 16), fused=False), same, reps, warmup))
  g = np.random.default_rng(3)
  hw = g.integers(8, 25, size=(256, 2))
  items = [y[i, :h, :w].contiguous() for i, (h, w) in enumerate(hw)]
  n_rag = sum(int(x.numel()) for x in items)

  def ragged(new):
    em._coder16_models = new
    try:
      return em.compress_ragged(items, return_decoded=True)
    finally:
      em._coder16_models = True

  def check_ragged(a, b):
    return same(a[0], b[0]) and len(a[1]) == len(b[1]) and all(same(u, v) for u, v in zip(a[1], b[1]))

  res.append(compare("compress_ragged(return_decoded=True), 256 items", n_rag, lambda: ragged(True),
                     lambda: ragged(False), check_ragged, reps, warmup))
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=9)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("coder16_bench needs a CUDA device")
  torch.cuda.set_device(0)
  result = dict(card_before=card(), results={})
  for dtype in (torch.bfloat16, torch.float16):
    result["results"][str(dtype).replace("torch.", "")] = run(dtype, args.reps, args.warmup)
  result["card_after"] = card()
  text = json.dumps(result, indent=1)
  print(text)
  if args.out:
    with open(args.out, "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
