"""UnboundedIndexRangeEncode / Decode throughput on the GPU against the compiled reference on the host cores.

Workloads (cfg2 tables: the 128 rows of tests/golden/cfg2_tables.npz, each a [-12, 0, c1, ..., 4096] lookup whose
last bin is already the escape, as cdf / cdf_size / offset = cdf_offset; data = cfg2's synthetic latents rounded,
channel c coded with row c):
  cfg2     256 strings x 32768 symbols: one ragged call, and a loop of 256 one-string ops
  single   one string of 32768 symbols and one of 1.4 M symbols (a single string is one serial chain)
  escape   the cfg2 latents times 200 (most symbols escape; |u| stays below 2^16, where the reference is defined at
           overflow_width 16), at overflow_width 1 and 16, 64 strings x 32768
GPU figures are medians of CUDA-event-timed calls (every call ends in its own host synchronisation); the reference is
oracle/unbounded's restatement of the op loop around the reference's RangeEncoder / RangeDecoder (built into
oracle/_ref/libubi_ref.so), on 1 thread and on the best of a few thread counts.  Prints one JSON object; --out also writes it to a file.

  python tools/unbounded_bench.py [--reps 7] [--out FILE]
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

from oracle import unbounded as ubi  # noqa: E402
from compression_b200 import functional as F  # noqa: E402
from compression_b200 import gen_ops  # noqa: E402

W_CFG2 = 4  # overflow_width of the cfg2 workloads


def card():
  q = "name,power.limit,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
  except Exception as e:  # pylint:disable=broad-except
    return {"name": torch.cuda.get_device_name(), "error": str(e)}


def cfg2_tables():
  g = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_tables.npz"))
  lookup, rows, at = g["lookup"], [], 0
  while at < lookup.size:
    p = abs(int(lookup[at]))
    end = at + 1
    while lookup[end] != 1 << p:
      end += 1
    rows.append(lookup[at + 1:end + 1])
    at = end + 1
    while at < lookup.size and lookup[at] == 1 << p:
      at += 1
  W = max(r.size for r in rows)
  cdf = np.full((len(rows), W), 1 << p, np.int32)
  for i, r in enumerate(rows):
    cdf[i, :r.size] = r
  return cdf, np.array([r.size for r in rows], np.int32), g["cdf_offset"].astype(np.int32), p


def latents(n_strings, n_per, scale=1.0):
  gen = torch.Generator().manual_seed(2)
  C = 128
  scales = torch.exp(torch.linspace(np.log(0.3), np.log(8.0), C))
  u = torch.rand(n_strings * n_per // C, C, generator=gen) - 0.5
  y = -scales * torch.sign(u) * torch.log1p(-2 * u.abs()).clamp_min(-17.0)
  data = torch.round(y * scale).to(torch.int32).reshape(-1).numpy()
  index = np.tile(np.arange(C, dtype=np.int32), data.size // C)
  return data, index


def gpu_ms(fn, reps):
  fn()
  torch.cuda.synchronize()
  ts = []
  for _ in range(reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    ts.append(a.elapsed_time(b))
  return float(np.median(ts))


def host_ms(fn, reps=3):
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    fn()
    ts.append((time.perf_counter() - t0) * 1e3)
  return float(np.median(ts))


def workload(name, data, index, lengths, tables, p, w, reps, loop=False):
  cdf, cdf_size, offset = tables
  n = int(sum(lengths))
  dev = torch.device("cuda")
  d_data, d_index = torch.from_numpy(data).to(dev), torch.from_numpy(index).to(dev)
  d_cdf, d_size, d_off = (torch.from_numpy(x).to(dev) for x in tables)
  args = (d_cdf, d_size, d_off, p, w)
  strings = F.unbounded_index_range_encode_ragged(d_data, d_index, lengths, *args)
  enc = gpu_ms(lambda: F.unbounded_index_range_encode_ragged(d_data, d_index, lengths, *args), reps)
  dec = gpu_ms(lambda: F.unbounded_index_range_decode_ragged(strings, d_index, lengths, *args), reps)
  back = F.unbounded_index_range_decode_ragged(strings, d_index, lengths, *args).cpu().numpy()
  R = ubi.ref()
  want = R.encode_batch(data, index, lengths, cdf, cdf_size, offset, p, w, threads=1)
  res = {"workload": name, "strings": len(lengths), "symbols": n, "precision": p, "overflow_width": w,
         "bytes": strings.nbytes(), "identical_to_oracle": strings.tolist() == want,
         "round_trip": bool(np.array_equal(back, data)),
         "gpu_encode_ms": enc, "gpu_decode_ms": dec,
         "gpu_encode_gsym_s": n / enc / 1e6, "gpu_decode_gsym_s": n / dec / 1e6}
  if loop:
    offs = np.concatenate([[0], np.cumsum(lengths)])
    res["gpu_encode_one_string_op_loop_ms"] = gpu_ms(
        lambda: [gen_ops.unbounded_index_range_encode(d_data[offs[i]:offs[i + 1]], d_index[offs[i]:offs[i + 1]], *args)
                 for i in range(len(lengths))], max(3, reps // 2))
  threads = sorted({1, 4, 16, 64, min(len(lengths), R.hardware_threads())})
  ref = {}
  for t in threads:
    if t > 1 and len(lengths) == 1:
      continue
    ref[t] = (host_ms(lambda: R.encode_batch(data, index, lengths, cdf, cdf_size, offset, p, w,
                                                                    threads=t)),
              host_ms(lambda: R.decode_batch(want, index, lengths, cdf, cdf_size, offset, p, w,
                                                                   threads=t)))
  best = min(ref, key=lambda t: ref[t][0])
  res.update({"ref_1_thread_encode_gsym_s": n / ref[1][0] / 1e6, "ref_1_thread_decode_gsym_s": n / ref[1][1] / 1e6,
              "ref_best_threads": best, "ref_best_encode_gsym_s": n / ref[best][0] / 1e6,
              "ref_best_decode_gsym_s": n / min(v[1] for v in ref.values()) / 1e6})
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=7)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  assert torch.cuda.is_available(), "this benchmark measures the GPU"
  cdf, cdf_size, offset, p = cfg2_tables()
  tables = (cdf, cdf_size, offset)
  out = {"card": card(), "host_threads": ubi.ref().hardware_threads(), "results": []}
  data, index = latents(256, 32768)
  out["results"].append(workload("cfg2 256 x 32768", data, index, [32768] * 256, tables, p, W_CFG2, a.reps, True))
  out["results"].append(workload("single 32768", data[:32768], index[:32768], [32768], tables, p, W_CFG2, a.reps))
  n1 = 1_400_000 // 128 * 128
  out["results"].append(workload("single 1.4M", data[:n1], index[:n1], [n1], tables, p, W_CFG2, max(3, a.reps // 2)))
  data, index = latents(64, 32768, scale=200.0)
  for w in (1, 16):
    out["results"].append(workload(f"escape-heavy 64 x 32768 w={w}", data, index, [32768] * 64, tables, p, w, a.reps))
  out["card_after"] = card()
  text = json.dumps(out, indent=1)
  print(text)
  if a.out:
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
      f.write(text)


if __name__ == "__main__":
  main()
