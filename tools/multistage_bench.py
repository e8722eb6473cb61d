"""Times MultistageModel against CheckerboardModel and MBT2018Model in one run, calls alternated between the models:
24 Kodak-shaped images (12 of 512x768, 12 of 768x512; random weights, synthetic content), N = M = 192 by default.

  python tools/multistage_bench.py [--reps 3] [--out FILE.json]

Per model: a one-image `compress` / `decompress`, `compress_images` / `decompress_images` of all 24 (also given per
image), and the library launches of each call.  For the multistage model also each stage's parameter pass alone on
one image (CUDA events around `functional.msc_params`).  Medians in ms; the card's name, power limit, SM clock and
clock-throttle reasons are read before and after in the same run.  Prints one JSON object."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import _lib, functional as F, models  # noqa: E402


def _card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active",
                        "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    q = torch.cuda.get_device_name()
  return q


def _images(n, seed=0):
  """tools/checkerboard_bench.py's images."""
  rng = np.random.default_rng(seed)
  out = []
  for i in range(n):
    h, w = (512, 768) if i % 2 == 0 else (768, 512)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 70 * np.sin(xx / (9.0 + i))[..., None] * np.cos(yy / 13.0)[..., None] * np.array([1.0, 0.8, 0.5])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 10, (h, w, 3)), 0, 255).astype(np.uint8)).cuda())
  return out


def _once(fn):
  """(ms, library launches, result) of one call ending in a synchronisation."""
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  t0 = time.perf_counter()
  out = fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t0) * 1e3, _lib.launch_count() - n0, out


def _stage_times(m, y_hat, psi, reps=20):
  """CUDA-event time of each stage's parameter pass."""
  res = {}
  for s in range(4):
    fn = lambda: F.msc_params(m._packed, y_hat, psi, s, m.num_scales)
    for _ in range(3):
      fn()
    ts = []
    for _ in range(reps):
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      fn()
      b.record()
      b.synchronize()
      ts.append(a.elapsed_time(b))
    res[f"stage_{s}"] = {"positions": F.msc_counts(*y_hat.shape[1:3])[s] * y_hat.shape[0], "ms": float(np.median(ts))}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--latent-depth", type=int, default=192)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--images", type=int, default=24)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("multistage_bench needs a CUDA device")
  imgs = _images(a.images)
  ms = {}
  for name, cls in (("mbt2018", models.MBT2018Model), ("checkerboard", models.CheckerboardModel),
                    ("multistage", models.MultistageModel)):
    torch.manual_seed(0)
    ms[name] = cls(num_filters=a.num_filters, latent_depth=a.latent_depth).build("cuda", patch=(64, 64)).fix_tables()
  res = {"card_before": _card(), "images": f"{a.images} Kodak-shaped (512x768 / 768x512), synthetic, random weights",
         "num_filters": a.num_filters, "latent_depth": a.latent_depth, "reps": a.reps}

  with torch.no_grad():
    items = {name: m.compress_images(imgs) for name, m in ms.items()}
    calls = {
        "compress_1": lambda m, it: m.compress(imgs[0]),
        "decompress_1": lambda m, it: m.decompress(*it[0]),
        "compress_images": lambda m, it: m.compress_images(imgs),
        "decompress_images": lambda m, it: m.decompress_images(it),
    }
    times = {n: {c: [] for c in calls} for n in ms}
    launches = {n: {} for n in ms}
    outs = {n: {} for n in ms}
    for name, m in ms.items():  # warm-up of every call
      for c, fn in calls.items():
        fn(m, items[name])
    for _ in range(a.reps):
      for c, fn in calls.items():
        for name, m in ms.items():  # the models alternate call by call
          t, l, out = _once(lambda: fn(m, items[name]))
          times[name][c].append(t)
          launches[name][c] = l
          outs[name][c] = out
    for name, m in ms.items():
      assert torch.equal(outs[name]["decompress_1"], outs[name]["decompress_images"][0]), name
      assert all(o.shape == x.shape for o, x in zip(outs[name]["decompress_images"], imgs))
      res[name] = {c: {"ms": float(np.median(ts)), "all_ms": ts, "launches": launches[name][c]}
                   for c, ts in times[name].items()}
      for c in ("compress_images", "decompress_images"):
        res[name][c]["ms_per_image"] = res[name][c]["ms"] / len(imgs)
      res[name]["bytes_24"] = sum(len(it[0].tolist()[0]) + len(it[1].tolist()[0]) for it in items[name])
    m = ms["multistage"]
    y = m.analysis_transform(imgs[0][None].float())
    psi = m._psi(m.side_entropy_model.quantize(m.hyper_analysis_transform(y)), tuple(y.shape[1:-1]))
    res["multistage"]["param_passes_1"] = _stage_times(m, torch.round(y).contiguous(), psi)
  res["card_after"] = _card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
