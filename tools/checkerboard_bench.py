"""Times CheckerboardModel against MBT2018Model in one run, calls alternated between the two models: 24 Kodak-shaped
images (12 of 512x768, 12 of 768x512; random weights, synthetic content), N = M = 192 by default.

  python tools/checkerboard_bench.py [--reps 3] [--out FILE.json]

Per model: latent encode and decode of 12 images of one shape (`_encode_latents` / `_decode_latents`),
`compress_images` / `decompress_images` of all 24, a one-image `compress` / `decompress`, and the library launches of
each call.  For the checkerboard model also the parameter passes alone (CUDA events around `functional.cb_params`)
with their FP32 rate on the multiply-adds the layer shapes give.  Medians in ms; the card's name, power limit and SM
clock are read in the same run.  Prints one JSON object."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    q = torch.cuda.get_device_name()
  return q


def _images(n, seed=0):
  """tools/mbt2018_bench.py's images."""
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


def _macs(M, anchors):
  """Multiply-adds per position of one pass: the anchors' layer 1 reads only psi (their ctx is zero)."""
  n3, n4 = 10 * M // 3, 8 * M // 3
  tail = n3 * n4 + n4 * 2 * M
  return 2 * M * n3 + tail if anchors else 12 * M * 2 * M + 4 * M * n3 + tail


def _pass_rates(m, y_hat, psi, reps=20):
  """CUDA-event time of each parameter pass over the batch, and its FP32 rate on _macs."""
  B, H, W, M = y_hat.shape
  res = {}
  for anchors in (True, False):
    fn = lambda: F.cb_params(m._packed, y_hat, psi, anchors, m.num_scales)
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
    ms = float(np.median(ts))
    n = F.cb_counts(H, W)[0 if anchors else 1] * B
    flops = 2.0 * _macs(M, anchors) * n
    res["anchors" if anchors else "non_anchors"] = {
        "positions": n, "ms": ms, "tflops": flops / ms / 1e9, "fraction_of_67_tflops": flops / ms / 1e9 / 67.0}
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
    raise SystemExit("checkerboard_bench needs a CUDA device")
  imgs = _images(a.images)
  ms = {}
  for name, cls in (("mbt2018", models.MBT2018Model), ("checkerboard", models.CheckerboardModel)):
    torch.manual_seed(0)
    ms[name] = cls(num_filters=a.num_filters, latent_depth=a.latent_depth).build("cuda", patch=(64, 64)).fix_tables()
  res = {"card_before": _card(), "images": f"{a.images} Kodak-shaped (512x768 / 768x512), synthetic, random weights",
         "num_filters": a.num_filters, "latent_depth": a.latent_depth, "reps": a.reps}

  with torch.no_grad():
    inputs = {}
    for name, m in ms.items():
      ys, psis = [], []
      for x in imgs[0::2]:
        y = m.analysis_transform(x[None].float())
        ys.append(y)
        psis.append(m._psi(m.side_entropy_model.quantize(m.hyper_analysis_transform(y)), tuple(y.shape[1:-1])))
      y, psi = torch.cat(ys).contiguous(), torch.cat(psis)
      strings = m._encode_latents(y, psi)[0]
      items = m.compress_images(imgs)
      inputs[name] = (y, psi, strings, items)
    calls = {
        "latent_encode_12": lambda m, i: m._encode_latents(i[0], i[1])[0],
        "latent_decode_12": lambda m, i: m._decode_latents(i[2], i[1]),
        "compress_images_24": lambda m, i: m.compress_images(imgs),
        "decompress_images_24": lambda m, i: m.decompress_images(i[3]),
        "compress_1": lambda m, i: m.compress(imgs[0]),
        "decompress_1": lambda m, i: m.decompress(*i[3][0]),
    }
    times = {n: {c: [] for c in calls} for n in ms}
    launches = {n: {} for n in ms}
    outs = {n: {} for n in ms}
    for name, m in ms.items():  # warm-up of every call
      for c, fn in calls.items():
        fn(m, inputs[name])
    for _ in range(a.reps):
      for c, fn in calls.items():
        for name, m in ms.items():  # the two models alternate call by call
          t, l, out = _once(lambda: fn(m, inputs[name]))
          times[name][c].append(t)
          launches[name][c] = l
          outs[name][c] = out
    for name in ms:
      y_dec = outs[name]["latent_decode_12"]
      assert torch.equal(y_dec, ms[name]._encode_latents(inputs[name][0], inputs[name][1])[1]), name
      res[name] = {c: {"ms": float(np.median(ts)), "all_ms": ts, "launches": launches[name][c]}
                   for c, ts in times[name].items()}
      assert all(o.shape == x.shape for o, x in zip(outs[name]["decompress_images_24"], imgs))
    cb = ms["checkerboard"]
    res["checkerboard"]["param_passes_12"] = _pass_rates(cb, outs["checkerboard"]["latent_decode_12"],
                                                         inputs["checkerboard"][1])
    y1, p1 = inputs["checkerboard"][0][:1], inputs["checkerboard"][1][:1]
    res["checkerboard"]["param_passes_1"] = _pass_rates(cb, torch.round(y1), p1)
    res["decompress_1_speedup"] = res["mbt2018"]["decompress_1"]["ms"] / res["checkerboard"]["decompress_1"]["ms"]
  res["card_after"] = _card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
