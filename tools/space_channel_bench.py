"""Times SpaceChannelModel against CheckerboardModel and MS2020Model in one run, calls alternated between the models:
24 Kodak-shaped images (12 of 512x768, 12 of 768x512; random weights, synthetic content), N = 192, M = 320 for the
space-channel and MS2020 models (groups 16, 16, 32, 64, 192) and M = 192 for the checkerboard model.

  python tools/space_channel_bench.py [--reps 3] [--out FILE.json]

Per model: a one-image `compress` / `decompress`, `compress_images` / `decompress_images` of all 24, and the library
launches of each call.  For the space-channel model also each group's parameter passes alone (CUDA events around
`functional.scc_params` over the 12 latents of one shape) with their FP32 rate on the multiply-adds the layer shapes
give.  Medians in ms; the card's name, power limit and SM clock are read in the same run.  Prints one JSON
object."""
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


def _macs(M, span, anchors):
  """Multiply-adds per position of one pass of group span = (offset, c): at the anchors the kernel skips the layer-1
  slices that lie wholly inside the zero spatial context, so those are not counted."""
  c = span[1]
  lay = F.scc_layout(M, span)
  k1, n3, n4 = lay["K1"], lay["N3"], lay["N4"]
  tail = n3 * n4 + n4 * 2 * c
  if not anchors:
    return 12 * c * 2 * c + k1 * n3 + tail
  slices = [(s * k1 // 8, (s + 1) * k1 // 8) for s in range(8)]
  return sum(hi - lo for lo, hi in slices if lo < k1 - 2 * c) * n3 + tail


def _pass_rates(m, y_hat, psi, reps=20):
  """CUDA-event time of each group's parameter passes over the batch, and their FP32 rate on _macs."""
  B, H, W, M = y_hat.shape
  res = []
  for k, (o, c) in enumerate(m.spans):
    ch = m._channel_context(k, y_hat) if k else None
    row = {"group": k, "channels": c}
    for anchors in (True, False):
      fn = lambda: F.scc_params(m._packed[k], (o, c), y_hat, psi, ch, anchors, m.num_scales)
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
      flops = 2.0 * _macs(M, (o, c), anchors) * n
      row["anchors" if anchors else "non_anchors"] = {"positions": n, "ms": ms, "tflops": flops / ms / 1e9}
    res.append(row)
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--images", type=int, default=24)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("space_channel_bench needs a CUDA device")
  imgs = _images(a.images)
  ms = {}
  for name, make in (("space_channel", lambda: models.SpaceChannelModel(num_filters=a.num_filters)),
                     ("checkerboard", lambda: models.CheckerboardModel(num_filters=a.num_filters, latent_depth=192)),
                     ("ms2020", lambda: models.MS2020Model(num_filters=a.num_filters))):
    torch.manual_seed(0)
    ms[name] = make().build("cuda", patch=(64, 64)).fix_tables()
  res = {"card_before": _card(), "images": f"{a.images} Kodak-shaped (512x768 / 768x512), synthetic, random weights",
         "num_filters": a.num_filters, "reps": a.reps,
         "latent_depth": {"space_channel": 320, "checkerboard": 192, "ms2020": 320},
         "groups": list(ms["space_channel"].groups)}

  with torch.no_grad():
    items = {name: m.compress_images(imgs) for name, m in ms.items()}
    calls = {
        "compress_1": lambda m, it: m.compress(imgs[0]),
        "decompress_1": lambda m, it: m.decompress(*it[0]),
        "compress_images_24": lambda m, it: m.compress_images(imgs),
        "decompress_images_24": lambda m, it: m.decompress_images(it),
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
    for name in ms:
      res[name] = {c: {"ms": float(np.median(ts)), "all_ms": ts, "launches": launches[name][c]}
                   for c, ts in times[name].items()}
      assert all(o.shape == x.shape for o, x in zip(outs[name]["decompress_images_24"], imgs))
      assert [o[0].tolist() for o in outs[name]["compress_images_24"]] == [o[0].tolist() for o in items[name]]
    sc = ms["space_channel"]
    ys, psis = [], []
    for x in imgs[0::2]:
      y = sc.analysis_transform(x[None].float())
      ys.append(y)
      psis.append(sc._psi(sc.side_entropy_model.quantize(sc.hyper_analysis_transform(y)), tuple(y.shape[1:-1])))
    y, psi = torch.cat(ys).contiguous(), torch.cat(psis)
    y_hat = sc._encode_latents(y, psi)[1]
    res["space_channel"]["param_passes_12"] = _pass_rates(sc, y_hat, psi)
    res["space_channel"]["param_passes_1"] = _pass_rates(sc, y_hat[:1].contiguous(), psi[:1].contiguous())
  res["card_after"] = _card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
