"""Times SpaceChannelMultistageModel against SpaceChannelModel and MultistageModel in one run, calls alternated
between the models: tools/multistage_bench.py's 24 Kodak-shaped images (12 of 512x768, 12 of 768x512; random weights,
synthetic content).  N = 192; M = 320 with groups (16, 16, 32, 64, 192) for the two space-channel models, and M = 192
for MultistageModel (its depth must be a multiple of 6).

  python tools/space_channel_multistage_bench.py [--reps 3] [--out FILE.json]

Per model: a one-image `compress` / `decompress`, `compress_images` / `decompress_images` of all 24 (also given per
image), and the library launches of each call.  For the space-channel multistage model also each group's and stage's
parameter pass alone on one image (CUDA events around `functional.mscc_params`).  Medians in ms; the card's name,
power limit, SM clock and clock-throttle reasons are read before and after in the same run.  Prints one JSON
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
from tools.multistage_bench import _card, _images, _once  # noqa: E402


def _stage_times(m, y_hat, psi, reps=20):
  """CUDA-event time of each group's and stage's parameter pass (the channel context computed beforehand)."""
  res = {}
  for k, (o, c) in enumerate(m.spans):
    ch = m._channel_context(k, y_hat) if k else None
    for s in range(4):
      fn = lambda: F.mscc_params(m._packed[k], (o, c), y_hat, psi, ch, s, m.num_scales)
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
      res[f"group_{k}_stage_{s}"] = {"channels": c, "positions": F.msc_counts(*y_hat.shape[1:3])[s] * y_hat.shape[0],
                                     "ms": float(np.median(ts))}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--latent-depth", type=int, default=320)
  ap.add_argument("--multistage-depth", type=int, default=192)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--images", type=int, default=24)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("space_channel_multistage_bench needs a CUDA device")
  imgs = _images(a.images)
  ms = {}
  for name, cls, depth in (("space_channel", models.SpaceChannelModel, a.latent_depth),
                           ("space_channel_multistage", models.SpaceChannelMultistageModel, a.latent_depth),
                           ("multistage", models.MultistageModel, a.multistage_depth)):
    torch.manual_seed(0)
    ms[name] = cls(num_filters=a.num_filters, latent_depth=depth).build("cuda", patch=(64, 64)).fix_tables()
  res = {"card_before": _card(), "images": f"{a.images} Kodak-shaped (512x768 / 768x512), synthetic, random weights",
         "num_filters": a.num_filters, "latent_depth": a.latent_depth, "groups": ms["space_channel"].groups,
         "multistage_depth": a.multistage_depth, "reps": a.reps}

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
    m = ms["space_channel_multistage"]
    y = m.analysis_transform(imgs[0][None].float())
    psi = m._psi(m.side_entropy_model.quantize(m.hyper_analysis_transform(y)), tuple(y.shape[1:-1]))
    res["space_channel_multistage"]["param_passes_1"] = _stage_times(m, torch.round(y).contiguous(), psi)
  res["card_after"] = _card()
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
