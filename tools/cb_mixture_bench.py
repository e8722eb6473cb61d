"""Times CheckerboardMixtureModel against MixtureHyperpriorModel and CheckerboardModel in one run, calls alternated
between the models: tools/multistage_bench.py's 24 Kodak-shaped images (12 of 512x768, 12 of 768x512, so 32 x 48 x
192 latents; random weights, synthetic content).  N = 192, M = 192, K = 3 Normal components for the mixture models.

  python tools/cb_mixture_bench.py [--reps 3] [--out FILE.json]

Per model: a one-image `decompress` at S = 1 and S = 16 substreams, and `compress_images` / `decompress_images` of
all 24 at S = 1, given per image, with the library launches of each call.  For the checkerboard mixture model also
each parameter pass alone on one image (CUDA events around `functional.cbm_params`).  Medians in ms; the card's
name, power limit, SM clock and clock-throttle reasons are read before and after in the same run.  Random weights
say nothing about rate, so the string sizes are reported only to show what was coded.  Prints one JSON object."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import functional as F, models  # noqa: E402
from tools.multistage_bench import _card, _images, _once  # noqa: E402

N, M, K = 192, 192, 3
BUILDERS = {
    "checkerboard_mixture": lambda S: models.CheckerboardMixtureModel(num_filters=N, latent_depth=M, num_components=K,
                                                                      substreams=S),
    "mixture_hyperprior": lambda S: models.MixtureHyperpriorModel(num_filters=N, latent_depth=M, num_components=K,
                                                                  substreams=S),
    "checkerboard": lambda S: models.CheckerboardModel(num_filters=N, latent_depth=M, substreams=S),
}


def _pass_times(m, x, reps=20):
  """CUDA-event time of the checkerboard mixture model's two parameter passes on one image."""
  with torch.no_grad():
    y = m.analysis_transform(x[None].float())
    z = m.hyper_analysis_transform(y)
    psi = m._psi(m.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
  y_hat = torch.round(y).contiguous()
  res = {}
  for name, anchors in (("anchors", True), ("non_anchors", False)):
    fn = lambda: F.cbm_params(m._packed, K, y_hat, psi, anchors)
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
    res[name + "_ms"] = float(np.median(ts))
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--out")
  a = ap.parse_args()
  res = {"card_before": _card(), "N": N, "M": M, "K": K, "images": "12 x 512x768 + 12 x 768x512"}
  images = _images(24)
  built = {}
  for name, make in BUILDERS.items():
    torch.manual_seed(0)
    base = make(1).build("cuda", patch=(64, 64)).fix_tables()
    for S in (1, 16):
      m = base if S == 1 else make(S).build("cuda", patch=(64, 64))
      if S > 1:
        m.load_state_dict(base.state_dict(), strict=False)
        m.fix_tables()
      built[(name, S)] = (m, m.compress(images[0]))
  times = {key: [] for key in built}
  lists = {name: ([], []) for name in BUILDERS}
  launches = {}
  items = {name: built[(name, 1)][0].compress_images(images) for name in BUILDERS}  # (warm-up)
  for name in BUILDERS:
    built[(name, 1)][0].decompress_images(items[name])
  for _ in range(a.reps):
    for (name, S), (m, item) in built.items():  # alternated between the models
      t, n, _ = _once(lambda: m.decompress(*item))
      times[(name, S)].append(t)
      launches[f"{name}_S{S}_decompress"] = n
    for name in BUILDERS:
      m = built[(name, 1)][0]
      t, n, items[name] = _once(lambda: m.compress_images(images))
      lists[name][0].append(t / len(images))
      launches[f"{name}_compress_images"] = n
      t, n, _ = _once(lambda: m.decompress_images(items[name]))
      lists[name][1].append(t / len(images))
      launches[f"{name}_decompress_images"] = n
  for (name, S), ts in times.items():
    res[f"{name}_S{S}_one_image_decompress_ms"] = float(np.median(ts))
  for name, (c, d) in lists.items():
    res[f"{name}_compress_images_ms_per_image"] = float(np.median(c))
    res[f"{name}_decompress_images_ms_per_image"] = float(np.median(d))
    res[f"{name}_y_bytes_per_image"] = float(np.mean([len(it[0].tolist()[0]) for it in items[name]]))
  res["launches"] = launches
  res["checkerboard_mixture_passes"] = _pass_times(built[("checkerboard_mixture", 1)][0], images[0])
  res["card_after"] = _card()
  out = json.dumps(res)
  if a.out:
    with open(a.out, "w") as f:
      f.write(out + "\n")
  print(out)


if __name__ == "__main__":
  main()
