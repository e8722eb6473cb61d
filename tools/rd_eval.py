"""Rate-distortion evaluation of a model on a list of images, printed as the reference's results files are written
(results/image_compression/<dataset>/<metric>_sRGB_<space>/*.txt): one block per metric and colour space of
`bpp, value` rows.  Here a block has one row, the dataset mean at the model's one lambda (`models.mean_metrics` over
`Model.evaluate_images`).

The model has random weights (seeded) unless --state-dict loads a torch state_dict saved from the same class and
arguments.  The images are the PNGs of --images DIR (read with PIL, converted to RGB) or, with --synthetic kodak,
24 seeded smooth-plus-noise images of Kodak's shapes, 12 of 512x768 and 12 of 768x512; with --synthetic mixed, 24
such images of seeded, all different shapes (sides multiples of 16 from 256 to 1024), as in a dataset of many image
sizes.  The context models (mbt2018, checkerboard, space_channel, multistage, space_channel_multistage,
checkerboard_mixture) code such a list with one ragged launch sequence.
--substreams S writes every string as S independently decodable streams (DESIGN §3.14); bpp includes their headers.
--tiles T (mbt2018 only) writes every y string as T column tiles, coded as a wavefront over many SMs (DESIGN §3.15).

--time also measures, alternating the two sides of each pair --reps times after --warmup calls (median ms, CUDA
events around a synchronised call):
  metrics   image.metrics_ragged (RGB) on the list of (original, reconstruction) pairs, against a loop of per-image
            image.psnr + image.ssim_multiscale calls;
  evaluate  Model.evaluate_images on the list, against a loop of Model.evaluate;
with the library's kernel launches and all CUDA kernels (torch.profiler, one call in a separate pass) of one call of
each side, and the card's name, power limit and SM clock read in the same run.

  python tools/rd_eval.py --synthetic kodak|mixed [--model bmshj2018] [--num-filters 192] [--state-dict F]
                          [--substreams S] [--tiles T] [--time]
  python tools/rd_eval.py --images DIR ...
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from compression_b200 import _lib, image, models  # noqa: E402

BLOCKS = [  # (metric, colour space, key in the evaluate_images dicts)
    ("PSNR", "RGB", "psnr"), ("PSNR", "Y", "psnr_y"), ("PSNR", "YCbCr-6:1:1", "psnr_ycbcr"),
    ("MS-SSIM", "RGB", "msssim"), ("MS-SSIM", "Y", "msssim_y"), ("MS-SSIM", "YCbCr-6:1:1", "msssim_ycbcr"),
]


MODELS = {"bls2017": models.BLS2017Model, "bmshj2018": models.BMSHJ2018Model, "ms2020": models.MS2020Model,
          "mbt2018": models.MBT2018Model, "checkerboard": models.CheckerboardModel,
          "space_channel": models.SpaceChannelModel, "multistage": models.MultistageModel,
          "space_channel_multistage": models.SpaceChannelMultistageModel,
          "checkerboard_mixture": models.CheckerboardMixtureModel}


def mixed_shapes(seed, n=24):
  """n seeded image shapes (h, w), sides multiples of 16 from 256 to 1024, no two alike (nor their latents)."""
  rng = np.random.default_rng(seed)
  sides = np.arange(256, 1025, 16)
  out = []
  while len(out) < n:
    s = (int(rng.choice(sides)), int(rng.choice(sides)))
    if s not in out:
      out.append(s)
  return out


def synthetic(seed, shapes=None):
  """Seeded smooth-plus-noise images of `shapes` (default: Kodak's, 12 of 512x768 and 12 of 768x512)."""
  g = torch.Generator().manual_seed(seed)
  out = []
  for h, w in shapes or [(512, 768)] * 12 + [(768, 512)] * 12:
    yy = torch.linspace(0, 1, h)[:, None, None]
    xx = torch.linspace(0, 1, w)[None, :, None]
    f = 2 + 6 * torch.rand(1, 1, 3, generator=g)
    a = 0.5 + 0.35 * torch.sin(f * xx + 4.0 * yy + 6.28 * torch.rand(1, 1, 3, generator=g)) * torch.cos(3.0 * yy - f * xx)
    a = (a + 0.06 * torch.randn(h, w, 3, generator=g)).clamp(0, 1)
    out.append(torch.round(a * 255).to(torch.uint8))
  return out


def png_images(directory):
  from PIL import Image
  names = sorted(n for n in os.listdir(directory) if n.lower().endswith(".png"))
  if not names:
    raise SystemExit(f"no PNG files in {directory}")
  return [torch.from_numpy(np.asarray(Image.open(os.path.join(directory, n)).convert("RGB")).copy()) for n in names]


def make_model(name, num_filters, state_dict, seed, substreams=1, tiles=1):
  torch.manual_seed(seed)
  kw = {} if num_filters is None else {"num_filters": num_filters}
  if substreams != 1:
    kw["substreams"] = substreams
  if tiles != 1:
    if name != "mbt2018":
      raise SystemExit(f"--tiles is for mbt2018 only, not {name}")
    kw["tiles"] = tiles
  m = MODELS[name](**kw)
  m.build("cuda")
  if state_dict:
    m.load_state_dict(torch.load(state_dict, map_location="cuda"))
  return m.fix_tables()


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  return dict(zip(("name", "power_limit", "sm_clock", "max_sm_clock"), (s.strip() for s in q.split(","))))


def timed_pair(fa, fb, reps, warmup):
  """Median ms of fa and of fb, run alternately."""
  for _ in range(warmup):
    fa()
    fb()
  ta, tb = [], []
  for _ in range(reps):
    for fn, t in ((fa, ta), (fb, tb)):
      torch.cuda.synchronize()
      s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      s.record()
      fn()
      e.record()
      e.synchronize()
      t.append(s.elapsed_time(e))
  return statistics.median(ta), statistics.median(tb)


def launches(fn):
  """(library kernel launches, all CUDA kernels) of one call."""
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  n1 = _lib.launch_count()
  kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and
                not e.name.startswith(("Memcpy", "Memset")))
  return n1 - n0, kernels


def parser():
  p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  src = p.add_mutually_exclusive_group(required=True)
  src.add_argument("--images", help="directory of PNG images")
  src.add_argument("--synthetic", choices=["kodak", "mixed"], help="seeded synthetic images of a dataset's shapes")
  p.add_argument("--model", choices=list(MODELS), default="bmshj2018")
  p.add_argument("--num-filters", type=int, default=None, help="the model's num_filters (default: its own)")
  p.add_argument("--state-dict", default=None, help="torch state_dict of the model to load")
  p.add_argument("--seed", type=int, default=0)
  p.add_argument("--substreams", type=int, default=1,
                 help="independently decodable streams per string (DESIGN §3.14; not mbt2018)")
  p.add_argument("--tiles", type=int, default=1, help="column tiles per y string (DESIGN §3.15; mbt2018 only)")
  p.add_argument("--time", action="store_true")
  p.add_argument("--reps", type=int, default=10)
  p.add_argument("--warmup", type=int, default=2)
  p.add_argument("--out", default=None, help="also write the results as JSON to this file")
  return p


def main():
  args = parser().parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("rd_eval.py needs a CUDA device")

  if args.synthetic:
    images = synthetic(args.seed, mixed_shapes(args.seed) if args.synthetic == "mixed" else None)
  else:
    images = png_images(args.images)
  model = make_model(args.model, args.num_filters, args.state_dict, args.seed, args.substreams, args.tiles)
  per_image = model.evaluate_images(images)
  mean = models.mean_metrics(per_image)
  dataset = args.synthetic or os.path.basename(os.path.normpath(args.images))
  weights = "state_dict " + args.state_dict if args.state_dict else f"random weights, seed {args.seed}"
  for metric, space, key in BLOCKS:
    print(f"# {metric}/sRGB/{space} of {args.model} ({weights}) on {dataset}, {len(images)} images.")
    print("# The first column contains bits per pixel (bpp) values; means over the images at one lambda.")
    print(f"{mean['bpp']:.6f}, {mean[key]:.6f}")
    print()
  result = {"model": args.model, "dataset": dataset, "n_images": len(images), "substreams": args.substreams,
            "tiles": args.tiles, "mean": mean}

  if args.time:
    gpu = card()
    dev = torch.device("cuda")
    xs = [x.to(dev, torch.float32) for x in images]
    x_hats = [x.to(torch.float32) for x in model.decompress_images(model.compress_images(images))]

    def ragged():
      image.metrics_ragged(xs, x_hats, 255)

    def loop():
      for x, x_hat in zip(xs, x_hats):
        image.psnr(x, x_hat, 255)
        image.ssim_multiscale(x, x_hat, 255)

    def eval_ragged():
      model.evaluate_images(images)

    def eval_loop():
      for x in images:
        model.evaluate(x)

    t_r, t_l = timed_pair(ragged, loop, args.reps, args.warmup)
    e_r, e_l = timed_pair(eval_ragged, eval_loop, max(3, args.reps // 3), 1)
    result["timing"] = {
        "gpu": gpu,
        "metrics_ragged_ms": t_r, "metrics_loop_ms": t_l,
        "metrics_ragged_launches": launches(ragged), "metrics_loop_launches": launches(loop),
        "evaluate_images_ms": e_r, "evaluate_loop_ms": e_l,
        "evaluate_images_launches": launches(eval_ragged), "evaluate_loop_launches": launches(eval_loop),
        "gpu_after": card(),
        "note": "launches are (library kernels, all CUDA kernels) of one call",
    }
    print(json.dumps(result["timing"]))
  if args.out:
    with open(args.out, "w") as f:
      json.dump(result, f, indent=1)


if __name__ == "__main__":
  main()
