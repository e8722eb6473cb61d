"""MS2020 over a list of images on the H100: the per-image compress / decompress loop against compress_images /
decompress_images, which code every slice of all images in one range-coder launch and take the encoder's slice
reconstructions from the encode itself instead of decoding them.

Workload: the default MS2020Model (192 filters, 320 latent channels, 10 slices) with randomly initialised weights
and fix_tables(), on 24 seeded synthetic uint8 images: 12 of 512x768 and 12 of 768x512 (H x W; Kodak's two
orientations).  Untrained weights give rates unlike a trained model's, and the decode time depends on the rate, so
the bits per symbol are reported beside the times.  For compress and decompress it reports
  - the median synchronised wall time of the per-image loop and of the list call, and whether their outputs are
    identical: the strings, the decoded latents handed to the synthesis transform, and the uint8 images (the
    synthesis transform's own run-to-run repeatability is reported beside them),
  - the range coder's kernel time per call (torch.profiler, in a separate run) and its share of that wall time,
  - the encode_kernel / decode_kernel launches per call (from the same profile),
and the card's name and power limit, read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/ms2020_bench.py [--reps 3] [--seed 0] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from compression_b200 import models  # noqa: E402

SIZES = [(512, 768)] * 12 + [(768, 512)] * 12
CODER_KERNELS = ("encode_kernel", "enc_offsets_kernel", "enc_write_kernel", "enc_init_state_kernel",
                 "decode_kernel", "dec_init_state_kernel", "dec_finalize_kernel")


def card():
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
  except Exception as e:  # pylint:disable=broad-except
    return {"name": torch.cuda.get_device_name(), "error": str(e)}


def timed(fn, reps):
  """Median wall time of `fn` ending in a device synchronisation, after one warm-up call."""
  out = fn()
  torch.cuda.synchronize()
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    ts.append(time.perf_counter() - t0)
  return sorted(ts)[len(ts) // 2] * 1e3, out


def coder_profile(fn):
  """Device time of the range coder's kernels in one call of `fn`, and how many encode_kernel / decode_kernel
  launches it made (torch.profiler, a run of its own)."""
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  ev = [e for e in prof.key_averages() if any(k in e.key for k in CODER_KERNELS)]
  return {"coder_kernel_ms": sum(e.device_time_total for e in ev) / 1e3,
          "encode_kernel_launches": sum(e.count for e in ev if "encode_kernel" in e.key),
          "decode_kernel_launches": sum(e.count for e in ev if "decode_kernel" in e.key)}


def synthesis_inputs(m, fn):
  """The latents `fn` hands to the synthesis transform, in order."""
  got, orig = [], m.synthesis_transform.forward
  m.synthesis_transform.forward = lambda x: (got.append(x.clone()), orig(x))[1]
  try:
    fn()
  finally:
    del m.synthesis_transform.forward
  return got


def same_item(a, b):
  if len(a) != len(b):
    return False
  for u, v in zip(a, b):
    if isinstance(u, torch.Tensor):
      if not torch.equal(u, v):
        return False
    elif u.shape != v.shape or u.tolist() != v.tolist():
      return False
  return True


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--seed", type=int, default=0)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("ms2020_bench needs a CUDA device")
  info_before = card()
  torch.manual_seed(args.seed)
  m = models.MS2020Model().build("cuda", patch=(64, 64)).fix_tables()
  g = torch.Generator().manual_seed(args.seed + 1)
  images = [torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).cuda() for h, w in SIZES]

  enc_loop, items_loop = timed(lambda: [m.compress(x) for x in images], args.reps)
  enc_list, items_list = timed(lambda: m.compress_images(images), args.reps)
  dec_loop, x_loop = timed(lambda: [m.decompress(*it) for it in items_loop], args.reps)
  dec_list, x_list = timed(lambda: m.decompress_images(items_list), args.reps)
  strings_identical = all(same_item(a, b) for a, b in zip(items_loop, items_list))
  images_identical = all(torch.equal(a, b) for a, b in zip(x_loop, x_list))
  # the decoded latents are the coder's output; the uint8 images also go through the synthesis transform, which is
  # checked for run-to-run repeatability on one input
  lat_loop = synthesis_inputs(m, lambda: [m.decompress(*it) for it in items_loop])
  lat_list = synthesis_inputs(m, lambda: m.decompress_images(items_list))
  latents_identical = len(lat_loop) == len(lat_list) and all(torch.equal(a, b) for a, b in zip(lat_loop, lat_list))
  synthesis_repeatable = torch.equal(m.synthesis_transform(lat_loop[0]), m.synthesis_transform(lat_loop[0]))

  n_y = sum(int(it[1][0]) * int(it[1][1]) for it in items_list) * 320
  n_z = sum(int(it[2][0]) * int(it[2][1]) for it in items_list) * 192
  n_bytes = sum(len(s.tolist()[0]) for it in items_list for s in it[3:])

  res = {
      "workload": f"default MS2020Model (random init, seed {args.seed}), {len(SIZES)} synthetic uint8 images: "
                  "12 of 512x768 and 12 of 768x512 (H x W)",
      "symbols": {"y": n_y, "z": n_z}, "bits_per_symbol": 8.0 * n_bytes / (n_y + n_z),
      "outputs_identical": {"strings": strings_identical, "decoded_latents": latents_identical,
                            "reconstructions": images_identical,
                            "synthesis_transform_repeatable_on_one_input": synthesis_repeatable},
      "compress_ms": {"per_image_loop": enc_loop, "compress_images": enc_list, "speedup": enc_loop / enc_list},
      "decompress_ms": {"per_image_loop": dec_loop, "decompress_images": dec_list, "speedup": dec_loop / dec_list},
  }
  runs = {"compress_per_image_loop": (lambda: [m.compress(x) for x in images], enc_loop),
          "compress_images": (lambda: m.compress_images(images), enc_list),
          "decompress_per_image_loop": (lambda: [m.decompress(*it) for it in items_loop], dec_loop),
          "decompress_images": (lambda: m.decompress_images(items_list), dec_list)}
  res["coder"] = {}
  for name, (fn, wall_ms) in runs.items():
    p = coder_profile(fn)
    p["share_of_wall"] = p["coder_kernel_ms"] / wall_ms
    res["coder"][name] = p
  res["card_before"], res["card_after"] = info_before, card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "ms2020_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
