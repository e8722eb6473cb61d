"""Ragged batches on the H100: one range-coder launch over a mixed-size image set against a per-image loop.

Workload: cfg2's committed tables (tests/golden/cfg2_tables.npz: 128 channel rows, precision 12, overflow on) on
Laplace(0, s_c) latents synthesised as bench.py does, for a seeded mix of image sizes (Kodak's two orientations,
1280x720, 1024x768 and 2048x1360; 256 images by default), latents [ceil(H/16), ceil(W/16), 128] per image.
For encode and decode it reports
  (a) one ragged call (functional.compress_ragged / decode_ragged),
  (b) the per-image loop through the existing single-item path (compress_f32 / decode_channel_f32),
  (c) the uniform cfg2 batch (256 streams x 32 768 symbols),
and the bound the ragged call cannot beat: the longest stream's symbols x the coder's cycles per symbol (measured
here, from the uniform batch's kernel time under torch.profiler) / the SM clock.  The card's name, power limit and
SM clock are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/ragged_bench.py [--images 256] [--seed 0] [--out DIR]
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

from compression_b200 import functional as F  # noqa: E402
from compression_b200 import gen_ops  # noqa: E402

SIZES = [(768, 512), (512, 768), (1280, 720), (1024, 768), (2048, 1360)]
C = 128


def card():
  q = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
    return dict(zip(q.split(","), [c.strip() for c in out.split(",")]))
  except Exception as e:  # pylint:disable=broad-except
    return {"name": torch.cuda.get_device_name(), "error": str(e)}


def latents(shapes, seed, dev):
  g = torch.Generator(device=dev).manual_seed(seed)
  scales = torch.exp(torch.linspace(np.log(0.3), np.log(8.0), C, device=dev))
  out = []
  for h, w in shapes:
    u = torch.rand(h, w, C, generator=g, device=dev) - 0.5
    out.append((-scales * torch.sign(u) * torch.log1p(-2 * u.abs()).clamp_min(-17.0)).contiguous())
  return out


def timed(fn, reps):
  """Median wall time of `fn` (each call ends in a device synchronisation), after one warm-up call."""
  out = fn()
  torch.cuda.synchronize()
  ts = []
  for _ in range(reps):
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    ts.append(time.perf_counter() - t0)
  return sorted(ts)[len(ts) // 2] * 1e3, out


def kernel_ms(fn, name, reps=5):
  """Mean device time of the kernels whose name contains `name`, per call of `fn` (torch.profiler)."""
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
  total = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
  return total / reps / 1e3


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--images", type=int, default=256)
  ap.add_argument("--seed", type=int, default=0)
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("ragged_bench needs a CUDA device")
  dev = torch.device("cuda")
  info_before = card()
  g = np.load(os.path.join(ROOT, "tests", "golden", "cfg2_tables.npz"))
  lookup = g["lookup"]
  coff = torch.from_numpy(g["cdf_offset"].astype(np.int32)).to(dev)
  qoff = torch.from_numpy(g["quantization_offset"]).to(dev) if bool(g["has_qoff"]) else None

  rng = np.random.default_rng(args.seed)
  sizes = [SIZES[i] for i in rng.integers(0, len(SIZES), args.images)]
  shapes = [(-(-h // 16), -(-w // 16)) for h, w in sizes]
  ys = latents(shapes, args.seed + 2, dev)
  lens = [y.numel() for y in ys]
  flat = torch.cat([y.reshape(-1) for y in ys])
  res = {"workload": f"{args.images} images, sizes drawn (seed {args.seed}) from {SIZES}; cfg2 tables; latents "
                     "[ceil(H/16), ceil(W/16), 128] fp32",
         "symbols": int(sum(lens)), "longest_stream": int(max(lens)), "shortest_stream": int(min(lens))}

  # ---- encode
  enc_a, strings = timed(lambda: F.compress_ragged(lookup, lens, flat, qoff, coff), args.reps)
  ragged_l = strings.tolist()

  def loop_encode():
    return [F.compress_f32((1,), lookup, y[None], qoff, coff) for y in ys]
  enc_b, per_image = timed(loop_encode, 1)
  res["strings_identical_to_per_image_path"] = [s.tolist()[0] for s in per_image] == ragged_l
  del per_image

  uni = latents([(16, 16)] * 256, args.seed + 3, dev)
  yu = torch.stack(uni)
  enc_c, _ = timed(lambda: F.compress_f32((256,), lookup, yu, qoff, coff), max(args.reps, 5))
  enc_kern = kernel_ms(lambda: F.compress_f32((256,), lookup, yu, qoff, coff), "encode_kernel")

  # ---- decode
  packed = gen_ops.Strings.from_bytes(ragged_l, (len(ragged_l),))

  def ragged_decode():
    h = gen_ops.create_range_decoder(packed, lookup)
    out = F.decode_ragged(h, lens, quant_offset=qoff, cdf_offset=coff)
    assert bool(gen_ops.entropy_decode_finalize(h).all())
    return out
  dec_a, dec = timed(ragged_decode, args.reps)
  singles = [gen_ops.Strings.from_bytes([s], (1,)) for s in ragged_l]

  def loop_decode():
    outs = []
    for s, y in zip(singles, ys):
      h = gen_ops.create_range_decoder(s, lookup)
      outs.append(F.decode_channel_f32(h, (1,) + tuple(y.shape), qoff, coff))
      gen_ops.entropy_decode_finalize(h)
    return outs
  dec_b, outs = timed(loop_decode, 1)
  res["decode_identical_to_per_image_path"] = bool(torch.equal(dec, torch.cat([o.reshape(-1) for o in outs])))
  del outs
  su = F.compress_f32((256,), lookup, yu, qoff, coff)

  def uniform_decode():
    h = gen_ops.create_range_decoder(su, lookup)
    out = F.decode_channel_f32(h, tuple(yu.shape), qoff, coff)
    gen_ops.entropy_decode_finalize(h)
    return out
  dec_c, _ = timed(uniform_decode, max(args.reps, 5))
  dec_kern = kernel_ms(uniform_decode, "decode_kernel")

  info_after = card()
  clock_mhz = float(str(info_after.get("clocks.sm", "1980")).split()[0] or 1980)
  n_uni = 16 * 16 * C
  cps_enc = enc_kern * 1e-3 * clock_mhz * 1e6 / n_uni
  cps_dec = dec_kern * 1e-3 * clock_mhz * 1e6 / n_uni
  res.update({
      "card_before": info_before, "card_after": info_after,
      "encode_ms": {"a_ragged_call": enc_a, "b_per_image_loop": enc_b, "c_uniform_cfg2_batch_256x32768": enc_c,
                    "bound_longest_stream": max(lens) * cps_enc / (clock_mhz * 1e3)},
      "decode_ms": {"a_ragged_call": dec_a, "b_per_image_loop": dec_b, "c_uniform_cfg2_batch_256x32768": dec_c,
                    "bound_longest_stream": max(lens) * cps_dec / (clock_mhz * 1e3)},
      "cycles_per_symbol": {"encode_kernel": cps_enc, "decode_kernel": cps_dec,
                            "source": f"uniform cfg2 kernel time (torch.profiler) x {clock_mhz:.0f} MHz / {n_uni}"},
      "speedup_ragged_vs_loop": {"encode": enc_b / enc_a, "decode": dec_b / dec_a},
  })
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "ragged_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
