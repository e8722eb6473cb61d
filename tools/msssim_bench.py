"""MS-SSIM on the fused kernels (compression_b200.image) against the same algorithm as an eager float32 torch graph on
the GPU (oracle/ssim_oracle.py run in float32 on CUDA), on three workloads:

  train  ssim_multiscale forward + backward on [8, 256, 256, 3] float32 in [0, 255] (a training batch's distortion)
  eval   ssim_multiscale forward on 24 Kodak-sized images, 12 of 512x768 and 12 of 768x512, one call per image as
         _Model.evaluate makes them
  step   one BLS2017Model training step (num_filters 128, batch 8, 256x256) with the loss bpp + lmbda (1 - MS-SSIM)

For each: median ms over --reps timed calls (CUDA events, after --warmup calls), the peak of allocated memory during
one call above what was allocated before it, and the CUDA kernels one call launches (counted with torch.profiler in a
separate pass).  The card's name and power limit are read in the same run.  Prints one JSON line per workload.

  python tools/msssim_bench.py [--reps 30] [--warmup 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from compression_b200 import image, models  # noqa: E402
from oracle import ssim_oracle as O  # noqa: E402


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True, check=True).stdout.strip().splitlines()[0]
  name, limit = [s.strip() for s in q.split(",")]
  return name, limit


def timed(fn, reps, warmup):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    times.append(s.elapsed_time(e))
  return statistics.median(times)


def peak_bytes(fn):
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  fn()
  torch.cuda.synchronize()
  return torch.cuda.max_memory_allocated() - base


def kernels(fn):
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    torch.cuda.synchronize()
  n = 0
  for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower() and \
        "memset" not in e.name.lower():
      n += 1
  return n


def measure(fn, reps, warmup):
  ms = timed(fn, reps, warmup)
  return {"median_ms": round(ms, 4), "peak_mib": round(peak_bytes(fn) / 2**20, 2), "kernels_per_call": kernels(fn)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  assert torch.cuda.is_available(), "msssim_bench needs a GPU"
  dev = torch.device("cuda")
  name, limit = card()
  g = torch.Generator(device=dev).manual_seed(0)
  results = []

  def report(workload, fused, graph):
    r = {"workload": workload, "card": name, "power_limit": limit, "fused": fused, "torch_graph": graph,
         "speedup": round(graph["median_ms"] / fused["median_ms"], 2)}
    print(json.dumps(r), flush=True)
    results.append(r)

  # -- train: forward + backward of the metric alone
  x = torch.rand(8, 256, 256, 3, device=dev, generator=g) * 255
  xh0 = (x + 8 * torch.randn(x.shape, device=dev, generator=g)).clamp(0, 255)

  def train(ms):
    xh = xh0.clone().requires_grad_()
    ms(x, xh).sum().backward()

  ok = (image.ssim_multiscale(x, xh0, 255).double() - O.ssim_multiscale(x, xh0, 255, dtype=torch.float32).double())
  assert float(ok.abs().max()) < 1e-4, float(ok.abs().max())
  report("train [8,256,256,3] fwd+bwd",
         measure(lambda: train(lambda a, b: image.ssim_multiscale(a, b, 255)), args.reps, args.warmup),
         measure(lambda: train(lambda a, b: O.ssim_multiscale(a, b, 255, dtype=torch.float32)), args.reps,
                 args.warmup))

  # -- eval: 24 Kodak-sized images, forward only, one call per image
  imgs = []
  for i in range(24):
    h, w = (512, 768) if i % 2 == 0 else (768, 512)
    a = torch.rand(h, w, 3, device=dev, generator=g) * 255
    imgs.append((a.round(), (a + 4 * torch.randn(a.shape, device=dev, generator=g)).clamp(0, 255).round()))

  def evaluate(ms):
    with torch.no_grad():
      for a, b in imgs:
        ms(a, b)

  report("eval 24 x 512x768/768x512 fwd",
         measure(lambda: evaluate(lambda a, b: image.ssim_multiscale(a, b, 255)), args.reps, args.warmup),
         measure(lambda: evaluate(lambda a, b: O.ssim_multiscale(a, b, 255, dtype=torch.float32)), args.reps,
                 args.warmup))

  # -- one BLS2017 training step with an MS-SSIM loss
  torch.manual_seed(0)
  m = models.BLS2017Model(num_filters=128).build("cuda")
  opt = torch.optim.Adam(m.parameters(), lr=1e-5)
  xb = (torch.rand(8, 256, 256, 3, device=dev, generator=g) * 255).round()

  def step(ms):
    _, bpp, _ = m(xb)
    loss = bpp + 100.0 * (1 - ms(xb, m._last_x_hat).mean())
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()

  report("BLS2017 step b8 256x256 MS-SSIM loss",
         measure(lambda: step(lambda a, b: image.ssim_multiscale(a, b, 255)), max(5, args.reps // 3), args.warmup),
         measure(lambda: step(lambda a, b: O.ssim_multiscale(a, b, 255, dtype=torch.float32)),
                 max(5, args.reps // 3), args.warmup))

  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
      json.dump(results, f, indent=1)


if __name__ == "__main__":
  main()
