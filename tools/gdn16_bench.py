"""Mixed-precision GDN at 128 and 192 channels on the H100: float32 activations, 16-bit activations on the native
kernels, and 16-bit activations on the conversion path (x.float(), the float32 kernels, .to(dtype)), alternated in
one process.

  (1) per call: `functional.gdn_forward` / `gdn_backward` at n_pix in {131072, 1048576}, median of --reps calls (CUDA
      events, after warm-up) per path, the three paths alternated three times.  GB/s on the algorithmic bytes (16-bit:
      4 B/element forward, 6 backward; float32: 8 and 12) with the fraction of 3.35 TB/s, beside the bytes the kernels
      move by design (BYTES_MOVED).  The native result is checked bitwise against the conversion path's on the timed
      inputs;
  (2) where the backward's time goes: device time per kernel from torch.profiler in a separate pass, 1048576 pixels;
  (3) model level: BLS2017Model(num_filters=128) and BMSHJ2018Model(num_filters=192) training steps (forward and
      loss.backward() under torch.autocast("cuda", dtype=torch.bfloat16)) at batch 8, 256x256, native against the
      conversion path alternated three times, with peak memory and the loss of each.
The card's name, power limit and SM clock are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/gdn16_bench.py [--reps 20] [--dtype bfloat16] [--out DIR]
"""
import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_PEAK = 3.35e12  # H100 SXM data sheet
WIDTHS = (128, 192)
SIZES = (131072, 1048576)
ALGO_BYTES = {("float32", "forward"): 8, ("float32", "backward"): 12, ("16bit", "forward"): 4,
              ("16bit", "backward"): 6}
# HBM bytes per element the kernels move by design (an L2 hit counts as none):
#   forward: x in, y out (the epilogue's re-read of x hits L2);
#   float32 backward: x, dy in, q, dx out (dx kernel; the read-back of dx hits L2), x, q in (dgamma kernel) = 24;
#   native 16-bit backward: x, dy in (2 + 2), q out (4), dx out (2), x, q in (2 + 4) = 16, plus the direct-term
#     scratch (4 out + 4 in) if it leaves L2 (at most 148 CTAs x 64 x C floats, about 14.5 MB);
#   conversion path: x.float() and dy.float() (2 in + 4 out each), the float32 backward (24), dx.to() (4 in, 2 out)
#     = 42 backward; forward 6 + 8 + 6 = 20.
BYTES_MOVED = {"float32": {"forward": "8", "backward": "24"},
               "native": {"forward": "4", "backward": "16 + up to 8 of scratch"},
               "conversion": {"forward": "20", "backward": "42"}}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--dtype", default="bfloat16", choices=("bfloat16", "float16"))
  ap.add_argument("--steps", type=int, default=10, help="training steps per timed window")
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tools"))
  import torch
  from torch.profiler import ProfilerActivity, profile
  from compression_b200 import functional as F
  from compression_b200 import models
  from ragged_bench import card
  assert torch.cuda.is_available(), "gdn16_bench needs a CUDA device"
  dev = torch.device("cuda")
  dt = getattr(torch, args.dtype)
  res = {"card_before": card(), "device": torch.cuda.get_device_name(), "dtype": args.dtype,
         "bytes_moved_per_element": BYTES_MOVED, "calls": {}, "profile": {}, "steps": {}}
  native16 = F._gdn_native16

  def route(native):
    F._gdn_native16 = native16 if native else (lambda *a, **k: False)

  def timed(fn, reps):
    ts = []
    for _ in range(reps):
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      fn()
      b.record()
      b.synchronize()
      ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]

  def same(a, b):
    nan = torch.isnan(b)
    return bool(torch.equal(torch.isnan(a), nan) and torch.equal(a[~nan], b[~nan]))

  for C in WIDTHS:
    g = torch.Generator().manual_seed(C)
    gamma = (0.1 * torch.eye(C) + (0.02 * torch.randn(C, C, generator=g)).abs()).to(dev)
    beta = (1.0 + 0.5 * torch.rand(C, generator=g)).to(dev)
    for n_pix in SIZES:
      x32 = torch.randn(n_pix, C, device=dev) * 2
      dy32 = torch.randn(n_pix, C, device=dev)
      x16, dy16 = x32.to(dt), dy32.to(dt)
      for kind in ("forward", "backward"):
        fns = {"float32": (True, (lambda: F.gdn_forward(x32, gamma, beta)) if kind == "forward" else
                           (lambda: F.gdn_backward(x32, gamma, beta, dy32))),
               "native": (True, (lambda: F.gdn_forward(x16, gamma, beta)) if kind == "forward" else
                          (lambda: F.gdn_backward(x16, gamma, beta, dy16))),
               "conversion": (False, (lambda: F.gdn_forward(x16, gamma, beta)) if kind == "forward" else
                              (lambda: F.gdn_backward(x16, gamma, beta, dy16)))}
        outs = {}
        for name, (native, fn) in fns.items():
          route(native)
          outs[name] = fn()
          fn()
        route(True)
        o_n = outs["native"] if kind == "backward" else (outs["native"],)
        o_c = outs["conversion"] if kind == "backward" else (outs["conversion"],)
        r = {"native_equals_conversion": all(same(a, b) for a, b in zip(o_n, o_c)), "ms": {}}
        del outs, o_n, o_c
        ts = {name: [] for name in fns}
        for _ in range(3):  # alternated
          for name, (native, fn) in fns.items():
            route(native)
            ts[name].append(timed(fn, args.reps))
        route(True)
        for name in fns:
          ms = sorted(ts[name])[1]
          scale = "float32" if name == "float32" else "16bit"
          gbps = ALGO_BYTES[(scale, kind)] * n_pix * C / (ms * 1e-3) / 1e9
          r["ms"][name] = ts[name]
          r[name] = {"ms_median": ms, "algorithmic_B_per_element": ALGO_BYTES[(scale, kind)], "GBps": gbps,
                     "fraction_of_3.35TBps": gbps * 1e9 / HBM_PEAK,
                     "moved_B_per_element": BYTES_MOVED[name][kind]}
        r["native_speedup_over_conversion"] = r["conversion"]["ms_median"] / r["native"]["ms_median"]
        r["native_speedup_over_float32"] = r["float32"]["ms_median"] / r["native"]["ms_median"]
        res["calls"][f"C{C}_n{n_pix}_{kind}"] = r
        print(json.dumps({f"C{C}_n{n_pix}_{kind}": r}), file=sys.stderr, flush=True)
      if n_pix == SIZES[-1]:
        per = {}
        for name, native, xx, dd in (("native", True, x16, dy16), ("float32", True, x32, dy32)):
          route(native)
          F.gdn_backward(xx, gamma, beta, dd)
          torch.cuda.synchronize()
          with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
              F.gdn_backward(xx, gamma, beta, dd)
            torch.cuda.synchronize()
          k = {}
          for e in prof.events():
            if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset")):
              m = re.search(r"(\w+)(<[^>]*>)?\(", e.name)
              kn = m.group(1) + (m.group(2) or "") if m else e.name
              k[kn] = k.get(kn, 0.) + e.device_time / 5 / 1e3
          per[name] = k
        route(True)
        res["profile"][f"C{C}_n{n_pix}_backward_ms_per_call"] = per
      del x32, dy32, x16, dy16

  for name, make in (("bls2017_128", lambda: models.BLS2017Model(num_filters=128).build("cuda")),
                     ("bmshj2018_192", lambda: models.BMSHJ2018Model(num_filters=192).build("cuda", patch=(64, 64)))):
    torch.manual_seed(0)
    m = make()
    x = torch.rand(8, 256, 256, 3, generator=torch.Generator().manual_seed(2)).mul(255).to(dev)

    def train():
      torch.manual_seed(3)
      m.zero_grad(set_to_none=True)
      with torch.autocast("cuda", dtype=torch.bfloat16):
        loss, _, _ = m(x, training=True)
      loss.backward()
      return loss

    r = {}
    for native in (True, False):
      route(native)
      train()
      torch.cuda.synchronize()
      m.zero_grad(set_to_none=True)
      torch.cuda.reset_peak_memory_stats()
      base = torch.cuda.memory_allocated()
      loss = train()
      torch.cuda.synchronize()
      r["native" if native else "conversion"] = {
          "ms": [], "loss": float(loss.detach()),
          "max_memory_allocated_MB": torch.cuda.max_memory_allocated() / 2**20,
          "peak_above_start_MB": (torch.cuda.max_memory_allocated() - base) / 2**20}
    for _ in range(3):
      for native in (True, False):
        route(native)
        r["native" if native else "conversion"]["ms"].append(timed(train, args.steps))
    route(True)
    r["speedup"] = sorted(r["conversion"]["ms"])[1] / sorted(r["native"]["ms"])[1]
    r["loss_equal"] = r["native"]["loss"] == r["conversion"]["loss"]
    res["steps"][name] = r
    print(json.dumps({name: r}), file=sys.stderr, flush=True)
    del m

  res["card_after"] = card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gdn16_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
