"""GDN at 192 / 256 / 320 channels on the H100: the tensor-core path against the fp32 CUDA-core path
(`TFCB_GDN_FP32=1`, read by the library on every call), alternated in one process.

  (1) kernel level: `functional.gdn_forward` / `gdn_backward` at n_pix in {8192, 32768, 131072, 1048576} (the GDN
      layers of a batch-8 256x256 training step, and 256x64x64): median of --reps calls (CUDA events, after warm-up),
      GB/s on the algorithmic bytes (forward 8 B/element: x in, y out; backward 12: x, dy in, dx out) and the fraction
      of 3.35 TB/s, and the largest difference between the two paths on the timed inputs.  An fp32-path size whose
      first call is predicted (from the next smaller size) or measured to take more than --max-call-s is not timed;
  (2) where the time goes: device time per kernel from torch.profiler in a separate pass, at 131072 pixels;
  (3) model level: BMSHJ2018Model(num_filters=320) and BLS2017Model(num_filters=256) training steps (forward and
      loss.backward()) at batch 8, 256x256, the two paths alternated three times, with peak memory.
The card's name, power limit and SM clock are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/gdn_wide_bench.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_PEAK = 3.35e12  # H100 SXM data sheet
WIDTHS = (192, 256, 320)
SIZES = (8192, 32768, 131072, 1048576)
ALGO_BYTES = {"forward": 8, "backward": 12}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--max-call-s", type=float, default=10.0)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tools"))
  import torch
  from torch.profiler import ProfilerActivity, profile
  from compression_b200 import functional as F
  from compression_b200 import models
  from ragged_bench import card
  assert torch.cuda.is_available(), "gdn_wide_bench needs a CUDA device"
  dev = torch.device("cuda")
  res = {"card_before": card(), "device": torch.cuda.get_device_name(), "kernels": {}, "profile": {}, "steps": {}}

  def path(old):
    if old:
      os.environ["TFCB_GDN_FP32"] = "1"
    else:
      os.environ.pop("TFCB_GDN_FP32", None)

  def once(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t

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

  for C in WIDTHS:
    g = torch.Generator().manual_seed(C)
    gamma = (0.1 * torch.eye(C) + (0.02 * torch.randn(C, C, generator=g)).abs()).to(dev)
    beta = (1.0 + 0.5 * torch.rand(C, generator=g)).to(dev)
    old_call_s = {}  # kind -> (n_pix, seconds) of the last fp32-path call
    for n_pix in SIZES:
      x = torch.randn(n_pix, C, device=dev) * 2
      dy = torch.randn(n_pix, C, device=dev)
      calls = {"forward": lambda: F.gdn_forward(x, gamma, beta),
               "backward": lambda: F.gdn_backward(x, gamma, beta, dy)}
      for kind, fn in calls.items():
        r = {}
        path(False)
        new_out, _ = once(fn)
        fn()
        prev = old_call_s.get(kind)
        if prev is not None and prev[1] * n_pix / prev[0] > args.max_call_s:
          r["fp32_path"] = f"not timed: one call predicted to take {prev[1] * n_pix / prev[0]:.0f} s"
          old_out = None
        else:
          path(True)
          old_out, s = once(fn)
          old_call_s[kind] = (n_pix, s)
          if s > args.max_call_s:
            r["fp32_path"] = f"not timed: one call took {s:.1f} s"
            old_out = None
        path(False)
        if old_out is not None:
          reps = args.reps if old_call_s[kind][1] < 0.05 else max(3, min(args.reps, int(2 / old_call_s[kind][1])))
          t_new, t_old = [], []
          for _ in range(3):  # alternated
            path(False)
            t_new.append(timed(fn, args.reps))
            path(True)
            t_old.append(timed(fn, reps))
          path(False)
          r["ms"] = sorted(t_new)[1]
          r["fp32_path_ms"] = sorted(t_old)[1]
          r["speedup"] = r["fp32_path_ms"] / r["ms"]
          outs = (new_out,) if kind == "forward" else new_out
          olds = (old_out,) if kind == "forward" else old_out
          r["max_diff_of_max"] = max(((a.double() - b.double()).abs().max() / b.double().abs().max()).item()
                                     for a, b in zip(outs, olds))
        else:
          r["ms"] = timed(fn, args.reps)
        gbps = ALGO_BYTES[kind] * n_pix * C / (r["ms"] * 1e-3) / 1e9
        r["GBps"] = gbps
        r["fraction_of_3.35TBps"] = gbps * 1e9 / HBM_PEAK
        res["kernels"][f"C{C}_n{n_pix}_{kind}"] = r
        print(json.dumps({f"C{C}_n{n_pix}_{kind}": r}), file=sys.stderr, flush=True)
      del x, dy

    # where the time goes (tensor-core path)
    n_pix = 131072
    x = torch.randn(n_pix, C, device=dev) * 2
    dy = torch.randn(n_pix, C, device=dev)
    path(False)
    F.gdn_backward(x, gamma, beta, dy)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for _ in range(5):
        F.gdn_forward(x, gamma, beta)
        F.gdn_backward(x, gamma, beta, dy)
      torch.cuda.synchronize()
    per = {}
    for e in prof.events():
      if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset")):
        m = re.search(r"(\w+)(<[^>]*>)?\(", e.name)
        name = m.group(1) + (m.group(2) or "") if m else e.name
        per[name] = per.get(name, 0.) + e.device_time / 5 / 1e3
    res["profile"][f"C{C}_n{n_pix}_ms_per_call"] = per
    del x, dy

  for name, make in (("bmshj2018_320", lambda: models.BMSHJ2018Model(num_filters=320)),
                     ("bls2017_256", lambda: models.BLS2017Model(num_filters=256))):
    torch.manual_seed(0)
    m = make().build("cuda", patch=(64, 64))
    x = torch.rand(8, 256, 256, 3, generator=torch.Generator().manual_seed(2)).mul(255).to(dev)

    def train():
      torch.manual_seed(3)
      m.zero_grad(set_to_none=True)
      loss, bpp, _ = m(x, training=True)
      loss.backward()
      return loss

    r = {}
    for old in (False, True):
      path(old)
      train()
      torch.cuda.synchronize()
      torch.cuda.reset_peak_memory_stats()
      loss, s = once(train)
      tag = "fp32_path" if old else "tensor_core"
      r[tag] = {"ms": [], "max_memory_allocated_MB": torch.cuda.max_memory_allocated() / 2**20,
                "loss": float(loss.detach()), "first_timed_step_s": s}
    for _ in range(3):
      for old in (False, True):
        path(old)
        tag = "fp32_path" if old else "tensor_core"
        r[tag]["ms"].append(timed(train, 10 if r[tag]["first_timed_step_s"] < 1 else 3))
    path(False)
    r["speedup"] = sorted(r["fp32_path"]["ms"])[1] / sorted(r["tensor_core"]["ms"])[1]
    r["loss_rel_diff"] = abs(r["tensor_core"]["loss"] - r["fp32_path"]["loss"]) / abs(r["fp32_path"]["loss"])
    res["steps"][name] = r
    print(json.dumps({name: r}), file=sys.stderr, flush=True)
    del m

  res["card_after"] = card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gdn_wide_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
