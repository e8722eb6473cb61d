"""GDN with trainable exponents: the literal-pow tensor-core kernels (gdn_tc.cu, gdn_tc_pow_*) against the CUDA-core
path (TFCB_GDN_FP32=1), alternated.

  (1) per width C in {128, 192, 256, 320} at 131 072 and 1 048 576 pixels: the forward and the five-gradient backward
      (functional.gdn_backward_exponents: dx, dgamma, dbeta, dalpha, depsilon), median of event-timed calls, with GB/s
      on the algorithmic 8 / 12 bytes per element.  A CUDA-core call predicted to take longer than --max-call-s is not
      timed.
  (2) batch-8 256x256 training steps (forward and loss.backward()) of BLS2017Model(128) and BMSHJ2018Model(320) with
      every GDN layer's alpha and epsilon trainable, the two paths alternated three times.
The card's name, power limit and SM clock are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/gdn_exponents_bench.py [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_PEAK = 3.35e12  # H100 SXM data sheet
WIDTHS = (128, 192, 256, 320)
SIZES = (131072, 1048576)
ALGO_BYTES = {"forward": 8, "backward": 12}
ALPHA, EPSILON = 1.25, 0.85


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--max-call-s", type=float, default=10.0)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tools"))
  import torch
  import compression_b200 as tfc
  from compression_b200 import functional as F
  from compression_b200 import models
  from ragged_bench import card
  assert torch.cuda.is_available(), "gdn_exponents_bench needs a CUDA device"
  dev = torch.device("cuda")
  res = {"card_before": card(), "device": torch.cuda.get_device_name(), "alpha": ALPHA, "epsilon": EPSILON,
         "kernels": {}, "steps": {}}

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
    old_call_s = {}
    for n_pix in SIZES:
      x = torch.randn(n_pix, C, device=dev) * 2
      dy = torch.randn(n_pix, C, device=dev)
      kw = dict(rectify=True, alpha=ALPHA, epsilon=EPSILON, pow_alpha=True, pow_epsilon=True)
      calls = {"forward": lambda: F.gdn_forward(x, gamma, beta, **kw),
               "backward": lambda: F.gdn_backward_exponents(x, gamma, beta, dy, **kw)}
      for kind, fn in calls.items():
        r = {}
        path(False)
        new_out, _ = once(fn)
        fn()
        prev = old_call_s.get(kind)
        old_out = None
        if prev is not None and prev[1] * n_pix / prev[0] > args.max_call_s:
          r["fp32_path"] = f"not timed: one call predicted to take {prev[1] * n_pix / prev[0]:.0f} s"
        else:
          path(True)
          old_out, s = once(fn)
          old_call_s[kind] = (n_pix, s)
          r["fp32_path_one_call_s"] = s
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

  for name, make in (("bls2017_128", lambda: models.BLS2017Model(num_filters=128)),
                     ("bmshj2018_320", lambda: models.BMSHJ2018Model(num_filters=320))):
    torch.manual_seed(0)
    m = make()
    for mod in m.modules():
      if isinstance(mod, tfc.GDN):
        mod.alpha_parameter = None
        mod.epsilon_parameter = None
    m.build("cuda", patch=(64, 64))
    x = torch.rand(8, 256, 256, 3, generator=torch.Generator().manual_seed(2)).mul(255).to(dev)

    def train():
      torch.manual_seed(3)
      m.zero_grad(set_to_none=True)
      loss, bpp, _ = m(x, training=True)
      loss.backward()
      return loss

    r = {"tensor_core": {"ms": []}, "fp32_path": {"ms": []}}
    for old in (False, True):
      path(old)
      train()
    for _ in range(3):
      for old in (False, True):
        path(old)
        loss, s = once(train)
        tag = "fp32_path" if old else "tensor_core"
        r[tag]["ms"].append(s * 1e3)
        r[tag]["loss"] = float(loss.detach())
    path(False)
    for tag in r:
      r[tag]["median_ms"] = sorted(r[tag]["ms"])[1]
    res["steps"][name] = r
    print(json.dumps({name: r}), file=sys.stderr, flush=True)
    del m, x

  res["card_after"] = card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gdn_exponents_bench.json"), "w") as f:
      f.write(text)


if __name__ == "__main__":
  main()
