"""The rate term of a training step on the H100: fused likelihood kernels against the graph of another tree.

Per tree (each run in a fresh process, the trees alternated three times):
  (1) the rate term alone, forward + backward (`entropy_model(y, training=True)`, `bits.sum().backward()`):
      bls2017 y [B,16,16,128] (ContinuousBatchedEntropyModel, NoisyDeepFactorized), bmshj2018 z [B,4,4,192] (the
      same) and y [B,16,16,192] (LocationScaleIndexedEntropyModel, NoisyNormal, 64 scales 0.11 ... 256), B = 8 and
      64: median time per call (CUDA events) and, from torch.profiler in a separate pass, CUDA kernels per call and
      the device time of the fused kernels (GB/s on their algorithmic bytes: deep factorized 4 + 4 B/element
      forward, 8 + 4 backward; location-scale 12 forward, 20 backward);
  (2) a full training step (forward + backward) of BLS2017Model and BMSHJ2018Model at batch 8, 256x256: median step
      time and torch.cuda.max_memory_allocated;
  (3) the losses and bits, so that the trees can be compared.
The card's name and power limit are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/rate_bench.py [--parent DIR] [--reps 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_PEAK = 3.35e12  # H100 SXM data sheet
SHAPES = {"bls2017_y": (16, 16, 128, "df"), "bmshj2018_z": (4, 4, 192, "df"), "bmshj2018_y": (16, 16, 192, "ls")}
ALGO_BYTES = {"df": (8, 12), "ls": (12, 20)}  # per element: forward, backward


def child(root, reps):
  """Measurements of the tree at `root` (its own library and Python package)."""
  sys.path.insert(0, root)
  import torch
  from torch.profiler import ProfilerActivity, profile
  from compression_b200 import distributions as D
  from compression_b200 import entropy_models as E
  from compression_b200 import models
  assert torch.cuda.is_available(), "rate_bench needs a CUDA device"
  dev = torch.device("cuda")
  scale_fn = lambda i: torch.exp(i * ((torch.log(torch.tensor(256.)) - torch.log(torch.tensor(.11))) / 63) +
                                 torch.log(torch.tensor(.11)))
  res = {"rate": {}, "step": {}}

  def timed(fn):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      fn()
      b.record()
      b.synchronize()
      ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]

  def profiled(fn, n=5):
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for _ in range(n):
        fn()
      torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type.name == "CUDA" and not e.name.startswith("Memcpy") and
          not e.name.startswith("Memset")]
    fused = {}
    for e in ev:
      if "noisy_" in e.name:
        k = "backward" if "bwd" in e.name or ", true>" in e.name or "Lb1E" in e.name else "forward"
        fused[k] = fused.get(k, 0.) + e.device_time / n / 1e3
    return len(ev) / n, fused

  for B in (8, 64):
    for name, (h, w, C, kind) in SHAPES.items():
      torch.manual_seed(0)
      y = (torch.randn(B, h, w, C, device=dev) * 3).requires_grad_(True)
      if kind == "df":
        prior = D.NoisyDeepFactorized(batch_shape=(C,), device=dev)
        em = E.ContinuousBatchedEntropyModel(prior, coding_rank=3, compression=False)
        args = ()
      else:
        em = E.LocationScaleIndexedEntropyModel(D.NoisyNormal, 64, scale_fn, coding_rank=3, compression=False)
        args = ((torch.rand(B, h, w, C, device=dev) * 63).requires_grad_(True),)

      def step():
        torch.manual_seed(1)
        _, bits = em(y, *args, training=True)
        bits.sum().backward()
        return bits

      bits = step()
      ms = timed(step)
      kernels, fused = profiled(step)
      n = y.numel()
      r = {"elements": n, "ms_per_call": ms, "cuda_kernels_per_call": kernels, "bits_sum": float(bits.sum())}
      if fused:
        fb, bb = ALGO_BYTES[kind]
        r["fused_kernel_ms"] = fused
        r["fused_GBps"] = {k: (fb if k == "forward" else bb) * n / (v * 1e-3) / 1e9 for k, v in fused.items()}
        r["fused_fraction_of_3.35TBps"] = {k: v * 1e9 / HBM_PEAK for k, v in r["fused_GBps"].items()}
      res["rate"][f"{name}_B{B}"] = r

  for name, make in (("bls2017", lambda: models.BLS2017Model(num_filters=128)),
                     ("bmshj2018", lambda: models.BMSHJ2018Model())):
    torch.manual_seed(0)
    m = make().build("cuda", patch=(64, 64))
    x = torch.rand(8, 256, 256, 3, generator=torch.Generator().manual_seed(2)).mul(255).to(dev)

    def train():
      torch.manual_seed(3)
      loss, bpp, _ = m(x, training=True)
      loss.backward()
      return loss, bpp

    train()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss, bpp = train()
    peak = torch.cuda.max_memory_allocated()
    res["step"][name] = {"ms": timed(train), "max_memory_allocated_MB": peak / 2**20, "loss": float(loss),
                         "bpp": float(bpp)}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--parent", default=None, help="root of another built tree to compare with")
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--child", default=None, help=argparse.SUPPRESS)  # child mode: tree root to measure
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if args.child:
    print(json.dumps(child(args.child, args.reps)))
    return
  sys.path.insert(0, os.path.join(ROOT, "tools"))
  import torch
  from ragged_bench import card
  trees = [("this", ROOT)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
  res = {"card_before": card(), "runs": {t: [] for t, _ in trees}}
  for _ in range(3 if args.parent else 1):
    for tag, root in trees:
      out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", root, "--reps", str(args.reps)],
                           check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1]
      res["runs"][tag].append(json.loads(out))
  summary = {}
  for tag, runs in res["runs"].items():
    s = {}
    for key in runs[0]["rate"]:
      s[key] = {"ms": [r["rate"][key]["ms_per_call"] for r in runs],
                "cuda_kernels_per_call": runs[0]["rate"][key]["cuda_kernels_per_call"]}
    for key in runs[0]["step"]:
      s[key + "_step"] = {"ms": [r["step"][key]["ms"] for r in runs],
                          "max_memory_allocated_MB": runs[0]["step"][key]["max_memory_allocated_MB"]}
    summary[tag] = s
  if args.parent:
    a, b = res["runs"]["this"][0], res["runs"]["parent"][0]
    rel = lambda u, v: abs(u - v) / max(abs(v), 1e-30)
    summary["relative_difference"] = {
        **{k: rel(a["rate"][k]["bits_sum"], b["rate"][k]["bits_sum"]) for k in a["rate"]},
        **{k + "_loss": rel(a["step"][k]["loss"], b["step"][k]["loss"]) for k in a["step"]}}
  res["summary"] = summary
  res["card_after"] = card()
  res["device"] = torch.cuda.get_device_name() if torch.cuda.is_available() else None
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "rate_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
