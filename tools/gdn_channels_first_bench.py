"""GDN on channels-first activations on the H100: the native path (kernels that read and write [N, C, H, W] in
place), the movedim path (a channels-last copy of x, the channels-last kernels, a channels-last-strided result;
forced by monkeypatching functional._gdn_native_cf), and channels-last on NHWC data, alternated in one process.

  (1) per call, [16, C, 256, 256] (1 048 576 pixels), C in {128, 192, 256, 320} float32 and {128, 192} bfloat16:
      `GDN(data_format=...)` forward (no grad) and forward + backward (torch.autograd.grad of the input and the
      parameters), median of --reps calls per path (CUDA events, after warm-up), the three paths alternated three
      times; the spread is the range of the three medians.  GB/s on the algorithmic bytes (float32 8 B/element
      forward, 12 backward; 16-bit 4 and 6; forward + backward counts both).  The three paths' outputs and gradients
      are compared bitwise on the timed inputs;
  (2) a training step of a bls2017-shaped NCHW model (Conv2d 5x5 / stride 2 and GDN, ConvTranspose2d and IGDN, 128
      channels, batch 8 at 256x256, MSE loss), native against the movedim path in --windows alternated windows of
      --steps steps (each window gives the median step time; reported: the median and range of the windows), with
      max_memory_allocated and the loss of each.
The card's name, power limit and SM clock are read in the same run.  Needs a CUDA device; prints one JSON object.

  python tools/gdn_channels_first_bench.py [--reps 20] [--steps 30] [--windows 9] [--out DIR]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_PEAK = 3.35e12  # H100 SXM data sheet
CONFIGS = (("float32", 128), ("float32", 192), ("float32", 256), ("float32", 320), ("bfloat16", 128),
           ("bfloat16", 192))
SHAPE = (16, 256, 256)  # N, H, W: 1 048 576 pixels
ALGO_BYTES = {("float32", "forward"): 8, ("float32", "forward_backward"): 20, ("bfloat16", "forward"): 4,
              ("bfloat16", "forward_backward"): 10}
PATHS = ("native", "movedim", "channels_last")


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--steps", type=int, default=30, help="training steps per timed window")
  ap.add_argument("--windows", type=int, default=9, help="timed windows per path of the training step")
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  sys.path.insert(0, ROOT)
  sys.path.insert(0, os.path.join(ROOT, "tools"))
  import torch
  from compression_b200 import functional as F
  from compression_b200.gdn import GDN
  from ragged_bench import card
  assert torch.cuda.is_available(), "gdn_channels_first_bench needs a CUDA device"
  dev = torch.device("cuda")
  res = {"card_before": card(), "device": torch.cuda.get_device_name(), "shape_NHW": SHAPE, "calls": {},
         "step": {}}
  native_cf = F._gdn_native_cf

  def route(native):
    F._gdn_native_cf = native_cf if native else (lambda *a, **k: False)

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
    a, b = a.contiguous(), b.contiguous()
    nan = torch.isnan(b)
    return bool(torch.equal(torch.isnan(a), nan) and torch.equal(a[~nan], b[~nan]))

  for dtype_name, C in CONFIGS:
    dt = getattr(torch, dtype_name)
    torch.manual_seed(C)
    n, h, w = SHAPE
    x_cf = (torch.randn(n, C, h, w, device=dev) * 2).to(dt)
    dy_cf = torch.randn(n, C, h, w, device=dev).to(dt)
    x_cl, dy_cl = x_cf.permute(0, 2, 3, 1).contiguous(), dy_cf.permute(0, 2, 3, 1).contiguous()
    layers = {"channels_first": GDN(data_format="channels_first"), "channels_last": GDN(data_format="channels_last")}
    for fmt, layer in layers.items():
      layer.build((1, C, 1, 1) if fmt == "channels_first" else (1, 1, 1, C), device=dev)
      with torch.no_grad():  # the same parameters in both, away from the initialiser
        layer.gamma_parameter.variable.add_(0.05 * torch.rand(C, C, generator=torch.Generator().manual_seed(1)).to(dev))
    cases = {"native": (True, layers["channels_first"], x_cf, dy_cf),
             "movedim": (False, layers["channels_first"], x_cf, dy_cf),
             "channels_last": (True, layers["channels_last"], x_cl, dy_cl)}

    def fns(path, kind):
      native, layer, x, dy = cases[path]
      params = [p for p in layer.parameters()]
      if kind == "forward":
        def run():
          with torch.no_grad():
            return (layer(x),)
      else:
        xg = x.detach().requires_grad_(True)

        def run():
          y = layer(xg)
          return (y,) + torch.autograd.grad(y, [xg] + params, dy)
      return native, run

    for kind in ("forward", "forward_backward"):
      runs = {p: fns(p, kind) for p in PATHS}
      outs = {}
      for p, (native, fn) in runs.items():
        route(native)
        outs[p] = fn()
        fn()
      route(True)
      to_cf = lambda t: t.permute(0, 3, 1, 2) if t.dim() == 4 else t  # noqa: E731
      r = {"native_equals_movedim": all(same(a, b) for a, b in zip(outs["native"], outs["movedim"])),
           "native_equals_channels_last": all(same(a, to_cf(b)) for a, b in zip(outs["native"], outs["channels_last"])),
           "native_output_contiguous": all(t.is_contiguous() for t in outs["native"][:2]), "ms": {}}
      del outs
      ts = {p: [] for p in PATHS}
      for _ in range(3):  # alternated
        for p, (native, fn) in runs.items():
          route(native)
          ts[p].append(timed(fn, args.reps))
      route(True)
      for p in PATHS:
        ms = sorted(ts[p])[1]
        gbps = ALGO_BYTES[(dtype_name, kind)] * n * h * w * C / (ms * 1e-3) / 1e9
        r["ms"][p] = ts[p]
        r[p] = {"ms_median": ms, "ms_spread": [min(ts[p]), max(ts[p])],
                "algorithmic_B_per_element": ALGO_BYTES[(dtype_name, kind)], "GBps": gbps,
                "fraction_of_3.35TBps": gbps * 1e9 / HBM_PEAK}
      r["native_speedup_over_movedim"] = r["movedim"]["ms_median"] / r["native"]["ms_median"]
      r["native_time_over_channels_last"] = r["native"]["ms_median"] / r["channels_last"]["ms_median"]
      key = f"{dtype_name}_C{C}_{kind}"
      res["calls"][key] = r
      print(json.dumps({key: r}), file=sys.stderr, flush=True)
    del x_cf, dy_cf, x_cl, dy_cl, cases, layers

  # a user's NCHW model: bls2017's transforms (analysis: 4 x Conv2d 5x5 stride 2 with GDN; synthesis: 4 x
  # ConvTranspose2d with IGDN), 128 channels
  def model():
    torch.manual_seed(0)
    nn = torch.nn
    Ch = 128
    enc = [nn.Conv2d(3, Ch, 5, 2, 2), GDN(data_format="channels_first"), nn.Conv2d(Ch, Ch, 5, 2, 2),
           GDN(data_format="channels_first"), nn.Conv2d(Ch, Ch, 5, 2, 2), GDN(data_format="channels_first"),
           nn.Conv2d(Ch, Ch, 5, 2, 2)]
    dec = [nn.ConvTranspose2d(Ch, Ch, 5, 2, 2, 1), GDN(inverse=True, data_format="channels_first"),
           nn.ConvTranspose2d(Ch, Ch, 5, 2, 2, 1), GDN(inverse=True, data_format="channels_first"),
           nn.ConvTranspose2d(Ch, Ch, 5, 2, 2, 1), GDN(inverse=True, data_format="channels_first"),
           nn.ConvTranspose2d(Ch, 3, 5, 2, 2, 1)]
    m = nn.Sequential(*enc, *dec).to(dev)
    m(torch.zeros(1, 3, 32, 32, device=dev))  # builds the GDN parameters
    return m

  m = model()
  x = torch.rand(8, 3, 256, 256, generator=torch.Generator().manual_seed(2)).to(dev)

  def train():
    m.zero_grad(set_to_none=True)
    loss = (m(x) - x).square().mean()
    loss.backward()
    return loss

  r = {}
  for native in (True, False):
    route(native)
    train()
    torch.cuda.synchronize()
    m.zero_grad(set_to_none=True)
    torch.cuda.reset_peak_memory_stats()
    loss = train()
    torch.cuda.synchronize()
    r["native" if native else "movedim"] = {"ms": [], "loss": float(loss.detach()),
                                           "max_memory_allocated_MB": torch.cuda.max_memory_allocated() / 2**20}
  for _ in range(args.windows):  # alternated
    for native in (True, False):
      route(native)
      r["native" if native else "movedim"]["ms"].append(timed(train, args.steps))
  route(True)
  for name in ("native", "movedim"):
    ms = sorted(r[name]["ms"])
    r[name]["ms_median"], r[name]["ms_spread"] = ms[len(ms) // 2], [ms[0], ms[-1]]
  r["speedup"] = r["movedim"]["ms_median"] / r["native"]["ms_median"]
  r["loss_equal"] = r["native"]["loss"] == r["movedim"]["loss"]
  res["step"]["bls2017_shaped_nchw_b8_256"] = r
  print(json.dumps({"step": r}), file=sys.stderr, flush=True)

  res["card_after"] = card()
  text = json.dumps(res, indent=1)
  print(text)
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gdn_channels_first_bench.json"), "w") as f:
      f.write(text + "\n")


if __name__ == "__main__":
  main()
