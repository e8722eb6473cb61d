"""Times MBT2018Model coding of 24 Kodak-shaped images (12 of 512x768, 12 of 768x512; random weights, synthetic
content) on the device-stepped path against a naive per-step path, and one-image decode latency.

  python tools/mbt2018_bench.py [--reps 3] [--latent-depth 192] [--out FILE.json]

Device path: compress_images / decompress_images (per image group of one latent shape: one encoder-loop launch and
one range encode; one decoder-loop launch).  Naive path, latent coding only: per position one tfcb_ar_params launch
plus torch quantisation (encoder) or tfcb_decode_index_f32 of M symbols per stream (decoder), with the same strings
and latents.  Prints one JSON object: medians in ms, library launches per call, and the card it ran on."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import _lib, functional as F, gen_ops, models  # noqa: E402


def _card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    q = torch.cuda.get_device_name()
  return q


def _images(n, seed=0):
  rng = np.random.default_rng(seed)
  out = []
  for i in range(n):
    h, w = (512, 768) if i % 2 == 0 else (768, 512)
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 70 * np.sin(xx / (9.0 + i)) [..., None] * np.cos(yy / 13.0)[..., None] * np.array([1.0, 0.8, 0.5])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 10, (h, w, 3)), 0, 255).astype(np.uint8)).cuda())
  return out


def _timed(fn, reps):
  """(median ms, library launches of one call, last result); one warm-up call first."""
  fn()
  torch.cuda.synchronize()
  ts, launches, out = [], None, None
  for _ in range(reps):
    n0 = _lib.launch_count()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    ts.append((time.perf_counter() - t0) * 1e3)
    launches = _lib.launch_count() - n0
  return float(np.median(ts)), launches, out


def _naive_encode(m, y, psi):
  B, H, W, M = y.shape
  y_hat = torch.zeros_like(y)
  loc = torch.zeros_like(y)
  index = torch.zeros(y.shape, dtype=torch.int32, device=y.device)
  fy, fh, fl, fi = (t.view(B, H * W, M) for t in (y, y_hat, loc, index))
  for p in range(H * W):
    l, _, i = F.ar_params(m._packed, y_hat, psi, p, m.num_scales)
    fh[:, p] = torch.round(fy[:, p] - l) + l
    fl[:, p], fi[:, p] = l, i
  em = m.entropy_model
  return F.compress_f32((B,), em._lookup_host(), y, loc, em.cdf_offset, index=index), y_hat


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--latent-depth", type=int, default=192)
  ap.add_argument("--num-filters", type=int, default=192)
  ap.add_argument("--images", type=int, default=24)
  ap.add_argument("--out", default=None)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("mbt2018_bench needs a CUDA device")
  torch.manual_seed(0)
  m = models.MBT2018Model(num_filters=a.num_filters, latent_depth=a.latent_depth).build("cuda", patch=(64, 64))
  m.fix_tables()
  imgs = _images(a.images)
  res = {"card": _card(), "images": f"{a.images} Kodak-shaped (512x768 / 768x512), synthetic, random weights",
         "num_filters": a.num_filters, "latent_depth": a.latent_depth, "reps": a.reps}

  with torch.no_grad():
    enc_ms, enc_l, items = _timed(lambda: m.compress_images(imgs), a.reps)
    dec_ms, dec_l, outs = _timed(lambda: m.decompress_images(items), a.reps)
    res["device"] = {"compress_images_ms": enc_ms, "decompress_images_ms": dec_ms,
                     "compress_ms_per_image": enc_ms / len(imgs), "decompress_ms_per_image": dec_ms / len(imgs),
                     "compress_launches": enc_l, "decompress_launches": dec_l}

    # latent coding alone, one group of each shape, device loop against the naive loop
    lat = {}
    for shape_imgs in (imgs[0::2], imgs[1::2]):
      ys, psis = [], []
      for x in shape_imgs:
        y = m.analysis_transform(x[None].float())
        z = m.hyper_analysis_transform(y)
        ys.append(y)
        psis.append(m._psi(m.side_entropy_model.quantize(z), tuple(y.shape[1:-1])))
      y, psi = torch.cat(ys).contiguous(), torch.cat(psis)
      key = "x".join(str(d) for d in y.shape[1:3])
      em = m.entropy_model
      d_enc, d_enc_l, (strings, y_hat, _, _) = _timed(lambda: m._encode_latents(y, psi), a.reps)
      d_dec, d_dec_l, y_dec = _timed(lambda: m._decode_latents(strings, psi), a.reps)
      n_enc, n_enc_l, (n_strings, n_y_hat) = _timed(lambda: _naive_encode(m, y, psi), max(1, a.reps - 2))

      def naive_decode():
        h = gen_ops.create_range_decoder(strings, em._lookup_host())
        out = F.ar_decode_naive(h, m._packed, psi, m.num_scales, em.cdf_offset)
        em._finish_decode(h)
        return out
      n_dec, n_dec_l, n_y_dec = _timed(naive_decode, max(1, a.reps - 2))
      assert n_strings.tolist() == strings.tolist() and torch.equal(n_y_hat, y_hat)
      assert torch.equal(y_dec, y_hat) and torch.equal(n_y_dec, y_hat)
      lat[key] = {"batch": y.shape[0], "device_encode_ms": d_enc, "device_decode_ms": d_dec,
                  "naive_encode_ms": n_enc, "naive_decode_ms": n_dec, "device_encode_launches": d_enc_l,
                  "device_decode_launches": d_dec_l, "naive_encode_launches": n_enc_l,
                  "naive_decode_launches": n_dec_l}
    res["latent_coding"] = lat

    one = items[0]
    res["one_image_decompress_ms"] = _timed(lambda: m.decompress(*one), a.reps)[0]
    y = m.analysis_transform(imgs[0][None].float())
    psi = m._psi(m.side_entropy_model.quantize(m.hyper_analysis_transform(y)), tuple(y.shape[1:-1]))
    res["one_image_latent_decode_ms"] = _timed(lambda: m._decode_latents(one[0], psi), a.reps)[0]
    res["round_trip_uint8"] = all(o.shape == x.shape for o, x in zip(outs, imgs))
  line = json.dumps(res)
  print(line)
  if a.out:
    with open(a.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
