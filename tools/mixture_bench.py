"""Times the mixture coder (DESIGN.md §3.18): K = 3 Normal mixtures on 24 latents of 32 x 48 x 192, encode and
decode in Gsym/s at S = 1 and S = 16 streams per image, the one-image decode, and the compiled reference coder on
the host cores with materialised rows at its best thread count.  What bounds a one-image decode is probed by the
same decode at K = 1: a third of the row building, with a chain of the same length.  Prints one JSON line with the
card's name, power limit and maximum SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from compression_b200 import functional as F  # noqa: E402


def card():
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    return q
  except Exception as e:  # pylint:disable=broad-except
    return f"unknown ({e})"


def compact(size, rows):
  """The rows of mixture_tables as the reference's 1-D lookup: each row's [-p, c_0 .. c_n] without its padding."""
  size, rows = size.cpu().numpy(), rows.cpu().numpy()
  return rows[np.arange(rows.shape[1])[None, :] < (size[:, None] + 3)]


def timed(fn, reps):
  fn()
  torch.cuda.synchronize()
  t = time.perf_counter()
  for _ in range(reps):
    fn()
  torch.cuda.synchronize()
  return (time.perf_counter() - t) / reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--images", type=int, default=24)
  ap.add_argument("--reps", type=int, default=3)
  ap.add_argument("--ref-images", type=int, default=0,
                  help="images the reference coder codes, one stream each (default: one per host core)")
  a = ap.parse_args()
  rng = np.random.default_rng(0)
  per = 32 * 48 * 192
  n, K = a.images * per, 3
  w = torch.from_numpy(rng.random((n, K), dtype=np.float32) + 0.05).cuda()
  mu = torch.from_numpy((rng.standard_normal((n, K)) * 2).astype(np.float32)).cuda()
  sg = torch.from_numpy(np.exp(rng.uniform(np.log(0.2), np.log(8.0), (n, K))).astype(np.float32)).cuda()
  y = (mu[:, 0] + sg[:, 0] * torch.randn(n, device="cuda")).contiguous()
  res = {"card": card(), "images": a.images, "latent": [32, 48, 192], "K": K}
  for S in (1, 16):
    lengths = [per // S] * (a.images * S)
    strings = F.mixture_encode_ragged(y, w, mu, sg, lengths)
    te = timed(lambda: F.mixture_encode_ragged(y, w, mu, sg, lengths), a.reps)
    td = timed(lambda: F.mixture_decode_ragged(strings, w, mu, sg, lengths), a.reps)
    out = F.mixture_decode_ragged(strings, w, mu, sg, lengths)
    assert torch.equal(out, torch.round(y).clamp(-2**31, 2**31 - 1))
    res[f"S{S}"] = {"encode_gsym_s": n / te / 1e9, "decode_gsym_s": n / td / 1e9,
                    "bytes": int(strings.offsets_dev[-1]), "encode_ms": te * 1e3, "decode_ms": td * 1e3}
  one = F.mixture_encode_ragged(y[:per], w[:per], mu[:per], sg[:per], [per])
  res["one_image_decode_ms"] = 1e3 * timed(lambda: F.mixture_decode_ragged(one, w[:per], mu[:per], sg[:per], [per]),
                                           a.reps)
  # K = 1: the first component alone (a third of the transcendentals per row)
  w1, mu1, sg1 = (t[:per, :1].contiguous() for t in (w, mu, sg))
  one1 = F.mixture_encode_ragged(y[:per], w1, mu1, sg1, [per])
  res["one_image_decode_k1_ms"] = 1e3 * timed(lambda: F.mixture_decode_ragged(one1, w1, mu1, sg1, [per]), a.reps)
  if oracle.have_ref():
    # one stream per host core over at most 8 images' symbols, rows built one image at a time and kept compact:
    # host memory stays near 8 images' compact lookup whatever the core count
    cores = os.cpu_count() or 1
    R = a.ref_images or cores
    m = min(R, 8) * per
    L = m // R
    parts, st = [], []
    for lo in range(0, R * L, per):
      hi = min(lo + per, R * L)
      s_, sz, _, rows = F.mixture_tables(w[lo:hi], mu[lo:hi], sg[lo:hi])
      parts.append(compact(sz, rows))
      st.append(s_.cpu().numpy().astype(np.int64))
      del rows
    lookup = np.concatenate(parts)
    del parts
    v = (torch.round(y[:R * L]).cpu().numpy().astype(np.int64) - np.concatenate(st)).astype(np.int32).reshape(R, L)
    idx = np.arange(R * L, dtype=np.int32).reshape(R, L)
    O = oracle.ref()
    rates = {}
    for threads in range(1, cores + 1):
      enc = O.encoder(lookup, R)
      t = time.perf_counter()
      enc.encode(v, index=idx, threads=threads)
      enc.finalize()
      rates[threads] = R * L / (time.perf_counter() - t) / 1e6
      enc.close()
    best = max(rates, key=rates.get)
    res["reference_encode_msym_s"] = rates[best]
    res["reference_threads"] = best
    res["reference_msym_s_by_threads"] = rates
    res["reference_streams"] = R
    res["reference_symbols"] = R * L
    res["host_cores"] = cores
  print(json.dumps(res))


if __name__ == "__main__":
  main()
