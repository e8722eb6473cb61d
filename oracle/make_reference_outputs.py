"""Generates tests/golden/reference_outputs.npz: the COMPILED REFERENCE's outputs (oracle/_ref, built by
`make -C oracle ref` where the reference tree exists) on the seeded cases of the tests that compare the product with
it, so that those tests run wherever the repository does:
    python oracle/make_reference_outputs.py
Each test regenerates its inputs from the same case generator and compares against what is stored here."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import oracle  # noqa: E402
import test_baseline_configs_gpu  # noqa: E402
import test_misc_gpu  # noqa: E402
import test_oracle_pin as pin  # noqa: E402
import test_pmf_tables_gpu  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "reference_outputs.npz")


def flat_bytes(strings):
  lens = np.asarray([len(s) for s in strings], np.int64)
  return np.frombuffer(b"".join(strings), np.uint8), lens


def flat_rows(arrays):
  return np.concatenate([a.reshape(-1) for a in arrays]), np.asarray([a.shape for a in arrays], np.int64)


def main():
  R = oracle.ref()
  out = {}
  triples, batches = pin.coder_fuzz_cases()
  out["triples_bytes"], out["triples_len"] = flat_bytes([R.encode_triples(lo, hi, p) for lo, hi, p in triples])
  streams = []
  for lookup, val, index in batches:
    s = R.encode(lookup, val, index, threads=2)
    back, ok = R.decode(lookup, s, val.shape[1], index, threads=2)
    assert np.array_equal(back, val) and ok.all()
    streams += s
  out["streams_bytes"], out["streams_len"] = flat_bytes(streams)

  rounded = [R.stochastic_round(x, 0.75, seed) for seed, x in pin.stochastic_round_cases(np.random.default_rng(0))]
  out["stochastic_round"] = np.stack(rounded).astype(np.int32)

  codes, digests = [], []
  for rl, mg, nz, _, d in pin.run_length_fuzz_cases():
    code = R.run_length_encode(d, rl, mg, nz)
    codes.append(code)
    for damaged, shape in pin.damaged_codes(code, d.size):
      digests.append(np.frombuffer(pin.decode_outcome_digest(R, damaged, shape, rl, mg, nz), np.uint8))
  out["rl_codes"], out["rl_codes_len"] = flat_bytes(codes)
  out["rl_damaged_sha256"] = np.stack(digests)

  P = oracle.port()
  out["long_rice_decoded"] = np.stack([R.run_length_decode(P.run_length_encode(d, rl, mg, False), d.shape, rl, mg, False)
                                       for rl, mg, d in pin.long_rice_cases()])

  out["pmf_tie_cdf"], out["pmf_tie_cdf_shape"] = flat_rows(
      [R.pmf_to_cdf(pmf, 12)[0] for pmf in test_baseline_configs_gpu.tie_row_pmfs()])
  out["pmf_cdf"], out["pmf_cdf_shape"] = flat_rows(
      [R.pmf_to_cdf(test_misc_gpu.pmf_case(n, scale), p) for n, p, scale in test_misc_gpu.PMF_CASES])
  # stored as counts (the CDF's differences), which compress far better than the CDF itself
  out["pmf_edge_counts"], out["pmf_edge_counts_shape"] = flat_rows(
      [np.diff(R.pmf_to_cdf(pmf, p), axis=-1) for p, pmf in test_pmf_tables_gpu.tie_free_reference_rows()])

  np.savez_compressed(OUT, **out)
  print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
  main()
