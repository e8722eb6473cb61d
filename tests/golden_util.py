"""Loads tests/golden/range_coder_golden.npz (generated from the compiled reference by oracle/make_golden.py) and
tests/golden/reference_outputs.npz (the compiled reference's outputs on the tests' seeded cases, written by
oracle/make_reference_outputs.py)."""
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "range_coder_golden.npz")
REFERENCE_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_outputs.npz")


def load():
  return dict(np.load(PATH))


def load_reference():
  return dict(np.load(REFERENCE_PATH))


def split(flat, lens):
  out, at = [], 0
  for n in lens:
    out.append(bytes(flat[at:at + int(n)]))
    at += int(n)
  return out


def split_rows(ref, key):
  """Arrays stored flat under `key` with their shapes under `key`_shape, in order."""
  out, at = [], 0
  for shape in ref[key + "_shape"]:
    n = int(np.prod(shape))
    out.append(ref[key][at:at + n].reshape(tuple(int(v) for v in shape)))
    at += n
  return out
