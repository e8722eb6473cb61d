"""CPU: the C-ABI shared library loads and exports every symbol include/tfcb200.h declares, and the
ctypes table in compression_b200/_lib.py covers exactly that set.  No compute calls (no GPU here)."""
import ctypes
import os
import re

import pytest

from compression_b200 import _lib

PROTO = re.compile(r"^\s*(?:const\s+)?[A-Za-z_][A-Za-z0-9_\s\*]*?\b(tfcb_[a-z0-9_]+)\s*\(", re.M)


def _declared():
  with open(_lib.HEADER_PATH) as f:
    text = f.read()
  text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
  return sorted(set(PROTO.findall(text)))


def test_library_loads_and_reports_the_header_abi_version():
  assert os.path.exists(_lib.LIB_PATH), "run `python -c 'import __graft_entry__ as g; g.build()'` first"
  lib = _lib.lib()
  with open(_lib.HEADER_PATH) as f:
    declared = int(re.search(r"^#define TFCB_ABI_VERSION (\d+)$", f.read(), re.M).group(1))
  assert lib.tfcb_abi_version() == declared == 2
  assert _lib.last_error() == ""
  assert _lib.launch_count() >= 0


def test_every_declared_symbol_is_exported_and_bound():
  names = _declared()
  assert len(names) >= 25
  raw = ctypes.CDLL(_lib.LIB_PATH)
  for n in names:
    assert hasattr(raw, n), f"{n} declared in tfcb200.h but not exported"
  assert sorted(_lib.SIGNATURES) == names


def test_argument_validation_that_needs_no_device():
  """Pure host-side checks return TFCB_INVALID_ARGUMENT before any CUDA call."""
  lib = _lib.lib()
  with pytest.raises(_lib.InvalidArgumentError, match="precision"):
    _lib.check(lib.tfcb_pmf_to_quantized_cdf(None, 1, 4, 0, None, None))
  with pytest.raises(_lib.InvalidArgumentError, match="at least 2"):
    _lib.check(lib.tfcb_pmf_to_quantized_cdf(None, 1, 1, 8, None, None))
  with pytest.raises(_lib.InvalidArgumentError, match="not an encoder"):
    _lib.check(lib.tfcb_encode_channel(None, None, 4, None))
  with pytest.raises(_lib.InvalidArgumentError, match="not a decoder"):
    _lib.check(lib.tfcb_decode_channel(None, None, 4, None))
  with pytest.raises(_lib.InvalidArgumentError, match="bad GDN shape"):
    _lib.check(lib.tfcb_gdn_forward(None, None, None, None, 4, 0, 0, 1.0, 1.0, None))


def test_product_never_imports_the_oracle():
  """The product path must not route through oracle/ (or any CPU fallback)."""
  root = os.path.dirname(os.path.dirname(_lib.HEADER_PATH))
  pkg = os.path.join(root, "compression_b200")
  for dirpath, _, files in os.walk(pkg):
    for fn in files:
      if fn.endswith((".py", ".cu", ".cuh", ".h")):
        with open(os.path.join(dirpath, fn)) as f:
          src = f.read()
        assert not re.search(r"^\s*(import|from)\s+oracle\b", src, re.M), f"{fn} imports the oracle"
        assert "oracle/" not in src or fn.endswith(".md"), f"{fn} references oracle/"
