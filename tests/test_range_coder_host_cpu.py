"""CPU: the range coder's compiled device code.  The host code between the C entry points and the kernels (the
operand description, the mode map, the compress and decode paths) may change; the kernels it instantiates may not."""
import hashlib
import os
import re
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compression_b200", "csrc")
NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)

# As compiled by CUDA 12.9: the number of functions and instructions, the sha256 of the instructions (functions sorted
# by name) and the sha256 of the sorted names.  The 50 functions are 18 encode_kernel and 20 decode_kernel (10 modes x
# SMEM) instantiations, the three legacy and three unbounded-index kernels, and enc_init_state, enc_offsets,
# enc_write, enc_grow, dec_init_state and dec_finalize.
RANGE_CODER_SASS = ("12.9", 50, 95648, "8e21575f06ab6c34b14955469cc6d102d09686c979c5c544d5fb38feb1198437",
                    "64e0dce3b4018d2a32b13be3409194af23c5f40a1134f6121b0277be55005f49")


@pytest.mark.skipif(NVCC is None, reason="nvcc is not installed")
def test_range_coder_sass_is_unchanged(tmp_path):
  version = re.search(r"release (\d+\.\d+)", subprocess.run([NVCC, "--version"], capture_output=True,
                                                             text=True).stdout).group(1)
  if version != RANGE_CODER_SASS[0]:
    pytest.skip(f"the reference hash is CUDA {RANGE_CODER_SASS[0]}'s, this is {version}")
  obj = str(tmp_path / "rc.o")
  subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler",
                  "-fPIC", "-I" + os.path.join(CSRC, "..", "..", "include"), "-I" + CSRC, "-c",
                  os.path.join(CSRC, "range_coder.cu"), "-o", obj], capture_output=True, text=True, check=True)
  cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
  sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
  funcs, cur = {}, None
  for line in sass.splitlines():
    m = re.match(r"\s+Function : (\S+)", line)
    if m:
      # the anonymous namespace's tag changes with the file's contents
      cur = re.sub(r"_GLOBAL__N__\w+?_cu_[0-9a-f]+", "_ANON_", m.group(1))
      funcs[cur] = []
      continue
    m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;?\s*(/\*.*\*/)?\s*$", line)
    if cur and m:
      funcs[cur].append(m.group(1))
  names = sorted(funcs)
  assert sum("9EncParams" in n for n in names) == 18 and sum("9DecParams" in n for n in names) == 20
  assert (len(names), sum(len(funcs[n]) for n in names)) == RANGE_CODER_SASS[1:3]
  assert hashlib.sha256("\n".join("\n".join(funcs[n]) for n in names).encode()).hexdigest() == RANGE_CODER_SASS[3]
  assert hashlib.sha256("\n".join(names).encode()).hexdigest() == RANGE_CODER_SASS[4]
