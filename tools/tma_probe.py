"""Scratch: bytes per microsecond one SM's async-copy engine moves into shared memory (tfcb_debug_tma_probe)."""
import ctypes as C, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from compression_b200 import _lib
lib = C.CDLL(_lib.LIB_PATH)
f = lib.tfcb_debug_tma_probe
f.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.c_void_p]
Cc = 192
names = {0: "2-D boxes 128 x 128 B (swizzled)", 1: "1-D bulk 16 KB", 2: "1-D bulk 96 KB", 3: "2-D boxes in + 2-D TMA store out"}
sms = torch.cuda.get_device_properties(0).multi_processor_count
for n_rows, label in ((128 * 132, "L2-resident (13 MB)"), (4096 * 64 * 64 // 4, "HBM (3.2 GB)")):
  x = torch.randn(n_rows, Cc, device="cuda"); y = torch.empty_like(x)
  for mode in (0, 1, 2, 3):
    for depth in ((1, 2) if mode == 2 else (1, 2, 4, 8)):
      iters = 400 if mode != 2 else 100
      ms = C.c_float(0)
      rc = f(x.data_ptr(), y.data_ptr(), n_rows, Cc, mode, depth, iters, C.byref(ms), None)
      assert rc == 0, _lib.last_error() if hasattr(_lib, "last_error") else rc
      unit = 96 * 1024 if mode == 2 else 16 * 1024
      per_sm = iters * unit / (ms.value * 1e3)  # bytes per microsecond per SM
      print(f"{label:22s} {names[mode]:36s} depth {depth}: {per_sm/1e3:7.1f} KB/us per SM  ({per_sm*sms/1e6:6.2f} TB/s chip)  {ms.value*1e3/iters:6.3f} us per copy", flush=True)
