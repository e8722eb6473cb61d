"""CPU: tfcb_gdn_backward_exponents (the five GDN gradients in one call) checks its host-side arguments before any
device work, so these run without a GPU.  The calls run on a worker thread: the library's last-error message is per
thread, and these tests leave the main thread's empty."""
import concurrent.futures
import ctypes as C

import pytest

from compression_b200 import _lib

_P = C.c_void_p(256)  # never dereferenced: every call below is rejected first


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _call(n_pix=100, C_=128, null=None):
  ptrs = [None if i == null else _P for i in range(9)]  # x, gamma, beta, dy, dx, dgamma, dbeta, dalpha_depsilon, ws
  return _lib.lib().tfcb_gdn_backward_exponents(*ptrs, n_pix, C_, 4 | 8, 1.2, 0.9, None)


@pytest.mark.parametrize("n_pix,C_", [(-1, 128), (100, 0), (100, -3)])
def test_rejects_bad_shapes_without_a_device(n_pix, C_):
  with pytest.raises(_lib.InvalidArgumentError, match="bad GDN shape"):
    _on_worker(lambda: _lib.check(_call(n_pix, C_)))


@pytest.mark.parametrize("null", range(9))
def test_rejects_null_pointers_without_a_device(null):
  with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
    _on_worker(lambda: _lib.check(_call(null=null)))


def test_rejects_a_width_the_exponent_kernel_cannot_hold():
  with pytest.raises(_lib.InvalidArgumentError, match="C too large"):
    _on_worker(lambda: _lib.check(_call(C_=4096)))


def test_workspace_extends_the_backward_workspace():
  L = _lib.lib()
  for n_pix, C_ in [(0, 128), (1, 192), (100_000, 320)]:
    assert (L.tfcb_gdn_backward_exponents_workspace_bytes(n_pix, C_) ==
            L.tfcb_gdn_backward_workspace_bytes(n_pix, C_) + L.tfcb_gdn_exponent_grads_workspace_bytes())
