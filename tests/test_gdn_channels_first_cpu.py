"""CPU: the channels-first GDN entries (tfcb_gdn_forward_cf / tfcb_gdn_backward_cf) check their host-side arguments
before any device work, and functional._gdn_native_cf decides which channels-first calls run on them.  The library
calls run on a worker thread: its last-error message is per thread, and these tests leave the main thread's empty.
The routing function looks at dtypes, shapes, strides, pointers and the environment only, so host tensors stand in
for device ones."""
import concurrent.futures
import ctypes as C

import pytest
import torch

from compression_b200 import _lib
from compression_b200 import functional as F

_P = C.c_void_p(256)  # 16-byte aligned and never dereferenced: every call below is rejected first
_ODD = C.c_void_p(260)  # 4 bytes past a 16-byte boundary


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _rejects(call, match):
  with pytest.raises(_lib.InvalidArgumentError, match=match):
    _on_worker(lambda: _lib.check(call()))


def _fwd(n=2, s=64, C_=128, dtype=0, flags=0, alpha=1.0, eps=1.0, ptrs=None):
  ptrs = ptrs or [_P] * 4  # x, gamma, beta, y
  return _lib.lib().tfcb_gdn_forward_cf(*ptrs, n, s, C_, dtype, flags, alpha, eps, None)


def _bwd(n=2, s=64, C_=128, dtype=0, flags=0, alpha=1.0, eps=1.0, ptrs=None):
  # x, gamma, beta, dy, dx, dgamma, dbeta, dalpha_depsilon, workspace
  ptrs = ptrs or [_P] * 7 + [None, _P]
  return _lib.lib().tfcb_gdn_backward_cf(*ptrs, n, s, C_, dtype, flags, alpha, eps, None)


@pytest.mark.parametrize("entry", [_fwd, _bwd])
@pytest.mark.parametrize("n,s,C_", [(-1, 64, 128), (2, -1, 128), (2, 64, 0), (2, 64, -128)])
def test_rejects_bad_shapes(entry, n, s, C_):
  _rejects(lambda: entry(n, s, C_), "bad GDN shape")


@pytest.mark.parametrize("entry", [_fwd, _bwd])
@pytest.mark.parametrize("n,s,C_", [(1 << 40, 1 << 20, 128), (1 << 62, 4, 128), (4, 1 << 62, 128),
                                    (1 << 28, 1 << 28, 256)])
def test_rejects_sizes_that_overflow(entry, n, s, C_):
  _rejects(lambda: entry(n, s, C_), "overflows")


@pytest.mark.parametrize("entry", [_fwd, _bwd])
@pytest.mark.parametrize("dtype", [-1, 3, 7])
def test_rejects_unknown_dtypes(entry, dtype):
  _rejects(lambda: entry(dtype=dtype), "dtype")


# (C, dtype, flags, alpha, epsilon) outside the tensor-core coverage: other widths, 16 bits at 256 / 320, 16 bits with
# a trainable or non-shortcut exponent
_UNCOVERED = [(64, 0, 0, 1.0, 1.0), (96, 0, 0, 1.0, 1.0), (3, 0, 4, 1.0, 1.0), (512, 0, 0, 1.0, 1.0),
              (256, 1, 0, 1.0, 1.0), (320, 2, 0, 1.0, 1.0), (128, 2, 4, 1.0, 1.0), (192, 1, 8, 1.0, 1.0),
              (128, 1, 0, 1.5, 1.0), (192, 2, 0, 1.0, 0.7)]


@pytest.mark.parametrize("entry", [_fwd, _bwd])
@pytest.mark.parametrize("C_,dtype,flags,alpha,eps", _UNCOVERED)
def test_rejects_configurations_without_kernels(entry, C_, dtype, flags, alpha, eps):
  _rejects(lambda: entry(C_=C_, dtype=dtype, flags=flags, alpha=alpha, eps=eps), "no kernel")


@pytest.mark.parametrize("entry", [_fwd, _bwd])
def test_the_fp32_switch_rejects_everything(entry, monkeypatch):
  monkeypatch.setenv("TFCB_GDN_FP32", "1")
  _rejects(lambda: entry(), "no kernel")
  _rejects(lambda: entry(C_=256, flags=4 | 8, alpha=1.2, eps=0.9), "no kernel")


@pytest.mark.parametrize("null", range(4))
def test_forward_rejects_null_pointers(null):
  _rejects(lambda: _fwd(ptrs=[None if i == null else _P for i in range(4)]), "null pointer")


@pytest.mark.parametrize("null", [0, 1, 2, 3, 4, 5, 6, 8])
def test_backward_rejects_null_pointers(null):
  _rejects(lambda: _bwd(ptrs=[None if i in (null, 7) else _P for i in range(9)]), "null pointer")


def test_backward_needs_the_exponent_output_with_a_pow_flag():
  _rejects(lambda: _bwd(flags=4, alpha=1.3), "null pointer")
  _rejects(lambda: _bwd(flags=8, eps=0.8), "null pointer")


def test_backward_refuses_an_exponent_output_for_the_shortcut_exponents():
  _rejects(lambda: _bwd(ptrs=[_P] * 9), "must be NULL")


def test_empty_tensors_may_come_with_null_activations_but_not_parameters():
  # accepted arguments reach the device, so only the rejections are exercised here
  _rejects(lambda: _fwd(n=0, ptrs=[None, None, _P, None]), "null pointer")
  _rejects(lambda: _bwd(s=0, ptrs=[None, _P, _P, None, None, None, _P, None, _P]), "null pointer")


@pytest.mark.parametrize("slot", [0, 2, 3])
def test_forward_rejects_unaligned_pointers(slot):
  _rejects(lambda: _fwd(ptrs=[_ODD if i == slot else _P for i in range(4)]), "16-byte aligned")


@pytest.mark.parametrize("slot", [0, 2, 3, 4, 8])
def test_backward_rejects_unaligned_pointers(slot):
  _rejects(lambda: _bwd(ptrs=[None if i == 7 else (_ODD if i == slot else _P) for i in range(9)]),
           "16-byte aligned")


def test_workspace_is_the_channels_last_workspace_of_the_same_pixels():
  """16 bits: the 16-bit backward's workspace; float32: the exponent backward's, followed by the same direct-term
  scratch (none at C = 256 / 320)."""
  L = _lib.lib()
  for n, s, C_ in [(0, 64, 128), (3, 0, 192), (1, 1, 256), (16, 65536, 320), (7, 4103, 128), (5, 999, 192)]:
    n_pix = n * s
    scratch = L.tfcb_gdn_backward_16bit_workspace_bytes(n_pix, C_) - L.tfcb_gdn_backward_workspace_bytes(n_pix, C_)
    assert scratch == 0 if C_ > 192 or n_pix == 0 else scratch > 0
    assert L.tfcb_gdn_backward_cf_workspace_bytes(n, s, C_, 0) == L.tfcb_gdn_backward_exponents_workspace_bytes(
        n_pix, C_) + scratch
    for dtype in (1, 2):
      assert L.tfcb_gdn_backward_cf_workspace_bytes(n, s, C_, dtype) == L.tfcb_gdn_backward_16bit_workspace_bytes(
          n_pix, C_)


@pytest.mark.parametrize("n,s,C_,dtype", [(-1, 4, 128, 0), (4, -1, 128, 0), (4, 4, 0, 0), (4, 4, 128, 3),
                                          (1 << 40, 1 << 20, 128, 0)])
def test_workspace_query_flags_rejected_arguments(n, s, C_, dtype):
  assert _lib.lib().tfcb_gdn_backward_cf_workspace_bytes(n, s, C_, dtype) == -1


# ---- routing: functional._gdn_native_cf ----


def _x(C_=128, dtype=torch.float32, shape=(2, None, 5, 7)):
  return torch.zeros(tuple(C_ if d is None else d for d in shape), dtype=dtype)


@pytest.mark.parametrize("C_", [128, 192, 256, 320])
@pytest.mark.parametrize("alpha,eps,pa,pe", [(1, 1, False, False), (2, 0.5, False, False), (1.5, 0.7, False, False),
                                             (1, 1, True, False), (1, 1, False, True), (1, 1, True, True)])
def test_float32_runs_natively_at_the_four_widths_with_any_exponents(C_, alpha, eps, pa, pe):
  x = _x(C_)
  assert F._gdn_native_cf(x, alpha, eps, pa, pe)
  assert F._gdn_native_cf(x, alpha, eps, pa, pe, dy=torch.zeros_like(x))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("C_", [128, 192])
@pytest.mark.parametrize("alpha,eps", [(1, 1), (2, 0.5), (1, 0.5), (2, 1)])
def test_16bit_runs_natively_at_128_and_192_with_the_shortcuts(dtype, C_, alpha, eps):
  x = _x(C_, dtype)
  assert F._gdn_native_cf(x, alpha, eps, False, False)
  assert F._gdn_native_cf(x, alpha, eps, False, False, dy=torch.zeros_like(x))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_16bit_elsewhere_takes_the_movedim_path(dtype):
  for C_ in (64, 256, 320):
    assert not F._gdn_native_cf(_x(C_, dtype), 1, 1, False, False)
  x = _x(128, dtype)
  assert not F._gdn_native_cf(x, 1.5, 1, False, False)
  assert not F._gdn_native_cf(x, 1, 0.7, False, False)
  assert not F._gdn_native_cf(x, 1, 1, True, False)
  assert not F._gdn_native_cf(x, 1, 1, False, True)


@pytest.mark.parametrize("C_", [3, 64, 96, 127, 129, 384])
def test_other_widths_take_the_movedim_path(C_):
  assert not F._gdn_native_cf(_x(C_), 1, 1, False, False)


def test_other_dtypes_take_the_movedim_path():
  assert not F._gdn_native_cf(_x(dtype=torch.float64), 1, 1, False, False)


@pytest.mark.parametrize("shape", [(2, None, 9), (2, None, 4, 4), (1, None, 2, 3, 4), (0, None, 8, 8),
                                   (3, None, 0, 5)])
def test_ranks_3_to_5_and_empty_tensors_run_natively(shape):
  assert F._gdn_native_cf(_x(shape=shape), 1, 1, False, False)


def test_rank_2_takes_the_channels_last_path():
  assert not F._gdn_native_cf(torch.zeros(10, 128), 1, 1, False, False)


def test_channels_last_memory_format_takes_the_movedim_path():
  x = _x(shape=(2, None, 5, 7)).to(memory_format=torch.channels_last)
  assert x.movedim(1, -1).is_contiguous()
  assert not F._gdn_native_cf(x, 1, 1, False, False)
  assert not F._gdn_native_cf(_x(), 1, 1, False, False, dy=x)


def test_non_contiguous_inputs_take_the_movedim_path():
  x = torch.zeros(2, 128, 6, 8)[..., :7]
  assert not F._gdn_native_cf(x, 1, 1, False, False)
  assert not F._gdn_native_cf(torch.zeros(2, 256, 8)[:, ::2], 1, 1, False, False)
  assert not F._gdn_native_cf(_x(shape=(2, None, 8)), 1, 1, False, False, dy=torch.zeros(2, 8, 128).transpose(1, 2))


def test_unaligned_storage_offsets_take_the_movedim_path():
  buf = torch.zeros(1 + 2 * 128 * 8)
  x = buf[1:].view(2, 128, 8)  # contiguous, 4 bytes past a 16-byte boundary
  assert x.is_contiguous() and x.data_ptr() % 16 != 0
  assert not F._gdn_native_cf(x, 1, 1, False, False)
  assert not F._gdn_native_cf(_x(shape=(2, None, 8)), 1, 1, False, False, dy=x)
  assert F._gdn_native_cf(torch.zeros(4 + 2 * 128 * 8)[4:].view(2, 128, 8), 1, 1, False, False)


def test_backward_needs_dy_in_the_activations_type_and_shape():
  x = _x(dtype=torch.bfloat16)
  assert not F._gdn_native_cf(x, 1, 1, False, False, dy=torch.zeros_like(x, dtype=torch.float32))
  assert not F._gdn_native_cf(x, 1, 1, False, False, dy=torch.zeros_like(x, dtype=torch.float16))
  assert not F._gdn_native_cf(x, 1, 1, False, False, dy=torch.zeros(2, 128, 7, 5, dtype=torch.bfloat16))


def test_exponent_gradients_need_the_literal_pow_kernels():
  x = _x()
  assert F._gdn_native_cf(x, 1, 1, True, False, exponent_grads=True)
  assert F._gdn_native_cf(x, 1.5, 1, False, False, exponent_grads=True)
  assert not F._gdn_native_cf(x, 1, 1, False, False, exponent_grads=True)
  assert not F._gdn_native_cf(x, 2, 0.5, False, False, exponent_grads=True)
  assert not F._gdn_native_cf(_x(dtype=torch.bfloat16), 1, 1, False, False, exponent_grads=True)


def test_fp32_switch_takes_the_movedim_path(monkeypatch):
  x = _x()
  monkeypatch.setenv("TFCB_GDN_FP32", "1")
  assert not F._gdn_native_cf(x, 1, 1, False, False)
  assert not F._gdn_native_cf(x, 1, 1, True, True, dy=torch.zeros_like(x), exponent_grads=True)
  monkeypatch.setenv("TFCB_GDN_FP32", "0")
  assert F._gdn_native_cf(x, 1, 1, False, False)


# ---- host tensors are refused before the library is reached ----


@pytest.fixture
def no_library(monkeypatch):
  """Makes any use of the shared library fail the test."""
  def refuse():
    raise AssertionError("the library was called")
  monkeypatch.setattr(_lib, "lib", refuse)


# a covered configuration (routed natively) and an uncovered one (the movedim path)
@pytest.mark.parametrize("C_", [128, 96])
def test_host_tensors_are_refused_in_both_directions(no_library, C_):
  x, dy = _x(C_), _x(C_)
  gamma, beta = torch.eye(C_), torch.ones(C_)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA tensors"):
    F.gdn_forward(x, gamma, beta, channels_first=True)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA tensors"):
    F.gdn_backward(x, gamma, beta, dy, channels_first=True)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA tensors"):
    F.gdn_backward_exponents(x, gamma, beta, dy, alpha=1.2, epsilon=0.9, channels_first=True)
  with pytest.raises(_lib.InvalidArgumentError, match="CUDA tensors"):
    F.gdn(x, gamma, beta, channels_first=True)


def test_the_channels_first_layer_refuses_host_tensors(no_library):
  from compression_b200.gdn import GDN
  for layer in (GDN(data_format="channels_first"), GDN(inverse=True, data_format="channels_first",
                                                           alpha_parameter=None, epsilon_parameter=None)):
    with pytest.raises(_lib.InvalidArgumentError, match="CUDA tensors"):
      layer(_x())

