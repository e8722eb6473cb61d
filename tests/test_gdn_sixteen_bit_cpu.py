"""CPU: which 16-bit GDN calls take the native kernels (functional._gdn_native16).  The predicate looks at dtypes,
shapes, pointers and the environment only, so host tensors stand in for device ones."""
import pytest
import torch

from compression_b200 import functional as F


def _x(C=128, n=10, dtype=torch.bfloat16):
  return torch.zeros(n, C, dtype=dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("C", [128, 192])
@pytest.mark.parametrize("alpha,epsilon", [(1, 1), (2, 0.5), (1, 0.5), (2, 1)])
def test_native_configurations(dtype, C, alpha, epsilon):
  x = _x(C, dtype=dtype)
  assert F._gdn_native16(x, C, 10, alpha, epsilon, False, False)
  assert F._gdn_native16(x, C, 10, alpha, epsilon, False, False, dy=torch.zeros_like(x))


@pytest.mark.parametrize("C", [3, 64, 256, 320])
def test_other_widths_convert(C):
  assert not F._gdn_native16(_x(C), C, 10, 1, 1, False, False)


def test_float32_and_exponents_and_empty_convert():
  assert not F._gdn_native16(_x(dtype=torch.float32), 128, 10, 1, 1, False, False)
  assert not F._gdn_native16(_x(), 128, 10, 1.5, 1, False, False)
  assert not F._gdn_native16(_x(), 128, 10, 1, 0.7, False, False)
  assert not F._gdn_native16(_x(), 128, 10, 1, 1, True, False)
  assert not F._gdn_native16(_x(), 128, 10, 1, 1, False, True)
  assert not F._gdn_native16(_x(n=0), 128, 0, 1, 1, False, False)


def test_backward_needs_dy_in_the_activations_type_and_shape():
  x = _x()
  assert not F._gdn_native16(x, 128, 10, 1, 1, False, False, dy=torch.zeros(10, 128))
  assert not F._gdn_native16(x, 128, 10, 1, 1, False, False, dy=torch.zeros(10, 128, dtype=torch.float16))
  assert not F._gdn_native16(x, 128, 10, 1, 1, False, False, dy=torch.zeros(5, 256, dtype=torch.bfloat16))


def test_unaligned_tensors_convert():
  buf = torch.zeros(11 * 128, dtype=torch.bfloat16)
  x = buf[1:1 + 10 * 128].view(10, 128)  # 2 bytes past a 16-byte boundary
  assert x.data_ptr() % 16 != 0
  assert not F._gdn_native16(x, 128, 10, 1, 1, False, False)
  assert not F._gdn_native16(_x(), 128, 10, 1, 1, False, False, dy=x)


def test_fp32_switch_converts_both_directions(monkeypatch):
  x = _x()
  monkeypatch.setenv("TFCB_GDN_FP32", "1")
  assert not F._gdn_native16(x, 128, 10, 1, 1, False, False)
  assert not F._gdn_native16(x, 128, 10, 1, 1, False, False, dy=torch.zeros_like(x))
  monkeypatch.setenv("TFCB_GDN_FP32", "0")
  assert F._gdn_native16(x, 128, 10, 1, 1, False, False)
