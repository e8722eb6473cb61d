"""CPU: which calls of UniformNoiseAdapter.log_prob the fused kernels take (routing decided from dtypes, shapes and the
device), that everything else is the graph bit for bit, and the host-side rejections of the new C entries."""
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import distributions as D


def _df(batch_shape=(4,), **kw):
  return D.NoisyDeepFactorized(batch_shape=batch_shape, **kw)


def test_deep_factorized_form():
  p = _df((4,))
  y = torch.zeros(2, 3, 4)
  assert D._fused_log_prob_form(p.base, y) == "deep_factorized"
  assert D._fused_log_prob_form(_df(()).base, y) == "deep_factorized"  # C = 1
  assert D._fused_log_prob_form(_df((3, 4)).base, y) == "deep_factorized"  # trailing dims [3, 4]
  assert D._fused_log_prob_form(p.base, torch.zeros(4)) == "deep_factorized"
  assert D._fused_log_prob_form(p.base, y.double()) is None
  assert D._fused_log_prob_form(_df((4,), dtype=torch.float64).base, y) is None
  assert D._fused_log_prob_form(_df((4,), num_filters=(3, 3, 3)).base, y) is None
  assert D._fused_log_prob_form(_df((4,), num_filters=(4, 3)).base, y) is None
  assert D._fused_log_prob_form(p.base, torch.zeros(4, 3)) is None            # channel not the trailing dim
  assert D._fused_log_prob_form(_df((2, 4)).base, torch.zeros(4)) is None      # fewer dims than the batch shape
  assert D._fused_log_prob_form(p.base, torch.zeros(4, 2, 3).permute(1, 2, 0)) is None  # not contiguous
  assert D._fused_log_prob_form(p.base, torch.zeros(2, 1)) is None             # broadcasts in the graph


def test_location_scale_form():
  y = torch.zeros(2, 5)
  full = torch.rand(2, 5) + 0.5
  for cls, kind in ((D.NoisyNormal, "normal"), (D.NoisyLogistic, "logistic"), (D.NoisyLaplace, "laplace")):
    assert D._fused_log_prob_form(cls(full, full).base, y) == kind
    assert D._fused_log_prob_form(cls(0., full).base, y) == kind                 # loc a broadcast scalar
    assert D._fused_log_prob_form(cls(torch.zeros(()), torch.ones(()), ).base, y) is None  # 0-d: y broadcasts
    assert D._fused_log_prob_form(cls(full, torch.ones(5)).base, y) is None      # scale broadcast along one dim
    assert D._fused_log_prob_form(cls(full.t().contiguous().t(), full).base, y) is None  # not contiguous
    assert D._fused_log_prob_form(cls(full, full, dtype=torch.float64).base, y.double()) is None
    assert D._fused_log_prob_form(cls(full, full).base, y.double()) is None
    assert D._fused_log_prob_form(cls(full, full).base, torch.zeros(5)) is None


def test_other_priors_are_not_routed():
  y = torch.zeros(2, 4)
  assert D._fused_log_prob_form(D.NoisyRoundedNormal(0., torch.ones(2, 4)).base, y) is None
  assert D._fused_log_prob_form(D.NoisySoftRoundedNormal(loc=torch.zeros(2, 4), scale=torch.ones(2, 4)).base, y) is None
  assert D._fused_log_prob_form(D.NoisyRoundedDeepFactorized(batch_shape=(4,)).base, y) is None
  assert D._fused_log_prob_form(D.NoisySoftRoundedDeepFactorized(batch_shape=(4,)).base, y) is None


def test_cpu_tensors_run_the_graph_bit_for_bit():
  torch.manual_seed(0)
  y = torch.randn(3, 4) * 3
  p = _df((4,))
  assert D._fused_log_prob_form(p.base, y) == "deep_factorized"
  assert D._fused_log_prob_kind(p.base, y) is None
  assert torch.equal(p.log_prob(y), p._log_prob_graph(y))
  q = D.NoisyNormal(torch.randn(3, 4), torch.rand(3, 4) + 0.2)
  assert D._fused_log_prob_kind(q.base, y) is None
  assert torch.equal(q.log_prob(y), q._log_prob_graph(y))


def test_packed_parameters_layout():
  p = _df((5,))
  with torch.no_grad():
    for t in p.parameters():
      t.copy_(torch.randn_like(t))
  b = p.base
  packed = b._packed_parameters()
  assert packed.shape == (5, 28)
  sp, th = torch.nn.functional.softplus, torch.tanh
  want = torch.cat([sp(b.matrices[0]).reshape(5, 3), sp(b.matrices[1]).reshape(5, 9), sp(b.matrices[2]).reshape(5, 3),
                    b.biases[0].reshape(5, 3), b.biases[1].reshape(5, 3), b.biases[2].reshape(5, 1),
                    th(b.factors[0]).reshape(5, 3), th(b.factors[1]).reshape(5, 3)], 1)
  assert torch.equal(packed, want)
  assert b.matrices[1].shape == (5, 3, 3)  # [channel, out, in]: row-major [out][in] per channel


def test_new_entries_reject_bad_arguments_before_device_work():
  lib = _lib.lib()
  fake = 0x1000  # never dereferenced: every call below fails its host-side checks first
  with pytest.raises(_lib.InvalidArgumentError, match="bad deep-factorized shape"):
    _lib.check(lib.tfcb_noisy_deep_factorized_log_prob(fake, fake, fake, 8, 0, None))
  with pytest.raises(_lib.InvalidArgumentError, match="bad deep-factorized shape"):
    _lib.check(lib.tfcb_noisy_deep_factorized_log_prob(fake, fake, fake, -4, 4, None))
  with pytest.raises(_lib.InvalidArgumentError, match="not a multiple"):
    _lib.check(lib.tfcb_noisy_deep_factorized_log_prob(fake, fake, fake, 10, 4, None))
  for args in ((None, fake, fake), (fake, None, fake), (fake, fake, None)):
    with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
      _lib.check(lib.tfcb_noisy_deep_factorized_log_prob(*args, 8, 4, None))
  with pytest.raises(_lib.InvalidArgumentError, match="bad deep-factorized shape"):
    _lib.check(lib.tfcb_noisy_deep_factorized_log_prob_backward(fake, fake, fake, fake, fake, fake, 8, -1, None))
  with pytest.raises(_lib.InvalidArgumentError, match="not a multiple"):
    _lib.check(lib.tfcb_noisy_deep_factorized_log_prob_backward(fake, fake, fake, fake, fake, fake, 9, 2, None))
  for i in range(6):
    args = [fake] * 6
    args[i] = None
    with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
      _lib.check(lib.tfcb_noisy_deep_factorized_log_prob_backward(*args, 8, 4, None))
  assert lib.tfcb_noisy_deep_factorized_workspace_bytes(0, 4) == 0
  assert lib.tfcb_noisy_deep_factorized_workspace_bytes(8, 0) == 0
  assert lib.tfcb_noisy_deep_factorized_workspace_bytes(1 << 20, 128) % (128 * 28 * 4) == 0

  for base in (-1, 3):
    with pytest.raises(_lib.InvalidArgumentError, match="unknown location-scale base"):
      _lib.check(lib.tfcb_noisy_loc_scale_log_prob(base, fake, fake, 0, fake, 0, fake, 8, None))
    with pytest.raises(_lib.InvalidArgumentError, match="unknown location-scale base"):
      _lib.check(lib.tfcb_noisy_loc_scale_log_prob_backward(base, fake, fake, 0, fake, 0, fake, fake, None, None, 8,
                                                            None))
  with pytest.raises(_lib.InvalidArgumentError, match="bad location-scale size"):
    _lib.check(lib.tfcb_noisy_loc_scale_log_prob(0, fake, fake, 0, fake, 0, fake, -1, None))
  for i in range(4):
    args = [fake] * 4
    args[i] = None
    with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
      _lib.check(lib.tfcb_noisy_loc_scale_log_prob(1, args[0], args[1], 0, args[2], 1, args[3], 8, None))
  for i in range(5):
    args = [fake] * 5
    args[i] = None
    with pytest.raises(_lib.InvalidArgumentError, match="null pointer"):
      _lib.check(lib.tfcb_noisy_loc_scale_log_prob_backward(2, args[0], args[1], 0, args[2], 0, args[3], args[4],
                                                            None, None, 8, None))
