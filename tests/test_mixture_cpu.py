"""CPU: the mixture coder's exact integer map from masses to the quantised CDF (oracle.mixture_oracle) at its edges,
and the host-side rejections of the C ABI and of MixtureEntropyModel, which all happen before any device work."""
import concurrent.futures
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from oracle import mixture_oracle as MO
from compression_b200 import _lib, entropy_models

TWO32 = 1 << 32


def _check_row(masses, p):
  c = MO.cdf_from_masses(masses, p)
  assert c[0] == 0 and c[-1] == 1 << p and len(c) == len(masses) + 1
  assert all(b - a >= 1 for a, b in zip(c, c[1:]))
  lookup = MO.lookup([c], p, len(masses) - 1)
  enc = oracle.port().encoder(lookup, 1)  # parses the row with the reference's lookup grammar
  enc.close()
  return c


@pytest.mark.parametrize("p", [1, 9, 12, 16])
def test_integer_map_edges(p):
  L = min(5, (1 << p) - 1)
  _check_row([0] * L + [TWO32], p)                        # all mass in the escape
  _check_row([TWO32 - 1] + [0] * (L - 1) + [1], p)        # all mass in one bin
  _check_row([TWO32 - 1] * L + [MO.escape_mass([TWO32 - 1] * L)], p)  # sum above 2^32: no escape mass
  assert MO.escape_mass([TWO32 - 1] * 2) == 0
  _check_row([0, MO.escape_mass([0])], p)                 # L = 1
  n = (1 << p) - 1                                        # n = 2^p - 1 bins: every bin 1 or 2
  if n >= 2:
    c = _check_row([TWO32 // n] * (n - 1) + [MO.escape_mass([TWO32 // n] * (n - 1))], p)
    assert max(b - a for a, b in zip(c, c[1:])) <= 2


def test_integer_map_fuzzed():
  rng = np.random.default_rng(0)
  for _ in range(300):
    p = int(rng.integers(1, 17))
    L = int(rng.integers(1, min(256, (1 << p) - 1) + 1))
    m = [int(x) for x in rng.integers(0, TWO32, L) * (rng.random(L) < 0.7) // int(rng.integers(1, L + 1))]
    _check_row(m + [MO.escape_mass(m)], p)


def test_integer_map_matches_the_formula_with_python_ints():
  m = [3, 0, 7, TWO32 - 10]
  c = MO.cdf_from_masses(m, 4)
  T = sum(m)
  assert c == [0] + [j + (16 - 4) * sum(m[:j]) // T for j in range(1, 5)]


def test_support_emulation_clips_around_the_rounded_mean():
  a, L = MO.support_f32("normal", [1.0, 1.0], [0.0, 1000.0], [1.0, 1.0], 2**-8, 256)
  assert (a, L) == (500 - 127, 256)
  a, L = MO.support_f32("logistic", [1.0], [2.3], [0.05], 2**-8, 16)
  assert L >= 1 and a <= 2 and a + L - 1 >= 2


# ---- ABI rejections: every call is refused on the host, so no pointer is dereferenced and nothing launches ----
_P = C.c_void_p(256)


def _on_worker(fn):
  with concurrent.futures.ThreadPoolExecutor(1) as ex:
    return ex.submit(fn).result()


def _call(entry, K=3, family=0, p=16, tail=2**-8, ms=256, items=(0, 4), null=None):
  it = np.asarray(items, np.int64)
  ptr = [None if i == null else _P for i in range(5)]
  L = _lib.lib()
  h, total = C.c_void_p(), C.c_int64(0)
  if entry == "encode":
    return L.tfcb_mixture_encode_ragged(ptr[0], ptr[1], ptr[2], ptr[3], K, family, p, tail, ms, it.size - 1,
                                        it.ctypes.data_as(C.c_void_p), ptr[4], None, C.byref(h), C.byref(total))
  if entry == "decode":
    return L.tfcb_mixture_decode_ragged(ptr[0], _P, it.size - 1, it.ctypes.data_as(C.c_void_p), ptr[1], ptr[2],
                                        ptr[3], K, family, p, tail, ms, ptr[4], None)
  return L.tfcb_mixture_tables(ptr[0], ptr[1], ptr[2], int(it[-1]), K, family, p, tail, ms, ptr[3], ptr[4], _P, _P,
                               None)


CASES = [
    (dict(family=2), "`family` must be 0"),
    (dict(K=0), "`K` must be in"),
    (dict(K=65), "`K` must be in"),
    (dict(ms=0), "`max_support` must be in"),
    (dict(ms=257), "`max_support` must be in"),
    (dict(p=0), "`precision` must be in"),
    (dict(p=17), "`precision` must be in"),
    (dict(p=8, ms=256), "2\\^precision > max_support"),
    (dict(tail=0.0), "`tail_mass` must be in"),
    (dict(tail=1.0), "`tail_mass` must be in"),
    (dict(tail=float("nan")), "`tail_mass` must be in"),
    (dict(null=0), "null pointer"),
    (dict(null=2), "null pointer"),
    (dict(null=4), "null pointer"),
]
ITEM_CASES = [
    (dict(items=(1, 3)), "symbol_offsets\\[0\\] must be 0"),
    (dict(items=(0, 3, 2)), "non-decreasing"),
    (dict(items=(0,)), "`n_streams` must be positive"),
]


@pytest.mark.parametrize("entry", ["tables", "encode", "decode"])
@pytest.mark.parametrize("kw,msg", CASES + ITEM_CASES, ids=lambda x: str(x))
def test_abi_rejects_before_any_launch(entry, kw, msg):
  if entry == "tables" and "items" in kw:
    pytest.skip("the tables entry takes an element count, not item offsets")
  n0 = _lib.launch_count()

  def run():
    rc = _call(entry, **kw)
    return rc, _lib.lib().tfcb_last_error().decode()
  rc, err = _on_worker(run)
  assert rc == _lib.INVALID_ARGUMENT
  assert __import__("re").search(msg, err), err
  assert _lib.launch_count() == n0


# ---- the entropy model's host checks ----
def test_model_constructor_checks():
  with pytest.raises(ValueError, match="family"):
    entropy_models.MixtureEntropyModel("laplace")
  with pytest.raises(ValueError, match="tail_mass"):
    entropy_models.MixtureEntropyModel(tail_mass=1.0)
  with pytest.raises(ValueError, match="max_support"):
    entropy_models.MixtureEntropyModel(max_support=300)
  with pytest.raises(ValueError, match="range_coder_precision"):
    entropy_models.MixtureEntropyModel(range_coder_precision=8, max_support=256)
  with pytest.raises(ValueError, match="coding_rank"):
    entropy_models.MixtureEntropyModel(coding_rank=-1)


def test_model_rejects_other_dtypes_and_shapes_before_the_device():
  em = entropy_models.MixtureEntropyModel(coding_rank=1)
  y = torch.zeros(2, 3)
  w = torch.ones(2, 3, 4)
  with pytest.raises(ValueError, match="float32 only"):
    em.compress(y.double(), w, w, w)
  with pytest.raises(ValueError, match="float32 only"):
    em.compress(y, w.half(), w, w)
  with pytest.raises(ValueError, match="share one shape"):
    em.compress(y, w, w[..., :2], w)
  with pytest.raises(ValueError, match="plus the components"):
    em.compress(y[:1], w, w, w)
  with pytest.raises(ValueError, match="coding_rank"):
    entropy_models.MixtureEntropyModel(coding_rank=3).compress(y, w, w, w)
  with pytest.raises(ValueError, match="float32 only"):
    em(y.double(), w, w, w)


def test_model_ragged_calls_reject_mixed_components_and_empty_lists():
  em = entropy_models.MixtureEntropyModel(coding_rank=1)
  ys = [torch.zeros(2, 6), torch.zeros(2, 9)]
  ws = [torch.ones(2, 6, 3), torch.ones(2, 9, 2)]  # 36 parameters each: only K tells them apart
  with pytest.raises(ValueError, match="same number of components"):
    em.compress_ragged(ys, ws, ws, ws)
  with pytest.raises(ValueError, match="same number of components"):
    em.decompress_ragged([b"", b""], ws, ws, ws)
  with pytest.raises(ValueError, match="at least one item"):
    em.decompress_ragged([], [], [], [])
  with pytest.raises(ValueError, match="at least one item"):
    em.compress_ragged([], [], [], [])


def test_mixture_model_constructor_checks():
  from compression_b200 import models
  with pytest.raises(ValueError, match="latent_depth"):
    models.MixtureHyperpriorModel(latent_depth=7)
  with pytest.raises(ValueError, match="num_components"):
    models.MixtureHyperpriorModel(num_components=0)
  with pytest.raises(ValueError, match="family"):
    models.MixtureHyperpriorModel(family="laplace")
  m = models.MixtureHyperpriorModel(num_filters=8, latent_depth=4, num_components=2)
  assert m.hyper_synthesis_transform[2].filters == 3 * 2 * 4
