"""GPU: the mixture coder (DESIGN.md §3.18) against its oracle and the compiled reference coder.  The device's masses
are held to a float64 bound, its rows to the exact integer map of its own masses, its strings byte for byte to the
reference RangeEncoder on those rows, and its decoder to the reference decoder, also on damaged strings."""
import math

import numpy as np
import pytest
import torch

import oracle
from oracle import mixture_oracle as MO

pytestmark = pytest.mark.gpu

F = pytest.importorskip("compression_b200.functional")
from compression_b200 import _lib, entropy_models, gen_ops  # noqa: E402


def _params(rng, n, K, sigma=(0.05, 1e3), loc_scale=20.0, zero_weights=True):
  w = rng.random((n, K)).astype(np.float32) + np.float32(0.01)
  if zero_weights and K > 1:
    w[rng.random((n, K)) < 0.2] = 0
    w[np.arange(n), rng.integers(0, K, n)] += 1  # never all zero
    dom = rng.random(n) < 0.2
    w[dom, 0] = 1e6  # dominant component
  mu = (rng.standard_normal((n, K)) * loc_scale).astype(np.float32)
  sg = np.exp(rng.uniform(math.log(sigma[0]), math.log(sigma[1]), (n, K))).astype(np.float32)
  return w, mu, sg


def _cuda(*a):
  return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


def _tables(w, mu, sg, family, p, ms, tail_mass=2**-8):
  st, sz, m, rows = F.mixture_tables(*_cuda(w, mu, sg), family=family, precision=p, tail_mass=tail_mass,
                                     max_support=ms)
  return st.cpu().numpy(), sz.cpu().numpy(), m.cpu().numpy(), rows.cpu().numpy()


MATRIX = [(fam, K, p, ms) for fam in MO.FAMILIES for K in (1, 2, 3, 5) for p, ms in
          ((9, 1), (12, 16), (16, 256), (9, 256), (16, 1))]


@pytest.mark.parametrize("family,K,p,ms", MATRIX)
def test_tables_match_the_oracle(family, K, p, ms):
  rng = np.random.default_rng(K * 1000 + p * 10 + ms)
  n = 300
  w, mu, sg = _params(rng, n, K)
  st, sz, m, rows = _tables(w, mu, sg, family, p, ms)
  worst = 0.0
  for e in range(n):
    a, L = MO.support_f32(family, w[e], mu[e], sg[e], 2**-8, ms)
    assert (st[e], sz[e]) == (a, L), e
    assert 1 <= L <= ms
    masses = [int(x) for x in m[e, :L + 1]]
    assert (m[e, L + 1:] == 0).all()
    assert masses[L] == MO.escape_mass(masses[:L])
    c = MO.cdf_from_masses(masses, p)
    assert rows[e, 0] == -p and list(rows[e, 1:L + 3]) == c and (rows[e, L + 3:] == 1 << p).all()
    assert all(c[j + 1] > c[j] for j in range(L + 1)) and c[-1] == 1 << p
    want, bound = MO.masses_bound(family, w[e], mu[e], sg[e], a, L)
    worst = max(worst, float((np.abs(np.asarray(masses[:L], np.float64) - want) / bound).max()))
  assert worst <= 1.0, worst
  print(f"worst mass error / bound: {worst:.3g}")


def _symbols(rng, w, mu, sg):
  k = np.array([rng.choice(len(r), p=r / r.sum()) for r in w.astype(np.float64)])
  i = np.arange(len(w))
  return (mu[i, k] + sg[i, k] * rng.standard_normal(len(w))).astype(np.float32)


def _ref_values(y, st):
  """What the reference codes: int32(rint(y)) - a, wrapping, with NaN -> 0 and saturation."""
  v = np.nan_to_num(np.rint(y.astype(np.float64)), nan=0.0)
  v = np.clip(v, -2**31, 2**31 - 1).astype(np.int64)
  return ((v - st.astype(np.int64) + 2**31) % 2**32 - 2**31).astype(np.int32)


def _ref_encode(lookup, d):
  O = oracle.best()
  enc = O.encoder(lookup, 1)
  enc.encode(d.reshape(1, -1), index=np.arange(d.size, dtype=np.int32).reshape(1, -1))
  return enc.finalize()[0]


def _ref_decode(lookup, s, n):
  O = oracle.best()
  dec = O.decoder([s], lookup)
  return dec.decode(n, index=np.arange(n, dtype=np.int32).reshape(1, -1))[0]


@pytest.mark.parametrize("family,K,p,ms", MATRIX)
def test_strings_equal_the_reference_and_round_trip(family, K, p, ms):
  rng = np.random.default_rng(7 + K * 100 + p + ms)
  n = 400
  w, mu, sg = _params(rng, n, K, sigma=(0.05, 50.0))
  y = _symbols(rng, w, mu, sg)
  y[::37] += np.float32(3000)          # escapes above
  y[5::41] -= np.float32(3000)         # and below
  st, sz, m, rows = _tables(w, mu, sg, family, p, ms)
  d = _ref_values(y, st)
  s = F.mixture_encode_ragged(*_cuda(y, w, mu, sg), [n], family=family, precision=p, max_support=ms)
  got = s.tolist()[0]
  assert got == _ref_encode(rows, d)
  dec = F.mixture_decode_ragged(s, *_cuda(w, mu, sg), [n], family=family, precision=p, max_support=ms)
  want = np.rint(y).astype(np.float32)
  np.testing.assert_array_equal(dec.cpu().numpy(), want)
  np.testing.assert_array_equal(_ref_decode(rows, got, n), d)


def test_saturated_and_non_finite_inputs_round_trip():
  rng = np.random.default_rng(3)
  n = 64
  w, mu, sg = _params(rng, n, 3, sigma=(0.5, 5.0))
  y = _symbols(rng, w, mu, sg)
  y[:8] = [np.nan, np.inf, -np.inf, 3e9, -3e9, 2.0**31, -2.0**31, 1e30]
  s = F.mixture_encode_ragged(*_cuda(y, w, mu, sg), [n])
  dec = F.mixture_decode_ragged(s, *_cuda(w, mu, sg), [n]).cpu().numpy()
  v = np.clip(np.nan_to_num(np.rint(y.astype(np.float64)), nan=0.0), -2**31, 2**31 - 1)
  np.testing.assert_array_equal(dec, v.astype(np.int64).astype(np.float32))
  # the elements whose payload the reference can code match it byte for byte
  st, sz, m, rows = _tables(w, mu, sg, "normal", 16, 256)
  y2 = y.copy()
  y2[:8] = [np.nan, 0, 0, 0, 0, 0, 0, 0]
  s2 = F.mixture_encode_ragged(*_cuda(y2, w, mu, sg), [n])
  assert s2.tolist()[0] == _ref_encode(rows, _ref_values(y2, st))


def test_ragged_lists_empty_and_one_element_streams_and_1025_streams():
  rng = np.random.default_rng(11)
  lengths = [0, 1, 33, 0, 257, 5] + [int(x) for x in rng.integers(0, 9, 1025 - 6)]
  n = sum(lengths)
  w, mu, sg = _params(rng, n, 3, sigma=(0.1, 20.0))
  y = _symbols(rng, w, mu, sg)
  y[::53] += np.float32(500)
  s = F.mixture_encode_ragged(*_cuda(y, w, mu, sg), lengths).tolist()
  st, sz, m, rows = _tables(w, mu, sg, "normal", 16, 256)
  d = _ref_values(y, st)
  at = 0
  for i, k in enumerate(lengths):
    if i < 40 or i % 97 == 0:
      one = F.mixture_encode_ragged(*_cuda(y[at:at + k], w[at:at + k], mu[at:at + k], sg[at:at + k]), [k]).tolist()[0]
      assert s[i] == one, i
      assert s[i] == _ref_encode(rows[at:at + k] if k else rows[:1], d[at:at + k]) if k else s[i] == b""
    at += k
  dec = F.mixture_decode_ragged(s, *_cuda(w, mu, sg), lengths).cpu().numpy()
  np.testing.assert_array_equal(dec, np.rint(y))


@pytest.mark.parametrize("kind", ["truncated", "flipped", "random"])
def test_damaged_strings_decode_as_the_reference(kind):
  rng = np.random.default_rng({"truncated": 1, "flipped": 2, "random": 3}[kind])
  n = 500
  w, mu, sg = _params(rng, n, 2, sigma=(0.3, 10.0), zero_weights=False)
  y = _symbols(rng, w, mu, sg)
  s = F.mixture_encode_ragged(*_cuda(y, w, mu, sg), [n]).tolist()[0]
  st, sz, m, rows = _tables(w, mu, sg, "normal", 16, 256)
  for trial in range(6):
    b = bytearray(s)
    if kind == "truncated":
      b = b[:int(rng.integers(0, len(b)))]
    elif kind == "flipped":
      for _ in range(1 + trial):
        i = int(rng.integers(0, len(b)))
        b[i] ^= 1 << int(rng.integers(0, 8))
    else:
      b = bytearray(rng.integers(0, 256, int(rng.integers(0, 2 * len(s)))).astype(np.uint8).tobytes())
    got = F.mixture_decode_ragged([bytes(b)], *_cuda(w, mu, sg), [n]).cpu().numpy()
    want = _ref_decode(rows, bytes(b), n).astype(np.int64) + st
    want = ((want + 2**31) % 2**32 - 2**31).astype(np.float32)
    np.testing.assert_array_equal(got, want)


def test_substreams_decode_to_the_same_values_and_cost_at_most_the_header_and_4_bytes_per_stream():
  rng = np.random.default_rng(5)
  em = entropy_models.MixtureEntropyModel("logistic", coding_rank=3)
  shape, K = (2, 12, 10, 8), 3
  n = int(np.prod(shape))
  w, mu, sg = _params(rng, n, K, sigma=(0.2, 8.0))
  y = _symbols(rng, w, mu, sg).reshape(shape)
  W, M, S_ = (torch.from_numpy(x.reshape(shape + (K,))).cuda() for x in (w, mu, sg))
  yt = torch.from_numpy(y).cuda()
  one = em.compress(yt, W, M, S_)
  np.testing.assert_array_equal(em.decompress(one, W, M, S_).cpu().numpy(), np.rint(y))
  for S in (2, 7):
    many = em.compress(yt, W, M, S_, substreams=S)
    np.testing.assert_array_equal(em.decompress(many, W, M, S_, substreams=S).cpu().numpy(), np.rint(y))
    for a, b in zip(one.tolist(), many.tolist()):
      parts = gen_ops.parse_substreams(b, S)
      header = len(b) - sum(len(x) for x in parts)
      assert len(b) <= len(a) + header + 4 * S


def test_ragged_model_strings_equal_the_one_image_strings_and_launch_counts_do_not_depend_on_items():
  rng = np.random.default_rng(9)
  em = entropy_models.MixtureEntropyModel("normal", coding_rank=3)
  K = 3
  shapes = [(4, 5, 6), (1, 1, 6), (7, 3, 6), (2, 9, 6)]
  items = []
  for sh in shapes:
    n = int(np.prod(sh))
    w, mu, sg = _params(rng, n, K, sigma=(0.2, 8.0))
    y = _symbols(rng, w, mu, sg).reshape(sh)
    items.append(tuple(torch.from_numpy(x.reshape(sh + ((K,) if x is not y else ()))).cuda()
                       for x in (y, w, mu, sg)))
  ys, ws, ls, ss = (list(t) for t in zip(*items))
  counts = {}
  for k in (1, len(items)):
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    strings = em.compress_ragged(ys[:k], ws[:k], ls[:k], ss[:k])
    n1 = _lib.launch_count()
    out = em.decompress_ragged(strings, ws[:k], ls[:k], ss[:k])
    counts[k] = (n1 - n0, _lib.launch_count() - n1)
  assert counts[1] == counts[len(items)], counts
  for i, (y, w, l, s) in enumerate(items):
    assert strings.tolist()[i] == em.compress(y[None], w[None], l[None], s[None]).tolist()[0]
    np.testing.assert_array_equal(out[i].cpu().numpy(), np.rint(y.cpu().numpy()))
  batch = em.compress(torch.stack([ys[0], ys[0]]), torch.stack([ws[0], ws[0]]), torch.stack([ls[0], ls[0]]),
                      torch.stack([ss[0], ss[0]])).tolist()
  assert batch[0] == batch[1] == strings.tolist()[0]


@pytest.mark.parametrize("family", MO.FAMILIES)
def test_string_length_is_within_1_percent_and_4_bytes_of_the_information_content(family):
  rng = np.random.default_rng(13)
  em = entropy_models.MixtureEntropyModel(family, coding_rank=1)
  B, n, K = 4, 5000, 3
  w, mu, sg = _params(rng, B * n, K, sigma=(0.5, 10.0))
  y = _symbols(rng, w, mu, sg).reshape(B, n)
  W, M, S_ = (torch.from_numpy(x.reshape(B, n, K)).cuda() for x in (w, mu, sg))
  _, bits = em(torch.from_numpy(y).cuda(), W, M, S_, training=False)
  strings = em.compress(torch.from_numpy(y).cuda(), W, M, S_)
  for s, b in zip(strings.tolist(), bits.cpu().numpy()):
    assert 8 * len(s) <= b * 1.01 + 32, (len(s), b / 8)


def test_forward_matches_the_mixture_graph():
  rng = np.random.default_rng(17)
  em = entropy_models.MixtureEntropyModel("normal", coding_rank=2)
  w, mu, sg = _params(rng, 60, 3, sigma=(0.5, 4.0))
  W, M, S_ = (torch.from_numpy(x.reshape(3, 4, 5, 3)).cuda() for x in (w, mu, sg))
  y = torch.from_numpy(_symbols(rng, w, mu, sg).reshape(3, 4, 5)).cuda()
  from compression_b200 import distributions as D
  prior = D.NoisyNormalMixture(M, S_, W / W.sum(-1, keepdim=True))
  yq, bits = em(y, W, M, S_, training=False)
  torch.testing.assert_close(yq, torch.round(y))
  torch.testing.assert_close(bits, prior.log_prob(torch.round(y)).sum((-2, -1)) / -math.log(2.0))
  yn, bits_t = em(y, W, M, S_, training=True)
  assert bits_t.shape == (3,) and ((yn - y).abs() <= 0.5).all()


@pytest.mark.parametrize("bad,what", [("nan_loc", "non-finite"), ("scale", "scale <= 0"), ("weight", "negative"),
                                      ("zero", "all weights 0")])
def test_bad_parameters_name_the_lowest_failing_string_and_element(bad, what):
  rng = np.random.default_rng(19)
  n = 100
  w, mu, sg = _params(rng, n, 2, zero_weights=False)
  e = 57
  if bad == "nan_loc":
    mu[e, 1] = np.nan
  elif bad == "scale":
    sg[e, 0] = 0
  elif bad == "weight":
    w[e, 1] = -1
  else:
    w[e] = 0
  y = np.zeros(n, np.float32)
  for fn in (lambda: F.mixture_encode_ragged(*_cuda(y, w, mu, sg), [50, 50]),
             lambda: F.mixture_decode_ragged([b"", b""], *_cuda(w, mu, sg), [50, 50])):
    with pytest.raises(_lib.InvalidArgumentError, match=f"{what}.*string 1, element 7"):
      fn()


# ---- host synchronisations: counted in the CUDA runtime trace (the library's own calls included) ----
_SYNCS = ("cudaStreamSynchronize", "cudaDeviceSynchronize", "cudaEventSynchronize", "cudaMemcpy")
_LAUNCHES = ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx")


def _runtime_calls(fn):
  """(result, host synchronisations, kernel launches) of fn() in the CUDA runtime trace, less those of an empty call
  (profiler start and stop).  torch's own synchronising calls raise (sync debug mode)."""
  from torch.profiler import ProfilerActivity, profile

  def trace(f):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
      torch.cuda.set_sync_debug_mode("error")
      try:
        out = f()
      finally:
        torch.cuda.set_sync_debug_mode(0)
    names = [e.name for e in prof.events()]
    return out, sum(n in _SYNCS for n in names), sum(n in _LAUNCHES for n in names)
  _, s0, l0 = trace(lambda: None)
  out, s, l = trace(fn)
  return out, s - s0, l - l0


def test_each_call_makes_exactly_one_host_synchronisation():
  rng = np.random.default_rng(23)
  lengths = [40, 0, 300, 7]
  n = sum(lengths)
  w, mu, sg = _params(rng, n, 3, sigma=(0.3, 10.0))
  y = _symbols(rng, w, mu, sg)
  y[::31] += np.float32(900)
  yd, wd, md, sd = _cuda(y, w, mu, sg)
  F.mixture_encode_ragged(yd, wd, md, sd, lengths)  # (warm: first-use set-up)
  strings, syncs, launches = _runtime_calls(lambda: F.mixture_encode_ragged(yd, wd, md, sd, lengths))
  assert syncs == 1 and launches >= 3, (syncs, launches)
  F.mixture_decode_ragged(strings, wd, md, sd, lengths)
  out, syncs, launches = _runtime_calls(lambda: F.mixture_decode_ragged(strings, wd, md, sd, lengths))
  assert syncs == 1 and launches >= 1, (syncs, launches)
  np.testing.assert_array_equal(out.cpu().numpy(), np.rint(y))


# ---- MixtureHyperpriorModel ----
from compression_b200 import distributions as D  # noqa: E402
from compression_b200 import models  # noqa: E402


def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  out = []
  for h, w in sizes:
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 60 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None] * np.array([1.0, 0.7, 0.4])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)))
  return out


@pytest.fixture(scope="module", params=["normal", "logistic"])
def model(request):
  torch.manual_seed(0)
  return models.MixtureHyperpriorModel(num_filters=16, latent_depth=12, num_components=3,
                                       family=request.param).build("cuda", patch=(64, 64)).fix_tables()


def test_model_forward_matches_the_mixture_graph(model):
  x = _images([(64, 48)], 1)[0][None].cuda().float()
  with torch.no_grad():
    loss, bpp, mse = model(x, training=False)
    y = model.analysis_transform(x)
    z = model.hyper_analysis_transform(y)
    side = model.side_entropy_model
    z_hat, side_bits = side(z, training=False)
    psi = model.hyper_synthesis_transform(z_hat)[:, :y.shape[1], :y.shape[2], :]
    K, M = 3, 12
    p = psi.reshape(psi.shape[:-1] + (M, 3, K))
    w, l, s = torch.softmax(p[..., 0, :], -1), p[..., 1, :], torch.clamp(p[..., 2, :], min=.11)
    cls = D.NoisyNormalMixture if model.family == "normal" else D.NoisyLogisticMixture
    bits = cls(l, s, w / w.sum(-1, keepdim=True)).log_prob(torch.round(y)).sum() / -math.log(2.0)
    want_bpp = (bits + side_bits.sum()) / (64 * 48)
  torch.testing.assert_close(bpp, want_bpp)
  xt = x.clone().requires_grad_(False)
  loss_t, _, _ = model(xt, training=True)
  assert torch.isfinite(loss_t)


def test_model_round_trip_is_exact_and_the_string_does_not_depend_on_the_batch(model):
  x = _images([(64, 80)], 3)[0]
  item = model.compress(x)
  got = model.decompress(*item)
  with torch.no_grad():
    y = model.analysis_transform(x[None].cuda().float())
    want = torch.clamp(torch.round(model.synthesis_transform(torch.round(y))), 0, 255).to(torch.uint8)[0, :64, :80]
  assert torch.equal(got, want)
  batch = model.compress_batch(torch.stack([x, _images([(64, 80)], 4)[0], x]))
  assert batch[0].tolist()[0] == batch[0].tolist()[2] == item[0].tolist()[0]
  assert batch[1].tolist()[0] == item[1].tolist()[0]
  assert torch.equal(model.decompress_batch(*batch)[2], got)


def test_model_compress_images_matches_the_one_image_strings_and_tfci_and_evaluate_work(model):
  images = _images([(64, 80), (40, 56), (17, 33)], 5)
  items = model.compress_images(images)
  for x, it in zip(images, items):
    one = model.compress(x)
    assert it[0].tolist() == one[0].tolist() and it[1].tolist() == one[1].tolist()
  outs = model.decompress_images(items)
  for x, out in zip(images, outs):
    assert torch.equal(out, model.decompress(*model.compress(x)))
    assert torch.equal(model.decompress_from_tfci(model.compress_to_tfci(x)), out)
  big = _images([(176, 192), (184, 176)], 8)  # (MS-SSIM's five scales need 176 pixels a side)
  ev = [model.evaluate(x) for x in big]
  evs = model.evaluate_images(big)
  for a, b in zip(ev, evs):
    assert a["bpp"] == b["bpp"] and a["msssim"] == b["msssim"]
    assert math.isfinite(a["psnr"])


def test_model_substreams_decode_to_the_same_image(model):
  x = _images([(64, 80)], 6)[0]
  want = model.decompress(*model.compress(x))
  m4 = models.MixtureHyperpriorModel(num_filters=16, latent_depth=12, num_components=3, family=model.family,
                                     substreams=4).build("cuda", patch=(64, 64))
  m4.load_state_dict(model.state_dict(), strict=False)
  m4.fix_tables()
  assert torch.equal(m4.decompress(*m4.compress(x)), want)
  items = m4.compress_images(_images([(64, 80), (40, 56)], 7))
  assert len(m4.decompress_images(items)) == 2


def test_tiny_weight_sums_are_rejected():
  w = np.full((4, 2), 1e-40, np.float32)
  mu = np.zeros((4, 2), np.float32)
  sg = np.ones((4, 2), np.float32)
  with pytest.raises(_lib.InvalidArgumentError, match="too small to normalise.*string 0, element 0"):
    F.mixture_encode_ragged(*_cuda(np.zeros(4, np.float32), w, mu, sg), [4])
