"""GPU: the space-channel multistage context model (SpaceChannelMultistageModel, functional.mscc_*).  Every stage of
every group equals the float32 emulation bit for bit, the one-group passes are tfcb_msc_params and the one-group
strings MultistageModel's, stage 0 is the space-channel anchor pass, the encoder is the emulated group-by-group,
stage-by-stage encoder, rows do not depend on the batch, the strings are the entropy model's of the coding-order
tensors, the 4K-call decoder returns the encoder's latents without host synchronisation in a fixed number of
launches, substreams decode to the same latents, and the model's coding calls fit together."""
import math

import numpy as np
import pytest
import torch

from compression_b200 import _lib
from compression_b200 import distributions as D
from compression_b200 import entropy_models as E
from compression_b200 import functional as F
from compression_b200 import gen_ops
from compression_b200 import models
from oracle import checkerboard_oracle as cbo
from oracle import multistage_oracle as mso
from oracle import space_channel_multistage_oracle as scmo

pytestmark = pytest.mark.gpu

NUM_SCALES = 64
SHAPES = [(1, 1), (1, 9), (7, 1), (2, 2), (3, 5), (32, 48)]
DEFAULT = (16, 16, 32, 64, 192)


@pytest.fixture(scope="module")
def em():
  scale_fn = models.BMSHJ2018Model(num_filters=24).scale_fn
  return E.LocationScaleIndexedEntropyModel(D.NoisyNormal, NUM_SCALES, scale_fn, coding_rank=3,
                                            compression=True).to("cuda")


def _weights(groups, seed):
  """Random per-group [ctx kernels (3), ctx biases (3), W1, b1, W2, b2, W3, b3] with loc of a few units and scale
  indexes spread over the table range."""
  g = torch.Generator().manual_seed(seed)
  M = sum(groups)
  out = []
  for k, c in enumerate(groups):
    k1, n3, n4 = scmo.widths(M, k, c)
    r = lambda *s: torch.randn(*s, generator=g).cuda()
    out.append([[r(5, 5, c, 2 * c) / math.sqrt(12 * c) for _ in range(3)], [0.1 * r(2 * c) for _ in range(3)],
                r(k1, n3) / math.sqrt(k1), 0.1 * r(n3), r(n3, n4) / math.sqrt(n3), 0.1 * r(n4),
                8 * r(n4, 2 * c) / math.sqrt(n4), torch.cat([0.5 * r(c), 24 + 4 * r(c)])])
  return out


def _np_weights(ws):
  return [[k.cpu().numpy() for k in ws[0]], [b.cpu().numpy() for b in ws[1]]] + [w.cpu().numpy() for w in ws[2:]]


_PACKED = {}


def _packed(groups, seed=0):
  if (groups, seed) not in _PACKED:
    ws = _weights(groups, seed)
    M = sum(groups)
    _PACKED[(groups, seed)] = ([F.mscc_pack_weights(M, s, *w) for s, w in zip(F.scc_spans(groups), ws)],
                               [_np_weights(w) for w in ws], ws)
  return _PACKED[(groups, seed)]


def _latents(B, H, W, M, seed):
  g = torch.Generator().manual_seed(1000 + seed)
  y = 3 * torch.randn(B, H, W, M, generator=g)
  big = torch.rand(B, H, W, M, generator=g) < 0.002  # a few escapes
  y[big] *= 40
  psi = torch.randn(B, H, W, 2 * M, generator=g)
  return y.cuda(), psi.cuda()


def _ch_ctx(groups):
  """A channel context the CPU reproduces exactly: channels of y_hat[..., :o_k] repeated and halved."""
  spans = F.scc_spans(groups)

  def fn(k, y_hat):
    o, c = spans[k]
    reps = -(-2 * c // o)
    if isinstance(y_hat, torch.Tensor):
      return y_hat[..., :o].repeat(1, 1, 1, reps)[..., :2 * c] * 0.5
    return np.tile(y_hat[..., :o], (1, 1, 1, reps))[..., :2 * c] * np.float32(0.5)

  return fn


def _np(t):
  return t.cpu().numpy()


def _bits(a):
  return np.asarray(a).view(np.int32)


def _encode(em, packed, groups, y, psi, ch_fn):
  y_hat, y_cc, loc, index, scale = F.mscc_encode(packed, groups, y, psi, ch_fn, NUM_SCALES, scale_index=True)
  strings = F.compress_f32((y.shape[0],), em._lookup_host(), y_cc, loc, em.cdf_offset, index=index)
  return strings, y_hat, y_cc, loc, index, scale


def _decode(em, packed, groups, strings, psi, ch_fn, S=1):
  if S > 1:
    strings = gen_ops.split_substreams(strings, S)
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  y_hat = F.mscc_decode(handle, packed, groups, psi, ch_fn, NUM_SCALES, em.cdf_offset, substreams=S)
  return y_hat, gen_ops.entropy_decode_finalize(handle)


def _check_params(packed, ws, groups, y_hat, psi):
  fn = _ch_ctx(groups)
  B, H, W, _ = y_hat.shape
  for k, (p, w, g) in enumerate(zip(packed, ws, F.scc_spans(groups))):
    ch = fn(k, y_hat).contiguous() if k else None
    for stage in range(4):
      got = F.mscc_params(p, g, y_hat, psi, ch, stage, NUM_SCALES)
      want = scmo.params32(w, g, _np(y_hat), _np(psi), None if ch is None else _np(ch), stage, NUM_SCALES)
      assert got[0].shape == (B, F.msc_counts(H, W)[stage], g[1])
      for a, b in zip(got, want):
        assert np.array_equal(_bits(_np(a)), _bits(b)), (groups, k, H, W, stage)


# ---------------------------------------------------------------------------------------------------------------
# 1. every stage of every group is the float32 emulation, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [(6,), (1, 5), (2, 4, 6, 12), DEFAULT], ids=str)
def test_params_are_the_float32_emulation_bit_for_bit(groups):
  packed, ws, _ = _packed(groups)
  M = sum(groups)
  shapes = SHAPES if M < 100 else [(1, 1), (1, 9), (7, 1), (2, 2), (5, 7)]
  for H, W in shapes:
    B = 3 if H * W < 100 else 1
    y, psi = _latents(B, H, W, M, M + H)
    _check_params(packed, ws, groups, torch.round(y), psi)


def test_position_counts_off_the_tile_are_the_emulation():
  groups = (2, 4, 6, 12)
  packed, ws, _ = _packed(groups)
  for B, (H, W) in ((3, (3, 5)), (5, (7, 11))):
    assert all((B * n) % 32 for n in F.msc_counts(H, W))
    y, psi = _latents(B, H, W, 24, 40 + B)
    _check_params(packed, ws, groups, torch.round(y), psi)


def test_ragged_params_equal_the_one_image_passes():
  groups = (2, 4, 6, 12)
  packed, ws, _ = _packed(groups)
  fn = _ch_ctx(groups)
  shapes = [(1, 1), (3, 5), (1, 6), (7, 1), (6, 8), (2, 2)]  # tiles of 32 positions straddle images; empty stages
  lat = [_latents(1, h, w, 24, i) for i, (h, w) in enumerate(shapes)]
  y_hats = [torch.round(y[0]) for y, _ in lat]
  psis = [p[0] for _, p in lat]
  for k, (p, w, g) in enumerate(zip(packed, ws, F.scc_spans(groups))):
    chs = [fn(k, yh[None])[0].contiguous() for yh in y_hats] if k else None
    for s in range(4):
      loc, scale, index, lengths = F.mscc_params_ragged(p, g, y_hats, psis, chs, s, NUM_SCALES)
      assert lengths == [F.msc_counts(h, w_)[s] * g[1] for h, w_ in shapes]
      at = 0
      for i, (yh, ps, n) in enumerate(zip(y_hats, psis, lengths)):
        ch = None if chs is None else _np(chs[i][None])
        want = scmo.params32(w, g, _np(yh[None]), _np(ps[None]), ch, s, NUM_SCALES)
        for a, b in zip((loc, scale, index), want):
          assert np.array_equal(_bits(_np(a[at:at + n])), _bits(b.reshape(-1)))
        at += n


def _msc_lib_params(packed, y_hat, psi, stage):
  """tfcb_msc_params itself (functional.msc_params is the one-group call of mscc_params)."""
  B, H, W, M = y_hat.shape
  lib = _lib.lib()
  n = F.msc_counts(H, W)[stage]
  loc, scale = (torch.empty((B, n, M), device="cuda") for _ in range(2))
  index = torch.empty((B, n, M), dtype=torch.int32, device="cuda")
  nw = int(lib.tfcb_msc_workspace_floats(M, B, H, W, stage))
  work = torch.empty(max(nw, 1), device="cuda")
  p = lambda t: None if t is None else t.data_ptr()
  _lib.check(lib.tfcb_msc_params(p(packed), packed.numel(), M, p(y_hat), p(psi), B, H, W, stage, NUM_SCALES, p(work),
                                 nw, 0, p(loc), p(scale), p(index), None, None, None, None))
  return loc, scale, index


@pytest.mark.parametrize("M", [6, 96, 192])
def test_one_group_is_the_multistage_pass_bit_for_bit(M):
  (packed,), _, (ws,) = _packed((M,))
  ms_packed = F.msc_pack_weights(*ws)
  assert torch.equal(packed, ms_packed)
  for H, W in ((1, 1), (1, 7), (5, 7), (32, 48)):
    y, psi = _latents(2, H, W, M, 3 * M + H)
    y_hat = torch.round(y)
    for stage in range(4):
      got = F.mscc_params(packed, (0, M), y_hat, psi, None, stage, NUM_SCALES)
      want = _msc_lib_params(ms_packed, y_hat, psi, stage)
      for a, b in zip(got, want):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
  y, psi = _latents(2, 6, 7, M, 5)
  got = F.mscc_encode([packed], (M,), y, psi, None, NUM_SCALES, scale_index=True)
  want = mso.encode32(_np_weights(ws), _np(y), _np(psi), NUM_SCALES)
  for a, b in zip(got, want):
    assert np.array_equal(_bits(_np(a)).reshape(-1), _bits(b).reshape(-1))


@pytest.mark.parametrize("groups", [(1, 5), (2, 4, 6, 12), DEFAULT], ids=str)
def test_stage_zero_is_the_space_channel_anchor_pass(groups):
  packed, _, ws = _packed(groups)
  M, (H, W) = sum(groups), (5, 7)
  fn = _ch_ctx(groups)
  y, psi = _latents(2, H, W, M, 9)
  y_hat = torch.round(y)
  anchors = cbo.positions(H, W, True)
  at = torch.tensor([anchors.index(p) for p in mso.positions(H, W, 0)], device="cuda")
  for k, (p, w, g) in enumerate(zip(packed, ws, F.scc_spans(groups))):
    ch = fn(k, y_hat).contiguous() if k else None
    scc = F.scc_pack_weights(M, g, w[0][1], w[1][1], *w[2:])  # any context kernel: the anchors read none
    got = F.mscc_params(p, g, y_hat, psi, ch, 0, NUM_SCALES)
    want = F.scc_params(scc, g, y_hat, psi, ch, True, NUM_SCALES)
    for a, b in zip(got, want):
      assert torch.equal(a.view(torch.int32), b[:, at].view(torch.int32))


@pytest.mark.parametrize("groups", [(1, 5), (2, 4, 6, 12), DEFAULT], ids=str)
def test_encoder_is_the_emulated_encoder(groups):
  packed, ws, _ = _packed(groups)
  M = sum(groups)
  B, H, W = 2, 5, 6
  y, psi = _latents(B, H, W, M, 21)
  fn = _ch_ctx(groups)
  got = F.mscc_encode(packed, groups, y, psi, fn, NUM_SCALES, scale_index=True)
  want = scmo.encode32(ws, groups, _np(y), _np(psi), fn, NUM_SCALES)
  for a, b in zip(got, want):
    assert np.array_equal(_bits(_np(a)), _bits(b))
  order = torch.from_numpy(scmo.coding_order(H, W, groups)).cuda()
  assert torch.equal(got[1], y.reshape(B, -1)[:, order])
  assert torch.equal(got[0].reshape(B, -1)[:, order], torch.round(got[1] - got[2]) + got[2])


def test_rows_do_not_depend_on_the_batch():
  groups = DEFAULT
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  y, psi = _latents(6, 5, 7, 320, 5)
  for B in (3, 6):
    batch = F.mscc_encode(packed, groups, y[:B], psi[:B], fn, NUM_SCALES, scale_index=True)
    for b in (0, B - 1):
      one = F.mscc_encode(packed, groups, y[b:b + 1].clone(), psi[b:b + 1].clone(), fn, NUM_SCALES, scale_index=True)
      for g, w in zip(one, batch):
        assert torch.equal(g[0], w[b])


# ---------------------------------------------------------------------------------------------------------------
# 2. strings and the decoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("groups", [(2, 4, 6, 12), DEFAULT], ids=str)
@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (2, 2), (5, 7)], ids=lambda s: f"{s[0]}x{s[1]}")
def test_strings_are_the_entropy_models_and_decode_to_the_encoders_latents(em, groups, shape):
  B, M = 3, sum(groups)
  y, psi = _latents(B, *shape, M, 7)
  y[0, 0, 0, :4] = torch.tensor([3e9, -3e9, 2.0**31, -2.0**31])  # saturated escapes
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  strings, y_hat_enc, y_cc, loc, index, scale = _encode(em, packed, groups, y, psi, fn)
  n = shape[0] * shape[1] * M
  assert torch.equal(em._flatten_indexes(em._normalize_indexes(scale)), index)
  want = em.compress(y_cc.view(B, n, 1, 1), scale.view(B, n, 1, 1), loc.view(B, n, 1, 1))
  assert strings.tolist() == want.tolist()
  y_hat, ok = _decode(em, packed, groups, strings, psi, fn)
  assert bool(ok.all())
  assert torch.equal(y_hat, y_hat_enc)


def test_batch_ragged_and_single_image_coding_interoperate(em):
  groups, (H, W), B = (2, 4, 6, 12), (5, 7), 4
  y, psi = _latents(B, H, W, 24, 3)
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  strings, y_hat_batch = _encode(em, packed, groups, y, psi, fn)[:2]
  for b, s in enumerate(strings.split()):  # batch encode, one-image decode
    y_hat, ok = _decode(em, packed, groups, s, psi[b:b + 1], fn)
    assert bool(ok.all()) and torch.equal(y_hat[0], y_hat_batch[b])
  singles = [_encode(em, packed, groups, y[b:b + 1], psi[b:b + 1], fn)[0] for b in range(B)]
  assert [s.tolist()[0] for s in singles] == strings.tolist()
  # a ragged list of other shapes: each image's string and latents are the one-image call's
  shapes = [(5, 7), (1, 1), (2, 9), (8, 1)]
  lat = [_latents(1, h, w, 24, 30 + i) for i, (h, w) in enumerate(shapes)]
  ys, psis = [t[0][0] for t in lat], [t[1][0] for t in lat]
  lists = lambda k, yhs: [fn(k, yh[None])[0].contiguous() for yh in yhs]
  lookup, coff = em._lookup_host(), em.cdf_offset
  y_hats, y_r, loc, index, lengths = F.mscc_encode_ragged(packed, groups, ys, psis, lists, NUM_SCALES)
  rs = F.compress_ragged(lookup, lengths, y_r, loc, coff, index=index)
  for i, (yi, pi) in enumerate(zip(ys, psis)):
    one_s, one_hat = _encode(em, packed, groups, yi[None], pi[None], fn)[:2]
    assert rs.tolist()[i] == one_s.tolist()[0] and torch.equal(y_hats[i], one_hat[0])
  handle = gen_ops.create_range_decoder(rs, lookup)
  got = F.mscc_decode_ragged(handle, packed, groups, psis, lists, NUM_SCALES, coff)
  assert bool(gen_ops.entropy_decode_finalize(handle).all())
  assert all(torch.equal(g, w) for g, w in zip(got, y_hats))


@pytest.mark.parametrize("S", [2, 7])
def test_substreams_decode_to_the_one_stream_latents(em, S):
  groups, B, H, W = (2, 4, 6, 12), 2, 6, 7
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  y, psi = _latents(B, H, W, 24, 40 + S)
  strings1, y_hat1 = _encode(em, packed, groups, y, psi, fn)[:2]
  y_hat, y_s, loc, index = F.mscc_encode(packed, groups, y, psi, fn, NUM_SCALES, substreams=S)
  assert torch.equal(y_hat, y_hat1)
  lengths = F.context_substreams(groups, [H] * B, [W] * B, S, multistage=True)[0]
  parts = F.compress_ragged(em._lookup_host(), lengths, y_s, loc, em.cdf_offset, index=index)
  strings = gen_ops.join_substreams(parts, S, (B,))
  for one, many in zip(strings1.tolist(), strings.tolist()):
    header = len(many) - sum(len(p) for p in gen_ops.parse_substreams(many, S))
    assert len(many) <= len(one) + header + 4 * S
  got, ok = _decode(em, packed, groups, strings, psi, fn, S)
  assert bool(ok.all()) and torch.equal(got, y_hat1)
  # the ragged encoder's substreams are the batch encoder's
  ys, psis = list(y), list(psi)
  lists = lambda k, yhs: [fn(k, yh[None])[0].contiguous() for yh in yhs]
  out = F.mscc_encode_ragged(packed, groups, ys, psis, lists, NUM_SCALES, substreams=S)
  assert out[4] == lengths.tolist() and torch.equal(out[1], y_s.reshape(-1))


@pytest.mark.parametrize("B", [1, 4])
def test_decode_runs_without_host_sync_in_a_fixed_number_of_launches(em, B):
  groups = (2, 4, 6, 12)
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  counts = {}
  for shape in ((1, 1), (1, 7), (5, 7), (32, 48)):
    y, psi = _latents(B, *shape, 24, 13)
    strings, y_hat_enc = _encode(em, packed, groups, y, psi, fn)[:2]
    handle = gen_ops.create_range_decoder(strings, em._lookup_host())
    coff = em.cdf_offset.cuda()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
      y_hat = F.mscc_decode(handle, packed, groups, psi, fn, NUM_SCALES, coff)
    finally:
      torch.cuda.set_sync_debug_mode(0)
    counts[shape] = _lib.launch_count() - n0
    assert bool(gen_ops.entropy_decode_finalize(handle).all())
    assert torch.equal(y_hat, y_hat_enc)
  # per group as the multistage decoder: stage 0 three parameter launches, a decode and a scatter; stages 1-3 four, a
  # decode and a scatter.  An empty stage launches nothing: at 1x1 stages 1-3 are empty, at 1x7 stages 1 and 3.
  assert counts[(5, 7)] == counts[(32, 48)] == (5 + 3 * 6) * len(groups)
  assert counts[(1, 1)] == 5 * len(groups)
  assert counts[(1, 7)] == (5 + 6) * len(groups)


def test_damaged_strings_are_reported(em):
  groups, B, H, W = (2, 4, 6, 12), 3, 5, 7
  y, psi = _latents(B, H, W, 24, 17)
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  good = _encode(em, packed, groups, y, psi, fn)[0].tolist()
  padded = gen_ops.Strings.from_bytes([good[0] + bytes(range(64)), good[1], good[2]], (B,))
  truncated = gen_ops.Strings.from_bytes([good[0], good[1][:len(good[1]) // 2], good[2]], (B,))
  y_hat, ok = _decode(em, packed, groups, padded, psi, fn)
  assert torch.isfinite(y_hat).all() and ok.tolist() == [False, True, True]
  y_hat, ok = _decode(em, packed, groups, truncated, psi, fn)
  assert torch.isfinite(y_hat).all() and ok.tolist()[0] and ok.tolist()[2]


def test_bad_arguments_raise_before_any_launch(em):
  groups, B, H, W = (2, 4, 6, 12), 2, 3, 4
  y, psi = _latents(B, H, W, 24, 19)
  packed = _packed(groups)[0]
  fn = _ch_ctx(groups)
  strings = _encode(em, packed, groups, y, psi, fn)[0]
  handle = gen_ops.create_range_decoder(strings, em._lookup_host())
  spans = F.scc_spans(groups)
  ch = fn(1, y).contiguous()
  n0 = _lib.launch_count()
  with pytest.raises(_lib.InvalidArgumentError, match="2 strings for a batch of 1"):
    F.mscc_decode(handle, packed, groups, psi[:1], fn, NUM_SCALES, em.cdf_offset)
  with pytest.raises(_lib.InvalidArgumentError, match="packed weights hold"):
    F.mscc_params(packed[2], spans[1], y, psi, ch, 0, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="ch_ctx"):
    F.mscc_params(packed[1], spans[1], y, psi, None, 0, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="no channel context"):
    F.mscc_params(packed[0], spans[0], y, psi, ch, 0, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="y_hat"):
    F.mscc_params(packed[0], spans[0], None, psi, None, 2, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="shape"):
    F.mscc_encode(packed, groups, y[:, :2], psi, fn, NUM_SCALES)
  with pytest.raises(_lib.InvalidArgumentError, match="substreams"):
    F.mscc_decode(handle, packed, groups, psi, fn, NUM_SCALES, em.cdf_offset, substreams=3)
  lib = _lib.lib()
  p = lambda t: None if t is None else t.data_ptr()
  o, c = spans[1]
  for stage in range(4):
    with pytest.raises(_lib.InvalidArgumentError, match="workspace of 4 floats"):
      _lib.check(lib.tfcb_mscc_params(p(packed[1]), packed[1].numel(), 24, o, c, p(y), p(psi), p(ch), B, H, W, stage,
                                      NUM_SCALES, p(y), 4, 0, p(y), None, None, None, None, None, None))
    with pytest.raises(_lib.InvalidArgumentError, match="chctx"):
      _lib.check(lib.tfcb_mscc_params(p(packed[1]), packed[1].numel(), 24, o, c, p(y), p(psi), None, B, H, W, stage,
                                      NUM_SCALES, p(y), 1 << 20, 0, p(y), None, None, None, None, None, None))
  hs, ws = np.array([3, 2], np.int64), np.array([4, 2], np.int64)
  with pytest.raises(_lib.InvalidArgumentError, match="aligned"):
    _lib.check(lib.tfcb_mscc_params_ragged(p(packed[1]), packed[1].numel(), 24, o, c, p(y), p(psi), p(ch), 2,
                                           hs.ctypes.data, ws.ctypes.data, 1, NUM_SCALES, p(y) + 4, 1 << 16, 0, None,
                                           None, None, None, None, None, None))
  assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# 3. the training path and the model
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_model():
  torch.manual_seed(0)
  return models.SpaceChannelMultistageModel(num_filters=24, latent_depth=24, groups=(2, 4, 6, 12)).build(
      "cuda", patch=(64, 64)).fix_tables()


def test_params_kernels_match_the_training_path(small_model):
  m = small_model
  M, H, W = m.latent_depth, 5, 6
  g = torch.Generator().manual_seed(2)
  y_hat = torch.round(3 * torch.randn(2, H, W, M, generator=g)).cuda()
  psi = torch.randn(2, H, W, 2 * M, generator=g).cuda()
  allow = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
  torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
  try:
    with torch.no_grad():
      loc_t, scale_t = m.entropy_parameters_of(y_hat, psi)
      # the training form's channel context, so that both sides read the same layer-1 inputs
      chs = [m.channel_context_transforms[k - 1](y_hat[..., :o]).contiguous() if k else None
             for k, (o, _) in enumerate(m.spans)]
  finally:
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = allow
  for k, (o, c) in enumerate(m.spans):
    cms = m.context_models[k]
    ws = [[_np(cm.kernel.detach()) for cm in cms], [_np(cm.bias.detach()) for cm in cms]]
    ws += [_np(t.detach()) for t in models._dense_weights(m.entropy_parameters[k])]
    for s in range(4):
      pos = mso.positions(H, W, s)
      loc, scale, _ = F.mscc_params(m._packed[k], (o, c), y_hat, psi, chs[k], s, NUM_SCALES)
      lb, sb = scmo.bound64(ws, (o, c), _np(y_hat), _np(psi), None if chs[k] is None else _np(chs[k]), s)
      # both sides are float32 evaluations of the same sums, each within the oracle's bound of the exact value
      for got, want, bound in ((loc, loc_t.view(2, H * W, M)[:, pos, o:o + c], lb),
                               (scale, scale_t.view(2, H * W, M)[:, pos, o:o + c], sb)):
        assert np.all(np.abs(_np(got).astype(np.float64) - _np(want)) <= 2 * bound), (k, s)


def test_training_reaches_every_parameter(small_model):
  m = small_model
  m.zero_grad()
  x = torch.randint(0, 256, (2, 64, 64, 3), device="cuda").float()
  loss, bpp, mse = m(x, training=True)
  assert math.isfinite(float(bpp.detach())) and math.isfinite(float(mse.detach()))
  loss.backward()
  for name, prm in m.named_parameters():
    assert prm.grad is not None, name
    assert torch.isfinite(prm.grad).all(), name
  for cms in m.context_models:  # exactly each stage's taps learn
    for s, cm in enumerate(cms, 1):
      grad = cm.kernel.grad.abs().sum((2, 3)).cpu()
      assert torch.equal(grad > 0, models.multistage_mask(s) > 0)
  m.zero_grad()


def _images(sizes, seed):
  rng = np.random.default_rng(seed)
  out = []
  for h, w in sizes:
    yy, xx = np.mgrid[0:h, 0:w]
    base = 128 + 60 * np.sin(xx / 7.0)[..., None] * np.cos(yy / 11.0)[..., None] * np.array([1.0, 0.7, 0.4])
    out.append(torch.from_numpy(np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)))
  return out


def test_model_round_trip_and_tfci(small_model):
  m = small_model
  x = _images([(64, 80)], 0)[0]
  packed = m.compress(x)
  assert len(packed) == 5
  x_hat = m.decompress(*packed)
  assert x_hat.shape == x.shape and x_hat.dtype == torch.uint8
  with torch.no_grad():
    y = m.analysis_transform(x[None].cuda().float())
    z = m.hyper_analysis_transform(y)
    psi = m._psi(m.side_entropy_model.quantize(z), tuple(y.shape[1:-1]))
    _, y_hat_enc, _, _ = m._encode_latents(y, psi)
    assert torch.equal(m._decode_latents(packed[0], psi), y_hat_enc)
    want = models._to_uint8(m.synthesis_transform(y_hat_enc)[:, :64, :80, :])[0]
  assert torch.equal(x_hat, want)
  assert torch.equal(m.decompress_from_tfci(m.compress_to_tfci(x)), x_hat)


def test_images_equal_the_one_image_calls_and_evaluate(small_model):
  m = small_model
  imgs = _images([(64, 80), (48, 64), (64, 80), (33, 47)], 1)
  items = m.compress_images(imgs)
  outs = m.decompress_images(items)
  for x, item, out in zip(imgs, items, outs):
    one = m.compress(x)
    assert one[0].tolist() == item[0].tolist() and one[1].tolist() == item[1].tolist()
    assert torch.equal(m.decompress(*one), out)
  batch = m.compress_batch(torch.stack([imgs[0], imgs[2]]))
  assert batch[0].tolist() == [items[0][0].tolist()[0], items[2][0].tolist()[0]]
  big = _images([(176, 192)], 2)
  d = m.evaluate_images(big)[0]
  e = m.evaluate(big[0])
  assert d["bpp"] == e["bpp"] and math.isfinite(e["psnr"])


def test_model_substreams_decode_the_one_stream_images(small_model):
  m = small_model
  x = _images([(64, 80)], 3)[0]
  want = m.decompress(*m.compress(x))
  m4 = models.SpaceChannelMultistageModel(num_filters=24, latent_depth=24, groups=(2, 4, 6, 12), substreams=4).build(
      "cuda", patch=(64, 64))
  keys = m4.state_dict().keys()
  m4.load_state_dict({k: v for k, v in m.state_dict().items() if k in keys})
  m4.fix_tables()
  assert torch.equal(m4.decompress(*m4.compress(x)), want)
  items = m4.compress_images(_images([(64, 80), (40, 56)], 4))
  assert len(m4.decompress_images(items)) == 2


def test_one_group_model_strings_are_the_multistage_models():
  torch.manual_seed(1)
  m = models.SpaceChannelMultistageModel(num_filters=24, latent_depth=24, groups=(24,)).build("cuda", patch=(64, 64))
  ms = models.MultistageModel(num_filters=24, latent_depth=24).build("cuda", patch=(64, 64))
  keys = ms.state_dict().keys()
  moved = {}
  for k, v in m.state_dict().items():
    for a, b in (("context_models.0.", "context_models."), ("entropy_parameters.0.", "entropy_parameters.")):
      if k.startswith(a):
        k = b + k[len(a):]
    moved[k] = v
  assert set(moved) == set(keys)
  ms.load_state_dict(moved)
  m.fix_tables()
  ms.fix_tables()
  x = _images([(64, 80), (48, 96)], 5)
  for a, b in zip(m.compress_images(x), ms.compress_images(x)):
    assert a[0].tolist() == b[0].tolist() and a[1].tolist() == b[1].tolist()
  one = m.compress(x[0])
  assert one[0].tolist() == ms.compress(x[0])[0].tolist()
  assert torch.equal(m.decompress(*one), ms.decompress(*one))


def test_default_model_codes_an_image():
  torch.manual_seed(0)
  m = models.SpaceChannelMultistageModel(num_filters=32).build("cuda", patch=(64, 64)).fix_tables()
  assert m.latent_depth == 320 and m.groups == DEFAULT
  x = _images([(96, 128)], 3)[0]
  items = m.compress(x)
  assert m.decompress(*items).shape == x.shape
  with torch.no_grad():
    y = m.analysis_transform(x[None].cuda().float())
    psi = m._psi(m.side_entropy_model.quantize(m.hyper_analysis_transform(y)), tuple(y.shape[1:-1]))
    assert torch.equal(m._decode_latents(items[0], psi), m._encode_latents(y, psi)[1])
