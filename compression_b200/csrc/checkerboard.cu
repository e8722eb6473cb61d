// Checkerboard context model (He, Zheng, Sun, Wang & Qin, CVPR 2021) and space-channel context model (He, Yang, Peng,
// Ma, Qin & Wang, CVPR 2022) on sm_90a: the entropy parameters of one colour of latent positions of one channel group,
// all images and positions of that colour at once.
//
// A position (r, c) is an anchor when r + c is even, else a non-anchor.  The latent y [B, H, W, M] is split into
// channel groups; group k holds the C = c_k channels [o, o + C) (the checkerboard model is the one group o = 0,
// C = M).  An image codes group 0's anchors in raster order, then group 0's non-anchors in raster order, then group
// 1's anchors, and so on ("coding order"); the j-th position of colour k (0 anchors, 1 non-anchors) lies in row
// 2 (j / W) or 2 (j / W) + 1, see cb_position.  Per position of group k (CH = 0 for k = 0, else 2C):
//   ctx   = 0 at an anchor (bias included); at a non-anchor bc + Wc · gather(ŷ[o, o + C), the 12 taps (dy, dx) in
//           [-2, 2]^2 with dy + dx odd, raster order, zeros outside the image), every tap an anchor  [12C] -> [2C]
//   h1    = leaky(b1 + W1 · [ψ_p (2M), chctx_p (CH), ctx])                      [K1 = 2M + CH + 2C]  -> [N3 = 5 K1 / 6]
//   h2    = leaky(b2 + W2 · h1)                                                                      [N3]  -> [N4 = 2 K1 / 3]
//   out   = b3 + W3 · h2 = [loc, scale_index]                                                        [N4]  -> [2C]
// (N3 and N4 rounded down; with one group they are 10M/3 and 8M/3) with the packed weights of one group, laid out
// by cb_net (Wc: the 12 checkerboard taps, gathered by the caller).  The channel context chctx [B, H, W, CH] comes
// from the caller.
//
// Every output is autoregressive.cu's fixed sequence of float32 operations: bias first, then the eight slices
// [s·K/8, (s+1)·K/8) in order, each an __fmaf_rn chain from +0.f in increasing k, added with __fadd_rn, then the
// LeakyReLU.  So an output depends only on its own position's inputs, never on the tile, the grid, B or the SM count.
// At an anchor, a slice of layer 1 that lies wholly in the ctx segment [2M + CH, K1) is a chain over zeros, which is
// +0 for finite weights: it is skipped and +0.f is added in its place (turning a -0 sum into +0, as the chain would).
// Any other slice runs its chain over the zeros.  With one group these are exactly slices 4-7.
//
// A pass is one launch per layer (three at anchors, four at non-anchors).  A CTA computes a tile of kCbTP positions ×
// kCbTN output columns of one layer, staging kCbKC inputs of each position and the matching weight rows in shared
// memory, so that each weight loaded from L2 serves kCbTP positions and a 32×48 image spreads over the SMs by
// position tiles and column tiles alike.  The layers' outputs go through a caller-provided workspace.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "autoregressive.cuh"
#include "checkerboard.cuh"
#include "checkerboard_schedule.cuh"
#include "common.cuh"

namespace tfcb {
namespace {

// One group's parameter network: its widths and the offsets of its packed buffer, in floats.
struct CbNet {
  int C, K1, N3, N4;
  long long wc, bc, w1, b1, w2, b2, w3, b3, total;
};

// The packed layout of group [o, o + C) of a latent of depth M: Wc [12C, 2C], bc [2C], W1 [K1, N3], b1, W2 [N3, N4],
// b2, W3 [N4, 2C], b3.  At o = 0, C = M (M a multiple of 6) it is ar_dims(M)'s, which tfcb_ar_pack_weights packs.
__host__ __device__ inline CbNet cb_net(int M, int o, int C) {
  CbNet d;
  d.C = C;
  d.K1 = 2 * M + (o > 0 ? 2 * C : 0) + 2 * C;
  d.N3 = 5 * d.K1 / 6;
  d.N4 = 2 * d.K1 / 3;
  d.wc = 0;
  d.bc = d.wc + (long long)kArTaps * C * 2 * C;
  d.w1 = d.bc + 2 * C;
  d.b1 = d.w1 + (long long)d.K1 * d.N3;
  d.w2 = d.b1 + d.N3;
  d.b2 = d.w2 + (long long)d.N3 * d.N4;
  d.w3 = d.b2 + d.N4;
  d.b3 = d.w3 + (long long)d.N4 * 2 * C;
  d.total = d.b3 + 2 * C;
  return d;
}

template <int IN, int OUT>
__global__ void __launch_bounds__(kCbThreads) cb_dense_kernel(const CbPass S, const CbLayer L) {
  cb_dense<IN, OUT, CbSchedule>(S, L);
}

// ŷ of one colour of group [o, o + C), [B, n_k, C] in coding order -> its positions and channels of [B, H, W, M];
// with `img` (a ragged list of n_img images) image i's n_k,i C values at C q_i -> its [H_i, W_i, M] at M pix_i
__global__ void cb_scatter_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n_k, int W,
                                  long long HW, int M, int o, int C, int colour, long long total,
                                  const CbImage* __restrict__ img, int n_img) {
  cb_scatter<CbSchedule>(src, dst, n_k, W, HW, M, o, C, colour, total, img, n_img);
}

constexpr int kSccMaxM = 1024;

long long cb_work_floats(const CbNet& d, const CbList& L, int colour) {
  return cb_table_floats(L) + cb_positions(L, colour) * ((colour ? 2 * d.C : 0) + d.N3 + d.N4);
}

bool scc_group_ok(int M, int o, int C) { return M > 0 && M % 2 == 0 && M <= kSccMaxM && o >= 0 && C >= 1 && o + C <= M; }

int scc_check_group(int M, int o, int C) {
  if (M <= 0 || M % 2 != 0 || M > kSccMaxM)
    return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be a positive even number and at most %d", M, kSccMaxM);
  if (o < 0 || C < 1 || o + C > M)
    return fail(TFCB_INVALID_ARGUMENT, "group of %d channels at offset %d does not fit a latent of depth %d", C, o, M);
  return TFCB_OK;
}

int scc_check_packed(const float* packed, int64_t packed_floats, int M, int o, int C) {
  if (!packed) return fail(TFCB_INVALID_ARGUMENT, "`packed` is null");
  const long long n = cb_net(M, o, C).total;
  if (packed_floats != n)
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, the group [%d, %d) of M=%d needs %lld",
                (long long)packed_floats, o, o + C, M, n);
  return TFCB_OK;
}

template <int IN, int OUT>
int cb_layer(const CbPass& S, const CbLayer& L, cudaStream_t s) {
  const dim3 grid((unsigned)((S.P + kCbTP - 1) / kCbTP), (unsigned)((L.N + kCbTN - 1) / kCbTN));
  cb_dense_kernel<IN, OUT><<<grid, kCbThreads, 0, s>>>(S, L);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// One pass over colour `colour` of group [o, o + C) of a latent of depth M, after the caller's checks of M, the group,
// the packed size, the images and num_scales.  Outputs [B, n_k, C] (whole == 0), or the coding order of every group,
// [B, H W M], at this pass's block H W o + (colour ? n_a C : 0) (whole != 0); for a ragged list, image by image at the
// offsets of cb_upload_table.
int cb_run(const float* packed, int M, int o, int C, const float* yhat, const float* psi, const float* chctx,
           const CbList& I, int colour, int num_scales, float* work, int64_t work_floats, int whole, float* loc,
           float* scale, int32_t* index, const float* y, float* y_cb, float* yhat_out, void* stream) {
  if (!psi || (colour && !yhat)) return fail(TFCB_INVALID_ARGUMENT, "`psi` or `yhat` is null");
  if (o > 0 && !chctx)
    return fail(TFCB_INVALID_ARGUMENT, "`chctx` is null: the group at channel offset %d needs its channel context", o);
  const CbNet d = cb_net(M, o, C);
  const long long need = cb_work_floats(d, I, colour);
  if (!work || work_floats < need)
    return fail(TFCB_INVALID_ARGUMENT, "workspace of %lld floats, this pass needs %lld", work ? (long long)work_floats : 0ll,
                need);
  if (I.hs) TFCB_TRY(ar_check_table_space(work, work_floats, need, alignof(CbImage)));
  if (y && (!y_cb || !yhat_out || !loc || !index))
    return fail(TFCB_INVALID_ARGUMENT, "the encoder needs `y_cb`, `yhat_out`, `loc` and `index`");
  const long long P = cb_positions(I, colour);
  if (P == 0) return TFCB_OK;
  cudaStream_t s = as_stream(stream);
  CbPass S{};
  S.B = (int)I.B;
  S.M = M;
  S.C = C;
  S.o = o;
  S.CH = o > 0 ? 2 * C : 0;
  S.colour = colour;
  S.num_scales = num_scales;
  S.P = P;
  if (I.hs) {
    TFCB_TRY(cb_upload_table(I, M, o, C, colour, whole, work, s));
    S.img = reinterpret_cast<const CbImage*>(work);
    S.n_img = (int)I.B;
  } else {
    const long long n_k = cb_count(I.H, I.W, colour);
    S.H = (int)I.H;
    S.W = (int)I.W;
    S.n_k = n_k;
    S.HW = I.H * I.W;
    S.out_stride = whole ? S.HW * M : n_k * C;
    S.out_base = whole ? S.HW * o + (colour ? cb_count(I.H, I.W, 0) * C : 0) : 0;
  }
  S.psi = psi;
  S.chctx = chctx;
  S.yhat = yhat;
  S.loc = loc;
  S.scale = scale;
  S.index = index;
  S.y = y;
  S.y_cb = y_cb;
  S.yhat_out = yhat_out;
  float* ctx = work + cb_table_floats(I);
  float* h1 = ctx + (colour ? S.P * 2 * C : 0);
  float* h2 = h1 + S.P * d.N3;
  if (colour)
    TFCB_TRY((cb_layer<kInTaps, kOutHidden>(
        S, {packed + d.wc, packed + d.bc, nullptr, ctx, kArTaps * C, 2 * C, kArTaps * C, false}, s)));
  TFCB_TRY((cb_layer<kInPsiCtx, kOutHidden>(
      S, {packed + d.w1, packed + d.b1, ctx, h1, d.K1, d.N3, colour ? d.K1 : d.K1 - 2 * C, true}, s)));
  TFCB_TRY((cb_layer<kInPlain, kOutHidden>(S, {packed + d.w2, packed + d.b2, h1, h2, d.N3, d.N4, d.N3, true}, s)));
  return cb_layer<kInPlain, kOutParams>(S, {packed + d.w3, packed + d.b3, h2, nullptr, d.N4, 2 * C, d.N4, false}, s);
}

// The scatter of one colour of group [o, o + C), after the caller's checks of the group and (for a ragged list) the
// images; a ragged list's table goes to `work`.
int cb_scatter(const float* src, const CbList& I, int M, int o, int C, int colour, float* dst, float* work,
               int64_t work_floats, void* stream) {
  if (!I.hs) {
    if (I.B <= 0 || I.B > 0x7FFFFFFF) return fail(TFCB_INVALID_ARGUMENT, "batch size %lld out of range", (long long)I.B);
    if (I.H <= 0 || I.W <= 0 || I.H * I.W > 0x7FFFFFFF)
      return fail(TFCB_INVALID_ARGUMENT, "latent shape %lld x %lld out of range", (long long)I.H, (long long)I.W);
  } else {
    TFCB_TRY(ar_check_table_space(work, work_floats, cb_table_floats(I), alignof(CbImage)));
  }
  const long long total = cb_positions(I, colour) * C;
  if (total == 0) return TFCB_OK;  // (the non-anchors of a 1x1 latent: empty tensors may have null pointers)
  if (!src || !dst) return fail(TFCB_INVALID_ARGUMENT, "`src` or `dst` is null");
  cudaStream_t s = as_stream(stream);
  const long long blocks = std::min<long long>((total + 255) / 256, 1ll << 16);
  if (I.hs) {
    TFCB_TRY(cb_upload_table(I, M, o, C, colour, 0, work, s));
    cb_scatter_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dst, 0, 0, 0, M, o, C, colour, total,
                                                       reinterpret_cast<const CbImage*>(work), (int)I.B);
  } else {
    cb_scatter_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dst, cb_count(I.H, I.W, colour), (int)I.W, I.H * I.W, M, o,
                                                       C, colour, total, nullptr, 0);
  }
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

int64_t tfcb_cb_workspace_floats(int M, int64_t B, int64_t H, int64_t W, int anchors) {
  if (M <= 0 || M % 6 != 0 || M > kArMaxM || B <= 0 || H <= 0 || W <= 0 || H * W > 0x7FFFFFFF) return -1;
  return cb_work_floats(cb_net(M, 0, M), {B, H, W, nullptr, nullptr}, anchors ? 0 : 1);
}

int tfcb_cb_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int anchors, int num_scales, float* work_dev,
                   int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev,
                   const float* y_dev, float* y_cb_dev, float* yhat_out_dev, void* stream) {
  TFCB_TRY(ar_check(M, packed_dev, packed_floats, B, H, W, num_scales));
  return cb_run(packed_dev, M, 0, M, yhat_dev, psi_dev, nullptr, {B, H, W, nullptr, nullptr}, anchors ? 0 : 1,
                num_scales, work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev, y_cb_dev,
                yhat_out_dev, stream);
}

int tfcb_cb_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int anchors, float* dst_dev,
                    void* stream) {
  if (M <= 0) return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be positive", M);
  return cb_scatter(src_dev, {B, H, W, nullptr, nullptr}, M, 0, M, anchors ? 0 : 1, dst_dev, nullptr, 0, stream);
}

int64_t tfcb_scc_packed_floats(int M, int offset, int C, int64_t* layout) {
  if (!scc_group_ok(M, offset, C)) return -1;
  const CbNet d = cb_net(M, offset, C);
  if (layout) {
    const int64_t v[11] = {d.K1, d.N3, d.N4, d.wc, d.bc, d.w1, d.b1, d.w2, d.b2, d.w3, d.b3};
    for (int i = 0; i < 11; ++i) layout[i] = v[i];
  }
  return d.total;
}

int tfcb_scc_pack_weights(int M, int offset, int C, const float* ctx_taps_dev, const float* ctx_bias_dev,
                          const float* w1_dev, const float* b1_dev, const float* w2_dev, const float* b2_dev,
                          const float* w3_dev, const float* b3_dev, float* packed_dev, int64_t packed_floats,
                          void* stream) {
  TFCB_TRY(scc_check_group(M, offset, C));
  const CbNet d = cb_net(M, offset, C);
  if (packed_floats != d.total)
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, the group [%d, %d) of M=%d needs %lld",
                (long long)packed_floats, offset, offset + C, M, (long long)d.total);
  const float* src[8] = {ctx_taps_dev, ctx_bias_dev, w1_dev, b1_dev, w2_dev, b2_dev, w3_dev, b3_dev};
  const long long at[9] = {d.wc, d.bc, d.w1, d.b1, d.w2, d.b2, d.w3, d.b3, d.total};
  return ar_pack_segments(src, at, packed_dev, as_stream(stream));
}

int64_t tfcb_scc_workspace_floats(int M, int offset, int C, int64_t B, int64_t H, int64_t W, int anchors) {
  if (!scc_group_ok(M, offset, C) || B <= 0 || H <= 0 || W <= 0 || H * W > 0x7FFFFFFF) return -1;
  return cb_work_floats(cb_net(M, offset, C), {B, H, W, nullptr, nullptr}, anchors ? 0 : 1);
}

int tfcb_scc_params(const float* packed_dev, int64_t packed_floats, int M, int offset, int C, const float* yhat_dev,
                    const float* psi_dev, const float* chctx_dev, int64_t B, int64_t H, int64_t W, int anchors,
                    int num_scales, float* work_dev, int64_t work_floats, int whole, float* loc_dev,
                    float* scale_index_dev, int32_t* index_dev, const float* y_dev, float* y_cb_dev,
                    float* yhat_out_dev, void* stream) {
  TFCB_TRY(scc_check_group(M, offset, C));
  TFCB_TRY(scc_check_packed(packed_dev, packed_floats, M, offset, C));
  TFCB_TRY(ar_check_batch(B, H, W, num_scales));
  return cb_run(packed_dev, M, offset, C, yhat_dev, psi_dev, chctx_dev, {B, H, W, nullptr, nullptr}, anchors ? 0 : 1,
                num_scales, work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev, y_cb_dev,
                yhat_out_dev, stream);
}

int tfcb_scc_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int offset, int C, int anchors,
                     float* dst_dev, void* stream) {
  TFCB_TRY(scc_check_group(M, offset, C));
  return cb_scatter(src_dev, {B, H, W, nullptr, nullptr}, M, offset, C, anchors ? 0 : 1, dst_dev, nullptr, 0, stream);
}

int64_t tfcb_scc_ragged_workspace_floats(int M, int offset, int C, int64_t n_images, const int64_t* heights_host,
                                         const int64_t* widths_host, int anchors) {
  if (!scc_group_ok(M, offset, C) || !ar_list_ok(n_images, heights_host, widths_host)) return -1;
  return cb_work_floats(cb_net(M, offset, C), {n_images, 0, 0, heights_host, widths_host}, anchors ? 0 : 1);
}

int tfcb_scc_params_ragged(const float* packed_dev, int64_t packed_floats, int M, int offset, int C,
                           const float* yhat_dev, const float* psi_dev, const float* chctx_dev, int64_t n_images,
                           const int64_t* heights_host, const int64_t* widths_host, int anchors, int num_scales,
                           float* work_dev, int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev,
                           int32_t* index_dev, const float* y_dev, float* y_cb_dev, float* yhat_out_dev,
                           void* stream) {
  TFCB_TRY(scc_check_group(M, offset, C));
  TFCB_TRY(scc_check_packed(packed_dev, packed_floats, M, offset, C));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  return cb_run(packed_dev, M, offset, C, yhat_dev, psi_dev, chctx_dev, {n_images, 0, 0, heights_host, widths_host},
                anchors ? 0 : 1, num_scales, work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev,
                y_cb_dev, yhat_out_dev, stream);
}

int tfcb_scc_scatter_ragged(const float* src_dev, int64_t n_images, const int64_t* heights_host,
                            const int64_t* widths_host, int M, int offset, int C, int anchors, float* work_dev,
                            int64_t work_floats, float* dst_dev, void* stream) {
  TFCB_TRY(scc_check_group(M, offset, C));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, 1));
  return cb_scatter(src_dev, {n_images, 0, 0, heights_host, widths_host}, M, offset, C, anchors ? 0 : 1, dst_dev,
                    work_dev, work_floats, stream);
}

}  // extern "C"
