// Checkerboard context model with mixture priors (DESIGN.md §3.19) on sm_90a: the per-latent mixtures of one colour
// of latent positions of all images at once, on checkerboard.cuh's tiles and the checkerboard schedule.
//
// Coding order and passes are the checkerboard model's (checkerboard.cu): an image's anchors (r + c even) in raster
// order, then its non-anchors, M channels per position.  Per position of colour k, with ŷ the decoded latents:
//   ctx   = 0 at an anchor (bias included); at a non-anchor bc + Wc · gather(ŷ, the 12 taps of odd parity)  [12M] -> [2M]
//   h1    = leaky(b1 + W1 · [ψ_p (2M), ctx])                                                  [4M] -> [N3 = 10M/3]
//   h2    = leaky(b2 + W2 · h1)                                                                  [N3] -> [N4 = 8M/3]
//   raw   = b3 + W3 · h2                                                                        [N4] -> [NO = 3KM]
// every output in checkerboard.cuh's fixed float32 order, so it depends only on its own position's inputs.  Channel c
// reads its K logits l, K locs and K scales from raw[3Kc .. 3Kc + 3K): the epilogue, per (position, channel), is
//   weight_k = expf(__fsub_rn(l_k, m)), m = fmaxf(.. fmaxf(l_0, l_1) .., l_{K-1}),
//   loc_k    = raw loc_k,
//   scale_k  = fmaxf(raw scale_k, 0.11f),
// written as [n, K] at the position's coding-order row: the operands of the mixture coder (mixture.cu), which
// normalises the weights itself.  The encoder's epilogue also writes y in coding order and ŷ = float((int)rintf(y))
// (saturating, NaN -> 0), the value the mixture decoder returns; so ŷ does not depend on the parameters and the
// anchors' ŷ is final before the non-anchor pass reads it.
//
// A pass is one launch per layer (three at anchors, four at non-anchors, the last one without LeakyReLU into the
// workspace), then one epilogue launch.  The scatter of decoded latents is tfcb_cb_scatter / tfcb_scc_scatter_ragged.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "autoregressive.cuh"
#include "checkerboard.cuh"
#include "checkerboard_schedule.cuh"
#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kCbmMaxK = 64;  // the mixture coder's component limit
constexpr float kCbmScaleMin = 0.11f;

// The packed layout: Wc [12M, 2M], bc [2M], W1 [4M, N3], b1, W2 [N3, N4], b2, W3 [N4, 3KM], b3 [3KM]; up to W3 it is
// ar_dims(M)'s (tfcb_cb_params' network with a wider last layer).
struct CbmNet {
  int K1, N3, N4, NO;
  long long wc, bc, w1, b1, w2, b2, w3, b3, total;
};

CbmNet cbm_net(int M, int K) {
  const ArDims a = ar_dims(M);
  CbmNet d;
  d.K1 = 4 * M;
  d.N3 = a.N3;
  d.N4 = a.N4;
  d.NO = 3 * K * M;
  d.wc = a.wc;
  d.bc = a.bc;
  d.w1 = a.w1;
  d.b1 = a.b1;
  d.w2 = a.w2;
  d.b2 = a.b2;
  d.w3 = a.w3;
  d.b3 = d.w3 + (long long)d.N4 * d.NO;
  d.total = d.b3 + d.NO;
  return d;
}

bool cbm_net_ok(int M, int K) { return M > 0 && M % 6 == 0 && M <= kArMaxM && K >= 1 && K <= kCbmMaxK; }

int cbm_check_net(int M, int K) {
  if (M <= 0 || M % 6 != 0 || M > kArMaxM)
    return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be a positive multiple of 6 and at most %d", M,
                kArMaxM);
  if (K < 1 || K > kCbmMaxK) return fail(TFCB_INVALID_ARGUMENT, "`K` must be in [1, %d]: %d", kCbmMaxK, K);
  return TFCB_OK;
}

int cbm_check_packed(const float* packed, int64_t packed_floats, int M, int K) {
  if (!packed) return fail(TFCB_INVALID_ARGUMENT, "`packed` is null");
  const long long n = cbm_net(M, K).total;
  if (packed_floats != n)
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, M=%d with K=%d needs %lld",
                (long long)packed_floats, M, K, n);
  return TFCB_OK;
}

long long cbm_work_floats(const CbmNet& d, int M, const CbList& L, int colour) {
  return cb_table_floats(L) + cb_positions(L, colour) * ((colour ? 2 * M : 0) + d.N3 + d.N4 + d.NO);
}

template <int IN>
__global__ void __launch_bounds__(kCbThreads) cbm_dense_kernel(const CbPass S, const CbLayer L) {
  cb_dense<IN, kOutHidden, CbSchedule>(S, L);
}

// The epilogue of one pass: raw [P, 3KM] -> weight / loc / scale at (row + c) K .. (row + c) K + K - 1.
struct CbmEpilogue {
  const float* raw;
  int M, K, W, colour;
  long long P, n_k, HW, out_stride, out_base;  // (fixed shape: B images of H × W, rows as CbPass)
  const CbImage* img;                          // a ragged list, or null
  int n_img;
  float* weight;
  float* loc;
  float* scale;
  const float* y;  // encoder: y [.., M] in, y in coding order and ŷ out (else null)
  float* y_cb;
  float* yhat;
};

__global__ void __launch_bounds__(256) cbm_epilogue_kernel(const CbmEpilogue E) {
  const long long total = E.P * E.M;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
       e += (long long)gridDim.x * blockDim.x) {
    const long long p = e / E.M;
    const int ch = (int)(e - p * E.M), K = E.K;
    long long row, j, pix0;
    int W;
    if (E.img) {
      const CbImage im = E.img[cb_image_of(E.img, E.n_img, p)];
      j = p - im.q;
      row = im.out + j * E.M;
      W = im.W;
      pix0 = im.pix;
    } else {
      const long long b = p / E.n_k;
      j = p - b * E.n_k;
      row = b * E.out_stride + E.out_base + j * E.M;
      W = E.W;
      pix0 = b * E.HW;
    }
    const float* r = E.raw + p * (3ll * K * E.M) + 3ll * K * ch;
    const long long at = (row + ch) * K;
    float m = __ldg(r);
    for (int k = 1; k < K; ++k) m = fmaxf(m, __ldg(r + k));
    for (int k = 0; k < K; ++k) {
      E.weight[at + k] = expf(__fsub_rn(__ldg(r + k), m));
      E.loc[at + k] = __ldg(r + K + k);
      E.scale[at + k] = fmaxf(__ldg(r + 2 * K + k), kCbmScaleMin);
    }
    if (E.y) {
      int rr, cc;
      cb_position(j, W, E.colour, &rr, &cc);
      const long long src = (pix0 + (long long)rr * W + cc) * E.M + ch;
      const float yv = __ldg(E.y + src);
      E.y_cb[row + ch] = yv;
      E.yhat[src] = (float)(int)rintf(yv);
    }
  }
}

template <int IN>
int cbm_layer(const CbPass& S, const CbLayer& L, cudaStream_t s) {
  const dim3 grid((unsigned)((S.P + kCbTP - 1) / kCbTP), (unsigned)((L.N + kCbTN - 1) / kCbTN));
  cbm_dense_kernel<IN><<<grid, kCbThreads, 0, s>>>(S, L);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// One pass over colour `colour` of the images I, after the caller's checks of M, K, the packed size and the images.
// Outputs per pass, image i's n_k,i M rows at M Q_i (whole == 0), or in the coding order of both colours, image i's
// at M P_i + (colour ? n_a,i M : 0) (whole != 0); weight / loc / scale hold K floats per row.
int cbm_run(const float* packed, int M, int K, const float* yhat, const float* psi, const CbList& I, int colour,
            float* work, int64_t work_floats, int whole, float* weight, float* loc, float* scale, const float* y,
            float* y_cb, float* yhat_out, void* stream) {
  if (!psi || (colour && !yhat)) return fail(TFCB_INVALID_ARGUMENT, "`psi` or `yhat` is null");
  const CbmNet d = cbm_net(M, K);
  const long long need = cbm_work_floats(d, M, I, colour);
  if (!work || work_floats < need)
    return fail(TFCB_INVALID_ARGUMENT, "workspace of %lld floats, this pass needs %lld", work ? (long long)work_floats : 0ll,
                need);
  if (I.hs) TFCB_TRY(ar_check_table_space(work, work_floats, need, alignof(CbImage)));
  const long long P = cb_positions(I, colour);
  if (P == 0) return TFCB_OK;  // (the non-anchors of 1x1 latents: empty outputs may have null pointers)
  if (!weight || !loc || !scale) return fail(TFCB_INVALID_ARGUMENT, "`weight`, `loc` or `scale` is null");
  if (y && (!y_cb || !yhat_out)) return fail(TFCB_INVALID_ARGUMENT, "the encoder needs `y_cb` and `yhat_out`");
  cudaStream_t s = as_stream(stream);
  CbPass S{};
  S.B = (int)I.B;
  S.M = M;
  S.C = M;
  S.colour = colour;
  S.P = P;
  CbmEpilogue E{};
  if (I.hs) {
    TFCB_TRY(cb_upload_table(I, M, 0, M, colour, whole, work, s));
    S.img = E.img = reinterpret_cast<const CbImage*>(work);
    S.n_img = E.n_img = (int)I.B;
  } else {
    S.H = (int)I.H;
    S.W = E.W = (int)I.W;
    S.n_k = E.n_k = cb_count(I.H, I.W, colour);
    S.HW = E.HW = I.H * I.W;
    E.out_stride = whole ? E.HW * M : E.n_k * M;
    E.out_base = whole && colour ? cb_count(I.H, I.W, 0) * M : 0;
  }
  S.psi = psi;
  S.yhat = yhat;
  float* ctx = work + cb_table_floats(I);
  float* h1 = ctx + (colour ? P * 2 * M : 0);
  float* h2 = h1 + P * d.N3;
  float* raw = h2 + P * d.N4;
  if (colour)
    TFCB_TRY(cbm_layer<kInTaps>(S, {packed + d.wc, packed + d.bc, nullptr, ctx, kArTaps * M, 2 * M, kArTaps * M, false},
                                s));
  TFCB_TRY(cbm_layer<kInPsiCtx>(
      S, {packed + d.w1, packed + d.b1, ctx, h1, d.K1, d.N3, colour ? d.K1 : d.K1 - 2 * M, true}, s));
  TFCB_TRY(cbm_layer<kInPlain>(S, {packed + d.w2, packed + d.b2, h1, h2, d.N3, d.N4, d.N3, true}, s));
  TFCB_TRY(cbm_layer<kInPlain>(S, {packed + d.w3, packed + d.b3, h2, raw, d.N4, d.NO, d.N4, false}, s));
  E.raw = raw;
  E.M = M;
  E.K = K;
  E.colour = colour;
  E.P = P;
  E.weight = weight;
  E.loc = loc;
  E.scale = scale;
  E.y = y;
  E.y_cb = y_cb;
  E.yhat = yhat_out;
  const long long blocks = std::min<long long>((P * M + 255) / 256, 1ll << 16);
  cbm_epilogue_kernel<<<(unsigned)blocks, 256, 0, s>>>(E);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

int64_t tfcb_cbm_packed_floats(int M, int K, int64_t* layout) {
  if (!cbm_net_ok(M, K)) return -1;
  const CbmNet d = cbm_net(M, K);
  if (layout) {
    const int64_t v[12] = {d.K1, d.N3, d.N4, d.NO, d.wc, d.bc, d.w1, d.b1, d.w2, d.b2, d.w3, d.b3};
    for (int i = 0; i < 12; ++i) layout[i] = v[i];
  }
  return d.total;
}

int tfcb_cbm_pack_weights(int M, int K, const float* ctx_taps_dev, const float* ctx_bias_dev, const float* w1_dev,
                          const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                          const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream) {
  TFCB_TRY(cbm_check_net(M, K));
  const CbmNet d = cbm_net(M, K);
  if (packed_floats != d.total)
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, M=%d with K=%d needs %lld",
                (long long)packed_floats, M, K, (long long)d.total);
  const float* src[8] = {ctx_taps_dev, ctx_bias_dev, w1_dev, b1_dev, w2_dev, b2_dev, w3_dev, b3_dev};
  const long long at[9] = {d.wc, d.bc, d.w1, d.b1, d.w2, d.b2, d.w3, d.b3, d.total};
  return ar_pack_segments(src, at, packed_dev, as_stream(stream));
}

int64_t tfcb_cbm_workspace_floats(int M, int K, int64_t B, int64_t H, int64_t W, int anchors) {
  if (!cbm_net_ok(M, K) || B <= 0 || B > 0x7FFFFFFF || H <= 0 || W <= 0 || H * W > 0x7FFFFFFF) return -1;
  return cbm_work_floats(cbm_net(M, K), M, {B, H, W, nullptr, nullptr}, anchors ? 0 : 1);
}

int tfcb_cbm_params(const float* packed_dev, int64_t packed_floats, int M, int K, const float* yhat_dev,
                    const float* psi_dev, int64_t B, int64_t H, int64_t W, int anchors, float* work_dev,
                    int64_t work_floats, int whole, float* weight_dev, float* loc_dev, float* scale_dev,
                    const float* y_dev, float* y_cb_dev, float* yhat_out_dev, void* stream) {
  TFCB_TRY(cbm_check_net(M, K));
  TFCB_TRY(cbm_check_packed(packed_dev, packed_floats, M, K));
  TFCB_TRY(ar_check_batch(B, H, W, 1));
  return cbm_run(packed_dev, M, K, yhat_dev, psi_dev, {B, H, W, nullptr, nullptr}, anchors ? 0 : 1, work_dev,
                 work_floats, whole, weight_dev, loc_dev, scale_dev, y_dev, y_cb_dev, yhat_out_dev, stream);
}

int64_t tfcb_cbm_ragged_workspace_floats(int M, int K, int64_t n_images, const int64_t* heights_host,
                                         const int64_t* widths_host, int anchors) {
  if (!cbm_net_ok(M, K) || !ar_list_ok(n_images, heights_host, widths_host)) return -1;
  return cbm_work_floats(cbm_net(M, K), M, {n_images, 0, 0, heights_host, widths_host}, anchors ? 0 : 1);
}

int tfcb_cbm_params_ragged(const float* packed_dev, int64_t packed_floats, int M, int K, const float* yhat_dev,
                           const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                           const int64_t* widths_host, int anchors, float* work_dev, int64_t work_floats, int whole,
                           float* weight_dev, float* loc_dev, float* scale_dev, const float* y_dev, float* y_cb_dev,
                           float* yhat_out_dev, void* stream) {
  TFCB_TRY(cbm_check_net(M, K));
  TFCB_TRY(cbm_check_packed(packed_dev, packed_floats, M, K));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, 1));
  return cbm_run(packed_dev, M, K, yhat_dev, psi_dev, {n_images, 0, 0, heights_host, widths_host}, anchors ? 0 : 1,
                 work_dev, work_floats, whole, weight_dev, loc_dev, scale_dev, y_dev, y_cb_dev, yhat_out_dev, stream);
}

}  // extern "C"
