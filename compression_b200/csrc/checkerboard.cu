// Checkerboard context model (He, Zheng, Sun, Wang & Qin, CVPR 2021) on sm_90a: the entropy parameters of one
// colour of latent positions, all images and positions of that colour at once.
//
// A position (r, c) is an anchor when r + c is even, else a non-anchor.  An image codes its anchors in raster order,
// then its non-anchors in raster order ("coding order"); the j-th position of colour k (0 anchors, 1 non-anchors)
// lies in row 2 (j / W) or 2 (j / W) + 1, see cb_position.  Per position (N2 = 2M, N3 = 10M/3, N4 = 8M/3):
//   ctx   = 0 at an anchor (bias included); at a non-anchor bc + Wc · gather(ŷ, the 12 taps (dy, dx) in [-2, 2]^2
//           with dy + dx odd, raster order, zeros outside the image), every tap an anchor            [12M] -> [2M]
//   h1    = leaky(b1 + W1 · [ψ_p, ctx])                                                              [4M]  -> [N3]
//   h2    = leaky(b2 + W2 · h1)                                                                      [N3]  -> [N4]
//   out   = b3 + W3 · h2 = [loc, scale_index]                                                        [N4]  -> [2M]
// with the packed weights of tfcb_ar_pack_weights (Wc: the 12 checkerboard taps, gathered by the caller).
//
// Every output is autoregressive.cu's fixed sequence of float32 operations: bias first, then the eight slices
// [s·K/8, (s+1)·K/8) in order, each an __fmaf_rn chain from +0.f in increasing k, added with __fadd_rn, then the
// LeakyReLU.  So an output depends only on its own position's inputs, never on the tile, the grid, B or the SM count.
// At an anchor, layer 1's slices 4-7 are exactly the ctx half [2M, 4M) (4M/8 = M/2), whose chains over zeros are +0
// for finite weights: they are skipped and +0.f is added in their place (turning a -0 sum into +0, as the chain would).
//
// A pass is one launch per layer (three at anchors, four at non-anchors).  A CTA computes a tile of kCbTP positions ×
// kCbTN output columns of one layer, staging kCbKC inputs of each position and the matching weight rows in shared
// memory, so that each weight loaded from L2 serves kCbTP positions and a 32×48 image spreads over the SMs by
// position tiles and column tiles alike.  The layers' outputs go through a caller-provided workspace.
#include <cuda_runtime.h>

#include <algorithm>

#include "autoregressive.cuh"
#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kCbTP = 32;        // positions per tile
constexpr int kCbTN = 64;        // output columns per tile
constexpr int kCbKC = 32;        // inputs per shared-memory stage
constexpr int kCbThreads = 256;  // thread (ty, tx) = (tid / 32, tid % 32): positions 4ty..4ty+3, columns tx, tx + 32

// the checkerboard taps in raster order: (dy, dx) in [-2, 2]^2 with dy + dx odd
__constant__ int8_t c_cb_dy[kArTaps] = {-2, -2, -1, -1, -1, 0, 0, 1, 1, 1, 2, 2};
__constant__ int8_t c_cb_dx[kArTaps] = {-1, 1, -2, 0, 2, -1, 1, -2, 0, 2, -1, 1};

enum : int { kInTaps = 0, kInPsiCtx = 1, kInPlain = 2 };  // what a layer reads
enum : int { kOutHidden = 0, kOutParams = 1 };             // what it writes

struct CbPass {
  int B, H, W, M, colour, num_scales;
  long long n_k, n_a, HW, P;  // positions of this colour per image, anchors per image, H·W, B·n_k
  const float* psi;           // [B, H, W, 2M]
  const float* yhat;          // [B, H, W, M]: the non-anchor pass gathers the anchors' ŷ
  // params epilogue: [B, out_rows, M] with this pass's rows at out_row0 + j
  long long out_rows, out_row0;
  float* loc;
  float* scale;
  int32_t* index;
  // encoder epilogue (y non-null): y [B, H, W, M] in, y in coding order and ŷ [B, H, W, M] out
  const float* y;
  float* y_cb;
  float* yhat_out;
};

struct CbLayer {
  const float* W;  // [K, N]
  const float* bias;
  const float* in;  // kInPsiCtx: ctx [P, 2M]; kInPlain: [P, K]
  float* out;       // kOutHidden: [P, N]
  int K, N;
  bool leaky, ctx_zero;  // ctx_zero: layer 1 at anchors
};

// the j-th position of colour k of an image of width W, in raster order
__host__ __device__ inline void cb_position(long long j, int W, int k, int* r, int* c) {
  const long long pair = j / W;
  const int rem = (int)(j - pair * W), even = (W + 1 - k) / 2;  // positions of colour k in an even row
  if (rem < even) {
    *r = (int)(2 * pair);
    *c = 2 * rem + k;
  } else {
    *r = (int)(2 * pair + 1);
    *c = 2 * (rem - even) + 1 - k;
  }
}

template <int IN, int OUT>
__global__ void __launch_bounds__(kCbThreads) cb_dense_kernel(const CbPass S, const CbLayer L) {
  __shared__ __align__(16) float xs[kCbKC][kCbTP + 4];  // (+4: a stage's stores hit 8 banks, rows stay 16-byte aligned)
  __shared__ __align__(16) float ws[kCbKC][kCbTN];
  __shared__ long long s_pix[kCbTP];  // b·H·W + r·W + c, or -1 past the last position
  __shared__ long long s_row[kCbTP];  // the position's row of the params outputs
  __shared__ int s_r[kCbTP], s_c[kCbTP];
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const long long p0 = (long long)blockIdx.x * kCbTP;
  const int j0 = blockIdx.y * kCbTN;
  if (tid < kCbTP) {
    const long long p = p0 + tid;
    long long pix = -1, row = 0;
    int r = 0, c = 0;
    if (p < S.P) {
      const long long b = p / S.n_k;
      cb_position(p - b * S.n_k, S.W, S.colour, &r, &c);
      pix = b * S.HW + (long long)r * S.W + c;
      row = b * S.out_rows + S.out_row0 + (p - b * S.n_k);
    }
    s_pix[tid] = pix;
    s_row[tid] = row;
    s_r[tid] = r;
    s_c[tid] = c;
  }
  __syncthreads();
  const int K = L.K, N = L.N, M = S.M;
  float v[4][2], acc[4][2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int j = j0 + tx + 32 * q;
    const float bj = j < N ? __ldg(L.bias + j) : 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i][q] = bj;
  }
  for (int s = 0; s < kArSlices; ++s) {
    const int k0 = s * K / kArSlices, k1 = (s + 1) * K / kArSlices;
    if (L.ctx_zero && s >= kArSlices / 2) {  // the ctx half of [ψ, ctx] at an anchor: a chain over zeros is +0
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 2; ++q) v[i][q] = __fadd_rn(v[i][q], 0.f);
      continue;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int q = 0; q < 2; ++q) acc[i][q] = 0.f;
    for (int kc = k0; kc < k1; kc += kCbKC) {
      const int n = min(kCbKC, k1 - kc);
      __syncthreads();  // the previous stage's reads are done
      for (int e = tid; e < kCbTP * kCbKC; e += kCbThreads) {
        const int pp = e / kCbKC, kk = e - pp * kCbKC;
        const long long pix = s_pix[pp];
        float x = 0.f;
        if (kk < n && pix >= 0) {
          const int k = kc + kk;
          if (IN == kInTaps) {
            const int t = k / M, ch = k - t * M;
            const int rr = s_r[pp] + c_cb_dy[t], cc = s_c[pp] + c_cb_dx[t];
            if (rr >= 0 && rr < S.H && cc >= 0 && cc < S.W)
              x = S.yhat[(pix + (long long)c_cb_dy[t] * S.W + c_cb_dx[t]) * M + ch];
          } else if (IN == kInPsiCtx) {
            x = k < 2 * M ? __ldg(S.psi + pix * (2 * M) + k) : L.in[(p0 + pp) * (2 * M) + (k - 2 * M)];
          } else {
            x = L.in[(p0 + pp) * K + k];
          }
        }
        xs[kk][pp] = x;
      }
      for (int e = tid; e < kCbKC * kCbTN; e += kCbThreads) {
        const int kk = e / kCbTN, jj = e - kk * kCbTN;
        ws[kk][jj] = (kk < n && j0 + jj < N) ? __ldg(L.W + (long long)(kc + kk) * N + j0 + jj) : 0.f;
      }
      __syncthreads();
      for (int kk = 0; kk < n; ++kk) {
        const float4 x4 = *reinterpret_cast<const float4*>(&xs[kk][4 * ty]);
        const float w0 = ws[kk][tx], w1 = ws[kk][tx + 32];
        const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[i][0] = __fmaf_rn(xv[i], w0, acc[i][0]);
          acc[i][1] = __fmaf_rn(xv[i], w1, acc[i][1]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int q = 0; q < 2; ++q) v[i][q] = __fadd_rn(v[i][q], acc[i][q]);
  }
  // ---- epilogue ----
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int pp = 4 * ty + i;
    const long long p = p0 + pp, pix = s_pix[pp];
    if (pix < 0) continue;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int j = j0 + tx + 32 * q;
      if (j >= N) continue;
      float val = v[i][q];
      if (L.leaky) val = val > 0.f ? val : __fmul_rn(val, kArLeakySlope);
      if (OUT == kOutHidden) {
        L.out[p * N + j] = val;
        continue;
      }
      const long long row = s_row[pp] * M;
      if (j < M) {
        if (S.loc) S.loc[row + j] = val;
        if (S.y) {
          const float yv = __ldg(S.y + pix * M + j);
          const int q32 = (int)rintf(__fsub_rn(yv, val));
          S.yhat_out[pix * M + j] = __fadd_rn((float)q32, val);
          S.y_cb[row + j] = yv;
        }
      } else {
        if (S.scale) S.scale[row + j - M] = val;
        if (S.index) S.index[row + j - M] = ar_table_index(val, S.num_scales);
      }
    }
  }
}

// ŷ of one colour, [B, n_k, M] in coding order -> its positions of [B, H, W, M]
__global__ void cb_scatter_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n_k, int W,
                                  long long HW, int M, int colour, long long total) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / M, b = row / n_k;
    int r, c;
    cb_position(row - b * n_k, W, colour, &r, &c);
    dst[(b * HW + (long long)r * W + c) * M + (e - row * M)] = src[e];
  }
}

long long cb_count(int64_t H, int64_t W, int colour) { return colour ? H * W / 2 : (H * W + 1) / 2; }

long long cb_work_floats(int M, int64_t B, int64_t H, int64_t W, int colour) {
  const ArDims d = ar_dims(M);
  return B * cb_count(H, W, colour) * ((colour ? d.N2 : 0) + d.N3 + d.N4);
}

template <int IN, int OUT>
int cb_layer(const CbPass& S, const CbLayer& L, cudaStream_t s) {
  const dim3 grid((unsigned)((S.P + kCbTP - 1) / kCbTP), (unsigned)((L.N + kCbTN - 1) / kCbTN));
  cb_dense_kernel<IN, OUT><<<grid, kCbThreads, 0, s>>>(S, L);
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
  return cb_work_floats(M, B, H, W, anchors ? 0 : 1);
}

int tfcb_cb_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int anchors, int num_scales, float* work_dev,
                   int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev,
                   const float* y_dev, float* y_cb_dev, float* yhat_out_dev, void* stream) {
  TFCB_TRY(ar_check(M, packed_dev, packed_floats, B, H, W, num_scales));
  const int colour = anchors ? 0 : 1;
  if (!psi_dev || (colour && !yhat_dev)) return fail(TFCB_INVALID_ARGUMENT, "`psi` or `yhat` is null");
  const long long need = cb_work_floats(M, B, H, W, colour);
  if (!work_dev || work_floats < need)
    return fail(TFCB_INVALID_ARGUMENT, "workspace of %lld floats, this pass needs %lld",
                work_dev ? (long long)work_floats : 0ll, need);
  if (y_dev && (!y_cb_dev || !yhat_out_dev || !loc_dev || !index_dev))
    return fail(TFCB_INVALID_ARGUMENT, "the encoder needs `y_cb`, `yhat_out`, `loc` and `index`");
  const long long n_k = cb_count(H, W, colour);
  if (n_k == 0) return TFCB_OK;
  const ArDims d = ar_dims(M);
  CbPass S{};
  S.B = (int)B;
  S.H = (int)H;
  S.W = (int)W;
  S.M = M;
  S.colour = colour;
  S.num_scales = num_scales;
  S.n_k = n_k;
  S.n_a = cb_count(H, W, 0);
  S.HW = H * W;
  S.P = B * n_k;
  S.psi = psi_dev;
  S.yhat = yhat_dev;
  S.out_rows = whole ? H * W : n_k;
  S.out_row0 = whole && colour ? S.n_a : 0;
  S.loc = loc_dev;
  S.scale = scale_index_dev;
  S.index = index_dev;
  S.y = y_dev;
  S.y_cb = y_cb_dev;
  S.yhat_out = yhat_out_dev;
  float* ctx = work_dev;
  float* h1 = ctx + (colour ? S.P * d.N2 : 0);
  float* h2 = h1 + S.P * d.N3;
  const float* Wp = packed_dev;
  cudaStream_t s = as_stream(stream);
  if (colour)
    TFCB_TRY((cb_layer<kInTaps, kOutHidden>(S, {Wp + d.wc, Wp + d.bc, nullptr, ctx, kArTaps * M, d.N2, false, false},
                                            s)));
  TFCB_TRY((cb_layer<kInPsiCtx, kOutHidden>(S, {Wp + d.w1, Wp + d.b1, ctx, h1, 4 * M, d.N3, true, !colour}, s)));
  TFCB_TRY((cb_layer<kInPlain, kOutHidden>(S, {Wp + d.w2, Wp + d.b2, h1, h2, d.N3, d.N4, true, false}, s)));
  return cb_layer<kInPlain, kOutParams>(S, {Wp + d.w3, Wp + d.b3, h2, nullptr, d.N4, d.N2, false, false}, s);
}

int tfcb_cb_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int anchors, float* dst_dev,
                    void* stream) {
  if (M <= 0) return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be positive", M);
  if (B <= 0 || B > 0x7FFFFFFF) return fail(TFCB_INVALID_ARGUMENT, "batch size %lld out of range", (long long)B);
  if (H <= 0 || W <= 0 || H * W > 0x7FFFFFFF)
    return fail(TFCB_INVALID_ARGUMENT, "latent shape %lld x %lld out of range", (long long)H, (long long)W);
  const int colour = anchors ? 0 : 1;
  const long long n_k = cb_count(H, W, colour), total = B * n_k * M;
  if (total == 0) return TFCB_OK;  // (the non-anchors of a 1x1 latent: empty tensors may have null pointers)
  if (!src_dev || !dst_dev) return fail(TFCB_INVALID_ARGUMENT, "`src` or `dst` is null");
  const long long blocks = std::min<long long>((total + 255) / 256, 1ll << 16);
  cb_scatter_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(src_dev, dst_dev, n_k, (int)W, H * W, M, colour,
                                                                     total);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

}  // extern "C"
