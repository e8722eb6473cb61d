// The tile machinery of the position-parallel context models: one dense layer of the entropy-parameter network over
// every position of one pass, kCbTP positions × kCbTN output columns per CTA, and the scatter of a pass's latents
// from coding order back to [B, H, W, M].  checkerboard.cu runs it over the checkerboard's colours (and the
// space-channel model's groups), multistage.cu over the four stages of the 2×2 schedule.  A pass's schedule is a
// compile-time policy with two members:
//   position(j, W, phase, &r, &c): the j-th position of pass `phase` of an image of width W, in raster order;
//   dy(phase, t), dx(phase, t):    the t-th context tap of pass `phase` (read only by kInTaps layers).
// Every output is autoregressive.cu's fixed sequence of float32 operations: bias first, then the eight slices
// [s·K/8, (s+1)·K/8) in order, each an __fmaf_rn chain from +0.f in increasing k, added with __fadd_rn, then the
// LeakyReLU.  So an output depends only on its own position's inputs, never on the tile, the grid, B or the SM count.
// A slice that lies wholly in [zero_from, K) of a kInPsiCtx layer (the ctx segment of a pass without context) is a
// chain over zeros, which is +0 for finite weights: it is skipped and +0.f is added in its place.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "autoregressive.cuh"
#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kCbTP = 32;        // positions per tile
constexpr int kCbTN = 64;        // output columns per tile
constexpr int kCbKC = 32;        // inputs per shared-memory stage
constexpr int kCbThreads = 256;  // thread (ty, tx) = (tid / 32, tid % 32): positions 4ty..4ty+3, columns tx, tx + 32

enum : int { kInTaps = 0, kInPsiCtx = 1, kInPlain = 2 };  // what a layer reads
enum : int { kOutHidden = 0, kOutParams = 1 };             // what it writes

// One image of a ragged list (§3.13): its first position of this pass (Q_i), its first pixel (P_i), its shape and
// the first element of its params outputs.
struct CbImage {
  long long q, pix, out;
  int H, W;
};

struct CbPass {
  int B, H, W, M, C, o, CH, colour, num_scales;  // latent depth M; the group's C channels from o; CH: chctx width;
                                                 // colour: the pass's phase (checkerboard colour, multistage stage)
  long long n_k, HW, P;                          // positions of this pass per image, H·W, B·n_k (ragged: Σ n_k,i)
  const CbImage* img;                            // a ragged list of n_img images, or null: B images of H × W
  int n_img;
  const float* psi;                              // [B, H, W, 2M]
  const float* chctx;                            // [B, H, W, CH] (CH > 0)
  const float* yhat;                             // [B, H, W, M]: a pass with taps gathers earlier passes' ŷ
  // params epilogue: channel c of this pass's j-th position of image b at out_stride·b + out_base + C·j + c
  long long out_stride, out_base;
  float* loc;
  float* scale;
  int32_t* index;
  // encoder epilogue (y non-null): y [B, H, W, M] in, y in coding order and ŷ [B, H, W, M] out, at channels o + c
  const float* y;
  float* y_cb;
  float* yhat_out;
};

struct CbLayer {
  const float* W;  // [K, N]
  const float* bias;
  const float* in;  // kInPsiCtx: ctx [P, 2C]; kInPlain: [P, K]
  float* out;       // kOutHidden: [P, N]
  int K, N;
  int zero_from;    // kInPsiCtx: inputs [zero_from, K) are zeros (the ctx segment of a pass without context), else K
  bool leaky;
};

// the image of a ragged list holding the pass's position p: the last i with img[i].q <= p (an image with no
// positions of this pass shares its q with the next one and is never chosen)
__device__ inline int cb_image_of(const CbImage* img, int n_img, long long p) {
  int lo = 0, hi = n_img - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&img[mid].q) <= p)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// One CTA of one dense layer of a pass (the body of each file's dense kernel).
template <int IN, int OUT, class Sched>
__device__ __forceinline__ void cb_dense(const CbPass& S, const CbLayer& L) {
  __shared__ __align__(16) float xs[kCbKC][kCbTP + 4];  // (+4: a stage's stores hit 8 banks, rows stay 16-byte aligned)
  __shared__ __align__(16) float ws[kCbKC][kCbTN];
  __shared__ long long s_pix[kCbTP];  // b·H·W + r·W + c, or -1 past the last position
  __shared__ long long s_row[kCbTP];  // the position's first element of the params outputs
  __shared__ int s_r[kCbTP], s_c[kCbTP];
  __shared__ int s_h[kCbTP], s_w[kCbTP];  // the position's image shape (a tile may straddle images of a list)
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const long long p0 = (long long)blockIdx.x * kCbTP;
  const int j0 = blockIdx.y * kCbTN;
  if (tid < kCbTP) {
    const long long p = p0 + tid;
    long long pix = -1, row = 0;
    int r = 0, c = 0, h = S.H, w = S.W;
    if (p < S.P) {
      if (S.img) {
        const CbImage im = S.img[cb_image_of(S.img, S.n_img, p)];
        h = im.H;
        w = im.W;
        Sched::position(p - im.q, w, S.colour, &r, &c);
        pix = im.pix + (long long)r * w + c;
        row = im.out + (p - im.q) * S.C;
      } else {
        const long long b = p / S.n_k;
        Sched::position(p - b * S.n_k, S.W, S.colour, &r, &c);
        pix = b * S.HW + (long long)r * S.W + c;
        row = b * S.out_stride + S.out_base + (p - b * S.n_k) * S.C;
      }
    }
    s_pix[tid] = pix;
    s_row[tid] = row;
    s_r[tid] = r;
    s_c[tid] = c;
    s_h[tid] = h;
    s_w[tid] = w;
  }
  __syncthreads();
  const int K = L.K, N = L.N, C = S.C;
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
    if (k0 >= L.zero_from) {  // wholly in the ctx segment of a pass without context: a chain over zeros is +0
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
            const int t = k / C, ch = k - t * C;
            const int rr = s_r[pp] + Sched::dy(S.colour, t), cc = s_c[pp] + Sched::dx(S.colour, t), w = s_w[pp];
            if (rr >= 0 && rr < s_h[pp] && cc >= 0 && cc < w)
              x = S.yhat[(pix + (long long)Sched::dy(S.colour, t) * w + Sched::dx(S.colour, t)) * S.M + S.o + ch];
          } else if (IN == kInPsiCtx) {
            const int PW = 2 * S.M, CH = S.CH;
            if (k < PW)
              x = __ldg(S.psi + pix * PW + k);
            else if (k < PW + CH)
              x = __ldg(S.chctx + pix * CH + (k - PW));
            else if (k < L.zero_from)
              x = L.in[(p0 + pp) * (2 * C) + (k - PW - CH)];
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
      const long long row = s_row[pp];
      if (j < C) {
        if (S.loc) S.loc[row + j] = val;
        if (S.y) {
          const long long at = pix * S.M + S.o + j;
          const float yv = __ldg(S.y + at);
          const int q32 = (int)rintf(__fsub_rn(yv, val));
          S.yhat_out[at] = __fadd_rn((float)q32, val);
          S.y_cb[row + j] = yv;
        }
      } else {
        if (S.scale) S.scale[row + j - C] = val;
        if (S.index) S.index[row + j - C] = ar_table_index(val, S.num_scales);
      }
    }
  }
}

// The scatter body: ŷ of one pass of group [o, o + C), [B, n_k, C] in coding order -> its positions and channels of
// [B, H, W, M]; with `img` (a ragged list of n_img images) image i's n_k,i C values at C q_i -> its [H_i, W_i, M] at
// M pix_i.
template <class Sched>
__device__ __forceinline__ void cb_scatter(const float* __restrict__ src, float* __restrict__ dst, long long n_k, int W,
                                           long long HW, int M, int o, int C, int colour, long long total,
                                           const CbImage* __restrict__ img, int n_img) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long row = e / C;
    int r, c;
    long long pix;
    if (img) {
      const CbImage im = img[cb_image_of(img, n_img, row)];
      Sched::position(row - im.q, im.W, colour, &r, &c);
      pix = im.pix + (long long)r * im.W + c;
    } else {
      const long long b = row / n_k;
      Sched::position(row - b * n_k, W, colour, &r, &c);
      pix = b * HW + (long long)r * W + c;
    }
    dst[pix * M + o + (e - row * C)] = src[e];
  }
}

// The images of a call: B of H × W (hs null), or a ragged list of B images of hs[i] × ws[i] (§3.13).
struct CbList {
  int64_t B, H, W;
  const int64_t* hs;
  const int64_t* ws;
};

// floats of a ragged list's image table at the start of the workspace
long long cb_table_floats(const CbList& L) { return L.hs ? L.B * (long long)(sizeof(CbImage) / sizeof(float)) : 0; }

}  // namespace
}  // namespace tfcb
