// SSIM / MS-SSIM statistics of tf.image.ssim and tf.image.ssim_multiscale (tensorflow/python/ops/image_ops_impl.py),
// forward and backward, fused.
//
// Per (image, channel, scale) the forward writes mean(cs) and mean(l * cs) over the VALID positions of a size x size
// Gaussian window (the softmax of -(i^2 + j^2) / (2 sigma^2), i.e. the outer product of two normalised 1-D Gaussians,
// applied separably):
//   l  = (2 mx my + c1) / (mx^2 + my^2 + c1)
//   cs = (2 (Sxy - mx my) + c2) / (S(x^2 + y^2) - mx^2 - my^2 + c2)
// with mx, my the windowed means and S(.) the windowed second moments.  Scale s + 1 is scale s padded at its end by
// one repeated row / column where odd, then 2x2 average pooled (TF's SYMMETRIC pad by the remainder + VALID avg_pool).
// The host combines the statistics (ReLU, pow, prod, channel mean) in torch; the backward turns the gradient of the
// statistics into gradients of the two images.
//
// Layout: images are channels-last [n_images, H, W, C] in their own dtype (uint8 widened as convert_image_dtype does,
// float32(u) * float32(1/255)); the pooled scales live in the workspace as planar float32 [n_images * C, Hs, Ws].  A
// plane is one (image, channel); element (r, c) of plane p is at ((p / cs) * Hs * Ws + r * Ws + c) * cs + p % cs with
// cs = C for the input and 1 for the pyramid, so one kernel reads both.  The forward also takes a list of images of
// their own sizes (tfcb_image_metrics_ragged): it runs from a table of per-image rows, the batch being its uniform
// case, can read Y' or Y'CbCr planes made from RGB as it loads scale 0, and can add the squared error of scale 0.
//
// Precision: the moments are filtered in double on values shifted by a per-tile constant (the mean of the two images
// at the tile's first pixel) and the shift is added back into the means.  The variances and the covariance are
// shift-invariant, so a bright flat region does not lose its digits to S(x^2) - mx^2.  The products feeding the
// second moments are rounded without contraction, so identical images give l = cs = 1 exactly.
//
// Determinism: each CTA covers one output tile of one plane and writes its sums as a double partial; one reduction
// kernel adds the partials of a plane in tile order.  Every gradient element is written by one thread.  A CTA's work
// depends on its (image, plane, tile) only (the forward walks that list by a grid-stride loop, the backward its planes
// in y), so an image's results do not depend on the batch or list it is in, and the launch count depends on the
// number of scales only.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kThreads = 256;
constexpr int kFwdTile = 32;  // forward output tile (kFwdTile x kFwdTile valid positions)
constexpr int kBwdTile = 16;  // backward output tile (one thread per input position)
constexpr int kMaxFilter = 32;
constexpr int kMaxScales = 16;
constexpr int kMaxPlaneBlocks = 65535;

struct Window {
  double g[kMaxFilter];  // normalised 1-D Gaussian (in double: float32 weights would not sum to 1 closely enough
                         // for the shifted variances of flat regions at small c2)
  int size;
};

// ---- element access ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
// One rounded multiply, never contracted into a following add: the pool kernel's sum of converted texels must be
// convert_image_dtype's float32 values added, or the uint8 pyramid differs from the converted images' by roundings.
__device__ __forceinline__ float to_f32(uint8_t v) { return __fmul_rn((float)v, 1.0f / 255.0f); }

template <typename T>
__device__ __forceinline__ T from_f32(float v);
template <>
__device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
__device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

struct Plane {
  long long base;  // offset of element (0, 0)
  int row, col;    // element strides
  __device__ __forceinline__ long long at(int r, int c) const { return base + (long long)r * row + (long long)c * col; }
};
__device__ __forceinline__ Plane plane_of(int p, int cstride, int Hs, int Ws) {
  Plane q;
  q.base = (long long)(p / cstride) * Hs * Ws * cstride + p % cstride;
  q.row = Ws * cstride;
  q.col = cstride;
  return q;
}

__device__ __forceinline__ void load_window(const Window& w, double* gs) {
  if (threadIdx.x < w.size) gs[threadIdx.x] = w.g[threadIdx.x];
}

// ---- the SSIM terms at one position, from the shifted moments ------------------------------------------------
struct Terms {
  double mx, my, ux, uy;  // shifted means (ux, uy) and true means (mx, my)
  double d1, d2, l, cs;
};
__device__ __forceinline__ Terms terms(double ux, double uy, double q, double sxy, double shift, double c1, double c2) {
  Terms t;
  t.ux = ux;
  t.uy = uy;
  t.mx = ux + shift;
  t.my = uy + shift;
  const double mxy = __dmul_rn(t.mx, t.my);
  t.d1 = __dadd_rn(__dadd_rn(__dmul_rn(t.mx, t.mx), __dmul_rn(t.my, t.my)), c1);
  t.l = __dadd_rn(2.0 * mxy, c1) / t.d1;
  const double uxy = __dmul_rn(ux, uy);
  t.d2 = __dadd_rn(__dsub_rn(q, __dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy))), c2);
  t.cs = __dadd_rn(2.0 * __dsub_rn(sxy, uxy), c2) / t.d2;
  return t;
}

// ---- lists of image pairs --------------------------------------------------------------------------------------
// The forward runs over a list of image pairs with one dtype and one C but sizes of their own; a batch of same-sized
// images is the uniform case.  Per scale, item i has a row: `src` is the element offset of its first element in the
// scale's source (the channels-last input at scale 0, otherwise a planar float32 pyramid level holding each item's
// planes [planes][h][w], items back to back), and `first` is the index of its first forward CTA in the scale.  Both
// grow strictly with i, so a CTA or a pool output finds its item by a binary search.
struct ItemRow {
  long long src, first;
  int h, w;         // size at this scale
  int ntx, tiles;   // forward tiles per tile row and per plane
};

// The item holding v: the last row whose `key` is <= v.
template <long long ItemRow::*key>
__device__ __forceinline__ int find_item(const ItemRow* rows, int n, long long v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (rows[mid].*key <= v) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Planes of an item at scale 0: kRgb reads the C channels, kY makes one Y' plane and kYCbCr three Y'CbCr planes from
// C = 3 as the pixels are read, so no converted copy is written.  The pyramid levels are read as kRgb.
enum ColorMode { kRgb = TFCB_COLOR_RGB, kY = TFCB_COLOR_Y, kYCbCr = TFCB_COLOR_YCBCR };

// Plane `ch` of BT.601 full-range (JFIF) Y'CbCr in float32, every product and sum rounded in the order written (no
// contraction), so that image.rgb_to_ycbcr's torch expression gives the same bits.  off = float32(128/255) * max_val.
__device__ __forceinline__ float ycbcr(float r, float g, float b, int ch, float off) {
  if (ch == 0)
    return __fadd_rn(__fadd_rn(__fmul_rn((float)0.299, r), __fmul_rn((float)0.587, g)), __fmul_rn((float)0.114, b));
  if (ch == 1)
    return __fadd_rn(off, __fadd_rn(__fsub_rn(__fmul_rn((float)-0.168736, r), __fmul_rn((float)0.331264, g)),
                                    __fmul_rn(0.5f, b)));
  return __fadd_rn(off, __fsub_rn(__fsub_rn(__fmul_rn(0.5f, r), __fmul_rn((float)0.418688, g)),
                                  __fmul_rn((float)0.081312, b)));
}

// Plane p of an item, interleaved (cstride = C) or planar (cstride = 1); a converted plane addresses the pixel's
// first channel.
template <int kMode>
__device__ __forceinline__ Plane item_plane(const ItemRow& it, int p, int cstride) {
  Plane q;
  q.base = it.src + (kMode == kRgb ? (long long)(p / cstride) * it.h * it.w * cstride + p % cstride : 0);
  q.row = it.w * cstride;
  q.col = cstride;
  return q;
}

template <int kMode, typename T>
__device__ __forceinline__ float texel(const T* __restrict__ x, const Plane& P, int r, int c, int p, float off) {
  const long long i = P.at(r, c);
  if (kMode == kRgb) return to_f32(x[i]);
  return ycbcr(to_f32(x[i]), to_f32(x[i + 1]), to_f32(x[i + 2]), kMode == kY ? 0 : p, off);
}

// Deterministic CTA sum of three doubles; thread 0 gets the result.
__device__ __forceinline__ void block_sum3(double& a, double& b, double& c, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    red[3 * warp] = a;
    red[3 * warp + 1] = b;
    red[3 * warp + 2] = c;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = 0.0;
    b = 0.0;
    c = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) {
      a += red[3 * w];
      b += red[3 * w + 1];
      c += red[3 * w + 2];
    }
  }
}

// ---- forward: one output tile of one plane of one item per CTA ------------------------------------------------
// Shared memory: window [kMaxFilter] f64, x and y [R][R] f32 (R = kFwdTile + F - 1), horizontal sums [4][R][kFwdTile]
// f64, reduction scratch.
size_t fwd_smem(int F) {
  const int R = kFwdTile + F - 1;
  return 4 * (size_t)R * kFwdTile * sizeof(double) + 3 * (kThreads / 32) * sizeof(double) + kMaxFilter * sizeof(double) +
         2 * (size_t)R * R * sizeof(float);
}

// CTA u of the scale writes its sums of cs and l * cs to part[2u], part[2u + 1].  With `sq` it also writes to sq[u]
// the sum of (x - y)^2 over the pixels its tile owns: rows y0 .. y0 + kFwdTile - 1, or to the plane's end in the last
// tile row, and likewise for columns, so the tiles of a plane partition its pixels.
template <typename T, int kMode>
__global__ void __launch_bounds__(kThreads)
ssim_fwd_kernel(const T* __restrict__ a, const T* __restrict__ b, int cstride, const ItemRow* __restrict__ rows,
                int n_items, long long ctas, Window win, double c1, double c2, float off, double* __restrict__ part,
                double* __restrict__ sq) {
  extern __shared__ double smd[];
  const int F = win.size, R = kFwdTile + F - 1;
  double* hs = smd;                        // [4][R][kFwdTile]
  double* red = hs + 4 * R * kFwdTile;     // [3 * warps]
  double* gs = red + 3 * (kThreads / 32);
  float* xs = reinterpret_cast<float*>(gs + kMaxFilter);  // [R][R]
  float* ys = xs + R * R;
  load_window(win, gs);
  const int hn = R * kFwdTile;
  for (long long u = blockIdx.x; u < ctas; u += gridDim.x) {
    const ItemRow it = rows[find_item<&ItemRow::first>(rows, n_items, u)];
    const int p = (int)((u - it.first) / it.tiles), tile = (int)((u - it.first) % it.tiles);
    const int Hs = it.h, Ws = it.w, Ho = Hs - F + 1, Wo = Ws - F + 1;
    const int y0 = (tile / it.ntx) * kFwdTile, x0 = (tile % it.ntx) * kFwdTile;
    const Plane P = item_plane<kMode>(it, p, cstride);
    const double shift =
        0.5 * ((double)texel<kMode>(a, P, y0, x0, p, off) + (double)texel<kMode>(b, P, y0, x0, p, off));
    for (int i = threadIdx.x; i < R * R; i += kThreads) {
      const int r = y0 + i / R, c = x0 + i % R;
      const bool in = r < Hs && c < Ws;
      xs[i] = in ? texel<kMode>(a, P, r, c, p, off) : 0.0f;
      ys[i] = in ? texel<kMode>(b, P, r, c, p, off) : 0.0f;
    }
    __syncthreads();
    double acc_sq = 0.0;
    if (sq) {
      const int rn = (y0 + kFwdTile >= Ho ? Hs : y0 + kFwdTile) - y0;
      const int cn = (x0 + kFwdTile >= Wo ? Ws : x0 + kFwdTile) - x0;
      for (int i = threadIdx.x; i < R * R; i += kThreads) {
        if (i / R < rn && i % R < cn) {
          const double d = (double)xs[i] - (double)ys[i];
          acc_sq = fma(d, d, acc_sq);
        }
      }
    }
    for (int i = threadIdx.x; i < hn; i += kThreads) {
      const int r = i / kFwdTile, c = i % kFwdTile;
      const float* xr = xs + r * R + c;
      const float* yr = ys + r * R + c;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      for (int k = 0; k < F; ++k) {
        const double g = gs[k], x = (double)xr[k] - shift, y = (double)yr[k] - shift;
        s0 = fma(g, x, s0);
        s1 = fma(g, y, s1);
        s2 = fma(g, __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), s2);
        s3 = fma(g, __dmul_rn(x, y), s3);
      }
      hs[i] = s0;
      hs[hn + i] = s1;
      hs[2 * hn + i] = s2;
      hs[3 * hn + i] = s3;
    }
    __syncthreads();
    double acc_cs = 0.0, acc_lcs = 0.0;
#pragma unroll 1
    for (int i = threadIdx.x; i < kFwdTile * kFwdTile; i += kThreads) {
      const int r = i / kFwdTile, c = i % kFwdTile;
      if (y0 + r >= Ho || x0 + c >= Wo) continue;
      double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0;
      for (int k = 0; k < F; ++k) {
        const double g = gs[k];
        const int j = (r + k) * kFwdTile + c;
        m0 = fma(g, hs[j], m0);
        m1 = fma(g, hs[hn + j], m1);
        m2 = fma(g, hs[2 * hn + j], m2);
        m3 = fma(g, hs[3 * hn + j], m3);
      }
      const Terms t = terms(m0, m1, m2, m3, shift, c1, c2);
      acc_cs += t.cs;
      acc_lcs += t.l * t.cs;
    }
    block_sum3(acc_cs, acc_lcs, acc_sq, red);
    if (threadIdx.x == 0) {
      part[2 * u] = acc_cs;
      part[2 * u + 1] = acc_lcs;
      if (sq) sq[u] = acc_sq;
    }
    __syncthreads();
  }
}

// ---- 2x2 average pool with end padding by repetition -> planar float32 -----------------------------------------
// Output element i is element i of the next level, so its item is found among the next scale's rows.
template <typename T, int kMode>
__global__ void __launch_bounds__(kThreads)
ssim_pool_kernel(const T* __restrict__ a, const T* __restrict__ b, int cstride, const ItemRow* __restrict__ rows,
                 const ItemRow* __restrict__ next, int n_items, long long total, float off, float* __restrict__ oa,
                 float* __restrict__ ob) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = find_item<&ItemRow::src>(next, n_items, i);
    const ItemRow it = rows[k];
    const int Hs = it.h, Ws = it.w, Hn = next[k].h, Wn = next[k].w;
    const long long e = i - next[k].src;
    const int p = (int)(e / ((long long)Hn * Wn));
    const int r = (int)(e / Wn % Hn), c = (int)(e % Wn);
    const Plane P = item_plane<kMode>(it, p, cstride);
    const int r0 = 2 * r, r1 = min(2 * r + 1, Hs - 1), c0 = 2 * c, c1 = min(2 * c + 1, Ws - 1);
    oa[i] = ((texel<kMode>(a, P, r0, c0, p, off) + texel<kMode>(a, P, r0, c1, p, off)) +
             (texel<kMode>(a, P, r1, c0, p, off) + texel<kMode>(a, P, r1, c1, p, off))) *
            0.25f;
    ob[i] = ((texel<kMode>(b, P, r0, c0, p, off) + texel<kMode>(b, P, r0, c1, p, off)) +
             (texel<kMode>(b, P, r1, c0, p, off) + texel<kMode>(b, P, r1, c1, p, off))) *
            0.25f;
  }
}

// ---- partials -> stats [items][planes][S][2] and, with `sq`, mse [items][planes] -------------------------------
struct ScaleParts {
  long long offset[kMaxScales];  // first partial of the scale, in doubles
  int n;
};

__global__ void __launch_bounds__(kThreads)
ssim_reduce_kernel(const double* __restrict__ part, const double* __restrict__ sq, const ItemRow* __restrict__ rows,
                   int n_items, int planes, int F, ScaleParts sp, float* __restrict__ stats, float* __restrict__ mse) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n_stats = (long long)n_items * planes * sp.n * 2;
  if (i < n_stats) {
    const int k = (int)(i % 2), s = (int)(i / 2 % sp.n);
    const long long ip = i / (2 * sp.n);
    const ItemRow& it = rows[(long long)s * n_items + ip / planes];
    const double* src = part + sp.offset[s] + (it.first + ip % planes * it.tiles) * 2 + k;
    double acc = 0.0;
    for (long long t = 0; t < it.tiles; ++t) acc += src[2 * t];
    stats[i] = (float)(acc / ((double)(it.h - F + 1) * (it.w - F + 1)));
  } else if (sq && i < n_stats + (long long)n_items * planes) {
    const long long ip = i - n_stats;
    const ItemRow& it = rows[ip / planes];
    const double* src = sq + it.first + ip % planes * it.tiles;
    double acc = 0.0;
    for (long long t = 0; t < it.tiles; ++t) acc += src[t];
    mse[ip] = (float)(acc / ((double)it.h * it.w));
  }
}

// ---- backward: one 16x16 tile of input positions of one plane per CTA ----------------------------------------
// For the tile's inputs q it recomputes the moments at every valid position p whose window covers q, forms there
//   Mx = dL/dmx', My = dL/dmy', A = dL/dS(x'^2 + y'^2), D = dL/dSx'y'
// (L = gA * mean(cs) + gB * mean(l cs)), applies the transposed window and combines
//   dx = G^T*Mx + 2 x' (G^T*A) + y' (G^T*D),   dy = G^T*My + 2 y' (G^T*A) + x' (G^T*D),
// plus the coarser scale's gradient through the pool's adjoint (1/4 to each of the 2x2, a padded row / column folded
// onto the last real one).  Shared memory: window, x and y [I][I] f32 (I = kBwdTile + 2 (F - 1)), horizontal moments
// [4][I][Pt] f64 (Pt = kBwdTile + F - 1; reused as the transposed pass [4][Pt][kBwdTile] f32), adjoints [4][Pt][Pt] f32.
size_t bwd_smem(int F) {
  const int I = kBwdTile + 2 * (F - 1), Pt = kBwdTile + F - 1;
  return 4 * (size_t)I * Pt * sizeof(double) + kMaxFilter * sizeof(double) + 2 * (size_t)I * I * sizeof(float) +
         4 * (size_t)Pt * Pt * sizeof(float);
}

template <typename T, typename TOut>
__global__ void __launch_bounds__(kThreads, 2)
ssim_bwd_kernel(const T* __restrict__ a, const T* __restrict__ b, int cstride, int planes, int Hs, int Ws,
                Window win, double c1, double c2, const float* __restrict__ g_stats, int n_scales, int scale,
                const float* __restrict__ gna, const float* __restrict__ gnb, TOut* __restrict__ da,
                TOut* __restrict__ db) {
  extern __shared__ double smd[];
  const int F = win.size, I = kBwdTile + 2 * (F - 1), Pt = kBwdTile + F - 1;
  double* hs = smd;                                  // [4][I][Pt] f64
  float* ts = reinterpret_cast<float*>(smd);         // [4][Pt][kBwdTile] f32, after hs is consumed
  double* gs = hs + 4 * I * Pt;
  float* xs = reinterpret_cast<float*>(gs + kMaxFilter);  // [I][I]
  float* ys = xs + I * I;
  float* adj = ys + I * I;                           // [4][Pt][Pt]
  load_window(win, gs);
  const int Ho = Hs - F + 1, Wo = Ws - F + 1;
  const int ntx = (Ws + kBwdTile - 1) / kBwdTile;
  const int q0r = (blockIdx.x / ntx) * kBwdTile, q0c = (blockIdx.x % ntx) * kBwdTile;
  const int o = F - 1;  // local index 0 of the inputs and of p is global q0 - o
  const int hn = I * Pt, an = Pt * Pt, tn = Pt * kBwdTile;
  const double inv_count = 1.0 / ((double)Ho * Wo);
  const int Hn = (Hs + 1) / 2, Wn = (Ws + 1) / 2;
  for (int p = blockIdx.y; p < planes; p += gridDim.y) {
    const Plane P = plane_of(p, cstride, Hs, Ws);
    const double shift = 0.5 * ((double)to_f32(a[P.at(q0r, q0c)]) + (double)to_f32(b[P.at(q0r, q0c)]));
    const double wA = (double)g_stats[((long long)p * n_scales + scale) * 2] * inv_count;
    const double wB = (double)g_stats[((long long)p * n_scales + scale) * 2 + 1] * inv_count;
    for (int i = threadIdx.x; i < I * I; i += kThreads) {
      const int r = q0r - o + i / I, c = q0c - o + i % I;
      const bool in = r >= 0 && c >= 0 && r < Hs && c < Ws;
      xs[i] = in ? to_f32(a[P.at(r, c)]) : 0.0f;
      ys[i] = in ? to_f32(b[P.at(r, c)]) : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < hn; i += kThreads) {
      const int r = i / Pt, c = i % Pt;
      const float* xr = xs + r * I + c;
      const float* yr = ys + r * I + c;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      for (int k = 0; k < F; ++k) {
        const double g = gs[k], x = (double)xr[k] - shift, y = (double)yr[k] - shift;
        s0 = fma(g, x, s0);
        s1 = fma(g, y, s1);
        s2 = fma(g, __dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), s2);
        s3 = fma(g, __dmul_rn(x, y), s3);
      }
      hs[i] = s0;
      hs[hn + i] = s1;
      hs[2 * hn + i] = s2;
      hs[3 * hn + i] = s3;
    }
    __syncthreads();
#pragma unroll 1
    for (int i = threadIdx.x; i < an; i += kThreads) {
      const int r = i / Pt, c = i % Pt;
      const int pr = q0r - o + r, pc = q0c - o + c;
      float mx = 0.0f, my = 0.0f, A = 0.0f, D = 0.0f;
      if (pr >= 0 && pc >= 0 && pr < Ho && pc < Wo) {
        double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0;
        for (int k = 0; k < F; ++k) {
          const double g = gs[k];
          const int j = (r + k) * Pt + c;
          m0 = fma(g, hs[j], m0);
          m1 = fma(g, hs[hn + j], m1);
          m2 = fma(g, hs[2 * hn + j], m2);
          m3 = fma(g, hs[3 * hn + j], m3);
        }
        const Terms t = terms(m0, m1, m2, m3, shift, c1, c2);
        const double dcs = wA + wB * t.l, dl = wB * t.cs;
        const double e1 = 2.0 * dl / t.d1, e2 = 2.0 * dcs / t.d2;
        mx = (float)(e1 * (t.my - t.l * t.mx) + e2 * (t.cs * t.ux - t.uy));
        my = (float)(e1 * (t.mx - t.l * t.my) + e2 * (t.cs * t.uy - t.ux));
        A = (float)(-0.5 * e2 * t.cs);
        D = (float)e2;
      }
      adj[i] = mx;
      adj[an + i] = my;
      adj[2 * an + i] = A;
      adj[3 * an + i] = D;
    }
    __syncthreads();
    // transposed window along rows: ts[m][r][c] = sum_k g[F-1-k] adj[m][r][c + k]
    for (int i = threadIdx.x; i < tn; i += kThreads) {
      const int r = i / kBwdTile, c = i % kBwdTile;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      for (int k = 0; k < F; ++k) {
        const double g = gs[F - 1 - k];
        const int j = r * Pt + c + k;
        s0 = fma(g, (double)adj[j], s0);
        s1 = fma(g, (double)adj[an + j], s1);
        s2 = fma(g, (double)adj[2 * an + j], s2);
        s3 = fma(g, (double)adj[3 * an + j], s3);
      }
      ts[i] = (float)s0;
      ts[tn + i] = (float)s1;
      ts[2 * tn + i] = (float)s2;
      ts[3 * tn + i] = (float)s3;
    }
    __syncthreads();
    {
      const int r = threadIdx.x / kBwdTile, c = threadIdx.x % kBwdTile;  // kThreads == kBwdTile^2
      const int qr = q0r + r, qc = q0c + c;
      if (qr < Hs && qc < Ws) {
        double tmx = 0.0, tmy = 0.0, tA = 0.0, tD = 0.0;
        for (int k = 0; k < F; ++k) {
          const double g = gs[F - 1 - k];
          const int j = (r + k) * kBwdTile + c;
          tmx = fma(g, (double)ts[j], tmx);
          tmy = fma(g, (double)ts[tn + j], tmy);
          tA = fma(g, (double)ts[2 * tn + j], tA);
          tD = fma(g, (double)ts[3 * tn + j], tD);
        }
        const int li = (r + o) * I + c + o;
        const double x = (double)xs[li] - shift, y = (double)ys[li] - shift;
        double gx = tmx + 2.0 * x * tA + y * tD;
        double gy = tmy + 2.0 * y * tA + x * tD;
        if (gna) {
          const long long n = ((long long)p * Hn + qr / 2) * Wn + qc / 2;
          const double w = 0.25 * ((Hs & 1) && qr == Hs - 1 ? 2.0 : 1.0) * ((Ws & 1) && qc == Ws - 1 ? 2.0 : 1.0);
          gx += w * (double)gna[n];
          gy += w * (double)gnb[n];
        }
        if (da) da[P.at(qr, qc)] = from_f32<TOut>((float)gx);
        if (db) db[P.at(qr, qc)] = from_f32<TOut>((float)gy);
      }
    }
    __syncthreads();
  }
}

// ---- host side --------------------------------------------------------------------------------------------------
struct Group {
  long long h, w, count;  // `count` consecutive items of size h x w
};

struct Layout {
  int n_scales, item_planes;
  long long n_items, planes;  // planes = n_items * item_planes
  long long C;
  std::vector<Group> groups;
  int h[kMaxScales], w[kMaxScales];  // the first item's sizes (a uniform batch's, for the backward)
  long long ctas[kMaxScales];        // forward CTAs of scale s
  long long elems[kMaxScales];       // elements of one side of pyramid level s (s >= 1)
  long long pyr[kMaxScales];  // byte offset of scale s's x plane set (s >= 1); y follows at + plane_bytes[s]
  long long grad[kMaxScales];  // byte offset of scale s's gradient pair (s >= 1)
  long long plane_bytes[kMaxScales];
  ScaleParts sp;
  long long rows;   // byte offset of the item rows [n_scales][n_items]
  long long part;   // byte offset of the partials
  long long sq;     // byte offset of the squared-error partials (with `mse`), [ctas[0]] doubles
  long long bytes;  // total
};

long long align256(long long v) { return (v + 255) & ~255LL; }

// Checks the filter, the scales and every item's size at every scale, then lays out the workspace.  `indexed` names
// the failing item in the message; `grads` adds the backward's gradient levels, `mse` the squared-error partials.
int plan(std::vector<Group> groups, long long C, int item_planes, int n_scales, int filter_size, bool indexed,
         bool grads, bool mse, Layout* L) {
  if (filter_size < 1 || filter_size > kMaxFilter)
    return fail(TFCB_INVALID_ARGUMENT, "filter_size=%d outside [1, %d]", filter_size, kMaxFilter);
  if (n_scales < 1 || n_scales > kMaxScales)
    return fail(TFCB_INVALID_ARGUMENT, "n_scales=%d outside [1, %d]", n_scales, kMaxScales);
  L->n_scales = n_scales;
  L->item_planes = item_planes;
  L->C = C;
  L->n_items = 0;
  for (const Group& g : groups) L->n_items += g.count;
  L->planes = L->n_items * item_planes;
  L->sp.n = n_scales;
  for (int s = 0; s < n_scales; ++s) L->ctas[s] = L->elems[s] = 0;
  for (size_t k = 0; k < groups.size(); ++k) {
    const Group& g = groups[k];
    int h = (int)g.h, w = (int)g.w;
    for (int s = 0; s < n_scales; ++s) {
      if (h < filter_size || w < filter_size) {
        char item[32] = "";
        if (indexed) snprintf(item, sizeof item, " %zu", k);
        return fail(TFCB_INVALID_ARGUMENT,
                    "image%s too small for %d scale(s) with filter_size=%d: scale %d is %dx%d (input %lldx%lld)", item,
                    n_scales, filter_size, s, h, w, g.h, g.w);
      }
      if (k == 0) {
        L->h[s] = h;
        L->w[s] = w;
      }
      const long long ho = h - filter_size + 1, wo = w - filter_size + 1;
      L->ctas[s] += g.count * item_planes * (((ho + kFwdTile - 1) / kFwdTile) * ((wo + kFwdTile - 1) / kFwdTile));
      L->elems[s] += g.count * item_planes * (long long)h * w;
      h = (h + 1) / 2;
      w = (w + 1) / 2;
    }
  }
  L->groups = std::move(groups);
  long long off = align256(L->n_items * n_scales * (long long)sizeof(ItemRow)), part = 0;
  L->rows = 0;
  for (int s = 0; s < n_scales; ++s) {
    L->sp.offset[s] = part;
    part += L->ctas[s] * 2;
    L->plane_bytes[s] = align256(L->elems[s] * (long long)sizeof(float));
    if (s > 0) {
      L->pyr[s] = off;
      off += 2 * L->plane_bytes[s];
      if (grads) {
        L->grad[s] = off;
        off += 2 * L->plane_bytes[s];
      }
    }
  }
  L->part = off;
  off += align256(part * (long long)sizeof(double));
  L->sq = off;
  if (mse) off += align256(L->ctas[0] * (long long)sizeof(double));
  L->bytes = off;
  return TFCB_OK;
}

// A batch of n_images same-sized images, one plane per channel.
int plan_uniform(int dtype, int64_t n_images, int64_t H, int64_t W, int64_t C, int n_scales, int filter_size,
                 Layout* L) {
  if (dtype < 0 || dtype > 3) return fail(TFCB_INVALID_ARGUMENT, "unsupported SSIM dtype %d", dtype);
  if (n_images < 0 || H <= 0 || W <= 0 || C <= 0)
    return fail(TFCB_INVALID_ARGUMENT, "bad SSIM shape: n_images=%lld H=%lld W=%lld C=%lld", (long long)n_images,
                (long long)H, (long long)W, (long long)C);
  if (H > INT32_MAX || W > INT32_MAX || C > INT32_MAX ||
      (n_images > 0 && (H * W > INT64_MAX / C || H * W * C > INT64_MAX / 8 / n_images)))
    return fail(TFCB_INVALID_ARGUMENT, "SSIM image too large: n_images=%lld H=%lld W=%lld C=%lld",
                (long long)n_images, (long long)H, (long long)W, (long long)C);
  if (n_images * C > INT32_MAX)
    return fail(TFCB_INVALID_ARGUMENT, "SSIM batch too large: n_images * C = %lld planes", (long long)(n_images * C));
  return plan({Group{H, W, n_images}}, C, (int)C, n_scales, filter_size, false, true, false, L);
}

// A list of n_items pairs of their own sizes; item_offsets_host may be NULL (a size query).
int plan_ragged(int dtype, int64_t n_items, const int64_t* item_offsets_host, const int64_t* heights_host,
                const int64_t* widths_host, int64_t C, int mode, int n_scales, int filter_size, Layout* L) {
  if (dtype < 0 || dtype > 3) return fail(TFCB_INVALID_ARGUMENT, "unsupported image dtype %d", dtype);
  if (mode != kRgb && mode != kY && mode != kYCbCr) return fail(TFCB_INVALID_ARGUMENT, "unknown colour mode %d", mode);
  if (C < 1 || C > INT32_MAX) return fail(TFCB_INVALID_ARGUMENT, "bad channel count C=%lld", (long long)C);
  if (mode != kRgb && C != 3)
    return fail(TFCB_INVALID_ARGUMENT, "colour mode %s needs C = 3 channels, got C=%lld", mode == kY ? "y" : "ycbcr",
                (long long)C);
  if (n_items < 0) return fail(TFCB_INVALID_ARGUMENT, "n_items=%lld is negative", (long long)n_items);
  const int item_planes = mode == kRgb ? (int)C : mode == kY ? 1 : 3;
  if (n_items * item_planes > INT32_MAX)
    return fail(TFCB_INVALID_ARGUMENT, "too many planes: n_items * planes = %lld", (long long)(n_items * item_planes));
  if (n_items > 0 && (!heights_host || !widths_host)) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  std::vector<Group> groups;
  groups.reserve(n_items);
  long long total = 0;
  for (int64_t i = 0; i < n_items; ++i) {
    const long long H = heights_host[i], W = widths_host[i];
    if (H < 1 || W < 1 || H > INT32_MAX || W > INT32_MAX)
      return fail(TFCB_INVALID_ARGUMENT, "image %lld: bad size %lldx%lld", (long long)i, H, W);
    if (H * W > (INT64_MAX / 8 - total) / C)
      return fail(TFCB_INVALID_ARGUMENT, "images too large: %lld elements before image %lld", total, (long long)i);
    if (item_offsets_host && item_offsets_host[i] != total)
      return fail(TFCB_INVALID_ARGUMENT, "inconsistent item_offsets: image %lld starts at %lld, expected %lld",
                  (long long)i, (long long)item_offsets_host[i], total);
    total += H * W * C;
    groups.push_back(Group{H, W, 1});
  }
  if (item_offsets_host && n_items > 0 && item_offsets_host[n_items] != total)
    return fail(TFCB_INVALID_ARGUMENT, "inconsistent item_offsets: the list ends at %lld, expected %lld",
                (long long)item_offsets_host[n_items], total);
  return plan(std::move(groups), C, item_planes, n_scales, filter_size, true, false, true, L);
}

// The rows of every scale, [n_scales][n_items].
std::vector<ItemRow> make_rows(const Layout& L, int filter_size) {
  std::vector<ItemRow> rows((size_t)(L.n_items * L.n_scales));
  for (int s = 0; s < L.n_scales; ++s) {
    long long src = 0, first = 0, i = 0;
    for (const Group& g : L.groups) {
      int h = (int)g.h, w = (int)g.w;
      for (int t = 0; t < s; ++t) {
        h = (h + 1) / 2;
        w = (w + 1) / 2;
      }
      const int ntx = (w - filter_size + 1 + kFwdTile - 1) / kFwdTile;
      const int tiles = ntx * ((h - filter_size + 1 + kFwdTile - 1) / kFwdTile);
      for (long long c = 0; c < g.count; ++c, ++i) {
        rows[(size_t)(s * L.n_items + i)] = ItemRow{src, first, h, w, ntx, tiles};
        src += (s == 0 ? L.C : L.item_planes) * (long long)h * w;
        first += (long long)L.item_planes * tiles;
      }
    }
  }
  return rows;
}

int stage_rows(const Layout& L, int filter_size, char* ws, cudaStream_t st) {
  const std::vector<ItemRow> rows = make_rows(L, filter_size);
  // (pageable source: staged before the call returns)
  TFCB_CUDA_TRY(cudaMemcpyAsync(ws + L.rows, rows.data(), rows.size() * sizeof(ItemRow), cudaMemcpyHostToDevice, st));
  return TFCB_OK;
}

int check_params(float max_val, float filter_sigma) {
  if (!(filter_sigma > 0.0f) || !isfinite(filter_sigma))
    return fail(TFCB_INVALID_ARGUMENT, "filter_sigma must be positive and finite, got %g", (double)filter_sigma);
  if (!isfinite(max_val)) return fail(TFCB_INVALID_ARGUMENT, "max_val must be finite, got %g", (double)max_val);
  return TFCB_OK;
}

// The exponent is taken relative to the smallest squared offset m^2 (0 for odd F, 1/4 for even F), as a softmax
// subtracts its maximum: the central taps are exp(0) = 1 for any sigma, so a tiny sigma at even F gives the box of the
// central taps instead of 0 / 0.  The difference is exact in double, and for odd F it leaves the window's bits alone.
Window make_window(int F, float sigma) {
  Window w;
  w.size = F;
  double g[kMaxFilter], sum = 0.0;
  const double s2 = (double)sigma * sigma, mid = 0.5 * (F - 1), m2 = F % 2 ? 0.0 : 0.25;
  for (int k = 0; k < F; ++k) {
    g[k] = exp(-0.5 * ((k - mid) * (k - mid) - m2) / s2);
    sum += g[k];
  }
  for (int k = 0; k < kMaxFilter; ++k) w.g[k] = k < F ? g[k] / sum : 0.0;
  return w;
}

int grid_y(long long planes) { return (int)std::min<long long>(planes, kMaxPlaneBlocks); }

template <typename K>
int allow_smem(K kernel, size_t bytes) {
  TFCB_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return TFCB_OK;
}

const ItemRow* rows_of(const Layout& L, int s, char* ws) {
  return reinterpret_cast<const ItemRow*>(ws + L.rows) + (long long)s * L.n_items;
}

// Source of scale s: the input for s = 0, the pyramid otherwise.
template <typename T, int kMode>
int launch_pool(const T* a, const T* b, int cstride, const Layout& L, int s, float off, char* ws, cudaStream_t st) {
  float* oa = reinterpret_cast<float*>(ws + L.pyr[s + 1]);
  float* ob = reinterpret_cast<float*>(ws + L.pyr[s + 1] + L.plane_bytes[s + 1]);
  const long long total = L.elems[s + 1];
  const int grid = (int)std::min<long long>((total + kThreads - 1) / kThreads, 1 << 16);
  ssim_pool_kernel<T, kMode><<<grid, kThreads, 0, st>>>(a, b, cstride, rows_of(L, s, ws), rows_of(L, s + 1, ws),
                                                        (int)L.n_items, total, off, oa, ob);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

template <typename T, int kMode>
int launch_fwd(const T* a, const T* b, int cstride, const Layout& L, int s, const Window& win, double c1, double c2,
               float off, bool mse, char* ws, cudaStream_t st) {
  const size_t smem = fwd_smem(win.size);
  TFCB_TRY((allow_smem(ssim_fwd_kernel<T, kMode>, smem)));
  double* part = reinterpret_cast<double*>(ws + L.part) + L.sp.offset[s];
  double* sq = mse ? reinterpret_cast<double*>(ws + L.sq) : nullptr;
  const unsigned grid = (unsigned)std::min<long long>(L.ctas[s], INT32_MAX);
  ssim_fwd_kernel<T, kMode><<<grid, kThreads, smem, st>>>(a, b, cstride, rows_of(L, s, ws), (int)L.n_items, L.ctas[s],
                                                          win, c1, c2, off, part, sq);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// stats [items][planes][S][2]; mse [items][planes] when not NULL (the layout must have been planned with `mse`).
template <typename T, int kMode>
int forward(const T* a, const T* b, const Layout& L, const Window& win, double c1, double c2, float off, float* stats,
            float* mse, char* ws, cudaStream_t st) {
  TFCB_TRY(stage_rows(L, win.size, ws, st));
  const int C = (int)L.C;
  for (int s = 0; s < L.n_scales; ++s) {
    if (s == 0) {
      TFCB_TRY((launch_fwd<T, kMode>(a, b, C, L, 0, win, c1, c2, off, mse != nullptr, ws, st)));
      if (L.n_scales > 1) TFCB_TRY((launch_pool<T, kMode>(a, b, C, L, 0, off, ws, st)));
    } else {
      const float* pa = reinterpret_cast<const float*>(ws + L.pyr[s]);
      const float* pb = reinterpret_cast<const float*>(ws + L.pyr[s] + L.plane_bytes[s]);
      TFCB_TRY((launch_fwd<float, kRgb>(pa, pb, 1, L, s, win, c1, c2, off, false, ws, st)));
      if (s + 1 < L.n_scales) TFCB_TRY((launch_pool<float, kRgb>(pa, pb, 1, L, s, off, ws, st)));
    }
  }
  const long long n = L.planes * L.n_scales * 2 + (mse ? L.planes : 0);
  ssim_reduce_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      reinterpret_cast<const double*>(ws + L.part), mse ? reinterpret_cast<const double*>(ws + L.sq) : nullptr,
      rows_of(L, 0, ws), (int)L.n_items, L.item_planes, win.size, L.sp, stats, mse);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

template <typename T, typename TOut>
int launch_bwd(const T* a, const T* b, int cstride, const Layout& L, int s, const Window& win, double c1, double c2,
               const float* g_stats, char* ws, TOut* da, TOut* db, cudaStream_t st) {
  const size_t smem = bwd_smem(win.size);
  TFCB_TRY((allow_smem(ssim_bwd_kernel<T, TOut>, smem)));
  const float* gna = nullptr;
  const float* gnb = nullptr;
  if (s + 1 < L.n_scales) {
    gna = reinterpret_cast<const float*>(ws + L.grad[s + 1]);
    gnb = reinterpret_cast<const float*>(ws + L.grad[s + 1] + L.plane_bytes[s + 1]);
  }
  const long long tiles =
      (long long)((L.h[s] + kBwdTile - 1) / kBwdTile) * ((L.w[s] + kBwdTile - 1) / kBwdTile);
  ssim_bwd_kernel<T, TOut><<<dim3((unsigned)tiles, grid_y(L.planes)), kThreads, smem, st>>>(
      a, b, cstride, (int)L.planes, L.h[s], L.w[s], win, c1, c2, g_stats, L.n_scales, s, gna, gnb, da, db);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// A uniform batch: the pyramid is then planar [planes][h][w] per level, the layout the backward kernel reads.
template <typename T>
int backward(const T* a, const T* b, int C, const Layout& L, const Window& win, double c1, double c2,
             const float* g_stats, T* da, T* db, char* ws, cudaStream_t st) {
  if (L.n_scales > 1) TFCB_TRY(stage_rows(L, win.size, ws, st));
  for (int s = 0; s + 1 < L.n_scales; ++s) {
    if (s == 0) {
      TFCB_TRY((launch_pool<T, kRgb>(a, b, C, L, 0, 0.0f, ws, st)));
    } else {
      TFCB_TRY((launch_pool<float, kRgb>(reinterpret_cast<const float*>(ws + L.pyr[s]),
                                         reinterpret_cast<const float*>(ws + L.pyr[s] + L.plane_bytes[s]), 1, L, s,
                                         0.0f, ws, st)));
    }
  }
  for (int s = L.n_scales - 1; s >= 1; --s) {
    const float* pa = reinterpret_cast<const float*>(ws + L.pyr[s]);
    const float* pb = reinterpret_cast<const float*>(ws + L.pyr[s] + L.plane_bytes[s]);
    float* ga = reinterpret_cast<float*>(ws + L.grad[s]);
    float* gb = reinterpret_cast<float*>(ws + L.grad[s] + L.plane_bytes[s]);
    TFCB_TRY((launch_bwd<float, float>(pa, pb, 1, L, s, win, c1, c2, g_stats, ws, ga, gb, st)));
  }
  return launch_bwd<T, T>(a, b, C, L, 0, win, c1, c2, g_stats, ws, da, db, st);
}

struct Call {
  Layout L;
  Window win;
  double c1, c2;
  float off;  // the Cb / Cr offset, float32(128/255) * max_val
};

int finish(float max_val, int filter_size, float filter_sigma, float k1, float k2, Call* call) {
  TFCB_TRY(check_params(max_val, filter_sigma));
  if (!isfinite(k1) || !isfinite(k2)) return fail(TFCB_INVALID_ARGUMENT, "k1 and k2 must be finite");
  call->win = make_window(filter_size, filter_sigma);
  const double a1 = (double)k1 * max_val, a2 = (double)k2 * max_val;
  call->c1 = a1 * a1;
  call->c2 = a2 * a2;
  call->off = (float)(128.0 / 255.0) * max_val;
  return TFCB_OK;
}

int prepare(int dtype, int64_t n_images, int64_t H, int64_t W, int64_t C, float max_val, int n_scales,
            int filter_size, float filter_sigma, float k1, float k2, Call* call) {
  TFCB_TRY(plan_uniform(dtype, n_images, H, W, C, n_scales, filter_size, &call->L));
  return finish(max_val, filter_size, filter_sigma, k1, k2, call);
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

#define TFCB_SSIM_DISPATCH(dtype, ...)                         \
  switch (dtype) {                                             \
    case 0: { using T = float; __VA_ARGS__; } break;           \
    case 1: { using T = __half; __VA_ARGS__; } break;          \
    case 2: { using T = __nv_bfloat16; __VA_ARGS__; } break;   \
    default: { using T = uint8_t; __VA_ARGS__; } break;        \
  }

extern "C" {

int64_t tfcb_ssim_workspace_bytes(int dtype, int64_t n_images, int64_t H, int64_t W, int64_t C, int n_scales,
                                  int filter_size) {
  Layout L{};
  const std::string saved = last_error();  // a size query leaves the last error as it was
  const int rc = plan_uniform(dtype, n_images, H, W, C, n_scales, filter_size, &L);
  last_error() = saved;
  return rc == TFCB_OK ? L.bytes : -1;
}

int tfcb_ssim_stats(const void* img1_dev, const void* img2_dev, int dtype, int64_t n_images, int64_t H, int64_t W,
                    int64_t C, float max_val, int n_scales, int filter_size, float filter_sigma, float k1, float k2,
                    float* stats_dev, void* workspace_dev, void* stream) {
  Call call;
  TFCB_TRY(prepare(dtype, n_images, H, W, C, max_val, n_scales, filter_size, filter_sigma, k1, k2, &call));
  if (n_images == 0) return TFCB_OK;
  if (!img1_dev || !img2_dev || !stats_dev || !workspace_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  char* ws = reinterpret_cast<char*>(workspace_dev);
  TFCB_SSIM_DISPATCH(dtype, {
    TFCB_TRY((forward<T, kRgb>(reinterpret_cast<const T*>(img1_dev), reinterpret_cast<const T*>(img2_dev), call.L,
                               call.win, call.c1, call.c2, call.off, stats_dev, nullptr, ws, as_stream(stream))));
  });
  return TFCB_OK;
}

int tfcb_ssim_stats_backward(const void* img1_dev, const void* img2_dev, int dtype, int64_t n_images, int64_t H,
                             int64_t W, int64_t C, float max_val, int n_scales, int filter_size, float filter_sigma,
                             float k1, float k2, const float* g_stats_dev, void* dimg1_dev, void* dimg2_dev,
                             void* workspace_dev, void* stream) {
  Call call;
  TFCB_TRY(prepare(dtype, n_images, H, W, C, max_val, n_scales, filter_size, filter_sigma, k1, k2, &call));
  if (dtype == 3) return fail(TFCB_INVALID_ARGUMENT, "uint8 images have no gradient");
  if (n_images == 0 || (!dimg1_dev && !dimg2_dev)) return TFCB_OK;
  if (!img1_dev || !img2_dev || !g_stats_dev || !workspace_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  char* ws = reinterpret_cast<char*>(workspace_dev);
  switch (dtype) {
#define TFCB_SSIM_BWD(TYPE)                                                                                       \
  TFCB_TRY(backward<TYPE>(reinterpret_cast<const TYPE*>(img1_dev), reinterpret_cast<const TYPE*>(img2_dev), (int)C, \
                          call.L, call.win, call.c1, call.c2, g_stats_dev, reinterpret_cast<TYPE*>(dimg1_dev),      \
                          reinterpret_cast<TYPE*>(dimg2_dev), ws, as_stream(stream)))
    case 0: TFCB_SSIM_BWD(float); break;
    case 1: TFCB_SSIM_BWD(__half); break;
    default: TFCB_SSIM_BWD(__nv_bfloat16); break;
#undef TFCB_SSIM_BWD
  }
  return TFCB_OK;
}

int64_t tfcb_image_metrics_ragged_workspace_bytes(int dtype, int64_t n_items, const int64_t* heights_host,
                                                  const int64_t* widths_host, int64_t C, int mode, int n_scales,
                                                  int filter_size) {
  Layout L{};
  const std::string saved = last_error();
  const int rc = plan_ragged(dtype, n_items, nullptr, heights_host, widths_host, C, mode, n_scales, filter_size, &L);
  last_error() = saved;
  return rc == TFCB_OK ? L.bytes : -1;
}

int tfcb_image_metrics_ragged(const void* img1_dev, const void* img2_dev, int dtype, int64_t n_items,
                              const int64_t* item_offsets_host, const int64_t* heights_host,
                              const int64_t* widths_host, int64_t C, int mode, float max_val, int n_scales,
                              int filter_size, float filter_sigma, float k1, float k2, float* stats_dev,
                              float* mse_dev, void* workspace_dev, void* stream) {
  if (n_items > 0 && !item_offsets_host) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  Call call;
  TFCB_TRY(plan_ragged(dtype, n_items, item_offsets_host, heights_host, widths_host, C, mode, n_scales, filter_size,
                       &call.L));
  TFCB_TRY(finish(max_val, filter_size, filter_sigma, k1, k2, &call));
  if (n_items == 0) return TFCB_OK;
  if (!img1_dev || !img2_dev || !stats_dev || !mse_dev || !workspace_dev)
    return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  char* ws = reinterpret_cast<char*>(workspace_dev);
#define TFCB_METRICS_MODE(M)                                                                                      \
  TFCB_SSIM_DISPATCH(dtype, {                                                                                     \
    TFCB_TRY((forward<T, M>(reinterpret_cast<const T*>(img1_dev), reinterpret_cast<const T*>(img2_dev), call.L,   \
                            call.win, call.c1, call.c2, call.off, stats_dev, mse_dev, ws, as_stream(stream))));   \
  })
  switch (mode) {
    case kRgb: TFCB_METRICS_MODE(kRgb); break;
    case kY: TFCB_METRICS_MODE(kY); break;
    default: TFCB_METRICS_MODE(kYCbCr); break;
  }
#undef TFCB_METRICS_MODE
  return TFCB_OK;
}

}  // extern "C"
