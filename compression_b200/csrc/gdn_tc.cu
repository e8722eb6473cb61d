// GDN / IGDN forward and backward on the Hopper tensor cores (wgmma), sm_90a.
//
//   n[pix, i] = sum_j p[pix, j] * gamma[j, i]      p = |x|, x^2 or relu(x) variants (py/layers/gdn.py:377-398)
//
// is a [n_pix x C] x [C x C] GEMM with 2*C^2 FLOP per 8*C bytes of HBM traffic: on fp32 CUDA cores it is compute
// bound well below the HBM roofline.  Here every contraction runs as  wgmma.mma_async .f32.bf16.bf16  on an
// error-compensated bf16 split (3 products: hi*hi + lo*hi + hi*lo, fp32 accumulation), which keeps the result within
// ~4e-6 of fp32 (SURVEY.md App. D; the contract is 1e-5) at bf16 tensor throughput.
//
// Forward and the dx half of the backward: persistent CTAs of 2 (C = 192) or 3 (C = 128) warpgroups; each warpgroup
// walks its own 64-pixel tiles (wgmma M = 64) with no block-level synchronisation after the prologue.  gamma's hi / lo
// bf16 planes are built once per CTA in shared memory in the no-swizzle core-matrix layout [j / 8][i][j % 8]: read
// K-major they are the B operand of p . gamma, read MN-major (transposed) the B operand of q . gamma^T, so one copy
// serves both products (two copies would not fit next to each other at C = 192).  The pixel-side operand comes from
// registers: a thread loads x at the positions of its wgmma A fragment, which are also the positions of its
// accumulator fragment, so q = dL/dn is turned into the A operand of q . gamma^T without leaving registers.
//
// dgamma = p^T . q reduces over pixels: a second kernel stages 64-pixel chunks of p and q as bf16 planes in shared
// memory (double-buffered, the next chunk is staged while the tensor cores work on the current one) and accumulates
// one [64 x C] slice of dgamma per warpgroup.
//
// C = 256 and 320 do not fit that layout (shared memory, registers) and split the work over blocks of output columns
// instead: see "Wide layers" below.
//
// At C in {128, 192, 256, 320}, trainable exponents and fixed ones outside alpha in {1, 2}, eps in {1, 0.5} run the
// literal-pow variant of every kernel (gdn_tc_pow_*, float32 only: powf / logf in the element functions, and the
// backward sums dL/dalpha and dL/depsilon in its epilogues).  Every other width falls back to the fp32 kernels in
// gdn.cu.  At C = 128 / 192 the forward, dx and dgamma kernels also take float16 / bfloat16 activations (IO = 1, 2):
// each element is widened exactly on load, the arithmetic is the float32 kernels', and the only rounding to 16 bits
// is the final store, so the result is the float32 result of the widened inputs rounded once.
//
// Host side: gdn_tc_route decides which of these kernels take a configuration, and gdn_tc_forward / gdn_tc_backward
// launch them through with_kernels, the one map from a route and a layout to the kernels' template arguments.  The C
// entry points, their argument checks and the backward workspace are gdn.cu's.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "gdn_tc.cuh"

namespace tfcb {
namespace {

constexpr int kTileM = 64;  // pixels per warpgroup tile (wgmma M)

struct TcFlags {
  int inverse, rectify, alpha_mode, eps_mode;  // alpha_mode: 1 |u|, 2 u^2; eps_mode: 1 identity, 2 sqrt
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma shared-memory matrix descriptor, no swizzle: bits [0,14) start >> 4, [16,30) leading-dimension byte offset >> 4
// (between core matrices along K), [32,46) stride-dimension byte offset >> 4 (between core matrices along M / N).
// A core matrix is 8 rows of 16 contiguous bytes.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// Keeps reads of the accumulators after the wait for the MMAs that write them.
template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N][32]) {
#pragma unroll
  for (int n = 0; n < N; ++n)
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[n][i])::"memory");
}

#define TFCB_WGMMA_D32                                                                                          \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, " \
  "%23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define TFCB_WGMMA_D32_OPS                                                                                         \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),    \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),     \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),    \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])

// d[64 x 64] += A[64 x 16] . B[16 x 64].  A: four bf16x2 registers per thread (the m16n8k16 A fragment of the
// warp's 16 rows); B: shared memory, K-major (TB = 0) or MN-major (TB = 1).
template <int TB>
__device__ __forceinline__ void wgmma_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " TFCB_WGMMA_D32
               ", {%32, %33, %34, %35}, %36, 1, 1, 1, %37;"
               : TFCB_WGMMA_D32_OPS
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "n"(TB)
               : "memory");
}

// d[64 x 64] += A[64 x 16] . B[16 x 64], both MN-major in shared memory.
__device__ __forceinline__ void wgmma_ss_mn(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " TFCB_WGMMA_D32 ", %32, %33, 1, 1, 1, 1, 1;"
               : TFCB_WGMMA_D32_OPS
               : "l"(a), "l"(b)
               : "memory");
}

// FAST = the default GDN / IGDN of bls2017 / bmshj2018 (alpha = 1, epsilon = 1, no rectification): no
// per-element branches.  Otherwise the runtime flags are honoured.
template <bool FAST>
__device__ __forceinline__ float tc_pool(float x, const TcFlags& f) {
  if (FAST) return fabsf(x);
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  if (f.alpha_mode == 2) return u * u;
  return f.rectify ? u : fabsf(u);
}

// The quotients use the hardware reciprocal (MUFU.RCP, <= 1 ulp): an IEEE divide costs ~20 instructions per element,
// and 2.4e-7 is far inside the 1e-5 contract.  n = beta + pool is a normal, moderate number.
__device__ __forceinline__ float rcp_approx(float v) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
  return r;
}

// y = u / m (GDN) or u * m (IGDN), m = n or sqrt(n).
template <bool FAST>
__device__ __forceinline__ float tc_out(float x, float n, const TcFlags& f) {
  if (FAST) return f.inverse ? x * n : x * rcp_approx(n);
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  const float m = (f.eps_mode == 2) ? sqrtf(n) : n;
  return f.inverse ? u * m : u * rcp_approx(m);
}

// Upstream gradient g at one element: *q = dL/dn, *d = the direct part of dL/du (through the division or product).
template <bool FAST>
__device__ __forceinline__ void tc_bwd_point(float x, float g, float n, const TcFlags& f, float* q, float* d) {
  if (FAST) {
    if (f.inverse) {
      *d = g * n;
      *q = g * x;
    } else {
      const float r = rcp_approx(n);
      *d = g * r;
      *q = -(*d) * x * r;
    }
    return;
  }
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  if (f.eps_mode == 2) {
    const float m = sqrtf(n);
    *d = f.inverse ? g * m : g / m;
    *q = f.inverse ? 0.5f * g * u / m : -0.5f * g * u / (n * m);
  } else {
    *d = f.inverse ? g * n : g / n;
    *q = f.inverse ? g * u : -g * u / (n * n);
  }
}

// d pool / d x, with the rectifier's mask folded in by the caller.
template <bool FAST>
__device__ __forceinline__ float tc_dpool(float x, const TcFlags& f) {
  if (FAST) return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f);  // TF's abs gradient is sign()
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  if (f.alpha_mode == 2) return 2.f * u;
  if (f.rectify) return 1.f;
  return (u > 0.f) ? 1.f : ((u < 0.f) ? -1.f : 0.f);
}

// Literal-pow variant: trainable exponents (TFCB_GDN_POW_*) and fixed exponents outside {1, 2} / {1, 1/2}.  Its own
// flags type selects the overloads below, so the kernels instantiated with TcFlags keep their code.  The element
// functions are the fp32 kernels' pool_of / norm_of / dpool_du / dl_dn (gdn.cu) with IEEE divides: a mode of 0 is
// powf, and a fixed exponent of a mixed configuration keeps its |u|, u^2 or sqrt shortcut.
struct TcPowFlags {
  int inverse, rectify, alpha_mode, eps_mode;  // alpha_mode: 0 powf(u, alpha), 1 |u|, 2 u^2; eps_mode: 0 powf, 1, 2 sqrt
  float alpha, eps;
  float* part_e;  // backward: per-CTA partials (dL/dalpha, dL/depsilon) [grid][2], or null
};

template <class F>
constexpr bool kPow = std::is_same_v<F, TcPowFlags>;

template <bool FAST>
__device__ __forceinline__ float tc_pool(float x, const TcPowFlags& f) {
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  if (f.alpha_mode == 1) return f.rectify ? u : fabsf(u);
  if (f.alpha_mode == 2) return u * u;
  return powf(u, f.alpha);
}

__device__ __forceinline__ float tc_norm(float n, const TcPowFlags& f) {
  if (f.eps_mode == 1) return n;
  if (f.eps_mode == 2) return sqrtf(n);
  return powf(n, f.eps);
}

template <bool FAST>
__device__ __forceinline__ float tc_out(float x, float n, const TcPowFlags& f) {
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  const float m = tc_norm(n, f);
  return f.inverse ? u * m : u / m;
}

template <bool FAST>
__device__ __forceinline__ void tc_bwd_point(float x, float g, float n, const TcPowFlags& f, float* q, float* d) {
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  const float m = tc_norm(n, f);
  *d = f.inverse ? g * m : g / m;
  if (!f.inverse) {
    if (f.eps_mode == 1)
      *q = -g * u / (n * n);
    else if (f.eps_mode == 2)
      *q = -0.5f * g * u / (n * sqrtf(n));
    else
      *q = -f.eps * g * u * powf(n, -f.eps - 1.f);
  } else {
    if (f.eps_mode == 1)
      *q = g * u;
    else if (f.eps_mode == 2)
      *q = 0.5f * g * u / sqrtf(n);
    else
      *q = f.eps * g * u * powf(n, f.eps - 1.f);
  }
}

template <bool FAST>
__device__ __forceinline__ float tc_dpool(float x, const TcPowFlags& f) {
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  if (f.alpha_mode == 1) {
    if (f.rectify) return 1.f;
    return (u > 0.f) ? 1.f : ((u < 0.f) ? -1.f : 0.f);
  }
  if (f.alpha_mode == 2) return 2.f * u;
  return f.alpha * powf(u, f.alpha - 1.f);
}

// The exponent gradients' terms of one element (gdn.cu gdn_bwd_exponents_kernel):
//   dL/depsilon += q n ln(n) / epsilon          from the epilogue that forms q
//   dL/dalpha   += dp p ln(u)   (u > 0)          from the epilogue that adds dpool/dx . dp
__device__ __forceinline__ float tc_deps_term(float q, float n, const TcPowFlags& f) { return q * n * logf(n) / f.eps; }

__device__ __forceinline__ float tc_dalpha_term(float x, float dp, const TcPowFlags& f) {
  const float u = f.rectify ? fmaxf(x, 0.f) : x;
  return (u > 0.f) ? dp * tc_pool<false>(x, f) * logf(u) : 0.f;
}

// Sums the CTA's (dL/dalpha, dL/depsilon) in a fixed order and writes them to part[0], part[1] (either may be
// skipped with WRITE_A / WRITE_E).  Called by every thread after its last MMA: reuses the start of `smem`.
template <bool WRITE_A, bool WRITE_E>
__device__ __forceinline__ void cta_exponent_partial(float dal, float dep, uint8_t* smem, float* part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    dal += __shfl_xor_sync(0xFFFFFFFFu, dal, o);
    dep += __shfl_xor_sync(0xFFFFFFFFu, dep, o);
  }
  float* red = reinterpret_cast<float*>(smem);
  const int warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    red[2 * warp] = dal;
    red[2 * warp + 1] = dep;
  }
  __syncthreads();
  if (threadIdx.x < 2 && (threadIdx.x == 0 ? WRITE_A : WRITE_E)) {
    float s = 0.f;
    for (int w = 0; w < n_warps; ++w) s += red[2 * w + threadIdx.x];
    part[threadIdx.x] = s;
  }
}

// Two floats -> bf16x2, the first in the low half (the lower column of a fragment).
__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
  return r;
}

// Error-compensated split of two values: hi = bf16(v), lo = bf16(v - hi).
__device__ __forceinline__ void split2(float a, float b, uint32_t* hi, uint32_t* lo) {
  *hi = pack_bf16x2(a, b);
  *lo = pack_bf16x2(a - __uint_as_float(*hi << 16), b - __uint_as_float(*hi & 0xFFFF0000u));
}

__device__ __forceinline__ void split8(const float (&v)[8], uint4* hi, uint4* lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) split2(v[2 * i], v[2 * i + 1], &h[i], &l[i]);
  *hi = make_uint4(h[0], h[1], h[2], h[3]);
  *lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// Element type of x / y in memory: 0 float32, 1 float16, 2 bfloat16 (the reference's mixed-precision policy keeps the
// variables in float32 and the activations in 16 bits, gdn_test.py:200-210; arithmetic is float32 here either way).
// Pairs of consecutive channels of one pixel; idx is the (even) element index.  Widening is exact, so a 16-bit
// element enters the arithmetic as the float32 value x.float() would give.
template <int IO>
__device__ __forceinline__ float2 widen2(uint32_t w) {
  if (IO == 2) return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u));
  return __half22float2(*reinterpret_cast<const __half2*>(&w));
}

template <int IO>
__device__ __forceinline__ float2 ld_pair(const void* base, long long idx) {
  if (IO == 0) return __ldg(reinterpret_cast<const float2*>(static_cast<const float*>(base) + idx));
  return widen2<IO>(__ldg(reinterpret_cast<const unsigned int*>(static_cast<const uint16_t*>(base) + idx)));
}

template <int IO>
__device__ __forceinline__ void st_pair(void* base, long long idx, float a, float b) {
  if (IO == 0) {
    *reinterpret_cast<float2*>(static_cast<float*>(base) + idx) = make_float2(a, b);
    return;
  }
  uint32_t w;
  if (IO == 2) {
    w = pack_bf16x2(a, b);
  } else {
    const __half2 h = __floats2half2_rn(a, b);
    w = *reinterpret_cast<const uint32_t*>(&h);
  }
  *reinterpret_cast<uint32_t*>(static_cast<uint16_t*>(base) + idx) = w;
}

// Layout of the activations x, y, dy and dx.  Channels-last (CF = false): element (pixel r, channel c) at r * C + c.
// Channels-first (CF = true, [N, C, S] with S the product of the spatial dimensions): pixel r of the flattened
// [N * S] order is position r % S of item r / S, and its channel c lives at (r / S) * C * S + c * S + r % S.  A row's
// base (its channel 0) takes the one division; channel c is then at base + ch_off(c).  Tiles run over the flattened
// pixel order either way (a tile may span two items), and q, the 16-bit scratch and the partials stay channels-last,
// so the channels-first kernels compute every value exactly as the channels-last kernels do on the transposed tensor.
template <bool CF>
__device__ __forceinline__ long long row_base(long long r, int C, long long S) {
  if constexpr (CF) {
    const long long item = r / S;
    return item * C * S + (r - item * S);
  } else {
    return r * C;
  }
}

template <bool CF>
__device__ __forceinline__ long long ch_off(int c, long long S) {
  if constexpr (CF) return (long long)c * S;
  else return c;
}

// The index of channel c of the row at `base` in layout CF, given the channels-last index `cl` of the same element:
// channels-last code keeps its own index expressions (and its instructions).
template <bool CF>
__device__ __forceinline__ long long cf_idx(long long cl, long long base, int c, long long S) {
  if constexpr (CF) return base + (long long)c * S;
  else return cl;
}

template <int IO>
__device__ __forceinline__ float ld_one(const void* base, long long idx) {
  if (IO == 0) return __ldg(static_cast<const float*>(base) + idx);
  const unsigned short w = __ldg(static_cast<const unsigned short*>(base) + idx);
  if (IO == 2) return __uint_as_float((uint32_t)w << 16);
  return __half2float(__ushort_as_half(w));
}

// One element, rounded to nearest as st_pair's paired conversions round each of theirs.
template <int IO>
__device__ __forceinline__ void st_one(void* base, long long idx, float v) {
  if (IO == 0) {
    static_cast<float*>(base)[idx] = v;
    return;
  }
  static_cast<unsigned short*>(base)[idx] =
      IO == 2 ? __bfloat16_as_ushort(__float2bfloat16_rn(v)) : __half_as_ushort(__float2half_rn(v));
}

// Channels c, c + 1 of one pixel at idx = row_base + ch_off(c): one access channels-last, two channels-first.
template <int IO, bool CF>
__device__ __forceinline__ float2 ld_px(const void* base, long long idx, long long S) {
  if constexpr (CF) return make_float2(ld_one<IO>(base, idx), ld_one<IO>(base, idx + S));
  else return ld_pair<IO>(base, idx);
}

template <int IO, bool CF>
__device__ __forceinline__ void st_px(void* base, long long idx, long long S, float a, float b) {
  if constexpr (CF) {
    st_one<IO>(base, idx, a);
    st_one<IO>(base, idx + S, b);
  } else {
    st_pair<IO>(base, idx, a, b);
  }
}

// float32 dx written, and read back in the kernel that wrote it (no read-only cache).
template <bool CF>
__device__ __forceinline__ float2 ld_px_rw(const float* base, long long idx, long long S) {
  if constexpr (CF) return make_float2(base[idx], base[idx + S]);
  else return *reinterpret_cast<const float2*>(base + idx);
}

template <bool CF>
__device__ __forceinline__ void st_px_f2(float* base, long long idx, long long S, float2 v) {
  if constexpr (CF) {
    base[idx] = v.x;
    base[idx + S] = v.y;
  } else {
    *reinterpret_cast<float2*>(base + idx) = v;
  }
}

template <int C>
struct TcCfg {
  static constexpr int kWG = C == 128 ? 3 : 2;  // warpgroups per CTA: as many as the registers allow
  static constexpr int kThreads = 128 * kWG;
  static constexpr int kSmem = 2 * C * C * 2;   // gamma hi / lo planes
  static_assert(kSmem <= 232448, "shared memory budget");
};

// gamma [C, C] fp32 (L2 resident) -> hi / lo bf16 planes [j / 8][i][j % 8] at smem, smem + C * C * 2.  Every CTA
// converts its own copy in the prologue: no per-call allocation and no separate preparation launch.
template <int C>
__device__ __forceinline__ void fill_planes(const float* __restrict__ gamma, uint8_t* smem) {
  for (int idx = threadIdx.x; idx < (C / 8) * C; idx += blockDim.x) {
    const int jc = idx / C, i = idx % C;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = __ldg(gamma + (jc * 8 + e) * C + i);
    uint4 hi, lo;
    split8(v, &hi, &lo);
    reinterpret_cast<uint4*>(smem)[idx] = hi;
    reinterpret_cast<uint4*>(smem + C * C * 2)[idx] = lo;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the planes are read by the tensor cores
  __syncthreads();
}

// A fragments of pool(x) for one tile: k-step kk covers channels 16 kk .. 16 kk + 15; register r of a step holds
// (row g, cols c, c+1), (row g+8, c, c+1), (row g, c+8, c+9), (row g+8, c+8, c+9), c = 16 kk + 2 t.  b0, b1: the
// row bases (row_base) of rows r0, r1 in layout CF.
template <int C, bool FAST, int IO, bool CF, class F>
__device__ __forceinline__ void pool_frags(const void* __restrict__ x, long long r0, long long r1, long long b0,
                                           long long b1, long long S, bool ok0, bool ok1, int t, const F& f,
                                           uint32_t (&ah)[C / 16][4], uint32_t (&al)[C / 16][4]) {
#pragma unroll
  for (int kk = 0; kk < C / 16; ++kk) {
    const int c = 16 * kk + 2 * t;
    const float2 z = make_float2(0.f, 0.f);
    const float2 v[4] = {ok0 ? ld_px<IO, CF>(x, cf_idx<CF>(r0 * C + c, b0, c, S), S) : z,
                         ok1 ? ld_px<IO, CF>(x, cf_idx<CF>(r1 * C + c, b1, c, S), S) : z,
                         ok0 ? ld_px<IO, CF>(x, cf_idx<CF>(r0 * C + c + 8, b0, c + 8, S), S) : z,
                         ok1 ? ld_px<IO, CF>(x, cf_idx<CF>(r1 * C + c + 8, b1, c + 8, S), S) : z};
#pragma unroll
    for (int r = 0; r < 4; ++r) split2(tc_pool<FAST>(v[r].x, f), tc_pool<FAST>(v[r].y, f), &ah[kk][r], &al[kk][r]);
  }
}

// acc[64 x C] = A . gamma (TB = 0) or A . gamma^T (TB = 1), A = ah + al, gamma = hi + lo planes at bh, bl; the
// lo . lo product is below fp32 resolution and skipped.  Issues the MMAs and waits for them.
template <int C, int TB>
__device__ __forceinline__ void gemm3(float (&acc)[C / 64][32], const uint32_t (&ah)[C / 16][4],
                                      const uint32_t (&al)[C / 16][4], uint32_t bh, uint32_t bl) {
#pragma unroll
  for (int n = 0; n < C / 64; ++n)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[n][i] = 0.f;
  // K-major: core matrix (k / 8, n / 8) at (k / 8) * C * 16 + (n / 8) * 128 bytes; MN-major (the same planes read as
  // gamma^T, k = i, n = j): at (n / 8) * C * 16 + (k / 8) * 128.
  constexpr uint32_t kLbo = TB ? 128 : C * 16, kSbo = TB ? C * 16 : 128;
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < C / 16; ++kk)
#pragma unroll
    for (int n = 0; n < C / 64; ++n) {
      const uint32_t off = TB ? (256u * kk + (uint32_t)n * C * 128) : ((uint32_t)kk * C * 32 + 1024u * n);
      wgmma_rs<TB>(acc[n], ah[kk], gmma_desc(bh + off, kLbo, kSbo));
      wgmma_rs<TB>(acc[n], al[kk], gmma_desc(bh + off, kLbo, kSbo));
      wgmma_rs<TB>(acc[n], ah[kk], gmma_desc(bl + off, kLbo, kSbo));
    }
  wgmma_commit();
  wgmma_wait_all();
  fence_acc(acc);
}

// Accumulator element (n, jj, h, e) of a thread: row g + 8 h of its warp's 16, column 64 n + 8 jj + 2 t + e.
#define TFCB_FOR_ACC_PAIRS(C)            \
  _Pragma("unroll") for (int n = 0; n < (C) / 64; ++n) \
  _Pragma("unroll") for (int jj = 0; jj < 8; ++jj)     \
  _Pragma("unroll") for (int h = 0; h < 2; ++h)

// The kernels' bodies take the flags type F: TcFlags for the fixed-exponent kernels, TcPowFlags for the literal-pow
// kernels (float32 I/O, FAST = false), which are named gdn_tc_pow_*.
// The kernels take the activations' layout CF (row_base) and S, the item size of the channels-first layout (unused
// channels-last).
template <int C, bool FAST, int IO, bool CF, class F>
__device__ __forceinline__ void tc_fwd_body(const void* __restrict__ x, const float* __restrict__ gamma,
                                            const float* __restrict__ beta, void* __restrict__ y, long long n_pix,
                                            const F& f, long long S) {
  using K = TcCfg<C>;
  extern __shared__ __align__(1024) uint8_t smem[];
  fill_planes<C>(gamma, smem);
  const uint32_t bh = smem_u32(smem), bl = bh + C * C * 2;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  for (long long tile = (long long)blockIdx.x * K::kWG + wg; tile < n_tiles; tile += (long long)gridDim.x * K::kWG) {
    const long long r0 = tile * kTileM + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < n_pix, ok1 = r1 < n_pix;
    const long long b0 = row_base<CF>(r0, C, S), b1 = row_base<CF>(r1, C, S);
    uint32_t ah[C / 16][4], al[C / 16][4];
    pool_frags<C, FAST, IO, CF>(x, r0, r1, b0, b1, S, ok0, ok1, t, f, ah, al);
    float acc[C / 64][32];
    gemm3<C, 0>(acc, ah, al, bh, bl);
    // accumulators are read on every thread (only the memory accesses are predicated): a read inside a divergent
    // branch makes ptxas serialise the MMAs
    TFCB_FOR_ACC_PAIRS(C) {
      const bool ok = h ? ok1 : ok0;
      const int col = 64 * n + 8 * jj + 2 * t;
      const long long idx = cf_idx<CF>((h ? r1 : r0) * C + col, h ? b1 : b0, col, S);
      const float2 xv = ok ? ld_px<IO, CF>(x, idx, S) : make_float2(0.f, 0.f);
      const float2 b = __ldg(reinterpret_cast<const float2*>(beta + col));
      const float y0 = tc_out<FAST>(xv.x, b.x + acc[n][4 * jj + 2 * h], f);
      const float y1 = tc_out<FAST>(xv.y, b.y + acc[n][4 * jj + 2 * h + 1], f);
      if (ok) st_px<IO, CF>(y, idx, S, y0, y1);
    }
  }
}

template <int C, bool FAST, int IO, bool CF>
__global__ void __launch_bounds__(TcCfg<C>::kThreads, 1)
gdn_tc_fwd_kernel(const void* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                  void* __restrict__ y, long long n_pix, TcFlags f, long long S) {
  tc_fwd_body<C, FAST, IO, CF>(x, gamma, beta, y, n_pix, f, S);
}

template <int C, bool CF>
__global__ void __launch_bounds__(TcCfg<C>::kThreads, 1)
gdn_tc_pow_fwd_kernel(const void* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                      void* __restrict__ y, long long n_pix, TcPowFlags f, long long S) {
  tc_fwd_body<C, false, 0, CF>(x, gamma, beta, y, n_pix, f, S);
}

// Backward, part 1: per 64-pixel tile
//   n = beta + p . gamma  ->  q = dL/dn (stored for part 2), the direct term of dx (stored)
//   dp = q . gamma^T      ->  dx = direct term + dpool/dx * dp (the direct term read back from the same thread's
//                             stores, L2 resident).
// x, dy and dx are float32 (IO = 0) or 16-bit (IO = 1 float16, 2 bfloat16; q stays float32).  With IO = 0 the direct
// term is stored in dx itself.  A 16-bit dx would round it before the second term is added, so with IO != 0 it goes
// to the warpgroup's own 64 x C float32 tile of `scratch` instead, and dx is stored once, rounded once: the result is
// the float32 kernel's on the widened inputs, rounded to the activation type.  No register can hold it through MMA2
// (the C = 192 FAST variant is at the 255-register limit) and no shared memory is left beside gamma's planes at C = 192.
// Channels-first (CF) float32 keeps the direct term in the scratch as well, so dx is only written: storing it in dx
// and reading it back would keep a second strided address per pair alive across MMA2, and those kernels spilled.
// The literal-pow variant also sums dL/depsilon in the first epilogue and dL/dalpha in the second, one partial per CTA.
template <int C, bool FAST, int IO, bool CF, class F>
__device__ __forceinline__ void tc_bwd_dx_body(const void* __restrict__ x, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, const void* __restrict__ dy,
                                               void* __restrict__ dx, float* __restrict__ q_ws, long long n_pix,
                                               const F& f, float* __restrict__ scratch, long long S) {
  using K = TcCfg<C>;
  extern __shared__ __align__(1024) uint8_t smem[];
  fill_planes<C>(gamma, smem);
  const uint32_t bh = smem_u32(smem), bl = bh + C * C * 2;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // IO != 0: this thread's row g, columns 2 t, 2 t + 1 of its warp's 16 rows in the warpgroup's scratch tile (the
  // accumulator pair (n, jj, h) is at + 8 h C + 64 n + 8 jj: immediate offsets)
  float* const dtile = scratch + ((long long)(blockIdx.x * K::kWG + wg) * kTileM + warp * 16 + g) * C + 2 * t;
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  float dal = 0.f, dep = 0.f;  // literal-pow variant: this thread's exponent-gradient sums
  for (long long tile = (long long)blockIdx.x * K::kWG + wg; tile < n_tiles; tile += (long long)gridDim.x * K::kWG) {
    const long long r0 = tile * kTileM + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < n_pix, ok1 = r1 < n_pix;
    const long long b0 = row_base<CF>(r0, C, S), b1 = row_base<CF>(r1, C, S);
    uint32_t ah[C / 16][4], al[C / 16][4];
    pool_frags<C, FAST, IO, CF>(x, r0, r1, b0, b1, S, ok0, ok1, t, f, ah, al);
    float acc[C / 64][32];
    gemm3<C, 0>(acc, ah, al, bh, bl);
    TFCB_FOR_ACC_PAIRS(C) {
      float* a = &acc[n][4 * jj + 2 * h];
      if (!(h ? ok1 : ok0)) {
        a[0] = a[1] = 0.f;
        continue;
      }
      const int col = 64 * n + 8 * jj + 2 * t;
      const long long idx = (h ? r1 : r0) * C + col;                // q (channels-last)
      const long long gi = cf_idx<CF>(idx, h ? b1 : b0, col, S);  // x, dy, dx
      const float2 xv = ld_px<IO, CF>(x, gi, S);
      const float2 gv = ld_px<IO, CF>(dy, gi, S);
      const float2 b = __ldg(reinterpret_cast<const float2*>(beta + col));
      float2 q, d;
      tc_bwd_point<FAST>(xv.x, gv.x, b.x + a[0], f, &q.x, &d.x);
      tc_bwd_point<FAST>(xv.y, gv.y, b.y + a[1], f, &q.y, &d.y);
      if constexpr (kPow<F>) dep += tc_deps_term(q.x, b.x + a[0], f) + tc_deps_term(q.y, b.y + a[1], f);
      *reinterpret_cast<float2*>(q_ws + idx) = q;
      if constexpr (IO == 0 && !CF)
        *reinterpret_cast<float2*>(static_cast<float*>(dx) + idx) = d;
      else
        *reinterpret_cast<float2*>(dtile + 8 * h * C + 64 * n + 8 * jj) = d;
      a[0] = q.x;
      a[1] = q.y;
    }
    // q's accumulator fragment is, register for register, the A fragment of q . gamma^T
#pragma unroll
    for (int kk = 0; kk < C / 16; ++kk) {
      const float* a = &acc[kk / 4][8 * (kk % 4)];
#pragma unroll
      for (int r = 0; r < 4; ++r) split2(a[2 * r], a[2 * r + 1], &ah[kk][r], &al[kk][r]);
    }
    gemm3<C, 1>(acc, ah, al, bh, bl);
    TFCB_FOR_ACC_PAIRS(C) {
      if (!(h ? ok1 : ok0)) continue;
      const long long idx = cf_idx<CF>((h ? r1 : r0) * C + 64 * n + 8 * jj + 2 * t, h ? b1 : b0,
                                       64 * n + 8 * jj + 2 * t, S);
      const float2 xv = ld_px<IO, CF>(x, idx, S);
      float2 d;
      if constexpr (IO == 0 && !CF)
        d = *reinterpret_cast<const float2*>(static_cast<const float*>(dx) + idx);
      else
        d = *reinterpret_cast<const float2*>(dtile + 8 * h * C + 64 * n + 8 * jj);
      d.x += tc_dpool<FAST>(xv.x, f) * acc[n][4 * jj + 2 * h];
      d.y += tc_dpool<FAST>(xv.y, f) * acc[n][4 * jj + 2 * h + 1];
      if constexpr (kPow<F>)
        dal += tc_dalpha_term(xv.x, acc[n][4 * jj + 2 * h], f) + tc_dalpha_term(xv.y, acc[n][4 * jj + 2 * h + 1], f);
      if (!FAST && f.rectify) {
        if (!(xv.x > 0.f)) d.x = 0.f;
        if (!(xv.y > 0.f)) d.y = 0.f;
      }
      st_px<IO, CF>(dx, idx, S, d.x, d.y);
    }
  }
  if constexpr (kPow<F>) {
    if (f.part_e != nullptr) cta_exponent_partial<true, true>(dal, dep, smem, f.part_e + 2 * blockIdx.x);
  }
}

template <int C, bool FAST, int IO, bool CF>
__global__ void __launch_bounds__(TcCfg<C>::kThreads, 1)
gdn_tc_bwd_dx_kernel(const void* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                     const void* __restrict__ dy, void* __restrict__ dx, float* __restrict__ q_ws, long long n_pix,
                     TcFlags f, float* __restrict__ scratch, long long S) {
  tc_bwd_dx_body<C, FAST, IO, CF>(x, gamma, beta, dy, dx, q_ws, n_pix, f, scratch, S);
}

template <int C, bool CF>
__global__ void __launch_bounds__(TcCfg<C>::kThreads, 1)
gdn_tc_pow_bwd_dx_kernel(const void* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                         const void* __restrict__ dy, void* __restrict__ dx, float* __restrict__ q_ws, long long n_pix,
                         TcPowFlags f, float* __restrict__ scratch, long long S) {
  tc_bwd_dx_body<C, false, 0, CF>(x, gamma, beta, dy, dx, q_ws, n_pix, f, scratch, S);
}

// Backward, part 2: per-CTA partials dgamma[j, i] = sum_pix p[pix, j] q[pix, i] and dbeta[i] = sum_pix q[pix, i].
// C / 64 warpgroups; warpgroup w accumulates rows 64 w .. 64 w + 63 of dgamma.  A 64-pixel chunk of p and q is staged
// as bf16 hi / lo planes [C / 8][64][8] (MN-major core matrices: 8 channels x 8 pixels); thread t stages channels
// 8 (t / 16) .. + 7 of pixels t % 16 + 16 s, s < 4, and keeps the dbeta sums of those channels.
template <int C>
struct DgCfg {
  static constexpr int kThreads = 2 * C;
  static constexpr int kPlane = C * kTileM * 2;
  static constexpr int kStage = 4 * kPlane;  // p hi, p lo, q hi, q lo
  static constexpr int kSmem = 2 * kStage;
  static_assert(kSmem <= 232448, "shared memory budget");
};

// The tensor core's fp32 accumulation is not round-to-nearest: a long-running accumulator drifts with the number of
// accumulation steps.  The accumulator is therefore added into the CTA's fp32 partial in global memory (round-to-
// nearest adds, L2 resident) every kDgFlush chunks and restarted.
constexpr int kDgFlush = 8;

// x in float32 (IO = 0) or 16 bits (IO = 1, 2: one 16-byte load of the 8 channels, widened exactly); q is float32.
template <int IO>
using IoElem = std::conditional_t<IO == 0, float, uint16_t>;

template <int C, bool FAST, int IO, bool CF, class F>
__device__ __forceinline__ void tc_dgamma_body(const IoElem<IO>* __restrict__ x, const float* __restrict__ q,
                                               float* __restrict__ part_g, float* __restrict__ part_b, long long n_pix,
                                               const F& f, long long S) {
  using L = DgCfg<C>;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int jc = tid >> 4, pl = tid & 15;
  const long long n_chunks = (n_pix + kTileM - 1) / kTileM;
  float bsum[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) bsum[e] = 0.f;

  auto stage = [&](long long chunk, int buf) {
    uint8_t* base = smem + buf * L::kStage;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int p = pl + 16 * s;
      const long long row = chunk * kTileM + p;
      float v[8], w[8];
      if (row < n_pix) {
        if constexpr (CF) {  // 8 element loads, one per channel; 16 lanes read 16 consecutive pixels of each
          const long long xb = row_base<true>(row, C, S) + ch_off<true>(8 * jc, S);
          const float4* qr = reinterpret_cast<const float4*>(q + row * C + 8 * jc);
          const float4 q0 = __ldg(qr), q1 = __ldg(qr + 1);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = ld_one<IO>(x, xb + e * S);
          w[0] = q0.x, w[1] = q0.y, w[2] = q0.z, w[3] = q0.w, w[4] = q1.x, w[5] = q1.y, w[6] = q1.z, w[7] = q1.w;
        } else if constexpr (IO == 0) {
          const float4* xr = reinterpret_cast<const float4*>(x + row * C + 8 * jc);
          const float4* qr = reinterpret_cast<const float4*>(q + row * C + 8 * jc);
          const float4 x0 = __ldg(xr), x1 = __ldg(xr + 1), q0 = __ldg(qr), q1 = __ldg(qr + 1);
          v[0] = x0.x, v[1] = x0.y, v[2] = x0.z, v[3] = x0.w, v[4] = x1.x, v[5] = x1.y, v[6] = x1.z, v[7] = x1.w;
          w[0] = q0.x, w[1] = q0.y, w[2] = q0.z, w[3] = q0.w, w[4] = q1.x, w[5] = q1.y, w[6] = q1.z, w[7] = q1.w;
        } else {
          const uint4 x8 = __ldg(reinterpret_cast<const uint4*>(x + row * C + 8 * jc));
          const float4* qr = reinterpret_cast<const float4*>(q + row * C + 8 * jc);
          const float4 q0 = __ldg(qr), q1 = __ldg(qr + 1);
          const float2 x01 = widen2<IO>(x8.x), x23 = widen2<IO>(x8.y), x45 = widen2<IO>(x8.z), x67 = widen2<IO>(x8.w);
          v[0] = x01.x, v[1] = x01.y, v[2] = x23.x, v[3] = x23.y, v[4] = x45.x, v[5] = x45.y, v[6] = x67.x, v[7] = x67.y;
          w[0] = q0.x, w[1] = q0.y, w[2] = q0.z, w[3] = q0.w, w[4] = q1.x, w[5] = q1.y, w[6] = q1.z, w[7] = q1.w;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = w[e] = 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        // pow(0, alpha) is inf for alpha < 0: rows past the end must stay 0
        if constexpr (kPow<F>)
          v[e] = row < n_pix ? tc_pool<FAST>(v[e], f) : 0.f;
        else
          v[e] = tc_pool<FAST>(v[e], f);
        bsum[e] += w[e];
      }
      const int slot = (jc * kTileM + p) * 16;
      uint4 hi, lo;
      split8(v, &hi, &lo);
      *reinterpret_cast<uint4*>(base + slot) = hi;
      *reinterpret_cast<uint4*>(base + L::kPlane + slot) = lo;
      split8(w, &hi, &lo);
      *reinterpret_cast<uint4*>(base + 2 * L::kPlane + slot) = hi;
      *reinterpret_cast<uint4*>(base + 3 * L::kPlane + slot) = lo;
    }
  };

  float acc[C / 64][32];
  float* pg = part_g + (long long)blockIdx.x * C * C;
  bool first_flush = true;
  stage(blockIdx.x, 0);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  int k = 0;
  for (long long chunk = blockIdx.x; chunk < n_chunks; chunk += gridDim.x, ++k) {
    if (k % kDgFlush == 0) {
#pragma unroll
      for (int n = 0; n < C / 64; ++n)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[n][i] = 0.f;
    }
    // core matrix (channel / 8, pixel / 8) at (channel / 8) * 1024 + (pixel / 8) * 128 bytes of a plane
    const uint32_t base = smem_u32(smem + (k & 1) * L::kStage);
    const uint32_t planes[3][2] = {{0, 2}, {1, 2}, {0, 3}};  // (p, q) plane pairs: hi.hi, lo.hi, hi.lo
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTileM / 16; ++kk)
#pragma unroll
      for (int pr = 0; pr < 3; ++pr) {
        const uint64_t a = gmma_desc(base + planes[pr][0] * L::kPlane + wg * 8 * 1024 + 256 * kk, 128, 1024);
#pragma unroll
        for (int n = 0; n < C / 64; ++n)
          wgmma_ss_mn(acc[n], a, gmma_desc(base + planes[pr][1] * L::kPlane + n * 8 * 1024 + 256 * kk, 128, 1024));
      }
    wgmma_commit();
    const bool last = chunk + gridDim.x >= n_chunks;
    if (!last) stage(chunk + gridDim.x, (k + 1) & 1);
    wgmma_wait_all();
    fence_acc(acc);
    if ((k + 1) % kDgFlush == 0 || last) {
      TFCB_FOR_ACC_PAIRS(C) {
        float2* dst = reinterpret_cast<float2*>(pg + (64 * wg + 16 * warp + g + 8 * h) * C + 64 * n + 8 * jj + 2 * t);
        float2 v = make_float2(acc[n][4 * jj + 2 * h], acc[n][4 * jj + 2 * h + 1]);
        if (!first_flush) {
          const float2 o = *dst;
          v.x += o.x;
          v.y += o.y;
        }
        *dst = v;
      }
      first_flush = false;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }
#pragma unroll
  for (int e = 0; e < 8; ++e)
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) bsum[e] += __shfl_xor_sync(0xFFFFFFFFu, bsum[e], o);
  if (pl == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) part_b[(long long)blockIdx.x * C + 8 * jc + e] = bsum[e];
  }
}

template <int C, bool FAST, int IO, bool CF>
__global__ void __launch_bounds__(DgCfg<C>::kThreads, 1)
gdn_tc_dgamma_kernel(const IoElem<IO>* __restrict__ x, const float* __restrict__ q, float* __restrict__ part_g,
                     float* __restrict__ part_b, long long n_pix, TcFlags f, long long S) {
  tc_dgamma_body<C, FAST, IO, CF>(x, q, part_g, part_b, n_pix, f, S);
}

template <int C, bool CF>
__global__ void __launch_bounds__(DgCfg<C>::kThreads, 1)
gdn_tc_pow_dgamma_kernel(const float* __restrict__ x, const float* __restrict__ q, float* __restrict__ part_g,
                         float* __restrict__ part_b, long long n_pix, TcPowFlags f, long long S) {
  tc_dgamma_body<C, false, 0, CF>(x, q, part_g, part_b, n_pix, f, S);
}

// ---- Wide layers, C in {256, 320}: the work is split over blocks of NB output columns ----
//
// At C > 192 neither gamma's planes (4 C^2 bytes: 256 / 400 KB) nor a warpgroup's A fragments of all K = C plus the
// accumulators of all C columns fit, so each CTA owns one block of NB channels:
//   forward / backward pass 1   columns [c0, c0 + NB):  planes of gamma[:, block], acc = pool(x) . gamma[:, block]
//   backward pass 2             rows J = [j0, j0 + NB):  planes of gamma[J, :],     dp[:, J] = q . gamma[J, :]^T
//   dgamma                      columns [c0, c0 + NB):  p over all C channels, q over the block's NB
// Pass 2 exists because with columns split over CTAs no CTA holds all of q, which every entry of dp needs.  A CTA's
// block is blockIdx.x % kBlocks, so the kBlocks CTAs of one group walk the same pixel tiles side by side: x (and q)
// come from HBM once and are re-read from L2 by the other blocks.
template <int C>
struct WideCfg {
  static constexpr int kNB = C == 256 ? 128 : 64;  // channels per block; accumulators: NB / 2 registers
  static constexpr int kBlocks = C / kNB;
  static constexpr int kKSlices = C == 320 ? 2 : 1;  // A fragments held at once: C / 16 / kKSlices k-steps
  static constexpr int kWG = 2;
  static constexpr int kThreads = 128 * kWG;
  static constexpr int kSmem = 2 * C * kNB * 2;  // hi / lo planes of a C x NB (or NB x C) block of gamma
  static constexpr int kDgPPlane = C * kTileM * 2;  // dgamma: one bf16 plane of p (all channels) ...
  static constexpr int kDgQPlane = kNB * kTileM * 2;  // ... and of q (the block's channels)
  static constexpr int kDgStage = 2 * kDgPPlane + 2 * kDgQPlane;  // p hi, p lo, q hi, q lo
  static constexpr int kDgSmem = 2 * kDgStage;
  static_assert(C % kNB == 0 && kNB % 64 == 0, "column blocks of whole wgmma N = 64 tiles");
  static_assert(kSmem <= 232448 && kDgSmem <= 232448, "shared memory budget");
};

// gamma rows [j0, j0 + NJ) x columns [i0, i0 + NI) -> hi / lo bf16 planes [j / 8][i][j % 8] (block-local j, i) at
// smem, smem + NJ * NI * 2: fill_planes restricted to one block.
template <int C, int NJ, int NI>
__device__ __forceinline__ void fill_planes_block(const float* __restrict__ gamma, int j0, int i0, uint8_t* smem) {
  for (int idx = threadIdx.x; idx < (NJ / 8) * NI; idx += blockDim.x) {
    const int jc = idx / NI, i = idx % NI;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = __ldg(gamma + (j0 + jc * 8 + e) * C + i0 + i);
    uint4 hi, lo;
    split8(v, &hi, &lo);
    reinterpret_cast<uint4*>(smem)[idx] = hi;
    reinterpret_cast<uint4*>(smem + NJ * NI * 2)[idx] = lo;
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
}

// A fragments of channels [16 k0, 16 k0 + KA) of a tile of a [n_pix, C] array in layout CF (row bases b0, b1), at
// the positions pool_frags uses: pool(x) (POOL) or the values themselves (q, always channels-last).
template <int C, int KA, bool POOL, bool FAST, bool CF, class F>
__device__ __forceinline__ void slice_frags(const float* __restrict__ src, long long r0, long long r1, long long b0,
                                            long long b1, long long S, bool ok0, bool ok1, int t, int k0, const F& f,
                                            uint32_t (&ah)[KA / 16][4], uint32_t (&al)[KA / 16][4]) {
#pragma unroll
  for (int kk = 0; kk < KA / 16; ++kk) {
    const int c = 16 * (k0 + kk) + 2 * t;
    const float2 z = make_float2(0.f, 0.f);
    const float2 v[4] = {ok0 ? ld_px<0, CF>(src, cf_idx<CF>(r0 * C + c, b0, c, S), S) : z,
                         ok1 ? ld_px<0, CF>(src, cf_idx<CF>(r1 * C + c, b1, c, S), S) : z,
                         ok0 ? ld_px<0, CF>(src, cf_idx<CF>(r0 * C + c + 8, b0, c + 8, S), S) : z,
                         ok1 ? ld_px<0, CF>(src, cf_idx<CF>(r1 * C + c + 8, b1, c + 8, S), S) : z};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (POOL)
        split2(tc_pool<FAST>(v[r].x, f), tc_pool<FAST>(v[r].y, f), &ah[kk][r], &al[kk][r]);
      else
        split2(v[r].x, v[r].y, &ah[kk][r], &al[kk][r]);
    }
  }
}

// acc[64 x NB] = A . B for one 64-pixel tile, K = C, A = split(pool(x)) (POOL) or split(q) from `src`, B = hi + lo
// planes at bh, bl laid out by fill_planes_block:
//   TB = 0: B = gamma[:, block]    (k = j, n = i; planes C x NB)
//   TB = 1: B = gamma[J, :]^T      (k = i, n = j; planes NB x C)
// K is walked in kKSlices slices, each loaded into registers, multiplied and waited for before the next is loaded:
// at C = 320 the A fragments of all K (160 registers) next to the accumulators leave ptxas too few registers to
// avoid spills.  Otherwise gemm3 with the plane extents of one block.
template <int C, int TB, bool POOL, bool FAST, bool CF, class F>
__device__ __forceinline__ void wide_gemm(float (&acc)[WideCfg<C>::kNB / 64][32], const float* __restrict__ src,
                                          long long r0, long long r1, long long b0, long long b1, long long S,
                                          bool ok0, bool ok1, int t, const F& f, uint32_t bh, uint32_t bl) {
  constexpr int NB = WideCfg<C>::kNB, KA = C / WideCfg<C>::kKSlices;
#pragma unroll
  for (int n = 0; n < NB / 64; ++n)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[n][i] = 0.f;
  // K-major: core matrix (k / 8, n / 8) at (k / 8) * NB * 16 + (n / 8) * 128 bytes; MN-major: at
  // (n / 8) * C * 16 + (k / 8) * 128.
  constexpr uint32_t kLbo = TB ? 128 : NB * 16, kSbo = TB ? C * 16 : 128;
#pragma unroll
  for (int s = 0; s < WideCfg<C>::kKSlices; ++s) {
    uint32_t ah[KA / 16][4], al[KA / 16][4];
    slice_frags<C, KA, POOL, FAST, CF>(src, r0, r1, b0, b1, S, ok0, ok1, t, s * KA / 16, f, ah, al);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < KA / 16; ++kk)
#pragma unroll
      for (int n = 0; n < NB / 64; ++n) {
        const uint32_t k = s * KA / 16 + kk;
        const uint32_t off = TB ? (256u * k + (uint32_t)n * C * 128) : (k * NB * 32 + 1024u * n);
        wgmma_rs<TB>(acc[n], ah[kk], gmma_desc(bh + off, kLbo, kSbo));
        wgmma_rs<TB>(acc[n], al[kk], gmma_desc(bh + off, kLbo, kSbo));
        wgmma_rs<TB>(acc[n], ah[kk], gmma_desc(bl + off, kLbo, kSbo));
      }
    wgmma_commit();
    wgmma_wait_all();
    fence_acc(acc);
  }
}

template <int C, bool FAST, bool CF, class F>
__device__ __forceinline__ void tc_wide_fwd_body(const float* __restrict__ x, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, float* __restrict__ y,
                                                 long long n_pix, const F& f, long long S) {
  using W = WideCfg<C>;
  constexpr int NB = W::kNB;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int c0 = (int)(blockIdx.x % W::kBlocks) * NB;
  fill_planes_block<C, C, NB>(gamma, 0, c0, smem);
  const uint32_t bh = smem_u32(smem), bl = bh + C * NB * 2;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const long long stride = (long long)(gridDim.x / W::kBlocks) * W::kWG;
  for (long long tile = (long long)(blockIdx.x / W::kBlocks) * W::kWG + wg; tile < n_tiles; tile += stride) {
    const long long r0 = tile * kTileM + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < n_pix, ok1 = r1 < n_pix;
    const long long b0 = row_base<CF>(r0, C, S), b1 = row_base<CF>(r1, C, S);
    float acc[NB / 64][32];
    wide_gemm<C, 0, true, FAST, CF>(acc, x, r0, r1, b0, b1, S, ok0, ok1, t, f, bh, bl);
    TFCB_FOR_ACC_PAIRS(NB) {
      const bool ok = h ? ok1 : ok0;
      const int col = c0 + 64 * n + 8 * jj + 2 * t;
      const long long idx = cf_idx<CF>((h ? r1 : r0) * C + col, h ? b1 : b0, col, S);
      const float2 xv = ok ? ld_px<0, CF>(x, idx, S) : make_float2(0.f, 0.f);
      const float2 b = __ldg(reinterpret_cast<const float2*>(beta + col));
      const float y0 = tc_out<FAST>(xv.x, b.x + acc[n][4 * jj + 2 * h], f);
      const float y1 = tc_out<FAST>(xv.y, b.y + acc[n][4 * jj + 2 * h + 1], f);
      if (ok) st_px<0, CF>(y, idx, S, y0, y1);
    }
  }
}

template <int C, bool FAST, bool CF>
__global__ void __launch_bounds__(WideCfg<C>::kThreads, 1)
gdn_tc_wide_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                       float* __restrict__ y, long long n_pix, TcFlags f, long long S) {
  tc_wide_fwd_body<C, FAST, CF>(x, gamma, beta, y, n_pix, f, S);
}

template <int C, bool CF>
__global__ void __launch_bounds__(WideCfg<C>::kThreads, 1)
gdn_tc_pow_wide_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                           const float* __restrict__ beta, float* __restrict__ y, long long n_pix, TcPowFlags f,
                           long long S) {
  tc_wide_fwd_body<C, false, CF>(x, gamma, beta, y, n_pix, f, S);
}

// Backward, pass 1: n[:, block] = beta + p . gamma[:, block]  ->  q[:, block] (workspace), dx[:, block] = direct term.
// The literal-pow variant also sums dL/depsilon over the block's columns: partial [blockIdx.x][1].
template <int C, bool FAST, bool CF, class F>
__device__ __forceinline__ void tc_wide_bwd_q_body(const float* __restrict__ x, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, const float* __restrict__ dy,
                                                   float* __restrict__ dx, float* __restrict__ q_ws, long long n_pix,
                                                   const F& f, long long S) {
  using W = WideCfg<C>;
  constexpr int NB = W::kNB;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int c0 = (int)(blockIdx.x % W::kBlocks) * NB;
  fill_planes_block<C, C, NB>(gamma, 0, c0, smem);
  const uint32_t bh = smem_u32(smem), bl = bh + C * NB * 2;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const long long stride = (long long)(gridDim.x / W::kBlocks) * W::kWG;
  float dep = 0.f;
  for (long long tile = (long long)(blockIdx.x / W::kBlocks) * W::kWG + wg; tile < n_tiles; tile += stride) {
    const long long r0 = tile * kTileM + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < n_pix, ok1 = r1 < n_pix;
    const long long b0 = row_base<CF>(r0, C, S), b1 = row_base<CF>(r1, C, S);
    float acc[NB / 64][32];
    wide_gemm<C, 0, true, FAST, CF>(acc, x, r0, r1, b0, b1, S, ok0, ok1, t, f, bh, bl);
    TFCB_FOR_ACC_PAIRS(NB) {
      const bool ok = h ? ok1 : ok0;
      const int col = c0 + 64 * n + 8 * jj + 2 * t;
      const long long idx = (h ? r1 : r0) * C + col;                // q (channels-last)
      const long long gi = cf_idx<CF>(idx, h ? b1 : b0, col, S);  // x, dy, dx
      const float2 xv = ok ? ld_px<0, CF>(x, gi, S) : make_float2(0.f, 0.f);
      const float2 gv = ok ? ld_px<0, CF>(dy, gi, S) : make_float2(0.f, 0.f);
      const float2 b = __ldg(reinterpret_cast<const float2*>(beta + col));
      float2 qv, d;
      tc_bwd_point<FAST>(xv.x, gv.x, b.x + acc[n][4 * jj + 2 * h], f, &qv.x, &d.x);
      tc_bwd_point<FAST>(xv.y, gv.y, b.y + acc[n][4 * jj + 2 * h + 1], f, &qv.y, &d.y);
      if constexpr (kPow<F>) {
        const float e = tc_deps_term(qv.x, b.x + acc[n][4 * jj + 2 * h], f) +
                        tc_deps_term(qv.y, b.y + acc[n][4 * jj + 2 * h + 1], f);
        if (ok) dep += e;
      }
      if (ok) {
        *reinterpret_cast<float2*>(q_ws + idx) = qv;
        st_px_f2<CF>(dx, gi, S, d);
      }
    }
  }
  if constexpr (kPow<F>) {
    if (f.part_e != nullptr) cta_exponent_partial<false, true>(0.f, dep, smem, f.part_e + 2 * blockIdx.x);
  }
}

template <int C, bool FAST, bool CF>
__global__ void __launch_bounds__(WideCfg<C>::kThreads, 1)
gdn_tc_wide_bwd_q_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                         const float* __restrict__ dy, float* __restrict__ dx, float* __restrict__ q_ws,
                         long long n_pix, TcFlags f, long long S) {
  tc_wide_bwd_q_body<C, FAST, CF>(x, gamma, beta, dy, dx, q_ws, n_pix, f, S);
}

template <int C, bool CF>
__global__ void __launch_bounds__(WideCfg<C>::kThreads, 1)
gdn_tc_pow_wide_bwd_q_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                             const float* __restrict__ beta, const float* __restrict__ dy, float* __restrict__ dx,
                             float* __restrict__ q_ws, long long n_pix, TcPowFlags f, long long S) {
  tc_wide_bwd_q_body<C, false, CF>(x, gamma, beta, dy, dx, q_ws, n_pix, f, S);
}

// Channels-first pass 2: pass 1's direct term in dx for columns c + 8 jj of rows r0, r1 (bases b0, b1), one 64-column
// block, all loaded before the block's stores.  With runtime strides the compiler cannot move a load above an earlier
// pair's store, and one memory round trip per pair made the kernel latency bound (2.8x the channels-last time).
__device__ __forceinline__ void wide_dx_prefetch(const float* dx, long long b0, long long b1, long long S, bool ok0,
                                                 bool ok1, int c, float2 (&dv)[8][2]) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      dv[jj][h] = (h ? ok1 : ok0) ? ld_px_rw<true>(dx, (h ? b1 : b0) + ch_off<true>(c + 8 * jj, S), S)
                                  : make_float2(0.f, 0.f);
}

// Backward, pass 2: dp[:, J] = q . gamma[J, :]^T  ->  dx[:, J] += dpool/dx * dp, then the rectifier's mask.  q is
// channels-last in either layout; x and dx are in layout CF.
template <int C, bool FAST, bool CF>
__global__ void __launch_bounds__(WideCfg<C>::kThreads, 1)
gdn_tc_wide_bwd_dp_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ q,
                          float* __restrict__ dx, long long n_pix, TcFlags f, long long S) {
  using W = WideCfg<C>;
  constexpr int NB = W::kNB;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int j0 = (int)(blockIdx.x % W::kBlocks) * NB;
  fill_planes_block<C, NB, C>(gamma, j0, 0, smem);
  const uint32_t bh = smem_u32(smem), bl = bh + C * NB * 2;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const long long stride = (long long)(gridDim.x / W::kBlocks) * W::kWG;
  for (long long tile = (long long)(blockIdx.x / W::kBlocks) * W::kWG + wg; tile < n_tiles; tile += stride) {
    const long long r0 = tile * kTileM + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < n_pix, ok1 = r1 < n_pix;
    const long long b0 = row_base<CF>(r0, C, S), b1 = row_base<CF>(r1, C, S);
    float acc[NB / 64][32];
    wide_gemm<C, 1, false, FAST, false>(acc, q, r0, r1, r0 * C, r1 * C, S, ok0, ok1, t, f, bh, bl);
    if constexpr (CF) {
#pragma unroll
      for (int n = 0; n < NB / 64; ++n) {
        float2 dv[8][2];
        wide_dx_prefetch(dx, b0, b1, S, ok0, ok1, j0 + 64 * n + 2 * t, dv);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const bool ok = h ? ok1 : ok0;
            const long long idx = (h ? b1 : b0) + ch_off<true>(j0 + 64 * n + 8 * jj + 2 * t, S);
            const float2 xv = ok ? ld_px<0, true>(x, idx, S) : make_float2(0.f, 0.f);
            float2 d = dv[jj][h];
            d.x += tc_dpool<FAST>(xv.x, f) * acc[n][4 * jj + 2 * h];
            d.y += tc_dpool<FAST>(xv.y, f) * acc[n][4 * jj + 2 * h + 1];
            if (!FAST && f.rectify) {
              if (!(xv.x > 0.f)) d.x = 0.f;
              if (!(xv.y > 0.f)) d.y = 0.f;
            }
            if (ok) st_px_f2<true>(dx, idx, S, d);
          }
      }
    } else {
      TFCB_FOR_ACC_PAIRS(NB) {
        const bool ok = h ? ok1 : ok0;
        const long long idx = (h ? r1 : r0) * C + j0 + 64 * n + 8 * jj + 2 * t;
        const float2 xv = ok ? __ldg(reinterpret_cast<const float2*>(x + idx)) : make_float2(0.f, 0.f);
        float2 d = ok ? *reinterpret_cast<const float2*>(dx + idx) : make_float2(0.f, 0.f);
        d.x += tc_dpool<FAST>(xv.x, f) * acc[n][4 * jj + 2 * h];
        d.y += tc_dpool<FAST>(xv.y, f) * acc[n][4 * jj + 2 * h + 1];
        if (!FAST && f.rectify) {
          if (!(xv.x > 0.f)) d.x = 0.f;
          if (!(xv.y > 0.f)) d.y = 0.f;
        }
        if (ok) *reinterpret_cast<float2*>(dx + idx) = d;
      }
    }
  }
}

// The literal-pow pass 2 also sums dL/dalpha over the block's rows: partial [blockIdx.x][0].  It is a copy of
// gdn_tc_wide_bwd_dp_kernel rather than a shared inline body: routed through one, the fixed-exponent kernel's
// instruction schedule changed.
template <int C, bool CF>
__global__ void __launch_bounds__(WideCfg<C>::kThreads, 1)
gdn_tc_pow_wide_bwd_dp_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                              const float* __restrict__ q, float* __restrict__ dx, long long n_pix, TcPowFlags f,
                              long long S) {
  using W = WideCfg<C>;
  constexpr int NB = W::kNB;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int j0 = (int)(blockIdx.x % W::kBlocks) * NB;
  fill_planes_block<C, NB, C>(gamma, j0, 0, smem);
  const uint32_t bh = smem_u32(smem), bl = bh + C * NB * 2;
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const long long stride = (long long)(gridDim.x / W::kBlocks) * W::kWG;
  float dal = 0.f;
  for (long long tile = (long long)(blockIdx.x / W::kBlocks) * W::kWG + wg; tile < n_tiles; tile += stride) {
    const long long r0 = tile * kTileM + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = r0 < n_pix, ok1 = r1 < n_pix;
    const long long b0 = row_base<CF>(r0, C, S), b1 = row_base<CF>(r1, C, S);
    float acc[NB / 64][32];
    wide_gemm<C, 1, false, false, false>(acc, q, r0, r1, r0 * C, r1 * C, S, ok0, ok1, t, f, bh, bl);
    if constexpr (CF) {  // the dx read-backs of a 64-column block first, as in gdn_tc_wide_bwd_dp_kernel
#pragma unroll
      for (int n = 0; n < NB / 64; ++n) {
        float2 dv[8][2];
        wide_dx_prefetch(dx, b0, b1, S, ok0, ok1, j0 + 64 * n + 2 * t, dv);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const bool ok = h ? ok1 : ok0;
            const long long idx = (h ? b1 : b0) + ch_off<true>(j0 + 64 * n + 8 * jj + 2 * t, S);
            const float2 xv = ok ? ld_px<0, true>(x, idx, S) : make_float2(0.f, 0.f);
            float2 d = dv[jj][h];
            const float dp0 = acc[n][4 * jj + 2 * h], dp1 = acc[n][4 * jj + 2 * h + 1];
            d.x += tc_dpool<false>(xv.x, f) * dp0;
            d.y += tc_dpool<false>(xv.y, f) * dp1;
            const float e = tc_dalpha_term(xv.x, dp0, f) + tc_dalpha_term(xv.y, dp1, f);
            if (ok) dal += e;
            if (f.rectify) {
              if (!(xv.x > 0.f)) d.x = 0.f;
              if (!(xv.y > 0.f)) d.y = 0.f;
            }
            if (ok) st_px_f2<true>(dx, idx, S, d);
          }
      }
    } else {
      TFCB_FOR_ACC_PAIRS(NB) {
        const bool ok = h ? ok1 : ok0;
        const long long idx = (h ? r1 : r0) * C + j0 + 64 * n + 8 * jj + 2 * t;
        const float2 xv = ok ? __ldg(reinterpret_cast<const float2*>(x + idx)) : make_float2(0.f, 0.f);
        float2 d = ok ? *reinterpret_cast<const float2*>(dx + idx) : make_float2(0.f, 0.f);
        const float dp0 = acc[n][4 * jj + 2 * h], dp1 = acc[n][4 * jj + 2 * h + 1];
        d.x += tc_dpool<false>(xv.x, f) * dp0;
        d.y += tc_dpool<false>(xv.y, f) * dp1;
        const float e = tc_dalpha_term(xv.x, dp0, f) + tc_dalpha_term(xv.y, dp1, f);
        if (ok) dal += e;
        if (f.rectify) {
          if (!(xv.x > 0.f)) d.x = 0.f;
          if (!(xv.y > 0.f)) d.y = 0.f;
        }
        if (ok) *reinterpret_cast<float2*>(dx + idx) = d;
      }
    }
  }
  if (f.part_e != nullptr) cta_exponent_partial<true, false>(dal, 0.f, smem, f.part_e + 2 * blockIdx.x);
}

// dgamma[:, block] and dbeta[block]: gdn_tc_dgamma_kernel with q staged for the block's NB channels only.  CTA
// (part, block) adds into columns [c0, c0 + NB) of partial `part`, so the partials keep the [n_parts][C][C] layout.
// Thread tid stages p channels 8 (tid / 16) .. + 7 of pixels tid % 16 + 16 s, and the same q channels of the block
// when tid / 16 < NB / 8.
template <int C, bool FAST, bool CF, class F>
__device__ __forceinline__ void tc_wide_dgamma_body(const float* __restrict__ x, const float* __restrict__ q,
                                                    float* __restrict__ part_g, float* __restrict__ part_b,
                                                    long long n_pix, const F& f, long long S) {
  using W = WideCfg<C>;
  constexpr int NB = W::kNB;
  constexpr int kP = W::kDgPPlane, kQ = W::kDgQPlane;
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int jc = tid >> 4, pl = tid & 15;
  const bool has_q = jc < NB / 8;
  const int c0 = (int)(blockIdx.x % W::kBlocks) * NB;
  const long long part = blockIdx.x / W::kBlocks, n_parts = gridDim.x / W::kBlocks;
  const long long n_chunks = (n_pix + kTileM - 1) / kTileM;
  float bsum[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) bsum[e] = 0.f;

  auto stage = [&](long long chunk, int buf) {
    uint8_t* base = smem + buf * W::kDgStage;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const int p = pl + 16 * s;
      const long long row = chunk * kTileM + p;
      float v[8], w[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = w[e] = 0.f;
      if (row < n_pix) {
        if constexpr (CF) {
          const long long xb = row_base<true>(row, C, S) + ch_off<true>(8 * jc, S);
#pragma unroll
          for (int e = 0; e < 8; ++e) v[e] = ld_one<0>(x, xb + e * S);
        } else {
          const float4* xr = reinterpret_cast<const float4*>(x + row * C + 8 * jc);
          const float4 x0 = __ldg(xr), x1 = __ldg(xr + 1);
          v[0] = x0.x, v[1] = x0.y, v[2] = x0.z, v[3] = x0.w, v[4] = x1.x, v[5] = x1.y, v[6] = x1.z, v[7] = x1.w;
        }
        if (has_q) {
          const float4* qr = reinterpret_cast<const float4*>(q + row * C + c0 + 8 * jc);
          const float4 q0 = __ldg(qr), q1 = __ldg(qr + 1);
          w[0] = q0.x, w[1] = q0.y, w[2] = q0.z, w[3] = q0.w, w[4] = q1.x, w[5] = q1.y, w[6] = q1.z, w[7] = q1.w;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        // pow(0, alpha) is inf for alpha < 0: rows past the end must stay 0
        if constexpr (kPow<F>)
          v[e] = row < n_pix ? tc_pool<FAST>(v[e], f) : 0.f;
        else
          v[e] = tc_pool<FAST>(v[e], f);
        bsum[e] += w[e];
      }
      const int slot = (jc * kTileM + p) * 16;
      uint4 hi, lo;
      split8(v, &hi, &lo);
      *reinterpret_cast<uint4*>(base + slot) = hi;
      *reinterpret_cast<uint4*>(base + kP + slot) = lo;
      if (has_q) {
        split8(w, &hi, &lo);
        *reinterpret_cast<uint4*>(base + 2 * kP + slot) = hi;
        *reinterpret_cast<uint4*>(base + 2 * kP + kQ + slot) = lo;
      }
    }
  };

  float acc[NB / 64][32];
  float* pg = part_g + part * C * C;
  bool first_flush = true;
  stage(part, 0);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  int k = 0;
  for (long long chunk = part; chunk < n_chunks; chunk += n_parts, ++k) {
    if (k % kDgFlush == 0) {
#pragma unroll
      for (int n = 0; n < NB / 64; ++n)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[n][i] = 0.f;
    }
    // core matrix (channel / 8, pixel / 8) at (channel / 8) * 1024 + (pixel / 8) * 128 bytes of a plane
    const uint32_t base = smem_u32(smem + (k & 1) * W::kDgStage);
    const uint32_t pp[3] = {0, kP, 0}, qp[3] = {2 * kP, 2 * kP, 2 * kP + kQ};  // hi.hi, lo.hi, hi.lo
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTileM / 16; ++kk)
#pragma unroll
      for (int pr = 0; pr < 3; ++pr) {
        const uint64_t a = gmma_desc(base + pp[pr] + wg * 8 * 1024 + 256 * kk, 128, 1024);
#pragma unroll
        for (int n = 0; n < NB / 64; ++n)
          wgmma_ss_mn(acc[n], a, gmma_desc(base + qp[pr] + n * 8 * 1024 + 256 * kk, 128, 1024));
      }
    wgmma_commit();
    const bool last = chunk + n_parts >= n_chunks;
    if (!last) stage(chunk + n_parts, (k + 1) & 1);
    wgmma_wait_all();
    fence_acc(acc);
    if ((k + 1) % kDgFlush == 0 || last) {
      TFCB_FOR_ACC_PAIRS(NB) {
        float2* dst =
            reinterpret_cast<float2*>(pg + (64 * wg + 16 * warp + g + 8 * h) * C + c0 + 64 * n + 8 * jj + 2 * t);
        float2 v = make_float2(acc[n][4 * jj + 2 * h], acc[n][4 * jj + 2 * h + 1]);
        if (!first_flush) {
          const float2 o = *dst;
          v.x += o.x;
          v.y += o.y;
        }
        *dst = v;
      }
      first_flush = false;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
  }
#pragma unroll
  for (int e = 0; e < 8; ++e)
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) bsum[e] += __shfl_xor_sync(0xFFFFFFFFu, bsum[e], o);
  if (has_q && pl == 0) {
#pragma unroll
    for (int e = 0; e < 8; ++e) part_b[part * C + c0 + 8 * jc + e] = bsum[e];
  }
}

template <int C, bool FAST, bool CF>
__global__ void __launch_bounds__(2 * C, 1)
gdn_tc_wide_dgamma_kernel(const float* __restrict__ x, const float* __restrict__ q, float* __restrict__ part_g,
                          float* __restrict__ part_b, long long n_pix, TcFlags f, long long S) {
  tc_wide_dgamma_body<C, FAST, CF>(x, q, part_g, part_b, n_pix, f, S);
}

template <int C, bool CF>
__global__ void __launch_bounds__(2 * C, 1)
gdn_tc_pow_wide_dgamma_kernel(const float* __restrict__ x, const float* __restrict__ q, float* __restrict__ part_g,
                              float* __restrict__ part_b, long long n_pix, TcPowFlags f, long long S) {
  tc_wide_dgamma_body<C, false, CF>(x, q, part_g, part_b, n_pix, f, S);
}

// The kernels of a configuration: gdn_tc_* for TcFlags, gdn_tc_pow_* (float32, FAST = false) for TcPowFlags, in the
// activation layout CF.
template <int C, bool FAST, int IO, bool CF, class F>
auto fwd_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_fwd_kernel<C, CF>;
  else return gdn_tc_fwd_kernel<C, FAST, IO, CF>;
}
template <int C, bool FAST, int IO, bool CF, class F>
auto bwd_dx_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_bwd_dx_kernel<C, CF>;
  else return gdn_tc_bwd_dx_kernel<C, FAST, IO, CF>;
}
template <int C, bool FAST, int IO, bool CF, class F>
auto dgamma_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_dgamma_kernel<C, CF>;
  else return gdn_tc_dgamma_kernel<C, FAST, IO, CF>;
}
template <int C, bool FAST, bool CF, class F>
auto wide_fwd_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_wide_fwd_kernel<C, CF>;
  else return gdn_tc_wide_fwd_kernel<C, FAST, CF>;
}
template <int C, bool FAST, bool CF, class F>
auto wide_bwd_q_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_wide_bwd_q_kernel<C, CF>;
  else return gdn_tc_wide_bwd_q_kernel<C, FAST, CF>;
}
template <int C, bool FAST, bool CF, class F>
auto wide_bwd_dp_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_wide_bwd_dp_kernel<C, CF>;
  else return gdn_tc_wide_bwd_dp_kernel<C, FAST, CF>;
}
template <int C, bool FAST, bool CF, class F>
auto wide_dgamma_kernel() {
  if constexpr (kPow<F>) return gdn_tc_pow_wide_dgamma_kernel<C, CF>;
  else return gdn_tc_wide_dgamma_kernel<C, FAST, CF>;
}

// The launchers take the layout CF and the channels-first item size S (1 channels-last); grids, partial counts and
// everything else depend on n_pix only, so both layouts run the same CTAs over the same tiles.
template <int C, bool FAST, int IO, bool CF, class F>
int launch_tc_fwd(const void* x, const float* gamma, const float* beta, void* y, long long n_pix, F f,
                  cudaStream_t s, long long S) {
  using K = TcCfg<C>;
  const auto kern = fwd_kernel<C, FAST, IO, CF, F>();
  TFCB_TRY(set_smem(kern, K::kSmem));
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const int grid = (int)std::min<long long>((n_tiles + K::kWG - 1) / K::kWG, sm_count());
  kern<<<grid, K::kThreads, K::kSmem, s>>>(x, gamma, beta, y, n_pix, f, S);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// The 16-bit backward's direct-term scratch (gdn_tc_bwd_dx_kernel): one 64 x C float32 tile per warpgroup of a dx
// grid of at most kMaxParts CTAs.
template <int C>
long long bwd16_scratch_floats(long long n_pix) {
  using K = TcCfg<C>;
  const long long n_tiles = (std::max(n_pix, 0LL) + kTileM - 1) / kTileM;
  return std::min<long long>((n_tiles + K::kWG - 1) / K::kWG, kMaxParts) * K::kWG * kTileM * C;
}

// IO != 0: x, dy, dx in 16 bits.  IO != 0 or CF: `scratch` holds bwd16_scratch_floats<C>(n_pix) floats.
// TcPowFlags: the dx kernel's CTAs write f.part_e[CTA][2] (when not null), *n_parts_e of them (at most kMaxParts).
template <int C, bool FAST, int IO, bool CF, class F>
int launch_tc_bwd(const void* x, const float* gamma, const float* beta, const void* dy, void* dx, float* q_ws,
                  float* part_g, float* part_b, float* scratch, int* n_parts, long long n_pix, F f,
                  cudaStream_t s, int* n_parts_e, long long S) {
  using K = TcCfg<C>;
  using L = DgCfg<C>;
  const auto dx_kern = bwd_dx_kernel<C, FAST, IO, CF, F>();
  const auto dg_kern = dgamma_kernel<C, FAST, IO, CF, F>();
  TFCB_TRY(set_smem(dx_kern, K::kSmem));
  TFCB_TRY(set_smem(dg_kern, L::kSmem));
  const int sms = sm_count();
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  // dx does not depend on the grid (every tile is computed the same way by whichever CTA takes it)
  const bool capped = IO != 0 || CF || kPow<F>;
  const int grid = (int)std::min<long long>((n_tiles + K::kWG - 1) / K::kWG, capped ? std::min(sms, kMaxParts) : sms);
  dx_kern<<<grid, K::kThreads, K::kSmem, s>>>(x, gamma, beta, dy, dx, q_ws, n_pix, f, scratch, S);
  TFCB_LAUNCHED();
  const int grid_g = (int)std::min<long long>(n_tiles, std::min(sms, kMaxParts));
  dg_kern<<<grid_g, L::kThreads, L::kSmem, s>>>(static_cast<const IoElem<IO>*>(x), q_ws, part_g, part_b, n_pix, f,
                                                S);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  *n_parts = grid_g;
  if (n_parts_e) *n_parts_e = grid;
  return TFCB_OK;
}

// Wide layers: groups of kBlocks CTAs (one per channel block), as many groups as fill the SMs once.
template <int C>
int wide_grid(long long n_tiles_per_group) {
  using W = WideCfg<C>;
  const long long groups = std::max(1, std::min(sm_count() / W::kBlocks, kMaxParts));
  return (int)(std::min<long long>(n_tiles_per_group, groups) * W::kBlocks);
}

template <int C, bool FAST, bool CF, class F>
int launch_tc_wide_fwd(const float* x, const float* gamma, const float* beta, float* y, long long n_pix, F f,
                       cudaStream_t s, long long S) {
  using W = WideCfg<C>;
  const auto kern = wide_fwd_kernel<C, FAST, CF, F>();
  TFCB_TRY(set_smem(kern, W::kSmem));
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const int grid = wide_grid<C>((n_tiles + W::kWG - 1) / W::kWG);
  kern<<<grid, W::kThreads, W::kSmem, s>>>(x, gamma, beta, y, n_pix, f, S);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// TcPowFlags: CTA b of pass 1 writes f.part_e[b][1] and CTA b of pass 2 f.part_e[b][0] (when not null), *n_parts_e
// partials (at most kMaxParts * kBlocks).
template <int C, bool FAST, bool CF, class F>
int launch_tc_wide_bwd(const float* x, const float* gamma, const float* beta, const float* dy, float* dx, float* q_ws,
                       float* part_g, float* part_b, int* n_parts, long long n_pix, F f, cudaStream_t s,
                       int* n_parts_e, long long S) {
  using W = WideCfg<C>;
  const auto q_kern = wide_bwd_q_kernel<C, FAST, CF, F>();
  const auto dp_kern = wide_bwd_dp_kernel<C, FAST, CF, F>();
  const auto dg_kern = wide_dgamma_kernel<C, FAST, CF, F>();
  TFCB_TRY(set_smem(q_kern, W::kSmem));
  TFCB_TRY(set_smem(dp_kern, W::kSmem));
  TFCB_TRY(set_smem(dg_kern, W::kDgSmem));
  const long long n_tiles = (n_pix + kTileM - 1) / kTileM;
  const int grid = wide_grid<C>((n_tiles + W::kWG - 1) / W::kWG);
  q_kern<<<grid, W::kThreads, W::kSmem, s>>>(x, gamma, beta, dy, dx, q_ws, n_pix, f, S);
  TFCB_LAUNCHED();
  dp_kern<<<grid, W::kThreads, W::kSmem, s>>>(x, gamma, q_ws, dx, n_pix, f, S);
  TFCB_LAUNCHED();
  // one partial per group of kBlocks CTAs (at most sms / kBlocks <= kMaxParts): fixed by n_pix, C and the SM count
  const int grid_g = wide_grid<C>(n_tiles);
  dg_kern<<<grid_g, 2 * C, W::kDgSmem, s>>>(x, q_ws, part_g, part_b, n_pix, f, S);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  *n_parts = grid_g / W::kBlocks;
  if (n_parts_e) *n_parts_e = grid;
  return TFCB_OK;
}

// One instantiation of the kernels: the template arguments with_kernels hands to its function.
template <int C_, bool FAST_, int IO_, bool CF_>
struct Inst {
  static constexpr int C = C_, IO = IO_;
  static constexpr bool FAST = FAST_, CF = CF_;
};

// TcPowFlags as gdn.cu's parse_flags fills GdnFlags (part_e null); a fixed-exponent route's TcFlags are its modes.
TcPowFlags route_flags(const TcRoute& r) {
  return {(r.flags & TFCB_GDN_INVERSE) ? 1 : 0,
          (r.flags & TFCB_GDN_RECTIFY) ? 1 : 0,
          (r.flags & TFCB_GDN_POW_ALPHA) ? 0 : (r.alpha == 1.f ? 1 : (r.alpha == 2.f ? 2 : 0)),
          (r.flags & TFCB_GDN_POW_EPSILON) ? 0 : (r.eps == 1.f ? 1 : (r.eps == 0.5f ? 2 : 0)),
          r.alpha,
          r.eps,
          nullptr};
}

template <int C, bool CF, class Fn>
int with_width(const TcRoute& r, Fn& fn) {
  const TcPowFlags pf = route_flags(r);
  if (r.family == TcRoute::kPow) return fn(Inst<C, false, 0, CF>{}, pf);
  const TcFlags f{pf.inverse, pf.rectify, pf.alpha_mode, pf.eps_mode};
  auto with_io = [&](auto io) {
    constexpr int IO = decltype(io)::value;
    return r.fast ? fn(Inst<C, true, IO, CF>{}, f) : fn(Inst<C, false, IO, CF>{}, f);
  };
  if constexpr (C <= 192) {
    if (r.dtype == 1) return with_io(std::integral_constant<int, 1>{});
    if (r.dtype == 2) return with_io(std::integral_constant<int, 2>{});
  }
  return with_io(std::integral_constant<int, 0>{});
}

// The one map from a route and a layout to the kernels: fn(Inst<C, FAST, IO, CF>{}, flags), flags TcFlags or
// TcPowFlags.  What it instantiates is the kernel set: at C = 128 / 192 the fixed-exponent kernels for FAST x IO and
// the literal-pow ones for IO = 0; at C = 256 / 320 both families for IO = 0; each in both layouts.
template <class Fn>
int with_kernels(const TcRoute& r, bool channels_first, Fn fn) {
  auto with_layout = [&](auto cf) {
    constexpr bool CF = decltype(cf)::value;
    switch (r.C) {
      case 128: return with_width<128, CF>(r, fn);
      case 192: return with_width<192, CF>(r, fn);
      case 256: return with_width<256, CF>(r, fn);
      default: return with_width<320, CF>(r, fn);
    }
  };
  return channels_first ? with_layout(std::true_type{}) : with_layout(std::false_type{});
}

}  // namespace

TcRoute gdn_tc_route(int C, int dtype, int flags, float alpha, float eps) {
  TcRoute r{TcRoute::kNone, false, C, dtype, flags, alpha, eps};
  const char* env = getenv("TFCB_GDN_FP32");  // debugging aid: force the CUDA-core kernels
  if ((env && env[0] == '1') || !(C == 128 || C == 192 || C == 256 || C == 320)) return r;
  const TcPowFlags f = route_flags(r);
  const bool pow = f.alpha_mode == 0 || f.eps_mode == 0;
  if (dtype != 0 && (pow || C > 192 || (dtype != 1 && dtype != 2))) return r;
  r.family = pow ? TcRoute::kPow : TcRoute::kFixed;
  r.fast = f.alpha_mode == 1 && f.eps_mode == 1 && !f.rectify;
  return r;
}

int gdn_tc_forward(const TcRoute& r, bool channels_first, const void* x, const float* gamma, const float* beta, void* y,
                   long long n_pix, long long S, cudaStream_t s) {
  return with_kernels(r, channels_first, [&](auto k, auto f) {
    using K = decltype(k);
    if constexpr (K::C > 192) {
      static_assert(K::IO == 0, "the wide kernels take float32 activations only");
      return launch_tc_wide_fwd<K::C, K::FAST, K::CF>(static_cast<const float*>(x), gamma, beta, static_cast<float*>(y),
                                                       n_pix, f, s, S);
    } else {
      return launch_tc_fwd<K::C, K::FAST, K::IO, K::CF>(x, gamma, beta, y, n_pix, f, s, S);
    }
  });
}

int gdn_tc_backward(const TcRoute& r, bool channels_first, const void* x, const float* gamma, const float* beta,
                    const void* dy, void* dx, float* q, float* part_g, float* part_b, float* part_e, float* scratch,
                    long long n_pix, long long S, cudaStream_t s, int* n_parts, int* n_parts_e) {
  return with_kernels(r, channels_first, [&](auto k, auto f) {
    using K = decltype(k);
    if constexpr (kPow<decltype(f)>) f.part_e = part_e;
    if constexpr (K::C > 192)
      return launch_tc_wide_bwd<K::C, K::FAST, K::CF>(static_cast<const float*>(x), gamma, beta,
                                                       static_cast<const float*>(dy), static_cast<float*>(dx), q,
                                                       part_g, part_b, n_parts, n_pix, f, s, n_parts_e, S);
    else
      return launch_tc_bwd<K::C, K::FAST, K::IO, K::CF>(x, gamma, beta, dy, dx, q, part_g, part_b, scratch, n_parts,
                                                         n_pix, f, s, n_parts_e, S);
  });
}

long long gdn_tc_scratch_floats(long long n_pix, int C) {
  if (C == 128) return bwd16_scratch_floats<128>(n_pix);
  if (C == 192) return bwd16_scratch_floats<192>(n_pix);
  return 0;
}

}  // namespace tfcb
