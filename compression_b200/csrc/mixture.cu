// Mixture priors on the range coder (DESIGN.md §3.18), sm_90a.  The chain, drain, finalize and escape code are the
// range coder's (range_coder.cuh); only the rows are new.
#include <algorithm>
#include <cmath>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "range_coder.cuh"

// ---------------------------------------------------------------------------------------------
// Mixture priors (DESIGN.md §3.18): every element coded with its own row, built on the device from K weights, locs
// and scales (family Normal or Logistic).  The row is the index-mode overflow row [-p, c_0 .. c_n] of the support
// a, .., a + L - 1 plus the escape bin, so the strings are the reference RangeEncoder's; nothing is tabulated.
//   support  lo = min_k (mu_k - t s_k), hi = max_k (mu_k + t s_k) over w_k > 0 (float32, __fmul_rn / __fsub_rn /
//            __fadd_rn); a = floorf(lo), L = ceilf(hi) - a + 1 when that is <= max_support, else L = max_support
//            and a = rintf(sum_k (w_k / W) mu_k) - (max_support - 1) / 2; a is clamped to [-2^30, 2^30].
//   masses   m_i = min(floor(2^32 q_i), 2^32 - 1), q_i = sum_k (w_k / W) dF_k(a + i) in float32, dF_k on the side of
//            mu_k away from the bin (cancellation-free); m_L = max(0, 2^32 - sum m_i); T = sum_{i <= L} m_i.
//   CDF      c_j = j + floor((2^p - n) S_j / T), S_j = sum_{i < j} m_i, n = L + 1: exact 64-bit integers.
// ---------------------------------------------------------------------------------------------
namespace tfcb {
namespace {

// Named barriers (bar.sync / bar.arrive) between the decoder's producer warps and its chain warp.  The id is an
// immediate, so ptxas reserves only the barriers used: 1 + b (rows of buffer b ready), 3 + b (buffer b free).
template <int ID>
__device__ __forceinline__ void bar_sync(int count) {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(count) : "memory");
}
template <int ID>
__device__ __forceinline__ void bar_arrive(int count) {
  asm volatile("bar.arrive %0, %1;" ::"n"(ID), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_sync_buf(int base, int b, int count) {
  if (base == 1) b ? bar_sync<2>(count) : bar_sync<1>(count);
  else b ? bar_sync<4>(count) : bar_sync<3>(count);
}
__device__ __forceinline__ void bar_arrive_buf(int base, int b, int count) {
  if (base == 1) b ? bar_arrive<2>(count) : bar_arrive<1>(count);
  else b ? bar_arrive<4>(count) : bar_arrive<3>(count);
}

constexpr int kMixMaxSupport = 256;
constexpr unsigned long long kMixNone = ~0ull;
constexpr int kMixMaxK = 64;
constexpr int kMixProducers = 8;  // row-building warps per decode CTA
enum : int { kMixNormal = 0, kMixLogistic = 1 };
// error key g << 3 | kind (g: element over the whole batch), kept with atomicMin in DevError::stream
enum : int { kMixNonFinite = 1, kMixScale = 2, kMixWeight = 3, kMixZero = 4, kMixTiny = 5 };

struct MixParams {
  const float* w;
  const float* loc;
  const float* scale;
  int K, family;
  uint32_t p;
  int max_support;
  float t;  // the family's upper quantile at tail_mass / 2
};

struct MixSupport {
  int a, L;  // L = 0: invalid parameters (recorded)
  float winv;  // 1 / W
};

// Standard CDF F(z) of the family.
__device__ __forceinline__ float mix_cdf(int family, float z) {
  if (family == kMixNormal) return __fmul_rn(0.5f, erfcf(__fmul_rn(z, -0.70710678118654752f)));
  return __frcp_rn(__fadd_rn(1.f, expf(-z)));
}

// Checks element e's parameters and finds its support; records the first failure of the element under atomicMin.
__device__ __forceinline__ MixSupport mix_support(const MixParams& P, long long e, long long g, DevError* err) {
  MixSupport s{0, 0, 0.f};
  const float* w = P.w + e * P.K;
  const float* mu = P.loc + e * P.K;
  const float* sg = P.scale + e * P.K;
  float W = 0.f;
  int kind = 0;
  for (int k = 0; k < P.K; ++k) {
    const float wk = w[k], mk = mu[k], sk = sg[k];
    if (!isfinite(wk) || !isfinite(mk) || !isfinite(sk)) kind = kind ? kind : kMixNonFinite;
    else if (!(sk > 0.f)) kind = kind ? kind : kMixScale;
    else if (wk < 0.f) kind = kind ? kind : kMixWeight;
    W = __fadd_rn(W, wk);
  }
  if (!kind && !(W > 0.f)) kind = kMixZero;
  if (!kind && !isfinite(W)) kind = kMixNonFinite;
  if (kind) {
    ubi_key(&err->stream, ((unsigned long long)g << 3) | (unsigned)kind);
    return s;
  }
  s.winv = __frcp_rn(W);
  if (!isfinite(s.winv)) {  // W below 2^-126: the normalised weights would overflow
    ubi_key(&err->stream, ((unsigned long long)g << 3) | (unsigned)kMixTiny);
    return s;
  }
  float lo = INFINITY, hi = -INFINITY, mean = 0.f;
  for (int k = 0; k < P.K; ++k) {
    const float wk = w[k];
    if (!(wk > 0.f)) continue;
    const float ts = __fmul_rn(P.t, sg[k]);
    lo = fminf(lo, __fsub_rn(mu[k], ts));
    hi = fmaxf(hi, __fadd_rn(mu[k], ts));
    mean = __fadd_rn(mean, __fmul_rn(__fmul_rn(wk, s.winv), mu[k]));
  }
  float af = floorf(lo);
  const float width = __fadd_rn(__fsub_rn(ceilf(hi), af), 1.f);
  if (width <= (float)P.max_support) {
    s.L = (int)width;
  } else {
    s.L = P.max_support;
    af = __fsub_rn(rintf(mean), (float)((P.max_support - 1) / 2));
  }
  s.a = (int)fminf(fmaxf(af, -1073741824.f), 1073741824.f);
  return s;
}

// m_x: the mass of integer x (a bin of the support) in units of 2^-32, truncated and clamped to [0, 2^32 - 1].
__device__ __forceinline__ uint32_t mix_mass(const MixParams& P, long long e, float winv, int x) {
  const float* w = P.w + e * P.K;
  const float* mu = P.loc + e * P.K;
  const float* sg = P.scale + e * P.K;
  const float xf = (float)x;
  float q = 0.f;
  for (int k = 0; k < P.K; ++k) {
    const float wk = w[k];
    if (!(wk > 0.f)) continue;
    const float d = __fsub_rn(xf, mu[k]);
    const float zl = __fdiv_rn(__fsub_rn(d, 0.5f), sg[k]);
    const float zh = __fdiv_rn(__fadd_rn(d, 0.5f), sg[k]);
    // above the median F(zh) - F(zl) = F(-zl) - F(-zh): both terms small, no cancellation
    const float df = d > 0.f ? __fsub_rn(mix_cdf(P.family, -zl), mix_cdf(P.family, -zh))
                             : __fsub_rn(mix_cdf(P.family, zh), mix_cdf(P.family, zl));
    q = __fadd_rn(q, __fmul_rn(__fmul_rn(wk, winv), fmaxf(df, 0.f)));
  }
  const float m = __fmul_rn(q, 4294967296.f);
  return m >= 4294967296.f ? 0xFFFFFFFFu : (uint32_t)m;
}

// c_j of the quantised CDF: j + floor((2^p - n) S_j / T).
__device__ __forceinline__ uint32_t mix_cdf_entry(uint32_t p, int n, int j, unsigned long long Sj,
                                                  unsigned long long T) {
  return (uint32_t)j + (uint32_t)((((1ull << p) - (unsigned long long)n) * Sj) / T);
}

// One row built by one warp, lanes over the bins: masses into row[1 .. L] (as uint32), their sum, then the CDF in
// place.  `mass_out` (tables entry only) receives m_0 .. m_L.  Returns the support (L = 0: invalid parameters).
__device__ __forceinline__ MixSupport mix_build_row(const MixParams& P, long long e, long long g, DevError* err, uint32_t* row,
                                    long long* mass_out, int lane) {
  const MixSupport sp = mix_support(P, e, g, err);
  if (sp.L == 0) return sp;
  unsigned long long sum = 0;
  for (int i = lane; i < sp.L; i += 32) {
    const uint32_t m = mix_mass(P, e, sp.winv, sp.a + i);
    row[i + 1] = m;
    sum += m;
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) sum += __shfl_xor_sync(kFull, sum, d);
  const unsigned long long two32 = 1ull << 32;
  const unsigned long long esc = sum < two32 ? two32 - sum : 0ull;
  const unsigned long long T = sum + esc;
  const int n = sp.L + 1;
  __syncwarp();
  unsigned long long carry = 0;
  for (int i0 = 0; i0 < sp.L; i0 += 32) {
    const int i = i0 + lane;
    const unsigned long long m = i < sp.L ? (unsigned long long)row[i + 1] : 0ull;
    if (mass_out && i < sp.L) mass_out[i] = (long long)m;
    unsigned long long incl = m;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const unsigned long long t = __shfl_up_sync(kFull, incl, d);
      if (lane >= d) incl += t;
    }
    __syncwarp();
    if (i < sp.L) row[i + 1] = mix_cdf_entry(P.p, n, i + 1, carry + incl, T);
    carry += __shfl_sync(kFull, incl, 31);
  }
  if (lane == 0) {
    row[0] = 0u;
    row[n] = 1u << P.p;
    if (mass_out) mass_out[sp.L] = (long long)esc;
  }
  __syncwarp();
  return sp;
}

// Tables entry: one warp per element; rows padded to max_support + 3 entries as the reference's 2-D lookup.
__global__ void __launch_bounds__(256) mix_tables_kernel(const MixParams P, long long n, int32_t* start,
                                                         int32_t* size, long long* mass, int32_t* rows,
                                                         DevError* err) {
  const int lane = threadIdx.x & 31;
  const long long e = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (e >= n) return;
  const int W = P.max_support + 3;
  int32_t* r = rows + e * W;
  long long* me = mass + e * (P.max_support + 1);
  const MixSupport sp = mix_build_row(P, e, e, err, reinterpret_cast<uint32_t*>(r + 1), me, lane);
  if (lane == 0) {
    start[e] = sp.a;
    size[e] = sp.L;
    r[0] = -(int32_t)P.p;
  }
  const int pad = sp.L == 0 ? 0 : (int32_t)(1u << P.p);
  for (int j = (sp.L == 0 ? 0 : sp.L + 2) + lane; j < W - 1; j += 32) r[1 + j] = pad;
  for (int j = (sp.L == 0 ? 0 : sp.L + 1) + lane; j <= P.max_support; j += 32) me[j] = 0;
}

// Coder operands of one element (12 bytes): lower | sign << 31, upper, and the Elias-gamma payload (0: no escape).
struct MixOps {
  uint32_t lo_sign, hi, gamma;
};

// Operand pass: one thread per element.  v = int32(rint(y)) (saturating, NaN -> 0), d = v - a (wrapping), coded as
// bin d when 0 <= d < L, else as the escape bin L followed by OverflowEncode's payload.
__global__ void __launch_bounds__(256) mix_operands_kernel(const MixParams P, const float* y, long long n,
                                                           MixOps* ops, DevError* err) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= n) return;
  MixOps o{0u, 1u << P.p, 0u};
  const MixSupport sp = mix_support(P, e, e, err);
  if (sp.L == 0) {
    ops[e] = o;
    return;
  }
  const int v = (int)rintf(y[e]);
  const int d = (int)((uint32_t)v - (uint32_t)sp.a);
  int bin = d;
  uint32_t sign = 0;
  if (d < 0) {
    o.gamma = (uint32_t)(-(long long)d);
    sign = 1;
    bin = sp.L;
  } else if (d >= sp.L) {
    o.gamma = (uint32_t)(d - sp.L + 1);
    bin = sp.L;
  }
  unsigned long long S0 = 0, S1 = 0, sum = 0;
  for (int i = 0; i < sp.L; ++i) {
    const uint32_t m = mix_mass(P, e, sp.winv, sp.a + i);
    if (i < bin) S0 += m;
    if (i <= bin) S1 += m;
    sum += m;
  }
  const unsigned long long two32 = 1ull << 32;
  const unsigned long long T = sum < two32 ? two32 : sum;
  const int nb = sp.L + 1;
  o.lo_sign = mix_cdf_entry(P.p, nb, bin, S0, T) | (sign << 31);
  o.hi = bin == sp.L ? (1u << P.p) : mix_cdf_entry(P.p, nb, bin + 1, S1, T);
  ops[e] = o;
}

// One warp per stream, ubi_encode_kernel's chain: every lane runs the recurrence, lane j keeps entry j of the
// current 32, and an escape is followed by gamma_record's bits (the encode kernel's escape records).
__global__ void __launch_bounds__(32) mix_encode_kernel(const MixOps* ops, uint32_t p, const long long* elem_off,
                                                        const long long* arena_off, EncState* state, uint16_t* words,
                                                        uint32_t* cbits, DevError* err) {
  __shared__ __align__(8) uint2 s_ent[32];
  const int lane = threadIdx.x;
  const long long s = blockIdx.x;
  const Extent e = stream_extent(elem_off, s, 0);
  const Extent a = stream_extent(arena_off, s, 0);
  const EncState st0 = enc_initial_state();
  EncChain c;
  c.s = st0.raw;
  EncDrain d;
  d.begin(st0, words + a.base, cbits + (a.base >> 5), (uint32_t)a.len, lane);
  uint2 mine = make_uint2(0u, 0u);
  int fill = 0;
  auto push = [&](uint4 o) {
    const uint2 ent = c.step(o);
    if (lane == fill) mine = ent;
    if (++fill == 32) {
      s_ent[lane] = mine;
      __syncwarp();
      d.drain<1>(s_ent, 32);
      __syncwarp();
      fill = 0;
    }
  };
  for (long long g0 = 0; g0 < e.len; g0 += 32) {
    const int count = (int)min(32ll, e.len - g0);
    MixOps m{0u, 0u, 0u};
    if (lane < count) m = ops[e.base + g0 + lane];
    for (int k = 0; k < count; ++k) {
      const uint32_t ls = __shfl_sync(kFull, m.lo_sign, k);
      push(enc_operands(ls & 0x7FFFFFFFu, __shfl_sync(kFull, m.hi, k), p));
      const uint32_t gk = __shfl_sync(kFull, m.gamma, k);
      if (gk) {
        const int nb = 32 - __clz(gk);
        for (int i = 0; i < 2 * nb; ++i) push(gamma_record(gk, ls >> 31, nb, i));
      }
    }
  }
  if (fill) {
    s_ent[lane] = mine;
    __syncwarp();
    d.drain<1>(s_ent, fill);
    __syncwarp();
  }
  d.end(err, s);
  if (lane == 0) {
    EncState st;
    st.base = d.dbase;
    st.span = (c.s < 65536u) ? ((c.s << 16) | 0xFFFFu) : c.s;
    st.cnt = d.cnt;
    st.raw = c.s;
    state[s] = st;
  }
}

// Decode: one CTA per stream.  Warp 0 runs the chain (dec_symbol / dec_update and the escape); warps 1 ..
// kMixProducers build the rows of the next group of 32 elements into a double-buffered shared-memory ring, so row
// building stays off the serial chain and rows never reach global memory.
struct MixDecMeta {
  int a, L;
};

__global__ void __launch_bounds__(32 * (kMixProducers + 1)) mix_decode_kernel(const MixParams P, const uint8_t* bytes,
                                                                             const long long* str_off,
                                                                             const long long* elem_off, float* out,
                                                                             DevError* err) {
  extern __shared__ __align__(16) uint32_t s_rows[];  // [2][32][max_support + 2]
  __shared__ MixDecMeta meta[2][32];
  __shared__ int stop;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const long long s = blockIdx.x;
  const Extent x = stream_extent(elem_off, s, 0);
  const long long n_groups = (x.len + 31) / 32;
  const int RW = P.max_support + 2;
  const int nthreads = 32 * (kMixProducers + 1);
  if (threadIdx.x == 0) stop = 0;
  __syncthreads();

  if (warp > 0) {
    for (long long g = 0; g < n_groups; ++g) {
      const int b = (int)(g & 1);
      if (g >= 2) bar_sync_buf(3, b, nthreads);
      const int count = (int)min(32ll, x.len - g * 32);
      if (!*(volatile int*)&stop) {
        for (int j = warp - 1; j < count; j += kMixProducers) {
          const long long el = x.base + g * 32 + j;
          const MixSupport sp = mix_build_row(P, el, el, err, s_rows + (b * 32 + j) * RW, nullptr, lane);
          if (lane == 0) meta[b][j] = MixDecMeta{sp.a, sp.L};
        }
      }
      bar_arrive_buf(1, b, nthreads);
    }
    return;
  }

  DecChain c;
  c.base = 0;
  c.span = 0xFFFFFFFFu;
  ByteWindow win;
  const Extent bx = stream_extent(str_off, s, 0);
  win.p = bytes + bx.base;
  win.len = bx.len;
  c.value = (bw_fetch(win, 0) << 16) | bw_fetch(win, 1);
  c.pos = 2;
  bw_seek(win, c.pos, lane);
  bool stopped = false;
  for (long long g = 0; g < n_groups; ++g) {
    const int b = (int)(g & 1);
    bar_sync_buf(1, b, nthreads);
    const int count = (int)min(32ll, x.len - g * 32);
    float my_val = 0.f;
    int done = stopped ? 0 : count;
    for (int k = 0; k < done; ++k) {
      const MixDecMeta m = meta[b][k];
      if (m.L == 0) {  // invalid parameters, recorded by the producer
        done = k;
        stopped = true;
        if (lane == 0) stop = 1;
        break;
      }
      const int sym = dec_symbol(c, win, reinterpret_cast<const int32_t*>(s_rows + (b * 32 + k) * RW), m.L + 2, P.p,
                                 lane);
      uint32_t v = (uint32_t)sym;
      if (sym == m.L) {  // OverflowDecode (range_coder_kernels.cc:449-471), capped as decode_kernel's
        int nb = 0;
        while (nb < 32 && ubi_dec_uniform(c, win, 1u, lane) == 0u) ++nb;
        uint32_t val = nb < 32 ? (1u << nb) : 0u;
        for (int t = nb - 1; t >= 0; --t) {
          const uint32_t bit = ubi_dec_uniform(c, win, 1u, lane);
          if (t < 32) val |= bit << t;
        }
        const uint32_t sg = ubi_dec_uniform(c, win, 1u, lane);
        v = sg ? 0u - val : val + (uint32_t)m.L - 1u;
      }
      v += (uint32_t)m.a;
      if (lane == k) my_val = (float)(int32_t)v;
    }
    if (lane < done) out[x.base + g * 32 + lane] = my_val;
    if (g + 2 < n_groups) bar_arrive_buf(3, b, nthreads);
  }
}

// ---- host side ----
// The family's upper quantile at tail_mass / 2 in double: Normal by bisection on erfc, Logistic in closed form.
double mix_quantile(int family, double tail_mass) {
  if (family == kMixLogistic) return std::log(2.0 / tail_mass - 1.0);
  double lo = 0.0, hi = 40.0;  // 0.5 erfc(z / sqrt 2) = tail_mass / 2
  for (int i = 0; i < 200; ++i) {
    const double mid = 0.5 * (lo + hi);
    if (std::erfc(mid / std::sqrt(2.0)) > tail_mass) lo = mid;
    else hi = mid;
  }
  return 0.5 * (lo + hi);
}

int mix_check(const float* w, const float* loc, const float* scale, long long n, int K, int family, int precision,
              double tail_mass, int max_support, MixParams* P) {
  if (family != kMixNormal && family != kMixLogistic)
    return fail(TFCB_INVALID_ARGUMENT, "`family` must be 0 (normal) or 1 (logistic): %d", family);
  if (!(1 <= K && K <= kMixMaxK)) return fail(TFCB_INVALID_ARGUMENT, "`K` must be in [1, %d]: %d", kMixMaxK, K);
  if (!(1 <= max_support && max_support <= kMixMaxSupport))
    return fail(TFCB_INVALID_ARGUMENT, "`max_support` must be in [1, %d]: %d", kMixMaxSupport, max_support);
  if (!(1 <= precision && precision <= 16) || (1 << precision) <= max_support)
    return fail(TFCB_INVALID_ARGUMENT, "`precision` must be in [1, 16] with 2^precision > max_support (%d): %d",
                max_support, precision);
  if (!(tail_mass > 0.0 && tail_mass < 1.0))
    return fail(TFCB_INVALID_ARGUMENT, "`tail_mass` must be in (0, 1): %g", tail_mass);
  if (n < 0 || n * (long long)K >= (1ll << 40)) return fail(TFCB_INVALID_ARGUMENT, "bad element count: %lld", n);
  if (n > 0 && (!w || !loc || !scale)) return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  P->w = w;
  P->loc = loc;
  P->scale = scale;
  P->K = K;
  P->family = family;
  P->p = (uint32_t)precision;
  P->max_support = max_support;
  P->t = (float)mix_quantile(family, tail_mass);
  return TFCB_OK;
}

// The error record's lowest key as a message naming the string and element.
int mix_error(const DevError& e, const int64_t* item_offsets, int64_t n_items) {
  if (e.code == kErrCapacity)
    return fail(TFCB_CUDA_ERROR, "internal: output arena too small (string %lld needs > %lld words)", e.stream,
                e.limit);
  const unsigned long long key = (unsigned long long)e.stream;
  if (key == kMixNone) return TFCB_OK;
  const long long g = (long long)(key >> 3);
  long long item = 0, elem = g;
  if (item_offsets) {
    const int64_t* hi = std::upper_bound(item_offsets, item_offsets + n_items + 1, (int64_t)g);
    item = (long long)(hi - item_offsets) - 1;
    elem = g - item_offsets[item];
  }
  static const char* const what[] = {"", "a non-finite weight, loc or scale", "a scale <= 0", "a negative weight",
                                     "all weights 0", "weights whose sum is too small to normalise (below 2^-126)"};
  const int kind = (int)(key & 7ull);
  return fail(TFCB_INVALID_ARGUMENT, "mixture parameters: %s (string %lld, element %lld)",
              kind >= 1 && kind <= 5 ? what[kind] : "unknown", item, elem);
}

// Synchronises once and reads the error record back.
int mix_sync_error(DevError* err, cudaStream_t s, DevError* out) {
  cudaError_t ce = cudaMemcpyAsync(out, err, sizeof *out, cudaMemcpyDeviceToHost, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(TFCB_CUDA_ERROR, "CUDA error '%s' in mixture coder", cudaGetErrorString(ce));
  }
  return TFCB_OK;
}

// The error record with every key at "none".
int mix_reset_error(DevError* err, cudaStream_t s) {
  TFCB_CUDA_TRY(cudaMemsetAsync(err, 0, sizeof(DevError), s));
  TFCB_CUDA_TRY(cudaMemsetAsync(&err->stream, 0xFF, 3 * sizeof(long long), s));
  return TFCB_OK;
}

int mix_check_items(int64_t n_items, const int64_t* item_offsets) {
  if (n_items >= (1ll << 31)) return fail(TFCB_INVALID_ARGUMENT, "too many strings: %lld", (long long)n_items);
  return check_symbol_offsets(item_offsets, n_items);
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

struct tfcb_mixture_encoder {
  long long n_streams = 0;
  EncState* state = nullptr;
  uint16_t* words = nullptr;
  uint32_t* cbits = nullptr;
  DevError* err = nullptr;
  long long* ext = nullptr;  // device [2 * (n_streams + 1)]: element offsets, then arena offsets
  const long long* arena_off = nullptr;
  long long* offsets = nullptr;
  MixOps* ops = nullptr;
  cudaStream_t s = nullptr;
};

namespace {
void mix_release(tfcb_mixture_encoder* h, cudaStream_t s) {
  dev_free(h->state, s);
  dev_free(h->words, s);
  dev_free(h->cbits, s);
  dev_free(h->err, s);
  dev_free(h->ext, s);
  dev_free(h->ops, s);
  delete h;
}
}  // namespace

extern "C" {

int tfcb_mixture_tables(const float* weight_dev, const float* loc_dev, const float* scale_dev, int64_t n, int K,
                        int family, int precision, double tail_mass, int max_support, int32_t* start_dev,
                        int32_t* size_dev, int64_t* mass_dev, int32_t* rows_dev, void* stream) {
  MixParams P{};
  TFCB_TRY(mix_check(weight_dev, loc_dev, scale_dev, n, K, family, precision, tail_mass, max_support, &P));
  if (n > 0 && (!start_dev || !size_dev || !mass_dev || !rows_dev))
    return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  cudaStream_t s = as_stream(stream);
  DevError* err = nullptr;
  int rc = dev_alloc((void**)&err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = mix_reset_error(err, s);
  DevError e{};
  if (rc == TFCB_OK && n > 0) {
    mix_tables_kernel<<<(unsigned)((n + 7) / 8), 256, 0, s>>>(P, n, start_dev, size_dev, reinterpret_cast<long long*>(mass_dev),
                                             rows_dev, err);
    TFCB_LAUNCHED();
  }
  if (rc == TFCB_OK) rc = mix_sync_error(err, s, &e);
  if (rc == TFCB_OK) rc = mix_error(e, nullptr, 0);
  dev_free(err, s);
  return rc;
}

int tfcb_mixture_encode_ragged(const float* y_dev, const float* weight_dev, const float* loc_dev,
                               const float* scale_dev, int K, int family, int precision, double tail_mass,
                               int max_support, int64_t n_items, const int64_t* item_offsets_host, int64_t* offsets_dev,
                               void* stream, tfcb_mixture_encoder** out, int64_t* total_bytes_host) {
  TFCB_TRY(mix_check_items(n_items, item_offsets_host));
  const long long S = n_items, n = item_offsets_host[S];
  MixParams P{};
  TFCB_TRY(mix_check(weight_dev, loc_dev, scale_dev, n, K, family, precision, tail_mass, max_support, &P));
  if (!out || !total_bytes_host || !offsets_dev || (!y_dev && n > 0))
    return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  const long long bits = bits_bound(precision, true);
  std::vector<long long> off(2 * (S + 1));
  long long* arena = off.data() + S + 1;
  long long total = 0;
  for (long long i = 0; i <= S; ++i) {
    off[i] = item_offsets_host[i];
    arena[i] = total;
    if (i == S) break;
    const long long m = item_offsets_host[i + 1] - item_offsets_host[i];
    if (m > ((kMaxStreamWords - 96) * 16) / bits)
      return fail(TFCB_INVALID_ARGUMENT, "string %lld: %lld elements may not fit one code stream (2^31 16-bit words)",
                  i, m);
    total += (words_for(bits, m) + 32 + 31) & ~31ll;
  }
  *out = nullptr;
  *total_bytes_host = 0;
  cudaStream_t s = as_stream(stream);
  auto* h = new tfcb_mixture_encoder;
  h->n_streams = S;
  h->s = s;
  h->offsets = reinterpret_cast<long long*>(offsets_dev);
  int rc = dev_alloc((void**)&h->state, (size_t)S * sizeof(EncState), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->words, (size_t)total * sizeof(uint16_t), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->cbits, (size_t)(total >> 5) * sizeof(uint32_t), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->ext, off.size() * sizeof(long long), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->ops, (size_t)std::max(n, 1ll) * sizeof(MixOps), s);
  if (rc == TFCB_OK) rc = mix_reset_error(h->err, s);
  if (rc == TFCB_OK) {
    const cudaError_t e = cudaMemcpyAsync(h->ext, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      rc = fail(TFCB_CUDA_ERROR, "mixture encode: %s", cudaGetErrorString(e));
    }
  }
  if (rc != TFCB_OK) {
    mix_release(h, s);
    return rc;
  }
  h->arena_off = h->ext + S + 1;
  if (n > 0) {
    mix_operands_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(P, y_dev, n, h->ops, h->err);
    TFCB_LAUNCHED();
  }
  mix_encode_kernel<<<(unsigned)S, 32, 0, s>>>(h->ops, P.p, h->ext, h->arena_off, h->state, h->words, h->cbits,
                                               h->err);
  TFCB_LAUNCHED();
  long long bytes = 0;
  DevError e{};
  rc = ragged_arena_offsets(S, h->state, h->words, h->cbits, h->err, h->arena_off, h->offsets, s, &bytes, &e);
  if (rc == TFCB_OK) rc = mix_error(e, item_offsets_host, n_items);
  if (rc != TFCB_OK) {
    mix_release(h, s);
    return rc;
  }
  *total_bytes_host = bytes;
  *out = h;
  return TFCB_OK;
}

int tfcb_mixture_write(tfcb_mixture_encoder* h, uint8_t* bytes_dev, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "mixture encode: not an encoder handle");
  cudaStream_t s = as_stream(stream);
  int rc = TFCB_OK;
  if (!bytes_dev) {
    rc = fail(TFCB_INVALID_ARGUMENT, "mixture encode: null output buffer");
  } else {
    ragged_arena_write(h->n_streams, h->state, h->words, h->cbits, h->err, h->arena_off, h->offsets, bytes_dev, s);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(TFCB_CUDA_ERROR, "mixture encode: %s", cudaGetErrorString(e));
  }
  mix_release(h, s);
  return rc;
}

void tfcb_mixture_encoder_destroy(tfcb_mixture_encoder* h) {
  if (h) mix_release(h, h->s);
}

int tfcb_mixture_decode_ragged(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_items,
                               const int64_t* item_offsets_host, const float* weight_dev, const float* loc_dev,
                               const float* scale_dev, int K, int family, int precision, double tail_mass,
                               int max_support, float* out_dev, void* stream) {
  TFCB_TRY(mix_check_items(n_items, item_offsets_host));
  const long long S = n_items, n = item_offsets_host[S];
  MixParams P{};
  TFCB_TRY(mix_check(weight_dev, loc_dev, scale_dev, n, K, family, precision, tail_mass, max_support, &P));
  if (!bytes_dev || !offsets_dev || (!out_dev && n > 0)) return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  cudaStream_t s = as_stream(stream);
  const size_t smem = (size_t)2 * 32 * (max_support + 2) * sizeof(uint32_t);
  static std::once_flag once;
  static cudaError_t attr = cudaSuccess;
  std::call_once(once, [] {
    attr = cudaFuncSetAttribute(mix_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                2 * 32 * (kMixMaxSupport + 2) * (int)sizeof(uint32_t));
  });
  if (attr != cudaSuccess) return fail(TFCB_CUDA_ERROR, "mixture decode: %s", cudaGetErrorString(attr));
  DevError* err = nullptr;
  long long* elem_off = nullptr;
  int rc = dev_alloc((void**)&err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&elem_off, (size_t)(S + 1) * sizeof(long long), s);
  if (rc == TFCB_OK) rc = mix_reset_error(err, s);
  if (rc == TFCB_OK &&
      cudaMemcpyAsync(elem_off, item_offsets_host, (size_t)(S + 1) * sizeof(long long), cudaMemcpyHostToDevice, s) !=
          cudaSuccess) {
    (void)cudaGetLastError();
    rc = fail(TFCB_CUDA_ERROR, "mixture decode: could not upload the item offsets");
  }
  DevError e{};
  if (rc == TFCB_OK) {
    mix_decode_kernel<<<(unsigned)S, 32 * (kMixProducers + 1), smem, s>>>(
        P, bytes_dev, reinterpret_cast<const long long*>(offsets_dev), elem_off, out_dev, err);
    TFCB_LAUNCHED();
    rc = mix_sync_error(err, s, &e);
  }
  if (rc == TFCB_OK) rc = mix_error(e, item_offsets_host, n_items);
  dev_free(err, s);
  dev_free(elem_off, s);
  return rc;
}

}  // extern "C"
