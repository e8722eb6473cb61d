// Range decoder device code shared by the decode kernels (range_coder.cu) and the autoregressive decoder step
// (autoregressive.cu): the decoder state, the coder's row descriptors, the byte window, and Dec2, the interval
// recurrence with its pre-scaled search keys.  One definition: the two decoders cannot drift apart.
#pragma once
#include <stdint.h>

#include "common.cuh"

struct tfcb_decoder;

namespace tfcb {

struct DecState {
  uint32_t base, span, value;
  uint32_t pos;  // 16-bit words consumed (starts at 2)
};

// What a kernel outside range_coder.cu needs of a decoder handle (tfcb_decoder is private to range_coder.cu): the
// coding tables as the decoder uploaded them, the strings, and the per-stream state and error record it continues.
struct DecoderView {
  const int2* rows;    // {start, meta} per table row
  const uint2* pairs;  // pre-scaled search keys of every row
  const int4* rows4;   // {key segment start, meta, first window index, irregular}
  int n_rows;
  long long n_pairs;
  const uint8_t* bytes;
  const long long* offsets;
  long long n_streams;
  DecState* state;
  DevError* err;
};

// Fills `v` from a decoder handle; TFCB_INVALID_ARGUMENT if `h` is null.
int decoder_view(tfcb_decoder* h, DecoderView* v);

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;

// meta = ncdf | |precision| << 24 | overflow << 31
__host__ __device__ inline int row_ncdf(int meta) { return meta & 0xFFFFFF; }
__host__ __device__ inline int row_prec(int meta) { return (meta >> 24) & 0x1F; }
__host__ __device__ inline bool row_ovf(int meta) { return meta < 0; }

struct ByteWindow {
  const uint8_t* p;
  long long len;
  uint32_t lane_word;  // word (pos & ~31) + lane
  uint32_t next;       // word at index pos
};

__device__ __forceinline__ uint32_t bw_fetch(const ByteWindow& w, long long word_idx) {
  const long long b = 2 * word_idx;
  uint32_t hi = 0, lo = 0;
  if (b < w.len) hi = w.p[b];
  if (b + 1 < w.len) lo = w.p[b + 1];
  return (hi << 8) | lo;
}

constexpr int kRing = 2048;       // words; the prepare warp keeps [pos, pos + kRingAhead) valid

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ uint32_t opaque(uint32_t x) {
  asm volatile("mov.u32 %0, %0;" : "+r"(x));
  return x;
}

__device__ __forceinline__ uint32_t key_bound(uint32_t span, uint2 q) {  // B'(c) = floor(size*c/2^p) - 1
  return (uint32_t)(((unsigned long long)span * q.x + (((unsigned long long)q.y << 32) | q.x)) >> 32);
}

__device__ __forceinline__ uint2 lds_v2(uint32_t addr) {
  uint2 r;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(addr));
  return r;
}
__device__ __forceinline__ void sts_v2(uint32_t addr, uint32_t x, uint32_t y) {
  asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(addr), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
  uint32_t r;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(r) : "r"(addr));
  return r;
}

// volatile: keeps the interval update ahead of the branch that follows it in program order
__device__ __forceinline__ uint32_t prmt(uint32_t x, uint32_t y, uint32_t sel) {
  uint32_t r;
  asm volatile("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(x), "r"(y), "r"(sel));
  return r;
}

struct Dec2 {
  uint32_t base, span, value;
  uint32_t pos2;       // stream position in BYTES (2 * word index)
  uint32_t next;       // word at that position
  uint32_t ring_addr;  // shared address of the word ring (4096-byte aligned)
  int lane;

  __device__ __forceinline__ void seek() { next = lds_u16(ring_addr | (pos2 & (2 * kRing - 2))); }
  // new interval [base + a, base + b1] and 16-bit renormalisation (range_coder.h:255-268); branch free:
  // all three 16-bit shifts are one byte permute with a shared selector
  __device__ __forceinline__ void update(uint32_t a, uint32_t b1) {
    const uint32_t nb = base + a;
    const uint32_t s = b1 - a;
    const bool renorm = s < 65536u;
    const uint32_t sel = renorm ? 0x1054u : 0x3210u;  // {x.b1, x.b0, y.b1, y.b0} : x
    span = prmt(s, 0xFFFFFFFFu, sel);
    base = prmt(nb, 0u, sel);
    value = prmt(value, next, sel);
    pos2 += renorm ? 2u : 0u;
    next = lds_u16(ring_addr | (pos2 & (2 * kRing - 2)));  // consumed at the next renormalisation, not before
  }
  // DecodeLinearly({0,1,2}, 1), range_coder_kernels.cc:450,461-469
  __device__ __forceinline__ uint32_t bit() {
    const uint32_t v = value - base;
    const uint32_t half = key_bound(span, make_uint2(0x80000000u, 0u)) ;  // floor(size / 2) ... see below
    // key_bound with addend_hi = 0 returns hi32(span*c' + c') = floor(size * 1 / 2) exactly (no "-1")
    const uint32_t b = (v < half) ? 0u : 1u;
    update(b ? half : 0u, b ? span : half - 1u);
    return b;
  }
  // Generic warp-parallel search over the whole row (pairs[start .. start + n]); returns the symbol.
  __device__ __forceinline__ int search_row(const uint2* pairs, int start, int n, uint32_t* a_out, uint32_t* b_out) {
    const uint32_t v = value - base;
    int lo_i = 0, hi_i = n;
    for (;;) {
      const int len = hi_i - lo_i;
      const bool final_round = len <= 63;
      const int stride = final_round ? 1 : ((len + 63) >> 6);
      int i0, i1;
      if (final_round) {
        i0 = lo_i + lane;
        i1 = lo_i + lane + 32;
      } else {
        i0 = lo_i + (lane + 1) * stride;
        i1 = lo_i + (lane + 33) * stride;
      }
      i0 = min(i0, hi_i);
      i1 = min(i1, hi_i);
      const uint2 q0 = pairs[start + i0], q1 = pairs[start + i1];
      const uint32_t B0 = key_bound(span, q0), B1 = key_bound(span, q1);
      const bool ge0 = (v <= B0) && q0.x != 0u, ge1 = (v <= B1) && q1.x != 0u;
      // distinct candidates below v (clamped duplicates sit at hi_i, which is never below)
      const int below = __popc(__ballot_sync(kFull, !ge0)) + __popc(__ballot_sync(kFull, !ge1));
      if (final_round) {
        const uint32_t m = ge0 ? B0 : (ge1 ? B1 : 0xFFFFFFFFu);
        const uint32_t am = ge1 ? (ge0 ? 0u : B0 + 1u) : B1 + 1u;
        *b_out = __reduce_min_sync(kFull, m);
        *a_out = __reduce_max_sync(kFull, am);
        int i = lo_i + below;  // smallest index whose bound is >= v
        i = max(1, min(i, n));
        return i - 1;
      }
      const int f = min(below, 63);
      const int nlo = (f == 0) ? lo_i : min(lo_i + f * stride, hi_i - 1);
      const int nhi = min(lo_i + (f + 1) * stride, hi_i);
      lo_i = nlo;
      hi_i = max(nhi, nlo + 1);
    }
  }
};

}  // namespace
}  // namespace tfcb
