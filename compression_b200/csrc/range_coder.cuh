// The range coder's serial recurrence and its helpers, shared by the coders built on it (range_coder.cu, and the
// mixture coder in mixture.cu): the encoder's chain and drain, the decoder's one-warp chain, the escape records and
// the host-side bounds.  Everything is in an anonymous namespace, so every translation unit has its own copy.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "common.cuh"
#include "range_decoder.cuh"

namespace tfcb {
namespace {

// ---------------------------------------------------------------------------------------------
// Encoder state and serial recurrence
// ---------------------------------------------------------------------------------------------
// Per stream the arena holds the UNRESOLVED 16-bit words (`words`) and one carry bit per word
// (`cbits`, bit w = "a carry left the 32-bit window while word w was its top half", i.e. +1 into
// word w-1; bit `cnt` is the pending carry of the not yet emitted top word).
struct EncState {
  uint32_t base;  // low end of the interval (32-bit window, wraps), renormalised
  uint32_t span;  // size - 1, renormalised (what RangeEncoder::Finalize looks at)
  uint32_t cnt;   // 16-bit words appended so far (a stream holds < 2^31 words = 4 GB)
  uint32_t raw;   // size - 1 BEFORE the renormalisation that followed the last symbol (what the chain resumes from)
};

__host__ __device__ inline EncState enc_initial_state() {
  EncState s;
  s.base = 0;
  s.span = 0xFFFFFFFFu;
  s.cnt = 0;
  s.raw = 0xFFFFFFFFu;
  return s;
}

// THE RECURRENCE.  The reference keeps (base, size - 1) and, after every Encode, multiplies both by 2^16 when
// size - 1 < 2^16 (range_coder.cc:69-84).  Only the interval SIZE feeds back into the next symbol, and the
// renormalisation is a select between two multiplies on that dependent chain.  Here the chain carries the
// UN-renormalised span `s` of the last symbol and never materialises the shifted one:
//
//   r    = s < 2^16                                 (the renormalisation the reference did after the last symbol)
//   Q(c) = s * ch + ch,   ch = c << (16 - p)        (64-bit: (s + 1) * c * 2^(16-p); c = 2^p fits: ch = 2^16)
//   floor(size * c / 2^p) = r ? Q : Q >> 16         (size = (s + 1) << 16r; exact; low 32 bits)
//   L = that for `lower`, U = that for `upper`;   s' = U - L - 1   (mod 2^32: a full-range symbol at size 2^32 wraps
//                                                                   to the right value)
// i.e. per symbol the dependent chain is  IADD3 -> IMAD.WIDE -> SHF (funnel by 0 or 16) -> IADD3, with the predicate
// of the shift amount evaluated beside the multiply -- no select between two multiplies.  {L, s'} per Encode is
// all the chain produces; the interval's low end, the carries, the emitted words and the word count are PREFIX
// computations over those entries and are done by the drain warp, 32 entries at a time (EncDrain).
// (Formula checked against the reference's on random triples: precisions 1..16, full-range, single-count and
// top-hugging symbols, from the initial state; the GPU tests compare whole streams with the compiled reference.)

// Pre-scaled operands of one Encode(lower, upper, p): {lower << (16-p), 0, upper << (16-p), 0}.  The zeros are
// the high halves of the two multiply-adds' 64-bit addends: one 128-bit shared-memory load puts each bound's
// addend in a register pair of its own.
__device__ __forceinline__ uint4 enc_operands(uint32_t lower, uint32_t upper, uint32_t p) {
  const uint32_t sh = 16u - p;
  return make_uint4(lower << sh, 0u, upper << sh, 0u);
}

struct EncChain {
  uint32_t s;  // un-renormalised span after the last symbol

  // One Encode(lower, upper, precision) of range_coder.cc:37-264 -> the entry {L, s'}.
  __device__ __forceinline__ uint2 step(uint2 ol, uint2 oh) {
    const unsigned long long ql = (unsigned long long)s * ol.x + (((unsigned long long)ol.y << 32) | ol.x);
    const unsigned long long qu = (unsigned long long)s * oh.x + (((unsigned long long)oh.y << 32) | oh.x);
    const uint32_t shift = (s < 65536u) ? 0u : 16u;
    const uint32_t L = __funnelshift_r((uint32_t)ql, (uint32_t)(ql >> 32), shift);
    const uint32_t U = __funnelshift_r((uint32_t)qu, (uint32_t)(qu >> 32), shift);
    // s' = U - L - 1 as ONE IADD3 (U, -L, -1).  Written in C the compiler turns it into U + ~L: a LOP3 and an add,
    // two dependent instructions on the chain instead of one.
    asm("{\n\t.reg .u32 t;\n\tsub.u32 t, %1, %2;\n\tsub.u32 %0, t, 1;\n\t}" : "=r"(s) : "r"(U), "r"(L));
    return make_uint2(L, s);
  }
  __device__ __forceinline__ uint2 step(uint4 o) { return step(make_uint2(o.x, o.y), make_uint2(o.z, o.w)); }
};

// x << s for s in [0, 32] (s == 32 gives 0): one funnel shift.
__device__ __forceinline__ uint32_t shl_clamp(uint32_t x, uint32_t s) { return __funnelshift_lc(0u, x, s); }

// Rebuilds everything the chain left out from its entries {L_k, s'_k}, 32 entries per pass, all lanes in parallel.
// Entry k renormalises iff s'_k < 2^16.  The low end obeys  base_{k+1} = (base_k + L_k) << sh_k  (sh_k = 16 or 0,
// mod 2^32), a composition of maps  x -> (x << S) + A  which is closed under composition
// ((x << S1) + A1) << S2) + A2 = (x << (S1 + S2)) + (A1 << S2) + A2,  so a warp-wide scan over (A, S) gives every
// lane the base its entry was added to; the carry out of the 32-bit window is then `base_k + L_k` overflowing, the
// emitted word is the top half of that sum, and the word index is a prefix popcount of the renormalisation flags.
struct EncDrain {
  uint32_t dbase;   // base before the first entry of the next pass
  uint32_t cnt;     // words emitted so far
  uint32_t cb_cur;  // carry bits of word group (cnt >> 5) accumulated so far
  uint16_t* words;
  uint32_t* cbits;
  uint32_t cap;  // capacity in words (multiple of 32)
  bool overflowed;
  int lane;

  __device__ __forceinline__ void begin(const EncState& st, uint16_t* w, uint32_t* cb, uint32_t cap_, int lane_) {
    dbase = st.base;
    cnt = st.cnt;
    words = w;
    cbits = cb;
    cap = cap_;
    overflowed = false;
    lane = lane_;
    cb_cur = (st.cnt == 0) ? 0u : cb[st.cnt >> 5];
  }

  // Entries [0, n) of `ent`, n <= kPasses * 32.  The scans of the passes do not depend on each other (only the
  // final application of `dbase` does), so they are issued together and their shuffle latencies overlap.
  template <int kPasses>
  __device__ __forceinline__ void drain(const uint2* ent, int n) {
    uint32_t Lk[kPasses], Ak[kPasses], Sk[kPasses], rmask[kPasses];
#pragma unroll
    for (int p = 0; p < kPasses; ++p) {
      const int k = p * 32 + lane;
      const bool act = k < n;
      const uint2 me = ent[act ? k : 0];
      const bool rr = act && me.y < 65536u;
      rmask[p] = __ballot_sync(kFull, rr);
      Lk[p] = act ? me.x : 0u;
      uint32_t S = rr ? 16u : 0u;
      uint32_t A = Lk[p] << S;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {  // inclusive scan of the maps: lane l ends with f_l o ... o f_0
        const uint32_t Ap = __shfl_up_sync(kFull, A, d);
        const uint32_t Sp = __shfl_up_sync(kFull, S, d);
        if (lane >= d) {
          A = shl_clamp(Ap, S) + A;
          S = min(Sp + S, 32u);
        }
      }
      Ak[p] = A;
      Sk[p] = S;
    }
#pragma unroll
    for (int p = 0; p < kPasses; ++p) {
      if (p * 32 >= n) break;
      // exclusive prefix = the map of the entries before this lane's
      uint32_t Ax = __shfl_up_sync(kFull, Ak[p], 1);
      uint32_t Sx = __shfl_up_sync(kFull, Sk[p], 1);
      if (lane == 0) {
        Ax = 0u;
        Sx = 0u;
      }
      const uint32_t before = shl_clamp(dbase, Sx) + Ax;  // base this entry's L was added to
      const uint32_t nb = before + Lk[p];
      const bool carry = nb < before;                     // (inactive lanes: L = 0, never)
      const bool ren = (rmask[p] >> lane) & 1u;
      const uint32_t my_cnt = cnt + __popc(rmask[p] & ((1u << lane) - 1u));  // word count before this entry
      if (ren) {
        if (my_cnt < cap) words[my_cnt] = (uint16_t)(nb >> 16);
        else overflowed = true;
      }
      const uint32_t g0 = cnt >> 5;
      const uint32_t bit = 1u << (my_cnt & 31u);
      const uint32_t m0 = __reduce_or_sync(kFull, (carry && (my_cnt >> 5) == g0) ? bit : 0u);
      const uint32_t m1 = __reduce_or_sync(kFull, (carry && (my_cnt >> 5) != g0) ? bit : 0u);
      const uint32_t pass_end = cnt + __popc(rmask[p]);
      cb_cur |= m0;
      if ((pass_end >> 5) != g0) {
        if (lane == 0 && g0 < (cap >> 5)) cbits[g0] = cb_cur;
        cb_cur = m1;
      }
      cnt = pass_end;
      // base after the last entry of this pass
      dbase = shl_clamp(dbase, __shfl_sync(kFull, Sk[p], 31)) + __shfl_sync(kFull, Ak[p], 31);
    }
  }

  __device__ __forceinline__ void end(DevError* err, long long stream) {
    if ((cnt >> 5) < (cap >> 5)) {
      if (lane == 0) cbits[cnt >> 5] = cb_cur;
    } else {
      overflowed = true;
    }
    if (__any_sync(kFull, overflowed)) report(err, kErrCapacity, stream, cnt, cnt, cap);
  }
};

// Where one stream's symbols (or arena words) are: resolved once per CTA from the offsets array when there is one,
// else from the uniform stride.
struct Extent {
  long long base, len;
};
__device__ __forceinline__ Extent stream_extent(const long long* off, long long s, long long stride) {
  if (off) return Extent{off[s], off[s + 1] - off[s]};
  return Extent{s * stride, stride};
}

// Record i of the escape tail of OverflowEncode (range_coder_kernels.cc:306-321): nb - 1 zero bits, the nb bits
// of g (MSB first), then the sign, each coded with the uniform binary CDF {0, 1, 2} at precision 1.
__device__ __forceinline__ uint4 gamma_record(uint32_t g, uint32_t sign, int nb, int i) {
  uint32_t bit;
  if (i < nb - 1) bit = 0u;
  else if (i < 2 * nb - 1) bit = (g >> (2 * nb - 2 - i)) & 1u;
  else bit = sign;
  return enc_operands(bit, bit + 1u, 1u);
}

__device__ __forceinline__ void bw_seek(ByteWindow& w, uint32_t pos, int lane) {
  w.lane_word = bw_fetch(w, (long long)(pos & ~31u) + lane);
  w.next = __shfl_sync(kFull, w.lane_word, pos & 31u);
}

struct DecChain {
  uint32_t base, span, value, pos;
};

__device__ __forceinline__ void dec_update(DecChain& c, ByteWindow& w, uint32_t a, uint32_t b, int lane) {
  c.base += a;
  c.span = b - a - 1u;
  if (c.span < 65536u) {
    c.base <<= 16;
    c.span = (c.span << 16) | 0xFFFFu;
    c.value = (c.value << 16) | w.next;
    c.pos += 1;
    if ((c.pos & 31u) == 0) {
      bw_seek(w, c.pos, lane);
    } else {
      w.next = __shfl_sync(kFull, w.lane_word, c.pos & 31u);
    }
  }
}

// Smallest i in [1, ncdf-1] with scale(cdf[i]) > value - base; identical to the reference's binary
// search (range_coder.h:204-222,241-251) for every monotone CDF.  Clamped for corrupt streams.
__device__ __forceinline__ int dec_symbol(DecChain& c, ByteWindow& w, const int32_t* cdf, int ncdf,
                                          uint32_t p, int lane) {
  const uint32_t v = c.value - c.base;
  int lo_i = 1;
  int n = ncdf - 1;
  int i;
  for (;;) {
    const int stride = (n + 31) >> 5;
    int off = (lane + 1) * stride - 1;
    if (off > n - 1) off = n - 1;
    const uint32_t cv = (uint32_t)cdf[lo_i + off];
    const bool pred = v < scale_cum(c.span, cv, p);
    // scale_cum truncates 2^32 to 0; that only happens for cv == 2^p with span == 2^32-1, where the
    // true value 2^32 exceeds every v.
    const bool full = (cv == (1u << p)) && (c.span == 0xFFFFFFFFu);
    const unsigned m = __ballot_sync(kFull, pred || full);
    const int f = m ? (__ffs(m) - 1) : 31;
    if (stride == 1) {
      i = lo_i + min(f, n - 1);
      break;
    }
    const int skip = min(f * stride, n - 1);
    lo_i += skip;
    n = min(stride, n - skip);
  }
  const uint32_t ca = (uint32_t)cdf[i - 1];
  const uint32_t cb = (uint32_t)cdf[i];
  dec_update(c, w, scale_cum(c.span, ca, p), scale_cum(c.span, cb, p), lane);
  return i - 1;
}

__device__ __forceinline__ void ubi_key(long long* field, unsigned long long key) {
  atomicMin(reinterpret_cast<unsigned long long*>(field), key);
}

// RangeDecoder::Decode over the uniform table 0, 1, ..., 2^w at precision w, computed instead of searched: the
// smallest i in [1, 2^w] with (value - base + 1) * 2^w <= size * i, which is what the reference's binary search finds.
__device__ __forceinline__ uint32_t ubi_dec_uniform(DecChain& c, ByteWindow& win, uint32_t w, int lane) {
  const unsigned long long size = (unsigned long long)c.span + 1ull;
  const unsigned long long want = ((unsigned long long)(c.value - c.base) + 1ull) << w;
  unsigned long long i = (want + size - 1ull) / size;
  if (i > (1ull << w)) i = 1ull << w;  // only on damaged strings; the reference reads past its table there
  const uint32_t sym = (uint32_t)i;
  dec_update(c, win, scale_cum(c.span, sym - 1u, w), scale_cum(c.span, sym, w), lane);
  return sym - 1u;
}

// Worst-case 16-bit words one call can append per stream: every Encode(.., p) shrinks the interval by
// at most 2^p, i.e. consumes at most p bits; an escape adds at most 65 one-bit symbols.
long long bits_bound(int max_prec, bool any_overflow) { return max_prec + (any_overflow ? 65 : 0); }
long long words_for(long long bits, long long n) { return (n * bits + 15) / 16 + 2; }
constexpr long long kMaxStreamWords = (1ll << 31) - 64;  // a stream's word count and positions fit 32 bits

int check_symbol_offsets(const int64_t* off, long long n_streams) {
  if (n_streams <= 0) return fail(TFCB_INVALID_ARGUMENT, "`n_streams` must be positive: %lld", n_streams);
  if (!off) return fail(TFCB_INVALID_ARGUMENT, "`symbol_offsets` is null");
  if (off[0] != 0) return fail(TFCB_INVALID_ARGUMENT, "symbol_offsets[0] must be 0: %lld", (long long)off[0]);
  for (long long i = 0; i < n_streams; ++i)
    if (off[i + 1] < off[i])
      return fail(TFCB_INVALID_ARGUMENT,
                  "symbol_offsets must be non-decreasing: symbol_offsets[%lld]=%lld > symbol_offsets[%lld]=%lld", i,
                  (long long)off[i], i + 1, (long long)off[i + 1]);
  return TFCB_OK;
}

}  // namespace

// Finalize of a ragged arena (per-stream word ranges `arena_off`) written by a chain in another translation unit:
// enc_offsets_kernel's lengths and offsets with the one host synchronisation, the raw error record in `err_out`, and
// enc_write_kernel into `out`.  `state` points at the streams' EncState.
int ragged_arena_offsets(long long n_streams, void* state, uint16_t* words, uint32_t* cbits, DevError* err,
                         const long long* arena_off, long long* offsets, cudaStream_t s, long long* total,
                         DevError* err_out);
void ragged_arena_write(long long n_streams, void* state, uint16_t* words, uint32_t* cbits, DevError* err,
                        const long long* arena_off, const long long* offsets, uint8_t* out, cudaStream_t s);

}  // namespace tfcb
