// Range coder for sm_90a: one CTA per code stream, the serial recurrence alone on one warp.
//
// Replaces (paths relative to /root/reference/tensorflow_compression):
//   cc/lib/range_coder.cc:37-307, cc/lib/range_coder.h:79-282          the coder
//   cc/kernels/range_coder_kernels.cc:110-164,168-322,334-471           multi-stream ops
//   cc/kernels/range_coding_kernels.cc:60-379 (+ _util.cc:34-91)        legacy single-stream ops
//
// ENCODER.  The reference emits bytes through a delayed-carry state machine.  Its output is exactly the
// big-number sum  SUM_k a_k * 2^-(16 r_k + 32)  of the per-symbol interval offsets a_k (r_k = number of 16-bit
// renormalisations before symbol k) followed by a short flush; only the recurrence on the interval size is
// inherently serial.  Per stream (encode_kernel, six warps):
//   * gather warps: coalesced symbol loads three passes ahead, fused quantisation, range checks, escape expansion
//     (an escaping symbol is followed by the records of its Elias-gamma bits), table gathers, operand pre-scaling;
//   * chain warp: nothing but the recurrence on the UN-renormalised span (EncChain::step: IADD3 -> IMAD.WIDE ->
//     funnel shift -> IADD3, no select between the multiplies), one entry {L, s'} per Encode;
//   * drain warp: base, carries, emitted 16-bit words and word count are prefix computations over those entries
//     (EncDrain: a warp scan over the maps x -> (x << S) + A), written as unresolved words + one carry bit each;
//   * finalize: warp-wide carry-lookahead over 32-word groups, RangeEncoder::Finalize's tail rule, compaction.
// DECODER.  Same recurrence plus a CDF search per symbol (decode_kernel, three warps: prepare / chain / resolve):
// pre-scaled search keys, a 64-key window per row around its median evaluated two keys per lane with one IMAD.HI
// each and two warp reductions; the symbol index itself is recovered off the chain by the resolve warp.
// The one-warp-per-stream helpers further down (ByteWindow, dec_symbol) serve the legacy single-stream ops only.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <type_traits>
#include <vector>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "range_coder.cuh"
#include "range_decoder.cuh"

namespace tfcb {
namespace {

// ---------------------------------------------------------------------------------------------
// Lookup tables
// ---------------------------------------------------------------------------------------------
struct HostRow {
  int32_t start;  // index of cdf[0] inside the lookup buffer
  int32_t ncdf;   // number of cdf entries (bins + 1)
  int32_t prec;   // signed precision entry
};

// Grammar of range_coder_kernels.cc:110-137 (one row) and :139-164 (1-D / 2-D containers).
int scan_row(const int32_t* base, const int32_t* end, const int32_t** cur, std::vector<HostRow>* rows) {
  const int32_t* p = *cur;
  if (end - p < 3) return fail(TFCB_INVALID_ARGUMENT, "CDF ended prematurely.");
  const int64_t ap = p[0] < 0 ? -(int64_t)p[0] : (int64_t)p[0];
  if (ap < 1 || ap >= 17)
    return fail(TFCB_INVALID_ARGUMENT, "precision=%lld not in range [1, 17)", (long long)ap);
  const int32_t last = 1 << ap;
  const int32_t* first = p;
  if (p[1] != 0) return fail(TFCB_INVALID_ARGUMENT, "CDF must start with 0.");
  p += 1;
  for (;;) {
    ++p;
    if (p == end) return fail(TFCB_INVALID_ARGUMENT, "CDF must end with 1 << precision.");
    if (p[0] < p[-1]) return fail(TFCB_INVALID_ARGUMENT, "CDF must be monotonically increasing.");
    if (*p == last) break;
  }
  ++p;
  rows->push_back(HostRow{(int32_t)(first + 1 - base), (int32_t)(p - first - 1), first[0]});
  while (p != end && *p == last) ++p;
  *cur = p;
  return TFCB_OK;
}

int parse_lookup(const int32_t* lookup, int64_t len, int64_t cols, std::vector<HostRow>* rows) {
  rows->clear();
  if (len < 0 || (len > 0 && lookup == nullptr))
    return fail(TFCB_INVALID_ARGUMENT, "`lookup` is null");
  if (len >= (1ll << 31)) return fail(TFCB_INVALID_ARGUMENT, "`lookup` too large");
  if (cols < 0 || (cols > 0 && len % cols != 0))
    return fail(TFCB_INVALID_ARGUMENT, "`lookup` must be rank 1 or 2");
  const int32_t* end = lookup + len;
  for (const int32_t* cur = lookup; cur != end;) {
    const int32_t* row_end = cols > 0 ? cur + cols : end;
    TFCB_TRY(scan_row(lookup, row_end, &cur, rows));
    if (cols > 0 && cur != row_end)
      return fail(TFCB_INVALID_ARGUMENT, "CDF must end with 1 << precision.");
  }
  return TFCB_OK;
}

struct DeviceLookup {
  int32_t* lookup = nullptr;  // device copy of the raw table
  int2* rows = nullptr;       // {start, meta}
  uint2* pairs = nullptr;     // decoder: per cdf entry {c', addend_hi} so that hi32(span*c' + {c',addend_hi}) = T(c) - 1
  int4* rows4 = nullptr;      // decoder: {key segment start, meta, first window index, irregular}
  long long n_pairs = 0;
  int zero_win = 0;  // key index of the all-zero window (decoder tables only)
  int n_rows = 0;
  long long len = 0;
  bool any_overflow = false;
  int max_prec = 0;
  int uniform_prec = 0;  // > 0 when every row shares one precision

  int upload(const int32_t* lookup_host, int64_t len_, int64_t cols, cudaStream_t s, bool for_decoder = false) {
    const int64_t len = len_;
    std::vector<HostRow> hr;
    TFCB_TRY(parse_lookup(lookup_host, len, cols, &hr));
    n_rows = (int)hr.size();
    this->len = len_;
    std::vector<int2> meta(std::max<size_t>(hr.size(), 1));
    for (size_t i = 0; i < hr.size(); ++i) {
      const int ap = hr[i].prec < 0 ? -hr[i].prec : hr[i].prec;
      any_overflow |= hr[i].prec < 0;
      max_prec = std::max(max_prec, ap);
      uniform_prec = (i == 0 || uniform_prec == ap) ? ap : -1;
      meta[i].x = hr[i].start;
      meta[i].y = hr[i].ncdf | (ap << 24) | (hr[i].prec < 0 ? (int)0x80000000 : 0);
    }
    if (uniform_prec < 0) uniform_prec = 0;
    TFCB_TRY(dev_alloc((void**)&lookup, std::max<int64_t>(len, 1) * sizeof(int32_t), s));
    TFCB_TRY(dev_alloc((void**)&rows, meta.size() * sizeof(int2), s));
    if (len > 0)
      TFCB_CUDA_TRY(cudaMemcpyAsync(lookup, lookup_host, len * sizeof(int32_t),
                                    cudaMemcpyHostToDevice, s));
    TFCB_CUDA_TRY(cudaMemcpyAsync(rows, meta.data(), meta.size() * sizeof(int2),
                                  cudaMemcpyHostToDevice, s));
    std::vector<uint2> hp;
    std::vector<int4> hr4;
    if (for_decoder) {
      // Pre-scaled search keys: B'(c) = floor(size*c/2^p) - 1 = hi32(span*c' + {c', 0xFFFFFFFF}) with
      // c' = c << (32-p); c == 2^p -> {0xFFFFFFFF, 0} (B' = span = size - 1).  Every row gets its own padded
      // segment: keys of cdf[0..n], then "full" keys up to index 64, so that the 64-key search window
      // [wfirst, wfirst + 63] (centred on the row's median, wfirst >= 1) never needs clamping.
      // Rows with zero-width bins at either end are marked irregular: slow path only.
      hr4.resize(meta.size());
      for (size_t i = 0; i < hr.size(); ++i) {
        const int ap = hr[i].prec < 0 ? -hr[i].prec : hr[i].prec;
        const int n = hr[i].ncdf - 1;
        const int pstart = (int)hp.size();
        int median = n, irregular = 0;
        for (int e = 0; e <= n; ++e) {
          const uint32_t c = (uint32_t)lookup_host[hr[i].start + e];
          hp.push_back((c == (1u << ap)) ? make_uint2(0xFFFFFFFFu, 0u) : make_uint2(c << (32 - ap), 0xFFFFFFFFu));
          if (e >= 1 && c == 0u) irregular = 1;
          if (e >= 1 && e < n && c == (1u << ap)) irregular = 1;  // trailing zero-width bins
          if (e >= 1 && median == n && c >= (1u << ap) / 2) median = e;
        }
        for (int e = n + 1; e <= 64; ++e) hp.push_back(make_uint2(0xFFFFFFFFu, 0u));
        int wfirst = median - 31;
        if (wfirst > n - 63) wfirst = n - 63;
        if (wfirst < 1) wfirst = 1;
        hr4[i] = make_int4(pstart, meta[i].y, wfirst, irregular);
      }
      // window of keys whose bound is 0: used for irregular rows so that the chain always takes the slow path
      zero_win = (int)hp.size();
      for (int e = 0; e < 64; ++e) hp.push_back(make_uint2(0u, 0u));
      n_pairs = (long long)hp.size();
      TFCB_TRY(dev_alloc((void**)&pairs, hp.size() * sizeof(uint2), s));
      TFCB_TRY(dev_alloc((void**)&rows4, hr4.size() * sizeof(int4), s));
      TFCB_CUDA_TRY(cudaMemcpyAsync(pairs, hp.data(), hp.size() * sizeof(uint2), cudaMemcpyHostToDevice, s));
      TFCB_CUDA_TRY(cudaMemcpyAsync(rows4, hr4.data(), hr4.size() * sizeof(int4), cudaMemcpyHostToDevice, s));
    }
    // the host vectors die at return: make sure the copies have been staged
    TFCB_CUDA_TRY(cudaStreamSynchronize(s));
    return TFCB_OK;
  }
  void release(cudaStream_t s) {
    dev_free(lookup, s);
    dev_free(rows, s);
    dev_free(pairs, s);
    dev_free(rows4, s);
    lookup = nullptr;
    rows = nullptr;
    pairs = nullptr;
    rows4 = nullptr;
  }
};

// kModeDecoded (encoder only, with kModeF32 or a 16-bit mode): the gather warp also writes every symbol's decoded
// value.  kModeH16 / kModeB16: the value is float16 / bfloat16, quantised and dequantised with the arithmetic of the
// entropy models' unfused 16-bit path (enc_gather, dequantise16).  kModeLocF32 (index mode with a 16-bit value): the
// loc is float32, and so is the decoded value (torch's type promotion); without it the loc is in the value's type.
enum : int { kModeIndex = 1, kModeF32 = 2, kModeDecoded = 4, kModeH16 = 8, kModeB16 = 16, kModeLocF32 = 32 };
constexpr int kMode16 = kModeH16 | kModeB16;
constexpr int kModeFloat = kModeF32 | kMode16;  // float values: quantised in the kernel, cdf_offset is read

struct EncParams {
  const int32_t* lookup;
  const int2* rows;
  int n_rows;
  int uniform_prec;        // > 0: every row has this precision
  const void* value;       // int32 or float [S, n]
  const int32_t* index;    // [S, n] or null
  const float* qoff;       // channel+f32: [n_rows] or null; index+f32: loc [S, n] or null
  const int32_t* coff;     // f32 modes: cdf_offset [n_rows]
  long long n;
  long long n_streams;
  int fresh;  // first encode of the handle: start from the initial state instead of reading `state`
  EncState* state;
  uint16_t* words;
  uint32_t* cbits;
  long long cap;  // words per stream
  DevError* err;
  // Ragged batches: stream s is symbols [sym_off[s], sym_off[s+1]) and arena words [arena_off[s], arena_off[s+1])
  // (multiples of 32).  Null: stream s is symbols [s * n, s * n + n) and words [s * cap, s * cap + cap).
  const long long* sym_off;
  const long long* arena_off;
  // kModeDecoded: float [n symbols in all], what the f32 decoder returns for each symbol (last: the other fields keep
  // their parameter offsets); in 16-bit modes only under kModeLocF32
  float* decoded;
  // 16-bit modes (after `decoded`, for the same reason): loc [S, n] in the value's type (index mode without
  // kModeLocF32; may be null), and kModeDecoded's output in the value's type (without kModeLocF32)
  const uint16_t* loc16;
  uint16_t* decoded16;
};

// 16-bit values as float32 (exact) and float32 rounded to the nearest 16-bit value (ties to even; overflow to inf,
// NaN stays NaN): the conversions torch's elementwise kernels make on the device.
template <int MODE>
__device__ __forceinline__ float widen16(uint32_t bits) {
  if (MODE & kModeH16) return __half2float(__ushort_as_half((unsigned short)bits));
  return __bfloat162float(__ushort_as_bfloat16((unsigned short)bits));
}
template <int MODE>
__device__ __forceinline__ uint16_t narrow16(float x) {
  if (MODE & kModeH16) return __half_as_ushort(__float2half_rn(x));
  return __bfloat16_as_ushort(__float2bfloat16_rn(x));
}

// The 16-bit dequantisation of entropy_models._dequantize: the int32 sum `sc` = symbol + cdf_offset cast to the
// value's type as torch casts int32 (to float, then to 16 bits: two roundings), then plus the offset `off` (widened
// to float32) in float32.  The caller rounds the result once to the value's type, or stores it as float32 under
// kModeLocF32, where torch promotes the sum with a float32 loc.
template <int MODE>
__device__ __forceinline__ float dequantise16(int sc, bool has_off, float off) {
  const float h = widen16<MODE>(narrow16<MODE>((float)sc));
  return has_off ? h + off : h;
}

// The gather of one pass of 32 symbols is split in two stages so that no global-memory latency is
// ever exposed to the (in-order) warp:
//   stage A, three passes ahead : the symbol itself (y / value, index, loc) and, in channel mode, the row
//                                 descriptor and the per-row offsets -- all independent loads;
//   stage B, current pass       : quantise, range-check, escape mapping, then the two table loads and the
//                                 operand records written to shared memory for the serial chain.
struct Fetched {
  float y;
  int v;
  float loc_or_q;
  int coff;
  int row;
  int2 ri;
  bool valid;
  // 16-bit modes: the value's (and a 16-bit loc's) bits as loaded, widened in stage B -- a conversion in stage A
  // would wait for the load there
  uint32_t y16, loc16;
};

struct Gathered {
  uint4 ops;       // pre-scaled operands (enc_operands)
  uint32_t prec;   // 0 = invalid / out of range
  uint32_t gamma;  // escape payload (0 = none)
  uint32_t sign;
};

// `at`: absolute symbol position; the stream's symbols end at `end`.
template <int MODE>
__device__ __forceinline__ Fetched enc_fetch(const EncParams& P, long long end, long long at, uint32_t chan_row) {
  Fetched f;
  f.y = 0.f;
  f.v = 0;
  f.loc_or_q = 0.f;
  f.coff = 0;
  f.row = (int)chan_row;
  f.ri = make_int2(0, 0);
  if (MODE & kMode16) {
    f.y16 = 0;
    f.loc16 = 0;
  }
  f.valid = at < end;
  if (!f.valid) return f;
  if (MODE & kModeF32) {
    f.y = __ldg(reinterpret_cast<const float*>(P.value) + at);
  } else if (MODE & kMode16) {
    f.y16 = __ldg(reinterpret_cast<const unsigned short*>(P.value) + at);
  } else {
    f.v = __ldg(reinterpret_cast<const int32_t*>(P.value) + at);
  }
  if (MODE & kModeIndex) {
    f.row = __ldg(P.index + at);
    if ((MODE & kMode16) && !(MODE & kModeLocF32)) {
      if (P.loc16) f.loc16 = __ldg(P.loc16 + at);
    } else if ((MODE & kModeFloat) && P.qoff) {
      f.loc_or_q = __ldg(P.qoff + at);
    }
  } else {
    f.ri = __ldg(P.rows + f.row);
    if (MODE & kModeFloat) {
      if (P.qoff) f.loc_or_q = __ldg(P.qoff + f.row);
      f.coff = __ldg(P.coff + f.row);
    }
  }
  return f;
}

// `at`: absolute symbol position.  Errors name the stream and the position inside it (the stream's start is looked
// up again there rather than kept live beside the gather loop).
template <int MODE>
__device__ __forceinline__ Gathered enc_gather(const EncParams& P, long long s, long long at, Fetched f) {
  Gathered g;
  g.ops = make_uint4(0u, 0u, 0u, 0u);
  g.prec = 0;
  g.gamma = 0;
  g.sign = 0;
  if (!f.valid) return g;
  if (MODE & kModeIndex) {
    if (f.row < 0 || f.row >= P.n_rows) {
      report(P.err, kErrIndex, s, at - stream_extent(P.sym_off, s, P.n).base, f.row, P.n_rows);
      return g;
    }
    f.ri = __ldg(P.rows + f.row);
    if (MODE & kModeFloat) f.coff = __ldg(P.coff + f.row);
  }
  if (MODE & kMode16) {
    f.y = widen16<MODE>(f.y16);
    if ((MODE & kModeIndex) && !(MODE & kModeLocF32)) f.loc_or_q = widen16<MODE>(f.loc16);  // (+0 without a loc)
  }
  int v = f.v;
  if (MODE & kModeFloat) {
    // 16-bit values: channel mode quantises the value widened to float32 against the float32 quantisation offset,
    // as does index mode with a float32 loc (torch promotes the difference to float32); with a loc in the value's
    // type (or none) index mode rounds the difference to that type first, as the unfused path's 16-bit subtraction
    float d = f.y - f.loc_or_q;
    if ((MODE & kMode16) && (MODE & kModeIndex) && !(MODE & kModeLocF32)) d = widen16<MODE>(narrow16<MODE>(d));
    v = (int)rintf(d) - f.coff;
  }
  if (MODE & kModeDecoded) {
    // the resolve warp's dequantisation of the symbol it decodes (v, before the escape mapping): the same integer
    // and the same float operations, so the value is bit-identical to the decoder's -- including the saturated
    // conversion of |y - loc| >= 2^31 and NaN -> 0, which recomputing rintf(y - loc) + loc would not reproduce
    if (MODE & kMode16) {
      const bool loc16 = (MODE & kModeIndex) && !(MODE & kModeLocF32);
      const bool has_off = loc16 ? P.loc16 != nullptr : P.qoff != nullptr;
      // channel mode adds the quantisation offset rounded to the value's type (_dequantize's off.to(out.dtype))
      const float off = (MODE & kModeIndex) ? f.loc_or_q : widen16<MODE>(narrow16<MODE>(f.loc_or_q));
      const float r = dequantise16<MODE>(v + f.coff, has_off, off);
      if (MODE & kModeLocF32) P.decoded[at] = r;
      else P.decoded16[at] = narrow16<MODE>(r);
    } else {
      float yv = (float)(v + f.coff);
      if (P.qoff) yv += f.loc_or_q;
      P.decoded[at] = yv;
    }
  }
  const int ncdf = row_ncdf(f.ri.y);
  if (!row_ovf(f.ri.y)) {
    if (v < 0 || v >= ncdf - 1) {
      report(P.err, kErrValue, s, at - stream_extent(P.sym_off, s, P.n).base, v, ncdf - 1);
      return g;
    }
  } else {
    const int esc = ncdf - 2;
    if (v < 0) {
      g.gamma = (uint32_t)(-(long long)v);
      g.sign = 1;
      v = esc;
    } else if (v >= esc) {
      g.gamma = (uint32_t)(v - esc + 1);
      v = esc;
    }
  }
  const uint32_t lower = (uint32_t)__ldg(P.lookup + f.ri.x + v);
  const uint32_t upper = (uint32_t)__ldg(P.lookup + f.ri.x + v + 1);
  g.prec = (uint32_t)row_prec(f.ri.y);
  g.ops = enc_operands(lower, upper, g.prec);
  return g;
}

// Named barriers (bar.sync / bar.arrive) for the warp-to-warp hand-offs.
__device__ __forceinline__ void bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Shared state of one code stream's CTA.  The unit of every hand-off is a BLOCK of up to kBlock operand records
// (gather -> chain) and the same number of entries (chain -> drain), double buffered; one barrier round trip per
// block and direction.  The gather warp writes the record stream the chain consumes blindly: an escaping symbol
// is followed by the records of its Elias-gamma bits (OverflowEncode, range_coder_kernels.cc:306-321), so the
// chain warp has no special cases at all.
constexpr int kBlock = 256;

struct BlockInfo {
  uint32_t n;     // records / entries in this block (kBlock except for the last one)
  uint32_t last;  // nonzero: no further block follows
};

// Records the chain warp loads ahead of the one it codes: enough to cover the shared-memory load latency while the
// gather and drain warps keep the SM's shared-memory pipe busy.
constexpr int kPrefetch = 4;
static_assert(kPrefetch == 2 || kPrefetch == 4 || kPrefetch == 8, "the chain loop unrolls by 8 records");

struct EncShared {
  uint4 ops[2][kBlock + kPrefetch];  // (the chain's operand prefetch may run kPrefetch records past the block)
  uint2 ent[2][kBlock];
  BlockInfo ops_info[2];
  BlockInfo ent_info[2];
};

enum : int { kBarOpsFull = 1, kBarOpsEmpty = 3, kBarEntFull = 5, kBarEntEmpty = 7 };

// Gather-warp helper: appends records to the block stream, handing full blocks to the chain warp.
struct RecordWriter {
  EncShared* sh;
  long long blocks;  // blocks published so far
  int fill;          // records in the current block

  __device__ __forceinline__ void begin(EncShared* sh_) {
    sh = sh_;
    blocks = 0;
    fill = 0;
  }
  __device__ __forceinline__ uint4* cur() { return sh->ops[blocks & 1]; }
  __device__ __forceinline__ void publish(bool last) {
    const int b = (int)(blocks & 1);
    if ((threadIdx.x & 31) == 0) {
      BlockInfo bi;
      bi.n = (uint32_t)fill;
      bi.last = last ? 1u : 0u;
      sh->ops_info[b] = bi;
    }
    bar_arrive(kBarOpsFull + b, 64);  // arrive orders the preceding shared-memory writes
    ++blocks;
    fill = 0;
    if (!last && blocks >= 2) bar_sync(kBarOpsEmpty + (int)(blocks & 1), 64);  // the chain is done with that buffer
  }
  // Appends this pass's records: lane's own record `first` at pass-local position `pre`, followed by `extra` more
  // produced by `rec(i)`; `total` = all lanes' records.  Blocks are filled exactly; a pass may straddle blocks.
  template <typename F>
  __device__ __forceinline__ void append(uint4 first, int pre, int extra, int total, bool has, F rec) {
    int done = 0;
    while (done < total) {
      const int room = kBlock - fill;
      const int take = min(room, total - done);
      uint4* dst = cur() + fill - done;  // record with pass-local position i goes to dst[i]
      if (has) {
        if (pre >= done && pre < done + take) dst[pre] = first;
        for (int i = 0; i < extra; ++i) {
          const int at = pre + 1 + i;
          if (at >= done && at < done + take) dst[at] = rec(i);
        }
      }
      fill += take;
      done += take;
      if (fill == kBlock) publish(false);
    }
  }
};


template <int MODE>
__global__ void __launch_bounds__(192) encode_kernel(const EncParams P) {
  __shared__ __align__(16) EncShared sh;
  const long long s = blockIdx.x;
  const int lane = threadIdx.x & 31;
  // Warp 0 chain, 1 gather, 5 drain; 2..4 exit at once.  Only the per-stream latency of the chain warp matters
  // (there are more schedulers than streams), so the layout keeps a chain warp alone on its sub-partition (warp slot
  // mod 4) when two CTAs share an SM: the first takes slots 0..5 (chain on sub-partition 0, gather + drain on 1), the
  // second slots 6..11 (chain on 2, gather + drain on 3).
  const int warp = threadIdx.x >> 5;
  if (warp != 0 && warp != 1 && warp != 5) return;

  if (warp == 1) {
    // ------------------------------- gather warp -------------------------------
    uint32_t row_a = 0, chan_step = 0;
    if (!(MODE & kModeIndex)) {
      row_a = (uint32_t)lane % (uint32_t)P.n_rows;
      chan_step = 32u % (uint32_t)P.n_rows;
    }
    auto advance_row = [&]() {
      if (!(MODE & kModeIndex)) {
        row_a += chan_step;
        if (row_a >= (uint32_t)P.n_rows) row_a -= (uint32_t)P.n_rows;
      }
    };
    // absolute symbol positions: only the stream's end stays live beside the loop
    const Extent x = stream_extent(P.sym_off, s, P.n);
    const long long end = x.base + x.len;
    // stage A (symbol loads) runs three 32-symbol passes ahead of stage B: no global latency is waited for
    Fetched f0 = enc_fetch<MODE>(P, end, x.base + lane, row_a);
    advance_row();
    Fetched f1 = enc_fetch<MODE>(P, end, x.base + 32 + lane, row_a);
    advance_row();
    Fetched f2 = enc_fetch<MODE>(P, end, x.base + 64 + lane, row_a);
    advance_row();
    RecordWriter w;
    w.begin(&sh);
    bool stop = false;
    for (long long j0 = x.base; j0 < end && !stop; j0 += 32) {
      const Fetched fcur = f0;
      f0 = f1;
      f1 = f2;
      f2 = enc_fetch<MODE>(P, end, j0 + 96 + lane, row_a);
      advance_row();
      const Gathered cur = enc_gather<MODE>(P, s, j0 + lane, fcur);
      const int count = (int)min(32ll, end - j0);
      const bool has = lane < count;
      const unsigned esc_mask = __ballot_sync(kFull, cur.gamma != 0);
      const unsigned bad_mask = __ballot_sync(kFull, cur.prec == 0 && has);
      if (bad_mask) {  // argument error already recorded: code nothing more of this stream
        stop = true;
        break;
      }
      if (esc_mask == 0) {
        if (w.fill + count <= kBlock) {  // the common case: one store per lane
          if (has) w.cur()[w.fill + lane] = cur.ops;
          w.fill += count;
          if (w.fill == kBlock) w.publish(false);
        } else {
          w.append(cur.ops, lane, 0, count, has, [&](int) { return cur.ops; });
        }
      } else {
        const int nb = cur.gamma ? 32 - __clz(cur.gamma) : 0;
        const int mine = has ? 1 + 2 * nb : 0;
        int incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          const int t = __shfl_up_sync(kFull, incl, d);
          if (lane >= d) incl += t;
        }
        const int total = __shfl_sync(kFull, incl, 31);
        w.append(cur.ops, incl - mine, 2 * nb, total, has,
                 [&](int i) { return gamma_record(cur.gamma, cur.sign, nb, i); });
      }
    }
    w.publish(true);  // (possibly empty) final block: lets the other two warps finish
    return;
  }

  if (warp == 5) {
    // ------------------------------- drain warp -------------------------------
    EncDrain d;
    const Extent a = stream_extent(P.arena_off, s, P.cap);
    d.begin(P.fresh ? enc_initial_state() : P.state[s], P.words + a.base, P.cbits + (a.base >> 5), (uint32_t)a.len,
            lane);
    for (long long k = 0;; ++k) {
      const int b = (int)(k & 1);
      bar_sync(kBarEntFull + b, 64);
      const BlockInfo bi = sh.ent_info[b];
      d.drain<kBlock / 32>(sh.ent[b], (int)bi.n);
      if (bi.last) break;
      bar_arrive(kBarEntEmpty + b, 64);
    }
    d.end(P.err, s);
    if (lane == 0) {
      P.state[s].base = d.dbase;
      P.state[s].cnt = d.cnt;
    }
    return;
  }

  // --------------------------------- chain warp ---------------------------------
  EncChain c;
  c.s = P.fresh ? enc_initial_state().raw : P.state[s].raw;
  for (long long k = 0;; ++k) {
    const int b = (int)(k & 1);
    bar_sync(kBarOpsFull + b, 64);
    const BlockInfo bi = sh.ops_info[b];
    if (k >= 2) bar_sync(kBarEntEmpty + b, 64);  // the drain warp is done with this entry buffer
    // operands are fetched kPrefetch records ahead so that the shared-memory latency stays off the chain; two 64-bit
    // loads per record: each multiply-add gets its addend in a register pair of its own
    const uint2* q = reinterpret_cast<const uint2*>(sh.ops[b]);
    uint2* e = sh.ent[b];
    const int n = (int)bi.n;
    int kk = 0;
    uint2 lo[kPrefetch], hi[kPrefetch];  // records kk .. kk + kPrefetch - 1
#pragma unroll
    for (int r = 0; r < kPrefetch; ++r) {
      lo[r] = q[2 * r];
      hi[r] = q[2 * r + 1];
    }
#pragma unroll 1
    for (; kk + 8 <= n; kk += 8) {
      const uint2* p = q + 2 * kk;
      uint2* const eo = e + kk;
#pragma unroll
      for (int j = 0; j < 8; j += 2) {  // immediates only
        const int r0 = j % kPrefetch, r1 = (j + 1) % kPrefetch;
        const uint2 a0 = lo[r0], b0 = hi[r0], a1 = lo[r1], b1 = hi[r1];
        lo[r0] = p[2 * (j + kPrefetch)];
        hi[r0] = p[2 * (j + kPrefetch) + 1];
        lo[r1] = p[2 * (j + 1 + kPrefetch)];
        hi[r1] = p[2 * (j + 1 + kPrefetch) + 1];
        eo[j] = c.step(a0, b0);
        eo[j + 1] = c.step(a1, b1);
      }
    }
    for (; kk < n; ++kk) e[kk] = c.step(sh.ops[b][kk]);
    if (lane == 0) sh.ent_info[b] = bi;
    bar_arrive(kBarEntFull + b, 64);  // arrive orders the preceding shared-memory writes
    if (bi.last) break;
    bar_arrive(kBarOpsEmpty + b, 64);
  }
  if (lane == 0) {
    P.state[s].span = (c.s < 65536u) ? ((c.s << 16) | 0xFFFFu) : c.s;
    P.state[s].raw = c.s;
  }
}

// ---------------------------------------------------------------------------------------------
// Encoder finalize
// ---------------------------------------------------------------------------------------------
__global__ void enc_init_state_kernel(EncState* st, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) st[i] = enc_initial_state();
}

// Tail rule of RangeEncoder::Finalize (range_coder.cc:266-307) expressed on (words, state).
// Returns the string length; `straddle` = the interval still contains 2^32 ("state 1").
__device__ __forceinline__ long long enc_final_length(const EncState& st, const uint16_t* words,
                                                      bool* straddle, uint32_t* tail, int* ntail) {
  const uint32_t top_end = st.base + st.span;
  *ntail = 0;
  *tail = 0;
  if (top_end < st.base) {
    // The reference picks 2^32: +1 ripples through the run of 0xFFFF words left of the window into
    // word d (the delayed word, < 0xFFFF); everything right of d becomes zero and is dropped, and so
    // is the low byte of word d when it is zero.
    *straddle = true;
    uint32_t d = st.cnt - 1u;
    while (d > 0 && words[d] == 0xFFFFu) --d;
    const uint32_t wd = ((uint32_t)words[d] + 1u) & 0xFFFFu;
    return 2ll * d + 1 + ((wd & 0xFFu) ? 1 : 0);
  }
  *straddle = false;
  if (st.base != 0) {
    const uint32_t r24 = ((st.base - 1u) >> 24) + 1u;
    if (r24 <= (top_end >> 24)) {
      *tail = r24 << 8;
      *ntail = 1;
    } else {
      const uint32_t r16 = ((st.base - 1u) >> 16) + 1u;
      *tail = r16;
      *ntail = (r16 & 0xFFu) ? 2 : 1;
    }
  }
  return 2ll * st.cnt + *ntail;
}

// What finalize needs on the host before it can size the output: the total and the first deferred error.
struct EncResult {
  long long total;
  DevError err;
};

// What finalize reads: the coded streams' state, unresolved words and carry bits, and the deferred error record.
// An encoder handle holds one; the legacy single-stream op sets one up per call.
struct EncArena {
  long long n_streams = 0;
  EncState* state = nullptr;
  uint16_t* words = nullptr;
  uint32_t* cbits = nullptr;
  long long cap = 0;  // words per stream (multiple of 32)
  DevError* err = nullptr;
  const long long* arena_off = nullptr;  // device [n_streams + 1]: per-stream word ranges of a ragged batch (else cap)
};

// Finalize in one block: every stream's string length (enc_final_length), their exclusive scan into
// offsets[0..n_streams], and {total, error} written straight into host-mapped memory, so that one stream
// synchronisation is the only round trip.  `reset_err` clears the error record for the next user of a recycled
// encoder.
__global__ void __launch_bounds__(1024) enc_offsets_kernel(const EncState* state, const uint16_t* words,
                                                           long long cap, const long long* arena_off,
                                                           long long n_streams, long long* offsets,
                                                           DevError* err, int reset_err, EncResult* res) {
  __shared__ long long warp_sums[32];
  __shared__ long long carry_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (long long base = 0; base < n_streams; base += blockDim.x) {
    const long long i = base + tid;
    long long v = 0;
    if (i < n_streams) {
      bool straddle;
      uint32_t tail;
      int ntail;
      v = enc_final_length(state[i], words + (arena_off ? arena_off[i] : i * cap), &straddle, &tail, &ntail);
    }
    long long x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long y = __shfl_up_sync(kFull, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
      long long w = (lane < (int)(blockDim.x >> 5)) ? warp_sums[lane] : 0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const long long y = __shfl_up_sync(kFull, w, d);
        if (lane >= d) w += y;
      }
      warp_sums[lane] = w;  // inclusive
    }
    __syncthreads();
    const long long before = carry_s + (wid ? warp_sums[wid - 1] : 0) + (x - v);
    if (i < n_streams) offsets[i] = before;
    __syncthreads();
    if (tid == blockDim.x - 1) carry_s = before + v;
    __syncthreads();
  }
  if (tid == 0) {
    offsets[n_streams] = carry_s;
    res->total = carry_s;
    res->err = *err;
    if (reset_err) *err = DevError{};
  }
}

// One CTA of kWriteWarps warps per stream.  The carry chain runs right to left over 32-word groups; it is cut into
// kWriteWarps segments: every warp first runs its segment's chain for BOTH possible carries entering it (two adds per
// group instead of one), the segments' carry-ins are then resolved through shared memory (a chain of kWriteWarps
// steps), and each warp resolves and writes its own segment.  (One warp per stream walked 200 groups serially:
// 46 us of the 714 us cfg2 step.)
constexpr int kWriteWarps = 8;

__global__ void __launch_bounds__(32 * kWriteWarps) enc_write_kernel(const EncState* state, const uint16_t* words,
                                                                    const uint32_t* cbits, long long cap,
                                                                    const long long* arena_off, long long n_streams,
                                                                    const long long* offsets, uint8_t* out) {
  __shared__ uint32_t seg_out[kWriteWarps][2];
  const long long s = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (s >= n_streams) return;
  const EncState st = state[s];
  const long long abase = arena_off ? arena_off[s] : s * cap;
  const uint16_t* w = words + abase;
  const uint32_t* cb = cbits + (abase >> 5);
  uint8_t* dst = out + offsets[s];
  bool straddle;
  uint32_t tail;
  int ntail;
  const long long len = enc_final_length(st, w, &straddle, &tail, &ntail);
  const long long body = straddle ? len : 2ll * st.cnt;  // bytes that come from resolved words

  const long long n_groups = ((long long)st.cnt + 31) >> 5;
  const long long per = (n_groups + kWriteWarps - 1) / kWriteWarps;
  const long long g_lo = min((long long)warp * per, n_groups), g_hi = min(g_lo + per, n_groups);  // this warp's groups
  const bool even = ((reinterpret_cast<uintptr_t>(dst)) & 1) == 0;
  constexpr int kBatch = 8;  // groups whose (independent) loads are in flight together

  // One pass over the segment [g_lo, g_hi), right to left.  WRITE = false: only the carries leaving the segment for a
  // carry of 0 and of 1 entering it; WRITE = true: resolve with the real carry `x0` and store the bytes.
  auto pass = [&](uint32_t& x0, uint32_t& x1, const bool write) {
    for (long long gt = g_hi; gt > g_lo; gt -= kBatch) {
      uint32_t word[kBatch], F[kBatch];
#pragma unroll
      for (int i = 0; i < kBatch; ++i) {
        const long long g = gt - 1 - i;
        const uint32_t idx = (uint32_t)(g << 5) + lane;
        word[i] = (g >= g_lo && idx < st.cnt) ? (uint32_t)w[idx] : 0u;
        F[i] = (g >= g_lo) ? cb[g] : 0u;
      }
#pragma unroll
      for (int i = 0; i < kBatch; ++i) {
        const long long g = gt - 1 - i;
        if (g < g_lo) break;
        const uint32_t idx = (uint32_t)(g << 5) + lane;
        const bool live = idx < st.cnt;
        uint32_t Fm = F[i];
        const uint32_t fill = st.cnt - (uint32_t)(g << 5);
        if (fill < 32u) Fm &= (1u << fill) - 1u;
        // P: word propagates a carry.  Dead lanes right of the last word must pass the carry through.
        const uint32_t Pm = __ballot_sync(kFull, live ? (word[i] == 0xFFFFu) : true);
        // position j = 31 - lane (bit 0 = right-most word); c[j+1] = F[31-j] | (P[31-j] & c[j])
        const uint32_t G = __brev(Fm);
        const uint32_t A = G | __brev(Pm);
        const unsigned long long sum = (unsigned long long)A + G + x0;
        if (!write) x1 = (uint32_t)(((unsigned long long)A + G + x1) >> 32) & 1u;
        const uint32_t cin = (uint32_t)sum ^ A ^ G;  // bit j = carry into position j
        const uint32_t my_c = (cin >> (31 - lane)) & 1u;
        x0 = (uint32_t)(sum >> 32) & 1u;
        if (write && live) {
          const uint32_t r = (word[i] + my_c) & 0xFFFFu;
          const long long b0 = 2ll * idx;
          if (even && b0 + 1 < body) {
            *reinterpret_cast<uint16_t*>(dst + b0) = (uint16_t)((r >> 8) | ((r & 0xFFu) << 8));  // big endian
          } else {
            if (b0 < body) dst[b0] = (uint8_t)(r >> 8);
            if (b0 + 1 < body) dst[b0 + 1] = (uint8_t)r;
          }
        }
      }
    }
  };
  uint32_t o0 = 0u, o1 = 1u;
  pass(o0, o1, false);
  if (lane == 0) {
    seg_out[warp][0] = o0;
    seg_out[warp][1] = o1;
  }
  __syncthreads();
  // carry entering the right-most word (index cnt - 1), then through the segments to the right of this one
  uint32_t x = straddle ? 1u : ((cb[st.cnt >> 5] >> (st.cnt & 31u)) & 1u);
  for (int k = kWriteWarps - 1; k > warp; --k) x = seg_out[k][x];
  uint32_t unused = 0u;
  pass(x, unused, true);
  if (!straddle && threadIdx.x == 0) {
    if (ntail >= 1) dst[body] = (uint8_t)(tail >> 8);
    if (ntail == 2) dst[body + 1] = (uint8_t)tail;
  }
}

__global__ void enc_grow_kernel(const uint16_t* src, const uint32_t* src_cb, long long src_cap,
                                uint16_t* dst, uint32_t* dst_cb, long long dst_cap,
                                const EncState* state) {
  const long long s = blockIdx.x;
  const uint32_t used = (state[s].cnt + 31u) & ~31u;
  for (uint32_t i = threadIdx.x; i < used; i += blockDim.x) dst[s * dst_cap + i] = src[s * src_cap + i];
  for (uint32_t i = threadIdx.x; i <= (state[s].cnt >> 5); i += blockDim.x)
    dst_cb[s * (dst_cap >> 5) + i] = src_cb[s * (src_cap >> 5) + i];
}

// ---------------------------------------------------------------------------------------------
// Decoder
// ---------------------------------------------------------------------------------------------
struct DecParams {
  const int32_t* lookup;
  const int2* rows;
  const uint2* pairs;
  const int4* rows4;
  int n_rows;
  long long lookup_len;
  long long n_pairs;
  int zero_win;
  const uint8_t* bytes;
  const long long* offsets;
  const int32_t* index;
  void* out;               // int32 or float [S, n]
  const float* qoff;       // channel: [n_rows]; index: loc [S, n]
  const int32_t* coff;     // [n_rows]
  long long n;
  long long n_streams;
  DecState* state;
  DevError* err;
  const long long* sym_off;  // ragged batches: stream s is symbols [sym_off[s], sym_off[s+1]); null: [s * n, s * n + n)
  // 16-bit index modes without kModeLocF32: loc [S, n] in the output's type, or null (last: the other fields keep
  // their parameter offsets).  `out` is in the value's type, float under kModeLocF32; `qoff` is float32 otherwise.
  const uint16_t* loc16;
};

// ---------------------------------------------------------------------------------------------
// Decoder: three warps per stream (prepare / chain / resolve), pre-scaled search keys
// ---------------------------------------------------------------------------------------------
// The decoder has the encoder's recurrence plus a search per symbol.  As in the encoder everything that
// is not the recurrence leaves the latency-critical warp:
//   prepare warp : per symbol the row's search window (64 pre-scaled keys around the row's median), and the
//                  stream's next 16-bit words in a shared-memory ring well ahead of the chain;
//   chain warp   : every lane evaluates two keys B'(c) = T(c) - 1 = hi32(span*c' + addend) (one IMAD.HI
//                  each), two warp reductions give the bracketing pair (a, b1) and the new interval; the
//                  SYMBOL INDEX is not needed to continue -- only {value - base, span} are recorded;
//   resolve warp : recovers the symbol index of 32 recorded symbols at a time by binary search over the
//                  window, applies cdf_offset / de-quantisation and writes the output coalesced.
// Rare cases (escape symbols, symbols outside the window, rows wider than the window) are handled on the
// chain warp by a generic warp-parallel search and hand the finished symbol to the resolve warp.
constexpr int kDecGroup = 128;
constexpr int kRingAhead = 1536;  // > words two groups can consume even if every symbol escapes (256 * 5.1)

struct DecDesc {      // one symbol's search window, prepared ahead of the chain
  int win;            // key index of the window's first key (segment start + wfirst; the zero window if irregular)
  uint32_t thr;       // the window's answer needs a candidate below v unless it starts the row: slow if a < thr
  int seg;            // key index of cdf[0]
  int n;              // ncdf - 1, bit 31: overflow row
};

struct DecShared {
  DecDesc desc[2][kDecGroup + 2];
  uint2 ent[2][kDecGroup];        // {value - base, span} before the symbol's update
  int ovr[2][kDecGroup];          // symbols finished on the chain warp (escapes, window misses)
  unsigned ovr_mask[2][kDecGroup / 32];
  unsigned bad[2];
  unsigned count[2];
  unsigned rbad[2];    // chain -> resolve copies (the prepare warp may already be two groups ahead)
  unsigned rcount[2];
  unsigned pos_pub[2]; // chain -> prepare: stream position (16-bit words) after the group that used buffer b
};

enum : int { kBarDescFull = 1, kBarDescEmpty = 3, kBarDecEntFull = 5, kBarDecEntEmpty = 7 };

template <int MODE, bool SMEM>
__global__ void __launch_bounds__(96) decode_kernel(const DecParams P) {
  extern __shared__ __align__(16) uint8_t s_dyn[];
  __shared__ __align__(16) DecShared sh;
  // The stream's next words, filled ahead by the prepare warp.  The chain warp addresses the ring as
  // base | offset, so its ABSOLUTE shared address must be 4096-byte aligned (static alignment is relative to the
  // CTA's window, which starts after the reserved 1 KB): carve an aligned ring out of a buffer twice the size.
  __shared__ __align__(16) uint16_t ring_buf[2 * kRing];
  uint16_t* const ring = ring_buf + (((4096u - (smem_addr(ring_buf) & 4095u)) & 4095u) >> 1);
  const long long s = blockIdx.x;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;  // 0 chain, 1 prepare, 2 resolve
  const Extent x = stream_extent(P.sym_off, s, P.n);
  const long long n_groups = (x.len + kDecGroup - 1) / kDecGroup;

  // tables: shared memory when they fit (loaded by all three warps), global (L1/L2) otherwise
  const uint2* pairs = P.pairs;
  const int4* rows4 = P.rows4;
  if (SMEM) {
    uint2* sp = reinterpret_cast<uint2*>(s_dyn);
    int4* sr = reinterpret_cast<int4*>(s_dyn + ((P.n_pairs * 8 + 15) & ~15ll));
    for (int i = threadIdx.x; i < (int)P.n_pairs; i += blockDim.x) sp[i] = P.pairs[i];
    for (int i = threadIdx.x; i < P.n_rows; i += blockDim.x) sr[i] = P.rows4[i];
    __syncthreads();
    pairs = sp;
    rows4 = sr;
  }

  if (warp == 1) {
    // ------------------------------- prepare warp -------------------------------
    uint32_t chan_row = (uint32_t)lane % (uint32_t)P.n_rows;
    const uint32_t chan_step = 32u % (uint32_t)P.n_rows;
    ByteWindow bw;
    bw.p = P.bytes + P.offsets[s];
    bw.len = P.offsets[s + 1] - P.offsets[s];
    long long filled = (long long)P.state[s].pos;  // ring holds words [.., filled)
    auto fill_ring = [&](long long upto) {
      for (long long wi = filled + lane; wi < upto; wi += 32) ring[wi & (kRing - 1)] = (uint16_t)bw_fetch(bw, wi);
      filled = max(filled, upto);
    };
    fill_ring(filled + kRingAhead);
    for (long long g = 0; g < n_groups; ++g) {
      const int b = (int)(g & 1);
      if (g >= 2) {
        bar_sync(kBarDescEmpty + b, 64);
        fill_ring((long long)sh.pos_pub[b] + kRingAhead);  // pos after group g-2; two groups consume < kRingAhead
      }
      unsigned bad = 0;
#pragma unroll
      for (int sub = 0; sub < kDecGroup / 32; ++sub) {
        const long long j = g * kDecGroup + sub * 32 + lane;
        int row = (int)chan_row;
        if (MODE & kModeIndex) {
          row = 0;
          if (j < x.len) {
            row = __ldg(P.index + x.base + j);
            if (row < 0 || row >= P.n_rows) {
              report(P.err, kErrIndex, s, j, row, P.n_rows);
              row = -1;
            }
          }
          bad |= __ballot_sync(kFull, row < 0);
          if (row < 0) row = 0;
        } else {
          chan_row += chan_step;
          if (chan_row >= (uint32_t)P.n_rows) chan_row -= (uint32_t)P.n_rows;
        }
        const int4 r4 = rows4[row];
        DecDesc d;
        d.win = r4.w ? P.zero_win : r4.x + r4.z;
        d.thr = (r4.z > 1 || r4.w) ? 1u : 0u;
        d.seg = r4.x;
        d.n = (row_ncdf(r4.y) - 1) | (row_ovf(r4.y) ? (int)0x80000000 : 0);
        sh.desc[b][sub * 32 + lane] = d;
        if (sub == kDecGroup / 32 - 1 && lane < 2) sh.desc[b][kDecGroup + lane] = d;  // pipeline overrun slots
      }
      if (lane == 0) {
        sh.bad[b] = bad;
        sh.count[b] = (unsigned)min((long long)kDecGroup, x.len - g * kDecGroup);
      }
      bar_arrive(kBarDescFull + b, 64);
      if (bad) break;
    }
    return;
  }

  if (warp == 2) {
    // ------------------------------- resolve warp -------------------------------
    for (long long g = 0; g < n_groups; ++g) {
      const int b = (int)(g & 1);
      bar_sync(kBarDecEntFull + b, 64);
      const int count = (int)sh.rcount[b];
      if (sh.rbad[b]) break;
      for (int sub = 0; sub * 32 < count; ++sub) {
        const int k = sub * 32 + lane;
        const long long j = g * kDecGroup + k;
        if (k < count) {
          const long long at = x.base + j;
          int row;
          if (MODE & kModeIndex) row = __ldg(P.index + at);
          else row = (int)(j % P.n_rows);
          int sym;
          if ((sh.ovr_mask[b][sub] >> lane) & 1u) {
            sym = sh.ovr[b][k];
          } else {
            // binary search inside the window: smallest key index whose bound is >= v.  The key just left of
            // the window is known to be below (cdf[0] = 0, or a below-candidate existed), the last one >= v.
            const int4 r4 = rows4[row];
            const uint2 e = sh.ent[b][k];
            const uint2* keys = pairs + r4.x;
            int lo = r4.z - 1, hi = r4.z + 63;
#pragma unroll
            for (int it = 0; it < 6; ++it) {
              const int mid = (lo + hi + 1) >> 1;
              const bool ge = e.x <= key_bound(e.y, keys[mid]);
              hi = ge ? mid : hi;
              lo = ge ? lo : mid;
            }
            sym = hi - 1;
          }
          if (MODE & kMode16) {
            const int sc = sym + __ldg(P.coff + row);
            float off = 0.f;
            bool has_off;
            if (!(MODE & kModeIndex)) {  // the quantisation offset rounded to the value's type, as in enc_gather
              has_off = P.qoff != nullptr;
              if (has_off) off = widen16<MODE>(narrow16<MODE>(__ldg(P.qoff + row)));
            } else if (MODE & kModeLocF32) {
              has_off = true;
              off = __ldg(P.qoff + at);
            } else {
              has_off = P.loc16 != nullptr;
              if (has_off) off = widen16<MODE>(__ldg(P.loc16 + at));
            }
            const float r = dequantise16<MODE>(sc, has_off, off);
            if (MODE & kModeLocF32) reinterpret_cast<float*>(P.out)[at] = r;
            else reinterpret_cast<uint16_t*>(P.out)[at] = narrow16<MODE>(r);
          } else if (MODE & kModeF32) {
            float yv = (float)(sym + __ldg(P.coff + row));
            if (P.qoff) yv += (MODE & kModeIndex) ? __ldg(P.qoff + at) : __ldg(P.qoff + row);
            reinterpret_cast<float*>(P.out)[at] = yv;
          } else {
            reinterpret_cast<int32_t*>(P.out)[at] = sym;
          }
        }
      }
      if (g + 2 < n_groups) bar_arrive(kBarDecEntEmpty + b, 64);
    }
    return;
  }

  // --------------------------------- chain warp ---------------------------------
  Dec2 c;
  c.lane = lane;
  {
    const DecState st = P.state[s];
    c.base = st.base;
    c.span = st.span;
    c.value = st.value;
    c.pos2 = st.pos << 1;
  }
  c.ring_addr = opaque(smem_addr(ring));
  bool started = false;

  for (long long g = 0; g < n_groups; ++g) {
    const int b = (int)(g & 1);
    bar_sync(kBarDescFull + b, 64);
    if (!started) {  // the ring is valid from here on
      started = true;
      if (c.pos2 == 0) {  // fresh stream: the constructor reads four bytes (range_coder.h:79-83)
        c.value = ((uint32_t)ring[0] << 16) | (uint32_t)ring[1];
        c.pos2 = 4;
      }
      c.seek();
    }
    const bool bad = sh.bad[b] != 0;
    const int count = bad ? 0 : (int)sh.count[b];
    if (g >= 2) bar_sync(kBarDecEntEmpty + b, 64);  // the resolve warp is done with this entry buffer
    const DecDesc* desc = sh.desc[b];
    unsigned om0 = 0, om1 = 0, om2 = 0, om3 = 0;  // symbols finished on this warp (bit per symbol)
    // opaque shared addresses: keeps them in registers instead of being re-derived every symbol
    const uint32_t desc_addr = opaque(smem_addr(sh.desc[b]));
    const uint32_t ent_addr = opaque(smem_addr(sh.ent[b]));
    const uint2* lkeys = pairs + lane;  // this lane's two candidates: lkeys[win], lkeys[win + 32]
    const uint32_t lkeys_addr = SMEM ? opaque(smem_addr(lkeys)) : 0u;
    auto load_keys = [&](uint32_t win, uint2& q0, uint2& q1) {
      if (SMEM) {
        q0 = lds_v2(lkeys_addr + win * 8u);
        q1 = lds_v2(lkeys_addr + win * 8u + 256u);
      } else {
        q0 = __ldg(lkeys + win);
        q1 = __ldg(lkeys + win + 32);
      }
    };
    // One symbol of the fast path.  dc = descriptor of this symbol (reloaded with the one two ahead once
    // used), dn = the next symbol's; qc* = this symbol's candidate keys, qn* = receives the next symbol's.
    // Called with the roles swapped on alternate symbols so that the software pipeline needs no register
    // moves.  The interval update is issued BEFORE the "is this symbol special" branch so that the branch
    // latency is off the serial chain; a special symbol restores the state and leaves the loop.
    uint32_t daddr = desc_addr + 32u;  // descriptor two symbols ahead
    uint32_t eaddr = ent_addr;         // this symbol's entry
    const uint32_t eend = ent_addr + (uint32_t)count * 8u;
    uint32_t ra = 0, rb1 = 0, rthr = 0;  // the special symbol's window answer
    auto step = [&](uint2& dc, const uint2& dn, const uint2& qc0, const uint2& qc1, uint2& qn0, uint2& qn1) -> bool {
      load_keys(dn.x, qn0, qn1);
      const uint32_t thr = dc.y;
      dc = lds_v2(daddr);
      daddr += 16u;
      const uint32_t v = c.value - c.base;
      const uint32_t span0 = c.span;
      const uint32_t B0 = key_bound(span0, qc0), B1 = key_bound(span0, qc1);
      const bool ge0 = v <= B0, ge1 = v <= B1;
      const uint32_t m = ge0 ? B0 : (ge1 ? B1 : 0xFFFFFFFFu);
      const uint32_t am = ge1 ? (ge0 ? 0u : B0 + 1u) : B1 + 1u;
      const uint32_t b1 = __reduce_min_sync(kFull, m);
      const uint32_t a = __reduce_max_sync(kFull, am);
      sts_v2(eaddr, v, span0);
      eaddr += 8u;
      // Fast path: the window holds a key >= v that is not the row's last one, and (unless the window starts
      // the row) a key below v.  b1 >= span0 covers "no key" (~0) and the last bin (escape of overflow rows).
      const bool special = !(b1 < span0 && a >= thr);
      const uint32_t base0 = c.base, value0 = c.value, pos0 = c.pos2, next0 = c.next;
      c.update(a, b1);
      if (special) {
        c.base = base0;
        c.span = span0;
        c.value = value0;
        c.pos2 = pos0;
        c.next = next0;
        ra = a;
        rb1 = b1;
        rthr = thr;
      }
      return special;
    };
    uint2 da, db, qa0, qa1, qb0, qb1;
    auto prime = [&](uint32_t k) {  // restart the software pipeline at symbol k
      daddr = desc_addr + k * 16u;
      da = lds_v2(daddr);
      db = lds_v2(daddr + 16u);
      daddr += 32u;
      load_keys(da.x, qa0, qa1);
    };
    prime(0u);
    for (;;) {
      bool special = false;
      for (;;) {
        if (eaddr == eend) break;
        special = step(da, db, qa0, qa1, qb0, qb1);
        if (special) break;
        if (eaddr == eend) break;
        special = step(db, da, qb0, qb1, qa0, qa1);
        if (special) break;
      }
      if (!special) break;
      // ---- special symbol k: its entry is stored, the coder state is the one before it ----
      const int k = (int)((eaddr - 8u - ent_addr) >> 3);
      uint32_t a = ra, b1 = rb1;
      const DecDesc df = desc[k];
      const int n = df.n & 0x7FFFFFFF;
      const bool ovf = df.n < 0;
      const bool miss = (b1 == 0xFFFFFFFFu) || (a < rthr);
      int sym = n - 1;  // in-window hit with b1 == span: the row's last bin (regular rows)
      if (miss) sym = c.search_row(pairs, df.seg, n, &a, &b1);
      c.update(a, b1);
      bool finished = miss;
      if (ovf && sym == n - 1) {  // OverflowDecode, range_coder_kernels.cc:449-471
        int nb = 0;
        while (c.bit() == 0 && nb < 32) ++nb;  // valid int32 gamma codes have <= 31 zeros; bounds what a corrupt stream can consume (kRingAhead)
        uint32_t val = (nb < 32) ? (1u << nb) : 0u;
        int t = nb;
        while (--t >= 0) {
          const uint32_t bitv = c.bit();
          if (t < 32) val |= bitv << t;
        }
        const uint32_t sg = c.bit();
        sym = sg ? -(int)val : (int)val + (n - 1) - 1;
        finished = true;
      }
      if (finished) {  // otherwise the resolve warp finds the (last) bin like any other
        sh.ovr[b][k] = sym;
        const unsigned bitk = 1u << (k & 31);
        om0 |= (k >> 5) == 0 ? bitk : 0u;
        om1 |= (k >> 5) == 1 ? bitk : 0u;
        om2 |= (k >> 5) == 2 ? bitk : 0u;
        om3 |= (k >> 5) == 3 ? bitk : 0u;
      }
      prime((uint32_t)k + 1u);
    }

    const unsigned omask[kDecGroup / 32] = {om0, om1, om2, om3};
    if (lane == 0) {
#pragma unroll
      for (int i = 0; i < kDecGroup / 32; ++i) sh.ovr_mask[b][i] = omask[i];
      sh.rbad[b] = bad ? 1u : 0u;
      sh.rcount[b] = (unsigned)count;
    }
    bar_arrive(kBarDecEntFull + b, 64);
    if (bad) break;
    if (g + 2 < n_groups) {
      if (lane == 0) sh.pos_pub[b] = c.pos2 >> 1;
      bar_arrive(kBarDescEmpty + b, 64);
    }
  }
  if (lane == 0) {
    DecState st;
    st.base = c.base;
    st.span = c.span;
    st.value = c.value;
    st.pos = c.pos2 >> 1;
    P.state[s] = st;
  }
}

__global__ void dec_init_state_kernel(DecState* st, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) {
    DecState s;
    s.base = 0;
    s.span = 0xFFFFFFFFu;
    s.value = 0;
    s.pos = 0;
    st[i] = s;
  }
}

// RangeDecoder::Finalize, range_coder.h:144-169.
__global__ void dec_finalize_kernel(const DecState* state, const uint8_t* bytes, const long long* offsets,
                                    long long n, uint8_t* ok) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= n) return;
  DecState st = state[s];
  const long long len = offsets[s + 1] - offsets[s];
  if (st.pos == 0) {  // never decoded from: only the constructor ran (four bytes, zero padded)
    const uint8_t* p = bytes + offsets[s];
    uint32_t v = 0;
    for (int i = 0; i < 4; ++i) v = (v << 8) | (i < len ? (uint32_t)p[i] : 0u);
    st.value = v;
    st.pos = 2;
  }
  bool good;
  if (2ll * st.pos < len) {
    good = false;  // did not read to the end
  } else {
    const uint32_t top_end = st.base + st.span;
    if (st.base == 0 || top_end < st.base) {
      good = (st.value == 0);
    } else {
      const int shift = (((st.base - 1u) >> 24) < (top_end >> 24)) ? 24 : 16;
      const uint32_t mid = ((st.base - 1u) >> shift) + 1u;
      good = ((mid << shift) == st.value);
    }
  }
  ok[s] = good ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------
// Legacy single-stream ops
// ---------------------------------------------------------------------------------------------
struct LegacyDims {
  int rank;               // merged rank (<= 6)
  long long data[6];      // merged data shape
  long long cdfd[6];      // merged cdf shape
  long long chip;         // strip length
};

__device__ __forceinline__ long long legacy_strip(const LegacyDims& d, long long lin) {
  long long off = 0, stride = d.chip;
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    if (i < d.rank) {
      const long long coord = lin % d.data[i];
      lin /= d.data[i];
      if (d.cdfd[i] > 1) off += coord * stride;
      stride *= d.cdfd[i];
    }
  }
  return off;
}

// CheckCdfValues, range_coding_kernels.cc:150-173.
__global__ void legacy_check_cdf_kernel(const int32_t* cdf, long long rows, long long size, int precision,
                                        DevError* err) {
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int32_t* s = cdf + r * size;
  const int32_t top = 1 << precision;
  if (s[0] != 0 || s[size - 1] != top) {
    report(err, kErrCdf, r, 0, s[0], s[size - 1], 1);
    return;
  }
  for (long long j = 0; j + 1 < size; ++j) {
    if (s[j + 1] <= s[j]) {
      report(err, kErrCdf, r, j, s[j], s[j + 1], 2);
      return;
    }
  }
}

__global__ void __launch_bounds__(32) legacy_encode_kernel(const int16_t* data, long long n,
                                                           const int32_t* cdf, LegacyDims dims,
                                                           int precision, int debug, EncState* state,
                                                           uint16_t* words, uint32_t* cbits,
                                                           long long cap, DevError* err) {
  __shared__ __align__(8) uint2 s_ent[32];
  const int lane = threadIdx.x;
  EncState st0;
  st0.base = 0;
  st0.span = 0xFFFFFFFFu;
  st0.cnt = 0;
  st0.raw = 0xFFFFFFFFu;
  EncChain c;
  c.s = st0.raw;
  EncDrain d;
  d.begin(st0, words, cbits, (uint32_t)cap, lane);
  for (long long g0 = 0; g0 < n; g0 += 32) {
    const int count = (int)min(32ll, n - g0);
    uint32_t lower = 0, upper = 1;
    bool bad = false;
    if (lane < count) {
      const long long j = g0 + lane;
      const long long v = data[j];
      if (v < 0 || dims.chip <= v + 1) {
        if (debug > 0) report(err, kErrValue, 0, j, v, dims.chip - 1);
        bad = true;  // without debug the reference has undefined behaviour; we stop instead
      } else {
        const int32_t* strip = cdf + legacy_strip(dims, j);
        lower = (uint32_t)strip[v];
        upper = (uint32_t)strip[v + 1];
        if (!(lower < upper) || upper > (1u << precision)) {
          bad = true;  // zero-probability symbol / invalid strip: UB in the reference
          report(err, kErrCdf, 0, j, lower, upper, 3);
        }
      }
    }
    if (__ballot_sync(kFull, bad)) break;
    uint2 mine = make_uint2(0u, 0u);
    for (int k = 0; k < count; ++k) {  // every lane runs the same recurrence; lane k keeps entry k
      const uint32_t lo = __shfl_sync(kFull, lower, k);
      const uint32_t hi = __shfl_sync(kFull, upper, k);
      const uint2 e = c.step(enc_operands(lo, hi, (uint32_t)precision));
      if (lane == k) mine = e;
    }
    s_ent[lane] = mine;
    __syncwarp();
    d.drain<1>(s_ent, count);
    __syncwarp();
  }
  d.end(err, 0);
  if (lane == 0) {
    EncState st;
    st.base = d.dbase;
    st.span = (c.s < 65536u) ? ((c.s << 16) | 0xFFFFu) : c.s;
    st.cnt = d.cnt;
    st.raw = c.s;
    state[0] = st;
  }
}

__global__ void __launch_bounds__(32) legacy_decode_kernel(const uint8_t* bytes, long long len,
                                                           long long n, const int32_t* cdf,
                                                           LegacyDims dims, int precision,
                                                           int16_t* out) {
  const int lane = threadIdx.x;
  DecChain c;
  c.base = 0;
  c.span = 0xFFFFFFFFu;
  ByteWindow w;
  w.p = bytes;
  w.len = len;
  c.value = (bw_fetch(w, 0) << 16) | bw_fetch(w, 1);
  c.pos = 2;
  bw_seek(w, c.pos, lane);
  for (long long g0 = 0; g0 < n; g0 += 32) {
    const int count = (int)min(32ll, n - g0);
    long long my_off = 0;
    if (lane < count) my_off = legacy_strip(dims, g0 + lane);
    int my_sym = 0;
    for (int k = 0; k < count; ++k) {
      const long long off = __shfl_sync(kFull, my_off, k);
      const int sym = dec_symbol(c, w, cdf + off, (int)dims.chip, (uint32_t)precision, lane);
      if (lane == k) my_sym = sym;
    }
    if (lane < count) out[g0 + lane] = (int16_t)my_sym;
  }
}

// ---------------------------------------------------------------------------------------------
// Host-side handles
// ---------------------------------------------------------------------------------------------
// Device-table cache.  A model creates a handle per compress()/decompress() call with the same `lookup`
// every time (continuous_batched.py:381, :408): parsing and uploading it again (plus the stream
// synchronisation that keeps the host staging alive) would sit on the host's critical path of every step.
// Entries are keyed by content (hash, then full compare), pinned while a handle uses them, and evicted
// least-recently-used beyond kMaxEntries.  Uploads are complete (stream-synchronised) before an entry becomes
// visible, so any stream may use it.
// ---------------------------------------------------------------------------------------------
struct LookupCache {
  struct Entry {
    uint64_t hash = 0;
    int64_t cols = 0;
    bool for_decoder = false;
    int device = 0;
    int pins = 0;
    uint64_t last_use = 0;
    std::vector<int32_t> host;
    DeviceLookup lut;
  };
  static constexpr size_t kMaxEntries = 16;
  std::mutex mu;
  std::vector<Entry*> entries;
  uint64_t clock = 0;

  static uint64_t hash_of(const int32_t* p, int64_t n) {
    uint64_t hsh = 1469598103934665603ull;
    for (int64_t i = 0; i < n; ++i) hsh = (hsh ^ (uint32_t)p[i]) * 1099511628211ull;
    return hsh;
  }

  int acquire(const int32_t* host, int64_t len, int64_t cols, bool for_decoder, cudaStream_t s, DeviceLookup* out,
              void** token) {
    *token = nullptr;
    if (len < 0 || (len > 0 && !host)) return fail(TFCB_INVALID_ARGUMENT, "bad lookup table");
    int device = 0;
    cudaGetDevice(&device);
    const uint64_t hsh = hash_of(host, len);
    std::lock_guard<std::mutex> lock(mu);
    for (Entry* e : entries) {
      if (e->hash == hsh && e->cols == cols && e->for_decoder == for_decoder && e->device == device &&
          (int64_t)e->host.size() == len && (len == 0 || std::memcmp(e->host.data(), host, len * sizeof(int32_t)) == 0)) {
        e->pins++;
        e->last_use = ++clock;
        *out = e->lut;
        *token = e;
        return TFCB_OK;
      }
    }
    Entry* e = new Entry;
    int rc = e->lut.upload(host, len, cols, s, for_decoder);  // synchronises s: the tables are resident on return
    if (rc != TFCB_OK) {
      e->lut.release(s);
      delete e;
      return rc;
    }
    e->hash = hsh;
    e->cols = cols;
    e->for_decoder = for_decoder;
    e->device = device;
    e->pins = 1;
    e->last_use = ++clock;
    e->host.assign(host, host + len);
    entries.push_back(e);
    while (entries.size() > kMaxEntries) {
      size_t victim = entries.size();
      for (size_t i = 0; i < entries.size(); ++i)
        if (entries[i]->pins == 0 && (victim == entries.size() || entries[i]->last_use < entries[victim]->last_use)) victim = i;
      if (victim == entries.size()) break;  // everything is in use
      cudaDeviceSynchronize();  // rare (> kMaxEntries distinct tables): no kernel of any stream may still read it
      entries[victim]->lut.release(s);
      delete entries[victim];
      entries.erase(entries.begin() + victim);
    }
    *out = e->lut;
    *token = e;
    return TFCB_OK;
  }

  // Whether the entry pinned by `token` holds exactly this encoder table.  (A pinned entry is never evicted, and
  // its fields do not change after it became visible.)
  bool same(const void* token, const int32_t* host, int64_t len, int64_t cols) {
    const Entry* e = static_cast<const Entry*>(token);
    if (!e || e->for_decoder || e->cols != cols || (int64_t)e->host.size() != len || (len > 0 && !host)) return false;
    int device = 0;
    cudaGetDevice(&device);
    return e->device == device && (len == 0 || std::memcmp(e->host.data(), host, len * sizeof(int32_t)) == 0);
  }

  void release(void* token) {
    if (!token) return;
    std::lock_guard<std::mutex> lock(mu);
    static_cast<Entry*>(token)->pins--;
  }
};

LookupCache& lookup_cache() {
  static LookupCache* c = new LookupCache;  // leaked on purpose: no destructor order problems at exit
  return *c;
}

int decode_error(const DevError& e, const char* what);

int fetch_error(DevError* d_err, cudaStream_t s, const char* what) {
  DevError e;
  TFCB_CUDA_TRY(cudaMemcpyAsync(&e, d_err, sizeof e, cudaMemcpyDeviceToHost, s));
  TFCB_CUDA_TRY(cudaStreamSynchronize(s));
  return decode_error(e, what);
}

int decode_error(const DevError& e, const char* what) {
  switch (e.code) {
    case kErrNone:
      return TFCB_OK;
    case kErrIndex:
      return fail(TFCB_INVALID_ARGUMENT, "index=%lld not in range [0, %lld) (stream %lld, element %lld)",
                  e.value, e.limit, e.stream, e.pos);
    case kErrValue:
      if (std::strcmp(what, "legacy") == 0)
        return fail(TFCB_INVALID_ARGUMENT, "'data' value not in [0, %lld): value=%lld", e.limit, e.value);
      return fail(TFCB_INVALID_ARGUMENT, "value=%lld not in range [0, %lld) (stream %lld, element %lld)",
                  e.value, e.limit, e.stream, e.pos);
    case kErrCapacity:
      return fail(TFCB_CUDA_ERROR, "internal: output arena too small (stream %lld needs > %lld words)",
                  e.stream, e.limit);
    case kErrCdf:
      if (e.aux == 1)
        return fail(TFCB_INVALID_ARGUMENT, "CDF should start from 0 and end at 2^precision: cdf[0]=%lld, cdf[^1]=%lld",
                    e.value, e.limit);
      if (e.aux == 2) return fail(TFCB_INVALID_ARGUMENT, "CDF is not monotonic");
      return fail(TFCB_INVALID_ARGUMENT,
                  "symbol with zero probability or invalid CDF strip at element %lld: lower=%lld upper=%lld",
                  e.pos, e.value, e.limit);
  }
  return fail(TFCB_CUDA_ERROR, "unknown device error %d", e.code);
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

struct tfcb_encoder : EncArena {
  DeviceLookup lut;      // shallow copy of a cache entry's tables
  void* lut_token = nullptr;
  long long bound = 0;  // worst-case words emitted so far per stream
  bool fresh = true;  // no encode yet: `state` is not initialised (the first encode starts from the initial state)
  bool finalized = false;  // tfcb_encode_finalize succeeded: only tfcb_encode_write (once) and destroy remain
  cudaStream_t home = nullptr;
  // tfcb_compress recycles its encoders: `device` keys the pool, `done` is recorded after the last kernel that
  // reads the word arena, and the next user's stream waits for it
  int device = 0;
  cudaEvent_t done = nullptr;
  long long arena_words = 0;  // words allocated in `words` (cbits: arena_words / 32): n_streams * cap, or more
  long long* ext = nullptr;   // ragged batches, device [2 * (n_streams + 1)]: symbol offsets, then arena offsets
};

namespace {

long long words_bound(const tfcb_encoder* h, long long n) {
  return words_for(bits_bound(h->lut.max_prec, h->lut.any_overflow), n);
}

int ensure_capacity(tfcb_encoder* h, long long extra_words, cudaStream_t s) {
  const long long need = h->bound + extra_words + 32;
  if (need <= h->cap) return TFCB_OK;
  if (need >= kMaxStreamWords)
    return fail(TFCB_INVALID_ARGUMENT, "a single code stream may not exceed 2^31 16-bit words");
  const long long new_cap = (std::max(need, h->cap * 2) + 31) & ~31ll;
  uint16_t* nw = nullptr;
  uint32_t* nc = nullptr;
  const long long S = std::max<long long>(h->n_streams, 1);
  TFCB_TRY(dev_alloc((void**)&nw, (size_t)S * new_cap * sizeof(uint16_t), s));
  TFCB_TRY(dev_alloc((void**)&nc, (size_t)S * (new_cap >> 5) * sizeof(uint32_t), s));
  if (h->cap > 0 && h->bound > 0 && h->n_streams > 0) {
    enc_grow_kernel<<<(unsigned)h->n_streams, 128, 0, s>>>(h->words, h->cbits, h->cap, nw, nc, new_cap,
                                                           h->state);
    TFCB_LAUNCHED();
    TFCB_CUDA_TRY(cudaGetLastError());
  }
  dev_free(h->words, s);
  dev_free(h->cbits, s);
  h->words = nw;
  h->cbits = nc;
  h->cap = new_cap;
  h->arena_words = S * new_cap;
  return TFCB_OK;
}

// Host-side checks of a ragged batch's symbol offsets [n_streams + 1].
// Lays out a ragged batch's arena on a fresh (pooled) encoder: stream s gets its own worst case rounded to 32
// words, so the arena is the sum of the per-stream bounds rather than n_streams times the longest one.  Uploads the
// symbol and arena offsets in one copy and points the encoder at them.  The arena only grows.
int prepare_ragged(tfcb_encoder* h, const int64_t* sym_off, cudaStream_t s) {
  const long long S = h->n_streams;
  std::vector<long long> off(2 * (S + 1));
  long long* arena = off.data() + S + 1;
  long long total = 0;
  for (long long i = 0; i <= S; ++i) {
    off[i] = sym_off[i];
    arena[i] = total;
    if (i < S) total += (words_bound(h, sym_off[i + 1] - sym_off[i]) + 32 + 31) & ~31ll;
  }
  if (total > h->arena_words) {
    uint16_t* nw = nullptr;
    uint32_t* nc = nullptr;
    TFCB_TRY(dev_alloc((void**)&nw, (size_t)total * sizeof(uint16_t), s));
    const int rc = dev_alloc((void**)&nc, (size_t)(total >> 5) * sizeof(uint32_t), s);
    if (rc != TFCB_OK) {
      dev_free(nw, s);
      return rc;
    }
    dev_free(h->words, s);
    dev_free(h->cbits, s);
    h->words = nw;
    h->cbits = nc;
    h->arena_words = total;
    h->cap = (total / S) & ~31ll;  // what a later uniform batch of this pooled encoder may use of the same arena
  }
  if (!h->ext) TFCB_TRY(dev_alloc((void**)&h->ext, off.size() * sizeof(long long), s));
  // (pageable source: staged before the call returns)
  TFCB_CUDA_TRY(cudaMemcpyAsync(h->ext, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice, s));
  h->arena_off = h->ext + S + 1;
  return TFCB_OK;
}

// Value types, numbered as the C ABI's `dtype` / `loc_dtype` (int32 values have no such argument).
enum Dtype : int { kInt32 = -1, kFloat32 = 0, kFloat16 = 1, kBFloat16 = 2 };

// What one encode or decode codes, besides the values themselves: each public entry converts its own arguments into
// this, and mode_of alone reads the kernel's mode from it.
struct Operands {
  Dtype type = kInt32;             // the value's (decoder: the output's) type
  bool indexed = false;            // index mode: `index` picks each symbol's table; channel mode: its position does
  const int32_t* index = nullptr;  // [S, n]
  const void* off = nullptr;       // channel mode: quantisation offsets [n_rows]; index mode: loc [S, n]; or null
  Dtype off_type = kFloat32;       // float32, or in index mode also the value's 16-bit type
  const int32_t* cdf_offset = nullptr;  // float values: [n_rows]
  void* decoded = nullptr;         // encoder, float values: each symbol's decoded value [S, n], or null
};

// The kernels' mode for a call.  A 16-bit index-mode call with a float32 loc runs under kModeLocF32, which also makes
// its decoded values float32 (torch's type promotion); in channel mode the offsets are float32 and the mode has no
// kModeLocF32.
int mode_of(const Operands& o) {
  int mode = (o.indexed ? kModeIndex : 0) | (o.decoded ? kModeDecoded : 0);
  if (o.type == kFloat32) mode |= kModeF32;
  if (o.type == kFloat16) mode |= kModeH16;
  if (o.type == kBFloat16) mode |= kModeB16;
  if ((mode & kMode16) && o.indexed && o.off && o.off_type == kFloat32) mode |= kModeLocF32;
  return mode;
}

template <int MODE>
using Mode = std::integral_constant<int, MODE>;

// The one map from a mode_of mode to the kernels' MODE: returns fn(Mode<MODE>{}).  It lists the modes the kernels are
// compiled for: decode_kernel's 10 below, and encode_kernel's 18, those 10 and each float one with kModeDecoded.
template <bool ENCODER, class Fn>
int with_mode(int mode, Fn fn) {
  const bool decoded = mode & kModeDecoded;
  if (decoded && !(ENCODER && (mode & kModeFloat)))
    return fail(TFCB_INVALID_ARGUMENT, "decoded values need float values");
  auto with_decoded = [&](auto m) {
    if constexpr (ENCODER) {
      if (decoded) return fn(Mode<decltype(m)::value | kModeDecoded>{});
    }
    return fn(m);
  };
  switch (mode & ~kModeDecoded) {
    case 0: return fn(Mode<0>{});
    case kModeIndex: return fn(Mode<kModeIndex>{});
    case kModeF32: return with_decoded(Mode<kModeF32>{});
    case kModeIndex | kModeF32: return with_decoded(Mode<kModeIndex | kModeF32>{});
    case kModeH16: return with_decoded(Mode<kModeH16>{});
    case kModeIndex | kModeH16: return with_decoded(Mode<kModeIndex | kModeH16>{});
    case kModeIndex | kModeH16 | kModeLocF32: return with_decoded(Mode<kModeIndex | kModeH16 | kModeLocF32>{});
    case kModeB16: return with_decoded(Mode<kModeB16>{});
    case kModeIndex | kModeB16: return with_decoded(Mode<kModeIndex | kModeB16>{});
    case kModeIndex | kModeB16 | kModeLocF32: return with_decoded(Mode<kModeIndex | kModeB16 | kModeLocF32>{});
  }
  return fail(TFCB_INVALID_ARGUMENT, "no kernel for mode %d", mode);
}

// `sym_off` (device, [n_streams + 1]) non-null: a ragged batch of `n` symbols in all, laid out by prepare_ragged.
template <int MODE>
int launch_encode(tfcb_encoder* h, const void* value, const Operands& o, long long n, cudaStream_t s,
                  const long long* sym_off) {
  // 16-bit values: a loc (index mode) and the decoded output are in the value's type, unless kModeLocF32
  constexpr bool in16 = (MODE & kMode16) && !(MODE & kModeLocF32);
  constexpr bool loc16 = in16 && (MODE & kModeIndex);
  if (h->finalized) return fail(TFCB_INVALID_ARGUMENT, "encoder handle was already finalized");
  if (n < 0) return fail(TFCB_INVALID_ARGUMENT, "negative element count");
  if (h->n_streams == 0 || n == 0) return TFCB_OK;
  if (h->lut.n_rows == 0) return fail(TFCB_INVALID_ARGUMENT, "index=0 not in range [0, 0)");
  if (value == nullptr) return fail(TFCB_INVALID_ARGUMENT, "`value` is null");
  if ((MODE & kModeIndex) && o.index == nullptr) return fail(TFCB_INVALID_ARGUMENT, "`index` is null");
  if ((MODE & kModeFloat) && o.cdf_offset == nullptr) return fail(TFCB_INVALID_ARGUMENT, "`cdf_offset` is null");
  if (!sym_off) {
    const long long extra = words_bound(h, n);
    TFCB_TRY(ensure_capacity(h, extra, s));
    h->bound += extra;
  }
  EncParams P;
  P.lookup = h->lut.lookup;
  P.rows = h->lut.rows;
  P.n_rows = h->lut.n_rows;
  P.uniform_prec = h->lut.uniform_prec;
  P.value = value;
  P.index = o.index;
  P.qoff = (MODE & kModeFloat) && !loc16 ? static_cast<const float*>(o.off) : nullptr;
  P.coff = (MODE & kModeFloat) ? o.cdf_offset : nullptr;
  P.n = n;
  P.n_streams = h->n_streams;
  P.fresh = h->fresh ? 1 : 0;
  P.state = h->state;
  P.words = h->words;
  P.cbits = h->cbits;
  P.cap = h->cap;
  P.err = h->err;
  P.sym_off = sym_off;
  P.arena_off = h->arena_off;
  P.decoded = in16 ? nullptr : static_cast<float*>(o.decoded);
  P.loc16 = loc16 ? static_cast<const uint16_t*>(o.off) : nullptr;
  P.decoded16 = in16 ? static_cast<uint16_t*>(o.decoded) : nullptr;
  if (h->n_streams > 0x7FFFFFFFll) return fail(TFCB_INVALID_ARGUMENT, "too many streams");
  encode_kernel<MODE><<<(unsigned)h->n_streams, 192, 0, s>>>(P);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  h->fresh = false;
  return TFCB_OK;
}

int encode(tfcb_encoder* h, const void* value, const Operands& o, long long n, cudaStream_t s,
           const long long* sym_off = nullptr) {
  return with_mode<true>(mode_of(o),
                         [&](auto m) { return launch_encode<decltype(m)::value>(h, value, o, n, s, sym_off); });
}

// Host-mapped {total, error} per host thread: written by enc_offsets_kernel, read after the stream synchronises.
EncResult* mapped_result(EncResult** dev) {
  thread_local EncResult* host = nullptr;
  thread_local EncResult* devp = nullptr;
  if (!host) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, sizeof(EncResult), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
        cudaHostGetDevicePointer((void**)&devp, p, 0) != cudaSuccess) {
      (void)cudaGetLastError();
      if (p) cudaFreeHost(p);
      return nullptr;
    }
    host = static_cast<EncResult*>(p);
  }
  *dev = devp;
  return host;
}

// Lengths, offsets (into `offsets`), the one host round trip, then the deferred argument errors (`what` selects their
// wording, see decode_error) and the total.  `err_out`, when given, receives the raw error record instead and no
// wording is applied (callers that keep their own error keys in it).
int enc_offsets(const EncArena& a, long long* offsets, bool reset_err, const char* what, cudaStream_t s,
                long long* total, DevError* err_out = nullptr) {
  EncResult* dres = nullptr;
  EncResult* res = mapped_result(&dres);
  if (!res) return fail(TFCB_CUDA_ERROR, "could not allocate host-mapped memory for the finalize result");
  enc_offsets_kernel<<<1, 1024, 0, s>>>(a.state, a.words, a.cap, a.arena_off, a.n_streams, offsets, a.err,
                                         reset_err ? 1 : 0, dres);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  TFCB_CUDA_TRY(cudaStreamSynchronize(s));
  EncResult r;
  std::memcpy(&r, res, sizeof r);
  *total = r.total;
  if (err_out) {
    *err_out = r.err;
    return TFCB_OK;
  }
  return decode_error(r.err, what);
}

void enc_write(const EncArena& a, const long long* offsets, uint8_t* out, cudaStream_t s) {
  if (a.n_streams > 0) {
    enc_write_kernel<<<(unsigned)a.n_streams, 32 * kWriteWarps, 0, s>>>(a.state, a.words, a.cbits, a.cap,
                                                                       a.arena_off, a.n_streams, offsets, out);
    TFCB_LAUNCHED();
  }
}

}  // namespace

namespace tfcb {
namespace {
EncArena ragged_arena(long long n_streams, void* state, uint16_t* words, uint32_t* cbits, DevError* err,
                      const long long* arena_off) {
  EncArena a;
  a.n_streams = n_streams;
  a.state = static_cast<EncState*>(state);
  a.words = words;
  a.cbits = cbits;
  a.err = err;
  a.arena_off = arena_off;
  return a;
}
}  // namespace

int ragged_arena_offsets(long long n_streams, void* state, uint16_t* words, uint32_t* cbits, DevError* err,
                         const long long* arena_off, long long* offsets, cudaStream_t s, long long* total,
                         DevError* err_out) {
  return enc_offsets(ragged_arena(n_streams, state, words, cbits, err, arena_off), offsets, false, "ragged", s, total,
                     err_out);
}

void ragged_arena_write(long long n_streams, void* state, uint16_t* words, uint32_t* cbits, DevError* err,
                        const long long* arena_off, const long long* offsets, uint8_t* out, cudaStream_t s) {
  enc_write(ragged_arena(n_streams, state, words, cbits, err, arena_off), offsets, out, s);
}
}  // namespace tfcb

namespace {

// Finalize of an encoder handle up to its output size: the initial state if nothing was encoded, an arena for
// enc_write_kernel to read even then, and enc_offsets.
int finalize_encoder(tfcb_encoder* h, long long* offsets, bool reset_err, cudaStream_t s, long long* total) {
  if (h->cap == 0) TFCB_TRY(ensure_capacity(h, 0, s));
  if (h->fresh && h->n_streams > 0) {
    enc_init_state_kernel<<<(unsigned)((h->n_streams + 255) / 256), 256, 0, s>>>(h->state, h->n_streams);
    TFCB_LAUNCHED();
    TFCB_CUDA_TRY(cudaGetLastError());
  }
  h->fresh = false;
  return enc_offsets(*h, offsets, reset_err, "encode", s, total);
}

}  // namespace

extern "C" {

int tfcb_encoder_create(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols,
                        int64_t n_streams, void* stream, tfcb_encoder** out) {
  if (!out) return fail(TFCB_INVALID_ARGUMENT, "null output handle");
  *out = nullptr;
  if (n_streams < 0) return fail(TFCB_INVALID_ARGUMENT, "negative stream count");
  cudaStream_t s = as_stream(stream);
  tfcb_encoder* h = new tfcb_encoder;
  h->home = s;
  h->n_streams = n_streams;
  int rc = lookup_cache().acquire(lookup_host, lookup_len, lookup_cols, /*for_decoder=*/false, s, &h->lut, &h->lut_token);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->state, std::max<int64_t>(n_streams, 1) * sizeof(EncState), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->err, sizeof(DevError), s);
  if (rc != TFCB_OK) {
    tfcb_encoder_destroy(h);
    return rc;
  }
  // (the state is initialised by the first encode, or by finalize when nothing was encoded)
  if (cudaMemsetAsync(h->err, 0, sizeof(DevError), s) != cudaSuccess) {
    (void)cudaGetLastError();
    tfcb_encoder_destroy(h);
    return fail(TFCB_CUDA_ERROR, "encoder initialisation failed");
  }
  *out = h;
  return TFCB_OK;
}

int tfcb_encode_channel(tfcb_encoder* h, const int32_t* value_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  return encode(h, value_dev, Operands{}, n, as_stream(stream));
}

int tfcb_encode_index(tfcb_encoder* h, const int32_t* index_dev, const int32_t* value_dev, int64_t n,
                      void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  return encode(h, value_dev, Operands{kInt32, true, index_dev}, n, as_stream(stream));
}

int tfcb_encode_channel_f32(tfcb_encoder* h, const float* y_dev, const float* quant_offset_dev,
                            const int32_t* cdf_offset_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  return encode(h, y_dev, Operands{kFloat32, false, nullptr, quant_offset_dev, kFloat32, cdf_offset_dev}, n,
                as_stream(stream));
}

int tfcb_encode_index_f32(tfcb_encoder* h, const int32_t* index_dev, const float* y_dev,
                          const float* loc_dev, const int32_t* cdf_offset_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  return encode(h, y_dev, Operands{kFloat32, true, index_dev, loc_dev, kFloat32, cdf_offset_dev}, n,
                as_stream(stream));
}

int tfcb_encoder_check(tfcb_encoder* h, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  return fetch_error(h->err, as_stream(stream), "encode");
}

int tfcb_encode_finalize(tfcb_encoder* h, int64_t* offsets_dev, void* stream, int64_t* total_bytes_host) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  if (h->finalized) return fail(TFCB_INVALID_ARGUMENT, "encoder handle was already finalized");
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  long long total = 0;
  // (the error record is not reset: a finalize retried after an argument error fails again)
  TFCB_TRY(finalize_encoder(h, reinterpret_cast<long long*>(offsets_dev), /*reset_err=*/false, as_stream(stream),
                            &total));
  h->finalized = true;
  if (total_bytes_host) *total_bytes_host = total;
  return TFCB_OK;
}

int tfcb_encode_write(tfcb_encoder* h, const int64_t* offsets_dev, uint8_t* bytes_dev, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  if (!h->finalized) return fail(TFCB_INVALID_ARGUMENT, "encoder handle is not finalized");
  // (the first write frees the word arena)
  if (!h->words) return fail(TFCB_INVALID_ARGUMENT, "encoder handle was already finalized");
  cudaStream_t s = as_stream(stream);
  enc_write(*h, reinterpret_cast<const long long*>(offsets_dev), bytes_dev, s);
  TFCB_CUDA_TRY(cudaGetLastError());
  dev_free(h->words, s);
  dev_free(h->cbits, s);
  h->words = nullptr;
  h->cbits = nullptr;
  return TFCB_OK;
}

void tfcb_encoder_destroy(tfcb_encoder* h) {
  if (!h) return;
  cudaStream_t s = h->home;
  lookup_cache().release(h->lut_token);
  dev_free(h->state, s);
  dev_free(h->words, s);
  dev_free(h->cbits, s);
  dev_free(h->err, s);
  dev_free(h->ext, s);
  if (h->done) cudaEventDestroy(h->done);
  delete h;
}

}  // extern "C"

namespace {

// Idle encoders of tfcb_compress, with their state, error record and word arena: a model compresses batch after
// batch of the same shape, and a recycled encoder saves the allocations and the initialisation of each call.
struct EncoderPool {
  static constexpr size_t kMaxIdle = 4;
  std::mutex mu;
  std::vector<tfcb_encoder*> idle;

  tfcb_encoder* take(long long n_streams, int device) {
    std::lock_guard<std::mutex> lock(mu);
    for (size_t i = idle.size(); i-- > 0;) {
      if (idle[i]->n_streams == n_streams && idle[i]->device == device) {
        tfcb_encoder* h = idle[i];
        idle.erase(idle.begin() + i);
        return h;
      }
    }
    return nullptr;
  }
  void give(tfcb_encoder* h) {
    {
      std::lock_guard<std::mutex> lock(mu);
      if (idle.size() < kMaxIdle) {
        idle.push_back(h);
        return;
      }
    }
    tfcb_encoder_destroy(h);
  }
};

EncoderPool& encoder_pool() {
  static EncoderPool* p = new EncoderPool;  // leaked on purpose, like the lookup cache
  return *p;
}

// A pooled encoder reset to a fresh handle for `lookup` on stream `s`.
int checkout_encoder(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                     cudaStream_t s, tfcb_encoder** out) {
  int device = 0;
  cudaGetDevice(&device);
  tfcb_encoder* h = encoder_pool().take(n_streams, device);
  if (!h) {
    TFCB_TRY(tfcb_encoder_create(lookup_host, lookup_len, lookup_cols, n_streams, s, &h));
    h->device = device;
    if (cudaEventCreateWithFlags(&h->done, cudaEventDisableTiming) != cudaSuccess) {
      (void)cudaGetLastError();
      h->done = nullptr;
      tfcb_encoder_destroy(h);
      return fail(TFCB_CUDA_ERROR, "encoder event creation failed");
    }
    *out = h;
    return TFCB_OK;
  }
  // Same table as the previous user (the common case: one model, batch after batch): a compare with the cache
  // entry the encoder already pins is cheaper than hashing the table again.
  if (!lookup_cache().same(h->lut_token, lookup_host, lookup_len, lookup_cols)) {
    DeviceLookup lut;
    void* token = nullptr;
    const int rc =
        lookup_cache().acquire(lookup_host, lookup_len, lookup_cols, /*for_decoder=*/false, s, &lut, &token);
    if (rc != TFCB_OK) {
      encoder_pool().give(h);
      return rc;
    }
    lookup_cache().release(h->lut_token);
    h->lut = lut;
    h->lut_token = token;
  }
  // the previous user's last kernel (enc_write_kernel) may still read the arena on another stream (on the same
  // stream, stream order is enough)
  if (h->home != s && cudaStreamWaitEvent(s, h->done, 0) != cudaSuccess) {
    (void)cudaGetLastError();
    tfcb_encoder_destroy(h);
    return fail(TFCB_CUDA_ERROR, "cudaStreamWaitEvent failed");
  }
  h->home = s;
  h->bound = 0;
  h->fresh = true;
  h->finalized = false;
  h->arena_off = nullptr;
  *out = h;
  return TFCB_OK;
}

// After the encode of a checked-out encoder (`rc` its result): finalize, and the encoder either handed to the caller
// or taken back.
int finish_compress(tfcb_encoder* h, int rc, int64_t* offsets_dev, cudaStream_t s, tfcb_encoder** out,
                    int64_t* total_bytes_host) {
  long long total = 0;
  if (rc == TFCB_OK)
    rc = finalize_encoder(h, reinterpret_cast<long long*>(offsets_dev), /*reset_err=*/true, s, &total);
  if (rc != TFCB_OK) {
    // argument errors leave the encoder clean (the finalize kernel cleared the error record): keep it
    if (rc == TFCB_INVALID_ARGUMENT) encoder_pool().give(h);
    else tfcb_encoder_destroy(h);
    return rc;
  }
  *out = h;
  *total_bytes_host = total;
  return TFCB_OK;
}

// The 16-bit value types' host-side arguments, checked before any device work: `dtype` 1 float16 or 2 bfloat16;
// `loc_dtype` 0 (float32), or in index mode also `dtype`; cdf_offset always, and the value (or output) whenever
// there are symbols.
int check16(int dtype, bool index_mode, int loc_dtype, const void* data, const char* data_name,
            const int32_t* cdf_offset_dev, long long n_symbols) {
  if (dtype != 1 && dtype != 2)
    return fail(TFCB_INVALID_ARGUMENT, "`dtype` must be 1 (float16) or 2 (bfloat16): %d", dtype);
  if (loc_dtype != 0 && !(index_mode && loc_dtype == dtype))
    return fail(TFCB_INVALID_ARGUMENT, "`loc_dtype` must be 0 (float32)%s: %d",
                index_mode ? " or the value's `dtype`" : " in channel mode", loc_dtype);
  if (!cdf_offset_dev) return fail(TFCB_INVALID_ARGUMENT, "`cdf_offset` is null");
  if (n_symbols > 0 && !data) return fail(TFCB_INVALID_ARGUMENT, "`%s` is null", data_name);
  return TFCB_OK;
}

// The compress of every tfcb_compress* entry, after its argument checks: `n` symbols per stream, or with
// `sym_off_host` [n_streams + 1] non-null a ragged batch.  A ragged batch's per-stream size limit needs the table's
// worst case bits per symbol, so the table is parsed for it here, before any device work.  Then one encode on a
// pooled encoder and finish_compress.
int compress(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams, long long n,
             const int64_t* sym_off_host, const void* value, const Operands& o, int64_t* offsets_dev, void* stream,
             tfcb_encoder** out, int64_t* total_bytes_host) {
  if (sym_off_host) {
    std::vector<HostRow> rows;
    TFCB_TRY(parse_lookup(lookup_host, lookup_len, lookup_cols, &rows));
    int max_prec = 0;
    bool any_overflow = false;
    for (const HostRow& r : rows) {
      max_prec = std::max(max_prec, r.prec < 0 ? -r.prec : r.prec);
      any_overflow |= r.prec < 0;
    }
    const long long bits = bits_bound(max_prec, any_overflow);
    for (long long i = 0; i < n_streams; ++i)
      if (words_for(bits, sym_off_host[i + 1] - sym_off_host[i]) + 32 >= kMaxStreamWords)
        return fail(TFCB_INVALID_ARGUMENT, "a single code stream may not exceed 2^31 16-bit words (stream %lld)", i);
  }
  cudaStream_t s = as_stream(stream);
  tfcb_encoder* h = nullptr;
  TFCB_TRY(checkout_encoder(lookup_host, lookup_len, lookup_cols, n_streams, s, &h));
  if (sym_off_host) {
    const int rc = prepare_ragged(h, sym_off_host, s);
    if (rc != TFCB_OK) {
      tfcb_encoder_destroy(h);
      return rc;
    }
    n = sym_off_host[n_streams];
  }
  return finish_compress(h, encode(h, value, o, n, s, sym_off_host ? h->ext : nullptr), offsets_dev, s, out,
                         total_bytes_host);
}

}  // namespace

extern "C" {

int tfcb_compress(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                  const int32_t* index_dev, const void* value_dev, int32_t value_is_f32, const float* qoff_dev,
                  const int32_t* cdf_offset_dev, int64_t n, int64_t* offsets_dev, void* stream,
                  tfcb_encoder** out, int64_t* total_bytes_host) {
  if (!out || !total_bytes_host) return fail(TFCB_INVALID_ARGUMENT, "null output pointer");
  *out = nullptr;
  *total_bytes_host = 0;
  if (n_streams < 0) return fail(TFCB_INVALID_ARGUMENT, "negative stream count");
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  const Operands o{value_is_f32 ? kFloat32 : kInt32, index_dev != nullptr, index_dev, qoff_dev, kFloat32,
                   cdf_offset_dev};
  return compress(lookup_host, lookup_len, lookup_cols, n_streams, n, nullptr, value_dev, o, offsets_dev, stream, out,
                  total_bytes_host);
}

int tfcb_compress_16bit(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                        const int32_t* index_dev, const void* value_dev, int dtype, const void* loc_dev, int loc_dtype,
                        const int32_t* cdf_offset_dev, int64_t n, int64_t* offsets_dev, void* stream,
                        tfcb_encoder** out, int64_t* total_bytes_host) {
  if (!out || !total_bytes_host) return fail(TFCB_INVALID_ARGUMENT, "null output pointer");
  *out = nullptr;
  *total_bytes_host = 0;
  if (n_streams < 0) return fail(TFCB_INVALID_ARGUMENT, "negative stream count");
  if (n < 0) return fail(TFCB_INVALID_ARGUMENT, "negative element count");
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  TFCB_TRY(check16(dtype, index_dev != nullptr, loc_dtype, value_dev, "value", cdf_offset_dev, n_streams * n));
  const Operands o{Dtype(dtype), index_dev != nullptr, index_dev, loc_dev, Dtype(loc_dtype), cdf_offset_dev};
  return compress(lookup_host, lookup_len, lookup_cols, n_streams, n, nullptr, value_dev, o, offsets_dev, stream, out,
                  total_bytes_host);
}

int tfcb_compress_ragged(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                         const int64_t* symbol_offsets_host, const int32_t* index_dev, const void* value_dev,
                         int32_t value_is_f32, const float* qoff_dev, const int32_t* cdf_offset_dev,
                         int64_t* offsets_dev, void* stream, tfcb_encoder** out, int64_t* total_bytes_host) {
  if (!out || !total_bytes_host) return fail(TFCB_INVALID_ARGUMENT, "null output pointer");
  *out = nullptr;
  *total_bytes_host = 0;
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  TFCB_TRY(check_symbol_offsets(symbol_offsets_host, n_streams));
  const Operands o{value_is_f32 ? kFloat32 : kInt32, index_dev != nullptr, index_dev, qoff_dev, kFloat32,
                   cdf_offset_dev};
  return compress(lookup_host, lookup_len, lookup_cols, n_streams, 0, symbol_offsets_host, value_dev, o, offsets_dev,
                  stream, out, total_bytes_host);
}

int tfcb_compress_ragged_decoded(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols,
                                 int64_t n_streams, const int64_t* symbol_offsets_host, const int32_t* index_dev,
                                 const void* value_dev, int32_t value_is_f32, const float* qoff_dev,
                                 const int32_t* cdf_offset_dev, int64_t* offsets_dev, void* stream,
                                 tfcb_encoder** out, int64_t* total_bytes_host, float* decoded_dev) {
  if (out) *out = nullptr;
  if (total_bytes_host) *total_bytes_host = 0;
  if (!value_is_f32) return fail(TFCB_INVALID_ARGUMENT, "decoded values need float32 values (`value_is_f32` is 0)");
  if (!decoded_dev) return fail(TFCB_INVALID_ARGUMENT, "`decoded` is null");
  if (!cdf_offset_dev) return fail(TFCB_INVALID_ARGUMENT, "`cdf_offset` is null");
  if (!out || !total_bytes_host) return fail(TFCB_INVALID_ARGUMENT, "null output pointer");
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  TFCB_TRY(check_symbol_offsets(symbol_offsets_host, n_streams));
  const Operands o{kFloat32, index_dev != nullptr, index_dev, qoff_dev, kFloat32, cdf_offset_dev, decoded_dev};
  return compress(lookup_host, lookup_len, lookup_cols, n_streams, 0, symbol_offsets_host, value_dev, o, offsets_dev,
                  stream, out, total_bytes_host);
}

int tfcb_compress_ragged_16bit(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                               const int64_t* symbol_offsets_host, const int32_t* index_dev, const void* value_dev,
                               int dtype, const void* loc_dev, int loc_dtype, const int32_t* cdf_offset_dev,
                               void* decoded_dev, int64_t* offsets_dev, void* stream, tfcb_encoder** out,
                               int64_t* total_bytes_host) {
  if (out) *out = nullptr;
  if (total_bytes_host) *total_bytes_host = 0;
  TFCB_TRY(check_symbol_offsets(symbol_offsets_host, n_streams));
  TFCB_TRY(check16(dtype, index_dev != nullptr, loc_dtype, value_dev, "value", cdf_offset_dev,
                   symbol_offsets_host[n_streams]));
  if (!out || !total_bytes_host) return fail(TFCB_INVALID_ARGUMENT, "null output pointer");
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  const Operands o{Dtype(dtype), index_dev != nullptr, index_dev, loc_dev, Dtype(loc_dtype), cdf_offset_dev,
                   decoded_dev};
  return compress(lookup_host, lookup_len, lookup_cols, n_streams, 0, symbol_offsets_host, value_dev, o, offsets_dev,
                  stream, out, total_bytes_host);
}

int tfcb_compress_write(tfcb_encoder* h, const int64_t* offsets_dev, uint8_t* bytes_dev, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not an encoder");
  cudaStream_t s = as_stream(stream);
  enc_write(*h, reinterpret_cast<const long long*>(offsets_dev), bytes_dev, s);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || cudaEventRecord(h->done, s) != cudaSuccess) {
    (void)cudaGetLastError();
    tfcb_encoder_destroy(h);
    return fail(TFCB_CUDA_ERROR, "enc_write_kernel launch failed: %s", cudaGetErrorString(e));
  }
  encoder_pool().give(h);
  return TFCB_OK;
}

}  // extern "C"

struct tfcb_decoder {
  DeviceLookup lut;      // shallow copy of a cache entry's tables
  void* lut_token = nullptr;
  long long n_streams = 0;
  const uint8_t* bytes = nullptr;
  const long long* offsets = nullptr;
  DecState* state = nullptr;
  DevError* err = nullptr;
  uint8_t* ok = nullptr;
  cudaStream_t home = nullptr;
  long long* sym_off = nullptr;  // ragged decodes: device copy of the symbol offsets [n_streams + 1]
};

int tfcb::decoder_view(tfcb_decoder* h, DecoderView* v) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  v->rows = h->lut.rows;
  v->pairs = h->lut.pairs;
  v->rows4 = h->lut.rows4;
  v->n_rows = h->lut.n_rows;
  v->n_pairs = h->lut.n_pairs;
  v->bytes = h->bytes;
  v->offsets = h->offsets;
  v->n_streams = h->n_streams;
  v->state = h->state;
  v->err = h->err;
  return TFCB_OK;
}

namespace {

// `sym_off` (device, [n_streams + 1]) non-null: a ragged batch of `n` symbols in all.
template <int MODE>
int launch_decode(tfcb_decoder* h, void* out, const Operands& o, long long n, cudaStream_t s,
                  const long long* sym_off) {
  // 16-bit index modes: the loc is in the output's type, unless kModeLocF32
  constexpr bool loc16 = (MODE & kMode16) && (MODE & kModeIndex) && !(MODE & kModeLocF32);
  if (n < 0) return fail(TFCB_INVALID_ARGUMENT, "negative element count");
  if (h->n_streams == 0 || n == 0) return TFCB_OK;
  if (h->lut.n_rows == 0) return fail(TFCB_INVALID_ARGUMENT, "index=0 not in range [0, 0)");
  if (out == nullptr) return fail(TFCB_INVALID_ARGUMENT, "output is null");
  if ((MODE & kModeIndex) && o.index == nullptr) return fail(TFCB_INVALID_ARGUMENT, "`index` is null");
  if ((MODE & kModeFloat) && o.cdf_offset == nullptr) return fail(TFCB_INVALID_ARGUMENT, "`cdf_offset` is null");
  DecParams P;
  P.lookup = h->lut.lookup;
  P.rows = h->lut.rows;
  P.pairs = h->lut.pairs;
  P.rows4 = h->lut.rows4;
  P.n_pairs = h->lut.n_pairs;
  P.zero_win = h->lut.zero_win;
  P.n_rows = h->lut.n_rows;
  P.lookup_len = h->lut.len;
  P.bytes = h->bytes;
  P.offsets = h->offsets;
  P.index = o.index;
  P.out = out;
  P.qoff = (MODE & kModeFloat) && !loc16 ? static_cast<const float*>(o.off) : nullptr;
  P.coff = (MODE & kModeFloat) ? o.cdf_offset : nullptr;
  P.n = n;
  P.n_streams = h->n_streams;
  P.state = h->state;
  P.err = h->err;
  P.sym_off = sym_off;
  P.loc16 = loc16 ? static_cast<const uint16_t*>(o.off) : nullptr;
  // Search keys live in shared memory whenever they fit beside the kernel's static 16 KB: up to 96 KB two CTAs
  // (streams) still share an SM; up to 200 KB one CTA per SM (cfg3's 64 NoisyNormal tables up to sigma = 256 take
  // 118 KB: from L1/L2 every slow-path search round cost a global-memory latency on the chain warp).
  const size_t smem = (size_t)((h->lut.n_pairs * 8 + 15) & ~15ll) + (size_t)h->lut.n_rows * sizeof(int4);
  if (smem <= 200 * 1024) {
    TFCB_CUDA_TRY(cudaFuncSetAttribute(decode_kernel<MODE, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    decode_kernel<MODE, true><<<(unsigned)h->n_streams, 96, smem, s>>>(P);
  } else {
    decode_kernel<MODE, false><<<(unsigned)h->n_streams, 96, 0, s>>>(P);
  }
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// A ragged decode's symbol offsets, checked and copied to the decoder (`*n`: the symbols in all; nothing is copied
// when there are none).
int upload_symbol_offsets(tfcb_decoder* h, const int64_t* symbol_offsets_host, cudaStream_t s, long long* n) {
  TFCB_TRY(check_symbol_offsets(symbol_offsets_host, h->n_streams));
  *n = symbol_offsets_host[h->n_streams];
  if (*n == 0) return TFCB_OK;
  if (!h->sym_off) TFCB_TRY(dev_alloc((void**)&h->sym_off, (h->n_streams + 1) * sizeof(long long), s));
  // (pageable source: staged before the call returns; an earlier decode on this stream has read the old offsets)
  TFCB_CUDA_TRY(cudaMemcpyAsync(h->sym_off, symbol_offsets_host, (h->n_streams + 1) * sizeof(long long),
                                cudaMemcpyHostToDevice, s));
  return TFCB_OK;
}

// The decode of every tfcb_decode_* entry, after its argument checks: `n` symbols per stream, or with `sym_off_host`
// [n_streams + 1] non-null a ragged batch.
int decode(tfcb_decoder* h, long long n, const int64_t* sym_off_host, void* out, const Operands& o, cudaStream_t s) {
  if (sym_off_host) TFCB_TRY(upload_symbol_offsets(h, sym_off_host, s, &n));
  return with_mode<false>(mode_of(o), [&](auto m) {
    return launch_decode<decltype(m)::value>(h, out, o, n, s, sym_off_host ? h->sym_off : nullptr);
  });
}

}  // namespace

extern "C" {

int tfcb_decoder_create(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_streams,
                        const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols,
                        void* stream, tfcb_decoder** out) {
  if (!out) return fail(TFCB_INVALID_ARGUMENT, "null output handle");
  *out = nullptr;
  if (n_streams <= 0) return fail(TFCB_INVALID_ARGUMENT, "`encoded` is empty");
  if (!offsets_dev) return fail(TFCB_INVALID_ARGUMENT, "`offsets` is null");
  cudaStream_t s = as_stream(stream);
  tfcb_decoder* h = new tfcb_decoder;
  h->home = s;
  h->n_streams = n_streams;
  h->bytes = bytes_dev;
  h->offsets = reinterpret_cast<const long long*>(offsets_dev);
  int rc = lookup_cache().acquire(lookup_host, lookup_len, lookup_cols, /*for_decoder=*/true, s, &h->lut, &h->lut_token);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->state, n_streams * sizeof(DecState), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->ok, n_streams, s);
  if (rc != TFCB_OK) {
    tfcb_decoder_destroy(h);
    return rc;
  }
  cudaMemsetAsync(h->err, 0, sizeof(DevError), s);
  dec_init_state_kernel<<<(unsigned)((n_streams + 255) / 256), 256, 0, s>>>(h->state, n_streams);
  TFCB_LAUNCHED();
  if (cudaGetLastError() != cudaSuccess) {
    tfcb_decoder_destroy(h);
    return fail(TFCB_CUDA_ERROR, "decoder state initialisation failed");
  }
  *out = h;
  return TFCB_OK;
}

int tfcb_decode_channel(tfcb_decoder* h, int32_t* out_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  return decode(h, n, nullptr, out_dev, Operands{}, as_stream(stream));
}

int tfcb_decode_index(tfcb_decoder* h, const int32_t* index_dev, int32_t* out_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  return decode(h, n, nullptr, out_dev, Operands{kInt32, true, index_dev}, as_stream(stream));
}

int tfcb_decode_channel_f32(tfcb_decoder* h, float* out_dev, const float* quant_offset_dev,
                            const int32_t* cdf_offset_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  return decode(h, n, nullptr, out_dev, Operands{kFloat32, false, nullptr, quant_offset_dev, kFloat32, cdf_offset_dev},
                as_stream(stream));
}

int tfcb_decode_index_f32(tfcb_decoder* h, const int32_t* index_dev, float* out_dev, const float* loc_dev,
                          const int32_t* cdf_offset_dev, int64_t n, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  return decode(h, n, nullptr, out_dev, Operands{kFloat32, true, index_dev, loc_dev, kFloat32, cdf_offset_dev},
                as_stream(stream));
}

int tfcb_decode_ragged(tfcb_decoder* h, const int64_t* symbol_offsets_host, const int32_t* index_dev, void* out_dev,
                       int32_t out_is_f32, const float* quant_offset_dev, const int32_t* cdf_offset_dev,
                       void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  const Operands o{out_is_f32 ? kFloat32 : kInt32, index_dev != nullptr, index_dev, quant_offset_dev, kFloat32,
                   cdf_offset_dev};
  return decode(h, 0, symbol_offsets_host, out_dev, o, as_stream(stream));
}

int tfcb_decode_16bit(tfcb_decoder* h, const int32_t* index_dev, void* out_dev, int dtype, const void* loc_dev,
                      int loc_dtype, const int32_t* cdf_offset_dev, int64_t n_per_stream, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  if (n_per_stream < 0) return fail(TFCB_INVALID_ARGUMENT, "negative element count");
  TFCB_TRY(check16(dtype, index_dev != nullptr, loc_dtype, out_dev, "out", cdf_offset_dev, h->n_streams * n_per_stream));
  const Operands o{Dtype(dtype), index_dev != nullptr, index_dev, loc_dev, Dtype(loc_dtype), cdf_offset_dev};
  return decode(h, n_per_stream, nullptr, out_dev, o, as_stream(stream));
}

int tfcb_decode_ragged_16bit(tfcb_decoder* h, const int64_t* symbol_offsets_host, const int32_t* index_dev,
                             void* out_dev, int dtype, const void* loc_dev, int loc_dtype,
                             const int32_t* cdf_offset_dev, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  TFCB_TRY(check_symbol_offsets(symbol_offsets_host, h->n_streams));
  TFCB_TRY(check16(dtype, index_dev != nullptr, loc_dtype, out_dev, "out", cdf_offset_dev,
                   symbol_offsets_host[h->n_streams]));
  const Operands o{Dtype(dtype), index_dev != nullptr, index_dev, loc_dev, Dtype(loc_dtype), cdf_offset_dev};
  return decode(h, 0, symbol_offsets_host, out_dev, o, as_stream(stream));
}

int tfcb_decode_finalize(tfcb_decoder* h, uint8_t* ok_host, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "'handle' is not a decoder");
  cudaStream_t s = as_stream(stream);
  TFCB_TRY(fetch_error(h->err, s, "decode"));
  dec_finalize_kernel<<<(unsigned)((h->n_streams + 127) / 128), 128, 0, s>>>(h->state, h->bytes, h->offsets,
                                                                             h->n_streams, h->ok);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  if (ok_host) TFCB_CUDA_TRY(cudaMemcpyAsync(ok_host, h->ok, h->n_streams, cudaMemcpyDeviceToHost, s));
  TFCB_CUDA_TRY(cudaStreamSynchronize(s));
  return TFCB_OK;
}

void tfcb_decoder_destroy(tfcb_decoder* h) {
  if (!h) return;
  cudaStream_t s = h->home;
  lookup_cache().release(h->lut_token);
  dev_free(h->state, s);
  dev_free(h->err, s);
  dev_free(h->ok, s);
  dev_free(h->sym_off, s);
  delete h;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// Legacy ops: host side
// ---------------------------------------------------------------------------------------------
namespace {

// MergeAxes of range_coding_kernels_util.cc:34-91 plus the argument checks of
// range_coding_kernels.cc:134-148,179-185.
int legacy_prepare(const int64_t* dshape, int rank, const int64_t* cshape, int crank, int precision,
                   int debug_level, LegacyDims* dims, long long* n_elems, long long* n_rows) {
  if (!(0 < precision && precision <= 16))
    return fail(TFCB_INVALID_ARGUMENT, "`precision` must be in [1, 16]: %d", precision);
  if (!(debug_level == 0 || debug_level == 1))
    return fail(TFCB_INVALID_ARGUMENT, "`debug_level` must be 0 or 1: %d", debug_level);
  if (rank < 0 || crank != rank + 1)
    return fail(TFCB_INVALID_ARGUMENT, "`cdf` should have one more axis than `data`: data rank=%d, cdf rank=%d",
                rank, crank);
  if (cshape[rank] <= 1)
    return fail(TFCB_INVALID_ARGUMENT, "The last dimension of `cdf` should be > 1: %lld",
                (long long)cshape[rank]);
  if (debug_level > 0 && cshape[rank] <= 2)
    return fail(TFCB_INVALID_ARGUMENT, "CDF size should be > 2: %lld", (long long)cshape[rank]);
  std::vector<long long> md(1, 1), mc(1, 1);
  long long n = 1, rows = 1;
  for (int j = 0; j < rank; ++j) {
    if (dshape[j] < 0) return fail(TFCB_INVALID_ARGUMENT, "negative dimension");
    if (dshape[j] != cshape[j] && cshape[j] != 1)
      return fail(TFCB_INVALID_ARGUMENT, "Cannot broadcast shape of `cdf` to the shape of `data` at axis %d (%lld vs %lld)",
                  j, (long long)cshape[j], (long long)dshape[j]);
    const bool was_b = mc.back() == 1, is_b = cshape[j] == 1;
    if (was_b == is_b || dshape[j] <= 1 || md.back() <= 1) {
      md.back() *= dshape[j];
      mc.back() *= cshape[j];
    } else {
      md.push_back(dshape[j]);
      mc.push_back(cshape[j]);
    }
    n *= dshape[j];
    rows *= cshape[j];
  }
  if (md.size() > 6)
    return fail(TFCB_INVALID_ARGUMENT, "Irregular broadcast pattern: more than 6 merged axis groups");
  dims->rank = (int)md.size();
  for (int i = 0; i < 6; ++i) {
    dims->data[i] = i < dims->rank ? md[i] : 1;
    dims->cdfd[i] = i < dims->rank ? mc[i] : 1;
  }
  dims->chip = cshape[rank];
  *n_elems = n;
  *n_rows = rows;
  return TFCB_OK;
}

}  // namespace

extern "C" {

int tfcb_range_encode(const int16_t* data_dev, const int64_t* data_shape_host, int rank,
                      const int32_t* cdf_dev, const int64_t* cdf_shape_host, int cdf_rank, int precision,
                      int debug_level, uint8_t* out_host, int64_t out_cap, int64_t* n_bytes_host,
                      void* stream) {
  cudaStream_t s = as_stream(stream);
  LegacyDims dims;
  long long n = 0, rows = 0;
  TFCB_TRY(legacy_prepare(data_shape_host, rank, cdf_shape_host, cdf_rank, precision, debug_level, &dims,
                          &n, &rows));
  EncArena a;
  a.n_streams = 1;
  a.cap = (((n * precision + 15) / 16 + 2 + 32) + 31) & ~31ll;
  if (a.cap >= (1ll << 31) - 64) return fail(TFCB_INVALID_ARGUMENT, "input too large for one code stream");
  long long* offsets = nullptr;
  uint8_t* out = nullptr;
  int rc = dev_alloc((void**)&a.state, sizeof(EncState), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&a.words, a.cap * sizeof(uint16_t), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&a.cbits, (a.cap >> 5) * sizeof(uint32_t), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&a.err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&offsets, 2 * sizeof(long long), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&out, (size_t)(2 * a.cap + 8), s);
  auto cleanup = [&]() {
    dev_free(a.state, s);
    dev_free(a.words, s);
    dev_free(a.cbits, s);
    dev_free(a.err, s);
    dev_free(offsets, s);
    dev_free(out, s);
  };
  if (rc != TFCB_OK) {
    cleanup();
    return rc;
  }
  cudaMemsetAsync(a.err, 0, sizeof(DevError), s);
  if (debug_level > 0 && rows > 0) {
    legacy_check_cdf_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, s>>>(cdf_dev, rows, dims.chip,
                                                                          precision, a.err);
    TFCB_LAUNCHED();
    rc = fetch_error(a.err, s, "legacy");
    if (rc != TFCB_OK) {
      cleanup();
      return rc;
    }
  }
  legacy_encode_kernel<<<1, 32, 0, s>>>(data_dev, n, cdf_dev, dims, precision, debug_level, a.state, a.words,
                                        a.cbits, a.cap, a.err);
  TFCB_LAUNCHED();
  long long total = 0;
  rc = enc_offsets(a, offsets, /*reset_err=*/false, "legacy", s, &total);
  if (rc == TFCB_OK) {
    if (n_bytes_host) *n_bytes_host = total;
    if (total > out_cap) rc = fail(TFCB_INVALID_ARGUMENT, "output buffer too small: need %lld bytes", total);
  }
  if (rc == TFCB_OK) {
    enc_write(a, offsets, out, s);
    if (total > 0) cudaMemcpyAsync(out_host, out, (size_t)total, cudaMemcpyDeviceToHost, s);
    const cudaError_t e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = fail(TFCB_CUDA_ERROR, "CUDA error '%s' in tfcb_range_encode", cudaGetErrorString(e));
  }
  cleanup();
  return rc;
}

int tfcb_range_decode(const uint8_t* encoded_host, int64_t n_bytes, const int64_t* shape_host, int rank,
                      const int32_t* cdf_dev, const int64_t* cdf_shape_host, int cdf_rank, int precision,
                      int debug_level, int16_t* out_dev, void* stream) {
  cudaStream_t s = as_stream(stream);
  LegacyDims dims;
  long long n = 0, rows = 0;
  TFCB_TRY(legacy_prepare(shape_host, rank, cdf_shape_host, cdf_rank, precision, debug_level, &dims, &n, &rows));
  if (n_bytes < 0) return fail(TFCB_INVALID_ARGUMENT, "negative string length");
  uint8_t* bytes = nullptr;
  DevError* err = nullptr;
  int rc = dev_alloc((void**)&bytes, (size_t)std::max<int64_t>(n_bytes, 1), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&err, sizeof(DevError), s);
  auto cleanup = [&]() {
    dev_free(bytes, s);
    dev_free(err, s);
  };
  if (rc != TFCB_OK) {
    cleanup();
    return rc;
  }
  cudaMemsetAsync(err, 0, sizeof(DevError), s);
  if (n_bytes > 0) cudaMemcpyAsync(bytes, encoded_host, (size_t)n_bytes, cudaMemcpyHostToDevice, s);
  if (debug_level > 0 && rows > 0) {
    legacy_check_cdf_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, s>>>(cdf_dev, rows, dims.chip,
                                                                          precision, err);
    TFCB_LAUNCHED();
    rc = fetch_error(err, s, "legacy");
    if (rc != TFCB_OK) {
      cleanup();
      return rc;
    }
  }
  if (n > 0) {
    legacy_decode_kernel<<<1, 32, 0, s>>>(bytes, n_bytes, n, cdf_dev, dims, precision, out_dev);
    TFCB_LAUNCHED();
  }
  cudaError_t e = cudaStreamSynchronize(s);
  cleanup();
  if (e != cudaSuccess) return fail(TFCB_CUDA_ERROR, "CUDA error '%s' in tfcb_range_decode", cudaGetErrorString(e));
  return TFCB_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// UnboundedIndexRangeEncode / UnboundedIndexRangeDecode (range_coding_ops.cc:126-247,
// unbounded_index_range_coding_kernels.cc), one warp per string over a ragged batch of strings.
//
// Element i of a string codes d = data[i] - offset[r] (r = index[i], m = cdf_size[r] - 2) with row r when
// 0 <= d < m, else the escape bin m followed by u = -2d - 1 (d < 0) or 2(d - m) (d >= m) as a run of
// widths = ceil(bitlen(u) / w) in w-bit symbols (runs of M = 2^w - 1, then the remainder) and the widths w-bit digits
// of u, least significant first.  The reference computes d, u and widths in signed 32-bit arithmetic and is undefined
// for d <= -2^30, d - m >= 2^30 and u >= 2^(w * floor(31 / w)); here d and u wrap as uint32 and widths comes from
// clz, which equals the reference wherever it is defined and extends the op to every int32 (DESIGN.md §3.8).
// ---------------------------------------------------------------------------------------------
namespace tfcb {
namespace {

// Error keys kept in a DevError with atomicMin, so that the lowest one wins whatever the schedule:
//   .stream  element key  g << 3 | kind   (g = element index over the whole batch: ordered by string, then element)
//   .pos     row key      r (cdf_size out of [3, W]), or 2^62 | r << 1 | (0: start / end, 1: not monotonic)
//   .value   the lowest element whose index is outside [0, R) (debug check only)
// All three start at ~0.  .code stays 0 unless the arena bound were ever exceeded (kErrCapacity).
enum : int { kUbiIndex = 1, kUbiCdfSize = 2, kUbiInterval = 3, kUbiPrefix = 4 };
constexpr unsigned long long kUbiNone = ~0ull;
constexpr unsigned long long kUbiCdfKey = 1ull << 62;

struct UbiParams {
  const int32_t* data;      // encoder: [elements]
  int32_t* out;             // decoder: [elements]
  const int32_t* index;     // [elements]
  const int32_t* cdf;       // [R, W]
  const int32_t* cdf_size;  // [R]
  const int32_t* offset;    // [R]
  long long R, W;
  int precision, width;
  const long long* elem_off;   // [strings + 1]: string s is elements [elem_off[s], elem_off[s + 1])
  const long long* arena_off;  // encoder: [strings + 1], words of string s (multiples of 32)
  EncState* state;
  uint16_t* words;
  uint32_t* cbits;
  const uint8_t* bytes;        // decoder: string s is bytes [str_off[s], str_off[s + 1])
  const long long* str_off;
  DevError* err;
};

// Row of element g, or -1 after recording why it cannot be coded.  Checked whatever debug_level is: an index or a
// cdf_size outside its range would make the kernels read outside `cdf`.
__device__ __forceinline__ int ubi_row(const UbiParams& P, long long g) {
  const int r = P.index[g];
  if (r < 0 || r >= P.R) {
    ubi_key(&P.err->stream, ((unsigned long long)g << 3) | kUbiIndex);
    return -1;
  }
  const int sz = P.cdf_size[r];
  if (sz < 3 || sz > P.W) {
    ubi_key(&P.err->stream, ((unsigned long long)g << 3) | kUbiCdfSize);
    return -1;
  }
  return r;
}

// debug_level 1: CheckIndex, CheckCdfSize and CheckCdf of the reference over the whole tensors, each row against its
// own cdf_size prefix; the keys order the failures the way the reference's sequential checks would meet them.
__global__ void ubi_check_kernel(const int32_t* index, long long n, const int32_t* cdf, const int32_t* cdf_size,
                                 long long R, long long W, int precision, DevError* err) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (long long i = t; i < n; i += stride) {
    const int r = index[i];
    if (r < 0 || r >= R) ubi_key(&err->value, (unsigned long long)i);
  }
  const int32_t top = 1 << precision;
  for (long long r = t; r < R; r += stride) {
    const int sz = cdf_size[r];
    if (sz < 3 || sz > W) {
      ubi_key(&err->pos, (unsigned long long)r);
      continue;
    }
    const int32_t* row = cdf + r * W;
    if (row[0] != 0 || row[sz - 1] != top) {
      ubi_key(&err->pos, kUbiCdfKey | ((unsigned long long)r << 1));
      continue;
    }
    for (int j = 0; j + 1 < sz; ++j) {
      if (row[j + 1] <= row[j]) {
        ubi_key(&err->pos, kUbiCdfKey | ((unsigned long long)r << 1) | 1ull);
        break;
      }
    }
  }
}

// One warp per string.  Lanes map 32 elements at a time; then every lane runs the same recurrence over the
// elements' records in order (main symbol at precision p, width prefix and digits at precision w), lane j keeping
// entry j of the current 32, and EncDrain turns each full set of 32 entries into words, as legacy_encode_kernel does.
__global__ void __launch_bounds__(32) ubi_encode_kernel(const UbiParams P) {
  __shared__ __align__(8) uint2 s_ent[32];
  const int lane = threadIdx.x;
  const long long s = blockIdx.x;
  const Extent e = stream_extent(P.elem_off, s, 0);
  const Extent a = stream_extent(P.arena_off, s, 0);
  const EncState st0 = enc_initial_state();
  EncChain c;
  c.s = st0.raw;
  EncDrain d;
  d.begin(st0, P.words + a.base, P.cbits + (a.base >> 5), (uint32_t)a.len, lane);
  const uint32_t p = (uint32_t)P.precision, w = (uint32_t)P.width, M = (1u << w) - 1u;
  uint2 mine = make_uint2(0u, 0u);
  int fill = 0;
  auto push = [&](uint32_t lo, uint32_t hi, uint32_t prec) {
    const uint2 ent = c.step(enc_operands(lo, hi, prec));
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
    uint32_t lower = 0, upper = 1, u = 0;
    int esc = 0;
    bool bad = false;
    if (lane < count) {
      const long long g = e.base + g0 + lane;
      const int r = ubi_row(P, g);
      if (r < 0) {
        bad = true;
      } else {
        const uint32_t m = (uint32_t)(P.cdf_size[r] - 2);
        const uint32_t du = (uint32_t)P.data[g] - (uint32_t)P.offset[r];
        const int32_t dd = (int32_t)du;
        uint32_t v = du;
        if (dd < 0) {
          u = 0u - 2u * du - 1u;
          v = m;
        } else if (du >= m) {
          u = 2u * (du - m);
          v = m;
        }
        esc = v == m;
        const int32_t* row = P.cdf + r * P.W;
        lower = (uint32_t)row[v];
        upper = (uint32_t)row[v + 1];
        if (!(lower < upper) || upper > (1u << p)) {  // an empty interval: the reference's output is garbage
          ubi_key(&P.err->stream, ((unsigned long long)g << 3) | kUbiInterval);
          bad = true;
        }
      }
    }
    if (__ballot_sync(kFull, bad)) break;
    for (int k = 0; k < count; ++k) {
      push(__shfl_sync(kFull, lower, k), __shfl_sync(kFull, upper, k), p);
      if (__shfl_sync(kFull, esc, k)) {
        const uint32_t uk = __shfl_sync(kFull, u, k);
        const uint32_t widths = (32u - __clz(uk) + w - 1u) / w;  // __clz(0) = 32: no digits
        uint32_t val = widths;
        for (; val >= M; val -= M) push(M, M + 1u, w);
        push(val, val + 1u, w);
        for (uint32_t j = 0; j < widths; ++j) {  // j * w < bitlen(u) <= 32
          const uint32_t digit = (uk >> (j * w)) & M;
          push(digit, digit + 1u, w);
        }
      }
    }
  }
  if (fill) {
    s_ent[lane] = mine;
    __syncwarp();
    d.drain<1>(s_ent, fill);
    __syncwarp();
  }
  d.end(P.err, s);
  if (lane == 0) {
    EncState st;
    st.base = d.dbase;
    st.span = (c.s < 65536u) ? ((c.s << 16) | 0xFFFFu) : c.s;
    st.cnt = d.cnt;
    st.raw = c.s;
    P.state[s] = st;
  }
}

// One warp per string, legacy_decode_kernel's chain.  The width prefix stops once its running total exceeds
// K = ceil(32 / w), the most any encoder writes: every symbol then takes at most 2K + 2 decode steps, on any bytes.
__global__ void __launch_bounds__(32) ubi_decode_kernel(const UbiParams P) {
  const int lane = threadIdx.x;
  const long long s = blockIdx.x;
  const Extent e = stream_extent(P.elem_off, s, 0);
  const Extent b = stream_extent(P.str_off, s, 0);
  DecChain c;
  c.base = 0;
  c.span = 0xFFFFFFFFu;
  ByteWindow win;
  win.p = P.bytes + b.base;
  win.len = b.len;
  c.value = (bw_fetch(win, 0) << 16) | bw_fetch(win, 1);
  c.pos = 2;
  bw_seek(win, c.pos, lane);
  const uint32_t p = (uint32_t)P.precision, w = (uint32_t)P.width, M = (1u << w) - 1u;
  const uint32_t K = (32u + w - 1u) / w;
  for (long long g0 = 0; g0 < e.len; g0 += 32) {
    const int count = (int)min(32ll, e.len - g0);
    int r = 0, m = 0, off = 0;
    bool bad = false;
    if (lane < count) {
      r = ubi_row(P, e.base + g0 + lane);
      if (r < 0) {
        bad = true;
      } else {
        m = P.cdf_size[r] - 2;
        off = P.offset[r];
      }
    }
    if (__ballot_sync(kFull, bad)) return;
    int32_t my_val = 0;
    int done = count;
    for (int k = 0; k < count; ++k) {
      const int rk = __shfl_sync(kFull, r, k);
      const int mk = __shfl_sync(kFull, m, k);
      const int sym = dec_symbol(c, win, P.cdf + rk * P.W, mk + 2, p, lane);
      uint32_t v = (uint32_t)sym;
      if (sym == mk) {
        uint32_t widths = 0, val;
        bool over = false;
        do {
          val = ubi_dec_uniform(c, win, w, lane);
          widths += val;
          if (widths > K) {
            over = true;
            break;
          }
        } while (val == M);
        if (over) {
          if (lane == 0) ubi_key(&P.err->stream, ((unsigned long long)(e.base + g0 + k) << 3) | kUbiPrefix);
          done = k;
          break;
        }
        uint32_t u = 0;
        for (uint32_t j = 0; j < widths; ++j) u |= ubi_dec_uniform(c, win, w, lane) << (j * w);
        v = u >> 1;
        v = (u & 1u) ? 0u - v - 1u : v + (uint32_t)mk;
      }
      v += (uint32_t)__shfl_sync(kFull, off, k);
      if (lane == k) my_val = (int32_t)v;
    }
    if (lane < done) P.out[e.base + g0 + lane] = my_val;
    if (done < count) return;
  }
}

// ---- host side ----
int ubi_check_attrs(int precision, int overflow_width, int debug_level) {
  if (!(0 < precision && precision <= 16))
    return fail(TFCB_INVALID_ARGUMENT, "`precision` must be in [1, 16]: %d", precision);
  if (!(0 < overflow_width && overflow_width <= 16))
    return fail(TFCB_INVALID_ARGUMENT, "`overflow_width` must be in [1, 16]: %d", overflow_width);
  if (!(debug_level == 0 || debug_level == 1))
    return fail(TFCB_INVALID_ARGUMENT, "`debug_level` must be 0 or 1: %d", debug_level);
  return TFCB_OK;
}

// CheckArgumentShapes of the reference on the host shapes, then the batch offsets and pointers.
int ubi_check_args(const int64_t* cdf_shape, int cdf_rank, int64_t cdf_size_len, int64_t offset_len,
                   int64_t n_items, const int64_t* item_offsets, const void* index, const void* cdf,
                   const void* cdf_size, const void* offset) {
  if (cdf_rank != 2 || !cdf_shape || cdf_shape[1] < 3 || cdf_shape[0] < 0)
    return fail(TFCB_INVALID_ARGUMENT, "'cdf' should be 2-D and cdf.dim_size(1) >= 3: rank %d", cdf_rank);
  if (cdf_size_len != cdf_shape[0])
    return fail(TFCB_INVALID_ARGUMENT,
                "'cdf_size' should be 1-D and its length should match the number of rows in 'cdf': [%lld]",
                (long long)cdf_size_len);
  if (offset_len != cdf_shape[0])
    return fail(TFCB_INVALID_ARGUMENT,
                "'offset' should be 1-D and its length should match the number of rows in 'cdf': offset.shape=[%lld], "
                "cdf.shape=[%lld,%lld]",
                (long long)offset_len, (long long)cdf_shape[0], (long long)cdf_shape[1]);
  if (cdf_shape[0] >= (1ll << 31) || cdf_shape[0] * cdf_shape[1] >= (1ll << 40))
    return fail(TFCB_INVALID_ARGUMENT, "'cdf' too large");
  if (n_items >= (1ll << 31)) return fail(TFCB_INVALID_ARGUMENT, "too many strings: %lld", (long long)n_items);
  TFCB_TRY(check_symbol_offsets(item_offsets, n_items));
  // (debug_level 1 reads every row even when there are no elements)
  if ((item_offsets[n_items] > 0 && !index) || (cdf_shape[0] > 0 && (!cdf || !cdf_size || !offset)))
    return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  return TFCB_OK;
}

// Worst-case bits per element: p for the main symbol, and for an escape floor(K / M) + 1 prefix symbols and K digits
// of w bits each (K = ceil(32 / w)): 65 + p at w = 1, 33 + p at w = 16.  Every Encode at precision q consumes at most
// q bits (see bits_bound).
long long ubi_bits_bound(int precision, int w) {
  const long long K = (32 + w - 1) / w, M = (1ll << w) - 1;
  return precision + (long long)w * (K / M + 1 + K);
}

// Reads what the messages name from the device (error path only) and returns the first failure in the order the
// reference would meet it.
int ubi_error(const DevError& e, int debug_level, const int64_t* item_offsets, int64_t n_items, const int32_t* index,
              const int32_t* cdf, const int32_t* cdf_size, long long R, long long W, int precision, int overflow_width,
              cudaStream_t s) {
  if (e.code == kErrCapacity)
    return fail(TFCB_CUDA_ERROR, "internal: output arena too small (string %lld needs > %lld words)", e.stream,
                e.limit);
  const unsigned long long ekey = (unsigned long long)e.stream, rkey = (unsigned long long)e.pos,
                           ikey = (unsigned long long)e.value;
  if (ekey == kUbiNone && rkey == kUbiNone && ikey == kUbiNone) return TFCB_OK;
  auto at = [&](const int32_t* p, long long i) {
    int32_t v = 0;
    if (cudaMemcpyAsync(&v, p + i, sizeof v, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess)
      (void)cudaGetLastError();
    return v;
  };
  auto where = [&](long long g, long long* item, long long* elem) {
    const int64_t* hi = std::upper_bound(item_offsets, item_offsets + n_items + 1, (int64_t)g);
    *item = (long long)(hi - item_offsets) - 1;
    *elem = g - item_offsets[*item];
  };
  long long item, elem;
  if (debug_level > 0 && ikey != kUbiNone) {
    where((long long)ikey, &item, &elem);
    return fail(TFCB_INVALID_ARGUMENT, "'index' has a value not in [0, %lld): value=%d (string %lld, element %lld)", R,
                at(index, (long long)ikey), item, elem);
  }
  if (debug_level > 0 && rkey != kUbiNone) {
    if (!(rkey & kUbiCdfKey))
      return fail(TFCB_INVALID_ARGUMENT, "'cdf_size' has a value not in [3, %lld]: value=%d", W,
                  at(cdf_size, (long long)rkey));
    const long long r = (long long)((rkey & ~kUbiCdfKey) >> 1);
    if (rkey & 1ull) return fail(TFCB_INVALID_ARGUMENT, "CDF is not monotonic");
    const int sz = at(cdf_size, r);
    return fail(TFCB_INVALID_ARGUMENT, "Each cdf should start from 0 and end at %d: cdf[0]=%d, cdf[^1]=%d",
                1 << precision, at(cdf, r * W), at(cdf, r * W + sz - 1));
  }
  const long long g = (long long)(ekey >> 3);
  where(g, &item, &elem);
  switch ((int)(ekey & 7ull)) {
    case kUbiIndex:
      return fail(TFCB_INVALID_ARGUMENT, "'index' has a value not in [0, %lld): value=%d (string %lld, element %lld)",
                  R, at(index, g), item, elem);
    case kUbiCdfSize:
      return fail(TFCB_INVALID_ARGUMENT, "'cdf_size' has a value not in [3, %lld]: value=%d (string %lld, element %lld)",
                  W, at(cdf_size, at(index, g)), item, elem);
    case kUbiInterval:
      return fail(TFCB_INVALID_ARGUMENT,
                  "symbol with zero probability or a CDF row beyond 2^precision (string %lld, element %lld)", item,
                  elem);
    case kUbiPrefix:
      return fail(TFCB_INVALID_ARGUMENT,
                  "damaged string: overflow width prefix exceeds %d digits of %d bits (string %lld, element %lld)",
                  (32 + overflow_width - 1) / overflow_width, overflow_width, item, elem);
  }
  return fail(TFCB_CUDA_ERROR, "internal: unknown error key %llx", ekey);
}

// The error record with every key at "none".
int ubi_reset_error(DevError* err, cudaStream_t s) {
  TFCB_CUDA_TRY(cudaMemsetAsync(err, 0, sizeof(DevError), s));
  TFCB_CUDA_TRY(cudaMemsetAsync(&err->stream, 0xFF, 3 * sizeof(long long), s));
  return TFCB_OK;
}

void ubi_launch_check(const UbiParams& P, long long n, cudaStream_t s) {
  const long long work = std::max<long long>(n, P.R);
  const unsigned blocks = (unsigned)std::min<long long>(std::max<long long>((work + 255) / 256, 1), 1024);
  ubi_check_kernel<<<blocks, 256, 0, s>>>(P.index, n, P.cdf, P.cdf_size, P.R, P.W, P.precision, P.err);
  TFCB_LAUNCHED();
}

}  // namespace
}  // namespace tfcb

struct tfcb_ubi_encoder : tfcb::EncArena {
  long long* ext = nullptr;  // device [2 * (n_streams + 1)]: element offsets, then arena offsets
  long long* offsets = nullptr;  // the caller's string offsets
  cudaStream_t s = nullptr;
};

namespace {
void ubi_release(tfcb_ubi_encoder* h, cudaStream_t s) {
  dev_free(h->state, s);
  dev_free(h->words, s);
  dev_free(h->cbits, s);
  dev_free(h->err, s);
  dev_free(h->ext, s);
  delete h;
}
}  // namespace

extern "C" {

int tfcb_unbounded_index_range_encode_ragged(const int32_t* data_dev, const int32_t* index_dev, int64_t n_items,
                                             const int64_t* item_offsets_host, const int32_t* cdf_dev,
                                             const int64_t* cdf_shape_host, int cdf_rank, const int32_t* cdf_size_dev,
                                             int64_t cdf_size_len, const int32_t* offset_dev, int64_t offset_len,
                                             int precision, int overflow_width, int debug_level, int64_t* offsets_dev,
                                             void* stream, tfcb_ubi_encoder** out, int64_t* total_bytes_host) {
  TFCB_TRY(ubi_check_attrs(precision, overflow_width, debug_level));
  TFCB_TRY(ubi_check_args(cdf_shape_host, cdf_rank, cdf_size_len, offset_len, n_items, item_offsets_host, index_dev,
                          cdf_dev, cdf_size_dev, offset_dev));
  if (!out || !total_bytes_host || !offsets_dev || (!data_dev && item_offsets_host[n_items] > 0))
    return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  const long long S = n_items, bits = ubi_bits_bound(precision, overflow_width);
  std::vector<long long> off(2 * (S + 1));
  long long* arena = off.data() + S + 1;
  long long total = 0;
  for (long long i = 0; i <= S; ++i) {
    off[i] = item_offsets_host[i];
    arena[i] = total;
    if (i == S) break;
    const long long n = item_offsets_host[i + 1] - item_offsets_host[i];
    if (n > ((kMaxStreamWords - 96) * 16) / bits)
      return fail(TFCB_INVALID_ARGUMENT, "string %lld: %lld elements may not fit one code stream (2^31 16-bit words)",
                  i, n);
    total += (words_for(bits, n) + 32 + 31) & ~31ll;
  }
  *out = nullptr;
  *total_bytes_host = 0;
  cudaStream_t s = as_stream(stream);
  auto* h = new tfcb_ubi_encoder;
  h->n_streams = S;
  h->s = s;
  h->offsets = reinterpret_cast<long long*>(offsets_dev);
  int rc = dev_alloc((void**)&h->state, (size_t)S * sizeof(EncState), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->words, (size_t)total * sizeof(uint16_t), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->cbits, (size_t)(total >> 5) * sizeof(uint32_t), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->ext, off.size() * sizeof(long long), s);
  if (rc == TFCB_OK) rc = ubi_reset_error(h->err, s);
  if (rc == TFCB_OK) {
    // (pageable source: staged before the call returns)
    const cudaError_t e = cudaMemcpyAsync(h->ext, off.data(), off.size() * sizeof(long long), cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
      (void)cudaGetLastError();
      rc = fail(TFCB_CUDA_ERROR, "UnboundedIndexRangeEncode: %s", cudaGetErrorString(e));
    }
  }
  if (rc != TFCB_OK) {
    ubi_release(h, s);
    return rc;
  }
  h->arena_off = h->ext + S + 1;
  UbiParams P{};
  P.data = data_dev;
  P.index = index_dev;
  P.cdf = cdf_dev;
  P.cdf_size = cdf_size_dev;
  P.offset = offset_dev;
  P.R = cdf_shape_host[0];
  P.W = cdf_shape_host[1];
  P.precision = precision;
  P.width = overflow_width;
  P.elem_off = h->ext;
  P.arena_off = h->arena_off;
  P.state = h->state;
  P.words = h->words;
  P.cbits = h->cbits;
  P.err = h->err;
  if (debug_level > 0) ubi_launch_check(P, item_offsets_host[S], s);
  ubi_encode_kernel<<<(unsigned)S, 32, 0, s>>>(P);
  TFCB_LAUNCHED();
  long long bytes = 0;
  DevError e{};
  rc = enc_offsets(*h, h->offsets, false, "unbounded", s, &bytes, &e);
  if (rc == TFCB_OK)
    rc = ubi_error(e, debug_level, item_offsets_host, n_items, index_dev, cdf_dev, cdf_size_dev, P.R, P.W, precision,
                   overflow_width, s);
  if (rc != TFCB_OK) {
    ubi_release(h, s);
    return rc;
  }
  *total_bytes_host = bytes;
  *out = h;
  return TFCB_OK;
}

int tfcb_unbounded_index_range_write(tfcb_ubi_encoder* h, uint8_t* bytes_dev, void* stream) {
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "UnboundedIndexRangeEncode: not an encoder handle");
  cudaStream_t s = as_stream(stream);
  int rc = TFCB_OK;
  if (!bytes_dev) {
    rc = fail(TFCB_INVALID_ARGUMENT, "UnboundedIndexRangeEncode: null output buffer");
  } else {
    enc_write(*h, h->offsets, bytes_dev, s);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(TFCB_CUDA_ERROR, "UnboundedIndexRangeEncode: %s", cudaGetErrorString(e));
  }
  ubi_release(h, s);
  return rc;
}

void tfcb_unbounded_index_range_encoder_destroy(tfcb_ubi_encoder* h) {
  if (h) ubi_release(h, h->s);
}

int tfcb_unbounded_index_range_decode_ragged(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_items,
                                             const int64_t* item_offsets_host, const int32_t* index_dev,
                                             const int32_t* cdf_dev, const int64_t* cdf_shape_host, int cdf_rank,
                                             const int32_t* cdf_size_dev, int64_t cdf_size_len,
                                             const int32_t* offset_dev, int64_t offset_len, int precision,
                                             int overflow_width, int debug_level, int32_t* out_dev, void* stream) {
  TFCB_TRY(ubi_check_attrs(precision, overflow_width, debug_level));
  TFCB_TRY(ubi_check_args(cdf_shape_host, cdf_rank, cdf_size_len, offset_len, n_items, item_offsets_host, index_dev,
                          cdf_dev, cdf_size_dev, offset_dev));
  if (!bytes_dev || !offsets_dev || (!out_dev && item_offsets_host[n_items] > 0))
    return fail(TFCB_INVALID_ARGUMENT, "null pointer argument");
  cudaStream_t s = as_stream(stream);
  const long long S = n_items;
  DevError* err = nullptr;
  long long* elem_off = nullptr;
  int rc = dev_alloc((void**)&err, sizeof(DevError), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&elem_off, (size_t)(S + 1) * sizeof(long long), s);
  if (rc == TFCB_OK) rc = ubi_reset_error(err, s);
  if (rc == TFCB_OK &&
      cudaMemcpyAsync(elem_off, item_offsets_host, (size_t)(S + 1) * sizeof(long long), cudaMemcpyHostToDevice, s) !=
          cudaSuccess) {
    (void)cudaGetLastError();
    rc = fail(TFCB_CUDA_ERROR, "UnboundedIndexRangeDecode: could not upload the item offsets");
  }
  DevError e{};
  if (rc == TFCB_OK) {
    UbiParams P{};
    P.out = out_dev;
    P.index = index_dev;
    P.cdf = cdf_dev;
    P.cdf_size = cdf_size_dev;
    P.offset = offset_dev;
    P.R = cdf_shape_host[0];
    P.W = cdf_shape_host[1];
    P.precision = precision;
    P.width = overflow_width;
    P.elem_off = elem_off;
    P.bytes = bytes_dev;
    P.str_off = reinterpret_cast<const long long*>(offsets_dev);
    P.err = err;
    if (debug_level > 0) ubi_launch_check(P, item_offsets_host[S], s);
    ubi_decode_kernel<<<(unsigned)S, 32, 0, s>>>(P);
    TFCB_LAUNCHED();
    cudaError_t ce = cudaMemcpyAsync(&e, err, sizeof e, cudaMemcpyDeviceToHost, s);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    if (ce != cudaSuccess) {
      (void)cudaGetLastError();
      rc = fail(TFCB_CUDA_ERROR, "CUDA error '%s' in UnboundedIndexRangeDecode", cudaGetErrorString(ce));
    }
  }
  if (rc == TFCB_OK)
    rc = ubi_error(e, debug_level, item_offsets_host, n_items, index_dev, cdf_dev, cdf_size_dev, cdf_shape_host[0],
                   cdf_shape_host[1], precision, overflow_width, s);
  dev_free(err, s);
  dev_free(elem_off, s);
  return rc;
}

}  // extern "C"
