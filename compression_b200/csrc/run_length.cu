// RunLengthEncode / RunLengthDecode (tensorflow_compression/cc/kernels/run_length_kernels.cc:52-262, op contract
// cc/ops/run_length_ops.cc:28-84, bit packing cc/lib/bit_coder.cc:50-191; RunLengthGammaEncode/Decode are the
// (-1, -1, false) special case, run_length_gamma_kernels.cc), for n coding units (strings) in one launch sequence.
// The one-string ops are the one-unit case of the same kernels.
//
// The reference walks the tensor once and appends variable-length codes (Elias gamma or Rice) LSB-first to a bit
// string.  Every code is a function of one element and of the run it belongs to, so the ENCODER is data parallel
// over all elements of all units at once:
//   1. run starts by a forward max-scan (a run = maximal stretch of zeros or of non-zeros that does not cross a unit
//      boundary: every unit start is a run start), run lengths scattered to the run starts by each run's last element;
//   2. the bit length of the token each element contributes (zero for most zeros; the last element of a unit that
//      ends in zeros carries the trailing run length);
//   3. an exclusive 64-bit prefix sum of the lengths = every token's bit offset in the concatenation of the units'
//      codes; unit u's code is bits off[start_u] .. off[end_u], padded to whole bytes, and an exclusive scan over the
//      units' byte lengths places the strings back to back;
//   4. every token ORs its few set bits into a zero-initialised word buffer at 8 * byte_offset[u] + (off[i] -
//      off[start_u]) (the long unary zero prefixes are never touched), two 32-bit atomics per field.
// The DECODER is inherently serial within a string (a code's position depends on all previous codes): one thread per
// string, all strings in one launch, reading through a 64-bit bit window.  A ragged launch takes as long as the
// longest string's walk.
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <new>

#include "common.cuh"

namespace tfcb {
namespace {

struct RlParams {
  int rl_code, mag_code, rl_nz;
};

__device__ __forceinline__ int bit_width_dev(uint32_t v) { return 32 - __clz(v); }

// bits of WriteRunLength(v), run_length_kernels.cc:66-72
__device__ __forceinline__ unsigned long long len_rl(uint32_t v, const RlParams& P) {
  if (P.rl_code >= 0) return (unsigned long long)(v >> P.rl_code) + 1ull + (unsigned long long)P.rl_code;
  return 2ull * (unsigned long long)bit_width_dev(v + 1u) - 1ull;
}
// magnitude payload of WriteNonZero(sample), :74-89
__device__ __forceinline__ uint32_t mag_value(int32_t s, const RlParams& P) {
  if (P.mag_code >= 0) return (uint32_t)(s > 0 ? s - 1 : -(s + 1));
  if (s == INT32_MIN) return (uint32_t)INT32_MAX;  // "We can't encode int32 minimum. Encode closest value instead."
  return (uint32_t)(s > 0 ? s : -s);
}
__device__ __forceinline__ unsigned long long len_mag(uint32_t m, const RlParams& P) {
  if (P.mag_code >= 0) return (unsigned long long)(m >> P.mag_code) + 1ull + (unsigned long long)P.mag_code;
  return 2ull * (unsigned long long)bit_width_dev(m) - 1ull;
}

struct MaxOp {
  __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; }
};

constexpr int kLaunchesPerScan = 2;  // cub's single-pass scans: an init kernel and the scan kernel

// first[unit_off[u]] = 1 for every unit with elements (empty units mark nothing)
__global__ void rl_unit_starts_kernel(const long long* __restrict__ unit_off, long long n_units,
                                      uint8_t* __restrict__ first) {
  const long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u < n_units && unit_off[u] < unit_off[u + 1]) first[unit_off[u]] = 1;
}

// start candidates: i where a unit starts or the zero-ness changes, else -1
__global__ void rl_boundaries_kernel(const int32_t* __restrict__ data, long long n, const uint8_t* __restrict__ first,
                                     int* __restrict__ cand) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  cand[i] = (first[i] || (data[i - 1] != 0) != (data[i] != 0)) ? (int)i : -1;  // first[0] is always set
}

__device__ __forceinline__ bool unit_last(const uint8_t* first, long long n, long long i) {
  return i == n - 1 || first[i + 1];
}

__global__ void rl_runlen_kernel(const int32_t* __restrict__ data, long long n, const uint8_t* __restrict__ first,
                                 const int* __restrict__ start, int* __restrict__ runlen) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (unit_last(first, n, i) || (data[i + 1] != 0) != (data[i] != 0))  // the run's last element
    runlen[start[i]] = (int)(i - start[i] + 1);
}

// The zero run that ends right before element i (0 if none) and whether a non-zero run precedes it in the unit.
__device__ __forceinline__ uint32_t zero_run_before(const int32_t* data, const uint8_t* first, const int* start,
                                                    long long i, bool* later_run) {
  *later_run = false;
  if (first[i] || data[i - 1] != 0) return 0u;
  const int s = start[i - 1];
  *later_run = !first[s];
  return (uint32_t)(i - s);
}

__global__ void rl_lengths_kernel(const int32_t* __restrict__ data, long long n, const uint8_t* __restrict__ first,
                                  const int* __restrict__ start, const int* __restrict__ runlen, RlParams P,
                                  unsigned long long* __restrict__ len) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t s = data[i];
  unsigned long long L = 0;
  if (s != 0) {
    L = 1ull + len_mag(mag_value(s, P), P);
    bool later;
    const uint32_t zr = zero_run_before(data, first, start, i, &later);
    if (!P.rl_nz) {
      L += len_rl(zr, P);
    } else if (start[i] == i) {  // first element of a non-zero run: both run lengths precede it
      L += len_rl(zr - (later ? 1u : 0u), P) + len_rl((uint32_t)runlen[i] - 1u, P);
    }
  } else if (unit_last(first, n, i)) {  // trailing zeros: one last run length
    const int st = start[i];
    const uint32_t zr = (uint32_t)(i + 1 - st);
    L = len_rl(zr - ((P.rl_nz && !first[st]) ? 1u : 0u), P);
  }
  len[i] = L;
}

// byte length of every unit's code; entry n_units is 0 so that the exclusive scan ends in the total
__global__ void rl_unit_bytes_kernel(const long long* __restrict__ unit_off, long long n_units,
                                     const unsigned long long* __restrict__ off, long long* __restrict__ bytes) {
  const long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u > n_units) return;
  bytes[u] = u < n_units ? (long long)((off[unit_off[u + 1]] - off[unit_off[u]] + 7ull) >> 3) : 0ll;
}

// ORs the low `nbits` (<= 32) bits of `value` into the bit string at bit position `pos` (LSB first, bit_coder.cc:50-66)
__device__ __forceinline__ void put_bits(uint32_t* out, unsigned long long pos, int nbits, uint32_t value) {
  if (nbits <= 0) return;
  const unsigned long long v = (unsigned long long)(nbits == 32 ? value : (value & ((1u << nbits) - 1u))) << (pos & 31ull);
  const unsigned long long w = pos >> 5;
  if ((uint32_t)v) atomicOr(out + w, (uint32_t)v);
  if ((uint32_t)(v >> 32)) atomicOr(out + w + 1, (uint32_t)(v >> 32));
}
// WriteRice / WriteGamma at `pos`; returns the position after the code
__device__ __forceinline__ unsigned long long put_code(uint32_t* out, unsigned long long pos, uint32_t value, int code) {
  if (code >= 0) {  // Rice: value >> code zeros, a one, `code` low bits
    pos += (unsigned long long)(value >> code);
    put_bits(out, pos, 1, 1u);
    put_bits(out, pos + 1, code, value);
    return pos + 1ull + (unsigned long long)code;
  }
  const int bw = bit_width_dev(value);  // gamma of value > 0: bw - 1 zeros, a one, bw - 1 low bits
  pos += (unsigned long long)(bw - 1);
  put_bits(out, pos, 1, 1u);
  put_bits(out, pos + 1, bw - 1, value);
  return pos + (unsigned long long)bw;
}
__device__ __forceinline__ unsigned long long put_rl(uint32_t* out, unsigned long long pos, uint32_t v, const RlParams& P) {
  return put_code(out, pos, P.rl_code >= 0 ? v : v + 1u, P.rl_code);
}

// the unit that holds element i: the largest u with unit_off[u] <= i (empty units share their offset with the next)
__device__ __forceinline__ long long unit_of(const long long* unit_off, long long n_units, long long i) {
  long long lo = 0, hi = n_units - 1;
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (unit_off[mid] <= i) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

__global__ void rl_emit_kernel(const int32_t* __restrict__ data, long long n, const uint8_t* __restrict__ first,
                               const int* __restrict__ start, const int* __restrict__ runlen, RlParams P,
                               const unsigned long long* __restrict__ off, const long long* __restrict__ unit_off,
                               long long n_units, const long long* __restrict__ str_off, uint32_t* __restrict__ out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t s = data[i];
  if (s == 0 && !unit_last(first, n, i)) return;  // a zero inside a run contributes no bits
  const long long u = unit_of(unit_off, n_units, i);
  unsigned long long pos = 8ull * (unsigned long long)str_off[u] + (off[i] - off[unit_off[u]]);
  if (s != 0) {
    bool later;
    const uint32_t zr = zero_run_before(data, first, start, i, &later);
    if (!P.rl_nz) {
      pos = put_rl(out, pos, zr, P);
    } else if (start[i] == i) {
      pos = put_rl(out, pos, zr - (later ? 1u : 0u), P);
      pos = put_rl(out, pos, (uint32_t)runlen[i] - 1u, P);
    }
    put_bits(out, pos, 1, s > 0 ? 1u : 0u);
    put_code(out, pos + 1, mag_value(s, P), P.mag_code);
  } else {
    const int st = start[i];
    put_rl(out, pos, (uint32_t)(i + 1 - st) - ((P.rl_nz && !first[st]) ? 1u : 0u), P);
  }
}

// ---- decoder: one thread per string, BitReader semantics of bit_coder.cc:92-189 (errors -> codes) ----
// `buf` holds the next `avail` bits of the string in its low bits, the bits above are zero.  Loads never leave the
// string's own bytes.
struct BitWindow {
  const uint8_t* p;
  long long nbytes, next;  // next: the first byte not yet in the window
  unsigned long long buf;
  int avail;

  __device__ __forceinline__ void refill() {
    if (next + 8 <= nbytes) {  // as many whole bytes as fit, as independent loads
      const int k = (64 - avail) >> 3;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (j < k) buf |= (unsigned long long)p[next + j] << (avail + 8 * j);
      next += k;
      avail += 8 * k;
      return;
    }
    while (avail <= 56 && next < nbytes) {
      buf |= (unsigned long long)p[next++] << avail;
      avail += 8;
    }
  }
  // Consumes zeros up to and including the next one; *zeros counts them.  False if the string ends first.  The
  // window is only reloaded once it holds no one, so most codes are read without waiting for a load.
  __device__ __forceinline__ bool unary(unsigned long long* zeros) {
    unsigned long long z = 0;
    while (!buf) {
      z += (unsigned long long)avail;
      avail = 0;
      if (next >= nbytes) return false;
      // a long Rice quotient (up to 2^32 zeros): skip whole zero bytes, 8 at a time once aligned
      while (next < nbytes && ((uintptr_t)(p + next) & 7) && p[next] == 0) ++next, z += 8;
      if (!((uintptr_t)(p + next) & 7))
        while (next + 8 <= nbytes && *reinterpret_cast<const unsigned long long*>(p + next) == 0ull) next += 8, z += 64;
      while (next < nbytes && p[next] == 0) ++next, z += 8;
      refill();
    }
    const int t = __ffsll((long long)buf) - 1;
    buf = (buf >> t) >> 1;
    avail -= t + 1;
    *zeros = z + (unsigned long long)t;
    return true;
  }
  __device__ __forceinline__ bool bits(int count, uint32_t* v) {  // count <= 31
    if (avail < count) refill();
    if (avail < count) return false;
    *v = (uint32_t)(buf & ((1ull << count) - 1ull));
    buf >>= count;
    avail -= count;
    return true;
  }
  // 0 ok, 1 out of bits, 2 gamma too wide (reported only once the terminating one has been read)
  __device__ __forceinline__ int gamma(uint32_t* v) {
    unsigned long long z;
    if (!unary(&z)) return 1;
    if (z + 1ull > 31ull) return 2;
    uint32_t lsbs;
    if (!bits((int)z, &lsbs)) return 1;
    *v = (1u << z) | lsbs;
    return 0;
  }
  __device__ __forceinline__ int rice(int k, uint32_t* v) {
    unsigned long long z;
    if (!unary(&z)) return 1;
    uint32_t lsbs;
    if (!bits(k, &lsbs)) return 1;
    *v = ((uint32_t)z << k) | lsbs;  // the quotient wraps at 2^32, as the reference's uint32 counter does
    return 0;
  }
};

// err: 0 ok, 1 "Out of bits to read.", 2 "Exceeded maximum gamma bit width.", 3 "Decoded past end of tensor."
// String u is bytes[str_off[u] .. str_off[u+1]) and decodes into data[unit_off[u] .. unit_off[u+1]), which the caller
// has zero-filled.  *first_err ends as min over failing units of (u << 2 | err) (all ones if none fails).
__global__ void rl_decode_kernel(const uint8_t* __restrict__ bytes, const long long* __restrict__ str_off,
                                 const long long* __restrict__ unit_off, long long n_units, RlParams P,
                                 int32_t* __restrict__ data, unsigned long long* __restrict__ first_err) {
  const long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u >= n_units) return;
  const long long n = unit_off[u + 1] - unit_off[u];
  if (n <= 0) return;
  data += unit_off[u];
  const long long b0 = str_off[u], b1 = str_off[u + 1];
  BitWindow rd = {bytes + b0, b1 > b0 ? b1 - b0 : 0, 0, 0ull, 0};
  auto read_rl = [&](uint32_t* v) -> int {
    if (P.rl_code >= 0) return rd.rice(P.rl_code, v);
    const int e = rd.gamma(v);
    if (e == 0) *v -= 1u;
    return e;
  };
  auto read_nz = [&](int32_t* s) -> int {
    uint32_t pos_bit, m;
    if (!rd.bits(1, &pos_bit)) return 1;
    const int e = (P.mag_code >= 0) ? rd.rice(P.mag_code, &m) : rd.gamma(&m);
    if (e) return e;
    if (P.mag_code >= 0) *s = pos_bit ? (int32_t)(m + 1u) : (int32_t)(0u - m - 1u);
    else *s = pos_bit ? (int32_t)m : (int32_t)(0u - m);
    return 0;
  };
  long long p = 0;
  uint32_t offset = 0;
  int e = 0;
  while (p < n) {
    uint32_t run;
    if ((e = read_rl(&run))) break;
    p += (long long)run + offset;
    if (!(p < n)) {
      if (p != n) e = 3;
      break;
    }
    if (P.rl_nz) {
      if ((e = read_rl(&run))) break;
      const long long next_zero = p + (long long)run + 1;
      if (next_zero > n) {
        e = 3;
        break;
      }
      while (p < next_zero) {
        int32_t s;
        if ((e = read_nz(&s))) break;
        data[p++] = s;
      }
      if (e) break;
      offset = 1;
    } else {
      int32_t s;
      if ((e = read_nz(&s))) break;
      data[p++] = s;
    }
  }
  if (e) atomicMin(first_err, ((unsigned long long)u << 2) | (unsigned long long)e);
}

const char* decode_message(int e) {
  return e == 1 ? "Out of bits to read." : e == 2 ? "Exceeded maximum gamma bit width." : "Decoded past end of tensor.";
}

// Host-side checks of the code parameters and of a batch's unit offsets [n_units + 1].
int check_units(const char* op, long long n_units, const int64_t* off, int rl_code, int mag_code) {
  if (n_units <= 0) return fail(TFCB_INVALID_ARGUMENT, "%s: `n_units` must be positive: %lld", op, n_units);
  if (n_units >= (1ll << 31) - 1) return fail(TFCB_INVALID_ARGUMENT, "%s: `n_units` must be below 2^31 - 1", op);
  if (!off) return fail(TFCB_INVALID_ARGUMENT, "%s: `unit_offsets` is null", op);
  if (off[0] != 0) return fail(TFCB_INVALID_ARGUMENT, "%s: unit_offsets[0] must be 0: %lld", op, (long long)off[0]);
  for (long long i = 0; i < n_units; ++i)
    if (off[i + 1] < off[i])
      return fail(TFCB_INVALID_ARGUMENT,
                  "%s: unit_offsets must be non-decreasing: unit_offsets[%lld]=%lld > unit_offsets[%lld]=%lld", op, i,
                  (long long)off[i], i + 1, (long long)off[i + 1]);
  if (off[n_units] >= (1ll << 31))
    return fail(TFCB_INVALID_ARGUMENT, "%s: the units hold %lld elements; at most 2^31 - 1 are supported", op,
                (long long)off[n_units]);
  if (rl_code > 31 || mag_code > 31) return fail(TFCB_INVALID_ARGUMENT, "%s: Rice parameter > 31", op);
  return TFCB_OK;
}

}  // namespace
}  // namespace tfcb

// Everything the emit pass needs, from the sizing pass (tfcb_run_length_encode_ragged) to the write.
struct tfcb_rl_encoder {
  const int32_t* data;  // borrowed: the caller keeps it until the write
  long long n, n_units;
  tfcb::RlParams P;
  long long* unit_off;      // [n_units + 1]
  long long* str_off;       // [n_units + 1], byte offsets of the strings
  uint8_t* first;           // [n], 1 at every unit's first element
  int* start;               // [n], start of every element's run
  int* runlen;              // [n], run lengths at the run starts
  unsigned long long* off;  // [n + 1], bit offsets of the tokens in the concatenated unit codes
  int64_t total_bytes;
  cudaStream_t s;
};

namespace tfcb {
namespace {

void rl_release(tfcb_rl_encoder* h, cudaStream_t s) {
  if (!h) return;
  dev_free(h->unit_off, s); dev_free(h->str_off, s); dev_free(h->first, s);
  dev_free(h->start, s); dev_free(h->runlen, s); dev_free(h->off, s);
  delete h;
}

// Steps 1-3 for units [unit_off_host[u], unit_off_host[u+1]) of `data` (arguments already checked): every string's
// byte offset lands in h->str_off, the total in h->total_bytes after one synchronisation.
int rl_encode_prepare(const int32_t* data, long long n_units, const int64_t* unit_off_host, RlParams P, cudaStream_t s,
                      tfcb_rl_encoder** out) {
  const long long n = unit_off_host[n_units];
  tfcb_rl_encoder* h = new (std::nothrow) tfcb_rl_encoder();
  if (!h) return fail(TFCB_OUT_OF_MEMORY, "RunLengthEncode: out of host memory");
  h->data = data, h->n = n, h->n_units = n_units, h->P = P, h->s = s;
  int* cand = nullptr;
  unsigned long long* len = nullptr;
  long long* unit_bytes = nullptr;
  void* tmp = nullptr;
  size_t t1 = 0, t2 = 0, t3 = 0;
  if (n > 0) {
    cub::DeviceScan::InclusiveScan(nullptr, t1, (int*)nullptr, (int*)nullptr, MaxOp(), (int)n, s);
    cub::DeviceScan::ExclusiveSum(nullptr, t2, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)(n + 1), s);
  }
  cub::DeviceScan::ExclusiveSum(nullptr, t3, (long long*)nullptr, (long long*)nullptr, (int)(n_units + 1), s);
  const size_t tmp_bytes = std::max(std::max(t1, t2), t3) + 16;
  const size_t units_bytes = (size_t)(n_units + 1) * sizeof(long long);
  int rc = dev_alloc((void**)&h->unit_off, units_bytes, s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&h->str_off, units_bytes, s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&unit_bytes, units_bytes, s);
  if (rc == TFCB_OK) rc = dev_alloc(&tmp, tmp_bytes, s);
  if (n > 0) {
    if (rc == TFCB_OK) rc = dev_alloc((void**)&h->first, (size_t)n, s);
    if (rc == TFCB_OK) rc = dev_alloc((void**)&h->start, (size_t)n * sizeof(int), s);
    if (rc == TFCB_OK) rc = dev_alloc((void**)&h->runlen, (size_t)n * sizeof(int), s);
    if (rc == TFCB_OK) rc = dev_alloc((void**)&h->off, (size_t)(n + 1) * sizeof(unsigned long long), s);
    if (rc == TFCB_OK) rc = dev_alloc((void**)&cand, (size_t)n * sizeof(int), s);
    if (rc == TFCB_OK) rc = dev_alloc((void**)&len, (size_t)(n + 1) * sizeof(unsigned long long), s);
  }
  auto cleanup = [&]() {
    dev_free(cand, s); dev_free(len, s); dev_free(unit_bytes, s); dev_free(tmp, s);
  };
  if (rc != TFCB_OK) {
    cleanup();
    rl_release(h, s);
    return rc;
  }
  cudaError_t e = cudaMemcpyAsync(h->unit_off, unit_off_host, units_bytes, cudaMemcpyHostToDevice, s);
  const unsigned ugrid = (unsigned)((n_units + 1 + 255) / 256);
  if (n > 0) {
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaMemsetAsync(h->first, 0, (size_t)n, s);
    rl_unit_starts_kernel<<<ugrid, 256, 0, s>>>(h->unit_off, n_units, h->first);
    rl_boundaries_kernel<<<grid, 256, 0, s>>>(data, n, h->first, cand);
    size_t t = tmp_bytes;
    cub::DeviceScan::InclusiveScan(tmp, t, cand, h->start, MaxOp(), (int)n, s);
    rl_runlen_kernel<<<grid, 256, 0, s>>>(data, n, h->first, h->start, h->runlen);
    rl_lengths_kernel<<<grid, 256, 0, s>>>(data, n, h->first, h->start, h->runlen, P, len);
    cudaMemsetAsync(len + n, 0, sizeof(unsigned long long), s);
    t = tmp_bytes;
    cub::DeviceScan::ExclusiveSum(tmp, t, len, h->off, (int)(n + 1), s);  // off[n] = total bits
    rl_unit_bytes_kernel<<<ugrid, 256, 0, s>>>(h->unit_off, n_units, h->off, unit_bytes);
    t = tmp_bytes;
    cub::DeviceScan::ExclusiveSum(tmp, t, unit_bytes, h->str_off, (int)(n_units + 1), s);
    for (int k = 0; k < 5 + 3 * kLaunchesPerScan; ++k) TFCB_LAUNCHED();
  } else {
    cudaMemsetAsync(h->str_off, 0, units_bytes, s);  // every string is empty
  }
  long long total = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&total, h->str_off + n_units, sizeof total, cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  cleanup();
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    rl_release(h, s);
    return fail(TFCB_CUDA_ERROR, "RunLengthEncode: %s", cudaGetErrorString(e));
  }
  h->total_bytes = total;
  *out = h;
  return TFCB_OK;
}

// Step 4: zeroes ceil(total / 4) words at `words` and ORs every token into them.
int rl_emit(const tfcb_rl_encoder* h, uint32_t* words, cudaStream_t s) {
  if (h->total_bytes == 0) return TFCB_OK;
  cudaMemsetAsync(words, 0, (size_t)((h->total_bytes + 3) / 4) * 4, s);
  rl_emit_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, s>>>(h->data, h->n, h->first, h->start, h->runlen, h->P,
                                                                 h->off, h->unit_off, h->n_units, h->str_off, words);
  TFCB_LAUNCHED();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TFCB_CUDA_ERROR, "RunLengthEncode launch failed: %s", cudaGetErrorString(e));
  return TFCB_OK;
}

// Decodes string u of `bytes` (byte offsets str_off_dev, or str_off_host uploaded here when given) into
// data[unit_off_host[u] ..] for every unit (arguments already checked), synchronises once and returns the lowest
// failing unit's (u << 2 | err), all ones if every string decoded.
int rl_decode(const uint8_t* bytes, const int64_t* str_off_dev, const int64_t* str_off_host, long long n_units,
              const int64_t* unit_off_host, RlParams P, int32_t* data, cudaStream_t s, unsigned long long* first_err) {
  const long long n = unit_off_host[n_units];
  *first_err = ~0ull;
  if (n == 0) return TFCB_OK;
  const size_t units_bytes = (size_t)(n_units + 1) * sizeof(long long);
  long long* buf = nullptr;  // unit offsets, [string offsets,] error word
  TFCB_TRY(dev_alloc((void**)&buf, units_bytes * (str_off_host ? 2 : 1) + 8, s));
  long long* unit_off = buf;
  const long long* str_off = str_off_host ? buf + (n_units + 1) : (const long long*)str_off_dev;
  unsigned long long* err = reinterpret_cast<unsigned long long*>(buf + (n_units + 1) * (str_off_host ? 2 : 1));
  cudaError_t e = cudaMemcpyAsync(unit_off, unit_off_host, units_bytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess && str_off_host)
    e = cudaMemcpyAsync(buf + (n_units + 1), str_off_host, units_bytes, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(err, 0xff, sizeof *err, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(data, 0, (size_t)n * sizeof(int32_t), s);  // "Fill data tensor with zeros."
  if (e == cudaSuccess) {
    rl_decode_kernel<<<(unsigned)((n_units + 127) / 128), 128, 0, s>>>(bytes, str_off, unit_off, n_units, P, data, err);
    TFCB_LAUNCHED();
    e = cudaMemcpyAsync(first_err, err, sizeof *err, cudaMemcpyDeviceToHost, s);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  dev_free(buf, s);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(TFCB_CUDA_ERROR, "RunLengthDecode: %s", cudaGetErrorString(e));
  }
  return TFCB_OK;
}

RlParams params(int run_length_code, int magnitude_code, int use_run_length_for_non_zeros) {
  return {run_length_code, magnitude_code, use_run_length_for_non_zeros ? 1 : 0};
}

}  // namespace
}  // namespace tfcb

extern "C" {

int tfcb_run_length_encode(const int32_t* data_dev, int64_t n, int run_length_code, int magnitude_code,
                           int use_run_length_for_non_zeros, uint8_t* code_dev, int64_t capacity, int64_t* n_bytes_host,
                           void* stream) {
  using namespace tfcb;
  if (n < 0 || n >= (1ll << 31) || capacity < 0 || !n_bytes_host) return fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: bad sizes");
  if (run_length_code > 31 || magnitude_code > 31) return fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: Rice parameter > 31");
  *n_bytes_host = 0;
  if (n == 0) return TFCB_OK;
  if (!data_dev || (!code_dev && capacity > 0)) return fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: null tensor");
  if (capacity & 3) capacity &= ~3ll;  // the bit string is assembled in 32-bit words
  cudaStream_t s = as_stream(stream);
  const int64_t unit_off[2] = {0, n};
  tfcb_rl_encoder* h = nullptr;
  TFCB_TRY(rl_encode_prepare(data_dev, 1, unit_off, params(run_length_code, magnitude_code, use_run_length_for_non_zeros),
                             s, &h));
  const int64_t n_bytes = h->total_bytes;
  *n_bytes_host = n_bytes;
  const int64_t words = (n_bytes + 3) / 4;
  int rc = words * 4 > capacity
               ? fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: the code needs %lld bytes (capacity %lld)",
                      (long long)(words * 4), (long long)capacity)
               : rl_emit(h, reinterpret_cast<uint32_t*>(code_dev), s);  // the one string starts at byte 0
  rl_release(h, s);
  return rc;
}

int tfcb_run_length_decode(const uint8_t* code_dev, int64_t n_bytes, int run_length_code, int magnitude_code,
                           int use_run_length_for_non_zeros, int32_t* data_dev, int64_t n, void* stream) {
  using namespace tfcb;
  if (n < 0 || n_bytes < 0) return fail(TFCB_INVALID_ARGUMENT, "RunLengthDecode: bad sizes");
  if (run_length_code > 31 || magnitude_code > 31) return fail(TFCB_INVALID_ARGUMENT, "RunLengthDecode: Rice parameter > 31");
  if (n == 0) return TFCB_OK;
  if (!data_dev || (!code_dev && n_bytes > 0)) return fail(TFCB_INVALID_ARGUMENT, "RunLengthDecode: null tensor");
  const int64_t unit_off[2] = {0, n}, str_off[2] = {0, n_bytes};
  unsigned long long first_err;
  TFCB_TRY(rl_decode(code_dev, nullptr, str_off, 1, unit_off,
                     params(run_length_code, magnitude_code, use_run_length_for_non_zeros), data_dev, as_stream(stream),
                     &first_err));
  if (first_err != ~0ull) return fail(TFCB_INVALID_ARGUMENT, "%s", decode_message((int)(first_err & 3ull)));
  return TFCB_OK;
}

int tfcb_run_length_encode_ragged(const int32_t* data_dev, int64_t n_units, const int64_t* unit_offsets_host,
                                  int run_length_code, int magnitude_code, int use_run_length_for_non_zeros,
                                  int64_t* offsets_dev, void* stream, tfcb_rl_encoder** out, int64_t* total_bytes_host) {
  using namespace tfcb;
  TFCB_TRY(check_units("RunLengthEncode", n_units, unit_offsets_host, run_length_code, magnitude_code));
  if (!offsets_dev || !out || !total_bytes_host || (!data_dev && unit_offsets_host[n_units] > 0))
    return fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: null pointer argument");
  *out = nullptr;
  *total_bytes_host = 0;
  cudaStream_t s = as_stream(stream);
  tfcb_rl_encoder* h = nullptr;
  TFCB_TRY(rl_encode_prepare(data_dev, n_units, unit_offsets_host,
                             params(run_length_code, magnitude_code, use_run_length_for_non_zeros), s, &h));
  const cudaError_t e = cudaMemcpyAsync(offsets_dev, h->str_off, (size_t)(n_units + 1) * sizeof(int64_t),
                                        cudaMemcpyDeviceToDevice, s);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    rl_release(h, s);
    return fail(TFCB_CUDA_ERROR, "RunLengthEncode: %s", cudaGetErrorString(e));
  }
  *total_bytes_host = h->total_bytes;
  *out = h;
  return TFCB_OK;
}

int tfcb_run_length_write(tfcb_rl_encoder* h, uint8_t* bytes_dev, void* stream) {
  using namespace tfcb;
  if (!h) return fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: not a run-length encoder");
  cudaStream_t s = as_stream(stream);
  int rc = TFCB_OK;
  if (h->total_bytes > 0) {
    // strings meet at byte granularity, so the words are assembled in a buffer of our own and only the caller's
    // [0, total) is written
    uint32_t* words = nullptr;
    if (!bytes_dev) rc = fail(TFCB_INVALID_ARGUMENT, "RunLengthEncode: null output buffer");
    if (rc == TFCB_OK) rc = dev_alloc((void**)&words, (size_t)((h->total_bytes + 3) / 4) * 4, s);
    if (rc == TFCB_OK) rc = rl_emit(h, words, s);
    if (rc == TFCB_OK) {
      const cudaError_t e = cudaMemcpyAsync(bytes_dev, words, (size_t)h->total_bytes, cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess) {
        (void)cudaGetLastError();
        rc = fail(TFCB_CUDA_ERROR, "RunLengthEncode: %s", cudaGetErrorString(e));
      }
    }
    dev_free(words, s);
  }
  rl_release(h, s);
  return rc;
}

void tfcb_run_length_encoder_destroy(tfcb_rl_encoder* h) {
  if (h) tfcb::rl_release(h, h->s);
}

int tfcb_run_length_decode_ragged(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_units,
                                  const int64_t* unit_offsets_host, int run_length_code, int magnitude_code,
                                  int use_run_length_for_non_zeros, int32_t* data_dev, void* stream) {
  using namespace tfcb;
  TFCB_TRY(check_units("RunLengthDecode", n_units, unit_offsets_host, run_length_code, magnitude_code));
  if (!bytes_dev || !offsets_dev || (!data_dev && unit_offsets_host[n_units] > 0))
    return fail(TFCB_INVALID_ARGUMENT, "RunLengthDecode: null pointer argument");
  unsigned long long first_err;
  TFCB_TRY(rl_decode(bytes_dev, offsets_dev, nullptr, n_units, unit_offsets_host,
                     params(run_length_code, magnitude_code, use_run_length_for_non_zeros), data_dev, as_stream(stream),
                     &first_err));
  if (first_err != ~0ull)
    return fail(TFCB_INVALID_ARGUMENT, "RunLengthDecode: unit %lld: %s", (long long)(first_err >> 2),
                decode_message((int)(first_err & 3ull)));
  return TFCB_OK;
}

}  // extern "C"
