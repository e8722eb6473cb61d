// Universal quantisation's coding tensors (tensorflow_compression/python/entropy_models/universal.py:30-62,147-170,
// 446-466) in one launch: per element the shared noise level (Philox-4x32-10 of its position within its item), the
// flat table index and the quantisation offset.  Element-parallel and memory-bound: 8 B written per element (12 B
// with float64 offsets), plus 4R or 8R B of indexes read in the indexed mode.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxRanges = 8;            // index dimensions of an indexed model, the noise level excluded
constexpr unsigned kMaxCtas = 1u << 20;  // grid-stride beyond this

// Philox-4x32-10 (Salmon et al., SC'11), the word order of entropy_models._philox4x32.
__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1) {
  uint32_t c2 = 0, c3 = 0;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

struct Params {
  // Items: either `per_item` elements each (elem_off null), or elem_off / block_off [k + 1] on the device, where
  // block_off counts the items' 4-element Philox blocks.
  const long long* elem_off;
  const long long* block_off;
  int k;
  long long per_item;
  long long n_blocks;
  uint32_t key0, key1;
  unsigned long long maxval;  // number of noise levels (any positive value for the bare draw)
  long long prior_size;       // batched mode: table index = level * prior_size + i % prior_size
  const void* indexes;        // indexed mode: [elements, n_ranges] in T
  int n_ranges;
  double bound[kMaxRanges + 1];     // range - 1 per coordinate, the level first (converted to T in the kernel)
  uint32_t stride[kMaxRanges + 1];  // strides of (levels,) + index_ranges, as int32 (wrapping like torch's sum)
  int32_t* levels;                  // bare draw: the levels
  int32_t* table;                   // coding tensors: table index
  void* offset;                     // and offset, float or double
};

__device__ __forceinline__ int32_t clamp_to_int(double x, double hi) {
  // max then min as _normalize_indexes does (NaN stays NaN), then the cast toward zero torch's .to(int32) makes
  return (int32_t)(x < 0.0 ? 0.0 : (x > hi ? hi : x));
}
__device__ __forceinline__ int32_t clamp_to_int(float x, float hi) {
  return (int32_t)(x < 0.f ? 0.f : (x > hi ? hi : x));
}

// MODE 0: bare draw (levels); 1: batched coding tensors; 2: indexed coding tensors with indexes of type T.
template <int MODE, typename T, bool OFF64>
__global__ void __launch_bounds__(kThreads) universal_kernel(const Params p) {
  for (long long b = blockIdx.x * (long long)kThreads + threadIdx.x; b < p.n_blocks;
       b += (long long)gridDim.x * kThreads) {
    long long item_start, n_item, q;
    if (p.elem_off == nullptr) {
      const long long per_block = (p.per_item + 3) >> 2;
      const long long j = b / per_block;
      q = b - j * per_block;
      item_start = j * p.per_item;
      n_item = p.per_item;
    } else {  // the last item whose first block is at or before b (empty items have none)
      int lo = 0, hi = p.k;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(p.block_off + mid) <= b) lo = mid; else hi = mid;
      }
      q = b - __ldg(p.block_off + lo);
      item_start = __ldg(p.elem_off + lo);
      n_item = __ldg(p.elem_off + lo + 1) - item_start;
    }
    const uint4 w4 = philox4x32_10((uint32_t)q, (uint32_t)((unsigned long long)q >> 32), p.key0, p.key1);
    const uint32_t words[4] = {w4.x, w4.y, w4.z, w4.w};
    const int cnt = (int)min(4ll, n_item - 4 * q);
    long long row = MODE == 1 ? (4 * q) % p.prior_size : 0;  // i % prior_size, advanced per element
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      if (w >= cnt) break;
      const long long e = item_start + 4 * q + w;  // position in the flat output (4q + w within the item)
      const uint32_t word = words[w];
      const int32_t level = (int32_t)(p.maxval > 0xFFFFFFFFull ? word : word % (uint32_t)p.maxval);
      if (MODE == 0) {
        p.levels[e] = level;
        continue;
      }
      double lv;  // the level as the offset formula reads it
      int32_t flat;
      if (MODE == 1) {
        lv = (double)level;
        flat = (int32_t)((uint32_t)level * (uint32_t)p.prior_size + (uint32_t)row);
        if (++row == p.prior_size) row = 0;
      } else {
        // _add_offset_indexes casts the level to the indexes' type; _normalize_indexes clips every coordinate
        const T* idx = static_cast<const T*>(p.indexes) + e * p.n_ranges;
        const T lt = (T)level;
        const T lc = lt < (T)0 ? (T)0 : (lt > (T)p.bound[0] ? (T)p.bound[0] : lt);
        lv = (double)lc;
        uint32_t acc = (uint32_t)clamp_to_int(lc, (T)p.bound[0]) * p.stride[0];
        for (int r = 0; r < p.n_ranges; ++r)
          acc += (uint32_t)clamp_to_int(idx[r], (T)p.bound[r + 1]) * p.stride[r + 1];
        flat = (int32_t)acc;
      }
      p.table[e] = flat;
      const double off = (lv + 1.0) / (double)(p.maxval + 1) - 0.5;  // universal.py:45-47, in double
      if (OFF64) static_cast<double*>(p.offset)[e] = off;
      else static_cast<float*>(p.offset)[e] = (float)off;
    }
  }
}

int check_item_offsets(const int64_t* off, long long n_items) {
  if (n_items <= 0) return fail(TFCB_INVALID_ARGUMENT, "`n_items` must be positive: %lld", n_items);
  if (!off) return fail(TFCB_INVALID_ARGUMENT, "`item_offsets` is null");
  if (off[0] != 0) return fail(TFCB_INVALID_ARGUMENT, "item_offsets[0] must be 0: %lld", (long long)off[0]);
  for (long long i = 0; i < n_items; ++i)
    if (off[i + 1] < off[i])
      return fail(TFCB_INVALID_ARGUMENT,
                  "item_offsets must be non-decreasing: item_offsets[%lld]=%lld > item_offsets[%lld]=%lld", i,
                  (long long)off[i], i + 1, (long long)off[i + 1]);
  if (n_items > 0x7FFFFFFFll) return fail(TFCB_INVALID_ARGUMENT, "too many items: %lld", n_items);
  return TFCB_OK;
}

template <int MODE, typename T, bool OFF64>
int launch(Params& p, const int64_t* item_off, long long n_items, cudaStream_t s) {
  // items of equal length (a batch of coding units) need no offsets on the device
  const long long per = item_off[1];
  bool uniform = per > 0;
  for (long long j = 1; uniform && j <= n_items; ++j) uniform = item_off[j] - item_off[j - 1] == per;
  long long* dev_off = nullptr;
  if (uniform) {
    p.elem_off = p.block_off = nullptr;
    p.per_item = per;
    p.n_blocks = n_items * ((per + 3) >> 2);
  } else {
    std::vector<long long> host(2 * (n_items + 1));
    long long nb = 0;
    for (long long j = 0; j <= n_items; ++j) {
      host[j] = item_off[j];
      host[n_items + 1 + j] = nb;
      if (j < n_items) nb += (item_off[j + 1] - item_off[j] + 3) >> 2;
    }
    TFCB_TRY(dev_alloc((void**)&dev_off, host.size() * sizeof(long long), s));
    const cudaError_t e = cudaMemcpyAsync(dev_off, host.data(), host.size() * sizeof(long long),
                                          cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
      dev_free(dev_off, s);
      TFCB_CUDA_TRY(e);
    }
    p.elem_off = dev_off;
    p.block_off = dev_off + n_items + 1;
    p.k = (int)n_items;
    p.n_blocks = nb;
  }
  const unsigned grid = (unsigned)std::min<long long>((p.n_blocks + kThreads - 1) / kThreads, kMaxCtas);
  universal_kernel<MODE, T, OFF64><<<grid, kThreads, 0, s>>>(p);
  TFCB_LAUNCHED();
  const cudaError_t e = cudaGetLastError();
  dev_free(dev_off, s);
  TFCB_CUDA_TRY(e);
  return TFCB_OK;
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

int tfcb_stateless_uniform_int(int32_t* out_dev, int64_t n, uint32_t seed0, uint32_t seed1, int64_t maxval,
                               void* stream) {
  if (n < 0) return fail(TFCB_INVALID_ARGUMENT, "`n` must be non-negative: %lld", (long long)n);
  if (maxval < 1) return fail(TFCB_INVALID_ARGUMENT, "`maxval` must be positive: %lld", (long long)maxval);
  if (n == 0) return TFCB_OK;
  if (!out_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  Params p{};
  p.key0 = seed0;
  p.key1 = seed1;
  p.maxval = (unsigned long long)maxval;
  p.levels = out_dev;
  const int64_t off[2] = {0, n};
  return launch<0, float, false>(p, off, 1, as_stream(stream));
}

int tfcb_universal_coding_tensors(int64_t n_items, const int64_t* item_offsets_host, uint32_t seed0, uint32_t seed1,
                                  int64_t num_noise_levels, int64_t prior_size, const void* indexes_dev,
                                  int32_t indexes_is_f64, const int64_t* index_ranges_host, int32_t n_ranges,
                                  int32_t* table_index_dev, void* offset_dev, int32_t offset_is_f64, void* stream) {
  TFCB_TRY(check_item_offsets(item_offsets_host, n_items));
  if (num_noise_levels < 1 || num_noise_levels > 0x7FFFFFFFll)
    return fail(TFCB_INVALID_ARGUMENT, "`num_noise_levels` must be in [1, 2^31): %lld", (long long)num_noise_levels);
  Params p{};
  p.key0 = seed0;
  p.key1 = seed1;
  p.maxval = (unsigned long long)num_noise_levels;
  const bool indexed = indexes_dev != nullptr || n_ranges != 0;
  if (indexed) {
    if (n_ranges < 1 || n_ranges > kMaxRanges)
      return fail(TFCB_INVALID_ARGUMENT, "`n_ranges` must be in [1, %d]: %d", kMaxRanges, n_ranges);
    if (!index_ranges_host) return fail(TFCB_INVALID_ARGUMENT, "`index_ranges` is null");
    long long ranges[kMaxRanges + 1];
    ranges[0] = num_noise_levels;
    for (int r = 0; r < n_ranges; ++r) {
      ranges[r + 1] = index_ranges_host[r];
      if (ranges[r + 1] < 1)
        return fail(TFCB_INVALID_ARGUMENT, "index_ranges[%d] must be positive: %lld", r, ranges[r + 1]);
    }
    unsigned long long stride = 1;  // np.cumprod of the reversed ranges, narrowed to int32 as _flatten_indexes does
    for (int r = n_ranges; r >= 0; --r) {
      p.stride[r] = (uint32_t)stride;
      p.bound[r] = (double)(ranges[r] - 1);
      stride *= (unsigned long long)ranges[r];
    }
    p.n_ranges = n_ranges;
  } else if (prior_size < 1) {
    return fail(TFCB_INVALID_ARGUMENT, "`prior_size` must be positive: %lld", (long long)prior_size);
  }
  p.prior_size = prior_size;
  if (item_offsets_host[n_items] == 0) return TFCB_OK;
  if (!table_index_dev || !offset_dev || (indexed && !indexes_dev)) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  p.indexes = indexes_dev;
  p.table = table_index_dev;
  p.offset = offset_dev;
  cudaStream_t s = as_stream(stream);
  if (!indexed) return offset_is_f64 ? launch<1, float, true>(p, item_offsets_host, n_items, s)
                                     : launch<1, float, false>(p, item_offsets_host, n_items, s);
  if (indexes_is_f64) return offset_is_f64 ? launch<2, double, true>(p, item_offsets_host, n_items, s)
                                           : launch<2, double, false>(p, item_offsets_host, n_items, s);
  return offset_is_f64 ? launch<2, float, true>(p, item_offsets_host, n_items, s)
                       : launch<2, float, false>(p, item_offsets_host, n_items, s);
}

}  // extern "C"
