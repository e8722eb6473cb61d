// PmfToQuantizedCdf on sm_90a: one thread block per PMF row.
//
// Replaces tensorflow_compression/cc/kernels/pmf_to_cdf_kernels.cc:58-208 (Compute / PerShard /
// PenaltyItem / GainItem) and, through tfcb_build_lookup, the per-row tf.while_loop of
// tensorflow_compression/python/entropy_models/continuous_base.py:282-294.
//
// Semantics kept bit for bit:
//   v_i = max(1, (int)rintf(pmf_i * 2^p))                       fp32 multiply, round-half-even
//   while sum > 2^p: decrement the bin with the smallest  mass * (log2 v - log2 (v-1))   (double)
//   while sum < 2^p: increment the bin with the largest   mass * (log2 (v+1) - log2 v)   (double)
//   cdf = prefix sum.
// The reference keeps a sorted queue and re-inserts a stepped item behind all items of equal key, so
// among equal keys the item that has waited longest goes first; the initial order among equal keys
// comes from an unstable std::sort.  Here: waited-longest first as well, initial ties broken by
// LOWEST BIN INDEX.  log2 of the integer arguments comes from a table computed on the host with the
// same libm the reference would use, so every double comparison is identical.  The shared table covers
// counts up to 65537; a row whose counts reach past it (a bin with mass above 1, or with a large
// multiple of 2^-p) is rerun with a larger table built for that call, up to kMaxLogTab entries.
#include <cmath>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kThreads = 256;
constexpr int kLogTab = 65538;       // shared table: log2(v) for v in [0, 65537]
constexpr int kMaxLogTab = 1 << 24;  // largest per-call table (128 MiB): counts up to 2^24 - 1

double* g_log2_dev = nullptr;
std::mutex g_log2_mu;

std::vector<double> log_table(int entries) {
  std::vector<double> tab(entries);
  tab[0] = 0.0;
  for (int v = 1; v < entries; ++v) tab[v] = std::log2(static_cast<double>(v));
  return tab;
}

int ensure_log_table(cudaStream_t s) {
  std::lock_guard<std::mutex> lock(g_log2_mu);
  if (g_log2_dev) return TFCB_OK;
  const std::vector<double> tab = log_table(kLogTab);
  double* d = nullptr;
  TFCB_CUDA_TRY(cudaMalloc((void**)&d, kLogTab * sizeof(double)));
  cudaError_t e = cudaMemcpyAsync(d, tab.data(), kLogTab * sizeof(double), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    cudaFree(d);
    return fail(TFCB_CUDA_ERROR, "log2 table upload failed: %s", cudaGetErrorString(e));
  }
  g_log2_dev = d;
  return TFCB_OK;
}

// What one launch reports to the host.  `err`: the first non-finite or negative mass.  Counts the
// log2 table does not cover: the largest one, and the lowest (row, bin) whose count is kMaxLogTab or
// more, stored complemented as ~(row << 20 | bin) so that atomicMax keeps the lowest and 0 means none.
// Only the DOWN adjustment can read past the table: a count of 65538 or more makes the row sum exceed
// 2^precision, and DOWN steps only lower counts.
struct RowsStatus {
  DevError err;
  unsigned long long max_count;
  unsigned long long first_over_cap;
};

struct Cand {
  double key;
  int age;
  int idx;
};

template <bool DOWN>
__device__ __forceinline__ bool better(const Cand& a, const Cand& b) {
  if (a.idx < 0) return false;
  if (b.idx < 0) return true;
  if (DOWN ? (a.key < b.key) : (a.key > b.key)) return true;
  if (a.key == b.key && a.age < b.age) return true;
  return false;
}

template <bool DOWN>
__device__ __forceinline__ Cand warp_best(Cand c) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    Cand o;
    o.key = __shfl_xor_sync(0xFFFFFFFFu, c.key, d);
    o.age = __shfl_xor_sync(0xFFFFFFFFu, c.age, d);
    o.idx = __shfl_xor_sync(0xFFFFFFFFu, c.idx, d);
    if (better<DOWN>(o, c)) c = o;
  }
  return c;
}

template <bool DOWN>
__device__ __forceinline__ double step_key(int v, double mass, const double* __restrict__ lg) {
  if (DOWN) {
    if (v <= 1) return INFINITY;
    return mass * (lg[v] - lg[v - 1]);
  }
  if (v < 1) return -INFINITY;
  return mass * (lg[v + 1] - lg[v]);
}

template <bool DOWN>
__device__ void adjust(int* q, const float* pmf, int len, float extra, int n, long long steps,
                       double* key, int* age, const double* __restrict__ lg) {
  __shared__ Cand s_warp[kThreads / 32];
  __shared__ Cand s_best;
  const int tid = threadIdx.x;
  for (int i = tid; i < n; i += kThreads) {
    const double mass = (double)(i < len ? pmf[i] : extra);
    key[i] = step_key<DOWN>(q[i], mass, lg);
    age[i] = i;
  }
  __syncthreads();
  int clock = n;
  for (long long it = 0; it < steps; ++it) {
    Cand c;
    c.idx = -1;
    c.key = 0;
    c.age = 0;
    for (int i = tid; i < n; i += kThreads) {
      Cand o;
      o.key = key[i];
      o.age = age[i];
      o.idx = i;
      if (better<DOWN>(o, c)) c = o;
    }
    c = warp_best<DOWN>(c);
    if ((tid & 31) == 0) s_warp[tid >> 5] = c;
    __syncthreads();
    if (tid < 32) {
      Cand w;
      if (tid < kThreads / 32) {
        w = s_warp[tid];
      } else {
        w.idx = -1;
        w.key = 0;
        w.age = 0;
      }
      w = warp_best<DOWN>(w);
      if (tid == 0) {
        s_best = w;
        const int b = w.idx;
        const int nv = q[b] + (DOWN ? -1 : 1);
        q[b] = nv;
        const double mass = (double)(b < len ? pmf[b] : extra);
        key[b] = step_key<DOWN>(nv, mass, lg);
        age[b] = clock;
      }
    }
    ++clock;
    __syncthreads();
  }
}

// One block per row.  `lens` == nullptr: dense rows of n bins, output stride n + 1 (the op).
// `lens` != nullptr: ragged rows with an appended overflow bin and a leading -precision entry
// written at out + out_off[r] (the table builder).
__global__ void __launch_bounds__(kThreads) pmf_rows_kernel(
    const float* __restrict__ pmf_all, long long row_stride, int n_fixed, const int* __restrict__ lens,
    const long long* __restrict__ out_off, int precision, int* __restrict__ out_all,
    double* __restrict__ key_all, int* __restrict__ age_all, long long scratch_stride,
    const double* __restrict__ lg, int lg_n, RowsStatus* st) {
  __shared__ long long s_red[kThreads / 32];
  __shared__ float s_redf[kThreads / 32];
  __shared__ long long s_sum;
  __shared__ float s_extra;
  __shared__ int s_bad;
  __shared__ int s_big;
  const long long r = blockIdx.x;
  const int tid = threadIdx.x;
  const float* pmf = pmf_all + r * row_stride;
  int len, n;
  int* cdf;
  if (lens) {
    len = lens[r];
    n = len + 1;
    int* o = out_all + out_off[r];
    if (tid == 0) o[0] = -precision;
    cdf = o + 1;
  } else {
    len = n_fixed;
    n = n_fixed;
    cdf = out_all + r * (long long)(n_fixed + 1);
  }
  int* q = cdf + 1;
  double* key = key_all + r * scratch_stride;
  int* age = age_all + r * scratch_stride;
  const int total = 1 << precision;

  if (tid == 0) {
    s_bad = 0;
    s_big = 0;
  }
  __syncthreads();
  // validation (pmf_to_cdf_kernels.cc:77-86) and, for ragged rows, the overflow mass
  float part = 0.f;
  for (int i = tid; i < len; i += kThreads) {
    const float m = pmf[i];
    if (!(isfinite(m) && m >= 0.f)) {
      s_bad = 1;
      report(&st->err, kErrValue, r, i, (long long)__float_as_int(m), 0);
    }
    part += m;
  }
  float extra = 0.f;
  if (lens) {
    // deterministic tree reduction in fp32 (continuous_base.py:285: max(1 - reduce_sum(p), 0))
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, d);
    if ((tid & 31) == 0) s_redf[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) t += s_redf[w];
      s_extra = fmaxf(1.f - t, 0.f);
    }
    __syncthreads();
    extra = s_extra;
  } else {
    __syncthreads();
  }
  if (s_bad) return;

  long long local = 0;
  for (int i = tid; i < n; i += kThreads) {
    const float m = i < len ? pmf[i] : extra;
    int v = (int)rintf(__fmul_rn(m, (float)total));
    v = max(v, 1);
    q[i] = v;
    local += v;
    if (v >= lg_n) {  // beyond the table: the host reruns with a larger one
      s_big = 1;
      atomicMax(&st->max_count, (unsigned long long)v);
      if (v >= kMaxLogTab) atomicMax(&st->first_over_cap, ~((unsigned long long)r << 20 | (unsigned)i));
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) local += __shfl_xor_sync(0xFFFFFFFFu, local, d);
  if ((tid & 31) == 0) s_red[tid >> 5] = local;
  __syncthreads();
  if (tid == 0) {
    long long t = 0;
    for (int w = 0; w < kThreads / 32; ++w) t += s_red[w];
    s_sum = t;
  }
  __syncthreads();
  const long long sum = s_sum;
  if (s_big) return;
  if (sum > total) {
    adjust<true>(q, pmf, len, extra, n, sum - total, key, age, lg);
  } else if (sum < total) {
    adjust<false>(q, pmf, len, extra, n, total - sum, key, age, lg);
  }
  __syncthreads();

  // prefix sum in place; cdf[0] = 0
  __shared__ int s_scan[kThreads / 32];
  __shared__ int s_carry;
  if (tid == 0) {
    s_carry = 0;
    cdf[0] = 0;
  }
  __syncthreads();
  for (int base = 0; base < n; base += kThreads) {
    const int i = base + tid;
    const int v = i < n ? q[i] : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
      if ((tid & 31) >= d) x += y;
    }
    if ((tid & 31) == 31) s_scan[tid >> 5] = x;
    __syncthreads();
    if (tid < 32) {
      int w = tid < kThreads / 32 ? s_scan[tid] : 0;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xFFFFFFFFu, w, d);
        if (tid >= d) w += y;
      }
      if (tid < kThreads / 32) s_scan[tid] = w;
    }
    __syncthreads();
    const int incl = s_carry + ((tid >> 5) ? s_scan[(tid >> 5) - 1] : 0) + x;
    if (i < n) q[i] = incl;
    __syncthreads();
    if (tid == kThreads - 1) s_carry = incl;
    __syncthreads();
  }
}

// One launch over all rows with the log2 table `lg` of `lg_n` entries; copies the status back and
// synchronises.
int launch_rows(const float* pmf, long long rows, long long row_stride, int n_fixed, const int* lens_dev,
                const long long* out_off_dev, long long max_n, int precision, int* out, double* key, int* age,
                const double* lg, int lg_n, RowsStatus* st_dev, RowsStatus* st, cudaStream_t s) {
  cudaMemsetAsync(st_dev, 0, sizeof(RowsStatus), s);
  pmf_rows_kernel<<<(unsigned)rows, kThreads, 0, s>>>(pmf, row_stride, n_fixed, lens_dev, out_off_dev, precision,
                                                      out, key, age, max_n, lg, lg_n, st_dev);
  TFCB_LAUNCHED();
  cudaError_t ce = cudaMemcpyAsync(st, st_dev, sizeof *st, cudaMemcpyDeviceToHost, s);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
  if (ce != cudaSuccess) {
    (void)cudaGetLastError();
    return fail(TFCB_CUDA_ERROR, "CUDA error '%s' in PmfToQuantizedCdf", cudaGetErrorString(ce));
  }
  if (st->err.code != kErrNone) {
    const int bits = (int)st->err.value;
    float f;
    memcpy(&f, &bits, sizeof f);
    return fail(TFCB_INVALID_ARGUMENT,
                "`pmf` has non-finite or negative element: %g (row %lld, bin %lld). Please check for "
                "numerical problems in the probability computation.",
                (double)f, st->err.stream, st->err.pos);
  }
  return TFCB_OK;
}

int run_rows(const float* pmf, long long rows, long long row_stride, int n_fixed, const int* lens_dev,
             const long long* out_off_dev, long long max_n, int precision, int* out, cudaStream_t s) {
  TFCB_TRY(ensure_log_table(s));
  double* key = nullptr;
  int* age = nullptr;
  RowsStatus* st_dev = nullptr;
  double* big_lg = nullptr;
  RowsStatus st;
  int rc = dev_alloc((void**)&key, (size_t)rows * max_n * sizeof(double), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&age, (size_t)rows * max_n * sizeof(int), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&st_dev, sizeof(RowsStatus), s);
  if (rc == TFCB_OK)
    rc = launch_rows(pmf, rows, row_stride, n_fixed, lens_dev, out_off_dev, max_n, precision, out, key, age,
                     g_log2_dev, kLogTab, st_dev, &st, s);
  if (rc == TFCB_OK && st.first_over_cap) {
    const unsigned long long at = ~st.first_over_cap;
    rc = fail(TFCB_INVALID_ARGUMENT,
              "`pmf` row %lld, bin %lld quantises to %d or more counts; at most %d counts per bin are supported",
              (long long)(at >> 20), (long long)(at & 0xFFFFF), kMaxLogTab, kMaxLogTab - 1);
  } else if (rc == TFCB_OK && st.max_count) {
    // Rows with counts past the shared table were left unadjusted: rerun every row with a table for this
    // call only (the shared one stays in place for concurrent calls on other streams).
    const int entries = (int)st.max_count + 1;
    const std::vector<double> tab = log_table(entries);
    rc = dev_alloc((void**)&big_lg, (size_t)entries * sizeof(double), s);
    if (rc == TFCB_OK) {
      cudaError_t ce = cudaMemcpyAsync(big_lg, tab.data(), (size_t)entries * sizeof(double),
                                       cudaMemcpyHostToDevice, s);
      if (ce != cudaSuccess) {
        (void)cudaGetLastError();
        rc = fail(TFCB_CUDA_ERROR, "log2 table upload failed: %s", cudaGetErrorString(ce));
      }
    }
    if (rc == TFCB_OK)
      rc = launch_rows(pmf, rows, row_stride, n_fixed, lens_dev, out_off_dev, max_n, precision, out, key, age,
                       big_lg, entries, st_dev, &st, s);
  }
  dev_free(big_lg, s);
  dev_free(key, s);
  dev_free(age, s);
  dev_free(st_dev, s);
  return rc;
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

int tfcb_pmf_to_quantized_cdf(const float* pmf_dev, int64_t rows, int64_t n, int precision,
                              int32_t* cdf_dev, void* stream) {
  if (!(0 < precision && precision <= 16))
    return fail(TFCB_INVALID_ARGUMENT, "`precision` must be in [1, 16]: %d", precision);
  if (rows < 0) return fail(TFCB_INVALID_ARGUMENT, "`pmf` should be at least 1-D.");
  if (n <= 1) return fail(TFCB_INVALID_ARGUMENT, "`pmf` size should be at least 2 in the last axis.");
  if (n > (1ll << precision))
    return fail(TFCB_INVALID_ARGUMENT,
                "`pmf` has %lld bins but 2^precision = %d: every bin needs at least one count",
                (long long)n, 1 << precision);
  if (rows == 0) return TFCB_OK;
  if (!pmf_dev || !cdf_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  return run_rows(pmf_dev, rows, n, (int)n, nullptr, nullptr, n, precision, cdf_dev, as_stream(stream));
}

int tfcb_build_lookup(const float* pmf_dev, int64_t rows, int64_t max_len, const int32_t* lens_host,
                      int precision, int32_t* lookup_dev, void* stream) {
  if (!(0 < precision && precision <= 16))
    return fail(TFCB_INVALID_ARGUMENT, "`precision` must be in [1, 16]: %d", precision);
  if (rows <= 0) return TFCB_OK;
  if (!pmf_dev || !lens_host || !lookup_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  cudaStream_t s = as_stream(stream);
  std::vector<long long> off(rows);
  long long at = 0, max_n = 0;
  for (int64_t r = 0; r < rows; ++r) {
    const long long len = lens_host[r];
    if (len < 1 || len > max_len)
      return fail(TFCB_INVALID_ARGUMENT, "pmf_length[%lld]=%lld not in [1, %lld]", (long long)r, len,
                  (long long)max_len);
    if (len + 1 > (1ll << precision))
      return fail(TFCB_INVALID_ARGUMENT, "PMF %lld has %lld bins, more than 2^precision", (long long)r,
                  len + 1);
    off[r] = at;
    at += len + 3;
    max_n = std::max(max_n, len + 1);
  }
  int* lens_dev = nullptr;
  long long* off_dev = nullptr;
  int rc = dev_alloc((void**)&lens_dev, rows * sizeof(int), s);
  if (rc == TFCB_OK) rc = dev_alloc((void**)&off_dev, rows * sizeof(long long), s);
  if (rc == TFCB_OK) {
    cudaMemcpyAsync(lens_dev, lens_host, rows * sizeof(int), cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(off_dev, off.data(), rows * sizeof(long long), cudaMemcpyHostToDevice, s);
    rc = run_rows(pmf_dev, rows, max_len, 0, lens_dev, off_dev, max_n, precision, lookup_dev, s);
  }
  dev_free(lens_dev, s);
  dev_free(off_dev, s);
  return rc;
}

}  // extern "C"
