// ORACLE / TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
//
// The UnboundedIndexRangeEncode / UnboundedIndexRangeDecode op loops (cc/kernels/unbounded_index_range_coding_kernels.cc
// needs TF headers and is not compiled) restated around the reference's own RangeEncoder / RangeDecoder, compiled in
// place like oracle/ref/ref_driver.cc, which is included here for its error plumbing and its persistent
// ParallelOverStreams pool; the library built from this file also exports everything ref_driver.cc does.
#include "../ref/ref_driver.cc"

// ------------------------------------------------------------------------------------------
// UnboundedIndexRangeEncode / UnboundedIndexRangeDecode op loops
// (cc/kernels/unbounded_index_range_coding_kernels.cc), restated around the reference's own RangeEncoder /
// RangeDecoder.  Every input on which the reference's loop would run undefined code (signed overflow of
// data - offset, -2d - 1, 2(d - m), u / 2 + m or value + offset; a shift by 32 or more; an index or cdf_size that
// reads outside the tables) or would not end is an error here instead, so the oracle never executes it.
// ------------------------------------------------------------------------------------------
namespace {

struct UbiArgs {
  const int32_t* cdf;
  int64_t R, W;
  const int32_t* cdf_size;
  const int32_t* offset;
  int precision, w, debug;
};

// CheckIndex / CheckCdfSize / CheckCdf over the whole tensors (debug_level 1).
bool UbiDebugCheck(const UbiArgs& a, const int32_t* index, int64_t n, std::string* err) {
  for (int64_t i = 0; i < n; ++i)
    if (index[i] < 0 || index[i] >= a.R) {
      *err = "'index' has a value not in [0, " + std::to_string(a.R) + "): value=" + std::to_string(index[i]);
      return false;
    }
  for (int64_t r = 0; r < a.R; ++r)
    if (a.cdf_size[r] < 3 || a.cdf_size[r] > a.W) {
      *err = "'cdf_size' has a value not in [3, " + std::to_string(a.W) + "]: value=" + std::to_string(a.cdf_size[r]);
      return false;
    }
  const int32_t top = 1 << a.precision;
  for (int64_t r = 0; r < a.R; ++r) {
    const int32_t* row = a.cdf + r * a.W;
    const int32_t sz = a.cdf_size[r];
    if (row[0] != 0 || row[sz - 1] != top) {
      *err = "Each cdf should start from 0 and end at " + std::to_string(top) + ": cdf[0]=" + std::to_string(row[0]) +
             ", cdf[^1]=" + std::to_string(row[sz - 1]);
      return false;
    }
    for (int32_t j = 0; j + 1 < sz; ++j)
      if (row[j + 1] <= row[j]) {
        *err = "CDF is not monotonic";
        return false;
      }
  }
  return true;
}

// The row element i codes with, or null (error set) where the reference would read outside the tables.
const int32_t* UbiRow(const UbiArgs& a, int32_t r, int32_t* m, std::string* err) {
  if (r < 0 || r >= a.R) {
    *err = "'index' has a value not in [0, " + std::to_string(a.R) + "): value=" + std::to_string(r);
    return nullptr;
  }
  if (a.cdf_size[r] < 3 || a.cdf_size[r] > a.W) {
    *err = "'cdf_size' has a value not in [3, " + std::to_string(a.W) + "]: value=" + std::to_string(a.cdf_size[r]);
    return nullptr;
  }
  *m = a.cdf_size[r] - 2;
  return a.cdf + static_cast<int64_t>(r) * a.W;
}

bool UbiEncodeOne(const UbiArgs& a, const int32_t* data, const int32_t* index, int64_t n, std::string* sink,
                  std::string* err) {
  tfc::RangeEncoder enc;
  const int K = (32 + a.w - 1) / a.w;
  const uint32_t max_overflow = (1u << a.w) - 1;
  for (int64_t i = 0; i < n; ++i) {
    int32_t m;
    const int32_t* row = UbiRow(a, index[i], &m, err);
    if (!row) return false;
    const int64_t d = static_cast<int64_t>(data[i]) - a.offset[index[i]];
    if (d < std::numeric_limits<int32_t>::min() || d > std::numeric_limits<int32_t>::max()) {
      *err = "undefined in the reference: data - offset overflows int32";
      return false;
    }
    int32_t value = static_cast<int32_t>(d);
    uint32_t overflow = 0;
    if (value < 0) {
      if (value <= -(1 << 30)) {
        *err = "undefined in the reference: -2 * (data - offset) - 1 overflows int32";
        return false;
      }
      overflow = -2 * value - 1;
      value = m;
    } else if (value >= m) {
      if (value - m >= (1 << 30)) {
        *err = "undefined in the reference: 2 * (data - offset - max_value) overflows int32";
        return false;
      }
      overflow = 2 * (value - m);
      value = m;
    }
    const int32_t lo = row[value], hi = row[value + 1];
    if (!(0 <= lo && lo < hi && hi <= (1 << a.precision))) {
      *err = "symbol with zero probability or a CDF row beyond 2^precision";
      return false;
    }
    enc.Encode(lo, hi, a.precision, sink);
    if (value == m) {
      if ((overflow >> ((K - 1) * a.w)) != 0) {  // the width loop would shift by K * w >= 32
        *err = "undefined in the reference: the overflow width loop shifts by 32 or more";
        return false;
      }
      int32_t widths = 0;
      while (overflow >> (widths * a.w) != 0) ++widths;
      uint32_t val = widths;
      while (val >= max_overflow) {
        enc.Encode(max_overflow, max_overflow + 1, a.w, sink);
        val -= max_overflow;
      }
      enc.Encode(val, val + 1, a.w, sink);
      for (int32_t j = 0; j < widths; ++j) {
        const uint32_t digit = (overflow >> (j * a.w)) & max_overflow;
        enc.Encode(digit, digit + 1, a.w, sink);
      }
    }
  }
  enc.Finalize(sink);
  return true;
}

bool UbiDecodeOne(const UbiArgs& a, const std::string& src, const int32_t* index, int64_t n, int32_t* out,
                  std::string* err) {
  tfc::RangeDecoder dec{absl::string_view(src)};
  const int K = (32 + a.w - 1) / a.w;
  const uint32_t max_overflow = (1u << a.w) - 1;
  std::vector<int32_t> overflow_cdf((1 << a.w) + 1);
  std::iota(overflow_cdf.begin(), overflow_cdf.end(), 0);
  const absl::Span<const int32_t> uniform(overflow_cdf.data(), overflow_cdf.size());
  for (int64_t i = 0; i < n; ++i) {
    int32_t m;
    const int32_t* row = UbiRow(a, index[i], &m, err);
    if (!row) return false;
    int32_t value = dec.Decode(absl::Span<const int32_t>(row, m + 2), a.precision);
    if (value == m) {
      int32_t widths = 0;
      uint32_t val;
      do {
        val = dec.Decode(uniform, a.w);
        widths += val;
        if (widths > K) {  // a digit would be shifted by 32 or more (and the prefix need not end)
          *err = "undefined in the reference: overflow width prefix longer than " + std::to_string(K) + " digits";
          return false;
        }
      } while (val == max_overflow);
      uint32_t overflow = 0;
      for (int32_t j = 0; j < widths; ++j) overflow |= static_cast<uint32_t>(dec.Decode(uniform, a.w)) << (j * a.w);
      value = overflow >> 1;
      if (overflow & 1) {
        value = -value - 1;
      } else {
        if (static_cast<int64_t>(value) + m > std::numeric_limits<int32_t>::max()) {
          *err = "undefined in the reference: overflow / 2 + max_value overflows int32";
          return false;
        }
        value += m;
      }
    }
    const int64_t v = static_cast<int64_t>(value) + a.offset[index[i]];
    if (v < std::numeric_limits<int32_t>::min() || v > std::numeric_limits<int32_t>::max()) {
      *err = "undefined in the reference: value + offset overflows int32";
      return false;
    }
    out[i] = static_cast<int32_t>(v);
  }
  return true;
}

// The lowest failing item's message, prefixed with the item when there are several.
int UbiFail(const std::vector<std::string>& errs, int64_t k) {
  for (int64_t u = 0; u < k; ++u)
    if (!errs[u].empty()) return Fail(k > 1 ? "string " + std::to_string(u) + ": " + errs[u] : errs[u]);
  return 0;
}

}  // namespace

extern "C" {

// Item u = elements [item_off[u], item_off[u+1]) -> string u at out[str_off[u] .. str_off[u+1]).  Returns 0, 1 (error,
// see last_error) or 2 (out_cap too small; str_off[k] holds the size needed).
int tfcref_unbounded_encode(const int32_t* data, const int32_t* index, const int64_t* item_off, int64_t k,
                            const int32_t* cdf, int64_t R, int64_t W, const int32_t* cdf_size, const int32_t* offset,
                            int precision, int w, int debug_level, int threads, int64_t* str_off, uint8_t* out,
                            int64_t out_cap) {
  const UbiArgs a{cdf, R, W, cdf_size, offset, precision, w, debug_level};
  std::string err;
  if (debug_level > 0 && !UbiDebugCheck(a, index, item_off[k], &err)) return Fail(err);
  std::vector<std::string> sinks(k), errs(k);
  ParallelOverStreams(k, threads, [&](int64_t lo, int64_t hi) {
    for (int64_t u = lo; u < hi; ++u)
      UbiEncodeOne(a, data + item_off[u], index + item_off[u], item_off[u + 1] - item_off[u], &sinks[u], &errs[u]);
  });
  if (UbiFail(errs, k)) return 1;
  str_off[0] = 0;
  for (int64_t u = 0; u < k; ++u) str_off[u + 1] = str_off[u] + static_cast<int64_t>(sinks[u].size());
  if (str_off[k] > out_cap) return 2;
  for (int64_t u = 0; u < k; ++u) std::memcpy(out + str_off[u], sinks[u].data(), sinks[u].size());
  g_error.clear();
  return 0;
}

int tfcref_unbounded_decode(const uint8_t* bytes, const int64_t* str_off, int64_t k, const int32_t* index,
                            const int64_t* item_off, const int32_t* cdf, int64_t R, int64_t W, const int32_t* cdf_size,
                            const int32_t* offset, int precision, int w, int debug_level, int threads, int32_t* out) {
  const UbiArgs a{cdf, R, W, cdf_size, offset, precision, w, debug_level};
  std::string err;
  if (debug_level > 0 && !UbiDebugCheck(a, index, item_off[k], &err)) return Fail(err);
  std::vector<std::string> errs(k);
  ParallelOverStreams(k, threads, [&](int64_t lo, int64_t hi) {
    for (int64_t u = lo; u < hi; ++u) {
      const std::string src(reinterpret_cast<const char*>(bytes) + str_off[u], str_off[u + 1] - str_off[u]);
      UbiDecodeOne(a, src, index + item_off[u], item_off[u + 1] - item_off[u], out + item_off[u], &errs[u]);
    }
  });
  if (UbiFail(errs, k)) return 1;
  g_error.clear();
  return 0;
}

}  // extern "C"
