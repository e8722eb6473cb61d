/* ORACLE / TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
 *
 * Plain-C restatement ("port") of the UnboundedIndexRangeEncode / UnboundedIndexRangeDecode op loops
 * (cc/kernels/unbounded_index_range_coding_kernels.cc).  The range coder itself is the port's (oracle/port/tfc_port.c,
 * included here so that its static coder routines are shared rather than copied); the library built from this file
 * also exports everything tfc_port.c does.  Pinned to the compiled reference by tests/test_unbounded_oracle_cpu.py.
 */
#include "../port/tfc_port.c"

/* ------------------------------------------------------------------------------------------ */
/* public: UnboundedIndexRangeEncode / Decode (unbounded_index_range_coding_kernels.cc).  Any input on which the */
/* reference's int32 arithmetic or shifts are undefined, or its width prefix need not end, returns an error.    */
/* ------------------------------------------------------------------------------------------ */
typedef struct {
  const int32_t* cdf;
  int64_t R, W;
  const int32_t* cdf_size;
  const int32_t* offset;
  int precision, w;
} ubi_t;

static int ubi_debug_check(const ubi_t* a, const int32_t* index, int64_t n) {
  for (int64_t i = 0; i < n; ++i)
    if (index[i] < 0 || index[i] >= a->R) {
      snprintf(g_err, sizeof g_err, "'index' has a value not in [0, %lld): value=%d", (long long)a->R, index[i]);
      return 1;
    }
  for (int64_t r = 0; r < a->R; ++r)
    if (a->cdf_size[r] < 3 || a->cdf_size[r] > a->W) {
      snprintf(g_err, sizeof g_err, "'cdf_size' has a value not in [3, %lld]: value=%d", (long long)a->W,
               a->cdf_size[r]);
      return 1;
    }
  for (int64_t r = 0; r < a->R; ++r) {
    const int32_t* row = a->cdf + r * a->W;
    const int32_t sz = a->cdf_size[r];
    if (row[0] != 0 || row[sz - 1] != (1 << a->precision)) {
      snprintf(g_err, sizeof g_err, "Each cdf should start from 0 and end at %d: cdf[0]=%d, cdf[^1]=%d",
               1 << a->precision, row[0], row[sz - 1]);
      return 1;
    }
    for (int32_t j = 0; j + 1 < sz; ++j)
      if (row[j + 1] <= row[j]) return fail("CDF is not monotonic");
  }
  return 0;
}

static const int32_t* ubi_row(const ubi_t* a, int32_t r, int32_t* m) {
  if (r < 0 || r >= a->R) {
    snprintf(g_err, sizeof g_err, "'index' has a value not in [0, %lld): value=%d", (long long)a->R, r);
    return NULL;
  }
  if (a->cdf_size[r] < 3 || a->cdf_size[r] > a->W) {
    snprintf(g_err, sizeof g_err, "'cdf_size' has a value not in [3, %lld]: value=%d", (long long)a->W,
             a->cdf_size[r]);
    return NULL;
  }
  *m = a->cdf_size[r] - 2;
  return a->cdf + (int64_t)r * a->W;
}

static int ubi_encode_one(const ubi_t* a, const int32_t* data, const int32_t* index, int64_t n, sink_t* s) {
  const int K = (32 + a->w - 1) / a->w;
  const uint32_t M = (1u << a->w) - 1u;
  enc_t e;
  enc_init(&e);
  for (int64_t i = 0; i < n; ++i) {
    int32_t m;
    const int32_t* row = ubi_row(a, index[i], &m);
    if (!row) return 1;
    const int64_t d = (int64_t)data[i] - a->offset[index[i]];
    if (d < INT32_MIN || d > INT32_MAX) return fail("undefined in the reference: data - offset overflows int32");
    int64_t v = d;
    uint32_t u = 0;
    if (d < 0) {
      if (d <= -(1ll << 30)) return fail("undefined in the reference: -2 * (data - offset) - 1 overflows int32");
      u = (uint32_t)(-2 * d - 1);
      v = m;
    } else if (d >= m) {
      if (d - m >= (1ll << 30))
        return fail("undefined in the reference: 2 * (data - offset - max_value) overflows int32");
      u = (uint32_t)(2 * (d - m));
      v = m;
    }
    const int32_t lo = row[v], hi = row[v + 1];
    if (!(0 <= lo && lo < hi && hi <= (1 << a->precision)))
      return fail("symbol with zero probability or a CDF row beyond 2^precision");
    enc_put(&e, s, lo, hi, a->precision);
    if (v == m) {
      if ((u >> ((K - 1) * a->w)) != 0)
        return fail("undefined in the reference: the overflow width loop shifts by 32 or more");
      uint32_t widths = 0;
      while ((u >> (widths * a->w)) != 0) ++widths;
      uint32_t rest = widths;
      for (; rest >= M; rest -= M) enc_put(&e, s, (int32_t)M, (int32_t)M + 1, a->w);
      enc_put(&e, s, (int32_t)rest, (int32_t)rest + 1, a->w);
      for (uint32_t j = 0; j < widths; ++j) {
        const uint32_t digit = (u >> (j * a->w)) & M;
        enc_put(&e, s, (int32_t)digit, (int32_t)digit + 1, a->w);
      }
    }
  }
  enc_flush(&e, s);
  return 0;
}

static int ubi_decode_one(const ubi_t* a, const uint8_t* bytes, int64_t nbytes, const int32_t* index, int64_t n,
                          const int32_t* uniform, int32_t* out) {
  const uint32_t K = (32u + (uint32_t)a->w - 1u) / (uint32_t)a->w;
  const uint32_t M = (1u << a->w) - 1u;
  dec_t d;
  dec_init(&d, bytes, (size_t)nbytes);
  for (int64_t i = 0; i < n; ++i) {
    int32_t m;
    const int32_t* row = ubi_row(a, index[i], &m);
    if (!row) return 1;
    int64_t v = dec_get(&d, row, m + 2, a->precision, 0);
    if (v == m) {
      uint32_t widths = 0, val;
      do {
        val = (uint32_t)dec_get(&d, uniform, (int64_t)M + 2, a->w, 0);
        widths += val;
        if (widths > K) {
          snprintf(g_err, sizeof g_err, "undefined in the reference: overflow width prefix longer than %u digits", K);
          return 1;
        }
      } while (val == M);
      uint32_t u = 0;
      for (uint32_t j = 0; j < widths; ++j) u |= (uint32_t)dec_get(&d, uniform, (int64_t)M + 2, a->w, 0) << (j * a->w);
      v = (int64_t)(u >> 1);
      if (u & 1u) {
        v = -v - 1;
      } else {
        v += m;
        if (v > INT32_MAX) return fail("undefined in the reference: overflow / 2 + max_value overflows int32");
      }
    }
    v += a->offset[index[i]];
    if (v < INT32_MIN || v > INT32_MAX) return fail("undefined in the reference: value + offset overflows int32");
    out[i] = (int32_t)v;
  }
  return 0;
}

static int ubi_item_fail(int64_t k, int64_t u) {
  if (k > 1) {
    char msg[sizeof g_err];
    snprintf(msg, sizeof msg, "string %lld: %.200s", (long long)u, g_err);
    memcpy(g_err, msg, sizeof g_err);
  }
  return 1;
}

/* Same contract as the reference flavour's tfcref_unbounded_encode; `threads` is ignored (one thread). */
int tfcport_unbounded_encode(const int32_t* data, const int32_t* index, const int64_t* item_off, int64_t k,
                             const int32_t* cdf, int64_t R, int64_t W, const int32_t* cdf_size, const int32_t* offset,
                             int precision, int w, int debug_level, int threads, int64_t* str_off, uint8_t* out,
                             int64_t out_cap) {
  (void)threads;
  const ubi_t a = {cdf, R, W, cdf_size, offset, precision, w};
  if (debug_level > 0 && ubi_debug_check(&a, index, item_off[k])) return 1;
  sink_t s = {0, 0, 0};
  str_off[0] = 0;
  for (int64_t u = 0; u < k; ++u) {
    if (ubi_encode_one(&a, data + item_off[u], index + item_off[u], item_off[u + 1] - item_off[u], &s)) {
      free(s.p);
      return ubi_item_fail(k, u);
    }
    str_off[u + 1] = (int64_t)s.n;
  }
  int rc = 0;
  if ((int64_t)s.n > out_cap) rc = 2;
  else if (s.n) memcpy(out, s.p, s.n);
  free(s.p);
  if (!rc) g_err[0] = 0;
  return rc;
}

int tfcport_unbounded_decode(const uint8_t* bytes, const int64_t* str_off, int64_t k, const int32_t* index,
                             const int64_t* item_off, const int32_t* cdf, int64_t R, int64_t W, const int32_t* cdf_size,
                             const int32_t* offset, int precision, int w, int debug_level, int threads, int32_t* out) {
  (void)threads;
  const ubi_t a = {cdf, R, W, cdf_size, offset, precision, w};
  if (debug_level > 0 && ubi_debug_check(&a, index, item_off[k])) return 1;
  const int64_t nu = ((int64_t)1 << w) + 1;
  int32_t* uniform = (int32_t*)malloc((size_t)nu * sizeof(int32_t));
  for (int64_t j = 0; j < nu; ++j) uniform[j] = (int32_t)j;
  int rc = 0;
  for (int64_t u = 0; u < k && !rc; ++u)
    if (ubi_decode_one(&a, bytes + str_off[u], str_off[u + 1] - str_off[u], index + item_off[u],
                       item_off[u + 1] - item_off[u], uniform, out + item_off[u]))
      rc = ubi_item_fail(k, u);
  free(uniform);
  if (!rc) g_err[0] = 0;
  return rc;
}
