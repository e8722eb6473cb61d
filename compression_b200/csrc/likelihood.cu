// Rate term of training: log p(y) of a prior convolved with U(-1/2, 1/2), forward and backward, fused.
//
// Replaces the eager graph of UniformNoiseAdapter.log_prob (tensorflow_compression/python/distributions/
// uniform_noise.py:128-151) for the two prior families every model trains with:
//   * NoisyDeepFactorized with num_filters (3, 3) (deep_factorized.py:166-193): a per-channel 1-3-3-1 MLP gives the
//     CDF logits l(x); log_cdf = logsigmoid(l), log_sf = logsigmoid(-l);
//   * NoisyNormal / NoisyLogistic / NoisyLaplace: z = (x - loc) / scale and the standard log-CDF s(z).
// Both then take the graph's select
//   right = log_sf(y+.5) < log_cdf(y+.5);  big = right ? log_sf(y-.5) : log_cdf(y+.5);
//   small = right ? log_sf(y+.5) : log_cdf(y-.5);  out = isinf(big) ? big : log1p(-exp(small - big)) + big.
//
// Every element is computed in double from the float32 inputs and rounded once.  The value is a difference of two
// CDFs taken in the log domain: far in a tail, or with a scale much wider than a bin, the two logs agree in most of
// their digits, and float32 arithmetic there loses more than the output's own rounding.  The backward passes are the
// chain rule of the same graph, operation by operation, including torch.where's zero gradient for the branch not
// taken (so a NaN the graph makes in that branch, e.g. at y = +-inf, is made here too).
//
// Deep-factorized parameters arrive packed, already transformed, one row of kNumParams floats per channel:
//   [ 0.. 3) softplus(matrices[0])  [3, 1]     [15..18) biases[0] [3]     [22..25) tanh(factors[0]) [3]
//   [ 3..12) softplus(matrices[1])  [3, 3]     [18..21) biases[1] [3]     [25..28) tanh(factors[1]) [3]
//   [12..15) softplus(matrices[2])  [1, 3]     [21..22) biases[2] [1]
// (matrices row-major [out][in]).  Element i belongs to channel i mod C.  Thread mapping: a CTA holds R sub-rows of
// `cpb` consecutive channels, so consecutive threads read consecutive elements and every thread keeps one channel's
// parameters in registers for its whole grid-stride walk over rows.
//
// Backward of the parameters is deterministic: every thread accumulates its channel's 28 gradients in double over
// its rows, the CTA adds its sub-rows in a fixed order and writes one float partial row [C][28], and
// reduce_partials_kernel adds the CTAs' partials in double in CTA order.  The grid depends on n and C only.
#include <algorithm>

#include "common.cuh"

namespace tfcb {
namespace {

enum : int { kM0 = 0, kM1 = 3, kM2 = 12, kB0 = 15, kB1 = 18, kB2 = 21, kF0 = 22, kF1 = 25, kNumParams = 28 };

constexpr int kMaxThreads = 256;       // per CTA
constexpr int kFwdMaxCtas = 8192;      // per channel chunk, forward
constexpr int kBwdMaxCtas = 512;       // per channel chunk, backward: bounds the partials to 512 rows of [C][28]
constexpr int kBwdRowsPerThread = 4;   // at least this many rows per thread before another CTA is added

// ---- CTA geometry of the deep-factorized kernels --------------------------------------------------------------
struct DfGeometry {
  int cpb;       // consecutive channels per CTA
  int subrows;   // rows a CTA covers per step (R)
  int chunks;    // channel chunks (grid.y)
  int grid_x;    // CTAs per chunk
  int threads() const { return cpb * subrows; }
};

DfGeometry df_geometry(long long n, int C, bool backward) {
  DfGeometry g;
  const int parts = (C + kMaxThreads - 1) / kMaxThreads;
  g.cpb = (C + parts - 1) / parts;
  g.subrows = kMaxThreads / g.cpb;
  g.chunks = (C + g.cpb - 1) / g.cpb;
  const long long rows = n / C;
  const long long per_cta = (long long)g.subrows * (backward ? kBwdRowsPerThread : 1);
  const int cap = std::max(1, (backward ? kBwdMaxCtas : kFwdMaxCtas) / g.chunks);
  g.grid_x = (int)std::max(1LL, std::min<long long>((rows + per_cta - 1) / per_cta, cap));
  return g;
}

// ---- the graph's pieces, in double --------------------------------------------------------------------------
// torch's logsigmoid: min(x, 0) - log1p(exp(-|x|)); log_sigmoid_backward: max_deriv - sign * z / (1 + z).
__device__ __forceinline__ double log_sigmoid(double x, double z) { return fmin(x, 0.0) - log1p(z); }
__device__ __forceinline__ double d_log_sigmoid(double x, double z) {
  return x < 0.0 ? 1.0 - z / (1.0 + z) : z / (1.0 + z);
}

// The select and log-difference; returns the output value.
__device__ __forceinline__ double combine(double lsf_p, double lcdf_p, double lsf_m, double lcdf_m) {
  const bool right = lsf_p < lcdf_p;
  const double big = right ? lsf_m : lcdf_p, small = right ? lsf_p : lcdf_m;
  return isinf(big) ? big : log1p(-exp(small - big)) + big;
}

// Gradient of combine() with respect to its four inputs for upstream g, as torch's autograd of the graph computes
// it: where -> zero for the branch not taken, log1p -> g / (1 + (-e)), neg, exp -> * e, sub.
struct Grad4 {
  double lsf_p, lcdf_p, lsf_m, lcdf_m;
};
__device__ __forceinline__ Grad4 combine_grad(double lsf_p, double lcdf_p, double lsf_m, double lcdf_m, double g) {
  const bool right = lsf_p < lcdf_p;
  const double big = right ? lsf_m : lcdf_p, small = right ? lsf_p : lcdf_m;
  const bool inf = isinf(big);
  const double e = exp(small - big);
  const double gv = inf ? 0.0 : g;
  const double gd = -(gv / (1.0 - e)) * e;
  const double gbig = (inf ? g : 0.0) + gv - gd;
  Grad4 r;
  r.lsf_m = right ? gbig : 0.0;
  r.lcdf_p = right ? 0.0 : gbig;
  r.lsf_p = right ? gd : 0.0;
  r.lcdf_m = right ? 0.0 : gd;
  return r;
}

// ---- deep factorized ----------------------------------------------------------------------------------------
struct Mlp {
  double t0[3], a0[3], t1[3], a1[3];  // tanh(h) and h + f * tanh(h) of the two hidden layers
  double l;
};

__device__ __forceinline__ void mlp(const float (&w)[kNumParams], double x, Mlp& s) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double h = fma((double)w[kM0 + i], x, (double)w[kB0 + i]);
    s.t0[i] = tanh(h);
    s.a0[i] = fma((double)w[kF0 + i], s.t0[i], h);
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    double h = (double)w[kB1 + i];
#pragma unroll
    for (int j = 0; j < 3; ++j) h = fma((double)w[kM1 + 3 * i + j], s.a0[j], h);
    s.t1[i] = tanh(h);
    s.a1[i] = fma((double)w[kF1 + i], s.t1[i], h);
  }
  double l = (double)w[kB2];
#pragma unroll
  for (int j = 0; j < 3; ++j) l = fma((double)w[kM2 + j], s.a1[j], l);
  s.l = l;
}

// Backpropagates dl through the MLP at input x: accumulates the parameter gradients, returns dl/dx * dl.
__device__ __forceinline__ double mlp_backward(const float (&w)[kNumParams], double x, const Mlp& s, double dl,
                                               double (&acc)[kNumParams]) {
  acc[kB2] += dl;
  double g1[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    acc[kM2 + i] = fma(dl, s.a1[i], acc[kM2 + i]);
    const double ga = dl * (double)w[kM2 + i];
    acc[kF1 + i] = fma(ga, s.t1[i], acc[kF1 + i]);
    g1[i] = ga * fma((double)w[kF1 + i], 1.0 - s.t1[i] * s.t1[i], 1.0);
    acc[kB1 + i] += g1[i];
  }
  double dx = 0.0;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    double ga = 0.0;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      acc[kM1 + 3 * i + j] = fma(g1[i], s.a0[j], acc[kM1 + 3 * i + j]);
      ga = fma(g1[i], (double)w[kM1 + 3 * i + j], ga);
    }
    acc[kF0 + j] = fma(ga, s.t0[j], acc[kF0 + j]);
    const double g0 = ga * fma((double)w[kF0 + j], 1.0 - s.t0[j] * s.t0[j], 1.0);
    acc[kB0 + j] += g0;
    acc[kM0 + j] = fma(g0, x, acc[kM0 + j]);
    dx = fma(g0, (double)w[kM0 + j], dx);
  }
  return dx;
}

struct DfLogs {
  double lsf_p, lcdf_p, lsf_m, lcdf_m, z_p, z_m;
};
__device__ __forceinline__ DfLogs df_logs(double l_p, double l_m) {
  DfLogs r;
  r.z_p = exp(-fabs(l_p));
  r.z_m = exp(-fabs(l_m));
  const double L_p = log1p(r.z_p), L_m = log1p(r.z_m);
  r.lcdf_p = fmin(l_p, 0.0) - L_p;
  r.lsf_p = fmin(-l_p, 0.0) - L_p;
  r.lcdf_m = fmin(l_m, 0.0) - L_m;
  r.lsf_m = fmin(-l_m, 0.0) - L_m;
  return r;
}

// Channel and first row of this thread; false if the thread has no channel.
__device__ __forceinline__ bool df_lane(int C, int cpb, int* ch, long long* row) {
  const int sub = threadIdx.x / cpb;
  *ch = blockIdx.y * cpb + threadIdx.x % cpb;
  *row = (long long)blockIdx.x * (blockDim.x / cpb) + sub;
  return *ch < C;
}

__device__ __forceinline__ void load_params(const float* __restrict__ packed, int ch, float (&w)[kNumParams]) {
#pragma unroll
  for (int p = 0; p < kNumParams; ++p) w[p] = __ldg(packed + (long long)ch * kNumParams + p);
}

__global__ void __launch_bounds__(kMaxThreads)
noisy_df_fwd_kernel(const float* __restrict__ y, const float* __restrict__ packed, float* __restrict__ out,
                    long long rows, int C, int cpb) {
  int ch;
  long long r;
  if (!df_lane(C, cpb, &ch, &r)) return;
  float w[kNumParams];
  load_params(packed, ch, w);
  const long long stride = (long long)gridDim.x * (blockDim.x / cpb);
  for (; r < rows; r += stride) {
    const long long i = r * C + ch;
    const double x = (double)y[i];
    Mlp sp, sm;
    mlp(w, x + 0.5, sp);
    mlp(w, x - 0.5, sm);
    const DfLogs v = df_logs(sp.l, sm.l);
    out[i] = (float)combine(v.lsf_p, v.lcdf_p, v.lsf_m, v.lcdf_m);
  }
}

__global__ void __launch_bounds__(kMaxThreads)
noisy_df_bwd_kernel(const float* __restrict__ y, const float* __restrict__ packed, const float* __restrict__ dout,
                    float* __restrict__ dy, float* __restrict__ part, long long rows, int C, int cpb) {
  __shared__ double red[kMaxThreads];
  int ch;
  long long r;
  const bool active = df_lane(C, cpb, &ch, &r);
  double acc[kNumParams];
#pragma unroll
  for (int p = 0; p < kNumParams; ++p) acc[p] = 0.0;
  if (active) {
    float w[kNumParams];
    load_params(packed, ch, w);
    const long long stride = (long long)gridDim.x * (blockDim.x / cpb);
    for (; r < rows; r += stride) {
      const long long i = r * C + ch;
      const double x = (double)y[i];
      Mlp sp, sm;
      mlp(w, x + 0.5, sp);
      mlp(w, x - 0.5, sm);
      const DfLogs v = df_logs(sp.l, sm.l);
      const Grad4 g = combine_grad(v.lsf_p, v.lcdf_p, v.lsf_m, v.lcdf_m, (double)dout[i]);
      // log_cdf = logsigmoid(l), log_sf = logsigmoid(-l): each term's own logsigmoid backward, the zeros included
      const double dl_p = g.lcdf_p * d_log_sigmoid(sp.l, v.z_p) - g.lsf_p * d_log_sigmoid(-sp.l, v.z_p);
      const double dl_m = g.lcdf_m * d_log_sigmoid(sm.l, v.z_m) - g.lsf_m * d_log_sigmoid(-sm.l, v.z_m);
      const double dx = mlp_backward(w, x + 0.5, sp, dl_p, acc) + mlp_backward(w, x - 0.5, sm, dl_m, acc);
      dy[i] = (float)dx;
    }
  }
  // CTA partial: sub-rows of the same channel added in sub-row order
  const int subrows = blockDim.x / cpb;
  float* prow = part + (long long)blockIdx.x * C * kNumParams;
#pragma unroll
  for (int p = 0; p < kNumParams; ++p) {
    red[threadIdx.x] = acc[p];
    __syncthreads();
    if (threadIdx.x < cpb && active) {
      double s = 0.0;
      for (int k = 0; k < subrows; ++k) s += red[k * cpb + threadIdx.x];
      prow[(long long)ch * kNumParams + p] = (float)s;
    }
    __syncthreads();
  }
}

// ---- location-scale ---------------------------------------------------------------------------------------------
// s(z) = log CDF of the standard base and ds = what torch's backward of that expression gives.
template <int BASE>
struct Std;

template <>
struct Std<TFCB_NOISY_NORMAL> {  // torch's special_log_ndtr and its derivative formula
  static __device__ __forceinline__ double s(double x) {
    const double t = x * 0.70710678118654752440;
    return x < -1.0 ? log(erfcx(-t) / 2.0) - t * t : log1p(-erfc(t) / 2.0);
  }
  static __device__ __forceinline__ double ds(double x, double sx) {
    return exp(-(sx + x * x / 2.0)) / 2.50662827463100050242;  // sqrt(2 pi)
  }
};

template <>
struct Std<TFCB_NOISY_LOGISTIC> {
  static __device__ __forceinline__ double s(double x) { return log_sigmoid(x, exp(-fabs(x))); }
  static __device__ __forceinline__ double ds(double x, double) { return d_log_sigmoid(x, exp(-fabs(x))); }
};

template <>
struct Std<TFCB_NOISY_LAPLACE> {  // where(z < 0, log(.5) + z, log1p(-.5 exp(-|z|))), distributions.py
  static __device__ __forceinline__ double s(double x) {
    return x < 0.0 ? -0.69314718055994530942 + x : log1p(-0.5 * exp(-fabs(x)));
  }
  static __device__ __forceinline__ double ds(double x, double) {
    if (x < 0.0) return 1.0;
    const double e = exp(-fabs(x));  // NaN for NaN x
    const double sgn = x > 0.0 ? 1.0 : 0.0;  // abs's backward is sgn(x), 0 at 0
    return 0.5 * e * sgn / (1.0 - 0.5 * e);
  }
};

template <int BASE, bool BACKWARD>
__global__ void __launch_bounds__(kMaxThreads)
noisy_loc_scale_kernel(const float* __restrict__ y, const float* __restrict__ loc, int loc_scalar,
                       const float* __restrict__ scale, int scale_scalar, const float* __restrict__ dout,
                       float* __restrict__ out_or_dy, float* __restrict__ dloc, float* __restrict__ dscale,
                       long long n) {
  using B = Std<BASE>;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += stride) {
    const double x = (double)y[i];
    const double mu = (double)loc[loc_scalar ? 0 : i];
    const double sigma = (double)scale[scale_scalar ? 0 : i];
    const double d_p = x + 0.5 - mu, d_m = x - 0.5 - mu;
    const double z_p = d_p / sigma, z_m = d_m / sigma;
    const double lcdf_p = B::s(z_p), lsf_p = B::s(-z_p), lcdf_m = B::s(z_m), lsf_m = B::s(-z_m);
    if (!BACKWARD) {
      out_or_dy[i] = (float)combine(lsf_p, lcdf_p, lsf_m, lcdf_m);
      continue;
    }
    const Grad4 g = combine_grad(lsf_p, lcdf_p, lsf_m, lcdf_m, (double)dout[i]);
    const double gz_p = g.lcdf_p * B::ds(z_p, lcdf_p) - g.lsf_p * B::ds(-z_p, lsf_p);
    const double gz_m = g.lcdf_m * B::ds(z_m, lcdf_m) - g.lsf_m * B::ds(-z_m, lsf_m);
    const double gd = gz_p / sigma + gz_m / sigma;  // z = (x - loc) / scale, per evaluation
    out_or_dy[i] = (float)gd;
    if (dloc) dloc[i] = (float)-gd;
    if (dscale) dscale[i] = (float)(-(gz_p * d_p) / (sigma * sigma) - (gz_m * d_m) / (sigma * sigma));
  }
}

int check_df(const float* packed, long long n, int C) {
  if (C <= 0 || n < 0) return fail(TFCB_INVALID_ARGUMENT, "bad deep-factorized shape: n=%lld C=%d", n, C);
  if (n % C != 0) return fail(TFCB_INVALID_ARGUMENT, "n=%lld is not a multiple of C=%d", n, C);
  if (!packed) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  return TFCB_OK;
}

int check_loc_scale(int base, long long n) {
  if (base != TFCB_NOISY_NORMAL && base != TFCB_NOISY_LOGISTIC && base != TFCB_NOISY_LAPLACE)
    return fail(TFCB_INVALID_ARGUMENT, "unknown location-scale base %d", base);
  if (n < 0) return fail(TFCB_INVALID_ARGUMENT, "bad location-scale size: n=%lld", n);
  return TFCB_OK;
}

int loc_scale_grid(long long n) { return (int)std::min<long long>((n + kMaxThreads - 1) / kMaxThreads, kFwdMaxCtas); }

}  // namespace
}  // namespace tfcb

using namespace tfcb;

#define DISPATCH_BASE(base, ...)                                                  \
  switch (base) {                                                                 \
    case TFCB_NOISY_NORMAL: { constexpr int BASE = TFCB_NOISY_NORMAL; __VA_ARGS__; } break;     \
    case TFCB_NOISY_LOGISTIC: { constexpr int BASE = TFCB_NOISY_LOGISTIC; __VA_ARGS__; } break; \
    default: { constexpr int BASE = TFCB_NOISY_LAPLACE; __VA_ARGS__; } break;                   \
  }

extern "C" {

int64_t tfcb_noisy_deep_factorized_workspace_bytes(int64_t n, int C) {
  if (C <= 0 || n <= 0) return 0;
  const DfGeometry g = df_geometry(n, C, true);
  return (int64_t)g.grid_x * C * kNumParams * (int64_t)sizeof(float);
}

int tfcb_noisy_deep_factorized_log_prob(const float* y_dev, const float* packed_dev, float* out_dev, int64_t n, int C,
                                        void* stream) {
  TFCB_TRY(check_df(packed_dev, n, C));
  if (n == 0) return TFCB_OK;
  if (!y_dev || !out_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  const DfGeometry g = df_geometry(n, C, false);
  noisy_df_fwd_kernel<<<dim3(g.grid_x, g.chunks), g.threads(), 0, as_stream(stream)>>>(y_dev, packed_dev, out_dev,
                                                                                      n / C, C, g.cpb);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

int tfcb_noisy_deep_factorized_log_prob_backward(const float* y_dev, const float* packed_dev, const float* dout_dev,
                                                 float* dy_dev, float* dpacked_dev, void* workspace_dev, int64_t n,
                                                 int C, void* stream) {
  TFCB_TRY(check_df(packed_dev, n, C));
  if (!dpacked_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  cudaStream_t s = as_stream(stream);
  if (n == 0) {
    TFCB_CUDA_TRY(cudaMemsetAsync(dpacked_dev, 0, (size_t)C * kNumParams * sizeof(float), s));
    return TFCB_OK;
  }
  if (!y_dev || !dout_dev || !dy_dev || !workspace_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  const DfGeometry g = df_geometry(n, C, true);
  float* part = reinterpret_cast<float*>(workspace_dev);
  noisy_df_bwd_kernel<<<dim3(g.grid_x, g.chunks), g.threads(), 0, s>>>(y_dev, packed_dev, dout_dev, dy_dev, part,
                                                                     n / C, C, g.cpb);
  const long long np = (long long)C * kNumParams;
  reduce_partials_kernel<<<(unsigned)((np + 255) / 256), 256, 0, s>>>(part, g.grid_x, np, dpacked_dev);
  TFCB_LAUNCHED();
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

int tfcb_noisy_loc_scale_log_prob(int base, const float* y_dev, const float* loc_dev, int loc_scalar,
                                  const float* scale_dev, int scale_scalar, float* out_dev, int64_t n, void* stream) {
  TFCB_TRY(check_loc_scale(base, n));
  if (n == 0) return TFCB_OK;
  if (!y_dev || !loc_dev || !scale_dev || !out_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  DISPATCH_BASE(base, {
    noisy_loc_scale_kernel<BASE, false><<<loc_scale_grid(n), kMaxThreads, 0, as_stream(stream)>>>(
        y_dev, loc_dev, loc_scalar, scale_dev, scale_scalar, nullptr, out_dev, nullptr, nullptr, n);
  });
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

int tfcb_noisy_loc_scale_log_prob_backward(int base, const float* y_dev, const float* loc_dev, int loc_scalar,
                                           const float* scale_dev, int scale_scalar, const float* dout_dev,
                                           float* dy_dev, float* dloc_dev, float* dscale_dev, int64_t n,
                                           void* stream) {
  TFCB_TRY(check_loc_scale(base, n));
  if (n == 0) return TFCB_OK;
  if (!y_dev || !loc_dev || !scale_dev || !dout_dev || !dy_dev) return fail(TFCB_INVALID_ARGUMENT, "null pointer");
  DISPATCH_BASE(base, {
    noisy_loc_scale_kernel<BASE, true><<<loc_scale_grid(n), kMaxThreads, 0, as_stream(stream)>>>(
        y_dev, loc_dev, loc_scalar, scale_dev, scale_scalar, dout_dev, dy_dev, dloc_dev, dscale_dev, n);
  });
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

}  // extern "C"
