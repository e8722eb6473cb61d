// The interface between the GDN entry points (gdn.cu) and the tensor-core kernels (gdn_tc.cu), and the host helpers
// both use.
#pragma once
#include "common.cuh"

namespace tfcb {

// Per-CTA dgamma / dbeta partials the backward workspace holds: no dgamma grid, and no dx grid that writes a partial
// or a scratch tile per CTA, has more CTAs.
constexpr int kMaxParts = 148;

// Which kernels take a configuration: none (the CUDA-core kernels of gdn.cu, or the entry rejects it), the fixed-
// exponent tensor-core kernels gdn_tc_* (fast: their branch-free variant for alpha = epsilon = 1 without
// rectification) or the literal-pow ones gdn_tc_pow_*.  Also the configuration it was made for.
struct TcRoute {
  enum Family { kNone, kFixed, kPow } family;
  bool fast;
  int C, dtype, flags;  // dtype of the activations: 0 float32, 1 float16, 2 bfloat16
  float alpha, eps;
};

// Float32 at C in {128, 192, 256, 320} with any exponents, float16 / bfloat16 at C in {128, 192} with alpha in {1, 2}
// and epsilon in {1, 1/2}; nothing under TFCB_GDN_FP32=1 (read on every call).  Pointer alignment is the caller's.
TcRoute gdn_tc_route(int C, int dtype, int flags, float alpha, float eps);

// y for a route other than kNone, n_pix > 0.  Channels-first: x and y are [n_pix / S, C, S].
int gdn_tc_forward(const TcRoute& r, bool channels_first, const void* x, const float* gamma, const float* beta, void* y,
                   long long n_pix, long long S, cudaStream_t s);

// dx, q and the per-CTA partials part_g [*n_parts][C][C] and part_b [*n_parts][C] for a route other than kNone,
// n_pix > 0, in dx's and dy's layout as for gdn_tc_forward.  The literal-pow kernels also write the exponent partials
// part_e [*n_parts_e][2] when part_e is not null.  At C = 128 / 192 with 16-bit or channels-first activations the dx
// kernel keeps its direct term in `scratch`, gdn_tc_scratch_floats(n_pix, C) floats.
int gdn_tc_backward(const TcRoute& r, bool channels_first, const void* x, const float* gamma, const float* beta,
                    const void* dy, void* dx, float* q, float* part_g, float* part_b, float* part_e, float* scratch,
                    long long n_pix, long long S, cudaStream_t s, int* n_parts, int* n_parts_e);
long long gdn_tc_scratch_floats(long long n_pix, int C);

// The persistent grids are sized by the SM count, so the partials, and the order they are summed in, depend on it.
inline int sm_count() {
  int dev = 0, n = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  return n > 0 ? n : 1;
}

template <class... P>
bool aligned16(P... p) {
  return ((reinterpret_cast<uintptr_t>(p) | ...) & 15) == 0;
}

template <typename K>
int set_smem(K kernel, size_t bytes) {
  TFCB_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return TFCB_OK;
}

}  // namespace tfcb
