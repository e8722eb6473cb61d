// What the joint autoregressive prior (autoregressive.cu) and the checkerboard and space-channel context models
// (checkerboard.cu) share: the packed parameter layout, the constants of the fixed reduction order, the table-index
// conversion, the packing copies and the argument checks.  Both files' kernels compute every dense output in the
// order of autoregressive.cu's file comment; with one channel group they read the same packed buffer
// (tfcb_ar_pack_weights).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kArSlices = 8;      // input slices per dense output (the fixed reduction order)
constexpr int kArTaps = 12;       // context taps: the causal ones of a 5x5 type-A mask, or the checkerboard ones
constexpr int kArMaxM = 384;
constexpr float kArLeakySlope = 0.01f;

struct ArDims {
  int M, N2, N3, N4;
  long long wc, bc, w1, b1, w2, b2, w3, b3, total;  // offsets into the packed buffer, in floats
};

__host__ __device__ inline ArDims ar_dims(int M) {
  ArDims d;
  d.M = M;
  d.N2 = 2 * M;
  d.N3 = 10 * M / 3;
  d.N4 = 8 * M / 3;
  d.wc = 0;
  d.bc = d.wc + (long long)kArTaps * M * d.N2;
  d.w1 = d.bc + d.N2;
  d.b1 = d.w1 + 4ll * M * d.N3;
  d.w2 = d.b1 + d.N3;
  d.b2 = d.w2 + (long long)d.N3 * d.N4;
  d.w3 = d.b2 + d.N4;
  d.b3 = d.w3 + (long long)d.N4 * d.N2;
  d.total = d.b3 + d.N2;
  return d;
}

// ContinuousIndexedEntropyModel._normalize_indexes (maximum with 0, minimum with num_scales - 1, both NaN-
// propagating like torch.maximum / minimum) followed by .to(torch.int32) on the GPU (truncation; NaN -> 0).
__device__ __forceinline__ int32_t ar_table_index(float s, int num_scales) {
  float v = (s != s) ? s : fmaxf(s, 0.f);
  v = (v != v) ? v : fminf(v, (float)(num_scales - 1));
  return (int32_t)v;
}

int ar_check_batch(int64_t B, int64_t H, int64_t W, int num_scales) {
  if (B <= 0 || B > 0x7FFFFFFF) return fail(TFCB_INVALID_ARGUMENT, "batch size %lld out of range", (long long)B);
  if (H <= 0 || W <= 0 || H * W > 0x7FFFFFFF)
    return fail(TFCB_INVALID_ARGUMENT, "latent shape %lld x %lld out of range", (long long)H, (long long)W);
  if (num_scales < 1) return fail(TFCB_INVALID_ARGUMENT, "num_scales=%d must be positive", num_scales);
  return TFCB_OK;
}

// A latent shape of a ragged list: positive sides and H W <= 2^31 - 1.
bool ar_shape_ok(int64_t H, int64_t W) { return H > 0 && W > 0 && H <= 0x7FFFFFFF && W <= 0x7FFFFFFF / H; }

bool ar_list_ok(int64_t n, const int64_t* hs, const int64_t* ws) {
  if (n <= 0 || n > 0x7FFFFFFF || !hs || !ws) return false;
  for (int64_t i = 0; i < n; ++i)
    if (!ar_shape_ok(hs[i], ws[i])) return false;
  return true;
}

// A ragged list of n images of latent shapes hs[i] x ws[i] (host arrays) and num_scales.
int ar_check_list(int64_t n, const int64_t* hs, const int64_t* ws, int num_scales) {
  if (n <= 0 || n > 0x7FFFFFFF) return fail(TFCB_INVALID_ARGUMENT, "a list of %lld images", (long long)n);
  if (!hs || !ws) return fail(TFCB_INVALID_ARGUMENT, "`heights` or `widths` is null");
  for (int64_t i = 0; i < n; ++i)
    if (!ar_shape_ok(hs[i], ws[i]))
      return fail(TFCB_INVALID_ARGUMENT, "image %lld: latent shape %lld x %lld out of range", (long long)i,
                  (long long)hs[i], (long long)ws[i]);
  if (num_scales < 1) return fail(TFCB_INVALID_ARGUMENT, "num_scales=%d must be positive", num_scales);
  return TFCB_OK;
}

int ar_check_packed(int M, const float* packed, int64_t packed_floats) {
  if (M <= 0 || M % 6 != 0 || M > kArMaxM)
    return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be a positive multiple of 6 and at most %d", M,
                kArMaxM);
  if (!packed) return fail(TFCB_INVALID_ARGUMENT, "`packed` is null");
  if (packed_floats != ar_dims(M).total)
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, M=%d needs %lld", (long long)packed_floats,
                M, (long long)ar_dims(M).total);
  return TFCB_OK;
}

int ar_check(int M, const float* packed, int64_t packed_floats, int64_t B, int64_t H, int64_t W, int num_scales) {
  TFCB_TRY(ar_check_packed(M, packed, packed_floats));
  return ar_check_batch(B, H, W, num_scales);
}

// A ragged list's per-image table, at least `need` floats of workspace: null and misaligned workspaces are refused.
int ar_check_table_space(const void* work, int64_t work_floats, long long need, size_t align) {
  if (!work || work_floats < need)
    return fail(TFCB_INVALID_ARGUMENT, "workspace of %lld floats, this call needs %lld",
                work ? (long long)work_floats : 0ll, need);
  if (reinterpret_cast<uintptr_t>(work) % align)
    return fail(TFCB_INVALID_ARGUMENT, "the workspace must be %d-byte aligned", (int)align);
  return TFCB_OK;
}

// Stream-ordered device copies of the eight weight operands (context weights, bias, W1, b1, W2, b2, W3, b3) into
// `packed` at the offsets at[i], each at[i + 1] - at[i] floats long.
int ar_pack_segments(const float* const src[8], const long long at[9], float* packed, cudaStream_t s) {
  for (int i = 0; i < 8; ++i)
    if (!src[i]) return fail(TFCB_INVALID_ARGUMENT, "weight operand %d is null", i);
  if (!packed) return fail(TFCB_INVALID_ARGUMENT, "`packed` is null");
  for (int i = 0; i < 8; ++i)
    TFCB_CUDA_TRY(cudaMemcpyAsync(packed + at[i], src[i], (at[i + 1] - at[i]) * sizeof(float),
                                  cudaMemcpyDeviceToDevice, s));
  return TFCB_OK;
}

int ar_check_range(int64_t p0, int64_t p1, int64_t H, int64_t W) {
  if (p0 < 0 || p1 < p0 || p1 > H * W)
    return fail(TFCB_INVALID_ARGUMENT, "positions [%lld, %lld) outside [0, %lld)", (long long)p0, (long long)p1,
                (long long)(H * W));
  return TFCB_OK;
}

}  // namespace
}  // namespace tfcb
