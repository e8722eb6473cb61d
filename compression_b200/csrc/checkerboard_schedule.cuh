// The checkerboard schedule (He et al. 2021) shared by checkerboard.cu and cb_mixture.cu: the 12 context taps, the
// j-th position of a colour, the checkerboard.cuh schedule policy, the positions of a colour of an image list and the
// upload of a ragged list's image table.  A position (r, c) is an anchor (colour 0) when r + c is even, else a
// non-anchor (colour 1).
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "autoregressive.cuh"
#include "checkerboard.cuh"
#include "common.cuh"

namespace tfcb {
namespace {

// the checkerboard taps in raster order: (dy, dx) in [-2, 2]^2 with dy + dx odd
__constant__ int8_t c_cb_dy[kArTaps] = {-2, -2, -1, -1, -1, 0, 0, 1, 1, 1, 2, 2};
__constant__ int8_t c_cb_dx[kArTaps] = {-1, 1, -2, 0, 2, -1, 1, -2, 0, 2, -1, 1};

// the j-th position of colour k of an image of width W, in raster order
__host__ __device__ inline void cb_position(long long j, int W, int k, int* r, int* c) {
  const long long pair = j / W;
  const int rem = (int)(j - pair * W), even = (W + 1 - k) / 2;  // positions of colour k in an even row
  if (rem < even) {
    *r = (int)(2 * pair);
    *c = 2 * rem + k;
  } else {
    *r = (int)(2 * pair + 1);
    *c = 2 * (rem - even) + 1 - k;
  }
}

// The checkerboard's schedule for checkerboard.cuh: pass `colour` (0 anchors, 1 non-anchors), the 12 taps of odd
// parity whatever the colour (only the non-anchor pass reads taps).
struct CbSchedule {
  __device__ static void position(long long j, int W, int colour, int* r, int* c) { cb_position(j, W, colour, r, c); }
  __device__ static int8_t dy(int, int t) { return c_cb_dy[t]; }
  __device__ static int8_t dx(int, int t) { return c_cb_dx[t]; }
};

long long cb_count(int64_t H, int64_t W, int colour) { return colour ? H * W / 2 : (H * W + 1) / 2; }

long long cb_positions(const CbList& L, int colour) {
  if (!L.hs) return L.B * cb_count(L.H, L.W, colour);
  long long n = 0;
  for (int64_t i = 0; i < L.B; ++i) n += cb_count(L.hs[i], L.ws[i], colour);
  return n;
}

}

// Uploads the image table of colour `colour` of group [o, o + C) of a ragged list to `work` (one stream-ordered copy
// from pageable memory, staged before the call returns).  Params outputs of image i start at C Q_i (whole == 0), or at
// M P_i + H_i W_i o + (colour ? n_a,i C : 0) in the coding order of every group (whole != 0).
int cb_upload_table(const CbList& L, int M, int o, int C, int colour, int whole, float* work, cudaStream_t s) {
  std::vector<CbImage> t((size_t)L.B);
  long long q = 0, pix = 0;
  for (int64_t i = 0; i < L.B; ++i) {
    const int64_t H = L.hs[i], W = L.ws[i];
    t[i].q = q;
    t[i].pix = pix;
    t[i].out = whole ? M * pix + H * W * o + (colour ? cb_count(H, W, 0) * C : 0) : C * q;
    t[i].H = (int)H;
    t[i].W = (int)W;
    q += cb_count(H, W, colour);
    pix += H * W;
  }
  TFCB_CUDA_TRY(cudaMemcpyAsync(work, t.data(), t.size() * sizeof(CbImage), cudaMemcpyHostToDevice, s));
  return TFCB_OK;
}  // namespace
}  // namespace tfcb
