// Joint autoregressive + hierarchical prior (Minnen, Ballé & Toderici 2018) on sm_90a: the entropy parameters of
// one latent position from its causal neighbours and the hyper feature, and the serial encoder / decoder loops over
// positions that need them.
//
// Per position p of an image with latents [H, W, M] (N2 = 2M, N3 = 10M/3, N4 = 8M/3):
//   ctx   = bc + Wc · gather(ŷ, the 12 taps of a 5x5 type-A mask)          [12M] -> [2M]
//   h1    = leaky(b1 + W1 · [ψ_p, ctx])                                     [4M]  -> [N3]
//   h2    = leaky(b2 + W2 · h1)                                             [N3]  -> [N4]
//   out   = b3 + W3 · h2 = [loc, scale_index]                               [N4]  -> [2M]
//   index = int32(min(max(scale_index, 0), num_scales - 1))   (the entropy model's _normalize_indexes + cast)
// Encoder: ŷ_p = float(int32(rint(y_p - loc))) + loc, the f32 coder's own dequantisation of the symbol it codes;
// the table indexes and locs of all positions go to ONE index-mode encode afterwards.  Decoder: the M symbols of p
// are decoded from the stream's saved state with the decode kernels' Dec2 recurrence (range_decoder.cuh) and
// dequantised as tfcb_decode_index_f32 does: float(sym + cdf_offset[index]) + loc.
//
// One CTA per image runs every position of its range in order: an image depends only on its own ŷ, so the loop
// needs no inter-CTA synchronisation, no host round trip and one launch.  Batch invariance is structural: CTA b
// reads only image b, and every output of a dense layer is computed by a fixed sequence of float32 operations that
// depends on the layer's shape alone (not on B, blockIdx, blockDim or the SM count):
//   out[j] = ((((bias[j] + P_0[j]) + P_1[j]) + ...) + P_7[j]),  P_s[j] = fma chain over k in [s*K/8, (s+1)*K/8)
//   in increasing k starting from 0.f, where K is the layer's input width.
#include <cuda_runtime.h>

#include <vector>

#include "autoregressive.cuh"
#include "common.cuh"
#include "range_decoder.cuh"

namespace tfcb {
namespace {

constexpr int kArThreads = 512;

enum : int { kArParams = 0, kArEncode = 1, kArDecode = 2 };

// floats of shared memory for activations: gathered taps, [ψ, ctx], h1, h2, out, and the slice partials
__host__ __device__ inline long long ar_act_floats(const ArDims& d) {
  return (long long)kArTaps * d.M + 2ll * d.N2 + d.N3 + d.N4 + d.N2 + (long long)kArSlices * d.N3;
}

// One image of a ragged list: its first pixel P_i (its elements start at M P_i) and its shape.
struct ArImage {
  long long pix;
  int H, W;
};

struct ArParams {
  const float* packed;
  const float* psi;    // [B, HW, 2M]
  const float* y;      // encoder: [B, HW, M]
  float* yhat;         // [B, HW, M]: read at earlier positions, written at the range's positions (not in params mode)
  float* loc_out;      // params: [B, M]; encoder: [B, HW, M]; optional in both
  float* scale_out;    // same layout, optional
  int32_t* index_out;  // same layout, optional
  const int32_t* cdf_offset;  // decoder: [n_rows]
  int H, W, M, num_scales;
  int p0, p1;
  // decoder
  const uint2* pairs;
  const int4* rows4;
  int n_rows;
  long long n_pairs;
  const uint8_t* bytes;
  const long long* offsets;
  DecState* state;
  const ArImage* img;  // ragged list: CTA b runs every position of image b (§3.13)
};

// out[j] for j < nout, in the fixed order of the file comment.  `in` and `out` are shared; W is [nin][nout].
__device__ __forceinline__ void ar_dense(const float* in, int nin, const float* __restrict__ W,
                                         const float* __restrict__ bias, int nout, float* part, float* out,
                                         bool leaky) {
  for (int item = threadIdx.x; item < kArSlices * nout; item += blockDim.x) {
    const int s = item / nout, j = item - s * nout;
    const int k0 = s * nin / kArSlices, k1 = (s + 1) * nin / kArSlices;
    const float* w = W + (long long)k0 * nout + j;
    float acc = 0.f;
#pragma unroll 8
    for (int k = k0; k < k1; ++k, w += nout) acc = __fmaf_rn(in[k], __ldg(w), acc);
    part[s * nout + j] = acc;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < nout; j += blockDim.x) {
    float v = __ldg(bias + j);
#pragma unroll
    for (int s = 0; s < kArSlices; ++s) v = __fadd_rn(v, part[s * nout + j]);
    if (leaky) v = v > 0.f ? v : __fmul_rn(v, kArLeakySlope);
    out[j] = v;
  }
  __syncthreads();
}

// The CTA of image b: positions [P.p0, P.p1) of B images of P.H × P.W, or (RAGGED) every position of image b of the
// list P.img.
template <int MODE, bool SMEM_KEYS, bool RAGGED>
__device__ __forceinline__ void ar_body(const ArParams& P) {
  extern __shared__ __align__(16) float s_act[];
  __shared__ __align__(16) uint16_t ring_buf[2 * kRing];  // decoder only: 4096-byte aligned ring, as decode_kernel
  const ArDims d = ar_dims(P.M);
  const int M = P.M;
  const long long b = blockIdx.x;
  const long long HW = (long long)P.H * P.W;
  // a ragged list's image b (the fixed-shape arithmetic below is left exactly as it was when RAGGED is false)
  ArImage im{};
  if (RAGGED) im = P.img[b];
  const long long pix0 = RAGGED ? im.pix : b * HW;  // the image's first pixel
  float* const taps = s_act;                    // [12M]
  float* const x1 = taps + kArTaps * M;         // [4M]: ψ then ctx
  float* const h1 = x1 + 2 * d.N2;              // [N3]
  float* const h2 = h1 + d.N3;                  // [N4]
  float* const out = h2 + d.N4;                 // [2M]: loc then scale_index
  float* const part = out + d.N2;               // [8 * N3]
  const float* const Wp = P.packed;

  // decoder state (warp 0 only; replicated across its lanes like the decode kernel's chain warp)
  const uint2* pairs = P.pairs;
  const int4* rows4 = P.rows4;
  uint16_t* ring = nullptr;
  Dec2 c;
  ByteWindow bw;
  long long filled = 0;
  const int lane = threadIdx.x & 31;
  if (MODE == kArDecode) {
    if (SMEM_KEYS) {
      uint2* sp = reinterpret_cast<uint2*>(part + (long long)kArSlices * d.N3);
      int4* sr = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(sp) + ((P.n_pairs * 8 + 15) & ~15ll));
      for (long long i = threadIdx.x; i < P.n_pairs; i += blockDim.x) sp[i] = P.pairs[i];
      for (int i = threadIdx.x; i < P.n_rows; i += blockDim.x) sr[i] = P.rows4[i];
      pairs = sp;
      rows4 = sr;
      __syncthreads();
    }
    ring = ring_buf + (((4096u - (smem_addr(ring_buf) & 4095u)) & 4095u) >> 1);
    if (threadIdx.x < 32) {
      bw.p = P.bytes + P.offsets[b];
      bw.len = P.offsets[b + 1] - P.offsets[b];
      const DecState st = P.state[b];
      c.lane = lane;
      c.base = st.base;
      c.span = st.span;
      c.value = st.value;
      c.pos2 = st.pos << 1;
      c.ring_addr = opaque(smem_addr(ring));
      filled = st.pos;
      for (long long wi = filled + lane; wi < filled + kRing; wi += 32) ring[wi & (kRing - 1)] = (uint16_t)bw_fetch(bw, wi);
      filled += kRing;
      __syncwarp();
      if (c.pos2 == 0) {  // fresh stream: the constructor reads four bytes (range_coder.h:79-83)
        c.value = ((uint32_t)ring[0] << 16) | (uint32_t)ring[1];
        c.pos2 = 4;
      }
      c.seek();
    }
  }

  for (int p = RAGGED ? 0 : P.p0; p < (RAGGED ? im.H * im.W : P.p1); ++p) {
    const int py = p / (RAGGED ? im.W : P.W), px = p - py * (RAGGED ? im.W : P.W);
    // ---- gather: the 12 causal neighbours of p (zeros outside the image) and ψ_p ----
    const float* yimg = P.yhat + (RAGGED ? pix0 * M : b * HW * M);
    for (int i = threadIdx.x; i < kArTaps * M; i += blockDim.x) {
      const int t = i / M, ch = i - t * M;
      const int yy = py + t / 5 - 2, xx = px + t % 5 - 2;
      float v = 0.f;
      if (yy >= 0 && xx >= 0 && xx < (RAGGED ? im.W : P.W))
        v = yimg[((long long)yy * (RAGGED ? im.W : P.W) + xx) * M + ch];  // (yy <= py always)
      taps[i] = v;
    }
    const float* psi = P.psi + (RAGGED ? pix0 + p : b * HW + p) * d.N2;
    for (int i = threadIdx.x; i < d.N2; i += blockDim.x) x1[i] = __ldg(psi + i);
    __syncthreads();
    // ---- context model and entropy parameters ----
    ar_dense(taps, kArTaps * M, Wp + d.wc, Wp + d.bc, d.N2, part, x1 + d.N2, false);
    ar_dense(x1, 4 * M, Wp + d.w1, Wp + d.b1, d.N3, part, h1, true);
    ar_dense(h1, d.N3, Wp + d.w2, Wp + d.b2, d.N4, part, h2, true);
    ar_dense(h2, d.N4, Wp + d.w3, Wp + d.b3, d.N2, part, out, false);
    // ---- epilogue ----
    const long long row = (MODE == kArParams) ? b * M : (RAGGED ? pix0 + p : b * HW + p) * M;
    if (MODE != kArDecode) {
      for (int ch = threadIdx.x; ch < M; ch += blockDim.x) {
        const float loc = out[ch], sc = out[M + ch];
        if (P.loc_out) P.loc_out[row + ch] = loc;
        if (P.scale_out) P.scale_out[row + ch] = sc;
        if (P.index_out) P.index_out[row + ch] = ar_table_index(sc, P.num_scales);
        if (MODE == kArEncode) {
          const int q = (int)rintf(__fsub_rn(__ldg(P.y + row + ch), loc));
          P.yhat[row + ch] = __fadd_rn((float)q, loc);
        }
      }
    } else if (threadIdx.x < 32) {
      // ---- decoder step: the M symbols of p, in channel order, from this stream's state ----
      float* yrow = P.yhat + row;
      for (int ch = 0; ch < M; ++ch) {
        if (filled - (long long)(c.pos2 >> 1) < 128) {  // a symbol consumes at most 66 words (escape with 32 zeros)
          const long long upto = (long long)(c.pos2 >> 1) + kRing - 64;
          for (long long wi = filled + lane; wi < upto; wi += 32) ring[wi & (kRing - 1)] = (uint16_t)bw_fetch(bw, wi);
          filled = upto;
          __syncwarp();
          c.seek();
        }
        const int ti = ar_table_index(out[M + ch], P.num_scales);  // < n_rows: checked on the host
        const int4 r4 = rows4[ti];
        const int n = row_ncdf(r4.y) - 1;
        uint32_t a, b1;
        int sym = c.search_row(pairs, r4.x, n, &a, &b1);
        c.update(a, b1);
        if (row_ovf(r4.y) && sym == n - 1) {  // OverflowDecode, range_coder_kernels.cc:449-471 (as decode_kernel)
          int nb = 0;
          while (c.bit() == 0 && nb < 32) ++nb;
          uint32_t val = (nb < 32) ? (1u << nb) : 0u;
          int t = nb;
          while (--t >= 0) {
            const uint32_t bitv = c.bit();
            if (t < 32) val |= bitv << t;
          }
          const uint32_t sg = c.bit();
          sym = sg ? -(int)val : (int)val + (n - 1) - 1;
        }
        if (lane == 0) {
          float yv = (float)(sym + __ldg(P.cdf_offset + ti));
          yv += out[ch];
          yrow[ch] = yv;
        }
      }
    }
    __syncthreads();  // ŷ_p is written before the next position gathers it; `out` / `taps` are free again
  }
  if (MODE == kArDecode && threadIdx.x == 0) {
    DecState st;
    st.base = c.base;
    st.span = c.span;
    st.value = c.value;
    st.pos = c.pos2 >> 1;
    P.state[b] = st;
  }
}

template <int MODE, bool SMEM_KEYS>
__global__ void __launch_bounds__(kArThreads) ar_kernel(const ArParams P) {
  ar_body<MODE, SMEM_KEYS, false>(P);
}

template <int MODE, bool SMEM_KEYS>
__global__ void __launch_bounds__(kArThreads) ar_ragged_kernel(const ArParams P) {
  ar_body<MODE, SMEM_KEYS, true>(P);
}

template <int MODE, bool SMEM_KEYS, bool RAGGED = false>
int ar_launch(const ArParams& P, long long B, size_t smem, cudaStream_t s) {
  auto kern = ar_kernel<MODE, SMEM_KEYS>;
  if constexpr (RAGGED) kern = ar_ragged_kernel<MODE, SMEM_KEYS>;
  TFCB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)B, kArThreads, smem, s>>>(P);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

constexpr size_t kArSmemLimit = 200 * 1024;  // dynamic shared memory beside the 8 KB ring (227 KB per CTA)

size_t ar_act_bytes(int M) { return (size_t)ar_act_floats(ar_dims(M)) * sizeof(float); }

constexpr long long kArImageFloats = sizeof(ArImage) / sizeof(float);

// Checks the workspace and uploads a ragged list's image table to it (one stream-ordered copy from pageable memory,
// staged before the call returns).
int ar_upload_table(int64_t n, const int64_t* hs, const int64_t* ws, float* work, int64_t work_floats, ArParams* P,
                    cudaStream_t s) {
  TFCB_TRY(ar_check_table_space(work, work_floats, n * kArImageFloats, alignof(ArImage)));
  std::vector<ArImage> t((size_t)n);
  long long pix = 0;
  for (int64_t i = 0; i < n; ++i) {
    t[i] = {pix, (int)hs[i], (int)ws[i]};
    pix += hs[i] * ws[i];
  }
  TFCB_CUDA_TRY(cudaMemcpyAsync(work, t.data(), t.size() * sizeof(ArImage), cudaMemcpyHostToDevice, s));
  P->img = reinterpret_cast<const ArImage*>(work);
  return TFCB_OK;
}

// The decoder's launch: search keys in shared memory when they fit beside the activations (64 NoisyNormal tables:
// 118 KB).
template <bool RAGGED>
int ar_launch_decode(const ArParams& P, const DecoderView& v, long long B, cudaStream_t s) {
  const size_t act = ar_act_bytes(P.M);
  const size_t keys = (size_t)((v.n_pairs * 8 + 15) & ~15ll) + (size_t)v.n_rows * sizeof(int4);
  if (act + keys <= kArSmemLimit) return ar_launch<kArDecode, true, RAGGED>(P, B, act + keys, s);
  return ar_launch<kArDecode, false, RAGGED>(P, B, act, s);
}

void ar_set_decoder(const DecoderView& v, ArParams* P) {
  P->pairs = v.pairs;
  P->rows4 = v.rows4;
  P->n_rows = v.n_rows;
  P->n_pairs = v.n_pairs;
  P->bytes = v.bytes;
  P->offsets = v.offsets;
  P->state = v.state;
}

int ar_check_decoder(const DecoderView& v, int64_t B, int num_scales) {
  if (v.n_streams != B)
    return fail(TFCB_INVALID_ARGUMENT, "the decoder holds %lld strings for a batch of %lld", v.n_streams,
                (long long)B);
  if (v.n_rows < num_scales)
    return fail(TFCB_INVALID_ARGUMENT, "the decoder's tables have %d rows for num_scales=%d", v.n_rows, num_scales);
  return TFCB_OK;
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

int64_t tfcb_ar_packed_floats(int M) {
  if (M <= 0 || M % 6 != 0 || M > kArMaxM) return -1;
  return ar_dims(M).total;
}

int tfcb_ar_pack_weights(int M, const float* ctx_kernel_dev, const float* ctx_bias_dev, const float* w1_dev,
                         const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                         const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream) {
  if (M <= 0 || M % 6 != 0 || M > kArMaxM)
    return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be a positive multiple of 6 and at most %d", M,
                kArMaxM);
  const ArDims d = ar_dims(M);
  if (packed_floats != d.total)
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, M=%d needs %lld", (long long)packed_floats,
                M, (long long)d.total);
  const float* src[8] = {ctx_kernel_dev, ctx_bias_dev, w1_dev, b1_dev, w2_dev, b2_dev, w3_dev, b3_dev};
  const long long at[9] = {d.wc, d.bc, d.w1, d.b1, d.w2, d.b2, d.w3, d.b3, d.total};
  // the context kernel [5, 5, M, 2M] holds the 12 causal taps first in raster order: [12M][2M] is its prefix
  return ar_pack_segments(src, at, packed_dev, as_stream(stream));
}

int tfcb_ar_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int64_t p, int num_scales, float* loc_dev, float* scale_index_dev,
                   int32_t* index_dev, void* stream) {
  TFCB_TRY(ar_check(M, packed_dev, packed_floats, B, H, W, num_scales));
  TFCB_TRY(ar_check_range(p, p + 1, H, W));
  if (!yhat_dev || !psi_dev) return fail(TFCB_INVALID_ARGUMENT, "`yhat` or `psi` is null");
  ArParams P{};
  P.packed = packed_dev;
  P.psi = psi_dev;
  P.yhat = const_cast<float*>(yhat_dev);  // read only in params mode
  P.loc_out = loc_dev;
  P.scale_out = scale_index_dev;
  P.index_out = index_dev;
  P.H = (int)H;
  P.W = (int)W;
  P.M = M;
  P.num_scales = num_scales;
  P.p0 = (int)p;
  P.p1 = (int)p + 1;
  return ar_launch<kArParams, false>(P, B, ar_act_bytes(M), as_stream(stream));
}

int tfcb_ar_encode(const float* packed_dev, int64_t packed_floats, int M, const float* y_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int64_t p_begin, int64_t p_end, int num_scales, float* yhat_dev,
                   float* loc_dev, int32_t* index_dev, float* scale_index_dev, void* stream) {
  TFCB_TRY(ar_check(M, packed_dev, packed_floats, B, H, W, num_scales));
  TFCB_TRY(ar_check_range(p_begin, p_end, H, W));
  if (!y_dev || !psi_dev || !yhat_dev || !loc_dev || !index_dev)
    return fail(TFCB_INVALID_ARGUMENT, "`y`, `psi`, `yhat`, `loc` or `index` is null");
  if (p_begin == p_end) return TFCB_OK;
  ArParams P{};
  P.packed = packed_dev;
  P.psi = psi_dev;
  P.y = y_dev;
  P.yhat = yhat_dev;
  P.loc_out = loc_dev;
  P.scale_out = scale_index_dev;
  P.index_out = index_dev;
  P.H = (int)H;
  P.W = (int)W;
  P.M = M;
  P.num_scales = num_scales;
  P.p0 = (int)p_begin;
  P.p1 = (int)p_end;
  return ar_launch<kArEncode, false>(P, B, ar_act_bytes(M), as_stream(stream));
}

int tfcb_ar_decode(tfcb_decoder* h, const float* packed_dev, int64_t packed_floats, int M, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int64_t p_begin, int64_t p_end, int num_scales,
                   const int32_t* cdf_offset_dev, float* yhat_dev, void* stream) {
  DecoderView v;
  TFCB_TRY(decoder_view(h, &v));
  TFCB_TRY(ar_check(M, packed_dev, packed_floats, B, H, W, num_scales));
  TFCB_TRY(ar_check_range(p_begin, p_end, H, W));
  TFCB_TRY(ar_check_decoder(v, B, num_scales));
  if (!psi_dev || !yhat_dev || !cdf_offset_dev)
    return fail(TFCB_INVALID_ARGUMENT, "`psi`, `yhat` or `cdf_offset` is null");
  if (p_begin == p_end) return TFCB_OK;
  ArParams P{};
  P.packed = packed_dev;
  P.psi = psi_dev;
  P.yhat = yhat_dev;
  P.cdf_offset = cdf_offset_dev;
  P.H = (int)H;
  P.W = (int)W;
  P.M = M;
  P.num_scales = num_scales;
  P.p0 = (int)p_begin;
  P.p1 = (int)p_end;
  ar_set_decoder(v, &P);
  return ar_launch_decode<false>(P, v, B, as_stream(stream));
}

int64_t tfcb_ar_ragged_workspace_floats(int64_t n_images) {
  if (n_images <= 0 || n_images > 0x7FFFFFFF) return -1;
  return n_images * kArImageFloats;
}

int tfcb_ar_encode_ragged(const float* packed_dev, int64_t packed_floats, int M, const float* y_dev,
                          const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                          const int64_t* widths_host, int num_scales, float* work_dev, int64_t work_floats,
                          float* yhat_dev, float* loc_dev, int32_t* index_dev, float* scale_index_dev, void* stream) {
  TFCB_TRY(ar_check_packed(M, packed_dev, packed_floats));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  if (!y_dev || !psi_dev || !yhat_dev || !loc_dev || !index_dev)
    return fail(TFCB_INVALID_ARGUMENT, "`y`, `psi`, `yhat`, `loc` or `index` is null");
  ArParams P{};
  P.packed = packed_dev;
  P.psi = psi_dev;
  P.y = y_dev;
  P.yhat = yhat_dev;
  P.loc_out = loc_dev;
  P.scale_out = scale_index_dev;
  P.index_out = index_dev;
  P.M = M;
  P.num_scales = num_scales;
  cudaStream_t s = as_stream(stream);
  TFCB_TRY(ar_upload_table(n_images, heights_host, widths_host, work_dev, work_floats, &P, s));
  return ar_launch<kArEncode, false, true>(P, n_images, ar_act_bytes(M), s);
}

int tfcb_ar_decode_ragged(tfcb_decoder* h, const float* packed_dev, int64_t packed_floats, int M, const float* psi_dev,
                          int64_t n_images, const int64_t* heights_host, const int64_t* widths_host, int num_scales,
                          const int32_t* cdf_offset_dev, float* work_dev, int64_t work_floats, float* yhat_dev,
                          void* stream) {
  DecoderView v;
  TFCB_TRY(decoder_view(h, &v));
  TFCB_TRY(ar_check_packed(M, packed_dev, packed_floats));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  TFCB_TRY(ar_check_decoder(v, n_images, num_scales));
  if (!psi_dev || !yhat_dev || !cdf_offset_dev)
    return fail(TFCB_INVALID_ARGUMENT, "`psi`, `yhat` or `cdf_offset` is null");
  ArParams P{};
  P.packed = packed_dev;
  P.psi = psi_dev;
  P.yhat = yhat_dev;
  P.cdf_offset = cdf_offset_dev;
  P.M = M;
  P.num_scales = num_scales;
  ar_set_decoder(v, &P);
  cudaStream_t s = as_stream(stream);
  TFCB_TRY(ar_upload_table(n_images, heights_host, widths_host, work_dev, work_floats, &P, s));
  return ar_launch_decode<true>(P, v, n_images, s);
}

}  // extern "C"
