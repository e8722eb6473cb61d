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

#include <algorithm>
#include <cstring>
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

// One work item of the column-tile kernel (§3.15): columns [c0, c1) of row `row` of image `img`, which is tile `tile`
// of the image (its stream img T + tile).  `self`, `left` and `upper` index the per-(image, non-empty tile) progress
// counters: the item's own tile, the tile before it in the row (-1 for the first), and the tile holding column
// min(W - 1, c1 + 1) (-1 in row 0).
struct ArTileItem {
  int img, row, c0, c1;
  int tile, self, left, upper;
};

// The CTA of image b: positions [P.p0, P.p1) of B images of P.H × P.W, or (RAGGED) every position of image b of the
// list P.img, or (TILE, with RAGGED) the positions of the work item `it`, continuing the stream of its tile.  With
// TILE the search keys are already in shared memory (SMEM_KEYS) and ŷ of other items is read with coherent loads.
template <int MODE, bool SMEM_KEYS, bool RAGGED, bool TILE = false>
__device__ __forceinline__ void ar_body(const ArParams& P, const ArTileItem& it = ArTileItem{}, int tiles = 1) {
  extern __shared__ __align__(16) float s_act[];
  __shared__ __align__(16) uint16_t ring_buf[2 * kRing];  // decoder only: 4096-byte aligned ring, as decode_kernel
  const ArDims d = ar_dims(P.M);
  const int M = P.M;
  const long long b = TILE ? (long long)it.img : (long long)blockIdx.x;
  const long long strm = TILE ? b * tiles + it.tile : b;  // the decoder's stream
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
      if (!TILE) {  // (the tile kernel copies them once per CTA: ar_tile_keys)
        for (long long i = threadIdx.x; i < P.n_pairs; i += blockDim.x) sp[i] = P.pairs[i];
        for (int i = threadIdx.x; i < P.n_rows; i += blockDim.x) sr[i] = P.rows4[i];
      }
      pairs = sp;
      rows4 = sr;
      if (!TILE) __syncthreads();
    }
    ring = ring_buf + (((4096u - (smem_addr(ring_buf) & 4095u)) & 4095u) >> 1);
    if (threadIdx.x < 32) {
      bw.p = P.bytes + P.offsets[strm];
      bw.len = P.offsets[strm + 1] - P.offsets[strm];
      const DecState st = P.state[strm];
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

  for (int p = TILE ? it.row * im.W + it.c0 : (RAGGED ? 0 : P.p0);
       p < (TILE ? it.row * im.W + it.c1 : (RAGGED ? im.H * im.W : P.p1)); ++p) {
    const int py = p / (RAGGED ? im.W : P.W), px = p - py * (RAGGED ? im.W : P.W);
    // ---- gather: the 12 causal neighbours of p (zeros outside the image) and ψ_p ----
    const float* yimg = P.yhat + (RAGGED ? pix0 * M : b * HW * M);
    for (int i = threadIdx.x; i < kArTaps * M; i += blockDim.x) {
      const int t = i / M, ch = i - t * M;
      const int yy = py + t / 5 - 2, xx = px + t % 5 - 2;
      float v = 0.f;
      if (yy >= 0 && xx >= 0 && xx < (RAGGED ? im.W : P.W)) {
        const float* src = yimg + ((long long)yy * (RAGGED ? im.W : P.W) + xx) * M + ch;  // (yy <= py always)
        v = TILE ? __ldcg(src) : *src;  // (other CTAs' ŷ: L2, never a stale L1 line)
      }
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
    P.state[strm] = st;
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

// ---- column tiles (§3.15): one persistent grid over a ticket-ordered table of (image, row, tile) items ----
struct ArTileParams {
  ArParams ar;               // ar.img: the image table
  const ArTileItem* items;   // in ticket order: sorted by (2 row + tile rank, row, image)
  int n_items, tiles;
  int* counters;             // rows done per (image, non-empty tile); kArTileFailed marks a tile with a failed item
  int* sched;                // [0] the next ticket, [1] the abort word, [2] CTAs that have finished
};

constexpr int kArTileFailed = 1 << 30;
constexpr unsigned long long kArTileWaitNs = 10000000000ull;  // 10 s: only a scheduling bug can wait this long

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int ld_relaxed(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void add_release(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Thread 0: waits until item `it` may run: tile u - 1 has finished row r and the tile holding column c1 + 1 has
// finished row r - 1.  False when the launch is aborted: the abort word is set, a tile it waits on failed, or the wait
// passes kArTileWaitNs (the first such CTA sets the abort word).  Every CTA then drains its remaining items.
__device__ __forceinline__ bool ar_tile_wait(const ArTileParams& T, const ArTileItem& it) {
  const unsigned long long t0 = global_ns();
  unsigned ns = 32;
  for (;;) {
    if (ld_relaxed(T.sched + 1)) return false;
    const int l = it.left < 0 ? it.row + 1 : ld_acquire(T.counters + it.left);
    const int u = it.upper < 0 ? it.row : ld_acquire(T.counters + it.upper);
    if ((l | u) & kArTileFailed) return false;
    if (l >= it.row + 1 && u >= it.row) return true;
    if (global_ns() - t0 > kArTileWaitNs) {
      atomicExch(T.sched + 1, 1);
      return false;
    }
    __nanosleep(ns);
    ns = min(ns * 2, 1024u);
  }
}

// The decoder's search keys, copied once per CTA to where ar_body<..., SMEM_KEYS> finds them (behind the activations).
__device__ __forceinline__ void ar_tile_keys(const ArParams& P) {
  extern __shared__ __align__(16) float s_act[];
  uint2* sp = reinterpret_cast<uint2*>(s_act + ar_act_floats(ar_dims(P.M)));
  int4* sr = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(sp) + ((P.n_pairs * 8 + 15) & ~15ll));
  for (long long i = threadIdx.x; i < P.n_pairs; i += blockDim.x) sp[i] = P.pairs[i];
  for (int i = threadIdx.x; i < P.n_rows; i += blockDim.x) sr[i] = P.rows4[i];
}

// Each CTA takes the next ticket, waits for the item's two dependencies, runs its positions left to right with
// ar_body (encoder: writes ŷ, loc, index; decoder: continues stream img T + tile from its saved state and saves it
// back), then publishes the row: ŷ and the state are written, a barrier, a fence and a release add on the counter.
// Tickets are in an order in which every item comes after the items it waits for, so the lowest unfinished ticket
// can always run: the schedule finishes for any grid size.  A failed item (aborted launch) writes no ŷ and marks its
// tile failed; the encoder sets its table indexes to -1, which the range encode rejects, and the last CTA to finish
// gives every failed tile's stream a state that tfcb_decode_finalize reports as not OK.
template <int MODE, bool SMEM_KEYS>
__global__ void __launch_bounds__(kArThreads) ar_tile_kernel(const ArTileParams T) {
  __shared__ int s_ticket, s_go;
  const ArParams& P = T.ar;
  if (MODE == kArDecode && SMEM_KEYS) ar_tile_keys(P);
  for (;;) {
    if (threadIdx.x == 0) s_ticket = atomicAdd(T.sched, 1);
    __syncthreads();
    const int k = s_ticket;
    if (k >= T.n_items) break;
    const ArTileItem it = T.items[k];
    if (threadIdx.x == 0) s_go = ar_tile_wait(T, it);
    __syncthreads();
    const bool go = s_go;
    if (go) {
      ar_body<MODE, SMEM_KEYS, true, true>(P, it, T.tiles);  // (ends with a barrier after the last position's ŷ)
    } else if (MODE == kArEncode) {
      const ArImage im = P.img[it.img];
      const long long at = (im.pix + (long long)it.row * im.W + it.c0) * P.M;
      for (long long e = threadIdx.x; e < (long long)(it.c1 - it.c0) * P.M; e += blockDim.x) P.index_out[at + e] = -1;
    }
    if (threadIdx.x == 0) {
      if (go) {
        __threadfence();
        add_release(T.counters + it.self, 1);
      } else {
        atomicOr(T.counters + it.self, kArTileFailed);
      }
    }
  }
  if (MODE == kArDecode) {
    __shared__ int s_last;
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = atomicAdd(T.sched + 2, 1) == (int)gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0 && ld_acquire(T.sched + 1)) {  // every other CTA has saved its states
      for (int k = 0; k < T.n_items; ++k) {
        const ArTileItem it = T.items[k];
        if (ld_relaxed(T.counters + it.self) & kArTileFailed) {
          DecState st;  // base 0 with value 1 (or not read to the end): RangeDecoder::Finalize fails
          st.base = 0;
          st.span = 0;
          st.value = 1;
          st.pos = 0x7FFFFFFFu;
          P.state[(long long)it.img * T.tiles + it.tile] = st;
        }
      }
    }
  }
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

// ---- column tiles: the schedule and the workspace (image table, item table, counters, ticket, abort, exits) ----
constexpr int64_t kArMaxTiles = 1024;  // gen_ops.MAX_SUBSTREAMS: the tiles are the substreams of a string

bool ar_tiles_ok(int64_t T) { return T >= 1 && T <= kArMaxTiles; }

int ar_check_tiles(int64_t T) {
  if (!ar_tiles_ok(T))
    return fail(TFCB_INVALID_ARGUMENT, "tiles=%lld must be in [1, %lld]", (long long)T, (long long)kArMaxTiles);
  return TFCB_OK;
}

// The items of a checked list in ticket order, and the number of progress counters (non-empty tiles of all images).
// Tile t of an image of width W holds columns [floor(t W / T), floor((t + 1) W / T)); item (i, r, u) is row r of the
// u-th non-empty tile.  False when the list has more than 2^31 - 1 items.
bool ar_tile_schedule(int64_t n, const int64_t* hs, const int64_t* ws, int64_t T, std::vector<ArTileItem>* items,
                      long long* n_counters) {
  long long total = 0;
  for (int64_t i = 0; i < n; ++i) {
    total += hs[i] * std::min<int64_t>(T, ws[i]);
    if (total > 0x7FFFFFFF) return false;
  }
  struct Keyed {
    long long diag;  // 2 r + u
    int row;
    ArTileItem it;
  };
  std::vector<Keyed> keyed;
  keyed.reserve((size_t)total);
  long long cbase = 0;
  std::vector<int> tile, c0, c1;
  for (int64_t i = 0; i < n; ++i) {
    const int64_t W = ws[i];
    tile.clear();
    c0.clear();
    c1.clear();
    for (int64_t t = 0; t < T; ++t) {
      const int64_t a = t * W / T, b = (t + 1) * W / T;
      if (b > a) {
        tile.push_back((int)t);
        c0.push_back((int)a);
        c1.push_back((int)b);
      }
    }
    const int U = (int)tile.size();
    for (int u = 0, ur = 0; u < U; ++u) {
      const int64_t need = std::min<int64_t>(W - 1, (int64_t)c1[u] + 1);  // column c_last + 2
      while (c1[ur] <= need) ++ur;
      for (int64_t r = 0; r < hs[i]; ++r) {
        const ArTileItem it{(int)i, (int)r, c0[u], c1[u], tile[u], (int)(cbase + u), u ? (int)(cbase + u - 1) : -1,
                            r ? (int)(cbase + ur) : -1};
        keyed.push_back({2 * r + u, (int)r, it});
      }
    }
    cbase += U;
  }
  std::sort(keyed.begin(), keyed.end(), [](const Keyed& x, const Keyed& y) {
    if (x.diag != y.diag) return x.diag < y.diag;
    if (x.row != y.row) return x.row < y.row;
    return x.it.img < y.it.img;
  });
  items->resize(keyed.size());
  for (size_t k = 0; k < keyed.size(); ++k) (*items)[k] = keyed[k].it;
  *n_counters = cbase;
  return true;
}

// Bytes of each workspace section: the image table, the item table, then counters and the three schedule words.
struct ArTileSpace {
  long long images, items, words;
  long long floats() const { return (images + items + words + 3) / 4; }
};

ArTileSpace ar_tile_space(int64_t n, long long n_items, long long n_counters) {
  return {n * (long long)sizeof(ArImage), n_items * (long long)sizeof(ArTileItem), (n_counters + 3) * 4};
}

// The tiles decoder's launch: keys in shared memory when they fit, as ar_launch_decode.
template <int MODE, bool SMEM_KEYS>
int ar_tile_launch(const ArTileParams& T, size_t smem, cudaStream_t s) {
  auto kern = ar_tile_kernel<MODE, SMEM_KEYS>;
  TFCB_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int dev = 0, sms = 0, per_sm = 0;
  TFCB_CUDA_TRY(cudaGetDevice(&dev));
  TFCB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  TFCB_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kArThreads, smem));
  const long long grid = std::min<long long>(T.n_items, (long long)std::max(per_sm, 1) * std::max(sms, 1));
  kern<<<(unsigned)grid, kArThreads, smem, s>>>(T);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// Checks the workspace, uploads the image and item tables (one stream-ordered copy from pageable memory, staged
// before the call returns, as ar_upload_table) and resets the counters and schedule words (one memset).
int ar_tile_prepare(int64_t n, const int64_t* hs, const int64_t* ws, int64_t T, float* work, int64_t work_floats,
                    ArTileParams* TP, cudaStream_t s) {
  std::vector<ArTileItem> items;
  long long n_counters = 0;
  if (!ar_tile_schedule(n, hs, ws, T, &items, &n_counters))
    return fail(TFCB_INVALID_ARGUMENT, "the list has more than 2^31 - 1 (row, tile) items");
  const ArTileSpace sp = ar_tile_space(n, (long long)items.size(), n_counters);
  TFCB_TRY(ar_check_table_space(work, work_floats, sp.floats(), alignof(ArImage)));
  std::vector<uint8_t> host((size_t)(sp.images + sp.items));
  long long pix = 0;
  for (int64_t i = 0; i < n; ++i) {
    const ArImage im{pix, (int)hs[i], (int)ws[i]};
    std::memcpy(host.data() + i * sizeof(ArImage), &im, sizeof(ArImage));
    pix += hs[i] * ws[i];
  }
  std::memcpy(host.data() + sp.images, items.data(), (size_t)sp.items);
  uint8_t* base = reinterpret_cast<uint8_t*>(work);
  TFCB_CUDA_TRY(cudaMemcpyAsync(base, host.data(), host.size(), cudaMemcpyHostToDevice, s));
  TFCB_CUDA_TRY(cudaMemsetAsync(base + sp.images + sp.items, 0, (size_t)sp.words, s));
  TP->ar.img = reinterpret_cast<const ArImage*>(base);
  TP->items = reinterpret_cast<const ArTileItem*>(base + sp.images);
  TP->n_items = (int)items.size();
  TP->tiles = (int)T;
  TP->counters = reinterpret_cast<int*>(base + sp.images + sp.items);
  TP->sched = TP->counters + n_counters;
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

int64_t tfcb_ar_tiles_workspace_floats(int64_t n_images, const int64_t* heights_host, const int64_t* widths_host,
                                       int64_t tiles) {
  if (!ar_list_ok(n_images, heights_host, widths_host) || !ar_tiles_ok(tiles)) return -1;
  std::vector<ArTileItem> items;
  long long n_counters = 0;
  if (!ar_tile_schedule(n_images, heights_host, widths_host, tiles, &items, &n_counters)) return -1;
  return ar_tile_space(n_images, (long long)items.size(), n_counters).floats();
}

int tfcb_ar_tiles_schedule(int64_t n_images, const int64_t* heights_host, const int64_t* widths_host, int64_t tiles,
                           int64_t* n_items_host, int64_t* items_host) {
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, 1));
  TFCB_TRY(ar_check_tiles(tiles));
  if (!n_items_host) return fail(TFCB_INVALID_ARGUMENT, "`n_items` is null");
  std::vector<ArTileItem> items;
  long long n_counters = 0;
  if (!ar_tile_schedule(n_images, heights_host, widths_host, tiles, &items, &n_counters))
    return fail(TFCB_INVALID_ARGUMENT, "the list has more than 2^31 - 1 (row, tile) items");
  *n_items_host = (int64_t)items.size();
  if (items_host)
    for (size_t k = 0; k < items.size(); ++k) {
      int64_t* o = items_host + 5 * k;
      o[0] = items[k].img;
      o[1] = items[k].row;
      o[2] = items[k].tile;
      o[3] = items[k].c0;
      o[4] = items[k].c1;
    }
  return TFCB_OK;
}

int tfcb_ar_encode_tiles(const float* packed_dev, int64_t packed_floats, int M, const float* y_dev,
                         const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                         const int64_t* widths_host, int64_t tiles, int num_scales, float* work_dev,
                         int64_t work_floats, float* yhat_dev, float* loc_dev, int32_t* index_dev,
                         float* scale_index_dev, void* stream) {
  TFCB_TRY(ar_check_packed(M, packed_dev, packed_floats));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  TFCB_TRY(ar_check_tiles(tiles));
  if (!y_dev || !psi_dev || !yhat_dev || !loc_dev || !index_dev)
    return fail(TFCB_INVALID_ARGUMENT, "`y`, `psi`, `yhat`, `loc` or `index` is null");
  ArTileParams T{};
  ArParams& P = T.ar;
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
  TFCB_TRY(ar_tile_prepare(n_images, heights_host, widths_host, tiles, work_dev, work_floats, &T, s));
  return ar_tile_launch<kArEncode, false>(T, ar_act_bytes(M), s);
}

int tfcb_ar_decode_tiles(tfcb_decoder* h, const float* packed_dev, int64_t packed_floats, int M, const float* psi_dev,
                         int64_t n_images, const int64_t* heights_host, const int64_t* widths_host, int64_t tiles,
                         int num_scales, const int32_t* cdf_offset_dev, float* work_dev, int64_t work_floats,
                         float* yhat_dev, void* stream) {
  DecoderView v;
  TFCB_TRY(decoder_view(h, &v));
  TFCB_TRY(ar_check_packed(M, packed_dev, packed_floats));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  TFCB_TRY(ar_check_tiles(tiles));
  TFCB_TRY(ar_check_decoder(v, n_images * tiles, num_scales));
  if (!psi_dev || !yhat_dev || !cdf_offset_dev)
    return fail(TFCB_INVALID_ARGUMENT, "`psi`, `yhat` or `cdf_offset` is null");
  ArTileParams T{};
  ArParams& P = T.ar;
  P.packed = packed_dev;
  P.psi = psi_dev;
  P.yhat = yhat_dev;
  P.cdf_offset = cdf_offset_dev;
  P.M = M;
  P.num_scales = num_scales;
  ar_set_decoder(v, &P);
  cudaStream_t s = as_stream(stream);
  TFCB_TRY(ar_tile_prepare(n_images, heights_host, widths_host, tiles, work_dev, work_floats, &T, s));
  const size_t act = ar_act_bytes(M);
  const size_t keys = (size_t)((v.n_pairs * 8 + 15) & ~15ll) + (size_t)v.n_rows * sizeof(int4);
  if (act + keys <= kArSmemLimit) return ar_tile_launch<kArDecode, true>(T, act + keys, s);
  return ar_tile_launch<kArDecode, false>(T, act, s);
}

}  // extern "C"
