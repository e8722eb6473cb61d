// Substreams (DESIGN §3.14): the split of a coding unit's symbols into S independently decodable streams, and the
// gather that rewrites whole-unit coding order into substream order for the encoder.
//
// A unit's symbols are in coding order, in phases (the order the decoder makes them: one phase for the batched,
// indexed and MS2020 strings, anchors then non-anchors per channel group for the context models).  Phase p has n_p
// positions of C_p symbols each.  Substream s of a unit is the concatenation over p of the positions
// [floor(s n_p / S), floor((s + 1) n_p / S)) of phase p.  So every stream holds whole positions (channel mode starts
// each stream at table row 0), and a per-phase ragged decode over units x S streams returns that phase in coding
// order, unit after unit: the layout the parameter passes and scatters already use.
//
// The gather is a segmented copy: each (unit, stream, phase) segment is contiguous in coding order and in substream
// order, so the host lists the non-empty segments' starts and every output element finds its segment by a binary
// search over them.  One launch for y, loc and index together; the range coder's and the parameter passes' kernels
// are untouched.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "common.cuh"

namespace tfcb {
namespace {

constexpr int64_t kMaxSubstreams = 1024;

struct SubSeg {
  long long dst;  // first element of the segment in substream order
  long long src;  // ... and in coding order
};

int sub_check(int64_t n_units, int64_t n_phases, const int64_t* pos, const int64_t* wid, int64_t S) {
  if (n_units <= 0 || n_units > 0x7FFFFFFF) return fail(TFCB_INVALID_ARGUMENT, "%lld coding units", (long long)n_units);
  if (n_phases <= 0 || n_phases > 0x7FFFFFFF)
    return fail(TFCB_INVALID_ARGUMENT, "%lld phases per unit", (long long)n_phases);
  if (S < 1 || S > kMaxSubstreams)
    return fail(TFCB_INVALID_ARGUMENT, "substreams=%lld must be in [1, %lld]", (long long)S, (long long)kMaxSubstreams);
  if (n_units * S * n_phases > 0x7FFFFFFF)
    return fail(TFCB_INVALID_ARGUMENT, "%lld units of %lld phases in %lld substreams: too many segments",
                (long long)n_units, (long long)n_phases, (long long)S);
  if (!pos || !wid) return fail(TFCB_INVALID_ARGUMENT, "`positions` or `widths` is null");
  long long total = 0;
  for (int64_t i = 0; i < n_units * n_phases; ++i) {
    if (pos[i] < 0 || pos[i] > 0x7FFFFFFF || wid[i] < 1 || wid[i] > 0x7FFFFFFF)
      return fail(TFCB_INVALID_ARGUMENT, "unit %lld, phase %lld: %lld positions of width %lld",
                  (long long)(i / n_phases), (long long)(i % n_phases), (long long)pos[i], (long long)wid[i]);
    total += pos[i] * wid[i];
    if (total > (1ll << 62)) return fail(TFCB_INVALID_ARGUMENT, "too many symbols");
  }
  return TFCB_OK;
}

// The layout after sub_check.  Any output may be null; `segs` receives the non-empty segments in substream order.
void sub_layout(int64_t U, int64_t P, const int64_t* pos, const int64_t* wid, int64_t S, int64_t* stream_off,
                int64_t* phase_len, std::vector<SubSeg>* segs) {
  long long unit_base = 0, dst = 0;
  if (stream_off) stream_off[0] = 0;
  for (int64_t u = 0; u < U; ++u) {
    const int64_t* n = pos + u * P;
    const int64_t* c = wid + u * P;
    for (int64_t s = 0; s < S; ++s) {
      long long phase_base = unit_base;
      for (int64_t p = 0; p < P; ++p) {
        const long long lo = s * n[p] / S, hi = (s + 1) * n[p] / S;
        const long long len = (hi - lo) * c[p];
        if (phase_len) phase_len[p * U * S + u * S + s] = len;
        if (segs && len) segs->push_back({dst, phase_base + lo * c[p]});
        dst += len;
        phase_base += n[p] * c[p];
      }
      if (stream_off) stream_off[u * S + s + 1] = dst;
    }
    for (int64_t p = 0; p < P; ++p) unit_base += n[p] * c[p];
  }
}

// out[e] = in[src(e)] for up to three 4-byte operands; src(e) from the segment that holds e (the last one starting
// at or before e).
__global__ void substream_gather_kernel(const SubSeg* __restrict__ seg, int n_seg, long long total,
                                        const uint32_t* __restrict__ a, const uint32_t* __restrict__ b,
                                        const uint32_t* __restrict__ c, uint32_t* __restrict__ ao,
                                        uint32_t* __restrict__ bo, uint32_t* __restrict__ co) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = n_seg - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (seg[mid].dst <= e) lo = mid; else hi = mid - 1;
    }
    const long long src = seg[lo].src + (e - seg[lo].dst);
    if (a) ao[e] = a[src];
    if (b) bo[e] = b[src];
    if (c) co[e] = c[src];
  }
}

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

int tfcb_substream_layout(int64_t n_units, int64_t n_phases, const int64_t* positions_host,
                          const int64_t* widths_host, int64_t substreams, int64_t* stream_offsets_host,
                          int64_t* phase_lengths_host) {
  TFCB_TRY(sub_check(n_units, n_phases, positions_host, widths_host, substreams));
  sub_layout(n_units, n_phases, positions_host, widths_host, substreams, stream_offsets_host, phase_lengths_host,
             nullptr);
  return TFCB_OK;
}

int64_t tfcb_substream_gather_workspace_bytes(int64_t n_units, int64_t n_phases, int64_t substreams) {
  if (n_units <= 0 || n_units > 0x7FFFFFFF || n_phases <= 0 || n_phases > 0x7FFFFFFF || substreams < 1 ||
      substreams > kMaxSubstreams || n_units * substreams * n_phases > 0x7FFFFFFF)
    return -1;
  return n_units * n_phases * substreams * (int64_t)sizeof(SubSeg);
}

int tfcb_substream_gather(int64_t n_units, int64_t n_phases, const int64_t* positions_host,
                          const int64_t* widths_host, int64_t substreams, const float* y_dev, const float* loc_dev,
                          const int32_t* index_dev, float* y_out_dev, float* loc_out_dev, int32_t* index_out_dev,
                          void* work_dev, int64_t work_bytes, void* stream) {
  TFCB_TRY(sub_check(n_units, n_phases, positions_host, widths_host, substreams));
  if (!y_dev && !loc_dev && !index_dev) return fail(TFCB_INVALID_ARGUMENT, "no operand to gather");
  if (!y_dev != !y_out_dev || !loc_dev != !loc_out_dev || !index_dev != !index_out_dev)
    return fail(TFCB_INVALID_ARGUMENT, "every operand given needs its output, and only those");
  const long long need = tfcb_substream_gather_workspace_bytes(n_units, n_phases, substreams);
  if (!work_dev || work_bytes < need)
    return fail(TFCB_INVALID_ARGUMENT, "workspace of %lld bytes, this call needs %lld",
                work_dev ? (long long)work_bytes : 0ll, need);
  if (reinterpret_cast<uintptr_t>(work_dev) % alignof(SubSeg))
    return fail(TFCB_INVALID_ARGUMENT, "the workspace must be %d-byte aligned", (int)alignof(SubSeg));
  std::vector<SubSeg> segs;
  sub_layout(n_units, n_phases, positions_host, widths_host, substreams, nullptr, nullptr, &segs);
  if (segs.empty()) return TFCB_OK;
  long long total = 0;
  for (int64_t i = 0; i < n_units * n_phases; ++i) total += positions_host[i] * widths_host[i];
  cudaStream_t s = as_stream(stream);
  // (pageable source: staged before the call returns)
  TFCB_CUDA_TRY(cudaMemcpyAsync(work_dev, segs.data(), segs.size() * sizeof(SubSeg), cudaMemcpyHostToDevice, s));
  const long long blocks = std::min<long long>((total + 255) / 256, 1ll << 16);
  substream_gather_kernel<<<(unsigned)blocks, 256, 0, s>>>(
      static_cast<const SubSeg*>(work_dev), (int)segs.size(), total, reinterpret_cast<const uint32_t*>(y_dev),
      reinterpret_cast<const uint32_t*>(loc_dev), reinterpret_cast<const uint32_t*>(index_dev),
      reinterpret_cast<uint32_t*>(y_out_dev), reinterpret_cast<uint32_t*>(loc_out_dev),
      reinterpret_cast<uint32_t*>(index_out_dev));
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

}  // extern "C"
