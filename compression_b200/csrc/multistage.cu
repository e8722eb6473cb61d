// Multistage spatial context model (Lin, Chen, Yang et al., ICASSP 2023) on sm_90a: the entropy parameters of one
// stage of a four-pass 2×2 schedule, all images and positions of that stage at once, on checkerboard.cuh's tiles;
// alone over the whole latent (tfcb_msc_*), or inside one channel group of the space-channel model (tfcb_mscc_*).
//
// Position (r, c) has phase (r mod 2, c mod 2) and stage (0,0) -> 0, (1,1) -> 1, (0,1) -> 2, (1,0) -> 3.  Stage s with
// phase (a, b) has ceil((H - a) / 2) · W_s positions, W_s = ceil((W - b) / 2); its j-th is (a + 2 (j / W_s),
// b + 2 (j mod W_s)).  The latent y [B, H, W, M] is split into channel groups; group k holds the C = c_k channels
// [o, o + C) (the multistage model is the one group o = 0, C = M).  An image codes group 0's stage 0 in raster order,
// then its stages 1, 2 and 3, then group 1's four stages, and so on ("coding order"), C channels per position.  Per
// position of stage s of group k (CH = 0 for k = 0, else 2C):
//   ctx   = 0 at stage 0 (bias included); else bc_s + Wc_s · (ŷ[o, o + C) at the stage's T_s taps, raster order, zeros
//           outside the image): the offsets (dy, dx) in [-2, 2]^2 whose neighbour lies in an earlier stage,
//           T_s = 4, 12, 16                                                                       [T_s C] -> [2C]
//   h1    = leaky(b1 + W1 · [ψ_p (2M), chctx_p (CH), ctx])                     [K1 = 2M + CH + 2C] -> [N3 = 5 K1 / 6]
//   h2    = leaky(b2 + W2 · h1)                                                                 [N3] -> [N4 = 2 K1 / 3]
//   out   = b3 + W3 · h2 = [loc, scale_index]                                                              [N4] -> [2C]
// (N3 and N4 rounded down; with one group they are 10M/3 and 8M/3.)  W1 .. b3 are shared by a group's stages; each
// stage s >= 1 has its own Wc_s and bc_s.  The channel context chctx [B, H, W, CH] comes from the caller.  Every
// output has the fixed float32 order of checkerboard.cuh, so stage 0 of a group is the space-channel model's anchor
// pass of that group at its positions, and stage s's outputs depend only on their own position's inputs.  A pass is
// one launch per layer: three at stage 0, four at stages 1-3, none for an empty stage (H = 1 or W = 1).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "autoregressive.cuh"
#include "checkerboard.cuh"
#include "common.cuh"

namespace tfcb {
namespace {

constexpr int kMsStages = 4;
constexpr int kMsMaxTaps = 16;

// The taps of stages 1-3 in raster order (row 0, stage 0, has none): dy and dx both odd; dy + dx odd; not both even.
__constant__ int8_t c_ms_dy[kMsStages][kMsMaxTaps] = {
    {},
    {-1, -1, 1, 1},
    {-2, -2, -1, -1, -1, 0, 0, 1, 1, 1, 2, 2},
    {-2, -2, -1, -1, -1, -1, -1, 0, 0, 1, 1, 1, 1, 1, 2, 2}};
__constant__ int8_t c_ms_dx[kMsStages][kMsMaxTaps] = {
    {},
    {-1, 1, -1, 1},
    {-1, 1, -2, 0, 2, -1, 1, -2, 0, 2, -1, 1},
    {-1, 1, -2, -1, 0, 1, 2, -1, 1, -2, -1, 0, 1, 2, -1, 1}};

__host__ __device__ inline int ms_row_phase(int stage) { return stage == 1 || stage == 3; }
__host__ __device__ inline int ms_col_phase(int stage) { return stage == 1 || stage == 2; }
int ms_taps(int stage) { return stage == 0 ? 0 : stage == 1 ? 4 : stage == 2 ? 12 : 16; }

// The multistage schedule for checkerboard.cuh: pass `stage`.
struct MsSchedule {
  __device__ static void position(long long j, int W, int stage, int* r, int* c) {
    const int a = ms_row_phase(stage), b = ms_col_phase(stage), ws = (W - b + 1) / 2;
    const long long row = j / ws;
    *r = a + 2 * (int)row;
    *c = b + 2 * (int)(j - row * ws);
  }
  __device__ static int8_t dy(int stage, int t) { return c_ms_dy[stage][t]; }
  __device__ static int8_t dx(int stage, int t) { return c_ms_dx[stage][t]; }
};

template <int IN, int OUT>
__global__ void __launch_bounds__(kCbThreads) ms_dense_kernel(const CbPass S, const CbLayer L) {
  cb_dense<IN, OUT, MsSchedule>(S, L);
}

// ŷ of one stage of group [o, o + C), [B, n_s, C] in coding order -> its positions and channels of [B, H, W, M];
// with `img` (a ragged list of n_img images) image i's n_s,i C values at C q_i -> its [H_i, W_i, M] at M pix_i
__global__ void ms_scatter_kernel(const float* __restrict__ src, float* __restrict__ dst, long long n_k, int W,
                                  long long HW, int M, int o, int C, int stage, long long total,
                                  const CbImage* __restrict__ img, int n_img) {
  cb_scatter<MsSchedule>(src, dst, n_k, W, HW, M, o, C, stage, total, img, n_img);
}

// One group's parameter network: its widths and packed layout.  Group [o, o + C) of a latent of depth M: Wc_1 [4C, 2C],
// bc_1 [2C], Wc_2 [12C, 2C], bc_2, Wc_3 [16C, 2C], bc_3, W1 [K1, N3], b1, W2 [N3, N4], b2, W3 [N4, 2C], b3; at[i] is
// segment i's first float, at[12] the total.  At o = 0, C = M (M a multiple of 6) it is tfcb_msc_packed_floats'.
struct MsNet {
  int C, CH, K1, N3, N4;
  long long at[13];
};

MsNet ms_net(int M, int o, int C) {
  MsNet d;
  d.C = C;
  d.CH = o > 0 ? 2 * C : 0;
  d.K1 = 2 * M + d.CH + 2 * C;
  d.N3 = 5 * d.K1 / 6;
  d.N4 = 2 * d.K1 / 3;
  const long long len[12] = {4ll * C * 2 * C, 2 * C, 12ll * C * 2 * C, 2 * C, 16ll * C * 2 * C, 2 * C,
                             (long long)d.K1 * d.N3, d.N3, (long long)d.N3 * d.N4, d.N4, (long long)d.N4 * 2 * C,
                             2 * C};
  d.at[0] = 0;
  for (int i = 0; i < 12; ++i) d.at[i + 1] = d.at[i] + len[i];
  return d;
}

bool ms_depth_ok(int M) { return M > 0 && M % 6 == 0 && M <= kArMaxM; }

// The space-channel model's groups (§3.12): M even and at most 1024, the group inside the latent.
constexpr int kMsccMaxM = 1024;

bool mscc_group_ok(int M, int o, int C) {
  return M > 0 && M % 2 == 0 && M <= kMsccMaxM && o >= 0 && C >= 1 && o + C <= M;
}

long long ms_count(int64_t H, int64_t W, int stage) {
  return ((H - ms_row_phase(stage) + 1) / 2) * ((W - ms_col_phase(stage) + 1) / 2);
}

long long ms_positions(const CbList& L, int stage) {
  if (!L.hs) return L.B * ms_count(L.H, L.W, stage);
  long long n = 0;
  for (int64_t i = 0; i < L.B; ++i) n += ms_count(L.hs[i], L.ws[i], stage);
  return n;
}

// the stages before `stage`'s positions of an H × W image: where its block of the group's coding order starts, per
// channel
long long ms_before(int64_t H, int64_t W, int stage) {
  long long n = 0;
  for (int s = 0; s < stage; ++s) n += ms_count(H, W, s);
  return n;
}

long long ms_work_floats(const MsNet& d, const CbList& L, int stage) {
  return cb_table_floats(L) + ms_positions(L, stage) * ((stage ? 2 * d.C : 0) + d.N3 + d.N4);
}

int ms_check_depth(int M) {
  if (!ms_depth_ok(M))
    return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be a positive multiple of 6 and at most %d", M,
                kArMaxM);
  return TFCB_OK;
}

int mscc_check_group(int M, int o, int C) {
  if (M <= 0 || M % 2 != 0 || M > kMsccMaxM)
    return fail(TFCB_INVALID_ARGUMENT, "latent depth M=%d must be a positive even number and at most %d", M,
                kMsccMaxM);
  if (o < 0 || C < 1 || o + C > M)
    return fail(TFCB_INVALID_ARGUMENT, "group of %d channels at offset %d does not fit a latent of depth %d", C, o, M);
  return TFCB_OK;
}

int ms_check_stage(int stage) {
  if (stage < 0 || stage >= kMsStages) return fail(TFCB_INVALID_ARGUMENT, "stage %d outside [0, 4)", stage);
  return TFCB_OK;
}

int ms_check_packed(const float* packed, int64_t packed_floats, int M, int o, int C) {
  if (!packed) return fail(TFCB_INVALID_ARGUMENT, "`packed` is null");
  const long long n = ms_net(M, o, C).at[12];
  if (packed_floats != n) {
    if (o == 0 && C == M)
      return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, M=%d needs %lld", (long long)packed_floats,
                  M, n);
    return fail(TFCB_INVALID_ARGUMENT, "packed weights hold %lld floats, the group [%d, %d) of M=%d needs %lld",
                (long long)packed_floats, o, o + C, M, n);
  }
  return TFCB_OK;
}

// Stream-ordered device copies of the twelve operands of ms_net's layout into `packed`, after the caller's checks of
// the group and the packed size.
int ms_pack(const MsNet& d, const float* const src[12], float* packed, void* stream) {
  for (int i = 0; i < 12; ++i)
    if (!src[i]) return fail(TFCB_INVALID_ARGUMENT, "weight operand %d is null", i);
  cudaStream_t s = as_stream(stream);
  for (int i = 0; i < 12; ++i)
    TFCB_CUDA_TRY(cudaMemcpyAsync(packed + d.at[i], src[i], (d.at[i + 1] - d.at[i]) * sizeof(float),
                                  cudaMemcpyDeviceToDevice, s));
  return TFCB_OK;
}

// Uploads the image table of stage `stage` of group [o, o + C) of a ragged list to `work` (one stream-ordered copy
// from pageable memory, staged before the call returns).  Params outputs of image i start at C Q_i (whole == 0), or at
// M P_i + H_i W_i o + C (the positions of its earlier stages) in the coding order of every group (whole != 0).
int ms_upload_table(const CbList& L, int M, int o, int C, int stage, int whole, float* work, cudaStream_t s) {
  std::vector<CbImage> t((size_t)L.B);
  long long q = 0, pix = 0;
  for (int64_t i = 0; i < L.B; ++i) {
    const int64_t H = L.hs[i], W = L.ws[i];
    t[i].q = q;
    t[i].pix = pix;
    t[i].out = whole ? M * pix + H * W * o + C * ms_before(H, W, stage) : C * q;
    t[i].H = (int)H;
    t[i].W = (int)W;
    q += ms_count(H, W, stage);
    pix += H * W;
  }
  TFCB_CUDA_TRY(cudaMemcpyAsync(work, t.data(), t.size() * sizeof(CbImage), cudaMemcpyHostToDevice, s));
  return TFCB_OK;
}

template <int IN, int OUT>
int ms_layer(const CbPass& S, const CbLayer& L, cudaStream_t s) {
  const dim3 grid((unsigned)((S.P + kCbTP - 1) / kCbTP), (unsigned)((L.N + kCbTN - 1) / kCbTN));
  ms_dense_kernel<IN, OUT><<<grid, kCbThreads, 0, s>>>(S, L);
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

// One pass over stage `stage` of group [o, o + C) of a latent of depth M, after the caller's checks of M, the group,
// the stage, the packed size, the images and num_scales.  Outputs [B, n_s, C] (whole == 0), or the coding order of
// every group, [B, H W M], at this pass's block H W o + C (the positions of the earlier stages) (whole != 0); for a
// ragged list, image by image at the offsets of ms_upload_table.
int ms_run(const float* packed, int M, int o, int C, const float* yhat, const float* psi, const float* chctx,
           const CbList& I, int stage, int num_scales, float* work, int64_t work_floats, int whole, float* loc,
           float* scale, int32_t* index, const float* y, float* y_ms, float* yhat_out, void* stream) {
  if (!psi || (stage && !yhat)) return fail(TFCB_INVALID_ARGUMENT, "`psi` or `yhat` is null");
  if (o > 0 && !chctx)
    return fail(TFCB_INVALID_ARGUMENT, "`chctx` is null: the group at channel offset %d needs its channel context", o);
  const MsNet d = ms_net(M, o, C);
  const long long need = ms_work_floats(d, I, stage);
  if (!work || work_floats < need)
    return fail(TFCB_INVALID_ARGUMENT, "workspace of %lld floats, this pass needs %lld", work ? (long long)work_floats : 0ll,
                need);
  if (I.hs) TFCB_TRY(ar_check_table_space(work, work_floats, need, alignof(CbImage)));
  if (y && (!y_ms || !yhat_out || !loc || !index))
    return fail(TFCB_INVALID_ARGUMENT, "the encoder needs `y_ms`, `yhat_out`, `loc` and `index`");
  const long long P = ms_positions(I, stage);
  if (P == 0) return TFCB_OK;
  cudaStream_t s = as_stream(stream);
  CbPass S{};
  S.B = (int)I.B;
  S.M = M;
  S.C = C;
  S.o = o;
  S.CH = d.CH;
  S.colour = stage;
  S.num_scales = num_scales;
  S.P = P;
  if (I.hs) {
    TFCB_TRY(ms_upload_table(I, M, o, C, stage, whole, work, s));
    S.img = reinterpret_cast<const CbImage*>(work);
    S.n_img = (int)I.B;
  } else {
    const long long n_s = ms_count(I.H, I.W, stage);
    S.H = (int)I.H;
    S.W = (int)I.W;
    S.n_k = n_s;
    S.HW = I.H * I.W;
    S.out_stride = whole ? S.HW * M : n_s * C;
    S.out_base = whole ? S.HW * o + ms_before(I.H, I.W, stage) * C : 0;
  }
  S.psi = psi;
  S.chctx = chctx;
  S.yhat = yhat;
  S.loc = loc;
  S.scale = scale;
  S.index = index;
  S.y = y;
  S.y_cb = y_ms;
  S.yhat_out = yhat_out;
  float* ctx = work + cb_table_floats(I);
  float* h1 = ctx + (stage ? S.P * 2 * C : 0);
  float* h2 = h1 + S.P * d.N3;
  if (stage)
    TFCB_TRY((ms_layer<kInTaps, kOutHidden>(S, {packed + d.at[2 * stage - 2], packed + d.at[2 * stage - 1], nullptr, ctx,
                                                ms_taps(stage) * C, 2 * C, ms_taps(stage) * C, false}, s)));
  TFCB_TRY((ms_layer<kInPsiCtx, kOutHidden>(
      S, {packed + d.at[6], packed + d.at[7], ctx, h1, d.K1, d.N3, stage ? d.K1 : d.K1 - 2 * C, true}, s)));
  TFCB_TRY((ms_layer<kInPlain, kOutHidden>(S, {packed + d.at[8], packed + d.at[9], h1, h2, d.N3, d.N4, d.N3, true}, s)));
  return ms_layer<kInPlain, kOutParams>(S, {packed + d.at[10], packed + d.at[11], h2, nullptr, d.N4, 2 * C, d.N4, false},
                                        s);
}

// The scatter of one stage of group [o, o + C), after the caller's checks of the group and the stage; a ragged list's
// table goes to `work`.
int ms_scatter(const float* src, const CbList& I, int M, int o, int C, int stage, float* dst, float* work,
               int64_t work_floats, void* stream) {
  if (!I.hs) {
    TFCB_TRY(ar_check_batch(I.B, I.H, I.W, 1));
  } else {
    TFCB_TRY(ar_check_table_space(work, work_floats, cb_table_floats(I), alignof(CbImage)));
  }
  const long long total = ms_positions(I, stage) * C;
  if (total == 0) return TFCB_OK;  // (an empty stage: empty tensors may have null pointers)
  if (!src || !dst) return fail(TFCB_INVALID_ARGUMENT, "`src` or `dst` is null");
  cudaStream_t s = as_stream(stream);
  const long long blocks = std::min<long long>((total + 255) / 256, 1ll << 16);
  if (I.hs) {
    TFCB_TRY(ms_upload_table(I, M, o, C, stage, 0, work, s));
    ms_scatter_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dst, 0, 0, 0, M, o, C, stage, total,
                                                       reinterpret_cast<const CbImage*>(work), (int)I.B);
  } else {
    ms_scatter_kernel<<<(unsigned)blocks, 256, 0, s>>>(src, dst, ms_count(I.H, I.W, stage), (int)I.W, I.H * I.W, M, o,
                                                       C, stage, total, nullptr, 0);
  }
  TFCB_LAUNCHED();
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}

bool ms_batch_ok(int64_t B, int64_t H, int64_t W) { return B > 0 && H > 0 && W > 0 && H * W <= 0x7FFFFFFF; }

}  // namespace
}  // namespace tfcb

using namespace tfcb;

extern "C" {

// ---- the multistage model: the one group (0, M), M a multiple of 6 ----

int64_t tfcb_msc_packed_floats(int M) { return ms_depth_ok(M) ? ms_net(M, 0, M).at[12] : -1; }

int tfcb_msc_pack_weights(int M, const float* wc1_dev, const float* bc1_dev, const float* wc2_dev,
                          const float* bc2_dev, const float* wc3_dev, const float* bc3_dev, const float* w1_dev,
                          const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                          const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream) {
  TFCB_TRY(ms_check_depth(M));
  TFCB_TRY(ms_check_packed(packed_dev, packed_floats, M, 0, M));
  const float* src[12] = {wc1_dev, bc1_dev, wc2_dev, bc2_dev, wc3_dev, bc3_dev,
                          w1_dev,  b1_dev,  w2_dev,  b2_dev,  w3_dev,  b3_dev};
  return ms_pack(ms_net(M, 0, M), src, packed_dev, stream);
}

int64_t tfcb_msc_workspace_floats(int M, int64_t B, int64_t H, int64_t W, int stage) {
  if (!ms_depth_ok(M) || stage < 0 || stage >= kMsStages || !ms_batch_ok(B, H, W)) return -1;
  return ms_work_floats(ms_net(M, 0, M), {B, H, W, nullptr, nullptr}, stage);
}

int tfcb_msc_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                    int64_t B, int64_t H, int64_t W, int stage, int num_scales, float* work_dev, int64_t work_floats,
                    int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev, const float* y_dev,
                    float* y_ms_dev, float* yhat_out_dev, void* stream) {
  TFCB_TRY(ms_check_depth(M));
  TFCB_TRY(ms_check_stage(stage));
  TFCB_TRY(ms_check_packed(packed_dev, packed_floats, M, 0, M));
  TFCB_TRY(ar_check_batch(B, H, W, num_scales));
  return ms_run(packed_dev, M, 0, M, yhat_dev, psi_dev, nullptr, {B, H, W, nullptr, nullptr}, stage, num_scales,
                work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev, y_ms_dev, yhat_out_dev,
                stream);
}

int tfcb_msc_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int stage, float* dst_dev,
                     void* stream) {
  TFCB_TRY(ms_check_depth(M));
  TFCB_TRY(ms_check_stage(stage));
  return ms_scatter(src_dev, {B, H, W, nullptr, nullptr}, M, 0, M, stage, dst_dev, nullptr, 0, stream);
}

int64_t tfcb_msc_ragged_workspace_floats(int M, int64_t n_images, const int64_t* heights_host,
                                         const int64_t* widths_host, int stage) {
  if (!ms_depth_ok(M) || stage < 0 || stage >= kMsStages || !ar_list_ok(n_images, heights_host, widths_host)) return -1;
  return ms_work_floats(ms_net(M, 0, M), {n_images, 0, 0, heights_host, widths_host}, stage);
}

int tfcb_msc_params_ragged(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev,
                           const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                           const int64_t* widths_host, int stage, int num_scales, float* work_dev,
                           int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev,
                           const float* y_dev, float* y_ms_dev, float* yhat_out_dev, void* stream) {
  TFCB_TRY(ms_check_depth(M));
  TFCB_TRY(ms_check_stage(stage));
  TFCB_TRY(ms_check_packed(packed_dev, packed_floats, M, 0, M));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  return ms_run(packed_dev, M, 0, M, yhat_dev, psi_dev, nullptr, {n_images, 0, 0, heights_host, widths_host}, stage,
                num_scales, work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev, y_ms_dev,
                yhat_out_dev, stream);
}

int tfcb_msc_scatter_ragged(const float* src_dev, int64_t n_images, const int64_t* heights_host,
                            const int64_t* widths_host, int M, int stage, float* work_dev, int64_t work_floats,
                            float* dst_dev, void* stream) {
  TFCB_TRY(ms_check_depth(M));
  TFCB_TRY(ms_check_stage(stage));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, 1));
  return ms_scatter(src_dev, {n_images, 0, 0, heights_host, widths_host}, M, 0, M, stage, dst_dev, work_dev,
                    work_floats, stream);
}

// ---- the space-channel multistage model: group [offset, offset + C) of a depth-M latent ----

int64_t tfcb_mscc_packed_floats(int M, int offset, int C, int64_t* layout) {
  if (!mscc_group_ok(M, offset, C)) return -1;
  const MsNet d = ms_net(M, offset, C);
  if (layout) {
    layout[0] = d.K1;
    layout[1] = d.N3;
    layout[2] = d.N4;
    for (int i = 0; i < 12; ++i) layout[3 + i] = d.at[i];
  }
  return d.at[12];
}

int tfcb_mscc_pack_weights(int M, int offset, int C, const float* wc1_dev, const float* bc1_dev, const float* wc2_dev,
                           const float* bc2_dev, const float* wc3_dev, const float* bc3_dev, const float* w1_dev,
                           const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                           const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream) {
  TFCB_TRY(mscc_check_group(M, offset, C));
  TFCB_TRY(ms_check_packed(packed_dev, packed_floats, M, offset, C));
  const float* src[12] = {wc1_dev, bc1_dev, wc2_dev, bc2_dev, wc3_dev, bc3_dev,
                          w1_dev,  b1_dev,  w2_dev,  b2_dev,  w3_dev,  b3_dev};
  return ms_pack(ms_net(M, offset, C), src, packed_dev, stream);
}

int64_t tfcb_mscc_workspace_floats(int M, int offset, int C, int64_t B, int64_t H, int64_t W, int stage) {
  if (!mscc_group_ok(M, offset, C) || stage < 0 || stage >= kMsStages || !ms_batch_ok(B, H, W)) return -1;
  return ms_work_floats(ms_net(M, offset, C), {B, H, W, nullptr, nullptr}, stage);
}

int tfcb_mscc_params(const float* packed_dev, int64_t packed_floats, int M, int offset, int C, const float* yhat_dev,
                     const float* psi_dev, const float* chctx_dev, int64_t B, int64_t H, int64_t W, int stage,
                     int num_scales, float* work_dev, int64_t work_floats, int whole, float* loc_dev,
                     float* scale_index_dev, int32_t* index_dev, const float* y_dev, float* y_cc_dev,
                     float* yhat_out_dev, void* stream) {
  TFCB_TRY(mscc_check_group(M, offset, C));
  TFCB_TRY(ms_check_stage(stage));
  TFCB_TRY(ms_check_packed(packed_dev, packed_floats, M, offset, C));
  TFCB_TRY(ar_check_batch(B, H, W, num_scales));
  return ms_run(packed_dev, M, offset, C, yhat_dev, psi_dev, chctx_dev, {B, H, W, nullptr, nullptr}, stage,
                num_scales, work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev, y_cc_dev,
                yhat_out_dev, stream);
}

int tfcb_mscc_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int offset, int C, int stage,
                      float* dst_dev, void* stream) {
  TFCB_TRY(mscc_check_group(M, offset, C));
  TFCB_TRY(ms_check_stage(stage));
  return ms_scatter(src_dev, {B, H, W, nullptr, nullptr}, M, offset, C, stage, dst_dev, nullptr, 0, stream);
}

int64_t tfcb_mscc_ragged_workspace_floats(int M, int offset, int C, int64_t n_images, const int64_t* heights_host,
                                          const int64_t* widths_host, int stage) {
  if (!mscc_group_ok(M, offset, C) || stage < 0 || stage >= kMsStages ||
      !ar_list_ok(n_images, heights_host, widths_host))
    return -1;
  return ms_work_floats(ms_net(M, offset, C), {n_images, 0, 0, heights_host, widths_host}, stage);
}

int tfcb_mscc_params_ragged(const float* packed_dev, int64_t packed_floats, int M, int offset, int C,
                            const float* yhat_dev, const float* psi_dev, const float* chctx_dev, int64_t n_images,
                            const int64_t* heights_host, const int64_t* widths_host, int stage, int num_scales,
                            float* work_dev, int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev,
                            int32_t* index_dev, const float* y_dev, float* y_cc_dev, float* yhat_out_dev,
                            void* stream) {
  TFCB_TRY(mscc_check_group(M, offset, C));
  TFCB_TRY(ms_check_stage(stage));
  TFCB_TRY(ms_check_packed(packed_dev, packed_floats, M, offset, C));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, num_scales));
  return ms_run(packed_dev, M, offset, C, yhat_dev, psi_dev, chctx_dev, {n_images, 0, 0, heights_host, widths_host},
                stage, num_scales, work_dev, work_floats, whole, loc_dev, scale_index_dev, index_dev, y_dev, y_cc_dev,
                yhat_out_dev, stream);
}

int tfcb_mscc_scatter_ragged(const float* src_dev, int64_t n_images, const int64_t* heights_host,
                             const int64_t* widths_host, int M, int offset, int C, int stage, float* work_dev,
                             int64_t work_floats, float* dst_dev, void* stream) {
  TFCB_TRY(mscc_check_group(M, offset, C));
  TFCB_TRY(ms_check_stage(stage));
  TFCB_TRY(ar_check_list(n_images, heights_host, widths_host, 1));
  return ms_scatter(src_dev, {n_images, 0, 0, heights_host, widths_host}, M, offset, C, stage, dst_dev, work_dev,
                    work_floats, stream);
}

}  // extern "C"
