// Microbenchmark (not part of the ABI header): how many bytes per microsecond can one SM's async-copy engine move
// into shared memory?  Modes: 0 = 2-D TMA boxes [128 rows x 128 B] with the 128-byte swizzle (what the GDN kernels
// use), 1 = 1-D bulk copies of 16 KB, 2 = 1-D bulk copies of 96 KB, 3 = 2-D boxes + a 2-D TMA store of every box.
// One elected thread per CTA keeps `depth` copies in flight over a ring; nothing is computed.
#include <cuda.h>

#include "common.cuh"

namespace tfcb {
namespace {

__device__ __forceinline__ uint32_t s32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void wait_parity(uint32_t mbar, uint32_t parity) {
  uint32_t done = 0;
  while (!done)
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(mbar), "r"(parity)
        : "memory");
}

__global__ void __launch_bounds__(32, 1) tma_probe_kernel(const __grid_constant__ CUtensorMap map,
                                                          const __grid_constant__ CUtensorMap out_map, const float* base,
                                                          long long n_rows, int C, int mode, int depth, int iters) {
  extern __shared__ __align__(1024) uint8_t smem[];
  __shared__ __align__(8) uint64_t bars[16];
  if (threadIdx.x != 0) return;
  const uint32_t unit = (mode == 2) ? 96u * 1024u : 16u * 1024u;
  for (int i = 0; i < depth; ++i) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(s32(bars + i)));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  const long long tiles = n_rows / 128;
  const int chunks = C / 32;
  for (int n = 0; n < iters + depth; ++n) {
    const int slot = n % depth;
    if (n >= depth) {
      wait_parity(s32(bars + slot), (uint32_t)((n / depth - 1) & 1));
      if (mode == 3) {
        const long long idx = ((long long)blockIdx.x + (long long)(n - depth) * gridDim.x);
        const long long tile = (idx / chunks) % tiles;
        asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(&out_map),
                     "r"((int)(idx % chunks) * 32), "r"((int)(tile * 128)), "r"(s32(smem + slot * unit))
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      }
    }
    if (n < iters) {
      const long long idx = ((long long)blockIdx.x + (long long)n * gridDim.x);
      const uint32_t full = s32(bars + slot);
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"(unit) : "memory");
      if (mode == 0 || mode == 3) {
        const long long tile = (idx / chunks) % tiles;
        asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
                         s32(smem + slot * unit)),
                     "l"(&map), "r"((int)(idx % chunks) * 32), "r"((int)(tile * 128)), "r"(full)
                     : "memory");
      } else {
        const long long off = (idx * (long long)unit) % ((n_rows * C * 4 / unit) * unit);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                         s32(smem + slot * unit)),
                     "l"(reinterpret_cast<const uint8_t*>(base) + off), "r"(unit), "r"(full)
                     : "memory");
      }
    }
  }
  if (mode == 3) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace
}  // namespace tfcb

extern "C" int tfcb_debug_tma_probe(const float* x_dev, float* y_dev, long long n_rows, int C, int mode, int depth, int iters,
                                    float* ms_out, void* stream) {
  using namespace tfcb;
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult st;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &st) != cudaSuccess || !fn)
    return fail(TFCB_CUDA_ERROR, "no cuTensorMapEncodeTiled");
  CUtensorMap maps[2];
  float* bases[2] = {const_cast<float*>(x_dev), y_dev};
  for (int i = 0; i < 2; ++i) {
    const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)n_rows};
    const cuuint64_t strides[1] = {(cuuint64_t)C * 4};
    const cuuint32_t box[2] = {32u, 128u}, es[2] = {1u, 1u};
    if (reinterpret_cast<EncodeFn>(fn)(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, bases[i], dims, strides, box, es,
                                       CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return fail(TFCB_CUDA_ERROR, "tensor map");
  }
  const size_t smem = (size_t)depth * ((mode == 2) ? 96 * 1024 : 16 * 1024);
  if (depth < 1 || depth > 14 || smem > 227 * 1024) return fail(TFCB_INVALID_ARGUMENT, "bad depth");
  TFCB_CUDA_TRY(cudaFuncSetAttribute(tma_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t s = as_stream(stream);
  int dev = 0, sms = 0;
  TFCB_CUDA_TRY(cudaGetDevice(&dev));
  TFCB_CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  tma_probe_kernel<<<sms, 32, smem, s>>>(maps[0], maps[1], x_dev, n_rows, C, mode, depth, 8);  // warm
  cudaEventRecord(a, s);
  tma_probe_kernel<<<sms, 32, smem, s>>>(maps[0], maps[1], x_dev, n_rows, C, mode, depth, iters);
  cudaEventRecord(b, s);
  TFCB_CUDA_TRY(cudaStreamSynchronize(s));
  cudaEventElapsedTime(ms_out, a, b);
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  TFCB_CUDA_TRY(cudaGetLastError());
  return TFCB_OK;
}
