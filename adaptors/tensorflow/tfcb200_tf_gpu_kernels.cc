// TensorFlow adaptor: DEVICE_GPU kernels for the reference's own op definitions, forwarding to the C ABI of
// libtfcb200.so (include/tfcb200.h).  NOT BUILT IN THIS REPOSITORY'S IMAGE (no TensorFlow headers here); it is the
// file a reference maintainer drops next to tensorflow_compression/cc/kernels/ -- see README.md in this directory
// for the build line.  The op DEFINITIONS stay where they are in the reference:
//   cc/ops/range_coder_ops.cc:28-247   CreateRangeEncoder, EntropyEncode{Channel,Index,Finalize},
//                                      CreateRangeDecoder, EntropyDecode{Channel,Index,Finalize}
//   cc/ops/pmf_to_cdf_ops.cc:28-57     PmfToQuantizedCdf
//   cc/ops/quantization_ops.cc:28-53   StochasticRound
//   cc/ops/run_length_ops.cc:28-84, run_length_gamma_ops.cc:26-58   RunLength{,Gamma}{Encode,Decode}
//   cc/ops/range_coding_ops.cc:30-124  RangeEncode, RangeDecode (legacy single-stream ops)
//   cc/ops/range_coding_ops.cc:126-247 UnboundedIndexRangeEncode, UnboundedIndexRangeDecode
// and their CPU kernels stay registered (cc/kernels/range_coder_kernels.cc:505-700 etc.); TensorFlow's placer picks
// the GPU kernel when the data tensors live on the GPU, so python/ops/gen_ops.py and models/*.py are unchanged.
// GDN has no op in the reference (python/layers/gdn.py:371-421 composes TF ops): GdnForward / GdnBackward are
// defined at the bottom of this file together with the tf.custom_gradient wrapper a maintainer would put in GDN.call.
#include <memory>
#include <string>
#include <vector>

#include "tensorflow/core/framework/op.h"
#include "tensorflow/core/framework/op_kernel.h"
#include "tensorflow/core/framework/shape_inference.h"
#include "tensorflow/core/framework/tensor.h"
#include "tensorflow/core/framework/tensor_shape.h"
#include "tensorflow/core/framework/variant.h"
#include "tensorflow/core/framework/variant_op_registry.h"
#include "tensorflow/core/platform/errors.h"
#include "tensorflow/core/platform/stream_executor.h"
#include "tfcb200.h"

namespace tfcb200_tf {
namespace {
namespace tf = tensorflow;
using tf::errors::InvalidArgument;

// cudaStream_t of the op's compute stream (what every tfcb_* entry takes as `void* stream`).
void* CudaStream(tf::OpKernelContext* ctx) {
  return reinterpret_cast<void*>(ctx->op_device_context()->stream()->platform_specific_handle().stream);
}

tf::Status FromRc(int rc) {
  if (rc == TFCB_OK) return tf::OkStatus();
  if (rc == TFCB_INVALID_ARGUMENT) return InvalidArgument(tfcb_last_error());
  if (rc == TFCB_OUT_OF_MEMORY) return tf::errors::ResourceExhausted(tfcb_last_error());
  return tf::errors::Internal(tfcb_last_error());
}

// The DT_VARIANT payloads: the counterpart of EntropyEncoderVariant / EntropyDecoderVariant
// (cc/kernels/range_coder_kernels.cc:62-78,326-329,475-478).  The C handle owns the per-stream coder state, the
// device arena and its copy of `lookup`; the variant keeps the handle shape for the shape checks.
struct GpuEncoderVariant {
  std::shared_ptr<tfcb_encoder> handle;
  tf::TensorShape shape;
  std::string TypeName() const { return "(anonymous)::tfcb200::GpuEncoderVariant"; }
  void Encode(tf::VariantTensorData*) const { LOG(ERROR) << "Encode() not implemented."; }
  bool Decode(const tf::VariantTensorData&) const { LOG(ERROR) << "Decode() not implemented."; return false; }
};
struct GpuDecoderVariant {
  std::shared_ptr<tfcb_decoder> handle;
  tf::TensorShape shape;
  tf::Tensor device_bytes, device_offsets;  // the strings, copied to the device once (the C handle borrows them)
  std::string TypeName() const { return "(anonymous)::tfcb200::GpuDecoderVariant"; }
  void Encode(tf::VariantTensorData*) const { LOG(ERROR) << "Encode() not implemented."; }
  bool Decode(const tf::VariantTensorData&) const { LOG(ERROR) << "Decode() not implemented."; return false; }
};

// `lookup` is 1-D (concatenated rows) or 2-D (stacked rows): cols = 0 or the row length (tfcb200.h).
tf::Status LookupArgs(const tf::Tensor& lookup, int64_t* len, int64_t* cols) {
  if (lookup.dims() != 1 && lookup.dims() != 2) return InvalidArgument("'lookup' should be 1-D or 2-D.");
  *len = lookup.NumElements();
  *cols = lookup.dims() == 2 ? lookup.dim_size(1) : 0;
  return tf::OkStatus();
}

// ---- CreateRangeEncoder (range_coder_kernels.cc:484-507) ----
class CreateRangeEncoderGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    tf::TensorShape shape;
    OP_REQUIRES_OK(ctx, tf::tensor::MakeShape(ctx->input(0), &shape));
    const tf::Tensor& lookup = ctx->input(1);  // host memory
    int64_t len, cols;
    OP_REQUIRES_OK(ctx, LookupArgs(lookup, &len, &cols));
    tfcb_encoder* raw = nullptr;
    OP_REQUIRES_OK(ctx, FromRc(tfcb_encoder_create(lookup.flat<int32_t>().data(), len, cols, shape.num_elements(),
                                                  CudaStream(ctx), &raw)));
    GpuEncoderVariant v;
    v.handle.reset(raw, tfcb_encoder_destroy);
    v.shape = shape;
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, tf::TensorShape({}), &out));
    out->scalar<tf::Variant>()() = std::move(v);
  }
};
REGISTER_KERNEL_BUILDER(
    Name("CreateRangeEncoder").Device(tf::DEVICE_GPU).HostMemory("shape").HostMemory("lookup").HostMemory("handle"),
    CreateRangeEncoderGpuOp);

tf::Status GetEncoder(tf::OpKernelContext* ctx, GpuEncoderVariant** v) {
  const tf::Tensor& h = ctx->input(0);
  if (h.dims() != 0) return InvalidArgument("'handle' must be a scalar.");
  *v = const_cast<tf::Variant&>(h.scalar<tf::Variant>()()).get<GpuEncoderVariant>();
  if (*v == nullptr || !(*v)->handle) return InvalidArgument("'handle' is not an encoder");
  return tf::OkStatus();
}

// ---- EntropyEncodeChannel / EntropyEncodeIndex (range_coder_kernels.cc:509-592) ----
template <bool kIndex>
class EntropyEncodeGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    GpuEncoderVariant* v;
    OP_REQUIRES_OK(ctx, GetEncoder(ctx, &v));
    const tf::Tensor& value = ctx->input(kIndex ? 2 : 1);
    OP_REQUIRES(ctx, tf::TensorShapeUtils::StartsWith(value.shape(), v->shape),
                InvalidArgument("'value' shape should start with 'handle' shape: value.shape=", value.shape().DebugString(),
                                " does not start with handle.shape=", v->shape.DebugString()));  // :528-535
    const int64_t streams = v->shape.num_elements();
    const int64_t n = streams ? value.NumElements() / streams : 0;
    int rc;
    if (kIndex) {
      const tf::Tensor& index = ctx->input(1);
      OP_REQUIRES(ctx, index.shape() == value.shape(),
                  InvalidArgument("'index' shape should match 'value' shape"));  // :545-549
      rc = tfcb_encode_index(v->handle.get(), index.flat<int32_t>().data(), value.flat<int32_t>().data(), n, CudaStream(ctx));
    } else {
      rc = tfcb_encode_channel(v->handle.get(), value.flat<int32_t>().data(), n, CudaStream(ctx));
    }
    OP_REQUIRES_OK(ctx, FromRc(rc));
    ctx->set_output(0, ctx->input(0));  // aliased handle
  }
};
REGISTER_KERNEL_BUILDER(Name("EntropyEncodeChannel").Device(tf::DEVICE_GPU).HostMemory("handle").HostMemory("aliased_handle"),
                        EntropyEncodeGpuOp<false>);
REGISTER_KERNEL_BUILDER(Name("EntropyEncodeIndex").Device(tf::DEVICE_GPU).HostMemory("handle").HostMemory("aliased_handle"),
                        EntropyEncodeGpuOp<true>);

// ---- EntropyEncodeFinalize (range_coder_kernels.cc:594-619): device-side range errors surface here ----
// The strings are packed on the device into temporaries and copied out, as RunLengthEncode does below.
class EntropyEncodeFinalizeGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    GpuEncoderVariant* v;
    OP_REQUIRES_OK(ctx, GetEncoder(ctx, &v));
    const int64_t streams = v->shape.num_elements();
    tf::Tensor offsets_dev, bytes_dev;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_INT64, tf::TensorShape({streams + 1}), &offsets_dev));
    int64_t total = 0;
    OP_REQUIRES_OK(ctx, FromRc(tfcb_encode_finalize(v->handle.get(), offsets_dev.flat<int64_t>().data(), CudaStream(ctx),
                                                   &total)));
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({total > 0 ? total : 1}), &bytes_dev));
    OP_REQUIRES_OK(ctx, FromRc(tfcb_encode_write(v->handle.get(), offsets_dev.flat<int64_t>().data(),
                                                bytes_dev.flat<uint8_t>().data(), CudaStream(ctx))));
    std::vector<uint8_t> bytes(total > 0 ? total : 1);
    std::vector<int64_t> offsets(streams + 1);
    auto* stream = ctx->op_device_context()->stream();
    stream_executor::DeviceMemoryBase src_bytes(bytes_dev.flat<uint8_t>().data(), static_cast<uint64_t>(total));
    stream_executor::DeviceMemoryBase src_offsets(offsets_dev.flat<int64_t>().data(), offsets.size() * sizeof(int64_t));
    if (total > 0) OP_REQUIRES_OK(ctx, stream->Memcpy(bytes.data(), src_bytes, static_cast<uint64_t>(total)));
    OP_REQUIRES_OK(ctx, stream->Memcpy(offsets.data(), src_offsets, offsets.size() * sizeof(int64_t)));
    OP_REQUIRES_OK(ctx, stream->BlockHostUntilDone());
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, v->shape, &out));
    auto flat = out->flat<tf::tstring>();
    for (int64_t i = 0; i < streams; ++i)
      flat(i).assign(reinterpret_cast<const char*>(bytes.data() + offsets[i]), offsets[i + 1] - offsets[i]);
  }
};
REGISTER_KERNEL_BUILDER(Name("EntropyEncodeFinalize").Device(tf::DEVICE_GPU).HostMemory("handle").HostMemory("encoded"),
                        EntropyEncodeFinalizeGpuOp);

// ---- CreateRangeDecoder (range_coder_kernels.cc:621-646) ----
class CreateRangeDecoderGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& encoded = ctx->input(0);  // host memory (tstring)
    const tf::Tensor& lookup = ctx->input(1);   // host memory
    int64_t len, cols;
    OP_REQUIRES_OK(ctx, LookupArgs(lookup, &len, &cols));
    const int64_t streams = encoded.NumElements();
    auto strings = encoded.flat<tf::tstring>();
    std::vector<int64_t> offsets(streams + 1, 0);
    for (int64_t i = 0; i < streams; ++i) offsets[i + 1] = offsets[i] + static_cast<int64_t>(strings(i).size());
    GpuDecoderVariant v;
    v.shape = encoded.shape();
    tf::AllocatorAttributes pinned;
    pinned.set_on_host(true);
    pinned.set_gpu_compatible(true);
    tf::Tensor host_bytes, host_offsets;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({offsets[streams] + 1}), &host_bytes, pinned));
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_INT64, tf::TensorShape({streams + 1}), &host_offsets, pinned));
    for (int64_t i = 0; i < streams; ++i)
      memcpy(host_bytes.flat<uint8_t>().data() + offsets[i], strings(i).data(), strings(i).size());
    memcpy(host_offsets.flat<int64_t>().data(), offsets.data(), offsets.size() * sizeof(int64_t));
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, host_bytes.shape(), &v.device_bytes));
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_INT64, host_offsets.shape(), &v.device_offsets));
    auto* dc = ctx->op_device_context();
    auto* dev = static_cast<tf::Device*>(ctx->device());
    tf::Status copy_status;
    dc->CopyCPUTensorToDeviceSync(&host_bytes, dev, &v.device_bytes);      // (any H2D primitive of the TF version at hand)
    dc->CopyCPUTensorToDeviceSync(&host_offsets, dev, &v.device_offsets);
    tfcb_decoder* raw = nullptr;
    OP_REQUIRES_OK(ctx, FromRc(tfcb_decoder_create(v.device_bytes.flat<uint8_t>().data(), v.device_offsets.flat<int64_t>().data(),
                                                  streams, lookup.flat<int32_t>().data(), len, cols, CudaStream(ctx), &raw)));
    v.handle.reset(raw, tfcb_decoder_destroy);
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, tf::TensorShape({}), &out));
    out->scalar<tf::Variant>()() = std::move(v);
  }
};
REGISTER_KERNEL_BUILDER(
    Name("CreateRangeDecoder").Device(tf::DEVICE_GPU).HostMemory("encoded").HostMemory("lookup").HostMemory("handle"),
    CreateRangeDecoderGpuOp);

tf::Status GetDecoder(tf::OpKernelContext* ctx, GpuDecoderVariant** v) {
  const tf::Tensor& h = ctx->input(0);
  if (h.dims() != 0) return InvalidArgument("'handle' must be a scalar.");
  *v = const_cast<tf::Variant&>(h.scalar<tf::Variant>()()).get<GpuDecoderVariant>();
  if (*v == nullptr || !(*v)->handle) return InvalidArgument("'handle' is not a decoder");
  return tf::OkStatus();
}

// ---- EntropyDecodeChannel / EntropyDecodeIndex (range_coder_kernels.cc:648-678) ----
template <bool kIndex>
class EntropyDecodeGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    GpuDecoderVariant* v;
    OP_REQUIRES_OK(ctx, GetDecoder(ctx, &v));
    tf::TensorShape suffix;
    OP_REQUIRES_OK(ctx, tf::tensor::MakeShape(ctx->input(kIndex ? 2 : 1), &suffix));  // `shape`, host memory
    tf::TensorShape out_shape = v->shape;
    out_shape.AppendShape(suffix);
    tf::Tensor* decoded;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(1, out_shape, &decoded));
    int rc;
    if (kIndex) {
      const tf::Tensor& index = ctx->input(1);
      OP_REQUIRES(ctx, index.shape() == out_shape,
                  InvalidArgument("'index' shape should be handle.shape + shape"));  // :656-661
      rc = tfcb_decode_index(v->handle.get(), index.flat<int32_t>().data(), decoded->flat<int32_t>().data(),
                             suffix.num_elements(), CudaStream(ctx));
    } else {
      rc = tfcb_decode_channel(v->handle.get(), decoded->flat<int32_t>().data(), suffix.num_elements(), CudaStream(ctx));
    }
    OP_REQUIRES_OK(ctx, FromRc(rc));
    ctx->set_output(0, ctx->input(0));
  }
};
REGISTER_KERNEL_BUILDER(Name("EntropyDecodeChannel").Device(tf::DEVICE_GPU).HostMemory("handle").HostMemory("shape").HostMemory("aliased_handle")
                            .TypeConstraint<int32_t>("Tdecoded"),
                        EntropyDecodeGpuOp<false>);
REGISTER_KERNEL_BUILDER(Name("EntropyDecodeIndex").Device(tf::DEVICE_GPU).HostMemory("handle").HostMemory("shape").HostMemory("aliased_handle")
                            .TypeConstraint<int32_t>("Tdecoded"),
                        EntropyDecodeGpuOp<true>);

// ---- EntropyDecodeFinalize (range_coder_kernels.cc:680-700) ----
class EntropyDecodeFinalizeGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    GpuDecoderVariant* v;
    OP_REQUIRES_OK(ctx, GetDecoder(ctx, &v));
    std::vector<uint8_t> ok(v->shape.num_elements() + 1);
    OP_REQUIRES_OK(ctx, FromRc(tfcb_decode_finalize(v->handle.get(), ok.data(), CudaStream(ctx))));
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, v->shape, &out));
    auto flat = out->flat<bool>();
    for (int64_t i = 0; i < flat.size(); ++i) flat(i) = ok[i] != 0;
  }
};
REGISTER_KERNEL_BUILDER(Name("EntropyDecodeFinalize").Device(tf::DEVICE_GPU).HostMemory("handle").HostMemory("success"),
                        EntropyDecodeFinalizeGpuOp);

// ---- PmfToQuantizedCdf (pmf_to_cdf_kernels.cc:58-101) ----
class PmfToCdfGpuOp : public tf::OpKernel {
 public:
  explicit PmfToCdfGpuOp(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    OP_REQUIRES_OK(c, c->GetAttr("precision", &precision_));
    OP_REQUIRES(c, 0 < precision_ && precision_ <= 16, InvalidArgument("`precision` must be in [1, 16]: ", precision_));
  }
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& pmf = ctx->input(0);
    OP_REQUIRES(ctx, pmf.dims() >= 1 && pmf.dim_size(pmf.dims() - 1) > 1,
                InvalidArgument("`pmf` size should be at least 2 in the last axis."));
    tf::TensorShape shape = pmf.shape();
    const int64_t n = shape.dim_size(shape.dims() - 1);
    shape.set_dim(shape.dims() - 1, n + 1);
    tf::Tensor* cdf;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, shape, &cdf));
    OP_REQUIRES_OK(ctx, FromRc(tfcb_pmf_to_quantized_cdf(pmf.flat<float>().data(), pmf.NumElements() / n, n, precision_,
                                                        cdf->flat<int32_t>().data(), CudaStream(ctx))));
  }
 private:
  int precision_;
};
REGISTER_KERNEL_BUILDER(Name("PmfToQuantizedCdf").Device(tf::DEVICE_GPU), PmfToCdfGpuOp);

// ---- StochasticRound (quantization_kernels.cc:48-108): same integers as the CPU kernel for the same seed ----
template <typename T, int kDtype>
class StochasticRoundGpuOp : public tf::OpKernel {
 public:
  using tf::OpKernel::OpKernel;
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& inputs = ctx->input(0);
    OP_REQUIRES(ctx, ctx->input(1).dims() == 0, InvalidArgument("step_size must be a scalar."));
    const float step = ctx->input(1).scalar<float>()();  // host memory
    auto seed = ctx->input(2).flat<int32_t>();            // host memory
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, inputs.shape(), &out));
    OP_REQUIRES_OK(ctx, FromRc(tfcb_stochastic_round(inputs.flat<T>().data(), kDtype, inputs.NumElements(), step, seed.data(),
                                                    seed.size(), out->flat<int32_t>().data(), CudaStream(ctx))));
  }
};
#define TFCB_REGISTER_SR(T, code)                                                                                   \
  REGISTER_KERNEL_BUILDER(Name("StochasticRound").Device(tf::DEVICE_GPU).TypeConstraint<T>("T").HostMemory("step_size") \
                              .HostMemory("seed"),                                                                   \
                          StochasticRoundGpuOp<T, code>)
TFCB_REGISTER_SR(float, 0);
TFCB_REGISTER_SR(Eigen::half, 1);
TFCB_REGISTER_SR(tf::bfloat16, 2);
#undef TFCB_REGISTER_SR

// ---- RunLengthEncode / RunLengthGammaEncode (run_length_kernels.cc:52-139, run_length_gamma_kernels.cc:51-101) ----
// `data` on the device, `code` (a scalar tf.string) in host memory: the bits are packed on the device into a
// temporary and copied out once the length is known (tfcb_run_length_encode synchronises to report it).
class RunLengthEncodeGpuOp : public tf::OpKernel {
 public:
  explicit RunLengthEncodeGpuOp(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    if (c->HasAttr("run_length_code")) {   // RunLengthGammaEncode has no attributes: gamma / gamma / false
      OP_REQUIRES_OK(c, c->GetAttr("run_length_code", &run_length_code_));
      OP_REQUIRES_OK(c, c->GetAttr("magnitude_code", &magnitude_code_));
      OP_REQUIRES_OK(c, c->GetAttr("use_run_length_for_non_zeros", &non_zero_runs_));
    }
  }
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& data = ctx->input(0);
    tf::Tensor* code;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, tf::TensorShape({}), &code));
    const int64_t n = data.NumElements();
    if (n == 0) return;
    int64_t cap = 4 * ((2 * n + 64 + 3) / 4), n_bytes = 0;
    tf::Tensor tmp;
    for (int attempt = 0; attempt < 2; ++attempt) {       // a second pass only if the first guess was too small
      OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({cap}), &tmp));
      const int rc = tfcb_run_length_encode(data.flat<int32_t>().data(), n, run_length_code_, magnitude_code_,
                                            non_zero_runs_ ? 1 : 0, tmp.flat<uint8_t>().data(), cap, &n_bytes,
                                            CudaStream(ctx));
      if (rc == TFCB_INVALID_ARGUMENT && n_bytes > cap - 4 && attempt == 0) {
        cap = 4 * ((n_bytes + 3) / 4) + 4;
        continue;
      }
      OP_REQUIRES_OK(ctx, FromRc(rc));
      break;
    }
    std::string host(static_cast<size_t>(n_bytes), '\0');
    auto* stream = ctx->op_device_context()->stream();
    stream_executor::DeviceMemoryBase src(tmp.flat<uint8_t>().data(), static_cast<uint64_t>(n_bytes));
    OP_REQUIRES_OK(ctx, stream->Memcpy(&host[0], src, static_cast<uint64_t>(n_bytes)));
    OP_REQUIRES_OK(ctx, stream->BlockHostUntilDone());
    code->scalar<tf::tstring>()() = std::move(host);
  }
 private:
  int run_length_code_ = -1, magnitude_code_ = -1;
  bool non_zero_runs_ = false;
};
REGISTER_KERNEL_BUILDER(Name("RunLengthEncode").Device(tf::DEVICE_GPU).HostMemory("code"), RunLengthEncodeGpuOp);
REGISTER_KERNEL_BUILDER(Name("RunLengthGammaEncode").Device(tf::DEVICE_GPU).HostMemory("code"), RunLengthEncodeGpuOp);

// ---- RunLengthDecode / RunLengthGammaDecode (run_length_kernels.cc:141-262) ----
class RunLengthDecodeGpuOp : public tf::OpKernel {
 public:
  explicit RunLengthDecodeGpuOp(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    if (c->HasAttr("run_length_code")) {
      OP_REQUIRES_OK(c, c->GetAttr("run_length_code", &run_length_code_));
      OP_REQUIRES_OK(c, c->GetAttr("magnitude_code", &magnitude_code_));
      OP_REQUIRES_OK(c, c->GetAttr("use_run_length_for_non_zeros", &non_zero_runs_));
    }
  }
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& code = ctx->input(0);   // host memory
    OP_REQUIRES(ctx, tf::TensorShapeUtils::IsScalar(code.shape()),
                InvalidArgument("Invalid `code` shape: ", code.shape().DebugString()));
    OP_REQUIRES(ctx, tf::TensorShapeUtils::IsVector(ctx->input(1).shape()),
                InvalidArgument("Invalid `shape` shape: ", ctx->input(1).shape().DebugString()));
    tf::TensorShape shape;
    OP_REQUIRES_OK(ctx, tf::tensor::MakeShape(ctx->input(1), &shape));
    tf::Tensor* data;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, shape, &data));
    const tf::tstring& bytes = code.scalar<tf::tstring>()();
    tf::Tensor dev;                            // the string on the device, padded so that word reads stay inside
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({static_cast<int64_t>(bytes.size()) + 4}), &dev));
    auto* stream = ctx->op_device_context()->stream();
    stream_executor::DeviceMemoryBase dst(dev.flat<uint8_t>().data(), bytes.size());
    if (!bytes.empty()) OP_REQUIRES_OK(ctx, stream->Memcpy(&dst, bytes.data(), bytes.size()));
    // decode errors come back as the reference's DataLoss messages ("Out of bits to read." ...)
    const int rc = tfcb_run_length_decode(dev.flat<uint8_t>().data(), static_cast<int64_t>(bytes.size()), run_length_code_,
                                          magnitude_code_, non_zero_runs_ ? 1 : 0, data->flat<int32_t>().data(),
                                          data->NumElements(), CudaStream(ctx));
    OP_REQUIRES(ctx, rc == TFCB_OK, rc == TFCB_INVALID_ARGUMENT ? tf::errors::DataLoss(tfcb_last_error())
                                                                : FromRc(rc));
  }
 private:
  int run_length_code_ = -1, magnitude_code_ = -1;
  bool non_zero_runs_ = false;
};
REGISTER_KERNEL_BUILDER(Name("RunLengthDecode").Device(tf::DEVICE_GPU).HostMemory("code").HostMemory("shape"),
                        RunLengthDecodeGpuOp);
REGISTER_KERNEL_BUILDER(Name("RunLengthGammaDecode").Device(tf::DEVICE_GPU).HostMemory("code").HostMemory("shape"),
                        RunLengthDecodeGpuOp);

// ---- RangeEncode / RangeDecode, the legacy single-stream ops (range_coding_kernels.cc:176-379) ----
std::vector<int64_t> Dims(const tf::TensorShape& shape) {
  std::vector<int64_t> d(shape.dims());
  for (int i = 0; i < shape.dims(); ++i) d[i] = shape.dim_size(i);
  return d;
}

class RangeEncodeGpuOp : public tf::OpKernel {
 public:
  explicit RangeEncodeGpuOp(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    OP_REQUIRES_OK(c, c->GetAttr("precision", &precision_));
    OP_REQUIRES_OK(c, c->GetAttr("debug_level", &debug_level_));
    OP_REQUIRES(c, 0 < precision_ && precision_ <= 16, InvalidArgument("`precision` must be in [1, 16]: ", precision_));
  }
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& data = ctx->input(0);
    const tf::Tensor& cdf = ctx->input(1);
    const std::vector<int64_t> ds = Dims(data.shape()), cs = Dims(cdf.shape());
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, tf::TensorShape({}), &out));
    // a symbol costs at most `precision` <= 16 bits; the coder flushes at most four more bytes
    std::string host(static_cast<size_t>(2 * data.NumElements() + 16), '\0');
    int64_t n_bytes = 0;
    OP_REQUIRES_OK(ctx, FromRc(tfcb_range_encode(data.flat<int16_t>().data(), ds.data(), data.dims(),
                                                cdf.flat<int32_t>().data(), cs.data(), cdf.dims(), precision_, debug_level_,
                                                reinterpret_cast<uint8_t*>(&host[0]), static_cast<int64_t>(host.size()),
                                                &n_bytes, CudaStream(ctx))));
    host.resize(static_cast<size_t>(n_bytes));
    out->scalar<tf::tstring>()() = std::move(host);
  }
 private:
  int precision_, debug_level_;
};
REGISTER_KERNEL_BUILDER(Name("RangeEncode").Device(tf::DEVICE_GPU).HostMemory("encoded"), RangeEncodeGpuOp);

class RangeDecodeGpuOp : public tf::OpKernel {
 public:
  explicit RangeDecodeGpuOp(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    OP_REQUIRES_OK(c, c->GetAttr("precision", &precision_));
    OP_REQUIRES_OK(c, c->GetAttr("debug_level", &debug_level_));
    OP_REQUIRES(c, 0 < precision_ && precision_ <= 16, InvalidArgument("`precision` must be in [1, 16]: ", precision_));
  }
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& encoded = ctx->input(0);   // host memory
    const tf::Tensor& cdf = ctx->input(2);
    OP_REQUIRES(ctx, tf::TensorShapeUtils::IsScalar(encoded.shape()),
                InvalidArgument("Invalid `encoded` shape: ", encoded.shape().DebugString()));
    OP_REQUIRES(ctx, tf::TensorShapeUtils::IsVector(ctx->input(1).shape()),
                InvalidArgument("Invalid `shape` shape: ", ctx->input(1).shape().DebugString()));
    tf::TensorShape shape;
    OP_REQUIRES_OK(ctx, tf::tensor::MakeShape(ctx->input(1), &shape));
    const std::vector<int64_t> ds = Dims(shape), cs = Dims(cdf.shape());
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, shape, &out));
    const tf::tstring& bytes = encoded.scalar<tf::tstring>()();
    OP_REQUIRES_OK(ctx, FromRc(tfcb_range_decode(reinterpret_cast<const uint8_t*>(bytes.data()),
                                                static_cast<int64_t>(bytes.size()), ds.data(), shape.dims(),
                                                cdf.flat<int32_t>().data(), cs.data(), cdf.dims(), precision_, debug_level_,
                                                out->flat<int16_t>().data(), CudaStream(ctx))));
  }
 private:
  int precision_, debug_level_;
};
REGISTER_KERNEL_BUILDER(Name("RangeDecode").Device(tf::DEVICE_GPU).HostMemory("encoded").HostMemory("shape"),
                        RangeDecodeGpuOp);

// ---- UnboundedIndexRangeEncode / Decode (unbounded_index_range_coding_kernels.cc): the one-item case of the
// library's ragged entries; `encoded` lives in host memory as for RangeEncode ----
class UnboundedIndexRangeGpuOpBase : public tf::OpKernel {
 public:
  explicit UnboundedIndexRangeGpuOpBase(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    OP_REQUIRES_OK(c, c->GetAttr("precision", &precision_));
    OP_REQUIRES_OK(c, c->GetAttr("overflow_width", &overflow_width_));
    OP_REQUIRES_OK(c, c->GetAttr("debug_level", &debug_level_));
  }
 protected:
  // cdf_size and offset must be vectors (the library sees their lengths only).
  tf::Status TableShapes(tf::OpKernelContext* ctx, int first, std::vector<int64_t>* cs) {
    const tf::Tensor& cdf = ctx->input(first);
    if (!tf::TensorShapeUtils::IsVector(ctx->input(first + 1).shape()))
      return InvalidArgument("'cdf_size' should be 1-D and its length should match the number of rows in 'cdf': ",
                             ctx->input(first + 1).shape().DebugString());
    if (!tf::TensorShapeUtils::IsVector(ctx->input(first + 2).shape()))
      return InvalidArgument("'offset' should be 1-D and its length should match the number of rows in 'cdf': "
                             "offset.shape=", ctx->input(first + 2).shape().DebugString());
    *cs = Dims(cdf.shape());
    return tf::OkStatus();
  }
  int precision_, overflow_width_, debug_level_;
};

class UnboundedIndexRangeEncodeGpuOp : public UnboundedIndexRangeGpuOpBase {
 public:
  using UnboundedIndexRangeGpuOpBase::UnboundedIndexRangeGpuOpBase;
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& data = ctx->input(0);
    const tf::Tensor& index = ctx->input(1);
    OP_REQUIRES(ctx, data.shape() == index.shape(),
                InvalidArgument("`data` and `index` should have the same shape: data.shape=",
                                data.shape().DebugString(), ", index.shape=", index.shape().DebugString()));
    std::vector<int64_t> cs;
    OP_REQUIRES_OK(ctx, TableShapes(ctx, 2, &cs));
    const int64_t items[2] = {0, data.NumElements()};
    tf::Tensor offsets;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_INT64, tf::TensorShape({2}), &offsets));
    tfcb_ubi_encoder* h = nullptr;
    int64_t total = 0;
    OP_REQUIRES_OK(ctx, FromRc(tfcb_unbounded_index_range_encode_ragged(
                            data.flat<int32_t>().data(), index.flat<int32_t>().data(), 1, items,
                            ctx->input(2).flat<int32_t>().data(), cs.data(), ctx->input(2).dims(),
                            ctx->input(3).flat<int32_t>().data(), ctx->input(3).NumElements(),
                            ctx->input(4).flat<int32_t>().data(), ctx->input(4).NumElements(), precision_,
                            overflow_width_, debug_level_, offsets.flat<int64_t>().data(), CudaStream(ctx), &h,
                            &total)));
    tf::Tensor bytes;
    tf::Status st = ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({std::max<int64_t>(total, 1)}), &bytes);
    if (!st.ok()) {
      tfcb_unbounded_index_range_encoder_destroy(h);
      ctx->SetStatus(st);
      return;
    }
    OP_REQUIRES_OK(ctx, FromRc(tfcb_unbounded_index_range_write(h, bytes.flat<uint8_t>().data(), CudaStream(ctx))));
    std::string host(static_cast<size_t>(total), '\0');
    if (total > 0) {
      auto* stream = ctx->op_device_context()->stream();
      stream_executor::DeviceMemoryBase src(bytes.flat<uint8_t>().data(), static_cast<uint64_t>(total));
      OP_REQUIRES_OK(ctx, stream->Memcpy(&host[0], src, static_cast<uint64_t>(total)));
      OP_REQUIRES_OK(ctx, stream->BlockHostUntilDone());
    }
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, tf::TensorShape({}), &out));
    out->scalar<tf::tstring>()() = std::move(host);
  }
};
REGISTER_KERNEL_BUILDER(Name("UnboundedIndexRangeEncode").Device(tf::DEVICE_GPU).HostMemory("encoded"),
                        UnboundedIndexRangeEncodeGpuOp);

class UnboundedIndexRangeDecodeGpuOp : public UnboundedIndexRangeGpuOpBase {
 public:
  using UnboundedIndexRangeGpuOpBase::UnboundedIndexRangeGpuOpBase;
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& encoded = ctx->input(0);  // host memory
    const tf::Tensor& index = ctx->input(1);
    OP_REQUIRES(ctx, tf::TensorShapeUtils::IsScalar(encoded.shape()),
                InvalidArgument("`encoded` should be a scalar: ", encoded.shape().DebugString()));
    std::vector<int64_t> cs;
    OP_REQUIRES_OK(ctx, TableShapes(ctx, 2, &cs));
    const tf::tstring& src = encoded.scalar<tf::tstring>()();
    const int64_t n_bytes = static_cast<int64_t>(src.size());
    tf::Tensor bytes, offsets;
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({std::max<int64_t>(n_bytes, 1)}), &bytes));
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_INT64, tf::TensorShape({2}), &offsets));
    auto* stream = ctx->op_device_context()->stream();
    const int64_t host_offsets[2] = {0, n_bytes};
    stream_executor::DeviceMemoryBase d_bytes(bytes.flat<uint8_t>().data(), static_cast<uint64_t>(n_bytes));
    stream_executor::DeviceMemoryBase d_offsets(offsets.flat<int64_t>().data(), 16);
    if (n_bytes > 0) OP_REQUIRES_OK(ctx, stream->Memcpy(&d_bytes, src.data(), static_cast<uint64_t>(n_bytes)));
    OP_REQUIRES_OK(ctx, stream->Memcpy(&d_offsets, host_offsets, 16));
    tf::Tensor* out;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, index.shape(), &out));
    const int64_t items[2] = {0, index.NumElements()};
    OP_REQUIRES_OK(ctx, FromRc(tfcb_unbounded_index_range_decode_ragged(
                            bytes.flat<uint8_t>().data(), offsets.flat<int64_t>().data(), 1, items,
                            index.flat<int32_t>().data(), ctx->input(2).flat<int32_t>().data(), cs.data(),
                            ctx->input(2).dims(), ctx->input(3).flat<int32_t>().data(), ctx->input(3).NumElements(),
                            ctx->input(4).flat<int32_t>().data(), ctx->input(4).NumElements(), precision_,
                            overflow_width_, debug_level_, out->flat<int32_t>().data(), CudaStream(ctx))));
  }
};
REGISTER_KERNEL_BUILDER(Name("UnboundedIndexRangeDecode").Device(tf::DEVICE_GPU).HostMemory("encoded"),
                        UnboundedIndexRangeDecodeGpuOp);

// ---- GDN: two new ops (the reference has none); see gdn_custom_gradient.py in this directory ----
REGISTER_OP("GdnForward")
    .Input("x: float32").Input("gamma: float32").Input("beta: float32").Output("y: float32")
    .Attr("inverse: bool = false").Attr("rectify: bool = false").Attr("alpha: float = 1.0").Attr("epsilon: float = 1.0")
    .SetShapeFn(tf::shape_inference::UnchangedShape)
    .Doc("y = u / (beta + pool(u) . gamma)^epsilon (IGDN: u * ...), channels last; python/layers/gdn.py:371-421.");
REGISTER_OP("GdnBackward")
    .Input("x: float32").Input("gamma: float32").Input("beta: float32").Input("dy: float32")
    .Output("dx: float32").Output("dgamma: float32").Output("dbeta: float32")
    .Attr("inverse: bool = false").Attr("rectify: bool = false").Attr("alpha: float = 1.0").Attr("epsilon: float = 1.0")
    .SetShapeFn([](tf::shape_inference::InferenceContext* c) {
      c->set_output(0, c->input(0));
      c->set_output(1, c->input(1));
      c->set_output(2, c->input(2));
      return tf::OkStatus();
    });

class GdnOpBase : public tf::OpKernel {
 public:
  explicit GdnOpBase(tf::OpKernelConstruction* c) : tf::OpKernel(c) {
    bool inverse, rectify;
    OP_REQUIRES_OK(c, c->GetAttr("inverse", &inverse));
    OP_REQUIRES_OK(c, c->GetAttr("rectify", &rectify));
    OP_REQUIRES_OK(c, c->GetAttr("alpha", &alpha_));
    OP_REQUIRES_OK(c, c->GetAttr("epsilon", &epsilon_));
    flags_ = (inverse ? TFCB_GDN_INVERSE : 0) | (rectify ? TFCB_GDN_RECTIFY : 0);
  }
 protected:
  int flags_;
  float alpha_, epsilon_;
};
class GdnForwardGpuOp : public GdnOpBase {
 public:
  using GdnOpBase::GdnOpBase;
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& x = ctx->input(0);
    OP_REQUIRES(ctx, x.dims() >= 2, InvalidArgument("Input tensor must have at least rank 2."));
    const int C = static_cast<int>(x.dim_size(x.dims() - 1));
    tf::Tensor* y;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, x.shape(), &y));
    OP_REQUIRES_OK(ctx, FromRc(tfcb_gdn_forward(x.flat<float>().data(), ctx->input(1).flat<float>().data(),
                                               ctx->input(2).flat<float>().data(), y->flat<float>().data(),
                                               x.NumElements() / C, C, flags_, alpha_, epsilon_, CudaStream(ctx))));
  }
};
class GdnBackwardGpuOp : public GdnOpBase {
 public:
  using GdnOpBase::GdnOpBase;
  void Compute(tf::OpKernelContext* ctx) override {
    const tf::Tensor& x = ctx->input(0);
    const int C = static_cast<int>(x.dim_size(x.dims() - 1));
    const int64_t n_pix = x.NumElements() / C;
    tf::Tensor *dx, *dgamma, *dbeta, ws;
    OP_REQUIRES_OK(ctx, ctx->allocate_output(0, x.shape(), &dx));
    OP_REQUIRES_OK(ctx, ctx->allocate_output(1, ctx->input(1).shape(), &dgamma));
    OP_REQUIRES_OK(ctx, ctx->allocate_output(2, ctx->input(2).shape(), &dbeta));
    OP_REQUIRES_OK(ctx, ctx->allocate_temp(tf::DT_UINT8, tf::TensorShape({tfcb_gdn_backward_workspace_bytes(n_pix, C)}), &ws));
    OP_REQUIRES_OK(ctx, FromRc(tfcb_gdn_backward(x.flat<float>().data(), ctx->input(1).flat<float>().data(),
                                                ctx->input(2).flat<float>().data(), ctx->input(3).flat<float>().data(),
                                                dx->flat<float>().data(), dgamma->flat<float>().data(),
                                                dbeta->flat<float>().data(), ws.flat<uint8_t>().data(), n_pix, C, flags_,
                                                alpha_, epsilon_, CudaStream(ctx))));
  }
};
REGISTER_KERNEL_BUILDER(Name("GdnForward").Device(tf::DEVICE_GPU), GdnForwardGpuOp);
REGISTER_KERNEL_BUILDER(Name("GdnBackward").Device(tf::DEVICE_GPU), GdnBackwardGpuOp);

}  // namespace
}  // namespace tfcb200_tf
