/* tfcb200.h -- C ABI of libtfcb200.so: the H100-native (sm_90a) replacement for the data-parallel hot path of
 * tensorflow/compression (range coder ops, PmfToQuantizedCdf, GDN/IGDN forward + backward).
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / TF types.  Every entry point
 * names the reference interface it replaces (paths relative to /root/reference).
 *
 * Conventions
 *   - `_dev` pointers are CUDA device pointers on the current device, `_host` pointers are host memory.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Calls are
 *     asynchronous on that stream unless stated otherwise.
 *   - Return value: TFCB_OK (0), TFCB_INVALID_ARGUMENT (1; the analogue of TF's InvalidArgument
 *     status), TFCB_CUDA_ERROR (2), TFCB_OUT_OF_MEMORY (3).  A message is available through
 *     tfcb_last_error() (thread local).
 *   - Handles are not thread safe; one consumer per handle, as the reference documents for its
 *     DT_VARIANT handles (tensorflow_compression/cc/ops/range_coder_ops.cc:94-95,190-192).
 *   - There is NO CPU fallback: without a CUDA device every compute entry returns TFCB_CUDA_ERROR.
 */
#ifndef TFCB200_H_
#define TFCB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFCB_OK 0
#define TFCB_INVALID_ARGUMENT 1
#define TFCB_CUDA_ERROR 2
#define TFCB_OUT_OF_MEMORY 3

#define TFCB_ABI_VERSION 2

/* Version of this ABI (TFCB_ABI_VERSION of the library that was loaded). */
int tfcb_abi_version(void);
/* Message of the last failing call on this thread ("" if none). */
const char* tfcb_last_error(void);

/* ------------------------------------------------------------------------------------------------
 * Range ENCODER.  Replaces CreateRangeEncoder / EntropyEncodeChannel / EntropyEncodeIndex /
 * EntropyEncodeFinalize:
 *   op contract   tensorflow_compression/cc/ops/range_coder_ops.cc:28-135
 *   CPU kernels   tensorflow_compression/cc/kernels/range_coder_kernels.cc:168-322,484-592
 *   coder         tensorflow_compression/cc/lib/range_coder.cc:37-307
 * One CTA per code stream (gather / chain / drain warps); streams = prod(handle shape); a stream holds < 2^31
 * 16-bit words (4 GB).
 * ---------------------------------------------------------------------------------------------- */
typedef struct tfcb_encoder tfcb_encoder;

/* `lookup_host`: the reference's `lookup` tensor, int32, either 1-D (lookup_cols == 0: rows
 * concatenated, each [+-precision, 0, c1, ..., 2^precision, (2^precision padding)*]) or 2-D
 * (lookup_cols == row width).  Negative precision enables the overflow (escape + Elias gamma)
 * code for that row.  Validated like ScanCDF / IndexCDFVector / IndexCDFMatrix
 * (range_coder_kernels.cc:110-164); violations -> TFCB_INVALID_ARGUMENT. */
int tfcb_encoder_create(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols,
                        int64_t n_streams, void* stream, tfcb_encoder** out);

/* EntropyEncodeChannel: `value_dev` is int32 [n_streams, n_per_stream] row-major; symbol j of every
 * stream uses lookup row (j mod n_rows), restarting at 0 for each call (range_coder_kernels.cc:
 * 244-267).  May be called repeatedly; the streams keep growing (state persists, :225-226). */
int tfcb_encode_channel(tfcb_encoder* h, const int32_t* value_dev, int64_t n_per_stream, void* stream);

/* EntropyEncodeIndex: `index_dev` has the shape of `value_dev`; row = index (range_coder_kernels.cc:
 * 219-242).  Out-of-range index / value are reported by tfcb_encode_finalize / tfcb_encoder_check as
 * TFCB_INVALID_ARGUMENT ("index=... not in range", "value=... not in range"), mirroring
 * REQUIRE_IN_RANGE (:204-210,231,235,260). */
int tfcb_encode_index(tfcb_encoder* h, const int32_t* index_dev, const int32_t* value_dev,
                      int64_t n_per_stream, void* stream);

/* Fused quantize + EntropyEncodeChannel: the symbol is
 *   int32(rintf(y - quant_offset[c])) - cdf_offset[c],   c = j mod n_rows
 * i.e. ContinuousBatchedEntropyModel.compress without materialising the int32 tensor
 * (tensorflow_compression/python/entropy_models/continuous_batched.py:375-382).
 * `quant_offset_dev` may be NULL (no offset). */
int tfcb_encode_channel_f32(tfcb_encoder* h, const float* y_dev, const float* quant_offset_dev,
                            const int32_t* cdf_offset_dev, int64_t n_per_stream, void* stream);

/* Fused quantize + EntropyEncodeIndex: symbol = int32(rintf(y - loc)) - cdf_offset[index]
 * (continuous_indexed.py:378-385; `loc_dev` may be NULL).  `index_dev` are already-clamped int32
 * table indexes. */
int tfcb_encode_index_f32(tfcb_encoder* h, const int32_t* index_dev, const float* y_dev,
                          const float* loc_dev, const int32_t* cdf_offset_dev, int64_t n_per_stream,
                          void* stream);

/* Synchronises `stream` and reports a pending device-side argument error, if any. */
int tfcb_encoder_check(tfcb_encoder* h, void* stream);

/* EntropyEncodeFinalize in two calls, into caller-owned device memory.  tfcb_encode_finalize flushes every
 * stream exactly like RangeEncoder::Finalize (range_coder.cc:266-307), writes where each string starts in the
 * packed output to `offsets_dev` int64 [n_streams + 1], synchronises `stream` once, reports deferred argument
 * errors (again on a retry) and returns the total size.  tfcb_encode_write then packs all strings back to back
 * into `bytes_dev` [total] (asynchronous; once, after a successful finalize).  After the write only destroy is
 * valid. */
int tfcb_encode_finalize(tfcb_encoder* h, int64_t* offsets_dev, void* stream, int64_t* total_bytes_host);
int tfcb_encode_write(tfcb_encoder* h, const int64_t* offsets_dev, uint8_t* bytes_dev, void* stream);
void tfcb_encoder_destroy(tfcb_encoder* h);

/* One whole compress() in two calls: create + one encode + finalize, with the result written into
 * caller-owned device memory.  tfcb_compress encodes `n_per_stream` symbols of every stream (channel mode when
 * `index_dev` is NULL, else index mode; `value_dev` is int32, or float32 quantised as in the *_f32 calls when
 * `value_is_f32` is nonzero), writes the offsets int64 [n_streams + 1] to `offsets_dev`, synchronises `stream`
 * once, reports argument errors like tfcb_encode_finalize and returns the total size and an encoder that holds
 * the unpacked streams.  tfcb_compress_write packs them into `bytes_dev` [total] and takes the encoder back;
 * the caller must not use it afterwards (tfcb_encoder_destroy releases one that is never written).
 * The library keeps such encoders, with their device buffers, between calls and reuses them in stream
 * order. */
int tfcb_compress(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                  const int32_t* index_dev, const void* value_dev, int32_t value_is_f32,
                  const float* quant_offset_dev, const int32_t* cdf_offset_dev, int64_t n_per_stream,
                  int64_t* offsets_dev, void* stream, tfcb_encoder** out, int64_t* total_bytes_host);
int tfcb_compress_write(tfcb_encoder* h, const int64_t* offsets_dev, uint8_t* bytes_dev, void* stream);

/* Ragged batch: one compress() over n_streams streams of different lengths (e.g. the latents of differently sized
 * images): stream s is symbols [symbol_offsets_host[s], symbol_offsets_host[s+1]) of value_dev (and of index_dev /
 * quant_offset_dev in index mode; in channel mode its rows restart at 0).  Otherwise exactly tfcb_compress: writes
 * offsets_dev [n_streams + 1], synchronises once, returns the total size and an encoder that tfcb_compress_write
 * packs and takes back.  String s is byte-identical to what tfcb_compress makes of stream s alone; a stream with
 * no symbols gives the empty string.  The offsets are host memory and are checked before any device work
 * (TFCB_INVALID_ARGUMENT): n_streams > 0, symbol_offsets_host[0] == 0, non-decreasing, every stream within the
 * per-stream limit.  The word arena is the sum of the streams' own worst cases. */
int tfcb_compress_ragged(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                         const int64_t* symbol_offsets_host, const int32_t* index_dev, const void* value_dev,
                         int32_t value_is_f32, const float* quant_offset_dev, const int32_t* cdf_offset_dev,
                         int64_t* offsets_dev, void* stream, tfcb_encoder** out, int64_t* total_bytes_host);
/* tfcb_compress_ragged that also hands back what decoding the strings would give, without decoding them: on success
 * `decoded_dev` (float32, one per symbol over all streams, symbol_offsets_host[n_streams] in all) holds exactly
 * what tfcb_decode_ragged(..., out_is_f32 = 1, the same quant_offset_dev and cdf_offset_dev) returns for these
 * strings, bit for bit: float(symbol + cdf_offset[row]) + quant_offset (or loc), with the integer the encoder
 * codes (so |y - loc| >= 2^31 saturates and NaN gives 0, as in the decoder).  An encoder that needs the decoded
 * values to condition what it codes next (channel-conditional models) saves a decode per step.  Offsets, the one
 * synchronisation, the returned encoder and the error messages are tfcb_compress_ragged's.  Checked before any
 * device work (TFCB_INVALID_ARGUMENT): `value_is_f32` nonzero, `decoded_dev` and `cdf_offset_dev` non-null. */
int tfcb_compress_ragged_decoded(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols,
                                 int64_t n_streams, const int64_t* symbol_offsets_host, const int32_t* index_dev,
                                 const void* value_dev, int32_t value_is_f32, const float* quant_offset_dev,
                                 const int32_t* cdf_offset_dev, int64_t* offsets_dev, void* stream,
                                 tfcb_encoder** out, int64_t* total_bytes_host, float* decoded_dev);
/* float16 / bfloat16 values (`dtype` 1 / 2), quantised in the encoder with the arithmetic of the entropy models'
 * unfused 16-bit path, so the strings are those of tfcb_compress on the int32 symbols that path computes:
 *   channel mode (index_dev NULL): int(rint(float(value) - loc[row])) - cdf_offset[row], `loc_dev` NULL or float32
 *     [rows] (the quantisation offsets; `loc_dtype` 0);
 *   index mode: `loc_dev` NULL, or shaped like the value in float32 (`loc_dtype` 0: the difference is taken in
 *     float32) or in the value's type (`loc_dtype` == dtype: the difference is rounded to that type first).
 * float -> int32 saturates and NaN gives 0, as in the *_f32 calls.  Otherwise exactly tfcb_compress (checks, offsets,
 * one synchronisation, the encoder tfcb_compress_write packs).  Checked before any device work
 * (TFCB_INVALID_ARGUMENT): `dtype` 1 or 2, `loc_dtype` 0 or (index mode) `dtype`, `cdf_offset_dev` non-null, and
 * `value_dev` non-null whenever there are symbols. */
int tfcb_compress_16bit(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                        const int32_t* index_dev, const void* value_dev, int dtype, const void* loc_dev, int loc_dtype,
                        const int32_t* cdf_offset_dev, int64_t n_per_stream, int64_t* offsets_dev, void* stream,
                        tfcb_encoder** out, int64_t* total_bytes_host);
/* tfcb_compress_16bit over a ragged batch, laid out and checked like tfcb_compress_ragged.  `decoded_dev` non-null:
 * the encoder also writes, per symbol, exactly what tfcb_decode_ragged_16bit with the same dtype, loc and cdf_offset
 * returns for these strings (as tfcb_compress_ragged_decoded does for float32): in the value's type, or float32 in
 * index mode with a float32 loc. */
int tfcb_compress_ragged_16bit(const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols, int64_t n_streams,
                               const int64_t* symbol_offsets_host, const int32_t* index_dev, const void* value_dev,
                               int dtype, const void* loc_dev, int loc_dtype, const int32_t* cdf_offset_dev,
                               void* decoded_dev, int64_t* offsets_dev, void* stream, tfcb_encoder** out,
                               int64_t* total_bytes_host);

/* ------------------------------------------------------------------------------------------------
 * Range DECODER.  Replaces CreateRangeDecoder / EntropyDecodeChannel / EntropyDecodeIndex /
 * EntropyDecodeFinalize:
 *   op contract   tensorflow_compression/cc/ops/range_coder_ops.cc:137-247
 *   CPU kernels   tensorflow_compression/cc/kernels/range_coder_kernels.cc:334-471,597-700
 *   coder         tensorflow_compression/cc/lib/range_coder.h:79-83,144-169,193-282
 * ---------------------------------------------------------------------------------------------- */
typedef struct tfcb_decoder tfcb_decoder;

/* `bytes_dev` / `offsets_dev` (int64 [n_streams + 1]) describe the encoded strings; the memory is
 * BORROWED and must outlive the handle (the reference also only holds a reference,
 * range_coder_kernels.cc:475-478). */
int tfcb_decoder_create(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_streams,
                        const int32_t* lookup_host, int64_t lookup_len, int64_t lookup_cols,
                        void* stream, tfcb_decoder** out);
/* EntropyDecodeChannel -> int32 [n_streams, n_per_stream]. */
int tfcb_decode_channel(tfcb_decoder* h, int32_t* out_dev, int64_t n_per_stream, void* stream);
/* EntropyDecodeIndex. */
int tfcb_decode_index(tfcb_decoder* h, const int32_t* index_dev, int32_t* out_dev,
                      int64_t n_per_stream, void* stream);
/* Fused decode + dequantize: out = float(sym + cdf_offset[c]) + quant_offset[c]
 * (continuous_batched.py:416-421); `quant_offset_dev` may be NULL. */
int tfcb_decode_channel_f32(tfcb_decoder* h, float* out_dev, const float* quant_offset_dev,
                            const int32_t* cdf_offset_dev, int64_t n_per_stream, void* stream);
/* Fused decode + dequantize, index mode: out = float(sym + cdf_offset[index]) + loc
 * (continuous_indexed.py:409-416); `loc_dev` may be NULL. */
int tfcb_decode_index_f32(tfcb_decoder* h, const int32_t* index_dev, float* out_dev,
                          const float* loc_dev, const int32_t* cdf_offset_dev, int64_t n_per_stream,
                          void* stream);
/* Ragged batch: decodes symbol_offsets_host[s+1] - symbol_offsets_host[s] more symbols of stream s into out_dev
 * at symbol_offsets_host[s], int32 (out_is_f32 == 0) or dequantised float as tfcb_decode_{channel,index}_f32;
 * index_dev NULL = channel mode (rows restart at 0 in every stream).  The offsets ([n_streams + 1], host memory)
 * are checked like tfcb_compress_ragged's.  State persists like the other decode calls; tfcb_decode_finalize
 * reports. */
int tfcb_decode_ragged(tfcb_decoder* h, const int64_t* symbol_offsets_host, const int32_t* index_dev, void* out_dev,
                       int32_t out_is_f32, const float* quant_offset_dev, const int32_t* cdf_offset_dev, void* stream);
/* Fused decode + dequantise of float16 / bfloat16 values (`dtype` 1 / 2; `index_dev` NULL: channel mode), the
 * inverse of tfcb_compress_16bit with the same loc operand and the arithmetic of the entropy models' unfused path:
 * h = to16(float(sym + cdf_offset[row])) (int32 -> float -> 16 bits, two roundings), then
 *   channel mode: out = to16(float(h) + float(to16(loc[row]))) (loc float32 [rows] or NULL: out = h);
 *   index mode, loc in the value's type (or NULL): out = to16(float(h) + float(loc));
 *   index mode, float32 loc: out = float(h) + loc, written as FLOAT32.
 * `out_dev` holds n_streams * n_per_stream outputs of that type.  Checked before any device work like
 * tfcb_compress_16bit (`out_dev` in place of `value_dev`). */
int tfcb_decode_16bit(tfcb_decoder* h, const int32_t* index_dev, void* out_dev, int dtype, const void* loc_dev,
                      int loc_dtype, const int32_t* cdf_offset_dev, int64_t n_per_stream, void* stream);
/* tfcb_decode_16bit over a ragged batch, with tfcb_decode_ragged's offsets and layout. */
int tfcb_decode_ragged_16bit(tfcb_decoder* h, const int64_t* symbol_offsets_host, const int32_t* index_dev,
                             void* out_dev, int dtype, const void* loc_dev, int loc_dtype,
                             const int32_t* cdf_offset_dev, void* stream);
/* EntropyDecodeFinalize: ok_host[s] = RangeDecoder::Finalize() of stream s (range_coder.h:144-169).
 * Synchronises; also reports a pending out-of-range index as TFCB_INVALID_ARGUMENT. */
int tfcb_decode_finalize(tfcb_decoder* h, uint8_t* ok_host, void* stream);
void tfcb_decoder_destroy(tfcb_decoder* h);

/* ------------------------------------------------------------------------------------------------
 * Joint autoregressive + hierarchical prior (Minnen, Ballé & Toderici 2018): the entropy parameters of a latent
 * position from its 12 causal neighbours (5x5 type-A mask) and the hyper feature psi, and the serial encoder /
 * decoder over positions.  M = latent depth, a multiple of 6 in [6, 384]; latents are channels-last float32
 * [B, H, W, M], psi [B, H, W, 2M]; positions p = y * W + x run in raster order.  Per position and image:
 *   ctx = Wc * taps + bc (2M); h1 = leaky(W1 * [psi_p, ctx] + b1) (10M/3); h2 = leaky(W2 * h1 + b2) (8M/3);
 *   [loc, scale_index] = W3 * h2 + b3 (M each); index = int32(min(max(scale_index, 0), num_scales - 1)),
 * leaky(x) = x > 0 ? x : 0.01 x.  Each output is one fixed sequence of float32 operations that depends only on
 * that image's inputs: results do not depend on B, an image's place in the batch, or the device's SM count.
 * Every call checks M, the packed size, shapes, the position range and null pointers before any device work.
 * ---------------------------------------------------------------------------------------------- */
/* Floats of the packed parameter buffer for latent depth M, or -1 if M is not supported. */
int64_t tfcb_ar_packed_floats(int M);
/* Packs the parameters into `packed_dev` (tfcb_ar_packed_floats(M) floats), stream-ordered device copies of the
 * values unchanged: the context kernel [5, 5, M, 2M] (its first 12 taps in raster order are the causal ones), its
 * bias [2M], then W1 [4M, 10M/3], b1, W2 [10M/3, 8M/3], b2, W3 [8M/3, 2M], b3 (inputs x outputs, row major). */
int tfcb_ar_pack_weights(int M, const float* ctx_kernel_dev, const float* ctx_bias_dev, const float* w1_dev,
                         const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                         const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream);
/* Parameter step: loc, scale_index and the table index [B, M] of position p for every image, from the decoded
 * latents `yhat_dev` at earlier positions (later positions are not read).  Each output may be NULL.  One launch. */
int tfcb_ar_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int64_t p, int num_scales, float* loc_dev, float* scale_index_dev,
                   int32_t* index_dev, void* stream);
/* Encoder steps p_begin <= p < p_end: per position the parameter step, then yhat = float(int32(rint(y - loc))) +
 * loc, the value tfcb_decode_index_f32 returns for the symbol an index-mode encode with this loc codes.  Writes
 * yhat, loc and index [B, H, W, M] (and scale_index, if not NULL) at those positions; yhat must hold the earlier
 * positions.  The strings are made afterwards by one index-mode encode (tfcb_compress) of y with index and loc.
 * One launch, no host synchronisation. */
int tfcb_ar_encode(const float* packed_dev, int64_t packed_floats, int M, const float* y_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int64_t p_begin, int64_t p_end, int num_scales, float* yhat_dev,
                   float* loc_dev, int32_t* index_dev, float* scale_index_dev, void* stream);
/* Decoder steps p_begin <= p < p_end: per position the parameter step, then the M symbols of each of the B streams
 * of `h` (which must hold B strings, made with index-mode tables of at least num_scales rows) are decoded from the
 * handle's state and dequantised like tfcb_decode_index_f32: yhat[b, p, c] = float(sym + cdf_offset[index]) + loc.
 * The handle's state advances as with the other decode calls, so steps may be mixed with them and
 * tfcb_decode_finalize reports each stream.  One launch, no host synchronisation. */
int tfcb_ar_decode(tfcb_decoder* h, const float* packed_dev, int64_t packed_floats, int M, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int64_t p_begin, int64_t p_end, int num_scales,
                   const int32_t* cdf_offset_dev, float* yhat_dev, void* stream);
/* Ragged lists: n_images > 0 images of latent shapes heights_host[i] x widths_host[i] (host arrays; every side
 * positive, H W <= 2^31 - 1).  Latents, yhat, loc, index and scale_index are flat: image i's [H_i, W_i, M] starts at
 * element M P_i with P_i = sum_{j<i} H_j W_j, psi likewise with 2M channels.  Each image's outputs equal the
 * fixed-shape call on that image alone, bit for bit.  The entries keep a table of the images in `work_dev`, uploaded
 * with one stream-ordered copy; there is no host synchronisation. */
/* Floats of workspace a ragged call over n_images images needs, or -1 if n_images is not positive. */
int64_t tfcb_ar_ragged_workspace_floats(int64_t n_images);
/* tfcb_ar_encode over every position of every image of the list, one CTA per image.  One launch. */
int tfcb_ar_encode_ragged(const float* packed_dev, int64_t packed_floats, int M, const float* y_dev,
                          const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                          const int64_t* widths_host, int num_scales, float* work_dev, int64_t work_floats,
                          float* yhat_dev, float* loc_dev, int32_t* index_dev, float* scale_index_dev, void* stream);
/* tfcb_ar_decode over every position of every image of the list: image i continues stream i of `h`, which must hold
 * n_images strings.  One launch. */
int tfcb_ar_decode_ragged(tfcb_decoder* h, const float* packed_dev, int64_t packed_floats, int M, const float* psi_dev,
                          int64_t n_images, const int64_t* heights_host, const int64_t* widths_host, int num_scales,
                          const int32_t* cdf_offset_dev, float* work_dev, int64_t work_floats, float* yhat_dev,
                          void* stream);
/* Column tiles (DESIGN §3.15): image i's latents coded as 1 <= tiles = T <= 1024 independent streams, decoded and
 * encoded as a wavefront over many CTAs.  Tile t of an image of width W holds columns [floor(t W / T),
 * floor((t + 1) W / T)) of every row (no columns when T > W); its stream is the tile's rows in order, M symbols per
 * position in channel order: tfcb_substream_layout with S = T and one phase per latent row of W positions of width M.
 * A work item is one row of one non-empty tile.  Item (i, r, u), u the tile's rank among the row's non-empty tiles,
 * waits for (i, r, u - 1) and for (i, r - 1, u_R), u_R the tile holding column min(W - 1, c_last + 2); the items run
 * in ticket order, sorted by (2 r + u, r, i), on a persistent grid (no co-residency is assumed).  ŷ, loc and index
 * equal tfcb_ar_encode_ragged's / tfcb_ar_decode_ragged's bit for bit.  Every wait is bounded (10 s) and polls an
 * abort word; an aborted encode sets the index of every position it skipped to -1 (which the range encode rejects),
 * an aborted decode leaves each failed tile's stream in a state tfcb_decode_finalize reports as not OK.  Per call:
 * one table upload, one reset of the counters, one launch; no host synchronisation. */
/* Floats of workspace a tiles call needs (image table, item table, progress counters and schedule words), or -1 if
 * the list or `tiles` is not supported.  The workspace must be 8-byte aligned. */
int64_t tfcb_ar_tiles_workspace_floats(int64_t n_images, const int64_t* heights_host, const int64_t* widths_host,
                                       int64_t tiles);
/* The ticket order on the host, no device work: *n_items_host receives the number of items and, if `items_host` is
 * not NULL, items_host [n_items][5] the items in ticket order as (image, row, tile t, first column, end column). */
int tfcb_ar_tiles_schedule(int64_t n_images, const int64_t* heights_host, const int64_t* widths_host, int64_t tiles,
                           int64_t* n_items_host, int64_t* items_host);
/* tfcb_ar_encode_ragged over column tiles: the same outputs in the same raster layout. */
int tfcb_ar_encode_tiles(const float* packed_dev, int64_t packed_floats, int M, const float* y_dev,
                         const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                         const int64_t* widths_host, int64_t tiles, int num_scales, float* work_dev,
                         int64_t work_floats, float* yhat_dev, float* loc_dev, int32_t* index_dev,
                         float* scale_index_dev, void* stream);
/* tfcb_ar_decode_ragged over column tiles: tile t of image i continues stream i T + t of `h`, which must hold
 * n_images T strings. */
int tfcb_ar_decode_tiles(tfcb_decoder* h, const float* packed_dev, int64_t packed_floats, int M, const float* psi_dev,
                         int64_t n_images, const int64_t* heights_host, const int64_t* widths_host, int64_t tiles,
                         int num_scales, const int32_t* cdf_offset_dev, float* work_dev, int64_t work_floats,
                         float* yhat_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Checkerboard context model (He et al. 2021) on the same packed parameters.  A latent position (r, c) is an
 * anchor when r + c is even, else a non-anchor; an image has ceil(H W / 2) anchors.  Coding order: the anchors in
 * raster order, then the non-anchors in raster order, M channels per position.  Anchors take ctx = 0 (bias
 * included); a non-anchor takes ctx = Wc * taps + bc over the 12 taps (dy, dx) in [-2, 2]^2 with dy + dx odd, in
 * raster order, zeros outside the image.  The packed Wc is those 12 taps [12, M, 2M]: pack them with
 * tfcb_ar_pack_weights, which reads the first 12 M 2M floats of its context-kernel operand.  The rest of the
 * network and its float32 order of operations are tfcb_ar_params'.
 * ---------------------------------------------------------------------------------------------- */
/* Floats of workspace one tfcb_cb_params pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_cb_workspace_floats(int M, int64_t B, int64_t H, int64_t W, int anchors);
/* One pass over every position of one colour (anchors != 0: the anchors) of all B images.  The non-anchor pass
 * reads the anchors' decoded latents from `yhat_dev` [B, H, W, M] (NULL is allowed for the anchor pass).  Writes
 * loc, scale_index and the table index (each may be NULL) in coding order: [B, n, M] with n the positions of this
 * colour per image (whole == 0), or [B, H W, M] at this pass's rows (whole != 0).  Encoder epilogue (y_dev not
 * NULL, [B, H, W, M]): also writes y in coding order to `y_cb_dev` (same layout as loc) and yhat = float(int32(rint(
 * y - loc))) + loc at this colour's positions of `yhat_out_dev` [B, H, W, M]; loc and index are then required.
 * Three launches for the anchors, four for the non-anchors, none for an empty pass; no host synchronisation. */
int tfcb_cb_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                   int64_t B, int64_t H, int64_t W, int anchors, int num_scales, float* work_dev,
                   int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev,
                   const float* y_dev, float* y_cb_dev, float* yhat_out_dev, void* stream);
/* Moves one colour's latents from coding order [B, n, M] to their positions of `dst_dev` [B, H, W, M] (the
 * other colour's positions are not written).  One launch; none when the colour has no positions. */
int tfcb_cb_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int anchors, float* dst_dev,
                    void* stream);

/* ------------------------------------------------------------------------------------------------
 * Space-channel context model (He et al. 2022): the checkerboard passes per channel group.  M = latent depth, even,
 * at most 1024; a group is the C >= 1 channels [offset, offset + C) of y, with offset + C <= M.  Per position of a
 * group, with CH = 0 for the group at offset 0 and CH = 2C otherwise:
 *   ctx = 0 at an anchor, else Wc * (the group's channels of yhat at the 12 checkerboard taps) + bc   [12C] -> [2C]
 *   h1 = leaky(W1 * [psi (2M), chctx (CH), ctx (2C)] + b1)                         [K1 = 2M + CH + 2C] -> [5 K1 / 6]
 *   h2 = leaky(W2 * h1 + b2) -> [2 K1 / 3];  [loc, scale_index] = W3 * h2 + b3 (C each)
 * (widths rounded down) in tfcb_ar_params' float32 order of operations; chctx [B, H, W, CH] is the caller's channel
 * context.  At offset 0 with C = M (M a multiple of 6) this is tfcb_cb_params, bit for bit, on the same packed
 * layout.  Coding order of all groups: per image, group 0's anchors, group 0's non-anchors, group 1's anchors, ...,
 * each in raster order with C channels per position: [B, H W M] in all.
 * ---------------------------------------------------------------------------------------------- */
/* Floats of one group's packed parameters, or -1 if the group is not supported.  If `layout` is not NULL it receives
 * 11 values: the widths K1, N3, N4, then the offsets of Wc [12, C, 2C], bc [2C], W1 [K1, N3], b1, W2 [N3, N4], b2,
 * W3 [N4, 2C] and b3 (inputs x outputs, row major); the buffer ends at the returned size. */
int64_t tfcb_scc_packed_floats(int M, int offset, int C, int64_t* layout);
/* Packs one group's parameters into `packed_dev`, stream-ordered device copies of the values unchanged, the
 * context taps already gathered as [12, C, 2C] in raster order of the taps. */
int tfcb_scc_pack_weights(int M, int offset, int C, const float* ctx_taps_dev, const float* ctx_bias_dev,
                          const float* w1_dev, const float* b1_dev, const float* w2_dev, const float* b2_dev,
                          const float* w3_dev, const float* b3_dev, float* packed_dev, int64_t packed_floats,
                          void* stream);
/* Floats of workspace one tfcb_scc_params pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_scc_workspace_floats(int M, int offset, int C, int64_t B, int64_t H, int64_t W, int anchors);
/* One pass over every position of one colour of one group of all B images; tfcb_cb_params' arguments, plus the
 * group and `chctx_dev` [B, H, W, 2C] (required unless offset is 0).  The non-anchor pass reads the group's
 * channels of the anchors of `yhat_dev` [B, H, W, M].  Writes loc, scale_index and the table index (each may be
 * NULL): [B, n, C] with n the positions of this colour (whole == 0), or [B, H W M] in the coding order of all groups
 * at this pass's block (whole != 0).  Encoder epilogue (y_dev not NULL, [B, H, W, M]): also writes the group's y in
 * coding order to `y_cb_dev` (same layout as loc) and yhat = float(int32(rint(y - loc))) + loc at this colour's
 * positions and the group's channels of `yhat_out_dev` [B, H, W, M]; loc and index are then required.  Three
 * launches for the anchors, four for the non-anchors, none for an empty pass; no host synchronisation. */
int tfcb_scc_params(const float* packed_dev, int64_t packed_floats, int M, int offset, int C, const float* yhat_dev,
                    const float* psi_dev, const float* chctx_dev, int64_t B, int64_t H, int64_t W, int anchors,
                    int num_scales, float* work_dev, int64_t work_floats, int whole, float* loc_dev,
                    float* scale_index_dev, int32_t* index_dev, const float* y_dev, float* y_cb_dev,
                    float* yhat_out_dev, void* stream);
/* Moves one colour of one group from coding order [B, n, C] to its positions and channels of `dst_dev`
 * [B, H, W, M] (nothing else is written).  One launch; none when the colour has no positions. */
int tfcb_scc_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int offset, int C, int anchors,
                     float* dst_dev, void* stream);
/* Ragged lists (the layout of tfcb_ar_encode_ragged): psi, chctx (2C channels), y and yhat are flat, image i's
 * starting at P_i times their channel count.  With n_k,i the positions of this colour of image i and
 * Q_i = sum_{j<i} n_k,j, a pass writes image i's n_k,i C values at C Q_i (whole == 0), or its block of the coding
 * order of all groups at M P_i + H_i W_i offset + (anchors ? 0 : n_a,i C) (whole != 0), whose streams are the images'
 * H_i W_i M values.  Each image's outputs equal the fixed-shape call on that image alone, bit for bit; a tile of
 * positions may span several images.  The checkerboard model is the group (0, M).  The table of the images goes to
 * `work_dev` with one stream-ordered copy; there is no host synchronisation. */
/* Floats of workspace one tfcb_scc_params_ragged pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_scc_ragged_workspace_floats(int M, int offset, int C, int64_t n_images, const int64_t* heights_host,
                                         const int64_t* widths_host, int anchors);
/* tfcb_scc_params over a ragged list of images in place of B, H, W.  Three launches for the anchors, four for the
 * non-anchors, none when no image has a position of this colour. */
int tfcb_scc_params_ragged(const float* packed_dev, int64_t packed_floats, int M, int offset, int C,
                           const float* yhat_dev, const float* psi_dev, const float* chctx_dev, int64_t n_images,
                           const int64_t* heights_host, const int64_t* widths_host, int anchors, int num_scales,
                           float* work_dev, int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev,
                           int32_t* index_dev, const float* y_dev, float* y_cb_dev, float* yhat_out_dev,
                           void* stream);
/* tfcb_scc_scatter of a ragged list: image i's n_k,i C values at C Q_i -> its positions and the group's channels of
 * its [H_i, W_i, M] in `dst_dev`.  `work_dev` holds at least 8 n_images floats (the workspace of a pass of the list
 * does).  One launch; none when no image has a position of this colour. */
int tfcb_scc_scatter_ragged(const float* src_dev, int64_t n_images, const int64_t* heights_host,
                            const int64_t* widths_host, int M, int offset, int C, int anchors, float* work_dev,
                            int64_t work_floats, float* dst_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Multistage context model (Lin et al. 2023): four position-parallel stages of a 2x2 schedule.  M = latent depth, a
 * multiple of 6, at most 384.  Position (r, c) has phase (r mod 2, c mod 2) and stage (0,0) -> 0, (1,1) -> 1,
 * (0,1) -> 2, (1,0) -> 3.  Stage s with phase (a, b) has ceil((H - a) / 2) W_s positions, W_s = ceil((W - b) / 2), the
 * j-th at (a + 2 floor(j / W_s), b + 2 (j mod W_s)); a stage may be empty (H = 1 or W = 1).  Coding order: per image,
 * stage 0, 1, 2, 3, each in raster order with M channels per position: [B, H W M] in all.  Per position of stage s:
 *   ctx = 0 at stage 0 (bias included), else Wc_s * (yhat at the stage's T_s taps) + bc_s            [T_s M] -> [2M]
 * with the taps (dy, dx) in [-2, 2]^2 whose neighbour lies in an earlier stage, in raster order, zeros outside the
 * image: T_1 = 4 (dy, dx both odd), T_2 = 12 (dy + dx odd), T_3 = 16 (dy, dx not both even).  Then tfcb_ar_params'
 * network on [psi, ctx] (4M -> 10M/3 -> 8M/3 -> [loc, scale_index]), shared by the stages, in its float32 order of
 * operations; stage 0 is tfcb_cb_params' anchor pass bit for bit on the same shared network.
 * ---------------------------------------------------------------------------------------------- */
/* Floats of the packed parameters, or -1 if M is not supported: Wc_1 [4, M, 2M], bc_1 [2M], Wc_2 [12, M, 2M], bc_2,
 * Wc_3 [16, M, 2M], bc_3, W1 [4M, 10M/3], b1, W2 [10M/3, 8M/3], b2, W3 [8M/3, 2M], b3, back to back. */
int64_t tfcb_msc_packed_floats(int M);
/* Packs the parameters into `packed_dev`, stream-ordered device copies of the values unchanged; each stage's context
 * taps already gathered as [T_s, M, 2M] in raster order of its taps. */
int tfcb_msc_pack_weights(int M, const float* wc1_dev, const float* bc1_dev, const float* wc2_dev,
                          const float* bc2_dev, const float* wc3_dev, const float* bc3_dev, const float* w1_dev,
                          const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                          const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream);
/* Floats of workspace one tfcb_msc_params pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_msc_workspace_floats(int M, int64_t B, int64_t H, int64_t W, int stage);
/* One pass over every position of stage `stage` (0 to 3) of all B images.  Stages 1-3 read the earlier stages'
 * decoded latents from `yhat_dev` [B, H, W, M] (NULL is allowed for stage 0).  Writes loc, scale_index and the table
 * index (each may be NULL): [B, n_s, M] (whole == 0), or [B, H W M] in coding order at this stage's block
 * (whole != 0).  Encoder epilogue (y_dev not NULL, [B, H, W, M]): also writes y in coding order to `y_ms_dev` (same
 * layout as loc) and yhat = float(int32(rint(y - loc))) + loc at this stage's positions of `yhat_out_dev`
 * [B, H, W, M]; loc and index are then required.  Three launches at stage 0, four at stages 1-3, none for an empty
 * stage; no host synchronisation. */
int tfcb_msc_params(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev, const float* psi_dev,
                    int64_t B, int64_t H, int64_t W, int stage, int num_scales, float* work_dev, int64_t work_floats,
                    int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev, const float* y_dev,
                    float* y_ms_dev, float* yhat_out_dev, void* stream);
/* Moves one stage's latents from coding order [B, n_s, M] to their positions of `dst_dev` [B, H, W, M] (nothing
 * else is written).  One launch; none for an empty stage. */
int tfcb_msc_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int stage, float* dst_dev,
                     void* stream);
/* Ragged lists, in the layout of tfcb_scc_params_ragged: image i's n_s,i M values at M Q_i (whole == 0), or its
 * block of its coding order at M (P_i + its positions of the earlier stages) (whole != 0).  Each image's outputs
 * equal the fixed-shape call on that image alone, bit for bit.  The image table goes to `work_dev` with one
 * stream-ordered copy; there is no host synchronisation. */
int64_t tfcb_msc_ragged_workspace_floats(int M, int64_t n_images, const int64_t* heights_host,
                                         const int64_t* widths_host, int stage);
int tfcb_msc_params_ragged(const float* packed_dev, int64_t packed_floats, int M, const float* yhat_dev,
                           const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                           const int64_t* widths_host, int stage, int num_scales, float* work_dev,
                           int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev, int32_t* index_dev,
                           const float* y_dev, float* y_ms_dev, float* yhat_out_dev, void* stream);
/* tfcb_msc_scatter of a ragged list: image i's n_s,i M values at M Q_i -> its [H_i, W_i, M] in `dst_dev`.
 * `work_dev` holds at least 8 n_images floats (the workspace of a pass of the list does). */
int tfcb_msc_scatter_ragged(const float* src_dev, int64_t n_images, const int64_t* heights_host,
                            const int64_t* widths_host, int M, int stage, float* work_dev, int64_t work_floats,
                            float* dst_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Space-channel multistage context model (DESIGN §3.17): the space-channel model's channel groups, each coded in the
 * four stages of the multistage schedule.  M = latent depth, even, at most 1024; group [offset, offset + C) of it.
 * Per position of stage s of the group (CH = 0 at offset 0, else 2C):
 *   ctx = 0 at stage 0 (bias included), else Wc_s * (the group's channels of yhat at the stage's T_s taps) + bc_s
 *                                                                                                 [T_s C] -> [2C]
 *   h1 = leaky(W1 * [psi (2M), chctx (CH), ctx (2C)] + b1) -> [N3 = 5 K1 / 6], K1 = 2M + CH + 2C;
 *   h2 = leaky(W2 * h1 + b2) -> [N4 = 2 K1 / 3];  [loc, scale_index] = W3 * h2 + b3 (C each)
 * (widths rounded down) with tfcb_msc_params' stages, taps and float32 order of operations; chctx [B, H, W, CH] is
 * the caller's channel context.  At offset 0 with C = M (M a multiple of 6) this is tfcb_msc_params, bit for bit, on
 * the same packed layout; stage 0 is tfcb_scc_params' anchor pass of the group at its positions.  Coding order of
 * all groups: per image, group 0's stages 0, 1, 2, 3, then group 1's, ..., each stage in raster order with C channels
 * per position: [B, H W M] in all.
 * ---------------------------------------------------------------------------------------------- */
/* Floats of one group's packed parameters, or -1 if the group is not supported.  If `layout` is not NULL it receives
 * 15 values: the widths K1, N3, N4, then the offsets of Wc_1 [4, C, 2C], bc_1 [2C], Wc_2 [12, C, 2C], bc_2,
 * Wc_3 [16, C, 2C], bc_3, W1 [K1, N3], b1, W2 [N3, N4], b2, W3 [N4, 2C] and b3 (inputs x outputs, row major); the
 * buffer ends at the returned size. */
int64_t tfcb_mscc_packed_floats(int M, int offset, int C, int64_t* layout);
/* Packs one group's parameters into `packed_dev`, stream-ordered device copies of the values unchanged; each stage's
 * context taps already gathered as [T_s, C, 2C] in raster order of its taps. */
int tfcb_mscc_pack_weights(int M, int offset, int C, const float* wc1_dev, const float* bc1_dev, const float* wc2_dev,
                           const float* bc2_dev, const float* wc3_dev, const float* bc3_dev, const float* w1_dev,
                           const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                           const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream);
/* Floats of workspace one tfcb_mscc_params pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_mscc_workspace_floats(int M, int offset, int C, int64_t B, int64_t H, int64_t W, int stage);
/* One pass over every position of stage `stage` (0 to 3) of one group of all B images; tfcb_msc_params' arguments,
 * plus the group and `chctx_dev` [B, H, W, 2C] (required unless offset is 0).  Stages 1-3 read the group's channels
 * of the earlier stages' positions of `yhat_dev` [B, H, W, M].  Writes loc, scale_index and the table index (each may
 * be NULL): [B, n_s, C] (whole == 0), or [B, H W M] in the coding order of all groups at this pass's block
 * H W offset + C (the positions of the earlier stages) (whole != 0).  Encoder epilogue (y_dev not NULL,
 * [B, H, W, M]): also writes the group's y in coding order to `y_cc_dev` (same layout as loc) and
 * yhat = float(int32(rint(y - loc))) + loc at this stage's positions and the group's channels of `yhat_out_dev`
 * [B, H, W, M]; loc and index are then required.  Three launches at stage 0, four at stages 1-3, none for an empty
 * stage; no host synchronisation. */
int tfcb_mscc_params(const float* packed_dev, int64_t packed_floats, int M, int offset, int C, const float* yhat_dev,
                     const float* psi_dev, const float* chctx_dev, int64_t B, int64_t H, int64_t W, int stage,
                     int num_scales, float* work_dev, int64_t work_floats, int whole, float* loc_dev,
                     float* scale_index_dev, int32_t* index_dev, const float* y_dev, float* y_cc_dev,
                     float* yhat_out_dev, void* stream);
/* Moves one stage of one group from coding order [B, n_s, C] to its positions and channels of `dst_dev`
 * [B, H, W, M] (nothing else is written).  One launch; none for an empty stage. */
int tfcb_mscc_scatter(const float* src_dev, int64_t B, int64_t H, int64_t W, int M, int offset, int C, int stage,
                      float* dst_dev, void* stream);
/* Ragged lists, in the layout of tfcb_scc_params_ragged: image i's n_s,i C values at C Q_i (whole == 0), or its block
 * of the coding order of all groups at M P_i + H_i W_i offset + C (its positions of the earlier stages)
 * (whole != 0).  Each image's outputs equal the fixed-shape call on that image alone, bit for bit.  The image table
 * goes to `work_dev` with one stream-ordered copy; there is no host synchronisation. */
int64_t tfcb_mscc_ragged_workspace_floats(int M, int offset, int C, int64_t n_images, const int64_t* heights_host,
                                          const int64_t* widths_host, int stage);
int tfcb_mscc_params_ragged(const float* packed_dev, int64_t packed_floats, int M, int offset, int C,
                            const float* yhat_dev, const float* psi_dev, const float* chctx_dev, int64_t n_images,
                            const int64_t* heights_host, const int64_t* widths_host, int stage, int num_scales,
                            float* work_dev, int64_t work_floats, int whole, float* loc_dev, float* scale_index_dev,
                            int32_t* index_dev, const float* y_dev, float* y_cc_dev, float* yhat_out_dev,
                            void* stream);
/* tfcb_mscc_scatter of a ragged list: image i's n_s,i C values at C Q_i -> its positions and the group's channels of
 * its [H_i, W_i, M] in `dst_dev`.  `work_dev` holds at least 8 n_images floats (the workspace of a pass of the list
 * does).  One launch; none when no image has a position of this stage. */
int tfcb_mscc_scatter_ragged(const float* src_dev, int64_t n_images, const int64_t* heights_host,
                             const int64_t* widths_host, int M, int offset, int C, int stage, float* work_dev,
                             int64_t work_floats, float* dst_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Substreams (DESIGN §3.14): a coding unit (one string of today's format: one image's y or z, one MS2020 slice)
 * split into S independently decodable streams.  A unit's symbols are in coding order, in phases p = 0 .. P-1
 * (the order in which the decoder makes them); phase p of unit u has positions[u P + p] positions of
 * widths[u P + p] symbols each.  Substream s of unit u is the concatenation, over p in order, of the positions
 * [floor(s n / S), floor((s + 1) n / S)) of phase p (n = its positions), all symbols of each.  Streams are numbered
 * u S + s.  1 <= S <= 1024; positions >= 0; widths >= 1.
 * ------------------------------------------------------------------------------------------------ */
/* The layout on the host, no device work: `stream_offsets_host` [n_units S + 1] the symbol offsets of the streams
 * for tfcb_compress_ragged (substream order, unit after unit); `phase_lengths_host` [n_phases][n_units S] the
 * symbols of stream u S + s in phase p, for one tfcb_decode_ragged per phase (whose output is then phase p's
 * coding order, unit after unit).  Either output may be NULL. */
int tfcb_substream_layout(int64_t n_units, int64_t n_phases, const int64_t* positions_host,
                          const int64_t* widths_host, int64_t substreams, int64_t* stream_offsets_host,
                          int64_t* phase_lengths_host);
/* Bytes of workspace tfcb_substream_gather needs, or -1 if the arguments are not supported. */
int64_t tfcb_substream_gather_workspace_bytes(int64_t n_units, int64_t n_phases, int64_t substreams);
/* Rewrites units held back to back in coding order (unit u's symbols after unit u - 1's) into substream order:
 * up to three 4-byte operands (y and loc float32, index int32; a NULL input skips that operand, whose output must
 * then be NULL too, and at least one is given).  One launch (none when there are no symbols), no host
 * synchronisation; the segment table goes to `work_dev` (8-byte aligned) with one stream-ordered copy. */
int tfcb_substream_gather(int64_t n_units, int64_t n_phases, const int64_t* positions_host,
                          const int64_t* widths_host, int64_t substreams, const float* y_dev, const float* loc_dev,
                          const int32_t* index_dev, float* y_out_dev, float* loc_out_dev, int32_t* index_out_dev,
                          void* work_dev, int64_t work_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Legacy single-stream ops RangeEncode / RangeDecode (int16 data, broadcastable N-D int32 CDF):
 *   op contract   tensorflow_compression/cc/ops/range_coding_ops.cc:30-124
 *   CPU kernels   tensorflow_compression/cc/kernels/range_coding_kernels.cc:60-379
 *   axis merging  tensorflow_compression/cc/kernels/range_coding_kernels_util.cc:34-91
 * Shapes are host arrays; `cdf_rank` must be `rank + 1`.  `debug_level` 1 validates the CDF values
 * and the data range (range_coding_kernels.cc:150-173,249-253).  Both calls synchronise.
 * ---------------------------------------------------------------------------------------------- */
/* Writes at most `out_cap` bytes to `out_host`; *n_bytes_host receives the string length. */
int tfcb_range_encode(const int16_t* data_dev, const int64_t* data_shape_host, int rank,
                      const int32_t* cdf_dev, const int64_t* cdf_shape_host, int cdf_rank,
                      int precision, int debug_level, uint8_t* out_host, int64_t out_cap,
                      int64_t* n_bytes_host, void* stream);
int tfcb_range_decode(const uint8_t* encoded_host, int64_t n_bytes, const int64_t* shape_host,
                      int rank, const int32_t* cdf_dev, const int64_t* cdf_shape_host, int cdf_rank,
                      int precision, int debug_level, int16_t* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * UnboundedIndexRangeEncode / UnboundedIndexRangeDecode over a ragged batch, one warp per string:
 *   op contract   tensorflow_compression/cc/ops/range_coding_ops.cc:126-247
 *   CPU kernels   tensorflow_compression/cc/kernels/unbounded_index_range_coding_kernels.cc
 * Item u is elements [item_offsets_host[u], item_offsets_host[u+1]) of data_dev / index_dev (int32, flat); string u is
 * byte-identical to the reference op on item u alone wherever the reference is defined, and an empty item gives the
 * empty string.  cdf_dev int32 [cdf_shape_host[0], cdf_shape_host[1]] (cdf_rank 2, at least 3 columns), cdf_size_dev
 * and offset_dev int32 [rows].  Outside the reference's defined domain (DESIGN.md §3.8) d and u wrap as uint32, so
 * decoding what the encoder wrote gives back every int32 input.
 * Checked before any device work (TFCB_INVALID_ARGUMENT, with the reference's messages): precision and
 * overflow_width in [1, 16], debug_level 0 or 1, the shapes, null pointers, and the item offsets as for
 * tfcb_compress_ragged.  On the device, whatever debug_level is: index in [0, rows), cdf_size in [3, cols], and a
 * non-empty interval for every coded bin; debug_level 1 also checks every index and, per row, the start, end and
 * monotonicity of its cdf_size prefix.  Failures name the lowest failing string and element.
 * tfcb_unbounded_index_range_encode_ragged writes where each string starts to `offsets_dev` int64 [n_items + 1],
 * synchronises once and returns the total size and a handle; tfcb_unbounded_index_range_write writes the strings
 * back to back into `bytes_dev` [total] (asynchronous) and takes the handle back, also when it fails;
 * tfcb_unbounded_index_range_encoder_destroy releases a handle that is never written.
 * tfcb_unbounded_index_range_decode_ragged decodes string u (bytes_dev[offsets_dev[u] .. offsets_dev[u+1]), device
 * offsets) into out_dev[item_offsets_host[u] ..) and synchronises once.  Damaged strings decode to what the
 * reference decoder gives, except that a width prefix longer than ceil(32 / overflow_width) digits (undefined in the
 * reference) is reported as TFCB_INVALID_ARGUMENT naming the lowest failing string and element.
 * ---------------------------------------------------------------------------------------------- */
typedef struct tfcb_ubi_encoder tfcb_ubi_encoder;
int tfcb_unbounded_index_range_encode_ragged(const int32_t* data_dev, const int32_t* index_dev, int64_t n_items,
                                             const int64_t* item_offsets_host, const int32_t* cdf_dev,
                                             const int64_t* cdf_shape_host, int cdf_rank, const int32_t* cdf_size_dev,
                                             int64_t cdf_size_len, const int32_t* offset_dev, int64_t offset_len,
                                             int precision, int overflow_width, int debug_level, int64_t* offsets_dev,
                                             void* stream, tfcb_ubi_encoder** out, int64_t* total_bytes_host);
int tfcb_unbounded_index_range_write(tfcb_ubi_encoder* h, uint8_t* bytes_dev, void* stream);
void tfcb_unbounded_index_range_encoder_destroy(tfcb_ubi_encoder* h);
int tfcb_unbounded_index_range_decode_ragged(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_items,
                                             const int64_t* item_offsets_host, const int32_t* index_dev,
                                             const int32_t* cdf_dev, const int64_t* cdf_shape_host, int cdf_rank,
                                             const int32_t* cdf_size_dev, int64_t cdf_size_len,
                                             const int32_t* offset_dev, int64_t offset_len, int precision,
                                             int overflow_width, int debug_level, int32_t* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Mixture priors (Cheng et al. 2020), DESIGN.md §3.18: element e is coded under its own mixture of K components of
 * one family (0 Normal, 1 Logistic) with float32 weight_dev, loc_dev and scale_dev [n, K] (components innermost; the
 * weights need not sum to 1).  The row of element e, built on the device, is the index-mode overflow row
 * [-precision, c_0, .., c_n] of the support start_e .. start_e + L_e - 1 plus the escape bin; y is quantised as
 * int32(rint(y)) (saturating, NaN -> 0) and coded as the reference RangeEncoder codes y - start_e with that row,
 * escapes with the Elias-gamma payload, so every int32 codes.  The decoded value is float32 of that int32.
 * Checked before any device work (TFCB_INVALID_ARGUMENT): family, K in [1, 64], max_support in [1, 256], precision
 * in [1, 16] with 2^precision > max_support, tail_mass in (0, 1), null pointers and the item offsets as for
 * tfcb_compress_ragged.  On the device: non-finite parameters, a scale <= 0, a negative weight, all weights 0 and
 * weights summing below 2^-126;
 * failures name the lowest failing string and element.
 * tfcb_mixture_tables writes start_dev / size_dev int32 [n], the masses mass_dev int64 [n, max_support + 1] (m_0 ..
 * m_{L-1}, the escape mass m_L, zeros after) and rows_dev int32 [n, max_support + 3] (the row, padded with
 * 2^precision: a 2-D lookup the reference coder takes), and synchronises once.
 * tfcb_mixture_encode_ragged codes item u (elements [item_offsets_host[u], item_offsets_host[u+1]) of y_dev and the
 * parameters) into string u, writes where each string starts to offsets_dev int64 [n_items + 1], synchronises once
 * and returns the total size and a handle; tfcb_mixture_write writes the strings back to back into bytes_dev
 * (asynchronous) and takes the handle back, also when it fails; tfcb_mixture_encoder_destroy releases a handle that
 * is never written.  tfcb_mixture_decode_ragged decodes string u into out_dev float32 [item_offsets_host[u] ..) and
 * synchronises once; a damaged string decodes to what the reference decoder gives on the same rows.
 * ---------------------------------------------------------------------------------------------- */
typedef struct tfcb_mixture_encoder tfcb_mixture_encoder;
int tfcb_mixture_tables(const float* weight_dev, const float* loc_dev, const float* scale_dev, int64_t n, int K,
                        int family, int precision, double tail_mass, int max_support, int32_t* start_dev,
                        int32_t* size_dev, int64_t* mass_dev, int32_t* rows_dev, void* stream);
int tfcb_mixture_encode_ragged(const float* y_dev, const float* weight_dev, const float* loc_dev,
                               const float* scale_dev, int K, int family, int precision, double tail_mass,
                               int max_support, int64_t n_items, const int64_t* item_offsets_host, int64_t* offsets_dev,
                               void* stream, tfcb_mixture_encoder** out, int64_t* total_bytes_host);
int tfcb_mixture_write(tfcb_mixture_encoder* h, uint8_t* bytes_dev, void* stream);
void tfcb_mixture_encoder_destroy(tfcb_mixture_encoder* h);
int tfcb_mixture_decode_ragged(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_items,
                               const int64_t* item_offsets_host, const float* weight_dev, const float* loc_dev,
                               const float* scale_dev, int K, int family, int precision, double tail_mass,
                               int max_support, float* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Checkerboard context model with mixture priors, DESIGN.md §3.19: the two checkerboard passes of tfcb_cb_params
 * (anchors r + c even, then non-anchors; coding order and float32 order as there) on a network whose last layer has
 * 3KM outputs, followed by an epilogue that writes each (position, channel)'s K components for the mixture coder:
 * weight_k = expf(l_k - max_j l_j) (unnormalised), loc_k, scale_k = fmaxf(raw, 0.11f), channel c reading its K logits,
 * K locs and K scales from outputs 3Kc .. 3Kc + 3K - 1.  M is a multiple of 6 in [6, 384], K in [1, 64].
 * tfcb_cbm_packed_floats returns the packed size (-1 if unsupported) and, with `layout`, writes int64 [12]: K1, N3,
 * N4, NO = 3KM and the offsets of Wc [12M, 2M] (the 12 checkerboard taps, raster order), bc, W1 [4M, N3], b1,
 * W2 [N3, N4], b2, W3 [N4, 3KM], b3; tfcb_cbm_pack_weights copies the eight operands there.
 * tfcb_cbm_params runs one pass over every position of one colour of B images of H x W: weight_dev, loc_dev and
 * scale_dev float32 [B, n_k, M, K] in coding order (whole == 0), or each image's [H W, M, K] block of both colours at
 * this pass's rows (whole != 0).  The non-anchor pass reads the anchors of yhat_dev [B, H, W, M].  With y_dev
 * [B, H, W, M] (the encoder, whole != 0) it also writes y in coding order to y_cb_dev [B, H W, M] and
 * float((int)rintf(y)) at this pass's positions of yhat_out_dev [B, H, W, M].  Four launches for the anchors, five
 * for the non-anchors, none for an empty pass.  The _ragged forms take a list of n_images latents of
 * heights_host[i] x widths_host[i] back to back, per-pass outputs at M Q_i K (Q_i: the images before i's positions
 * of this colour), whole outputs at M P_i K (+ n_a,i M K for the non-anchors); the workspace holds the image table,
 * which tfcb_scc_scatter_ragged (offset 0, C = M) reads for the scatter of decoded latents.  Every argument is
 * checked before any launch (TFCB_INVALID_ARGUMENT).
 * ---------------------------------------------------------------------------------------------- */
int64_t tfcb_cbm_packed_floats(int M, int K, int64_t* layout);
int tfcb_cbm_pack_weights(int M, int K, const float* ctx_taps_dev, const float* ctx_bias_dev, const float* w1_dev,
                          const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_dev,
                          const float* b3_dev, float* packed_dev, int64_t packed_floats, void* stream);
/* Floats of workspace one tfcb_cbm_params pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_cbm_workspace_floats(int M, int K, int64_t B, int64_t H, int64_t W, int anchors);
int tfcb_cbm_params(const float* packed_dev, int64_t packed_floats, int M, int K, const float* yhat_dev,
                    const float* psi_dev, int64_t B, int64_t H, int64_t W, int anchors, float* work_dev,
                    int64_t work_floats, int whole, float* weight_dev, float* loc_dev, float* scale_dev,
                    const float* y_dev, float* y_cb_dev, float* yhat_out_dev, void* stream);
/* Floats of workspace one tfcb_cbm_params_ragged pass needs, or -1 if the arguments are not supported. */
int64_t tfcb_cbm_ragged_workspace_floats(int M, int K, int64_t n_images, const int64_t* heights_host,
                                         const int64_t* widths_host, int anchors);
int tfcb_cbm_params_ragged(const float* packed_dev, int64_t packed_floats, int M, int K, const float* yhat_dev,
                           const float* psi_dev, int64_t n_images, const int64_t* heights_host,
                           const int64_t* widths_host, int anchors, float* work_dev, int64_t work_floats, int whole,
                           float* weight_dev, float* loc_dev, float* scale_dev, const float* y_dev, float* y_cb_dev,
                           float* yhat_out_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * PmfToQuantizedCdf:
 *   op contract   tensorflow_compression/cc/ops/pmf_to_cdf_ops.cc:28-57
 *   CPU kernel    tensorflow_compression/cc/kernels/pmf_to_cdf_kernels.cc:58-208
 * pmf float32 [rows, n] -> cdf int32 [rows, n + 1].  Exact ties between bins are broken by lowest
 * bin index (the reference uses an unstable std::sort; see DESIGN.md).  Synchronises (it must
 * report non-finite / negative mass as TFCB_INVALID_ARGUMENT, pmf_to_cdf_kernels.cc:77-86).
 * ---------------------------------------------------------------------------------------------- */
int tfcb_pmf_to_quantized_cdf(const float* pmf_dev, int64_t rows, int64_t n, int precision,
                              int32_t* cdf_dev, void* stream);

/* The per-row loop of ContinuousEntropyModelBase._build_tables in one launch
 * (tensorflow_compression/python/entropy_models/continuous_base.py:282-294): for row r take
 * pmf[r, :lens[r]], append the overflow mass max(1 - sum, 0), quantise, and emit
 * [-precision, cdf...] into a 1-D concatenated lookup.  `lens_host` int32 [rows];
 * `lookup_dev` must hold sum(lens[r] + 3) int32.  Synchronises. */
int tfcb_build_lookup(const float* pmf_dev, int64_t rows, int64_t max_len, const int32_t* lens_host,
                      int precision, int32_t* lookup_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * RunLengthEncode / RunLengthDecode (and RunLengthGammaEncode/Decode = codes (-1, -1), use_run_length_for_non_zeros 0):
 *   op contract   tensorflow_compression/cc/ops/run_length_ops.cc:28-84
 *   CPU kernels   tensorflow_compression/cc/kernels/run_length_kernels.cc:52-262, bit packing cc/lib/bit_coder.cc:50-191
 * data int32 [n] (flattened) <-> one bit string.  run_length_code / magnitude_code >= 0: Rice code with that parameter,
 * < 0: Elias gamma.  Encode: `code_dev` has room for `capacity` bytes (a multiple of 4 is used); *n_bytes_host receives
 * the length of the code; TFCB_INVALID_ARGUMENT with the needed size in the message (and in *n_bytes_host) when it
 * does not fit.  The encoder is data parallel (scans + atomics); the decoder is serial within a string, as in the
 * reference.  Decode errors carry the reference's DataLoss messages.  Both calls synchronise `stream`.
 * ---------------------------------------------------------------------------------------------- */
int tfcb_run_length_encode(const int32_t* data_dev, int64_t n, int run_length_code, int magnitude_code,
                           int use_run_length_for_non_zeros, uint8_t* code_dev, int64_t capacity,
                           int64_t* n_bytes_host, void* stream);
int tfcb_run_length_decode(const uint8_t* code_dev, int64_t n_bytes, int run_length_code, int magnitude_code,
                           int use_run_length_for_non_zeros, int32_t* data_dev, int64_t n, void* stream);

/* Many strings in one launch (the reference has no batched op; this is an extension, e.g. for all coding units of
 * a tensor, or differently sized items).  Unit u is data_dev[unit_offsets_host[u] .. unit_offsets_host[u+1]); string u
 * is byte-identical to what tfcb_run_length_encode makes of unit u alone, and a unit with no elements gives the empty
 * string.  The host offsets are checked before any device work (TFCB_INVALID_ARGUMENT): n_units > 0, non-null
 * pointers, unit_offsets_host[0] == 0, non-decreasing, fewer than 2^31 elements in all, Rice parameters <= 31.
 * tfcb_run_length_encode_ragged writes where each string starts to `offsets_dev` int64 [n_units + 1], synchronises
 * once and returns the total size and a handle; data_dev must stay valid until tfcb_run_length_write packs the
 * strings back to back into `bytes_dev` [total] (asynchronous; only [0, total) is written) and takes the handle back,
 * also when it fails.  tfcb_run_length_encoder_destroy releases a handle that is never written. */
typedef struct tfcb_rl_encoder tfcb_rl_encoder;
int tfcb_run_length_encode_ragged(const int32_t* data_dev, int64_t n_units, const int64_t* unit_offsets_host,
                                  int run_length_code, int magnitude_code, int use_run_length_for_non_zeros,
                                  int64_t* offsets_dev, void* stream, tfcb_rl_encoder** out, int64_t* total_bytes_host);
int tfcb_run_length_write(tfcb_rl_encoder* h, uint8_t* bytes_dev, void* stream);
void tfcb_run_length_encoder_destroy(tfcb_rl_encoder* h);
/* Decodes string u (bytes_dev[offsets_dev[u] .. offsets_dev[u+1]), device offsets) into
 * data_dev[unit_offsets_host[u] .. unit_offsets_host[u+1]), one thread per string, and synchronises once.  The
 * unit offsets are checked like the encoder's.  A damaged string gives TFCB_INVALID_ARGUMENT naming the
 * lowest-numbered failing unit ("unit k: Out of bits to read.", as tfcb_run_length_decode would say of it). */
int tfcb_run_length_decode_ragged(const uint8_t* bytes_dev, const int64_t* offsets_dev, int64_t n_units,
                                  const int64_t* unit_offsets_host, int run_length_code, int magnitude_code,
                                  int use_run_length_for_non_zeros, int32_t* data_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * StochasticRound:
 *   op contract   tensorflow_compression/cc/ops/quantization_ops.cc:28-53
 *   CPU kernel    tensorflow_compression/cc/kernels/quantization_kernels.cc:48-95
 * outputs[i] = floor(inputs[i] / step_size) + (u_i < frac), u_i the i-th draw of the reference's xoshiro256+
 * stream seeded through std::seed_seq(seed) -- the same integers as the CPU op for the same seed (the
 * sequential stream is entered in parallel through GF(2) jump matrices).  `dtype` 0 float32, 1 float16,
 * 2 bfloat16; `seed_host` int32 [seed_len] in host memory, seed_len == 0 seeds from the clock
 * (quantization_kernels.cc:71-78).
 * ---------------------------------------------------------------------------------------------- */
int tfcb_stochastic_round(const void* inputs_dev, int dtype, int64_t n, float step_size,
                          const int32_t* seed_host, int64_t seed_len, int32_t* outputs_dev, void* stream);

/* ------------------------------------------------------------------------------------------------
 * GDN / IGDN (tensorflow_compression/python/layers/gdn.py:371-421), channels-last:
 *   u = rectify ? relu(x) : x;  p = |u|^alpha;  n_i = beta_i + sum_j p_j gamma[j,i];
 *   y_i = u_i / n_i^eps  (GDN)   or   u_i * n_i^eps  (IGDN)
 * x, y: float32 [n_pix, C] row-major;  gamma float32 [C, C] (row j, column i);  beta float32 [C].
 * alpha in {1, 2} and eps in {1, 0.5} take the reference's fast paths; other values use powf.
 * C in {128, 192, 256, 320} with 16-byte aligned pointers run on the tensor cores (bf16 split with fp32
 * accumulation: <= 1e-5 relative forward, <= 2e-5 of the largest gradient backward), with literal powf kernels for
 * trainable exponents and fixed ones outside those values; every other shape runs the fp32 kernels.
 * TFCB_GDN_FP32=1 in the environment forces the fp32 kernels.
 * The reference has no native GDN code (TF graph of abs / conv1x1 / bias_add / div); the backward
 * pass replaces TF autodiff of that graph.
 * ---------------------------------------------------------------------------------------------- */
#define TFCB_GDN_INVERSE 1
#define TFCB_GDN_RECTIFY 2
/* trainable exponents: compute `u ** alpha` / `n ** epsilon` literally even when the current value is 1, 2 or 1/2
 * (gdn.py:380-388,406-411 take the |u| / u^2 / sqrt shortcuts only for fixed exponents) */
#define TFCB_GDN_POW_ALPHA 4
#define TFCB_GDN_POW_EPSILON 8

int tfcb_gdn_forward(const float* x_dev, const float* gamma_dev, const float* beta_dev, float* y_dev,
                     int64_t n_pix, int C, int flags, float alpha, float epsilon, void* stream);

/* Gradients for upstream dy: dx [n_pix, C], dgamma [C, C], dbeta [C] (dgamma / dbeta are
 * OVERWRITTEN, reduced over all pixels).  `workspace_dev` must hold
 * tfcb_gdn_backward_workspace_bytes(n_pix, C) bytes. */
/* Mixed-precision variant (gdn_test.py:200-210: float32 variables, float16 / bfloat16 activations): x and y in
 * 16 bits (dtype 1 float16, 2 bfloat16), arithmetic in float32 -- 4 bytes of HBM traffic per element instead of 8.
 * Native kernel for C = 128 or 192 with alpha in {1, 2}, epsilon in {1, 1/2}; TFCB_INVALID_ARGUMENT otherwise (the
 * caller converts to float32).  y is exactly the float32 result for the widened x, rounded once to dtype. */
int tfcb_gdn_forward_16bit(const void* x_dev, const float* gamma_dev, const float* beta_dev, void* y_dev,
                           int64_t n_pix, int C, int dtype, int flags, float alpha, float epsilon, void* stream);

int64_t tfcb_gdn_backward_workspace_bytes(int64_t n_pix, int C);
int tfcb_gdn_backward(const float* x_dev, const float* gamma_dev, const float* beta_dev,
                      const float* dy_dev, float* dx_dev, float* dgamma_dev, float* dbeta_dev,
                      void* workspace_dev, int64_t n_pix, int C, int flags, float alpha,
                      float epsilon, void* stream);

/* Mixed-precision backward: x, dy and dx in 16 bits (dtype 1 float16, 2 bfloat16), dgamma / dbeta and the arithmetic
 * in float32 -- 6 bytes of algorithmic HBM traffic per element instead of 12.  dx is exactly the float32 backward's dx
 * for the widened x and dy, rounded once to dtype; dgamma / dbeta are the float32 backward's, bit for bit.  Native
 * kernels for C = 128 or 192 with alpha in {1, 2}, epsilon in {1, 1/2} and 16-byte aligned pointers;
 * TFCB_INVALID_ARGUMENT otherwise (the caller converts to float32), and under TFCB_GDN_FP32=1.  n_pix = 0 launches
 * nothing and sets dgamma / dbeta to zero, as tfcb_gdn_backward does.  `workspace_dev` must hold
 * tfcb_gdn_backward_16bit_workspace_bytes(n_pix, C) bytes. */
int64_t tfcb_gdn_backward_16bit_workspace_bytes(int64_t n_pix, int C);
int tfcb_gdn_backward_16bit(const void* x_dev, const float* gamma_dev, const float* beta_dev, const void* dy_dev,
                            void* dx_dev, float* dgamma_dev, float* dbeta_dev, void* workspace_dev, int64_t n_pix,
                            int C, int dtype, int flags, float alpha, float epsilon, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rate term of training: log p(y) of a prior convolved with U(-1/2, 1/2), forward and backward, fused.
 * Replaces UniformNoiseAdapter.log_prob (tensorflow_compression/python/distributions/uniform_noise.py:128-151)
 * and its autograd for the two families the models train with.  Each element is computed in double from float32
 * inputs and rounded once; the backward is the chain rule of the same expression (NaN and +-inf propagate as in
 * autograd of the graph).  Zero-size input does nothing (the parameter gradient is zeroed).
 *
 * Deep factorized, num_filters (3, 3) (deep_factorized.py:166-193): y float32 [n], element i in channel i mod C.
 * `packed_dev` float32 [C, 28], already transformed, per channel:
 *   softplus(matrices[0]) [3,1], softplus(matrices[1]) [3,3], softplus(matrices[2]) [1,3]  (row-major [out][in]),
 *   biases[0] [3], biases[1] [3], biases[2] [1], tanh(factors[0]) [3], tanh(factors[1]) [3].
 * The backward writes dy [n] and OVERWRITES dpacked [C, 28] with the gradient summed over all elements, in a fixed
 * order (bitwise reproducible); `workspace_dev` holds tfcb_noisy_deep_factorized_workspace_bytes(n, C) bytes.
 * Checked before any device work (TFCB_INVALID_ARGUMENT): C > 0, n >= 0, n mod C == 0, non-null pointers.
 * ---------------------------------------------------------------------------------------------- */
int tfcb_noisy_deep_factorized_log_prob(const float* y_dev, const float* packed_dev, float* out_dev, int64_t n,
                                        int C, void* stream);
int64_t tfcb_noisy_deep_factorized_workspace_bytes(int64_t n, int C);
int tfcb_noisy_deep_factorized_log_prob_backward(const float* y_dev, const float* packed_dev, const float* dout_dev,
                                                 float* dy_dev, float* dpacked_dev, void* workspace_dev, int64_t n,
                                                 int C, void* stream);

/* Location-scale bases: z = (y +- 1/2 - loc) / scale and the standard log-CDF of `base` (log_ndtr, log-sigmoid, or
 * the two-branch Laplace form).  y float32 [n]; loc / scale float32 [n], or one value read at [0] for every
 * element when `loc_scalar` / `scale_scalar` is nonzero.  The backward writes dy [n] and, where the pointer is not
 * NULL, the elementwise dloc [n] and dscale [n] (the caller sums them for a scalar operand).  Checked before any
 * device work (TFCB_INVALID_ARGUMENT): a known base, n >= 0, non-null y, loc, scale, out / dout, dy. */
#define TFCB_NOISY_NORMAL 0
#define TFCB_NOISY_LOGISTIC 1
#define TFCB_NOISY_LAPLACE 2
int tfcb_noisy_loc_scale_log_prob(int base, const float* y_dev, const float* loc_dev, int loc_scalar,
                                  const float* scale_dev, int scale_scalar, float* out_dev, int64_t n, void* stream);
int tfcb_noisy_loc_scale_log_prob_backward(int base, const float* y_dev, const float* loc_dev, int loc_scalar,
                                           const float* scale_dev, int scale_scalar, const float* dout_dev,
                                           float* dy_dev, float* dloc_dev, float* dscale_dev, int64_t n,
                                           void* stream);

/* ------------------------------------------------------------------------------------------------
 * Universal quantisation (tensorflow_compression/python/entropy_models/universal.py:30-62,147-170,446-466): the
 * shared noise levels and the coding tensors of UniversalBatchedEntropyModel / UniversalIndexedEntropyModel.
 * The level of the element at position i of its item is word (i mod 4) of Philox-4x32-10(counter = {lo32(i/4),
 * hi32(i/4), 0, 0}, key = {seed0, seed1}) mod the number of levels L, the stream entropy_models.stateless_uniform_int
 * draws on the CPU.  One launch, asynchronous.
 *
 * tfcb_stateless_uniform_int: the levels alone, one item of n elements, as int32 (reduced modulo `maxval` only when
 * maxval <= 2^32; wrapped to int32 like torch's cast).  Checked (TFCB_INVALID_ARGUMENT): n >= 0, maxval >= 1.
 *
 * tfcb_universal_coding_tensors: items split by host `item_offsets_host` [n_items + 1] (checked like
 * tfcb_compress_ragged's symbol offsets, before any device work); the noise position restarts in every item.  Writes
 * per element the int32 table index and the offset (level + 1) / (L + 1) - 1/2, computed in double and written as
 * float32, or as float64 when `offset_is_f64` is nonzero.
 *   batched (indexes_dev NULL, n_ranges 0): index = level * prior_size + i mod prior_size.
 *   indexed: indexes_dev [elements, n_ranges] float32 (or float64 when `indexes_is_f64`), 1 <= n_ranges <= 8; the
 *     coordinates (level, indexes...) are read in that type, clipped to [0, range - 1] (max then min; NaN stays NaN)
 *     and truncated to int32 (NaN gives 0, as torch's cast on the device), and summed with the int32 strides of
 *     (L,) + index_ranges_host.  The offset uses the clipped level in that type.
 * Checked (TFCB_INVALID_ARGUMENT): 1 <= L < 2^31, prior_size >= 1 (batched), positive index ranges, non-null
 * outputs (and indexes) when there are elements. */
int tfcb_stateless_uniform_int(int32_t* out_dev, int64_t n, uint32_t seed0, uint32_t seed1, int64_t maxval,
                               void* stream);
int tfcb_universal_coding_tensors(int64_t n_items, const int64_t* item_offsets_host, uint32_t seed0, uint32_t seed1,
                                  int64_t num_noise_levels, int64_t prior_size, const void* indexes_dev,
                                  int32_t indexes_is_f64, const int64_t* index_ranges_host, int32_t n_ranges,
                                  int32_t* table_index_dev, void* offset_dev, int32_t offset_is_f64, void* stream);

/* Number of kernel launches issued by this library since load (bench.py's `gpu_launches`). */
/* Gradients of the loss with respect to the scalar exponents alpha and epsilon (gdn.py:345-367 makes them
 * trainable GDNParameters; TF autodiff differentiates through pow): dalpha_depsilon_dev float32 [2].
 * workspace_dev: tfcb_gdn_exponent_grads_workspace_bytes() bytes. */
int64_t tfcb_gdn_exponent_grads_workspace_bytes(void);
int tfcb_gdn_exponent_grads(const float* x_dev, const float* gamma_dev, const float* beta_dev,
                            const float* dy_dev, float* dalpha_depsilon_dev, void* workspace_dev,
                            int64_t n_pix, int C, int flags, float alpha, float epsilon, void* stream);

/* All five gradients in one call: dx, dgamma, dbeta as tfcb_gdn_backward and dalpha_depsilon_dev float32 [2] as
 * tfcb_gdn_exponent_grads, for any configuration.  C in {128, 192, 256, 320} with a trainable exponent (or a fixed one
 * outside {1, 2} / {1, 1/2}) and 16-byte aligned pointers runs the tensor-core backward with both exponent sums fused
 * into its epilogues (bitwise reproducible from call to call); everything else, and TFCB_GDN_FP32=1, runs
 * tfcb_gdn_backward's kernels followed by tfcb_gdn_exponent_grads' and gives their results.  `workspace_dev` holds
 * tfcb_gdn_backward_exponents_workspace_bytes(n_pix, C) bytes: tfcb_gdn_backward's workspace followed by
 * tfcb_gdn_exponent_grads_workspace_bytes() bytes.  Shapes, pointers and C <= 3072 are checked before any device work
 * (TFCB_INVALID_ARGUMENT); n_pix = 0 launches nothing and sets dgamma, dbeta, dalpha and depsilon to zero. */
int64_t tfcb_gdn_backward_exponents_workspace_bytes(int64_t n_pix, int C);
int tfcb_gdn_backward_exponents(const float* x_dev, const float* gamma_dev, const float* beta_dev, const float* dy_dev,
                                float* dx_dev, float* dgamma_dev, float* dbeta_dev, float* dalpha_depsilon_dev,
                                void* workspace_dev, int64_t n_pix, int C, int flags, float alpha, float epsilon,
                                void* stream);

/* Channels-first GDN / IGDN (the reference's data_format="channels_first", gdn.py:127-175): x, y, dy, dx are
 * [n_items, C, spatial] contiguous, spatial the product of the spatial dimensions, so element (item b, channel c,
 * position s) is at (b * C + c) * spatial + s.  `dtype` 0 float32, 1 float16, 2 bfloat16 (parameters, dgamma, dbeta
 * and the arithmetic float32).  The same kernels as the channels-last entries read and write this layout in place:
 * every output (y, dx, dgamma, dbeta, dalpha / depsilon) is bit for bit what tfcb_gdn_forward / tfcb_gdn_backward /
 * tfcb_gdn_backward_exponents (float32) or the _16bit entries (16 bits) give for the same tensors transposed to
 * [n_items * spatial, C], so the channels-last accuracy bounds above hold as they are.
 * Covered exactly where the channels-last tensor-core kernels run: float32 at C in {128, 192, 256, 320} with any
 * exponents, float16 / bfloat16 at C in {128, 192} with alpha in {1, 2} and epsilon in {1, 1/2} and no POW flag.
 * Checked before any device work (TFCB_INVALID_ARGUMENT): n_items, spatial >= 0, C > 0, n_items * spatial * C within
 * int64; a covered configuration (never under TFCB_GDN_FP32=1: transpose to channels-last there); non-null pointers
 * (x, y, dy, dx may be NULL when n_items * spatial = 0); x, y, dy, dx, beta and the workspace 16-byte aligned.
 * An empty tensor launches nothing; the backward then sets dgamma, dbeta (and dalpha / depsilon) to zero.
 * Backward: dalpha_depsilon_dev float32 [2] receives (dL/dalpha, dL/depsilon) and is required with a POW flag; it may
 * be NULL without one, and must be NULL when both exponents take the shortcuts.  `workspace_dev` holds
 * tfcb_gdn_backward_cf_workspace_bytes(n_items, spatial, C, dtype) bytes (-1 for arguments the entries reject). */
int tfcb_gdn_forward_cf(const void* x_dev, const float* gamma_dev, const float* beta_dev, void* y_dev, int64_t n_items,
                        int64_t spatial, int C, int dtype, int flags, float alpha, float epsilon, void* stream);
int64_t tfcb_gdn_backward_cf_workspace_bytes(int64_t n_items, int64_t spatial, int C, int dtype);
int tfcb_gdn_backward_cf(const void* x_dev, const float* gamma_dev, const float* beta_dev, const void* dy_dev,
                         void* dx_dev, float* dgamma_dev, float* dbeta_dev, float* dalpha_depsilon_dev,
                         void* workspace_dev, int64_t n_items, int64_t spatial, int C, int dtype, int flags,
                         float alpha, float epsilon, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Image quality: the statistics behind tf.image.ssim and tf.image.ssim_multiscale
 * (tensorflow/python/ops/image_ops_impl.py), which the model scripts print after compressing an image
 * (models/bls2017.py:294-295, bmshj2018.py:370-371, ms2020.py:540-541).  The host combines them into the metrics:
 *   ssim            = mean over channels of stats[..., 0, 1]
 *   ssim_multiscale = mean over channels of prod_k v_k ** power_factors[k], v_k = relu(stats[..., k, 0]) for
 *                     k < n_scales - 1 and relu(stats[..., n_scales - 1, 1]) for the last scale.
 * img1_dev, img2_dev: [n_images, H, W, C] channels-last, `dtype` 0 float32, 1 float16, 2 bfloat16, 3 uint8 (widened to
 * float32(u) * float32(1/255) like convert_image_dtype; `max_val` is given after that conversion, 1.0 for 255).
 * Window: filter_size x filter_size, the softmax of -(i^2 + j^2) / (2 filter_sigma^2) around (filter_size - 1) / 2,
 * VALID, per channel.  With c1 = (k1 max_val)^2, c2 = (k2 max_val)^2 and mx, my, S(.) the windowed means and moments:
 *   l = (2 mx my + c1) / (mx^2 + my^2 + c1),  cs = (2 (Sxy - mx my) + c2) / (S(x^2 + y^2) - mx^2 - my^2 + c2).
 * Scale s + 1 is scale s padded at its end by one repeated row / column where odd, then 2x2 average pooled.
 * stats_dev float32 [n_images, C, n_scales, 2] receives (mean(cs), mean(l * cs)) over each scale's valid positions,
 * summed in double in a fixed order and rounded once: bitwise reproducible, and an image's values do not depend on the
 * batch it is in.  The launch count depends on n_scales only.
 *
 * The backward takes g_stats_dev float32 [n_images, C, n_scales, 2] (the loss gradient of stats) and writes dimg1 /
 * dimg2 in the image dtype (computed in float32, rounded once); either may be NULL, and with both NULL nothing runs.
 * uint8 images have no gradient (TFCB_INVALID_ARGUMENT).
 *
 * `workspace_dev` holds tfcb_ssim_workspace_bytes(dtype, n_images, H, W, C, n_scales, filter_size) bytes (the same
 * size serves both directions; -1 for arguments the entries reject).  Checked before any device work
 * (TFCB_INVALID_ARGUMENT): a known dtype; n_images >= 0, H, W, C >= 1, n_images * H * W * C within int64 and
 * n_images * C < 2^31; 1 <= filter_size <= 32; 1 <= n_scales <= 16; every scale at least filter_size in H and W (as
 * TF asserts: with the defaults 161 passes and 160 fails); filter_sigma > 0 and finite; finite max_val, k1, k2; non-null
 * pointers.  n_images = 0 launches nothing. */
int64_t tfcb_ssim_workspace_bytes(int dtype, int64_t n_images, int64_t H, int64_t W, int64_t C, int n_scales,
                                  int filter_size);
int tfcb_ssim_stats(const void* img1_dev, const void* img2_dev, int dtype, int64_t n_images, int64_t H, int64_t W,
                    int64_t C, float max_val, int n_scales, int filter_size, float filter_sigma, float k1, float k2,
                    float* stats_dev, void* workspace_dev, void* stream);
int tfcb_ssim_stats_backward(const void* img1_dev, const void* img2_dev, int dtype, int64_t n_images, int64_t H,
                             int64_t W, int64_t C, float max_val, int n_scales, int filter_size, float filter_sigma,
                             float k1, float k2, const float* g_stats_dev, void* dimg1_dev, void* dimg2_dev,
                             void* workspace_dev, void* stream);

/* Rate-distortion evaluation of a list of image pairs of their own sizes: the forward statistics above and the mean
 * squared error of every image and plane, with one launch per kernel per scale whatever the number of images (at most
 * 2 n_scales launches).  Pair i is img1_dev / img2_dev [item_offsets_host[i] .. item_offsets_host[i + 1]), channels-last
 * [heights_host[i], widths_host[i], C] in `dtype` (as tfcb_ssim_stats; uint8 is widened the same way).  The offsets and
 * sizes are host arrays [n_items + 1] and [n_items].  `mode` selects the planes:
 *   TFCB_COLOR_RGB    the C channels;
 *   TFCB_COLOR_Y      one Y' plane from C = 3;
 *   TFCB_COLOR_YCBCR  three Y'CbCr planes from C = 3.
 * Y'CbCr is BT.601 full range (JFIF) in the images' units after the dtype conversion, m = max_val, evaluated in float32
 * left to right with every product and sum rounded:
 *   Y' = 0.299 R + 0.587 G + 0.114 B
 *   Cb = float32(128/255) m + (-0.168736 R - 0.331264 G + 0.5 B)
 *   Cr = float32(128/255) m + (0.5 R - 0.418688 G - 0.081312 B)
 * It is applied as scale 0 is read; nothing converted is written to memory.
 * stats_dev float32 [n_items, planes, n_scales, 2] receives what tfcb_ssim_stats gives for the planes (for RGB, bit
 * for bit what it gives for each image alone).  mse_dev float32 [n_items, planes] receives mean((x - y)^2) over each
 * plane, summed in double in a fixed order and rounded once.  Results are bitwise reproducible, and an image's values
 * do not depend on the list it is in.  There is no backward.
 * `workspace_dev` holds tfcb_image_metrics_ragged_workspace_bytes(...) bytes (-1 for arguments the entry rejects).
 * Checked before any device work (TFCB_INVALID_ARGUMENT): a known dtype and mode; C >= 1, and C = 3 for Y' and Y'CbCr;
 * n_items >= 0; every size at least 1 and, at every scale, at least filter_size (the message names the image);
 * item_offsets_host[0] = 0 and each item spanning H W C elements; the other arguments as tfcb_ssim_stats; non-null
 * pointers.  n_items = 0 launches nothing.  The offsets and sizes are staged into the workspace (pageable copies). */
#define TFCB_COLOR_RGB 0
#define TFCB_COLOR_Y 1
#define TFCB_COLOR_YCBCR 2
int64_t tfcb_image_metrics_ragged_workspace_bytes(int dtype, int64_t n_items, const int64_t* heights_host,
                                                  const int64_t* widths_host, int64_t C, int mode, int n_scales,
                                                  int filter_size);
int tfcb_image_metrics_ragged(const void* img1_dev, const void* img2_dev, int dtype, int64_t n_items,
                              const int64_t* item_offsets_host, const int64_t* heights_host,
                              const int64_t* widths_host, int64_t C, int mode, float max_val, int n_scales,
                              int filter_size, float filter_sigma, float k1, float k2, float* stats_dev,
                              float* mse_dev, void* workspace_dev, void* stream);

int64_t tfcb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* TFCB200_H_ */
