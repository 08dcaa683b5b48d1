/*
 * gpujpegx.h -- extension entry points of the H100-native libgpujpeg (additive: nothing here exists in the reference;
 * every name carries the prefix gpujpegx_).  The reference API itself is in libgpujpeg/gpujpeg.h.
 *
 *   * resident re-runs and coefficient read-back: used by bench.py and the parity tests
 *   * gpujpegx_transcode*: lossless JPEG-to-JPEG rewrite (restart markers, fitted Huffman tables, baseline from progressive,
 *     lossless turns and mirrors)
 *   * gpujpegx_batch_*: a batch of independent frames sharded over the GPUs of one box (SURVEY.md section 8e,
 *     BASELINE.json config 5).  The reference's only multi-device affordances are gpujpeg_init_device /
 *     gpujpeg_set_device (src/gpujpeg_common.c:219-288) and "one coder per host thread with its own stream"
 *     (test/misc/mt_encode.c:12-43); this is that pattern packaged: one host thread + one stream + one coder pair per
 *     device, frames assigned round-robin, no collective on the data path.  Frames that all live on the first device
 *     are moved to their owners by peer copies (NVLink) -- the scatter / gather of section 8e.
 */
#ifndef GPUJPEGX_H
#define GPUJPEGX_H

#include "gpujpeg_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- resident re-runs (no copies, no synchronisation; the caller times the coder's stream) ---- */
/* stage_mask: bit 0 = K1 (colour + FDCT + quantisation), bit 3 = the symbol statistics of enc_opt_huffman=optimized alone,
 * bit 1 = K2 (Huffman encode + scan assembly, with the tables the last gpujpeg_encoder_encode chose); d_raw == NULL
 * re-uses the device copy of the last host image */
GPUJPEG_API int gpujpegx_encoder_run_resident(struct gpujpeg_encoder* encoder, const uint8_t* d_raw, int stage_mask);
/* the symbol counts of the last frame's statistics (enc_opt_huffman=optimized, or a resident run with bit 3), indexed
 * [table class][DC 0 / AC 1][symbol] (parity tests); -1 when no statistics have run since the last encode */
GPUJPEG_API int gpujpegx_encoder_get_symbol_counts(struct gpujpeg_encoder* encoder, uint64_t out[2][2][256]);
/* stage_mask: bit 2 = K0 (marker list + clean stream from the JPEG bytes on the device), bit 0 = K3 (Huffman decode),
 * bit 1 = K4 (dequantisation + IDCT + colour); d_out == NULL writes into the decoder's own buffer */
GPUJPEG_API int gpujpegx_decoder_run_resident(struct gpujpeg_decoder* decoder, uint8_t* d_out, int stage_mask);
/* the JPEG stream of the last frame as the last K2 launch left it (resident re-runs included), the same bytes
 * gpujpeg_encoder_encode returns: its size, copied into `out` when `out` is not NULL and holds it; -1 on error or when
 * the encoder writes segment-info tables (those are completed on the host) */
GPUJPEG_API long long gpujpegx_encoder_get_stream(struct gpujpeg_encoder* encoder, uint8_t* out, size_t capacity);
/* quantised coefficients of the last frame, natural order, block-major (parity tests).  The decoder variant returns 1
 * when the values are already multiplied by the quantiser (integer IDCT flavour), 0 otherwise, -1 on error */
GPUJPEG_API int gpujpegx_encoder_get_coefficients(struct gpujpeg_encoder* encoder, int16_t* out, size_t count);
GPUJPEG_API int gpujpegx_decoder_get_coefficients(struct gpujpeg_decoder* decoder, int16_t* out, size_t count);
/* 1 if the scans of the last decoded frame were split by the stream's own segment-info tables (struct
 * gpujpeg_parameters.segment_info of the encoder; reference: src/gpujpeg_reader.c:1168-1215) -- then no marker scan ran on
 * the device --, 0 if by the marker scan, -1 on error */
GPUJPEG_API int gpujpegx_decoder_used_segment_info(const struct gpujpeg_decoder* decoder);
/* 1 if the Huffman stage of the last decoded frame ran the sub-sequence kernel (dec_opt_huffman: restart segments of any
 * length, several threads per segment), 0 if another kernel, -1 on error */
GPUJPEG_API int gpujpegx_decoder_used_subsequences(const struct gpujpeg_decoder* decoder);
/* measurement aid: rounds the sub-sequence kernel needed to reach its fixed point on the last frame (or on its last resident
 * re-run); 129 when it finished a segment in one thread.  Waits for the decoder's stream.  -1 if the frame did not run it */
GPUJPEG_API int gpujpegx_decoder_subsequence_rounds(struct gpujpeg_decoder* decoder);

/* ---- lossless JPEG-to-JPEG rewrite (what jpegtran -restart N -optimize -trim / -perfect does on a CPU) ----
 * Every stream gpujpeg_decoder_decode takes (baseline with or without restart markers, progressive, 1, 3 or 4 components) is
 * rewritten as one baseline frame with its quantised coefficients unchanged: the source's quantisation tables and COM
 * segments, its interleaving (a progressive frame of several components becomes one interleaved scan), the restart interval
 * and Huffman tables asked for, optionally turned and mirrored in the DCT domain.  One device and one stream per instance, not
 * thread-safe per instance; a refused frame leaves the instance usable. */
struct gpujpegx_transcoder;

/* "none" (default), "auto" (the stream's SPIFF / Exif orientation) or "<deg>[-]" (deg 0, 90, 180, 270): turn clockwise, then
 * mirror horizontally -- the grammar of dec_opt_orientation.  jpegtran's -flip horizontal = "0-", -flip vertical = "180-",
 * -transpose = "90-", -transverse = "270-".  Orientation metadata is kept with "none" and dropped after any other transform. */
#define GPUJPEGX_TRAN_OPT_TRANSFORM "tran_opt_transform"
/* "0" (default): partial edge iMCUs that a transform would move are dropped (jpegtran -trim); "1": such a frame is refused
 * (jpegtran -perfect) */
#define GPUJPEGX_TRAN_OPT_PERFECT "tran_opt_perfect"
/* "auto" (default: what RESTART_AUTO gives the encoder for the output's size, sampling and interleaving) or N >= 0 MCUs (0: no
 * restart markers) */
#define GPUJPEGX_TRAN_OPT_RESTART "tran_opt_restart"
/* "standard" (default: T.81 Annex K tables) or "optimized" (tables fitted to the frame, as enc_opt_huffman=optimized) */
#define GPUJPEGX_TRAN_OPT_HUFFMAN "tran_opt_huffman"
/* "none" (default) or "WxH+X+Y" (the grammar of dec_opt_crop): jpegtran -crop with -trim, a rectangle of the transformed image
 * (after tran_opt_transform, so "auto" crops the upright image) rewritten without re-encoding.  With W_u x H_u the transformed
 * source and W_t x H_t the output without a crop (W_u x H_u trimmed to whole output iMCUs along a reversed axis):
 *   - refused unless X + W <= W_u and Y + H <= H_u;
 *   - the origin is rounded down to the output's iMCU grid (8 * max h x 8 * max v samples after the transform): X0, Y0; refused
 *     if X0 >= W_t or Y0 >= H_t (the rectangle starts in the edge strip the trim drops);
 *   - the output is (min(X + W, W_t) - X0) x (min(Y + H, H_t) - Y0): the uncropped output's blocks from (X0, Y0) on, whole iMCUs
 *     of the source's MCU padding included, a block past the source's grid keeping only its clamped neighbour's DC;
 *   - everything else as without a crop (tables, COM segments, orientation metadata, perfect -- checked on the whole frame --,
 *     the automatic restart interval for the output's size); only the rectangle's coefficients are range-checked, and only the
 *     restart segments that hold its blocks are Huffman-decoded;
 *   - a rectangle of all of W_t x H_t gives the bytes of no crop. */
#define GPUJPEGX_TRAN_OPT_CROP "tran_opt_crop"

/* NULL without a device */
GPUJPEG_API struct gpujpegx_transcoder* gpujpegx_transcoder_create(cudaStream_t stream);
GPUJPEG_API void gpujpegx_transcoder_destroy(struct gpujpegx_transcoder* t);
/* 0 / -1 */
GPUJPEG_API int gpujpegx_transcoder_set_option(struct gpujpegx_transcoder* t, const char* opt, const char* val);
/* jpeg: host memory.  *out: transcoder-owned host buffer, valid until the next call or destroy.  0 / -1. */
GPUJPEG_API int gpujpegx_transcode(struct gpujpegx_transcoder* t, const uint8_t* jpeg, size_t size, uint8_t** out,
                                   size_t* out_size);

/* ---- batches of independent frames over several GPUs ---- */
struct gpujpegx_batch;

/* where the frames of a batch call live */
enum gpujpegx_location {
    GPUJPEGX_HOST = 0,          /* host memory (pinned or not): every worker copies over its own PCIe link */
    GPUJPEGX_DEVICE_OWNER = 1,  /* device memory of the GPU that processes the frame (frame f -> devices[f % count]) */
    GPUJPEGX_DEVICE_FIRST = 2   /* device memory of devices[0]: moved to / from the owner by peer copies */
};

/* One worker (host thread, CUDA stream, encoder, decoder) per entry of `devices`; NULL / 0 = every visible device.
 * Returns NULL when a device cannot be initialised. */
GPUJPEG_API struct gpujpegx_batch* gpujpegx_batch_create(const int* devices, int device_count);
GPUJPEG_API void gpujpegx_batch_destroy(struct gpujpegx_batch* batch);
GPUJPEG_API int gpujpegx_batch_device_count(const struct gpujpegx_batch* batch);
/* device that processes frame f */
GPUJPEG_API int gpujpegx_batch_owner(const struct gpujpegx_batch* batch, int frame);

/* Encodes images[0..count) with the same parameters (as gpujpeg_encoder_encode).  jpegs[f] / sizes[f] receive a
 * batch-owned host buffer holding frame f's stream, valid until the next gpujpegx_batch_encode or the destroy.
 * Returns 0, or -1 if any frame failed. */
GPUJPEG_API int gpujpegx_batch_encode(struct gpujpegx_batch* batch, const struct gpujpeg_parameters* param,
                                      const struct gpujpeg_image_parameters* param_image, const uint8_t* const* images, int count,
                                      enum gpujpegx_location where, uint8_t** jpegs, size_t* sizes);
/* Decodes jpegs[0..count) (host memory) into outputs[f] (caller-owned, in `where`; each must hold the decoded image:
 * default output format, as gpujpeg_decoder_decode with a custom buffer).  Returns 0, or -1 if any frame failed. */
GPUJPEG_API int gpujpegx_batch_decode(struct gpujpegx_batch* batch, const uint8_t* const* jpegs, const size_t* sizes, int count,
                                      uint8_t* const* outputs, enum gpujpegx_location where);
/* wall-clock milliseconds of the last batch call (first job handed out -> last worker done) */
GPUJPEG_API double gpujpegx_batch_last_ms(const struct gpujpegx_batch* batch);

#ifdef __cplusplus
}
#endif
#endif
