/*
 * gpujpegx.h -- extension entry points of the H100-native libgpujpeg (additive: nothing here exists in the reference;
 * every name carries the prefix gpujpegx_).  The reference API itself is in libgpujpeg/gpujpeg.h.
 *
 *   * resident re-runs and coefficient read-back: used by bench.py and the parity tests
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
/* stage_mask: bit 0 = K1 (colour + FDCT + quantisation), bit 1 = K2 (Huffman encode + scan assembly); d_raw == NULL
 * re-uses the device copy of the last host image */
GPUJPEG_API int gpujpegx_encoder_run_resident(struct gpujpeg_encoder* encoder, const uint8_t* d_raw, int stage_mask);
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
