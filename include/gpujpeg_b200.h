/*
 * gpujpeg_b200.h -- the C ABI of the H100-native JPEG hot path.
 *
 * This single header declares, in one place, every type and entry point that a
 * caller of libgpujpeg binds against.  It is written from scratch (no text
 * taken from the reference) but is ABI-identical to the reference interface it
 * replaces -- same identifiers, same enum values, same struct layouts, same
 * calling convention -- so that code written against
 *     #include <libgpujpeg/gpujpeg.h>
 * recompiles (or simply re-links) against this library unchanged.  The five
 * headers under include/libgpujpeg/ are thin forwarders to this file.
 *
 * Every declaration cites the reference interface it replaces as
 *     [ref: <file>:<line>]   (paths relative to the reference tree root).
 *
 * Struct sizes on x86-64 (checked by tests/test_abi.py):
 *   gpujpeg_parameters 40, gpujpeg_image_parameters 20, gpujpeg_encoder_input 24,
 *   gpujpeg_decoder_output 64, gpujpeg_decoder_init_parameters 16,
 *   gpujpeg_image_info 512, gpujpeg_duration_stats 72, gpujpeg_devices_info 3048,
 *   gpujpeg_image_metadata 8.
 */
#ifndef GPUJPEG_B200_H_ABI
#define GPUJPEG_B200_H_ABI

#ifdef __cplusplus
#include <cstddef>
#include <cstdint>
#else
#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>
#endif

#ifndef __DRIVER_TYPES_H__
struct CUstream_st;
typedef struct CUstream_st* cudaStream_t;
#endif

#if defined(__GNUC__) || defined(__clang__)
#define GPUJPEG_API __attribute__((visibility("default")))
#define GPUJPEG_DEPRECATED __attribute__((deprecated))
#define ATTRIBUTE_UNUSED __attribute__((unused))
#else
#define GPUJPEG_API
#define GPUJPEG_DEPRECATED
#define ATTRIBUTE_UNUSED
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------- */
/* version                                         [ref: libgpujpeg/gpujpeg_version.h.cmakein:31-42] */
#define GPUJPEG_VERSION_MAJOR 0
#define GPUJPEG_VERSION_MINOR 27
#define GPUJPEG_VERSION_PATCH 13
#define GPUJPEG_MK_VERSION_INT(major, minor, patch) ((major) << 16U | (minor) << 8U | (patch))
#define GPUJPEG_VERSION_INT \
    GPUJPEG_MK_VERSION_INT(GPUJPEG_VERSION_MAJOR, GPUJPEG_VERSION_MINOR, GPUJPEG_VERSION_PATCH)
#define LIBGPUJPEG_API_VERSION ((GPUJPEG_VERSION_MAJOR << 8U) | GPUJPEG_VERSION_MINOR)

/* ------------------------------------------------------------------------- */
/* scalar constants                                [ref: libgpujpeg/gpujpeg_type.h:52-82] */
#define GPUJPEG_MAX_COMPONENT_COUNT 4
#define GPUJPEG_INIT_DEV_VERBOSE 1
#define GPUJPEG_OPENGL_INTEROPERABILITY 2
#define GPUJPEG_VERBOSE GPUJPEG_INIT_DEV_VERBOSE
#define GPUJPEG_MAX_SEGMENT_INFO_HEADER_COUNT 100
#define GPUJPEG_NOERR 0
#define GPUJPEG_ERROR (-1)
#define GPUJPEG_ERR_RESTART_CHANGE (-2)
#define GPUJPEG_VAL_TRUE "1"
#define GPUJPEG_VAL_FALSE "0"

/* colour spaces                                   [ref: libgpujpeg/gpujpeg_type.h:87-96] */
enum gpujpeg_color_space {
    GPUJPEG_NONE = 0,
    GPUJPEG_RGB = 1,
    GPUJPEG_YCBCR_BT601 = 2,
    GPUJPEG_YCBCR_BT601_256LVLS = 3,
    GPUJPEG_YCBCR_JPEG = GPUJPEG_YCBCR_BT601_256LVLS,
    GPUJPEG_YCBCR_BT709 = 4,
    GPUJPEG_YCBCR = GPUJPEG_YCBCR_BT709,
    GPUJPEG_YUV = 5
};

/* file header flavours                            [ref: libgpujpeg/gpujpeg_type.h:98-105] */
enum gpujpeg_header_type {
    GPUJPEG_HEADER_DEFAULT = 0,
    GPUJPEG_HEADER_JFIF = 1 << 0,
    GPUJPEG_HEADER_SPIFF = 1 << 1,
    GPUJPEG_HEADER_ADOBE = 1 << 2,
    GPUJPEG_HEADER_EXIF = 1 << 3
};

/* raw pixel layouts                               [ref: libgpujpeg/gpujpeg_type.h:110-137] */
enum gpujpeg_pixel_format {
    GPUJPEG_PIXFMT_NONE = -1,
    GPUJPEG_U8 = 0,             /* 1 x u8                                  */
    GPUJPEG_444_U8_P012 = 1,    /* c0 c1 c2 c0 c1 c2 ...  (the hot path)   */
    GPUJPEG_444_U8_P0P1P2 = 2,  /* three full planes                       */
    GPUJPEG_422_U8_P1020 = 3,   /* c1 c0 c2 c0 packed 4:2:2                */
    GPUJPEG_422_U8_P0P1P2 = 4,  /* planar 4:2:2                            */
    GPUJPEG_420_U8_P0P1P2 = 5,  /* planar 4:2:0                            */
    GPUJPEG_4444_U8_P0123 = 6   /* 4 x u8 per pixel                        */
};

/* [ref: libgpujpeg/gpujpeg_type.h:140-144] */
struct gpujpeg_component_sampling_factor {
    uint8_t horizontal;
    uint8_t vertical;
};

/* metadata carried next to the pixels             [ref: libgpujpeg/gpujpeg_type.h:146-165] */
enum { GPUJPEG_METADATA_ORIENTATION, GPUJPEG_METADATA_COUNT };
struct gpujpeg_orientation {
    unsigned rotation : 2;
    unsigned flip : 1;
};
struct gpujpeg_image_metadata {
    struct {
        union {
            struct gpujpeg_orientation orient;
        };
        unsigned set : 1;
    } vals[GPUJPEG_METADATA_COUNT];
};

/* ------------------------------------------------------------------------- */
/* library-wide helpers                            [ref: libgpujpeg/gpujpeg_common.h:82-100] */
GPUJPEG_API int gpujpeg_version(void);
GPUJPEG_API const char* gpujpeg_version_to_string(int version);
GPUJPEG_API double gpujpeg_get_time(void);

/* device enumeration                              [ref: libgpujpeg/gpujpeg_common.h:102-158] */
#define GPUJPEG_MAX_DEVICE_COUNT 10
struct gpujpeg_device_info {
    int id;
    char name[256];
    int cc_major;
    int cc_minor;
    size_t global_memory;
    size_t constant_memory;
    size_t shared_memory;
    int register_count;
    int multiprocessor_count;
};
struct gpujpeg_devices_info {
    int device_count;
    struct gpujpeg_device_info device[GPUJPEG_MAX_DEVICE_COUNT];
};
GPUJPEG_API struct gpujpeg_devices_info gpujpeg_get_devices_info(void);
GPUJPEG_API int gpujpeg_print_devices_info(void);
GPUJPEG_API int gpujpeg_init_device(int device_id, int flags);

/* coder parameters                                [ref: libgpujpeg/gpujpeg_common.h:160-232] */
enum restart_int { RESTART_AUTO = -1, RESTART_NONE = 0 };
enum verbosity {
    GPUJPEG_LL_QUIET = -1,
    GPUJPEG_LL_INFO = 0,
    GPUJPEG_LL_STATUS = 1,
    GPUJPEG_LL_VERBOSE = 2,
    GPUJPEG_LL_DEBUG = 3,
    GPUJPEG_LL_DEBUG2 = 4
};
struct gpujpeg_parameters {
    int verbose;           /* enum verbosity                                        */
    int perf_stats;        /* keep per-stage timers                                 */
    int quality;           /* 0..100                                                */
    int restart_interval;  /* MCUs per restart segment; RESTART_AUTO; RESTART_NONE  */
    int interleaved;       /* 1 = single scan, 0 = one scan per component           */
    int segment_info;      /* emit APP13 segment offset tables                      */
    int comp_count;        /* 0 = derive from pixel format                          */
    struct gpujpeg_component_sampling_factor sampling_factor[GPUJPEG_MAX_COMPONENT_COUNT];
    enum gpujpeg_color_space color_space_internal;
};
GPUJPEG_API void gpujpeg_set_default_parameters(struct gpujpeg_parameters* param);
GPUJPEG_API struct gpujpeg_parameters gpujpeg_default_parameters(void);

/* chroma subsampling shorthands                   [ref: libgpujpeg/gpujpeg_common.h:234-278] */
typedef uint32_t gpujpeg_sampling_factor_t;
#define MK_SUBSAMPLING(h1, v1, h2, v2, h3, v3, h4, v4)                                               \
    ((h1) << 28U | (v1) << 24U | (h2) << 20U | (v2) << 16U | (h3) << 12U | (v3) << 8U | (h4) << 4U | \
     (v4) << 0U)
#define GPUJPEG_SUBSAMPLING_UNKNOWN 0U
#define GPUJPEG_SUBSAMPLING_4444 MK_SUBSAMPLING(1, 1, 1, 1, 1, 1, 1, 1)
#define GPUJPEG_SUBSAMPLING_444 MK_SUBSAMPLING(1, 1, 1, 1, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_440 MK_SUBSAMPLING(1, 2, 1, 1, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_422 MK_SUBSAMPLING(2, 1, 1, 1, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_420 MK_SUBSAMPLING(2, 2, 1, 1, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_411 MK_SUBSAMPLING(4, 1, 1, 1, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_410 MK_SUBSAMPLING(4, 2, 1, 1, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_400 MK_SUBSAMPLING(1, 1, 0, 0, 0, 0, 0, 0)
#define GPUJPEG_SUBSAMPLING_442 MK_SUBSAMPLING(1, 2, 1, 2, 1, 1, 0, 0)
#define GPUJPEG_SUBSAMPLING_421 MK_SUBSAMPLING(2, 2, 2, 1, 1, 1, 0, 0)
GPUJPEG_API void gpujpeg_parameters_chroma_subsampling(struct gpujpeg_parameters* param,
                                                       gpujpeg_sampling_factor_t subsampling);
GPUJPEG_API const char* gpujpeg_subsampling_get_name(
    int comp_count, const struct gpujpeg_component_sampling_factor* sampling_factor);
GPUJPEG_API gpujpeg_sampling_factor_t gpujpeg_subsampling_from_name(const char* subsampling);

/* raw image description                           [ref: libgpujpeg/gpujpeg_common.h:280-310] */
struct gpujpeg_image_parameters {
    int width;
    int height;
    enum gpujpeg_color_space color_space;
    enum gpujpeg_pixel_format pixel_format;
    int width_padding; /* bytes appended to every row */
};
GPUJPEG_API void gpujpeg_image_set_default_parameters(struct gpujpeg_image_parameters* param);
GPUJPEG_API struct gpujpeg_image_parameters gpujpeg_default_image_parameters(void);

/* file formats known to the helper I/O            [ref: libgpujpeg/gpujpeg_common.h:312-360] */
enum gpujpeg_image_file_format {
    GPUJPEG_IMAGE_FILE_UNKNOWN = 0,
    GPUJPEG_IMAGE_FILE_JPEG = 1,
    GPUJPEG_IMAGE_FILE_RAW = 2,
    GPUJPEG_IMAGE_FILE_GRAY,
    GPUJPEG_IMAGE_FILE_RGB,
    GPUJPEG_IMAGE_FILE_RGBA,
    GPUJPEG_IMAGE_FILE_BMP,
    GPUJPEG_IMAGE_FILE_GIF,
    GPUJPEG_IMAGE_FILE_PNG,
    GPUJPEG_IMAGE_FILE_TGA,
    GPUJPEG_IMAGE_FILE_PGM,
    GPUJPEG_IMAGE_FILE_PPM,
    GPUJPEG_IMAGE_FILE_PNM,
    GPUJPEG_IMAGE_FILE_PAM,
    GPUJPEG_IMAGE_FILE_Y4M,
    GPUJPEG_IMAGE_FILE_YUV,
    GPUJPEG_IMAGE_FILE_YUVA,
    GPUJPEG_IMAGE_FILE_UYVY,
    GPUJPEG_IMAGE_FILE_I420,
    GPUJPEG_IMAGE_FILE_TST
};
#define GPUJPEG_IMAGE_FORMAT_IS_RAW(format) ((format) >= GPUJPEG_IMAGE_FILE_RAW)

/* per-stage timing, milliseconds                  [ref: libgpujpeg/gpujpeg_common.h:365-375] */
struct gpujpeg_duration_stats {
    double duration_memory_to;
    double duration_memory_from;
    double duration_memory_map;
    double duration_memory_unmap;
    double duration_preprocessor;
    double duration_dct_quantization;
    double duration_huffman_coder;
    double duration_stream;
    double duration_in_gpu;
};

/* image helpers                                   [ref: libgpujpeg/gpujpeg_common.h:377-470] */
GPUJPEG_API enum gpujpeg_image_file_format gpujpeg_image_get_file_format(const char* filename);
GPUJPEG_API void gpujpeg_set_device(int index);
GPUJPEG_API size_t gpujpeg_image_calculate_size(struct gpujpeg_image_parameters* param);
GPUJPEG_API int gpujpeg_image_load_from_file(const char* filename, uint8_t** image, size_t* image_size);
GPUJPEG_API int gpujpeg_image_save_to_file(const char* filename, const uint8_t* image, size_t image_size,
                                           const struct gpujpeg_image_parameters* param_image);
GPUJPEG_API int gpujpeg_image_get_properties(const char* filename,
                                             struct gpujpeg_image_parameters* param_image, int file_exists);
GPUJPEG_API int gpujpeg_image_destroy(uint8_t* image);
GPUJPEG_API void gpujpeg_image_range_info(const char* filename, int width, int height,
                                          enum gpujpeg_pixel_format sampling_factor);
GPUJPEG_API int gpujpeg_image_convert(const char* input, const char* output,
                                      struct gpujpeg_image_parameters param_image_from,
                                      struct gpujpeg_image_parameters param_image_to);

/* OpenGL interop: present for link compatibility; this build has no GL, so
 * gpujpeg_opengl_init() returns -2 exactly as the reference built without GL.
 *                                                 [ref: libgpujpeg/gpujpeg_common.h:472-640] */
struct gpujpeg_opengl_context;
GPUJPEG_API int gpujpeg_opengl_init(struct gpujpeg_opengl_context** ctx);
GPUJPEG_API void gpujpeg_opengl_destroy(struct gpujpeg_opengl_context*);
GPUJPEG_API int gpujpeg_opengl_texture_create(int width, int height, uint8_t* data);
GPUJPEG_API int gpujpeg_opengl_texture_set_data(int texture_id, uint8_t* data);
GPUJPEG_API int gpujpeg_opengl_texture_get_data(int texture_id, uint8_t* data, size_t* data_size);
GPUJPEG_API void gpujpeg_opengl_texture_destroy(int texture_id);
enum gpujpeg_opengl_texture_type { GPUJPEG_OPENGL_TEXTURE_READ = 1, GPUJPEG_OPENGL_TEXTURE_WRITE = 2 };
struct gpujpeg_opengl_texture {
    int texture_id;
    enum gpujpeg_opengl_texture_type texture_type;
    int texture_width;
    int texture_height;
    int texture_pbo_type;
    int texture_pbo_id;
    struct cudaGraphicsResource* texture_pbo_resource;
    void* texture_callback_param;
    void (*texture_callback_attach_opengl)(void* param);
    void (*texture_callback_detach_opengl)(void* param);
};
GPUJPEG_API struct gpujpeg_opengl_texture* gpujpeg_opengl_texture_register(
    int texture_id, enum gpujpeg_opengl_texture_type texture_type);
GPUJPEG_API void gpujpeg_opengl_texture_unregister(struct gpujpeg_opengl_texture* texture);
GPUJPEG_API uint8_t* gpujpeg_opengl_texture_map(struct gpujpeg_opengl_texture* texture, size_t* data_size);
GPUJPEG_API void gpujpeg_opengl_texture_unmap(struct gpujpeg_opengl_texture* texture);

/* name tables                                     [ref: libgpujpeg/gpujpeg_common.h:642-691] */
GPUJPEG_API const char* gpujpeg_color_space_get_name(enum gpujpeg_color_space color_space);
GPUJPEG_API enum gpujpeg_pixel_format gpujpeg_pixel_format_by_name(const char* name);
GPUJPEG_API enum gpujpeg_header_type gpujpeg_header_type_by_name(const char* name);
GPUJPEG_API const char* gpujpeg_header_type_get_name(enum gpujpeg_header_type header_type);
GPUJPEG_API void gpujpeg_print_pixel_formats(void);
GPUJPEG_API enum gpujpeg_color_space gpujpeg_color_space_by_name(const char* name);
GPUJPEG_API int gpujpeg_pixel_format_get_comp_count(enum gpujpeg_pixel_format pixel_format);
GPUJPEG_API const char* gpujpeg_pixel_format_get_name(enum gpujpeg_pixel_format pixel_format);
GPUJPEG_API int gpujpeg_pixel_format_is_planar(enum gpujpeg_pixel_format pixel_format);
GPUJPEG_API void gpujpeg_device_reset(void);
GPUJPEG_API const char* gpujpeg_orientation_get_name(struct gpujpeg_orientation orientation);

/* ------------------------------------------------------------------------- */
/* ENCODER                                         [ref: libgpujpeg/gpujpeg_encoder.h:44-267] */
struct gpujpeg_encoder; /* opaque */

enum gpujpeg_encoder_input_type {
    GPUJPEG_ENCODER_INPUT_IMAGE,           /* host pointer  */
    GPUJPEG_ENCODER_INPUT_OPENGL_TEXTURE,  /* not supported in this build */
    GPUJPEG_ENCODER_INPUT_GPU_IMAGE        /* device pointer */
};
struct gpujpeg_encoder_input {
    enum gpujpeg_encoder_input_type type;
    uint8_t* image;
    struct gpujpeg_opengl_texture* texture;
};
/* [ref: libgpujpeg/gpujpeg_encoder.h:78-131] */
GPUJPEG_API void gpujpeg_encoder_input_set_image(struct gpujpeg_encoder_input* input, uint8_t* image);
GPUJPEG_API void gpujpeg_encoder_input_set_gpu_image(struct gpujpeg_encoder_input* input, uint8_t* image);
GPUJPEG_API void gpujpeg_encoder_input_set_texture(struct gpujpeg_encoder_input* input,
                                                   struct gpujpeg_opengl_texture* texture);
GPUJPEG_API struct gpujpeg_encoder_input gpujpeg_encoder_input_image(uint8_t* image);
GPUJPEG_API struct gpujpeg_encoder_input gpujpeg_encoder_input_gpu_image(uint8_t* image);
GPUJPEG_API struct gpujpeg_encoder_input gpujpeg_encoder_input_texture(struct gpujpeg_opengl_texture* texture);

/* [ref: libgpujpeg/gpujpeg_encoder.h:133-142] one encoder = one device (current at create) + one stream */
GPUJPEG_API struct gpujpeg_encoder* gpujpeg_encoder_create(cudaStream_t stream);
/* [ref: libgpujpeg/gpujpeg_encoder.h:144-161] */
GPUJPEG_API size_t gpujpeg_encoder_max_pixels(struct gpujpeg_parameters* param,
                                              struct gpujpeg_image_parameters* param_image,
                                              enum gpujpeg_encoder_input_type image_input_type,
                                              size_t memory_size, int* max_pixels);
GPUJPEG_API size_t gpujpeg_encoder_max_memory(struct gpujpeg_parameters* param,
                                              struct gpujpeg_image_parameters* param_image,
                                              enum gpujpeg_encoder_input_type image_input_type,
                                              int max_pixels);
/* [ref: libgpujpeg/gpujpeg_encoder.h:163-174] */
GPUJPEG_API int gpujpeg_encoder_allocate(struct gpujpeg_encoder* encoder,
                                         const struct gpujpeg_parameters* param,
                                         const struct gpujpeg_image_parameters* param_image,
                                         enum gpujpeg_encoder_input_type image_input_type);
/* [ref: libgpujpeg/gpujpeg_encoder.h:176-193; impl src/gpujpeg_encoder.c:351-646]
 * Blocks until the JPEG is complete in host memory.  *image_compressed points
 * into an encoder-owned buffer valid until the next encode/destroy. */
GPUJPEG_API int gpujpeg_encoder_encode(struct gpujpeg_encoder* encoder,
                                       const struct gpujpeg_parameters* param,
                                       const struct gpujpeg_image_parameters* param_image,
                                       const struct gpujpeg_encoder_input* input,
                                       uint8_t** image_compressed, size_t* image_compressed_size);
/* [ref: libgpujpeg/gpujpeg_encoder.h:195-215] */
GPUJPEG_DEPRECATED GPUJPEG_API int gpujpeg_encoder_get_stats(struct gpujpeg_encoder* encoder,
                                                             struct gpujpeg_duration_stats* stats);
GPUJPEG_DEPRECATED GPUJPEG_API void gpujpeg_encoder_set_jpeg_header(struct gpujpeg_encoder* encoder,
                                                                    enum gpujpeg_header_type header_type);
/* [ref: libgpujpeg/gpujpeg_encoder.h:217-228; impl src/gpujpeg_encoder.c:290-317] */
GPUJPEG_API int gpujpeg_encoder_suggest_restart_interval(const struct gpujpeg_image_parameters* param_image,
                                                         gpujpeg_sampling_factor_t subsampling,
                                                         bool interleaved, int verbose);
/* string options                                  [ref: libgpujpeg/gpujpeg_encoder.h:230-253] */
#define GPUJPEG_ENCODER_OPT_OUT_PINNED "enc_out_pinned"
#define GPUJPEG_ENC_OPT_OUT "enc_opt_out"
#define GPUJPEG_ENC_OUT_VAL_PAGEABLE "enc_out_val_pageable"
#define GPUJPEG_ENC_OUT_VAL_PINNED "enc_out_val_pinned"
#define GPUJPEG_ENC_OPT_HDR "enc_hdr"
#define GPUJPEG_ENC_HDR_VAL_JFIF "JFIF"
#define GPUJPEG_ENC_HDR_VAL_EXIF "Exif"
#define GPUJPEG_ENC_HDR_VAL_ADOBE "Adobe"
#define GPUJPEG_ENC_HDR_VAL_SPIFF "SPIFF"
#define GPUJPEG_ENC_OPT_FLIPPED_BOOL "enc_opt_flipped"
#define GPUJPEG_ENC_OPT_EXIF_TAG "enc_exif_tag"
#define GPUJPEG_ENC_OPT_METADATA "enc_metadata"
#define GPUJPEG_ENC_OPT_CHANNEL_REMAP "enc_opt_channel_remap"
GPUJPEG_API int gpujpeg_encoder_set_option(struct gpujpeg_encoder* encoder, const char* opt, const char* val);
GPUJPEG_API void gpujpeg_encoder_print_options(void);
GPUJPEG_API int gpujpeg_encoder_destroy(struct gpujpeg_encoder* encoder);

/* ------------------------------------------------------------------------- */
/* DECODER                                         [ref: libgpujpeg/gpujpeg_decoder.h:46-320] */
struct gpujpeg_decoder; /* opaque */

enum gpujpeg_decoder_output_type {
    GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER,    /* decoder-owned pinned host buffer */
    GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER,      /* caller-owned host buffer         */
    GPUJPEG_DECODER_OUTPUT_OPENGL_TEXTURE,     /* not supported in this build      */
    GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER,        /* decoder-owned device buffer      */
    GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER  /* caller-owned device buffer       */
};
struct gpujpeg_decoder_output {
    enum gpujpeg_decoder_output_type type;
    uint8_t* data;
    size_t data_size;
    struct gpujpeg_image_parameters param_image;
    struct gpujpeg_opengl_texture* texture;
    const struct gpujpeg_image_metadata* metadata;
};
struct gpujpeg_decoder_init_parameters {
    cudaStream_t stream;
    int verbose;
    bool perf_stats;
    bool ff_cs_itu601_is_709;
};
/* [ref: libgpujpeg/gpujpeg_decoder.h:96-141] */
GPUJPEG_API void gpujpeg_decoder_output_set_default(struct gpujpeg_decoder_output* output);
GPUJPEG_API void gpujpeg_decoder_output_set_custom(struct gpujpeg_decoder_output* output, uint8_t* custom_buffer);
GPUJPEG_API void gpujpeg_decoder_output_set_texture(struct gpujpeg_decoder_output* output,
                                                    struct gpujpeg_opengl_texture* texture);
GPUJPEG_API void gpujpeg_decoder_output_set_cuda_buffer(struct gpujpeg_decoder_output* output);
GPUJPEG_API void gpujpeg_decoder_output_set_custom_cuda(struct gpujpeg_decoder_output* output,
                                                        uint8_t* d_custom_buffer);
/* [ref: libgpujpeg/gpujpeg_decoder.h:143-170] */
GPUJPEG_API struct gpujpeg_decoder* gpujpeg_decoder_create(cudaStream_t stream);
GPUJPEG_API struct gpujpeg_decoder_init_parameters gpujpeg_decoder_default_init_parameters(void);
GPUJPEG_API struct gpujpeg_decoder* gpujpeg_decoder_create_with_params(
    const struct gpujpeg_decoder_init_parameters* params);
/* [ref: libgpujpeg/gpujpeg_decoder.h:172-188; impl src/gpujpeg_decoder.c:184-231] */
GPUJPEG_API int gpujpeg_decoder_init(struct gpujpeg_decoder* decoder, const struct gpujpeg_parameters* param,
                                     const struct gpujpeg_image_parameters* param_image);
/* [ref: libgpujpeg/gpujpeg_decoder.h:190-204; impl src/gpujpeg_decoder.c:234-469] */
GPUJPEG_API int gpujpeg_decoder_decode(struct gpujpeg_decoder* decoder, uint8_t* image, size_t image_size,
                                       struct gpujpeg_decoder_output* output);
GPUJPEG_DEPRECATED GPUJPEG_API int gpujpeg_decoder_get_stats(struct gpujpeg_decoder* decoder,
                                                             struct gpujpeg_duration_stats* stats);
GPUJPEG_API int gpujpeg_decoder_destroy(struct gpujpeg_decoder* decoder);

/* pseudo pixel formats / colour spaces for set_output_format   [ref: libgpujpeg/gpujpeg_decoder.h:222-249] */
#define GPUJPEG_PIXFMT_AUTODETECT ((enum gpujpeg_pixel_format)(GPUJPEG_PIXFMT_NONE - 1))
#define GPUJPEG_PIXFMT_NO_ALPHA ((enum gpujpeg_pixel_format)(GPUJPEG_PIXFMT_NONE - 2))
#define GPUJPEG_PIXFMT_STD ((enum gpujpeg_pixel_format)(GPUJPEG_PIXFMT_NONE - 3))
#define GPUJPEG_PIXFMT_NATIVE ((enum gpujpeg_pixel_format)(GPUJPEG_PIXFMT_NONE - 4))
#define GPUJPEG_CS_DEFAULT ((enum gpujpeg_color_space)(GPUJPEG_NONE - 1))
GPUJPEG_API void gpujpeg_decoder_set_output_format(struct gpujpeg_decoder* decoder,
                                                   enum gpujpeg_color_space color_space,
                                                   enum gpujpeg_pixel_format pixel_format);

/* stream probing                                  [ref: libgpujpeg/gpujpeg_decoder.h:251-291] */
enum { GPUJPEG_COUNT_SEG_COUNT_REQ = 1 << 0 };
struct gpujpeg_image_info {
    union {
        struct {
            struct gpujpeg_image_parameters param_image;
            struct gpujpeg_parameters param;
            int segment_count;
            enum gpujpeg_header_type header_type;
            const char* comment;
            struct gpujpeg_image_metadata metadata;
        };
        char reserved[512];
    };
};
GPUJPEG_API int gpujpeg_decoder_get_image_info2(uint8_t* image, size_t image_size,
                                                struct gpujpeg_image_info* info, int verbose, unsigned flags);
GPUJPEG_API int gpujpeg_decoder_get_image_info(uint8_t* image, size_t image_size,
                                               struct gpujpeg_image_parameters* param_image,
                                               struct gpujpeg_parameters* param, int* segment_count);

/* string options                                  [ref: libgpujpeg/gpujpeg_decoder.h:293-314] */
#define GPUJPEG_DEC_OPT_TGA_RLE_BOOL "dec_opt_tga_rle"
#define GPUJPEG_DEC_OPT_FLIPPED_BOOL "dec_opt_flipped"
#define GPUJPEG_DEC_OPT_CHANNEL_REMAP "dec_opt_channel_remap"
#define GPUJPEG_DEC_OPT_ALIGNMENT_BYTES_INT "dec_opt_alignment_bytes"
/* Extension of this build (not in the reference): selects which inverse DCT the
 * decoder runs.  "int" (default) is bit-exact with the reference's
 * gpujpeg_idct_cpu [src/gpujpeg_dct_cpu.c:55-189]; "float_gpuref" reproduces the
 * float lifting IDCT of the reference CUDA kernel [src/gpujpeg_dct_gpu.cu:312-363]. */
#define GPUJPEG_DEC_OPT_IDCT "dec_opt_idct"
#define GPUJPEG_DEC_IDCT_VAL_INT "int"
#define GPUJPEG_DEC_IDCT_VAL_FLOAT_GPUREF "float_gpuref"
/* extension: which Huffman decoder kernel runs.  "auto" (default): several lanes per restart segment, self-synchronising,
 * for segments of at most 40 blocks, one thread per segment otherwise; "thread_per_segment": always the latter */
#define GPUJPEG_DEC_OPT_HUFFMAN "dec_opt_huffman"
#define GPUJPEG_DEC_HUFFMAN_VAL_AUTO "auto"
#define GPUJPEG_DEC_HUFFMAN_VAL_THREAD_PER_SEGMENT "thread_per_segment"
/* extension (tuning): lanes that share one restart segment in the self-synchronising decoder: 0 = chosen per scan from
 * the scan's bytes per segment (default), or 4, 8, 16, 32 for every scan */
#define GPUJPEG_DEC_OPT_HUFFMAN_LANES "dec_opt_huffman_lanes"
GPUJPEG_API int gpujpeg_decoder_set_option(struct gpujpeg_decoder* decoder, const char* opt, const char* val);
GPUJPEG_API void gpujpeg_decoder_print_options(void);

#ifdef __cplusplus
}
#endif
#endif /* GPUJPEG_B200_H_ABI */
