/*
 * gj_internal.h -- internal structures of the H100-native libgpujpeg replacement.
 *
 * Host code is plain C (north_star: "host code stays C calling into a thin C-ABI layer of
 * hand-written sm_90a CUDA kernels").  The stage launchers at the bottom are that thin layer:
 * extern "C", plain pointers and sizes, implemented in the .cu files.
 *
 * Data layout in HBM (see DESIGN.md section 3):
 *   raw      u8   RGB interleaved, row pitch 3*W+padding                      (3 B/pixel)
 *   coef     i16  [comp][block][64], blocks in raster order, coefficients in ZIG-ZAG order
 *                 (the reference keeps natural order, src/gpujpeg_dct_gpu.cu:286-293; zig-zag is
 *                 free for the producer here and removes the gather from both Huffman kernels)
 *   scan tmp u8   one fixed-stride slot per restart segment (encoder only)
 *   stream   u8   the finished JPEG byte stream (encoder) / the input file bytes (decoder)
 */
#ifndef GJ_INTERNAL_H
#define GJ_INTERNAL_H

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/gpujpeg_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define GJ_MAX_COMP 4
#define GJ_SOS_LEN_1 10 /* bytes of an SOS header with one component */

/* ---- logging [ref: src/gpujpeg_common_internal.h:125-150] ---- */
#define GJ_ERR(...) (void)(fprintf(stderr, "[GPUJPEG] [Error] " __VA_ARGS__))
#define GJ_WARN(...) (void)(fprintf(stderr, "[GPUJPEG] [Warning] " __VA_ARGS__))
#define GJ_VERBOSE(v, ...) do { if ( (v) >= GPUJPEG_LL_VERBOSE ) (void)fprintf(stderr, "[GPUJPEG] [Verbose] " __VA_ARGS__); } while ( 0 )
#define GJ_DEBUG(v, ...) do { if ( (v) >= GPUJPEG_LL_DEBUG ) (void)fprintf(stderr, "[GPUJPEG] [Debug] " __VA_ARGS__); } while ( 0 )

/* ---- tables (gj_tables.c) ---- */
extern const uint8_t gj_zigzag_to_natural[64];
extern const uint8_t gj_natural_to_zigzag[64];

/* Huffman specification as carried by a DHT marker */
struct gj_huff_spec {
    uint8_t bits[17]; /* bits[1..16] */
    uint8_t vals[256];
    int nvals;
};
void gj_huff_spec_default(int cls /*0 lum,1 chroma*/, int kind /*0 DC,1 AC*/, struct gj_huff_spec* spec);
/* the table T.81 Annex K.2 fits to a symbol histogram, byte for byte what libjpeg's optimize_coding writes (enc_opt_huffman) */
void gj_huff_spec_optimal(const uint64_t freq[256], struct gj_huff_spec* spec);

/* quantisation: raw zig-zag u8 table for a quality [ref: src/gpujpeg_table.c:83-99] */
void gj_quant_raw(int cls, int quality, uint8_t raw_zz[64]);
/* forward table in ZIG-ZAG coefficient order: fwd_zz[k] = 1/(raw[k]*aan[x]*aan[y]*8) as float
 * (same values as the reference's transposed table, src/gpujpeg_table.c:112-120, re-indexed) */
void gj_quant_forward_zz(const uint8_t raw_zz[64], float fwd_zz[64]);

/* Encoder LUTs for the device: per table set (0 = luminance, 1 = chrominance)
 *   ac[sym]  = (code << 5) | len   (len 0 = symbol has no code)
 *   dc[cat]  = (code << 5) | len */
struct gj_enc_lut {
    uint32_t ac[256];
    uint32_t dc[16];
};
void gj_enc_lut_build(const struct gj_huff_spec* dc, const struct gj_huff_spec* ac, struct gj_enc_lut* lut);

/* Decoder LUT for the device, one per (class, id):
 *   look[peek9] = (symbol << 4) | len for codes of length <= 9, 0 if longer
 *   maxcode[l]  = exclusive upper bound of all codes of length <= l, left-justified to 16 bits
 *   valoff[l]   = valptr[l] - mincode[l]
 *   vals[]      = HUFFVAL
 * (a two-level table and a cp.async staging ring were measured as well: both lengthen the
 * per-warp instruction stream, which is what bounds the decoder, and lost against this variant) */
#define GJ_DEC_LOOK_BITS 9
struct gj_dec_lut {
    uint16_t look[1 << GJ_DEC_LOOK_BITS];
    uint32_t maxcode[18];
    int32_t valoff[18];
    uint8_t vals[256];
};
int gj_dec_lut_build(const struct gj_huff_spec* spec, struct gj_dec_lut* lut);

/* Fast decoder table, one per (class, id), indexed by the next GJ_DEC_FAST_BITS bits of the stream.  One entry tells
 * the decoder everything it needs to step over a symbol AND its value bits:
 *   bits  0-6   advance of the zig-zag index: DC 1; AC run + 1, ZRL 16, EOB (and the invalid run/0 symbols) 64
 *   bits  7-11  code length + value size (bits to consume), never 0 for a code
 *   bits 16-19  value size
 * so that a decoder which keeps its state as (zig-zag index | bit position << 7) advances it with ONE addition of the
 * entry's low half (a 16-bit load of it for a walk that does not need the value).
 * Codes longer than GJ_DEC_FAST_BITS: the entry of their 10-bit prefix has bits 7-11 == 0 and names a second-level
 * table (bits 0-6 = its number + 1) indexed by the following 16 - GJ_DEC_FAST_BITS bits, same entry format; the
 * standard tables need 4 of them.  0 = no such code / more prefixes than second-level tables: canonical search in
 * gj_dec_lut. */
#define GJ_DEC_FAST_BITS 10
#define GJ_DEC_FAST_SUBS 8
#define GJ_DEC_FAST_TOTAL_SHIFT 7
#define GJ_DEC_FAST_TOTAL_MASK (31u << GJ_DEC_FAST_TOTAL_SHIFT)
#define GJ_DEC_FAST_SIZE_SHIFT 16
struct gj_dec_fast {
    uint32_t e[1 << GJ_DEC_FAST_BITS];
    uint32_t sub[GJ_DEC_FAST_SUBS][1 << (16 - GJ_DEC_FAST_BITS)];
};
void gj_dec_fast_build(const struct gj_huff_spec* spec, int is_ac, struct gj_dec_fast* fast);

/* ---- geometry (gj_codestream.c)  [ref: src/gpujpeg_common.c:628-1106] ---- */
#define GJ_MAX_MCU_BLOCKS 10  /* T.81 B.2.3: at most 10 data units per MCU */

/* one component's plane of 8x8 blocks [ref: src/gpujpeg_common.c:671-736] */
struct gj_comp_geo {
    int hs, vs;         /* sampling factors as in SOF0 */
    int width, height;  /* samples that carry image data */
    int bcx, bcy;       /* block grid (interleaved: padded to whole MCUs) */
    int nblk;           /* bcx * bcy */
    int blk_off;        /* index of the component's first block in the coefficient / mask buffers */
};

/* What the entropy kernels need to turn "block number j of segment s of scan k" into a block index; passed to
 * K2/K3 by value.  For the 4:4:4 case (`simple`) they keep the closed form comp * nblk + first_mcu + mcu. */
struct gj_scan_layout {
    int simple;               /* every component 1x1: MCU index == block index in every plane */
    int interleaved;
    int comp_count;
    int scan_count;
    int bpm;                  /* blocks per MCU of an interleaved scan (1 otherwise) */
    int mcu_x;                /* MCUs per MCU row (interleaved) */
    int blk_off[GJ_MAX_COMP];
    int bcx[GJ_MAX_COMP];
    int scan_seg_begin[GJ_MAX_COMP + 1];  /* first global segment of scan k; entries >= scan_count hold seg_count */
    int scan_mcus[GJ_MAX_COMP];           /* MCUs of scan k */
    /* interleaved MCU, block i in coding order [ref: src/gpujpeg_common.c:1062-1084]:
     * component, block offset inside the MCU, distance (in blocks of the scan) to the previous block of the
     * same component = the DC predictor */
    uint8_t idx_comp[GJ_MAX_MCU_BLOCKS], idx_dx[GJ_MAX_MCU_BLOCKS], idx_dy[GJ_MAX_MCU_BLOCKS], idx_pred[GJ_MAX_MCU_BLOCKS];
    uint8_t comp_hs[GJ_MAX_COMP], comp_vs[GJ_MAX_COMP];
    uint8_t comp_tbl[GJ_MAX_COMP];   /* quantisation / Huffman table class of the component: 0 luminance, 1 chrominance */
};

struct gj_geometry {
    int width, height, comp_count;
    int pitch;            /* bytes per raw row */
    int data_width, data_height;
    int bcx, bcy, nblk;   /* 8x8 blocks of component 0 */
    int interleaved;
    int restart_interval; /* as given (0 = none) */
    int seg_mcu;          /* MCUs per segment (restart_interval or all) */
    int scan_count;
    int comps_per_scan;   /* 1 (non-interleaved) or comp_count */
    int seg_per_scan;     /* segments of scan 0 (all scans when `lay.simple`) */
    int seg_count;        /* all scans */
    int max_hs, max_vs;   /* MCU size in blocks of the full-resolution plane */
    int subsampled;       /* some component has fewer samples than the image */
    struct gj_comp_geo comp[GJ_MAX_COMP];
    struct gj_scan_layout lay;
    size_t raw_size;      /* bytes of the raw image */
    size_t coef_count;    /* int16 coefficients, all components */
    size_t slot_stride;   /* bytes reserved per segment in the encoder's scan tmp buffer */
    size_t stream_cap;    /* capacity of the finished stream buffer */
};
/* Where the samples of component c live in a raw image of a given pixel format [ref: src/gpujpeg_preprocessor.cu:78-160
 * (loads per format), :409-455 (planar copy)]: sample (x, y) is the byte at off + y * pitch + x * xs. */
struct gj_raw_comp {
    size_t off;
    size_t pitch;
    int xs;
};
struct gj_raw_layout {
    int comp_count;
    struct gj_raw_comp comp[GJ_MAX_COMP];
    struct gpujpeg_component_sampling_factor sampling[GJ_MAX_COMP];  /* the format's own sampling */
    size_t size;   /* bytes of the whole image */
    int alpha_off; /* 4444-u8-p0123: byte offset of the alpha sample inside a pixel (ignored on input, 255 on output); 0 = none */
};
/* 0 on success, -1 for a format/size combination this build does not take */
int gj_raw_layout_init(struct gj_raw_layout* l, const struct gpujpeg_image_parameters* pi);

int gj_geometry_init(struct gj_geometry* g, const struct gpujpeg_parameters* param,
                     const struct gpujpeg_image_parameters* param_image);

/* dec_opt_crop: the blocks of every component plane that an output rectangle needs -- columns [bx0, bx1), rows [by0, by1).
 * Output pixel (x, y) reads component c at sample (x / (max_hs / hs), y / (max_vs / vs)), n samples per block side (8, or
 * 8 / scale for a scaled decode). */
struct gj_blk_rect {
    int bx0, by0, bx1, by1;
};
void gj_crop_blocks(const struct gj_geometry* g, int n, int x, int y, int w, int h, struct gj_blk_rect win[GJ_MAX_COMP]);
/* dec_opt_pixels=libjpeg: fancy upsampling reads one chroma sample on every side of the one under a pixel, so the blocks a
 * rectangle needs are those of r = {x, y, w, h} widened by max_hs pixels and max_vs rows, clamped to the width x height image
 * (in place) */
void gj_crop_widen(int width, int height, int max_hs, int max_vs, int r[4]);
/* The restart segments of a scan that hold a unit (MCU) of the rectangle [ux0, ux1) x [uy0, uy1) of its units_x-wide unit
 * grid, seg_units units per segment, bpm blocks per unit: pairs {seg_base + segment, blocks to decode} in ascending order,
 * the block count reaching up to and including the segment's last needed unit.  Returns the number of pairs. */
int gj_crop_pick_units(int units_x, int units, int seg_units, int bpm, int ux0, int uy0, int ux1, int uy1, int seg_base,
                       uint32_t* out);
/* the pick list of baseline scan k (pairs as above, global segment numbers), from the blocks gj_crop_blocks gave */
int gj_crop_pick(const struct gj_geometry* g, int k, const struct gj_blk_rect win[GJ_MAX_COMP], uint32_t* out);

/* dec_opt_orientation: the output pixel (ox, oy) -- counted from the output rectangle's origin -- shows the source pixel
 * (sxx * ox + sxy * oy + sx0, syx * ox + syy * oy + sy0) of the unoriented (scaled) image; o.. is the inverse map, from a source
 * pixel to its output pixel.  The matrices are signed permutations. */
struct gj_orient_map {
    int sxx, sxy, sx0, syx, syy, sy0;
    int oxx, oxy, ox0, oyx, oyy, oy0;
};
/* value of dec_opt_orientation: "none" -> mode 0, "auto" -> mode 1, "<deg>[-]" (0, 90, 180, 270; '-' = mirrored) -> mode 2 with
 * rot = deg / 90 and flip; 0 on success */
int gj_parse_orientation(const char* val, int* mode, int* rot, int* flip);
/* value of dec_opt_crop / tran_opt_crop other than "none": djpeg's -crop syntax "WxH+X+Y", decimal, v = {W, H, X, Y} with W, H >= 1;
 * 0 on success */
int gj_parse_crop(const char* val, int v[4]);
/* The w x h image turned rot quarter turns clockwise, then mirrored horizontally if flip: its size *ow x *oh; the map of the
 * rectangle crop = {x, y, w, h} of it (NULL: all of it) and src = {x, y, w, h}, the rectangle of the w x h image it shows.
 * Returns -1 (and leaves the outputs alone) if crop does not lie inside the oriented image. */
int gj_orient_frame(int w, int h, int rot, int flip, const int* crop, int* ow, int* oh, struct gj_orient_map* m, int src[4]);

/* The transcoder's lossless turn / mirror (gj_transcoder.c, k_coef_transform).  Output block (bx, by) of component c shows the
 * source block (sx, sy) = (axx * bx + axy * by + ax0, ayx * bx + ayy * by + ay0) of the same component when that lies in the
 * source's src_bcx x src_bcy block grid of c; otherwise it is a dummy block, whose DC is that of the output block
 * (min(bx, vis_bx - 1), min(by, vis_by - 1)) and whose AC coefficients are zero.  Coefficient signs and the transpose follow
 * gj_coef_src (gj_device.cuh): transpose = output x runs along source y, neg_x / neg_y = the source's x / y axis is reversed. */
struct gj_blk_map {
    int axx, axy, ax0, ayx, ayy, ay0;
    int src_bcx, src_bcy;              /* the source's block grid of the component */
    int out_bcx, out_bcy;              /* the output's */
    int vis_bx, vis_by;                /* output blocks [0, vis_bx) x [0, vis_by) show source blocks */
};
struct gj_transcode_plan {
    int width, height;                 /* the output */
    int hs[GJ_MAX_COMP], vs[GJ_MAX_COMP];
    int transpose, neg_x, neg_y;
    int src_w, src_h;                  /* the source after the trim */
    struct gj_blk_map blk[GJ_MAX_COMP];
};
/* A w x h source of comp_count components with sampling hs / vs, its block grids those of gj_geometry_init (interleaved or not),
 * turned rot quarter turns clockwise, then mirrored horizontally if flip, into an output of the same interleaving flag
 * out_interleaved.  Without perfect, partial edge iMCUs that would move are dropped; with it such a frame is refused, as is a
 * frame trimmed to nothing.  Returns 0, or -1 with the reason in why (GJ_WHY_BYTES). */
#define GJ_WHY_BYTES 160
int gj_transcode_plan(int w, int h, int comp_count, const int* hs, const int* vs, int src_interleaved, int out_interleaved, int rot,
                      int flip, int perfect, struct gj_transcode_plan* plan, char* why);
/* tran_opt_crop (jpegtran -crop with -trim): the plan `full` of a w x h source (gj_transcode_plan's output) cut to the rectangle
 * rect = {x, y, w, h} of the transformed image.  Refused unless the rectangle lies inside the untrimmed transformed image; its
 * origin is rounded down to the output's iMCU grid, and refused if that lies in the strip the trim drops; the output reaches to
 * the rectangle's far edge, clipped to full's output.  Every component's block map is full's, shifted by the origin's blocks,
 * over the smaller output grid.  Returns 0, or -1 with the reason in why (GJ_WHY_BYTES). */
int gj_transcode_crop(const struct gj_transcode_plan* full, int w, int h, int comp_count, int out_interleaved, const int rect[4],
                      struct gj_transcode_plan* plan, char* why);
/* the source blocks the block maps of plan read (dummy blocks read their clamped neighbours), per component */
void gj_transcode_window(const struct gj_transcode_plan* plan, int comp_count, struct gj_blk_rect win[GJ_MAX_COMP]);
/* the COM segments of a JPEG file in front of its first SOS, markers included, copied to out (NULL: size only); their size */
size_t gj_com_segments(const uint8_t* data, size_t size, uint8_t* out);

/* ---- codestream writer (gj_writer.c)  [ref: src/gpujpeg_writer.c] ---- */
/* what a header may carry besides the coding parameters: orientation (SPIFF directory entry / Exif tag) and user Exif tags */
struct gj_exif_tags;
struct gj_header_extras {
    struct gpujpeg_image_metadata metadata;
    const struct gj_exif_tags* exif_tags;
    /* the transcoder: component c's quantisation table (zig-zag) and its table id, in place of raw_q by class (NULL: raw_q) */
    const uint8_t (*comp_q)[64];
    const uint8_t* comp_tq;
    /* whole COM segments (markers included) that replace the writer's own comments; NULL: the writer's */
    const uint8_t* com;
    size_t com_size;
    int libjpeg;   /* enc_opt_writer=libjpeg: the header libjpeg-turbo writes for a JFIF frame (gj_write_header) */
};
#define GJ_HEADER_BASE_CAP 1024   /* bytes a header needs at most without user Exif tags */
size_t gj_write_header(uint8_t* out, const struct gpujpeg_parameters* param,
                       const struct gpujpeg_image_parameters* param_image, const uint8_t raw_q[2][64],
                       const struct gj_huff_spec spec[2][2], enum gpujpeg_header_type header_type,
                       const struct gj_header_extras* extras /* may be NULL */);
/* ---- Exif (gj_exif.c)  [ref: src/gpujpeg_exif.c] ---- */
int gj_exif_add_tag(struct gj_exif_tags** tags, const char* cfg);   /* enc_exif_tag option value; 0 on success */
void gj_exif_tags_destroy(struct gj_exif_tags* tags);
size_t gj_exif_tags_bytes(const struct gj_exif_tags* tags);          /* what the user tags add to the header, at most */
size_t gj_exif_write(uint8_t* out, const struct gpujpeg_parameters* param, const struct gpujpeg_image_parameters* pi,
                     const struct gpujpeg_image_metadata* metadata, const struct gj_exif_tags* tags);
void gj_exif_parse(const uint8_t* seg, size_t len, const uint8_t* file_end, int verbose, struct gpujpeg_image_metadata* metadata);
unsigned gj_exif_orientation_code(const struct gpujpeg_orientation* o);
size_t gj_write_sos(uint8_t* out, const struct gpujpeg_parameters* param, int scan_index);
/* APP13 "segment info" headers of a scan (the positions left zero) [ref: src/gpujpeg_writer.c:553-599]; out == NULL: size only */
#define GJ_SEGINFO_CHUNK (65536 - 100)   /* position bytes per header [ref: src/gpujpeg_common_internal.h:91] */
size_t gj_write_segment_info_headers(uint8_t* out, int scan_index, int segment_count);
/* where position number `index` of a scan's table lies, relative to the first header's first byte */
size_t gj_segment_info_entry_offset(int index);

/* ---- codestream reader (gj_reader.c)  [ref: src/gpujpeg_reader.c] ---- */
/* Scans a progressive (SOF2) frame may have: libjpeg's scripts use 6-10, hand-written ones rarely more than about 20.  A
 * baseline frame keeps its limit of GJ_MAX_COMP scans. */
#define GJ_MAX_SCANS 64
struct gj_scan_info {
    int ncomp;
    int comp[GJ_MAX_COMP];
    int td[GJ_MAX_COMP], ta[GJ_MAX_COMP];
    int ss, se, ah, al;   /* spectral selection and successive approximation (T.81 B.2.3); baseline: 0, 63, 0, 0 */
    /* progressive frames: file offset of the DHT entry (its Tc/Th byte) in force at the SOS for the table component k of
     * the scan uses -- DC for a DC-first scan, AC for an AC scan --, 0 = no such table was defined (a DC refinement uses none) */
    size_t huff_at[GJ_MAX_COMP];
    size_t begin, end; /* entropy-coded bytes [begin,end) in the file */
    int first_segment, segment_count;
};
/* the table a DHT entry at file offset `at` (as recorded in gj_scan_info.huff_at) defines; the walk has checked it */
void gj_huff_spec_at(const uint8_t* data, size_t at, struct gj_huff_spec* spec);
/* APP13 "segment info" headers met in front of a scan [ref: src/gpujpeg_reader.c:229-249]: pieces of one table of
 * big-endian 32-bit positions (every restart segment's first byte relative to the scan's first byte, then the scan's end) */
#define GJ_SEGINFO_MAX_PIECES 64
struct gj_seginfo {
    const uint8_t* piece[GJ_SEGINFO_MAX_PIECES];
    uint32_t piece_bytes[GJ_SEGINFO_MAX_PIECES];
    int pieces;
    size_t bytes;
};
struct gj_stream {
    int width, height, comp_count;
    int restart_interval;
    int comp_id[GJ_MAX_COMP], comp_hv[GJ_MAX_COMP], comp_tq[GJ_MAX_COMP];
    uint8_t qt[4][64];
    int have_qt[4];
    struct gj_huff_spec huff[2][4]; /* [class][id] */
    int have_huff[2][4];
    size_t huff_at[2][4];           /* file offset of the DHT entry that defined [class][id] */
    int progressive;                /* SOF2: Huffman-coded progressive DCT (T.81 Annex G) */
    /* progressive frames: per component and zig-zag coefficient, 1 + the Al of the last scan that coded it (0 = none yet),
     * as T.81 G.1.1.1.2 requires every refinement to continue; and the quantisation table latched at the component's first
     * scan (have_comp_qt) */
    uint8_t coef_bits[GJ_MAX_COMP][64];
    uint8_t comp_qt[GJ_MAX_COMP][64];
    int have_comp_qt[GJ_MAX_COMP];
    int scan_count;
    struct gj_scan_info scan[GJ_MAX_SCANS];
    struct gj_seginfo seginfo[GJ_MAX_COMP];   /* [scan]: the table in front of the scan's SOS, if any (baseline scans only) */
    struct gj_seginfo seginfo_pending;        /* headers met since the last SOS */
    enum gpujpeg_color_space color_space;
    int spiff_color_space;   /* colour space named by a SPIFF header, GPUJPEG_NONE (0) if there is none */
    int in_spiff_directory;  /* between the SPIFF header and its end-of-directory entry */
    int exif_seen;           /* an Exif APP1 header: the components are YCbCr JPEG whatever their ids say */
    int verbose;             /* in: log level of the reader's messages */
    struct gpujpeg_image_metadata metadata;   /* orientation from a SPIFF directory entry or an Exif header */
    int com_color_space;     /* colour space named by FFmpeg's COM "CS=ITU601", GPUJPEG_NONE (0) if there is none */
    int ff_cs_itu601_is_709; /* in: read that comment as BT.709 [ref: libgpujpeg/gpujpeg_decoder.h:95] */
    enum gpujpeg_header_type header_type;
    const char* comment;
    size_t header_size;
    int interleaved;
};
/* incremental pieces: begin, walk marker segments up to the next SOS, finish */
void gj_reader_begin(struct gj_stream* s, int ff_cs_itu601_is_709);
int gj_reader_walk(const uint8_t* data, size_t size, size_t* pos, struct gj_stream* s, int* adobe_transform);
int gj_reader_finish(struct gj_stream* s, int adobe_transform, int verbose);
enum gpujpeg_color_space gj_stream_color_space(const struct gj_stream* s, int adobe_transform);
/* parse all markers; does not split scans into segments */
int gj_reader_parse(const uint8_t* data, size_t size, struct gj_stream* s, int verbose);
/* split scan data at RSTn markers: fills seg_off/seg_len (file offsets of stuffed entropy bytes) */
int gj_reader_split(const uint8_t* data, struct gj_stream* s, uint32_t* seg_off, uint32_t* seg_len, int max_segments);

/* ---- image files (gj_imageio.c)  [ref: src/utils/image_delegate.c, src/utils/pam.c, src/utils/y4m.c] ---- */
enum { GJ_IMGFILE_PNM = 1, GJ_IMGFILE_PAM, GJ_IMGFILE_Y4M };
struct gj_imgfile {
    int kind;
    int width, height;
    int channels, maxval;              /* Netpbm */
    int subsampling, bitdepth, limited; /* Y4M: 400 / 420 / 422 / 444 / 4444 */
    size_t data_offset, data_bytes;    /* where the samples are in the file */
};
int gj_imgfile_probe(const char* filename, struct gj_imgfile* f);
int gj_imgfile_params(const char* filename, const struct gj_imgfile* f, struct gpujpeg_image_parameters* pi);
int gj_imgfile_load(const char* filename, uint8_t** image, size_t* image_size, void* (*alloc)(size_t));
int gj_imgfile_save_pam(const char* filename, const struct gpujpeg_image_parameters* pi, const uint8_t* data, int pnm);
int gj_imgfile_save_y4m(const char* filename, const struct gpujpeg_image_parameters* pi, const uint8_t* data);

/* ---- device side: the C-ABI stage launchers (implemented in *.cu) ---- */
typedef struct CUstream_st* gj_stream_t;

/* constant tables a coder instance keeps on the device */
struct gj_dev_enc_tables {
    float fwd_zz[2][64];      /* forward quant tables, zig-zag order */
    struct gj_enc_lut lut[2]; /* Huffman encoder LUTs */
};
struct gj_dev_dec_tables {
    uint16_t qinv_zz[4][64];  /* dequantisation tables by table id, zig-zag order */
    struct gj_dec_lut lut[2][4];
    struct gj_dec_fast fast[2][4];
};

/* K1, the transform stage: the input classes of the encoder (params_supported, gj_encoder.c) -- RGB u8 interleaved into a
 * YCbCr JPEG, a raw image that already holds the JPEG's components, any other pixel format / colour space through the generic
 * pass (gj_convert.cu) -- and the frame's options */
enum { GJ_IN_UNSUPPORTED = 0, GJ_IN_RGB = 1, GJ_IN_SAMPLES = 2, GJ_IN_GENERIC = 3 };
struct gj_k1_request {
    int in;                     /* GJ_IN_* */
    int libjpeg;                /* enc_opt_writer=libjpeg: libjpeg-turbo's coefficients */
    int flipped;                /* enc_opt_flipped */
    int channel_remap;          /* enc_opt_channel_remap is set */
    int coef_input;             /* the coefficients come from the transcoder: no K1 */
};
enum { GJ_K1_FUSED = 1, GJ_K1_BLOCKS = 2 };
enum { GJ_K1_FLIP_NONE = 0, GJ_K1_FLIP_PITCH = 1, GJ_K1_FLIP_PLANES = 2 };
#define GJ_FDCT_ISLOW 1         /* libjpeg's jpeg_fdct_islow and quantiser (k_fdct_libjpeg) */
/* Everything K1 does with a frame: the generic pass into the planes, the flip of the planes, then gj_launch_fdct_fused or
 * gj_launch_fdct_blocks (gj_encoder.c launch_k1) */
struct gj_k1_plan {
    int kernel;                 /* 0 (no K1), GJ_K1_FUSED (k_fdct_rgb444 / k_fdct_rgb_ss / k_fdct_libjpeg by the sampling and
                                 * the flavour) or GJ_K1_BLOCKS (k_fdct_samples) */
    int flavour;                /* 0 this library's FDCT, GJ_FDCT_ISLOW */
    int convert;                /* gj_launch_convert_in writes the padded component planes (planes_bytes) first */
    size_t planes_bytes;
    int flip;                   /* GJ_K1_FLIP_*: rows read last to first, or the planes flipped */
    int stripes;                /* the host image may arrive stripe by stripe (fused rows, as stored) */
    int mcu_rows;               /* MCU rows of the frame: the fused kernels' row range */
    int raw_layout;             /* the kernels read the raw image through its gj_raw_layout */
};
/* The one place K1 is chosen (gj_codestream.c), for a frame the encoder accepted */
void gj_k1_choose(const struct gj_geometry* g, const struct gj_k1_request* r, struct gj_k1_plan* p);
/* K1 as a frame's plan says, into quantised zig-zag coefficients and their non-zero masks.
 * The fused kernels (this library's flavour: RGB u8 interleaved, luminance 1x1, 2x1, 2x2 or 1x2 and chrominance 1x1, the colour
 * transform fused with the FDCT; GJ_FDCT_ISLOW: the same RGB input, or grey u8, through libjpeg-turbo's colour conversion,
 * downsampling, ISLOW FDCT and quantiser (raw_q: the DQT tables, zig-zag), with its edge replication and the dummy blocks of
 * interleaved MCUs): MCU rows [my0, my1) of the frame (an MCU row = 8 * comp[0].vs image rows), `pitch` bytes per image row
 * [replaces ref: src/gpujpeg_preprocessor.cu:241-253, 562-586 + src/gpujpeg_dct_gpu.cu:621-678] */
int gj_launch_fdct_fused(const struct gj_k1_plan* plan, const struct gj_geometry* g, const uint8_t* d_raw, int pitch, int my0, int my1,
                         const struct gj_dev_enc_tables* h_tables, const uint8_t raw_q[2][64], int16_t* d_coef, uint64_t* d_nzmask,
                         gj_stream_t stream);
/* The per-block kernel, no colour transform, any pixel format gj_raw_layout_init describes or the component planes
 * (gj_planes_layout), any sampling: one thread per 8x8 block reads its samples straight from the image of layout `raw`
 * [replaces the "matching format" memcpy path + DCT launches, ref: src/gpujpeg_preprocessor.cu:409-455,
 *  src/gpujpeg_postprocessor.cu:406-433, and the GPUJPEG_NONE colour-transform kernels] */
int gj_launch_fdct_blocks(const struct gj_k1_plan* plan, const uint8_t* d_src, const struct gj_raw_layout* raw, const struct gj_comp_geo* comp,
                          int comp_count, const uint8_t* comp_tbl, const struct gj_dev_enc_tables* h_tables, int16_t* d_coef,
                          uint64_t* d_nzmask, gj_stream_t stream);

/* K2: Huffman-encode every restart segment and assemble the finished scan data
 * [replaces ref: src/gpujpeg_huffman_gpu_encoder.cu:1071-1167 + host loop src/gpujpeg_encoder.c:567-626]
 * d_stream receives [header gap][SOS][scan 0]...[EOI]; d_info[0] = total bytes, d_info[1] = error flag */
struct gj_huff_enc_args {
    const int16_t* d_coef;
    const uint64_t* d_nzmask; /* [comp][block]: bit k set <=> zig-zag coefficient k is non-zero (written by K1) */
    struct gj_scan_layout lay; /* scans, segments and the block order inside them */
    int seg_mcu;
    uint8_t* d_tmp;
    size_t slot_stride;
    uint32_t* d_spill;      /* [seg_count][blocks per segment, or 32 lanes for long segments][32 words]: overflow of the
                             * per-block bit strings (rarely touched) */
    uint32_t* d_seg_bytes;  /* [seg_count] */
    uint64_t* d_seg_off;    /* [seg_count] */
    uint8_t* d_stream;
    size_t stream_cap;
    uint32_t header_size;
    const uint8_t* d_sos;   /* what precedes every scan's data: [APP13 segment-info headers] SOS header; scan s: pre_len[s]
                             * bytes at d_sos + pre_off[s] */
    int pre_len[GJ_MAX_COMP], pre_off[GJ_MAX_COMP];
    uint64_t* d_seg_pos;    /* [seg_count] or NULL: receives the stream offset of every segment's first byte (segment info) */
    uint64_t* d_info;       /* [4]: total, error, reserved */
    uint64_t* d_info_next;  /* [4] or NULL: cleared by this launch for the next one */
    int info_is_zero;       /* d_info has been cleared by the previous launch */
    const struct gj_dev_enc_tables* d_tables;
    uint64_t* d_split;      /* segments longer than 40 blocks: status words of the chunks and tiles, split_bytes bytes */
    size_t split_bytes;
};
int gj_launch_huffman_encode(const struct gj_huff_enc_args* a, gj_stream_t stream);
/* bytes of d_split a frame needs whose slots grow to at most max_slot_stride bytes (0: short segments) */
size_t gj_huffman_split_status_bytes(int seg_count, int segblk, size_t max_slot_stride);
/* the same in pieces (the encoder's stripe pipeline): K2 on scan k's segments [lo[k], lo[k] + n[k]) -- `first` marks the first
 * piece of a frame --, then the tail kernel once; only for frames gj_huffman_encode_parts_eligible() accepts */
int gj_huffman_encode_parts_eligible(const struct gj_huff_enc_args* a);
int gj_launch_huffman_encode_part(const struct gj_huff_enc_args* a, int first, const int lo[GJ_MAX_COMP], const int n[GJ_MAX_COMP],
                                  gj_stream_t stream);
int gj_launch_huffman_place(const struct gj_huff_enc_args* a, gj_stream_t stream);
/* symbol statistics of the frame K1 left in place, exactly as K2 would emit the symbols: d_counts[table class][DC 0 / AC 1]
 * [symbol] (2 x 2 x 256 64-bit counters, cleared by the launch) -- the input of enc_opt_huffman=optimized */
#define GJ_HUFF_COUNTS_BYTES (2 * 2 * 256 * sizeof(uint64_t))
int gj_launch_huffman_stats(const struct gj_huff_enc_args* a, uint64_t* d_counts, gj_stream_t stream);

/* Block extent, the decoder's format between K3 and K4: next to its coefficient buffer the decoder keeps one byte per
 * 64-coefficient block, at the block's index in the coefficient buffer.  Its value n (0..GJ_CEXT_FULL) says that the
 * 16-byte chunks 0..n-1 of the block (chunk i = zig-zag coefficients 8i..8i+7) are valid in the coefficient buffer and
 * that every coefficient past them is zero, whatever the buffer holds there.  Every decode path writes the extent of
 * every block of the frame on every frame, blocks it leaves zero included, so that chunks a denser earlier frame left
 * behind are never read.  Helpers: gj_cext_of, gj_load_coef_block (gj_device.cuh). */
#define GJ_CEXT_FULL 8

/* K3: Huffman-decode every restart segment into zig-zag coefficients and block extents
 * [replaces ref: src/gpujpeg_huffman_gpu_decoder.cu:663-746] */
struct gj_huff_dec_args {
    const uint8_t* d_file;      /* the JPEG bytes */
    size_t file_size;
    const uint32_t* d_seg_off;  /* host-built table: [seg_count] file offset of each segment (or NULL) */
    /* resynchronised streams: [seg_count] {file offset, clean start, clean end} per segment, file offset 0xFFFFFFFF = the
     * segment does not exist in the stream (its blocks are zero); NULL = positions come from the marker list */
    const uint32_t* d_seg_tab;
    uint32_t* d_unit_ctr;       /* 8 words, all zero between launches: work counters of the self-synchronising kernel */
    const uint32_t* d_seg_len;  /* informative: the decoder stops after the segment's block count */
    /* device-built marker list (K0): segment j of scan s starts at scan_begin[s] (j = 0) or two bytes
     * after marker number first_rank[s] + j - 1 */
    const uint32_t* d_list_pos;
    const uint8_t* d_list_code;
    uint32_t first_rank[GJ_MAX_COMP];  /* markers in front of the scan's first byte (host, from K0's marker report) */
    uint32_t scan_begin[GJ_MAX_COMP];
    uint32_t* d_error;            /* set to non-zero by K3 when the RSTn sequence is broken */
    /* the clean stream (K0): stuffing, fill bytes and markers removed, big-endian words.  Segment j of scan s occupies
     * the clean bytes [scan_cbegin[s] or d_list_cpos[first_rank[s] + j - 1], d_list_cpos[first_rank[s] + j]) */
    const uint32_t* d_clean;
    const uint32_t* d_list_cpos;
    uint32_t scan_cbegin[GJ_MAX_COMP];
    /* self-synchronising kernel: lanes that share one restart segment in scan s (2, 4, 8, 16 or 32; gj_k3_choose) */
    uint8_t scan_lanes[GJ_MAX_COMP];
    uint32_t scan_bytes[GJ_MAX_COMP];  /* entropy-coded bytes of scan s (as in the file) */
    uint8_t scan_dense[GJ_MAX_COMP];   /* >= 16 bytes of entropy-coded data per block: worth staging blocks in shared memory */
    int kernel;                 /* GJ_K3_THREAD_PER_SEGMENT, GJ_K3_SELF_SYNC or GJ_K3_SUBSEQUENCE (gj_k3_choose) */
    /* the decoder's stripe pipeline (self-synchronising kernel only): this launch decodes scan s's segments
     * [part_seg_lo[s], part_seg_hi[s]) -- rounded outwards to whole units, so launches must hand over at multiples of 32
     * segments --, part_seg_hi[s] == 0: all of the scan */
    int part_seg_lo[GJ_MAX_COMP], part_seg_hi[GJ_MAX_COMP];
    int dequantize;             /* 1: store coefficient*quantiser wrapped to int16 (integer IDCT flavour) */
    struct gj_scan_layout lay;  /* scans, segments and the block order inside them */
    int seg_count, seg_mcu;
    int scan_comp[GJ_MAX_COMP][GJ_MAX_COMP]; /* component index of the i-th component of scan s */
    int scan_td[GJ_MAX_COMP][GJ_MAX_COMP], scan_ta[GJ_MAX_COMP][GJ_MAX_COMP];
    int scan_tq[GJ_MAX_COMP][GJ_MAX_COMP]; /* quantisation table id of that component */
    int16_t* d_coef;
    uint8_t* d_cext;            /* the extent of every block of d_coef (GJ_CEXT_FULL) */
    const struct gj_dev_dec_tables* d_tables;
    /* dec_opt_crop: decode only the pick_count pairs {global segment, blocks} of d_pick (gj_crop_pick), one thread per
     * segment; the caller clears d_cext first.  With positions from the marker list the launch also checks the number of
     * every restart marker of the frame, as a full decode would.  NULL: every segment. */
    const uint32_t* d_pick;
    int pick_count;
    /* the sub-sequence kernel (gj_huffscan.cu) for every scan: segments of any length, several threads per segment; positions
     * from the marker list only.  d_ss_scratch holds gj_subseq_scratch_bytes(seg_count, ecs_bytes, gj_subseq_grid()) bytes.
     * A cropped frame decodes whole segments then (d_pick is not used). */
    void* d_ss_scratch;
    size_t ss_scratch_bytes, ecs_bytes;
};
int gj_launch_huffman_decode(const struct gj_huff_dec_args* a, gj_stream_t stream);
/* K3's kernel.  GJ_K3_AUTO is a request only (dec_opt_huffman=auto). */
enum { GJ_K3_AUTO = 0, GJ_K3_THREAD_PER_SEGMENT = 1, GJ_K3_SELF_SYNC = 2, GJ_K3_SUBSEQUENCE = 3 };
/* where K3 finds the restart segments: K0's marker list, the stream's segment-info tables, the resynchronised table */
enum { GJ_K3_MARKER_LIST = 0, GJ_K3_SEGMENT_INFO = 1, GJ_K3_RESYNC_TABLE = 2 };
#define GJ_K3_SYNC_MAXBLK 40   /* blocks per restart segment the self-synchronising kernel takes (every RESTART_AUTO setting) */
/* The one place K3's kernel is chosen (gj_codestream.c), from the frame (geometry, a->scan_bytes), the request
 * (dec_opt_huffman: GJ_K3_AUTO, GJ_K3_THREAD_PER_SEGMENT or GJ_K3_SUBSEQUENCE; dec_opt_huffman_lanes: force_lanes, 0 =
 * automatic), where the segment positions come from (GJ_K3_MARKER_LIST ..) and whether the frame is cropped.  Sets
 * a->kernel, scan_lanes and scan_dense of the frame's scans, ecs_bytes.  Returns 1 if K3 decodes only the segments of a crop
 * (gj_crop_pick), 0 if every segment, -1 for GJ_K3_SEGMENT_INFO if the frame is not to be decoded from those tables. */
int gj_k3_choose(const struct gj_geometry* g, int request, const int force_lanes[GJ_MAX_COMP], int positions, int crop,
                 struct gj_huff_dec_args* a);

/* K4, the pixel stage: what the decoder's output negotiation (choose_output) gives -- RGB u8 interleaved from a 3-component YCbCr
 * stream, the stream's own samples in a pixel format of its sampling, or any other format / colour space through component
 * planes and the generic pass (gj_convert.cu) -- and the frame's options */
enum { GJ_OUT_RGB = 1, GJ_OUT_SAMPLES = 2, GJ_OUT_GENERIC = 3 };
struct gj_k4_request {
    int out;                    /* GJ_OUT_* */
    int libjpeg;                /* dec_opt_pixels=libjpeg: GPUJPEG_RGB 444-u8-p012 or GPUJPEG_U8, libjpeg-turbo's pixels */
    int scale;                  /* dec_opt_scale: 1, 2, 4 or 8 */
    int crop;                   /* dec_opt_crop, a rectangle smaller than the image: src */
    int src[4];                 /* x, y, w, h of the (scaled) image the output shows */
    int orient;                 /* dec_opt_orientation turns or mirrors the image: map */
    struct gj_orient_map map;   /* output pixel <-> image pixel (gj_orient_frame) */
    int flipped;                /* dec_opt_flipped */
    int idct_flavour;           /* dec_opt_idct: 0 int, 1 float */
    int coef_only;              /* the frame stops after the Huffman stage */
    int channel_remap;          /* dec_opt_channel_remap is set */
};
/* dec_opt_crop: K4 on a window -- only the blocks blk[c] of every component are transformed, and sample (sx, sy) of
 * component c goes to (sx - ox[c], sy - oy[c]) of the raw image, kept where that lies inside comp[c].width x comp[c].height */
struct gj_k4_window {
    struct gj_blk_rect blk[GJ_MAX_COMP];
    int ox[GJ_MAX_COMP], oy[GJ_MAX_COMP];
};
enum { GJ_K4_FUSED = 1, GJ_K4_SAMPLES = 2, GJ_K4_SCALED = 3 };
enum { GJ_K4_FLIP_NONE = 0, GJ_K4_FLIP_PITCH = 1, GJ_K4_FLIP_PLANES = 2 };
enum { GJ_K4_POST_NONE = 0, GJ_K4_POST_CONVERT = 1, GJ_K4_POST_LIBJPEG = 2 };
/* IDCT flavour of k_idct_samples for dec_opt_pixels=libjpeg: libjpeg's jpeg_idct_islow (gj_idct_islow_block) on raw coefficients */
#define GJ_IDCT_ISLOW 2
/* Everything K4 does with a frame: gj_launch_idct_fused or gj_launch_idct_blocks, then the flip of the planes, then the pass from
 * the planes to the output (gj_decoder.c launch_k4) */
struct gj_k4_plan {
    int kernel;                 /* GJ_K4_FUSED (k_idct_rgb444 / k_idct_rgb_ss by the sampling), GJ_K4_SAMPLES (k_idct_samples)
                                 * or GJ_K4_SCALED (k_idct_scaled<n>) */
    int window;                 /* the WIN instance: fused, the rectangle rect; the others, the window win */
    int orient;                 /* fused: 0 as stored, 1 the ORIENT instance of a half turn or a mirror, 2 of a quarter turn */
    int flavour;                /* 0 int, 1 float, GJ_IDCT_ISLOW */
    int dequantize;             /* K3 (or the progressive scans) store coefficient * quantiser wrapped to int16 */
    int n;                      /* samples per block side: 8, or 8 / scale */
    int to_planes;              /* the IDCT writes the padded component planes (gj_planes_layout), else the output */
    int scomp;                  /* ... the output, through the components at the output's size (else the stream's geometry) */
    int rect[4];                /* fused: x, y, w, h of the image the output shows */
    struct gj_orient_map map;
    struct gj_k4_window win;    /* the blocks a cropped frame needs (K3 decodes the segments that hold them) and the origins */
    int flip;                   /* GJ_K4_FLIP_*: rows written last to first, or the planes flipped */
    int post;                   /* GJ_K4_POST_*: gj_launch_convert_out, gj_launch_libjpeg_out */
    int post_map;               /* the post pass takes map */
    int stripes;                /* the frame may leave for the host stripe by stripe (fused rows, as stored) */
    int mcu_rows;               /* MCU rows of the frame: the fused kernels' row range */
    size_t planes_bytes;        /* the component planes */
};
/* The one place K4 is chosen (gj_codestream.c), for a request the decoder accepted */
void gj_k4_choose(const struct gj_geometry* g, const struct gj_k4_request* r, struct gj_k4_plan* p);
/* sub-sequence kernel: bytes per sub-sequence (a tuning value; GPUJPEG_B200_SUBSEQ_BYTES overrides it for experiments), the
 * smallest value the scratch is sized for, warm-up of a sub-sequence's first walk */
#define GJ_SS_SUB_BYTES 32
#define GJ_SS_MIN_BYTES 16
#define GJ_SS_WARM_BITS 256
size_t gj_subseq_scratch_bytes(int seg_count, size_t ecs_bytes, int grid_ctas);
int gj_subseq_grid(void);   /* CTAs of its cooperative grid on the current device, -1 on error */
int gj_subseq_rounds(const void* d_scratch, gj_stream_t stream);   /* rounds of the last launch on that scratch */
int gj_launch_huffman_decode_subseq(const struct gj_huff_dec_args* a, void* d_scratch, size_t scratch_bytes, size_t ecs_bytes,
                                    gj_stream_t stream);

/* Progressive frames (gj_progressive.cu): one scan of a SOF2 frame as k_prog_decode sees it.  An interleaved scan (DC
 * only) codes MCUs of the frame's MCU grid; a non-interleaved one codes the component's own ceil(w_c/8) x ceil(h_c/8)
 * blocks -- one block per MCU, so that the restart interval counts blocks -- inside its (possibly MCU-padded) plane. */
enum { GJ_PROG_DC_FIRST = 0, GJ_PROG_DC_REFINE = 1, GJ_PROG_AC_FIRST = 2, GJ_PROG_AC_REFINE = 3 };
struct gj_prog_scan {
    int kind;                      /* GJ_PROG_* */
    int ss, se, ah, al;
    int ncomp;                     /* components in the scan */
    int bpm;                       /* blocks per MCU */
    int units, units_x;            /* MCUs of the scan, MCUs per row */
    int seg_units;                 /* MCUs per restart segment */
    int seg_count;
    int lut0;                      /* component i of the scan decodes with table lut0 + i of the frame's table array */
    uint32_t first_rank, cbegin;   /* K0: markers in front of the scan, clean-stream position of its first byte */
    int blk_off[GJ_MAX_COMP], bcx[GJ_MAX_COMP], nblk[GJ_MAX_COMP], hs[GJ_MAX_COMP], vs[GJ_MAX_COMP];   /* by scan component */
    uint8_t idx_ci[GJ_MAX_MCU_BLOCKS], idx_dx[GJ_MAX_MCU_BLOCKS], idx_dy[GJ_MAX_MCU_BLOCKS];          /* block i of an MCU */
};
/* scan k of a progressive stream on the frame geometry g (which must be the interleaved one if any scan interleaves);
 * 0 on success, -1 if the scan does not fit the geometry */
int gj_prog_scan_init(const struct gj_geometry* g, const struct gj_stream* s, int k, int restart_interval, struct gj_prog_scan* out);
/* dec_opt_crop: the pick list of progressive scan S (pairs as gj_crop_pick_units, segment numbers of the scan); comp[i] is the
 * frame component of scan component i */
int gj_prog_crop_pick(const struct gj_prog_scan* S, const int comp[GJ_MAX_COMP], const struct gj_blk_rect win[GJ_MAX_COMP],
                      uint32_t* out);

struct gj_prog_args {
    const struct gj_prog_scan* scans;   /* host array, scan_count entries */
    int scan_count;
    const struct gj_dec_lut* d_luts;    /* every scan's Huffman tables, one copy per frame */
    const uint32_t* d_clean;            /* K0's clean stream and marker list */
    const uint32_t* d_list_cpos;
    const uint8_t* d_list_code;
    uint32_t* d_error;                  /* set when a restart marker carries the wrong number */
    int16_t* d_coef;
    uint8_t* d_cext;                    /* block extents: all GJ_CEXT_FULL (the scans accumulate into the dense buffer) */
    size_t coef_count;
    int dequantize;                     /* 1: finish with coefficient * quantiser wrapped to int16 (integer IDCT flavour) */
    int comp_count;
    int comp_blk_off[GJ_MAX_COMP];      /* first block of every component (dequantisation table qinv_zz[component]) */
    const struct gj_dev_dec_tables* d_tables;
    /* dec_opt_crop: scan k decodes only the pairs {segment, blocks} d_pick[2 * pick_off[k] ..] (pick_n[k] of them); NULL: all */
    const uint32_t* d_pick;
    int pick_off[GJ_MAX_SCANS], pick_n[GJ_MAX_SCANS];
};
/* zero the coefficients, decode every scan in stream order, dequantise */
int gj_launch_progressive_decode(const struct gj_prog_args* a, gj_stream_t stream);

/* K0: marker list of the entropy-coded part of the file, built on the device (gj_markers.cu)
 * [replaces ref: src/gpujpeg_reader.c:1038-1155] */
int gj_launch_marker_scan(const uint8_t* d_file, size_t begin, size_t end, unsigned long long* d_cta, uint32_t* d_list_pos,
                          uint8_t* d_list_code, uint32_t* d_list_cpos, uint32_t list_cap, uint8_t* d_clean, uint32_t* d_result,
                          uint32_t* d_other, uint32_t other_cap, gj_stream_t stream);

/* K4 as a frame's plan (gj_k4_choose) says, from the zig-zag coefficients and their block extents.
 * The fused kernels (k_idct_rgb444 for 4:4:4, else k_idct_rgb_ss; comp: luminance 1x1, 2x1, 2x2 or 1x2, chrominance 1x1):
 * dequantisation, IDCT, colour transform and interleave into RGB u8 of `pitch` bytes per row, MCU rows [my0, my1) of the
 * width x height image (an MCU row = 8 * comp[0].vs image rows; a window or orientation instance takes the whole frame and
 * writes the rectangle plan->rect, pitch 3 * its width, or 3 * its height after a quarter turn)
 * [replaces ref: src/gpujpeg_dct_gpu.cu:681-727 + src/gpujpeg_postprocessor.cu:183-216, 271-282, 444-496] */
int gj_launch_idct_fused(const struct gj_k4_plan* plan, const int16_t* d_coef, const uint8_t* d_cext, const struct gj_comp_geo comp[3],
                         const int comp_tq[3], uint8_t* d_out, int width, int height, int pitch, int my0, int my1,
                         const struct gj_dev_dec_tables* h_tables, gj_stream_t stream);
/* The per-block kernels, one thread per 8x8 block, no colour transform (k_idct_samples, plan->n = 8; k_idct_scaled<n>, n = 4,
 * 2 or 1 for dec_opt_scale, from raw coefficients): the plan->n x plan->n samples of every block (of the window plan->win)
 * straight into the raw image of layout `raw`, any pixel format gj_raw_layout_init describes or the component planes
 * (gj_planes_layout); comp[c].width / height are the component's sample extents at that size
 * [replaces the "matching format" memcpy path + DCT launches, ref: src/gpujpeg_postprocessor.cu:406-433] */
int gj_launch_idct_blocks(const struct gj_k4_plan* plan, const int16_t* d_coef, const uint8_t* d_cext, const struct gj_comp_geo* comp,
                          int comp_count, const int* comp_tq, uint8_t* d_raw, const struct gj_raw_layout* raw,
                          const struct gj_dev_dec_tables* h_tables, gj_stream_t stream);
/* dec_opt_pixels=libjpeg behind the ISLOW planes (gj_planes_layout, n = 8; comp = the stream's geometry, whose width / height are
 * every component's real samples): the width x height output, RGB u8 interleaved (3 components) or grey u8, pixel (x, y) showing
 * source pixel `map` (x, y) -- luminance, fancy-upsampled chroma (gj_fancy_sample), jdcolor's YCbCr -> RGB unless rgb_internal */
int gj_launch_libjpeg_out(const uint8_t* d_planes, uint8_t* d_out, const struct gj_comp_geo* comp, int comp_count, int max_hs, int max_vs,
                          int width, int height, int rgb_internal, const struct gj_orient_map* map, gj_stream_t stream);

/* Generic pre-/post-processing pass (gj_convert.cu): raw image in any supported pixel format and colour space <-> the
 * component planes of the YCbCr JPEG (plane c at byte comp[c].blk_off * n * n, pitch comp[c].bcx * n, n samples per block
 * side: 8, or fewer for the planes of a scaled decode)
 * [replaces the generic kernels of ref: src/gpujpeg_preprocessor.cu:163-201, src/gpujpeg_postprocessor.cu:183-216] */
int gj_launch_convert_in(const uint8_t* d_raw, const struct gj_raw_layout* raw, enum gpujpeg_pixel_format fmt, int color_space,
                         int color_space_internal, int width, int height, uint8_t* d_planes, size_t planes_size,
                         const struct gj_comp_geo* comp, int comp_count, int max_hs, int max_vs, gj_stream_t stream);
/* map: the image pixel each raw pixel shows -- dec_opt_crop converts only its rectangle, dec_opt_orientation turns and mirrors
 * (the raw image is then width x height of the oriented output); NULL: raw pixel (x, y) is image pixel (x, y) */
int gj_launch_convert_out(const uint8_t* d_planes, uint8_t* d_raw, const struct gj_raw_layout* raw, enum gpujpeg_pixel_format fmt,
                          int color_space, int color_space_internal, int width, int height, const struct gj_comp_geo* comp,
                          int comp_count, int max_hs, int max_vs, int n, const struct gj_orient_map* map, gj_stream_t stream);
/* enc/dec_opt_flipped: vertical flip of the (padded) component planes; enc/dec_opt_channel_remap: channel permutation of
 * the raw image in place.  gj_launch_channel_remap returns -2 when the channel count does not match the pixel format and
 * -3 for pixel formats with chroma subsampling [replaces ref: src/gpujpeg_preprocessor.cu:456-559] */
int gj_launch_flip_planes(uint8_t* d_planes, const struct gj_comp_geo* padded, int comp_count, gj_stream_t stream);
int gj_launch_channel_remap(uint8_t* d_raw, const struct gj_raw_layout* raw, enum gpujpeg_pixel_format fmt, int width, int height,
                            unsigned remap, gj_stream_t stream);
/* option value -> (channel count << 24) | selector nibbles [ref: src/gpujpeg_encoder.c:662-698]; 0 on error */
unsigned gj_parse_channel_remap(const char* val, const char* optname);
/* "1" / "0" / "true" / "false" ... -> 0 / 1, -1 on error [ref: src/gpujpeg_common.c gpujpeg_parse_bool_opt] */
int gj_parse_bool(const char* val, const char* optname);
/* the planes above described as a raw layout, so that the sample kernels can run on them (n samples per block side) */
void gj_planes_layout(struct gj_raw_layout* l, struct gj_comp_geo padded[GJ_MAX_COMP], const struct gj_comp_geo* comp,
                      int comp_count, int n);

/* The transcoder (gj_transcode.cu): the decoder's raw coefficients and block extents -> the encoder's coefficient buffer and
 * non-zero masks, every output block through the plan's block map and coefficient map (the identity included).  *d_range is
 * set non-zero when an output coefficient leaves the 8-bit baseline range (DC [-1024, 1023], AC [-1023, 1023]). */
struct gj_coef_transform_args {
    const int16_t* d_src;
    const uint8_t* d_cext;
    int src_blk_off[GJ_MAX_COMP];
    int16_t* d_dst;
    uint64_t* d_nzmask;
    int dst_blk_off[GJ_MAX_COMP];
    int comp_count;
    int dst_blocks;
    int transpose, neg_x, neg_y;
    struct gj_blk_map blk[GJ_MAX_COMP];
    uint32_t* d_range;
};
int gj_launch_coef_transform(const struct gj_coef_transform_args* a, gj_stream_t stream);

/* The decoder up to its raw quantised coefficients (gj_decoder.c): every stream gpujpeg_decoder_decode takes, no IDCT, no output.
 * The pointers stay valid until the decoder's next call. */
struct gj_coef_frame {
    const struct gj_geometry* geo;    /* block grids and their offsets in d_coef */
    const int16_t* d_coef;            /* zig-zag, not dequantised */
    const uint8_t* d_cext;
    int progressive;
    enum gpujpeg_color_space color_space;
    uint8_t qt[GJ_MAX_COMP][64];      /* component c's quantisation table (zig-zag) and its table id */
    int tq[GJ_MAX_COMP];
    struct gpujpeg_image_metadata metadata;
    const uint8_t* com;               /* the COM segments in front of the first SOS, markers included */
    size_t com_size;
};
/* window: NULL, or called once per frame when its geometry g is set (progressive: the block grids the scans decode into) and
 * before any Huffman decoding, with the stream's metadata read so far.  It returns -1 to refuse the frame, 0 to decode every
 * block, or 1 to decode only the restart segments that hold the blocks win[c] of every component (gj_crop_pick,
 * gj_prog_crop_pick); the extents of the blocks left undecoded are 0, so they read as zero. */
typedef int (*gj_coef_window_fn)(void* ctx, const struct gj_geometry* g, int progressive, const struct gpujpeg_image_metadata* md,
                                 struct gj_blk_rect win[GJ_MAX_COMP]);
int gj_decoder_decode_coefficients(struct gpujpeg_decoder* d, const uint8_t* image, size_t image_size, gj_coef_window_fn window,
                                   void* ctx, struct gj_coef_frame* f);

/* The encoder from coefficients (gj_encoder.c): gj_encoder_setup_coefficients sizes the encoder for a frame of parameters p
 * (RESTART_AUTO as gpujpeg_encoder_encode resolves it for the frame, no segment info) and width x height with the header composed from comp_q / comp_tq, the COM
 * segments com (replacing the writer's comments) and the metadata, and hands out where the coefficients and non-zero masks go
 * (comp-major zig-zag blocks of *geo).  gj_encoder_finish runs what follows K1 in gpujpeg_encoder_encode. */
int gj_encoder_setup_coefficients(struct gpujpeg_encoder* e, const struct gpujpeg_parameters* p, int width, int height,
                                  const uint8_t comp_q[GJ_MAX_COMP][64], const uint8_t comp_tq[GJ_MAX_COMP], const uint8_t* com,
                                  size_t com_size, const struct gpujpeg_image_metadata* metadata, int16_t** d_coef,
                                  uint64_t** d_nzmask, const struct gj_geometry** geo);
int gj_encoder_finish(struct gpujpeg_encoder* e, uint8_t** out, size_t* out_size);

/* debug/test helper: device coefficient buffer (zig-zag) -> host natural order, block-major; coefficients past a block's
 * extent read as zero: the decoder's extent bytes d_cext, or the encoder's non-zero masks d_nzmask (gj_coef_live_chunks) */
int gj_coef_to_host_natural(const int16_t* d_coef, const uint8_t* d_cext, const uint64_t* d_nzmask, size_t count, int16_t* h_out,
                            gj_stream_t stream);

/* thin wrappers over the CUDA runtime so the host files stay plain C without cuda headers */
int gj_cuda_malloc(void** p, size_t size);
int gj_cuda_free(void* p);
int gj_cuda_malloc_host(void** p, size_t size);
int gj_cuda_free_host(void* p);
int gj_cuda_memcpy_h2d_async(void* dst, const void* src, size_t size, gj_stream_t s);
int gj_cuda_memcpy_d2h_async(void* dst, const void* src, size_t size, gj_stream_t s);
int gj_cuda_memcpy_d2d_async(void* dst, const void* src, size_t size, gj_stream_t s);
int gj_cuda_memset_async(void* dst, int v, size_t size, gj_stream_t s);
int gj_cuda_stream_sync(gj_stream_t s);
int gj_cuda_stream_create(gj_stream_t* s);   /* non-blocking: runs next to the legacy default stream */
int gj_cuda_event_create(void** ev);          /* timing disabled */
void gj_cuda_event_destroy(void* ev);
int gj_cuda_event_record(void* ev, gj_stream_t s);
int gj_cuda_stream_wait_event(gj_stream_t s, void* ev);
void gj_cuda_stream_destroy(gj_stream_t s);
int gj_cuda_enable_peer(int peer);
int gj_cuda_memcpy_peer_async(void* dst, int dst_dev, const void* src, int src_dev, size_t size, gj_stream_t s);
int gj_cuda_pointer_is_device(const void* p);
const char* gj_cuda_last_error(void);
/* event timers [ref: src/gpujpeg_common_internal.h:156-205] */
struct gj_timer { void* start; void* stop; int armed; };
int gj_timer_create(struct gj_timer* t);
void gj_timer_destroy(struct gj_timer* t);
void gj_timer_start(struct gj_timer* t, gj_stream_t s);
void gj_timer_stop(struct gj_timer* t, gj_stream_t s);
double gj_timer_ms(struct gj_timer* t);
int gj_cuda_device_count(void);
int gj_cuda_sm_count(void);   /* multiprocessors of the current device (132 on an H100 SXM); 1 on failure */
int gj_cuda_device_props(int dev, struct gpujpeg_device_info* info);
int gj_cuda_set_device(int dev);
int gj_cuda_get_device(void);
void gj_cuda_device_reset(void);

#ifdef __cplusplus
}
#endif
#endif
