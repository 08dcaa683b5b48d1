/*
 * gj_encoder.c -- the public encoder API on top of the sm_90a stage launchers.  Host C.
 *
 * Mirrors the reference orchestrator's contract (src/gpujpeg_encoder.c:351-646): same parameter
 * handling (comp_count 0 => from pixel format, RESTART_AUTO heuristic), same re-initialisation
 * rules, one stream, blocks until the JPEG is complete in an encoder-owned host buffer.
 * What differs is the pipeline behind it:
 *
 *     H2D raw  ->  K1 (colour+FDCT+quant, one launch for all components)
 *              ->  K2 (Huffman encode -> scan -> finished byte stream on the device)
 *              ->  D2H 32-byte info, D2H payload (one copy; the reference copies 43 200 segments
 *                  one by one on the host, src/gpujpeg_encoder.c:567-623)
 *
 * Supported (anything else fails loudly with GPUJPEG_ERROR, never a CPU fallback): see params_supported() --
 * internal colour space YCbCr JPEG (BT.601 full range), JFIF header, 1 or 3 components, 4:4:4 / 4:2:2 / 4:2:0 /
 * 4:4:0, interleaved or not, any restart interval; input GPUJPEG_RGB 444-u8-p012 through the fused kernels, grey /
 * planar / packed YCbCr input without colour transform straight into the DCT, every other pixel format x colour
 * space combination through the generic pass.
 */
#include <assert.h>
#include <stdlib.h>
#include <string.h>

#include "gj_internal.h"

#define GJ_STRIPES 8
#define GJ_STRIPE_MIN_BYTES ((size_t)8 << 20)

struct gpujpeg_encoder {
    gj_stream_t stream;
    int device;
    struct gpujpeg_parameters param;           /* as adjusted */
    struct gpujpeg_image_parameters param_image;
    int initialised;
    struct gj_geometry geo;
    struct gj_k1_request k1_req;               /* what the K1 plan was chosen for */
    struct gj_k1_plan k1;                      /* what K1 does with the frame (gj_k1_choose) */
    uint8_t* d_planes; size_t d_planes_size;   /* component planes between the generic pass and the DCT */
    struct gj_raw_layout raw;                  /* where the samples live (k1.raw_layout) */
    int quality;                               /* quality the tables were built for (-1 = none) */
    enum gpujpeg_header_type header_type;      /* enc_hdr: forced header flavour, GPUJPEG_HEADER_DEFAULT = by colour space */
    enum gpujpeg_header_type header_written;   /* flavour the cached header bytes were composed with */
    int flipped;                               /* enc_opt_flipped */
    unsigned channel_remap;                    /* enc_opt_channel_remap: (count << 24) | selector nibbles, 0 = none */
    int out_pinned;

    uint8_t raw_q[2][64];
    struct gj_huff_spec spec[2][2];
    struct gj_dev_enc_tables h_tab;            /* host copy (K1 takes it by value) */
    struct gj_dev_enc_tables* d_tab;           /* device copy (K2 LUTs) */
    int huff_optimized;                        /* enc_opt_huffman=optimized: tables fitted to every frame */
    int writer_libjpeg;                        /* enc_opt_writer=libjpeg: libjpeg-turbo's coefficients and header */
    int spec_custom;                           /* spec / LUTs / header hold fitted tables, not Annex K */
    uint64_t* d_counts;                        /* [2][2][256] symbol counts of the statistics kernel */
    uint64_t* h_counts;                        /* pinned copy */
    int counts_valid;                          /* the statistics kernel has run on the current geometry */

    /* device buffers */
    uint8_t* d_raw; size_t d_raw_size;
    int16_t* d_coef; size_t d_coef_size;
    uint64_t* d_nzmask; size_t d_nzmask_size;
    uint8_t* d_tmp; size_t d_tmp_size;
    size_t slot_stride;              /* bytes per restart segment in d_tmp: starts at 48 bytes per block (photographic and noisy
                                      * content at any common quality), grows to what a frame needed when K2 reports an overflow;
                                      * the worst case (geo.slot_stride, 416 bytes per block: 648 MB for an 8K frame) is only ever
                                      * allocated for content that needs it.  Segments on K2's chunk path (gj_huffman.cu) split
                                      * their slot into equal parts per block, one per chunk of 128 blocks: there the DENSEST
                                      * chunk sets the size (a photo with one noisy region can outgrow 48 bytes per block where
                                      * the whole segment would not, and then re-runs K2 once with slots of up to 216 bytes
                                      * per block) */
    uint32_t* d_spill; size_t d_spill_size;
    uint64_t* d_split; size_t d_split_size;  /* status words of the long-segment path of K2 */
    uint32_t* d_seg_bytes; uint64_t* d_seg_off; int seg_alloc;
    uint8_t* d_stream; size_t d_stream_size;
    uint8_t* d_sos; size_t d_sos_size;        /* per scan: [APP13 segment-info headers] SOS header */
    uint8_t* h_pre; size_t h_pre_size;         /* the same on the host */
    int pre_len[GJ_MAX_COMP], pre_off[GJ_MAX_COMP];
    int with_segment_info;                     /* param.segment_info && restart_interval > 0 [ref: src/gpujpeg_writer.c:553] */
    uint64_t* d_seg_pos; uint64_t* h_seg_pos; size_t seg_pos_size;   /* segment info: stream offset of every segment (pinned copy) */
    uint64_t* d_info;                          /* two blocks of 4 words: K2's tail clears the one the next launch uses */
    uint64_t* d_info_cur;                      /* the block the last K2 launch reported into */
    int info_parity, info_clean;
    uint64_t* h_info;                          /* pinned */

    /* host output */
    uint8_t* out; size_t out_size; int out_is_pinned;
    uint8_t* header; size_t header_cap; size_t header_size;   /* file header, composed on the host */
    /* stripe pipeline of host images (RGB frames of GJ_STRIPE_MIN_BYTES or more on the fused kernels): the image arrives in GJ_STRIPES pieces
     * on a copy stream, K1 runs on every piece as soon as it is there -- the transform hides behind the PCIe transfer */
    gj_stream_t copy_stream;
    void* ev_begin; void* ev_stripe[GJ_STRIPES];
    int stripes;                               /* GPUJPEG_B200_STRIPES (1 = off), default GJ_STRIPES */
    int k2_parts;                              /* GPUJPEG_B200_STRIPES_K2 (0 = K2 behind the last stripe only); -1 = not read yet */
    size_t stripe_min_bytes;                   /* GPUJPEG_B200_STRIPE_MIN_BYTES (tests), default GJ_STRIPE_MIN_BYTES */
    struct gj_header_extras extras;            /* enc_metadata (orientation), enc_exif_tag (user tags, owned) */
    int extras_dirty;                          /* an option changed what the header carries */
    /* gj_encoder_setup_coefficients: the frame's coefficients come from the transcoder, not from K1; the header carries these
     * quantisation tables and COM segments (extras points at them) */
    int coef_input;
    uint8_t comp_q[GJ_MAX_COMP][64];
    uint8_t comp_tq[GJ_MAX_COMP];
    uint8_t* com; size_t com_cap;

    /* timers [ref: src/gpujpeg_common_internal.h:414-422] */
    struct gj_timer t_to, t_from, t_pre, t_huff, t_gpu;
    int timers_ok;
    double t_stream_ms;
    struct gpujpeg_duration_stats stats;
    int stats_valid;
};

/* ---- small public helpers [ref: src/gpujpeg_encoder.c:47-110] ---- */
void gpujpeg_encoder_input_set_image(struct gpujpeg_encoder_input* input, uint8_t* image)
{
    input->type = GPUJPEG_ENCODER_INPUT_IMAGE;
    input->image = image;
    input->texture = NULL;
}
void gpujpeg_encoder_input_set_gpu_image(struct gpujpeg_encoder_input* input, uint8_t* image)
{
    input->type = GPUJPEG_ENCODER_INPUT_GPU_IMAGE;
    input->image = image;
    input->texture = NULL;
}
void gpujpeg_encoder_input_set_texture(struct gpujpeg_encoder_input* input, struct gpujpeg_opengl_texture* texture)
{
    input->type = GPUJPEG_ENCODER_INPUT_OPENGL_TEXTURE;
    input->image = NULL;
    input->texture = texture;
}
struct gpujpeg_encoder_input gpujpeg_encoder_input_image(uint8_t* image)
{
    struct gpujpeg_encoder_input r;
    gpujpeg_encoder_input_set_image(&r, image);
    return r;
}
struct gpujpeg_encoder_input gpujpeg_encoder_input_gpu_image(uint8_t* image)
{
    struct gpujpeg_encoder_input r;
    gpujpeg_encoder_input_set_gpu_image(&r, image);
    return r;
}
struct gpujpeg_encoder_input gpujpeg_encoder_input_texture(struct gpujpeg_opengl_texture* texture)
{
    struct gpujpeg_encoder_input r;
    gpujpeg_encoder_input_set_texture(&r, texture);
    return r;
}

/* [ref: src/gpujpeg_encoder.c:113-181] */
struct gpujpeg_encoder* gpujpeg_encoder_create(cudaStream_t stream)
{
    struct gpujpeg_encoder* e = (struct gpujpeg_encoder*)calloc(1, sizeof *e);
    if ( !e ) return NULL;
    e->stream = (gj_stream_t)stream;
    e->device = gj_cuda_get_device();
    e->quality = -1;
    e->header_type = GPUJPEG_HEADER_DEFAULT;
    e->k2_parts = -1;
    if ( e->device < 0 ) {
        GJ_ERR("Cannot get CUDA device: %s\n", gj_cuda_last_error());
        free(e);
        return NULL;
    }
    for ( int t = 0; t < 2; t++ )
        for ( int k = 0; k < 2; k++ )
            gj_huff_spec_default(t, k, &e->spec[t][k]);
    for ( int t = 0; t < 2; t++ )
        gj_enc_lut_build(&e->spec[t][0], &e->spec[t][1], &e->h_tab.lut[t]);
    if ( gj_cuda_malloc((void**)&e->d_tab, sizeof *e->d_tab) || gj_cuda_malloc((void**)&e->d_info, 64) ||
         gj_cuda_malloc_host((void**)&e->h_info, 64) || gj_cuda_malloc((void**)&e->d_counts, GJ_HUFF_COUNTS_BYTES) ||
         gj_cuda_malloc_host((void**)&e->h_counts, GJ_HUFF_COUNTS_BYTES) ) {
        GJ_ERR("Encoder allocation failed: %s\n", gj_cuda_last_error());
        gpujpeg_encoder_destroy(e);
        return NULL;
    }
    e->timers_ok = !(gj_timer_create(&e->t_to) || gj_timer_create(&e->t_from) || gj_timer_create(&e->t_pre) ||
                     gj_timer_create(&e->t_huff) || gj_timer_create(&e->t_gpu));
    return e;
}

int gpujpeg_encoder_destroy(struct gpujpeg_encoder* e)
{
    if ( !e ) return -1;
    gj_cuda_free(e->d_tab);
    gj_cuda_free(e->d_info);
    gj_cuda_free(e->d_counts);
    if ( e->h_counts ) gj_cuda_free_host(e->h_counts);
    gj_cuda_free(e->d_sos);
    free(e->h_pre);
    free(e->header);
    if ( e->copy_stream ) gj_cuda_stream_destroy(e->copy_stream);
    gj_cuda_event_destroy(e->ev_begin);
    for ( int i = 0; i < GJ_STRIPES; i++ )
        gj_cuda_event_destroy(e->ev_stripe[i]);
    gj_exif_tags_destroy((struct gj_exif_tags*)e->extras.exif_tags);
    free(e->com);
    gj_cuda_free(e->d_seg_pos);
    if ( e->h_seg_pos ) gj_cuda_free_host(e->h_seg_pos);
    gj_cuda_free_host(e->h_info);
    gj_cuda_free(e->d_raw);
    gj_cuda_free(e->d_coef);
    gj_cuda_free(e->d_planes);
    gj_cuda_free(e->d_nzmask);
    gj_cuda_free(e->d_tmp);
    gj_cuda_free(e->d_spill);
    gj_cuda_free(e->d_split);
    gj_cuda_free(e->d_seg_bytes);
    gj_cuda_free(e->d_seg_off);
    gj_cuda_free(e->d_stream);
    if ( e->out ) {
        if ( e->out_is_pinned ) gj_cuda_free_host(e->out);
        else free(e->out);
    }
    gj_timer_destroy(&e->t_to);
    gj_timer_destroy(&e->t_from);
    gj_timer_destroy(&e->t_pre);
    gj_timer_destroy(&e->t_huff);
    gj_timer_destroy(&e->t_gpu);
    free(e);
    return 0;
}

/* [ref: src/gpujpeg_encoder.c:290-317] */
int gpujpeg_encoder_suggest_restart_interval(const struct gpujpeg_image_parameters* param_image,
                                             gpujpeg_sampling_factor_t subsampling, bool interleaved, int verbose)
{
    const int comp_count = gpujpeg_pixel_format_get_comp_count(param_image->pixel_format);
    const double mpix = ((double)param_image->width * param_image->height * comp_count) / (1000000.0 * 3.0);
    int rst = mpix < 1.0 ? 4 : mpix < 3.0 ? 8 : mpix < 9.0 ? 10 : 12;
    if ( subsampling != GPUJPEG_SUBSAMPLING_444 && interleaved ) rst /= 2;
    if ( !interleaved ) rst *= comp_count;
    GJ_VERBOSE(verbose, "Auto-adjusting restart interval to %d for better performance.\n", rst);
    return rst;
}

static int grow(void** p, size_t* have, size_t want)
{
    if ( *have >= want ) return 0;
    gj_cuda_free(*p);
    *p = NULL;
    *have = 0;
    if ( gj_cuda_malloc(p, want) ) return -1;
    *have = want;
    return 0;
}

/* What this build encodes, and the input class gj_k1_choose turns into the frame's K1 (anything else fails loudly, there is no
 * CPU fallback):
 *   GJ_IN_RGB      GPUJPEG_444_U8_P012 + GPUJPEG_RGB -> YCbCr (BT.601 full range) JPEG, 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0:
 *                  the fused colour + FDCT kernels
 *   GJ_IN_SAMPLES  the image already holds the JPEG's components (colour space == internal colour space, or a single
 *                  component): GPUJPEG_U8, 444-u8-p012, 444/422/420-u8-p0p1p2, 422-u8-p1020; the JPEG takes the
 *                  format's own sampling [ref: src/gpujpeg_preprocessor.cu:296-311 "no transform" rule]
 *   GJ_IN_GENERIC  any of those pixel formats in GPUJPEG_RGB / _YCBCR_BT601 / _YCBCR_BT601_256LVLS / _YCBCR_BT709 with any of
 *                  the four samplings: one extra pass converts to the JPEG's component planes (gj_convert.cu), then
 *                  the sample kernel runs on the planes */
static int params_supported(const struct gpujpeg_parameters* p, const struct gpujpeg_image_parameters* pi)
{
    if ( pi->width < 1 || pi->height < 1 || pi->width > 65535 || pi->height > 65535 || pi->width_padding < 0 ) {
        GJ_ERR("Unsupported image size %dx%d.\n", pi->width, pi->height);
        return GJ_IN_UNSUPPORTED;
    }
    if ( p->restart_interval < 0 || p->restart_interval > 65535 ) {
        GJ_ERR("Restart interval %d cannot be stored in a DRI marker.\n", p->restart_interval);
        return GJ_IN_UNSUPPORTED;
    }
    /* YCbCr JPEG (JFIF header), RGB (Adobe APP14 header, every component coded with the luminance tables), or the
     * limited-range YCbCr spaces BT.601 / BT.709 (SPIFF header) [ref: src/gpujpeg_writer.c:456-475] */
    if ( p->color_space_internal != GPUJPEG_YCBCR_BT601_256LVLS &&
         !(p->comp_count >= 3 && (p->color_space_internal == GPUJPEG_RGB || p->color_space_internal == GPUJPEG_YCBCR_BT601 ||
                                  p->color_space_internal == GPUJPEG_YCBCR_BT709)) ) {
        GJ_ERR("Internal color space %s is not taken by this build.\n", gpujpeg_color_space_get_name(p->color_space_internal));
        return GJ_IN_UNSUPPORTED;
    }
    if ( pi->color_space == GPUJPEG_YCBCR_BT601 && p->color_space_internal == GPUJPEG_YCBCR_BT709 ) {
        /* the reference converts this pair with the full-range matrix (src/gpujpeg_colorspace.h:386-394); not restated */
        GJ_ERR("BT.601 input into a BT.709-internal JPEG is not taken by this build.\n");
        return GJ_IN_UNSUPPORTED;
    }
    if ( p->comp_count != 3 && p->comp_count != 1 && p->comp_count != 4 ) {
        GJ_ERR("This build encodes 1-, 3- and 4-component images only (comp_count = %d).\n", p->comp_count);
        return GJ_IN_UNSUPPORTED;
    }
    if ( pi->pixel_format == GPUJPEG_444_U8_P012 && pi->color_space == GPUJPEG_RGB && p->comp_count == 3 &&
         p->color_space_internal == GPUJPEG_YCBCR_BT601_256LVLS ) {
        /* luminance 1x1, 2x1, 1x2 or 2x2 with 1x1 chrominance: the sampling modes the reference has precompiled
         * preprocessor kernels for [ref: src/gpujpeg_preprocessor.cu:241-253] */
        const int lh = p->sampling_factor[0].horizontal, lv = p->sampling_factor[0].vertical;
        if ( lh < 1 || lh > 2 || lv < 1 || lv > 2 || p->sampling_factor[1].horizontal != 1 ||
             p->sampling_factor[1].vertical != 1 || p->sampling_factor[2].horizontal != 1 || p->sampling_factor[2].vertical != 1 ) {
            GJ_ERR("This build encodes 4:4:4, 4:2:2, 4:2:0 and 4:4:0 only (got %s).\n",
                   gpujpeg_subsampling_get_name(3, p->sampling_factor));
            return GJ_IN_UNSUPPORTED;
        }
        return GJ_IN_RGB;
    }
    struct gj_raw_layout rl;
    if ( gj_raw_layout_init(&rl, pi) ) {
        GJ_ERR("Pixel format %s (%dx%d, row padding %d) is not taken by this build.\n",
               gpujpeg_pixel_format_get_name(pi->pixel_format), pi->width, pi->height, pi->width_padding);
        return GJ_IN_UNSUPPORTED;
    }
    /* comp_count = 4: the alpha samples of a 4444-u8-p0123 image are coded as a fourth component (with the luminance tables
     * and the first component's sampling); with comp_count = 3 they are ignored [ref: src/gpujpeg_common.c:692-694,
     * src/gpujpeg_preprocessor.cu:131-138] */
    const int four = p->comp_count == 4;
    if ( four ? !(rl.comp_count == 3 && rl.alpha_off) : rl.comp_count != p->comp_count ) {
        GJ_ERR("Pixel format %s has %d components, the JPEG parameters ask for %d.\n",
               gpujpeg_pixel_format_get_name(pi->pixel_format), rl.comp_count + (rl.alpha_off ? 1 : 0), p->comp_count);
        return GJ_IN_UNSUPPORTED;
    }
    int needs_pass = four || (p->comp_count == 3 && pi->color_space != p->color_space_internal && pi->color_space != GPUJPEG_NONE);
    for ( int c = 0; c < p->comp_count && c < 3; c++ )
        if ( p->sampling_factor[c].horizontal != rl.sampling[c].horizontal ||
             p->sampling_factor[c].vertical != rl.sampling[c].vertical )
            needs_pass = 1;
    if ( needs_pass ) {
        const int lh = p->sampling_factor[0].horizontal, lv = p->sampling_factor[0].vertical;
        if ( p->comp_count < 3 || lh < 1 || lh > 2 || lv < 1 || lv > 2 || p->sampling_factor[1].horizontal != 1 ||
             p->sampling_factor[1].vertical != 1 || p->sampling_factor[2].horizontal != 1 || p->sampling_factor[2].vertical != 1 ||
             (four && (p->sampling_factor[3].horizontal != lh || p->sampling_factor[3].vertical != lv)) ) {
            GJ_ERR("This build encodes 4:4:4, 4:2:2, 4:2:0 and 4:4:0 only (got %s).\n",
                   gpujpeg_subsampling_get_name(p->comp_count, p->sampling_factor));
            return GJ_IN_UNSUPPORTED;
        }
        if ( pi->color_space != GPUJPEG_NONE && pi->color_space != GPUJPEG_RGB && pi->color_space != GPUJPEG_YCBCR_BT601 &&
             pi->color_space != GPUJPEG_YCBCR_BT601_256LVLS && pi->color_space != GPUJPEG_YCBCR_BT709 ) {
            GJ_ERR("Colour space %s is not taken by this build.\n", gpujpeg_color_space_get_name(pi->color_space));
            return GJ_IN_UNSUPPORTED;
        }
        if ( (pi->width & 1) && rl.sampling[0].horizontal == 2 && pi->pixel_format != GPUJPEG_420_U8_P0P1P2 ) {
            /* the reference's generic kernel and its planar copy disagree on odd widths of 4:2:2 data */
            GJ_ERR("Odd widths are only taken without colour / sampling conversion for this pixel format.\n");
            return GJ_IN_UNSUPPORTED;
        }
        return GJ_IN_GENERIC;
    }
    return GJ_IN_SAMPLES;
}

/* enc_opt_writer=libjpeg takes what libjpeg-turbo's jpeg_write_scanlines takes with jpeg_set_defaults: RGB 444-u8-p012 into an
 * interleaved YCbCr JFIF frame at 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0, or GPUJPEG_U8 samples into a grey frame; the header libjpeg
 * writes, so nothing that changes it.  Checked before anything of the encoder changes: a refused frame leaves it as it was. */
static int libjpeg_supported(const struct gpujpeg_encoder* e, const struct gpujpeg_parameters* p, const struct gpujpeg_image_parameters* pi)
{
    const char* why = NULL;
    if ( p->color_space_internal != GPUJPEG_YCBCR_BT601_256LVLS ) why = "an internal colour space other than YCbCr JPEG";
    else if ( p->comp_count == 3 ) {
        if ( pi->pixel_format != GPUJPEG_444_U8_P012 || pi->color_space != GPUJPEG_RGB ) why = "input other than RGB 444-u8-p012";
        else if ( !p->interleaved ) why = "a non-interleaved colour frame";
    }
    else if ( p->comp_count == 1 ) {
        if ( pi->pixel_format != GPUJPEG_U8 || pi->color_space == GPUJPEG_YCBCR_BT601 || pi->color_space == GPUJPEG_YCBCR_BT709 )
            why = "grey input other than full-range GPUJPEG_U8";
    }
    else why = "a component count other than 1 or 3";
    if ( !why && (e->flipped || e->channel_remap) ) why = "enc_opt_flipped / enc_opt_channel_remap";
    if ( !why && p->segment_info ) why = "segment info";
    if ( !why && ((e->header_type != GPUJPEG_HEADER_DEFAULT && e->header_type != GPUJPEG_HEADER_JFIF) || e->extras.exif_tags ||
                  e->extras.metadata.vals[GPUJPEG_METADATA_ORIENTATION].set) )
        why = "a header other than JFIF (enc_hdr, enc_exif_tag, enc_metadata)";
    if ( why ) {
        GJ_ERR(GPUJPEG_ENC_OPT_WRITER "=" GPUJPEG_ENC_WRITER_VAL_LIBJPEG " does not take %s.\n", why);
        return 0;
    }
    return 1;
}

/* K1 as the frame's plan says: the generic pass into the planes and their flip, then the fused kernels on MCU rows [my0, my1) or
 * the per-block one on the image or the planes */
static int launch_k1(struct gpujpeg_encoder* e, const uint8_t* d_raw, int my0, int my1)
{
    const struct gj_geometry* g = &e->geo;
    const struct gj_k1_plan* p = &e->k1;
    if ( p->kernel == GJ_K1_FUSED )   /* (grey input: rows of the U8 image) */
        return gj_launch_fdct_fused(p, g, d_raw, g->comp_count == 1 ? (int)e->raw.comp[0].pitch : g->pitch, my0, my1, &e->h_tab,
                                    (const uint8_t(*)[64])e->raw_q, e->d_coef, e->d_nzmask, e->stream);
    if ( !p->convert )
        return gj_launch_fdct_blocks(p, d_raw, &e->raw, g->comp, g->comp_count, g->lay.comp_tbl, &e->h_tab, e->d_coef, e->d_nzmask,
                                     e->stream);
    struct gj_raw_layout pl;
    struct gj_comp_geo padded[GJ_MAX_COMP];
    gj_planes_layout(&pl, padded, g->comp, g->comp_count, 8);
    if ( gj_launch_convert_in(d_raw, &e->raw, e->param_image.pixel_format, e->param_image.color_space, e->param.color_space_internal,
                              g->width, g->height, e->d_planes, pl.size, g->comp, g->comp_count, g->max_hs, g->max_vs, e->stream) )
        return -1;
    if ( p->flip == GJ_K1_FLIP_PLANES && gj_launch_flip_planes(e->d_planes, padded, g->comp_count, e->stream) ) return -1;
    return gj_launch_fdct_blocks(p, e->d_planes, &pl, padded, g->comp_count, g->lay.comp_tbl, &e->h_tab, e->d_coef, e->d_nzmask,
                                 e->stream);
}

static void fill_huff_args(const struct gpujpeg_encoder* e, struct gj_huff_enc_args* ha);

/* The stripe pipeline applies to what the fused RGB kernels (either writer's) take as it comes (k1.stripes), on frames large enough */
static int stripes_usable(struct gpujpeg_encoder* e)
{
    const struct gj_geometry* g = &e->geo;
    if ( !e->k1.stripes ) return 0;
    if ( e->stripes == 0 ) {
        const char* v = getenv("GPUJPEG_B200_STRIPES");
        const char* m = getenv("GPUJPEG_B200_STRIPE_MIN_BYTES");
        e->stripe_min_bytes = m ? (size_t)strtoull(m, NULL, 0) : GJ_STRIPE_MIN_BYTES;
        e->stripes = v ? atoi(v) : GJ_STRIPES;
        if ( e->stripes < 1 ) e->stripes = 1;
        if ( e->stripes > GJ_STRIPES ) e->stripes = GJ_STRIPES;
    }
    if ( e->stripes < 2 || g->bcy / g->max_vs < 2 * e->stripes || g->raw_size < e->stripe_min_bytes ) return 0;
    if ( !e->copy_stream ) {
        if ( gj_cuda_stream_create(&e->copy_stream) || gj_cuda_event_create(&e->ev_begin) ) {
            e->stripes = 1;
            return 0;
        }
        for ( int i = 0; i < GJ_STRIPES; i++ )
            if ( gj_cuda_event_create(&e->ev_stripe[i]) ) {
                e->stripes = 1;
                return 0;
            }
    }
    return 1;
}

/* H2D of the host image in stripes of whole block rows on the copy stream; K1 of a stripe on the coder's stream as soon as the
 * stripe has arrived.  The copy stream starts behind everything the coder's stream holds (the previous frame's K1 reads d_raw). */
static int encode_striped(struct gpujpeg_encoder* e, const uint8_t* h_image, int* k2_done)
{
    const struct gj_geometry* g = &e->geo;
    if ( gj_cuda_event_record(e->ev_begin, e->stream) || gj_cuda_stream_wait_event(e->copy_stream, e->ev_begin) ) return -1;
    /* K2 as well, stripe by stripe, where a stripe's restart segments can be told from its rows (4:4:4: MCU = block position) and
     * are short enough for the packed kernel: the segments that lie completely inside the rows transformed so far */
    struct gj_huff_enc_args ha;
    fill_huff_args(e, &ha);
    if ( e->k2_parts < 0 ) {
        const char* v = getenv("GPUJPEG_B200_STRIPES_K2");
        e->k2_parts = !(v && v[0] == '0');
    }
    /* (fitted tables are known only when the last stripe has been counted: then K2 runs behind the stripes) */
    const int parts = e->k2_parts && !e->huff_optimized && gj_huffman_encode_parts_eligible(&ha);
    int segs_done[GJ_MAX_COMP] = {0, 0, 0, 0};
    const int mcu_h = 8 * g->max_vs;                                  /* image rows per MCU row (4:4:4: one block row) */
    const int mcu_rows = e->k1.mcu_rows;
    for ( int i = 0; i < e->stripes; i++ ) {
        const int my0 = (int)((long long)mcu_rows * i / e->stripes), my1 = (int)((long long)mcu_rows * (i + 1) / e->stripes);
        const size_t row0 = (size_t)my0 * mcu_h, row1 = (size_t)my1 * mcu_h < (size_t)g->height ? (size_t)my1 * mcu_h : (size_t)g->height;
        const size_t off = row0 * (size_t)g->pitch;
        const size_t bytes = (i + 1 == e->stripes ? g->raw_size : row1 * (size_t)g->pitch) - off;
        if ( gj_cuda_memcpy_h2d_async(e->d_raw + off, h_image + off, bytes, e->copy_stream) ||
             gj_cuda_event_record(e->ev_stripe[i], e->copy_stream) || gj_cuda_stream_wait_event(e->stream, e->ev_stripe[i]) )
            return -1;
        if ( launch_k1(e, e->d_raw, my0, my1) ) return -1;
        if ( parts ) {
            int lo[GJ_MAX_COMP] = {0, 0, 0, 0}, n[GJ_MAX_COMP] = {0, 0, 0, 0};
            for ( int k = 0; k < g->scan_count; k++ ) {
                const int segs = g->lay.scan_seg_begin[k + 1] - g->lay.scan_seg_begin[k];
                long long hi = i + 1 == e->stripes ? segs : (long long)my1 * g->bcx / g->seg_mcu;   /* whole segments in rows [0, my1) */
                if ( hi > segs ) hi = segs;
                lo[k] = segs_done[k];
                n[k] = (int)hi - segs_done[k];
                segs_done[k] = (int)hi;
            }
            if ( gj_launch_huffman_encode_part(&ha, i == 0, lo, n, e->stream) ) {
                e->info_clean = 0;
                return -1;
            }
        }
    }
    if ( parts ) {
        const int rc = gj_launch_huffman_place(&ha, e->stream);
        e->d_info_cur = ha.d_info;
        e->info_parity ^= 1;
        e->info_clean = rc == 0;
        if ( rc ) return -1;
        *k2_done = 1;
    }
    return 0;
}

/* K2 on the frame K1 left in place.  The 32-byte result block alternates between two halves of d_info: the tail kernel of
 * one launch clears the half the next launch accumulates into, so no memset stands between K1 and K2. */
static int launch_k2(struct gpujpeg_encoder* e)
{
    struct gj_huff_enc_args ha;
    fill_huff_args(e, &ha);
    const int rc = gj_launch_huffman_encode(&ha, e->stream);
    e->d_info_cur = ha.d_info;
    e->info_parity ^= 1;
    e->info_clean = rc == 0;   /* after a failed launch nothing is known about either half: the next launch clears its own */
    return rc;
}

static void fill_huff_args(const struct gpujpeg_encoder* e, struct gj_huff_enc_args* ha)
{
    const struct gj_geometry* g = &e->geo;
    memset(ha, 0, sizeof *ha);
    ha->d_coef = e->d_coef;
    ha->d_nzmask = e->d_nzmask;
    ha->lay = g->lay;
    ha->seg_mcu = g->seg_mcu;
    ha->d_tmp = e->d_tmp;
    ha->d_spill = e->d_spill;
    ha->slot_stride = e->slot_stride;
    ha->d_seg_bytes = e->d_seg_bytes;
    ha->d_seg_off = e->d_seg_off;
    ha->d_stream = e->d_stream;
    ha->stream_cap = g->stream_cap;
    ha->header_size = (uint32_t)e->header_size;
    ha->d_sos = e->d_sos;
    for ( int s = 0; s < GJ_MAX_COMP; s++ ) {
        ha->pre_len[s] = e->pre_len[s];
        ha->pre_off[s] = e->pre_off[s];
    }
    ha->d_seg_pos = e->with_segment_info ? e->d_seg_pos : NULL;
    ha->d_info = e->d_info + 4 * e->info_parity;
    ha->d_info_next = e->d_info + 4 * (e->info_parity ^ 1);
    ha->info_is_zero = e->info_clean;
    ha->d_tables = e->d_tab;
    ha->d_split = e->d_split;
    ha->split_bytes = e->d_split_size;
}

/* the symbol statistics of the frame K1 left in place (enqueued only) */
static int launch_stats(struct gpujpeg_encoder* e)
{
    struct gj_huff_enc_args ha;
    fill_huff_args(e, &ha);
    if ( gj_launch_huffman_stats(&ha, e->d_counts, e->stream) ) return -1;
    e->counts_valid = 1;
    return 0;
}

/* enc_opt_huffman=optimized, between K1 and K2: statistics -> (one synchronisation) -> the tables T.81 Annex K.2 fits to them
 * for the classes the frame's components use (Annex K for an unused class) -> encoder LUTs on the device and the file header.
 * One table set per class per frame, in the file header, as libjpeg writes baseline streams. */
static int fit_huffman_tables(struct gpujpeg_encoder* e)
{
    const struct gj_geometry* g = &e->geo;
    if ( launch_stats(e) || gj_cuda_memcpy_d2h_async(e->h_counts, e->d_counts, GJ_HUFF_COUNTS_BYTES, e->stream) ||
         gj_cuda_stream_sync(e->stream) )
        return -1;
    int used[2] = {0, 0};
    for ( int c = 0; c < g->comp_count; c++ )
        used[g->lay.comp_tbl[c]] = 1;
    for ( int t = 0; t < 2; t++ ) {
        for ( int k = 0; k < 2; k++ ) {
            if ( used[t] ) gj_huff_spec_optimal(e->h_counts + (t * 2 + k) * 256, &e->spec[t][k]);
            else gj_huff_spec_default(t, k, &e->spec[t][k]);
        }
        gj_enc_lut_build(&e->spec[t][0], &e->spec[t][1], &e->h_tab.lut[t]);
    }
    e->spec_custom = 1;
    /* the DHT segments of fitted tables are longer than Annex K's: up to 256 values each */
    const size_t need = GJ_HEADER_BASE_CAP + 4 * 256 + gj_exif_tags_bytes(e->extras.exif_tags) + e->extras.com_size;
    if ( need > e->header_cap ) {
        free(e->header);
        e->header = (uint8_t*)malloc(need);
        e->header_cap = e->header ? need : 0;
        if ( !e->header ) return -1;
    }
    e->header_size = gj_write_header(e->header, &e->param, &e->param_image, e->raw_q, e->spec, e->header_type, &e->extras);
    if ( e->header_size + 64 > g->stream_cap ) {
        GJ_ERR("The header (%zu bytes) does not fit the stream buffer of a %dx%d image.\n", e->header_size, g->width, g->height);
        return -1;
    }
    return gj_cuda_memcpy_h2d_async(e->d_tab, &e->h_tab, sizeof e->h_tab, e->stream);
}

/* the K1 request of a frame of input class `in` (params_supported; ignored for the transcoder's coefficients) */
static struct gj_k1_request k1_request(const struct gpujpeg_encoder* e, int in)
{
    struct gj_k1_request r;
    memset(&r, 0, sizeof r);
    r.in = in;
    r.libjpeg = e->writer_libjpeg;
    r.flipped = e->flipped != 0;
    r.channel_remap = e->channel_remap != 0;
    r.coef_input = e->coef_input;
    return r;
}

/* the host output buffer: at least `size` bytes, pinned or not as asked */
static int reserve_out(struct gpujpeg_encoder* e, size_t size)
{
    if ( e->out_size >= size && e->out_is_pinned == e->out_pinned ) return 0;
    if ( e->out ) {
        if ( e->out_is_pinned ) gj_cuda_free_host(e->out);
        else free(e->out);
    }
    e->out = NULL;
    e->out_size = 0;
    e->out_is_pinned = e->out_pinned;
    if ( e->out_pinned ) {
        if ( gj_cuda_malloc_host((void**)&e->out, size) ) return -1;
    }
    else if ( !(e->out = (uint8_t*)malloc(size)) ) {
        return -1;
    }
    e->out_size = size;
    return 0;
}

/* (re)build everything that depends on geometry [ref: src/gpujpeg_common.c:628-1106] */
static int encoder_init_image(struct gpujpeg_encoder* e, const struct gpujpeg_parameters* p,
                              const struct gpujpeg_image_parameters* pi, const struct gj_k1_request* k1)
{
    gj_geometry_init(&e->geo, p, pi);
    e->geo.stream_cap += e->extras.com_size;
    e->k1_req = *k1;
    gj_k1_choose(&e->geo, k1, &e->k1);
    if ( e->k1.raw_layout && gj_raw_layout_init(&e->raw, pi) ) return -1;
    if ( e->k1.convert && grow((void**)&e->d_planes, &e->d_planes_size, e->k1.planes_bytes) ) return -1;
    const struct gj_geometry* g = &e->geo;
    size_t coef_bytes = g->coef_count * sizeof(int16_t);
    const size_t segblk_all = (size_t)g->seg_mcu * (size_t)g->lay.bpm;
    size_t first_stride = (segblk_all * 48 + 2 + 127) / 128 * 128;
    if ( first_stride > g->slot_stride ) first_stride = g->slot_stride;
    if ( e->slot_stride < first_stride || e->slot_stride > g->slot_stride ) e->slot_stride = first_stride;
    size_t tmp_bytes = (size_t)g->seg_count * e->slot_stride + 256;
    /* overflow area of the per-block bit strings: 32 words per block of a short segment (packed kernel, <= 40 blocks),
     * per lane of a warp otherwise (streaming kernel); the chunks of few long segments need status words instead */
    const int segblk = g->seg_mcu * g->lay.bpm;
    size_t spill_bytes = (size_t)g->seg_count * (segblk <= 40 ? segblk : 32) * 32 * sizeof(uint32_t);
    const size_t split_bytes = gj_huffman_split_status_bytes(g->seg_count, segblk, g->slot_stride);
    if ( grow((void**)&e->d_coef, &e->d_coef_size, coef_bytes) ||
         grow((void**)&e->d_nzmask, &e->d_nzmask_size, g->coef_count / 64 * sizeof(uint64_t)) ||
         grow((void**)&e->d_tmp, &e->d_tmp_size, tmp_bytes) ||
         grow((void**)&e->d_spill, &e->d_spill_size, spill_bytes) ||
         grow((void**)&e->d_split, &e->d_split_size, split_bytes) ||
         grow((void**)&e->d_stream, &e->d_stream_size, g->stream_cap + 64) ) {
        GJ_ERR("Encoder device allocation failed (%zu + %zu + %zu bytes): %s\n", coef_bytes, tmp_bytes, g->stream_cap,
               gj_cuda_last_error());
        return -1;
    }
    if ( g->seg_count > e->seg_alloc ) {
        gj_cuda_free(e->d_seg_bytes);
        gj_cuda_free(e->d_seg_off);
        e->d_seg_bytes = NULL;
        e->d_seg_off = NULL;
        e->seg_alloc = 0;
        if ( gj_cuda_malloc((void**)&e->d_seg_bytes, (size_t)g->seg_count * 4) ||
             gj_cuda_malloc((void**)&e->d_seg_off, (size_t)g->seg_count * 8) )
            return -1;
        e->seg_alloc = g->seg_count;
    }
    if ( reserve_out(e, g->stream_cap) ) return -1;
    e->param = *p;
    e->param_image = *pi;
    e->initialised = 1;
    return 0;
}

static int same_image(const struct gpujpeg_image_parameters* a, const struct gpujpeg_image_parameters* b)
{
    return a->width == b->width && a->height == b->height && a->color_space == b->color_space &&
           a->pixel_format == b->pixel_format && a->width_padding == b->width_padding;
}
/* sampling factors in the packed form of GPUJPEG_SUBSAMPLING_* (one nibble pair per component) */
static gpujpeg_sampling_factor_t packed_sampling(const struct gpujpeg_parameters* p)
{
    gpujpeg_sampling_factor_t r = 0;
    for ( int c = 0; c < p->comp_count && c < 4; c++ )
        r |= (gpujpeg_sampling_factor_t)p->sampling_factor[c].horizontal << (28 - 8 * c) |
             (gpujpeg_sampling_factor_t)p->sampling_factor[c].vertical << (24 - 8 * c);
    return r;
}

static int same_param(const struct gpujpeg_parameters* a, const struct gpujpeg_parameters* b)
{
    /* everything but verbose / perf_stats / quality [ref: src/gpujpeg_common.c:348-367] */
    if ( a->restart_interval != b->restart_interval || a->interleaved != b->interleaved ||
         a->segment_info != b->segment_info || a->comp_count != b->comp_count ||
         a->color_space_internal != b->color_space_internal )
        return 0;
    for ( int c = 0; c < a->comp_count; c++ )
        if ( a->sampling_factor[c].horizontal != b->sampling_factor[c].horizontal ||
             a->sampling_factor[c].vertical != b->sampling_factor[c].vertical )
            return 0;
    return 1;
}

/* [ref: src/gpujpeg_encoder.c:319-348] */
static struct gpujpeg_parameters adjust_params(struct gpujpeg_encoder* e, const struct gpujpeg_parameters* param,
                                               const struct gpujpeg_image_parameters* pi, int img_changed)
{
    struct gpujpeg_parameters a = *param;
    if ( param->comp_count == 0 ) {
        if ( img_changed || !e->initialised ) {
            const int n = gpujpeg_pixel_format_get_comp_count(pi->pixel_format);
            a.comp_count = n > 3 ? 3 : n;
            /* the pixel format's own sampling [ref: src/gpujpeg_encoder.c:327-330] */
            struct gj_raw_layout rl;
            const int known = gj_raw_layout_init(&rl, pi) == 0;
            memset(a.sampling_factor, 0, sizeof a.sampling_factor);
            for ( int c = 0; c < a.comp_count; c++ ) {
                a.sampling_factor[c].horizontal = known ? rl.sampling[c].horizontal : 1;
                a.sampling_factor[c].vertical = known ? rl.sampling[c].vertical : 1;
            }
        }
        else {
            a.comp_count = e->param.comp_count;
            memcpy(a.sampling_factor, e->param.sampling_factor, sizeof a.sampling_factor);
        }
    }
    if ( param->restart_interval == RESTART_AUTO ) {
        if ( img_changed || !e->initialised || a.interleaved != e->param.interleaved )
            a.restart_interval =
                gpujpeg_encoder_suggest_restart_interval(pi, packed_sampling(&a), a.interleaved, a.verbose);
        else
            a.restart_interval = e->param.restart_interval;
    }
    return a;
}

int gpujpeg_encoder_allocate(struct gpujpeg_encoder* encoder, const struct gpujpeg_parameters* param,
                             const struct gpujpeg_image_parameters* param_image,
                             enum gpujpeg_encoder_input_type image_input_type)
{
    struct gpujpeg_parameters a = adjust_params(encoder, param, param_image, 1);
    const int in = params_supported(&a, param_image);
    if ( !in ) return -1;
    const struct gj_k1_request k1 = k1_request(encoder, in);
    if ( encoder_init_image(encoder, &a, param_image, &k1) ) return -1;
    if ( image_input_type == GPUJPEG_ENCODER_INPUT_IMAGE &&
         grow((void**)&encoder->d_raw, &encoder->d_raw_size, encoder->geo.raw_size) )
        return -1;
    return 0;
}

/* [ref: src/gpujpeg_encoder.c:183-288] memory model of this build: raw + coefficients + scan tmp + stream */
size_t gpujpeg_encoder_max_memory(struct gpujpeg_parameters* param, struct gpujpeg_image_parameters* param_image,
                                  enum gpujpeg_encoder_input_type image_input_type, int max_pixels)
{
    struct gpujpeg_image_parameters pi = *param_image;
    struct gpujpeg_parameters p = *param;
    if ( p.comp_count == 0 ) p.comp_count = 3;
    pi.width = 8 * (int)((max_pixels > 0 ? (size_t)max_pixels : 0) / 8 / 8 + 1);
    pi.height = 8 * 8;
    if ( pi.width < 8 ) pi.width = 8;
    /* use a squarish estimate: memory is linear in pixel count */
    struct gj_geometry g;
    pi.width = 4096;
    pi.height = (max_pixels + 4095) / 4096;
    if ( pi.height < 1 ) pi.height = 1;
    if ( p.restart_interval == RESTART_AUTO ) p.restart_interval = 36;
    gj_geometry_init(&g, &p, &pi);
    /* scan slots at their initial size (48 bytes per block); denser content grows them, up to 416 bytes per block */
    size_t total = g.coef_count * 2 + (size_t)g.seg_count * (((size_t)g.seg_mcu * g.lay.bpm * 48 + 2 + 127) / 128 * 128) + g.stream_cap +
                   (size_t)g.seg_count * 12;
    if ( image_input_type == GPUJPEG_ENCODER_INPUT_IMAGE ) total += g.raw_size;
    return total;
}

size_t gpujpeg_encoder_max_pixels(struct gpujpeg_parameters* param, struct gpujpeg_image_parameters* param_image,
                                  enum gpujpeg_encoder_input_type image_input_type, size_t memory_size, int* max_pixels)
{
    /* bisection over the linear model above [ref: src/gpujpeg_encoder.c:183-262] */
    int lo = 0, hi = 1 << 30;
    while ( hi - lo > 4096 ) {
        const int mid = lo + (hi - lo) / 2;
        if ( gpujpeg_encoder_max_memory(param, param_image, image_input_type, mid) <= memory_size ) lo = mid;
        else hi = mid;
    }
    if ( max_pixels ) *max_pixels = lo;
    return lo ? gpujpeg_encoder_max_memory(param, param_image, image_input_type, lo) : 0;
}

/* enc_opt_huffman=standard after fitted tables: back to Annex K (LUTs, header and device copy are to be rebuilt); 1 if so */
static int standard_tables_back(struct gpujpeg_encoder* e)
{
    if ( e->huff_optimized || !e->spec_custom ) return 0;
    for ( int t = 0; t < 2; t++ ) {
        for ( int k = 0; k < 2; k++ )
            gj_huff_spec_default(t, k, &e->spec[t][k]);
        gj_enc_lut_build(&e->spec[t][0], &e->spec[t][1], &e->h_tab.lut[t]);
    }
    e->spec_custom = 0;
    return 1;
}

/* the file header and what precedes every scan, composed on the host, and the tables uploaded */
static int compose_headers(struct gpujpeg_encoder* e)
{
    const struct gj_geometry* g = &e->geo;
    e->header_written = e->header_type;
    e->extras_dirty = 0;
    const size_t need = GJ_HEADER_BASE_CAP + gj_exif_tags_bytes(e->extras.exif_tags) + e->extras.com_size;
    if ( need > e->header_cap ) {
        free(e->header);
        e->header = (uint8_t*)malloc(need);
        e->header_cap = e->header ? need : 0;
        if ( !e->header ) {
            GJ_ERR("Encoder header allocation failed (%zu bytes).\n", need);
            return -1;
        }
    }
    /* host codestream writer: file header + SOS headers, composed once per parameter change */
    e->header_size = gj_write_header(e->header, &e->param, &e->param_image, e->raw_q, e->spec, e->header_type, &e->extras);
    if ( e->header_size + 64 > g->stream_cap ) {
        GJ_ERR("The header (%zu bytes) does not fit the stream buffer of a %dx%d image.\n", e->header_size, g->width, g->height);
        return -1;
    }
    /* what precedes every scan's data: [APP13 segment-info headers, positions filled in after the frame is coded] SOS */
    e->with_segment_info = e->param.segment_info && e->param.restart_interval > 0;
    size_t pre_total = 0;
    for ( int s = 0; s < GJ_MAX_COMP; s++ ) {
        e->pre_off[s] = (int)pre_total;
        e->pre_len[s] = 0;
        if ( s >= g->scan_count ) continue;
        const int segs = g->lay.scan_seg_begin[s + 1] - g->lay.scan_seg_begin[s];
        e->pre_len[s] = (int)((e->with_segment_info ? gj_write_segment_info_headers(NULL, s, segs) : 0) + 16);
        pre_total += (size_t)e->pre_len[s];
    }
    if ( pre_total > e->h_pre_size ) {
        free(e->h_pre);
        e->h_pre = (uint8_t*)malloc(pre_total);
        e->h_pre_size = e->h_pre ? pre_total : 0;
    }
    if ( !e->h_pre || grow((void**)&e->d_sos, &e->d_sos_size, pre_total) ) {
        GJ_ERR("Encoder scan header allocation failed (%zu bytes).\n", pre_total);
        return -1;
    }
    pre_total = 0;
    for ( int s = 0; s < g->scan_count; s++ ) {
        const int segs = g->lay.scan_seg_begin[s + 1] - g->lay.scan_seg_begin[s];
        uint8_t* p = e->h_pre + pre_total;
        size_t n = e->with_segment_info ? gj_write_segment_info_headers(p, s, segs) : 0;
        n += gj_write_sos(p + n, &e->param, s);
        e->pre_off[s] = (int)pre_total;
        e->pre_len[s] = (int)n;
        pre_total += n;
    }
    if ( e->with_segment_info && (size_t)g->seg_count * 8 > e->seg_pos_size ) {
        gj_cuda_free(e->d_seg_pos);
        if ( e->h_seg_pos ) gj_cuda_free_host(e->h_seg_pos);
        e->d_seg_pos = NULL;
        e->h_seg_pos = NULL;
        e->seg_pos_size = 0;
        if ( gj_cuda_malloc((void**)&e->d_seg_pos, (size_t)g->seg_count * 8) ||
             gj_cuda_malloc_host((void**)&e->h_seg_pos, (size_t)g->seg_count * 8) ) {
            GJ_ERR("Encoder segment info allocation failed: %s\n", gj_cuda_last_error());
            return -1;
        }
        e->seg_pos_size = (size_t)g->seg_count * 8;
    }
    if ( gj_cuda_memcpy_h2d_async(e->d_tab, &e->h_tab, sizeof e->h_tab, e->stream) ||
         gj_cuda_memcpy_h2d_async(e->d_sos, e->h_pre, pre_total, e->stream) ||
         gj_cuda_stream_sync(e->stream) ) {
        GJ_ERR("Encoder table upload failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    return 0;
}

/* What follows K1: the fitted tables (enc_opt_huffman=optimized), K2 (again with larger slots if a segment did not fit), the size,
 * the payload and the header into the host buffer, the segment-info tables.  k2_done: the stripe pipeline has run K2. */
static int encode_tail(struct gpujpeg_encoder* e, int k2_done, int stats, uint8_t** out, size_t* out_size)
{
    const struct gj_geometry* g = &e->geo;
    if ( !k2_done && e->huff_optimized && fit_huffman_tables(e) ) {
        GJ_ERR("Huffman statistics / table construction failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( !k2_done && launch_k2(e) ) {
        GJ_ERR("Huffman encoder launch failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( stats && e->timers_ok ) {
        gj_timer_stop(&e->t_huff, e->stream);
        gj_timer_stop(&e->t_gpu, e->stream);
        gj_timer_start(&e->t_from, e->stream);
    }
    /* the only two synchronisation points of a frame: size, then payload */
    if ( gj_cuda_memcpy_d2h_async(e->h_info, e->d_info_cur, 32, e->stream) || gj_cuda_stream_sync(e->stream) ) {
        GJ_ERR("Encoder failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( e->h_info[1] & 2 ) {
        /* a restart segment did not fit its slot: K2 counted what it needs (h_info[2]); enlarge the slots and run K2 again on
         * the coefficients K1 left in place.  Happens once per encoder for unusually dense content. */
        size_t need = ((size_t)e->h_info[2] + 127) / 128 * 128;
        if ( need > g->slot_stride ) need = g->slot_stride;
        if ( need <= e->slot_stride ) need = g->slot_stride;
        GJ_VERBOSE(e->param.verbose, "Enlarging the scan buffer to %zu bytes per restart segment.\n", need);
        e->slot_stride = need;
        if ( grow((void**)&e->d_tmp, &e->d_tmp_size, (size_t)g->seg_count * e->slot_stride + 256) ) {
            GJ_ERR("Encoder device allocation failed (%zu bytes): %s\n", (size_t)g->seg_count * e->slot_stride, gj_cuda_last_error());
            return -1;
        }
        if ( launch_k2(e) || gj_cuda_memcpy_d2h_async(e->h_info, e->d_info_cur, 32, e->stream) ||
             gj_cuda_stream_sync(e->stream) ) {
            GJ_ERR("Encoder failed: %s\n", gj_cuda_last_error());
            return -1;
        }
    }
    if ( e->h_info[1] == 1 && e->h_info[0] > g->stream_cap ) {
        /* the finished stream outgrew the reference's budget of 2 bytes per sample (K2 counted it all, h_info[0]): a legal
         * frame can code to more -- a transcoded stream of blocks with 63 AC coefficients at +-1023 takes about 207 bytes per
         * block, and the worst 8-bit pixel blocks at q100 with short restart intervals exceed 128 bytes per block too.  Grow
         * the device stream and the host output buffer to that size and run K2 again; the size stays for the encoder's
         * later frames of this geometry, as the slot size above does. */
        const size_t need = ((size_t)e->h_info[0] + 4095) / 4096 * 4096;
        GJ_VERBOSE(e->param.verbose, "Enlarging the stream buffer to %zu bytes.\n", need);
        if ( grow((void**)&e->d_stream, &e->d_stream_size, need + 64) || reserve_out(e, need) ) {
            GJ_ERR("Encoder allocation failed (%zu bytes): %s\n", need, gj_cuda_last_error());
            return -1;
        }
        e->geo.stream_cap = need;
        if ( launch_k2(e) || gj_cuda_memcpy_d2h_async(e->h_info, e->d_info_cur, 32, e->stream) ||
             gj_cuda_stream_sync(e->stream) ) {
            GJ_ERR("Encoder failed: %s\n", gj_cuda_last_error());
            return -1;
        }
    }
    const size_t total = (size_t)e->h_info[0];
    if ( e->h_info[1] || total > e->out_size || total < e->header_size + 2 ) {
        GJ_ERR("Compressed image (%zu bytes) does not fit the output buffer (%zu bytes)!\n", total, e->out_size);
        return -1;
    }
    if ( gj_cuda_memcpy_d2h_async(e->out + e->header_size, e->d_stream + e->header_size, total - e->header_size,
                                  e->stream) ||
         (e->with_segment_info && gj_cuda_memcpy_d2h_async(e->h_seg_pos, e->d_seg_pos, (size_t)g->seg_count * 8, e->stream)) ) {
        GJ_ERR("Encoder copy of compressed data failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( stats && e->timers_ok ) gj_timer_stop(&e->t_from, e->stream);
    const double t_fmt = stats ? gpujpeg_get_time() : 0.0;
    memcpy(e->out, e->header, e->header_size); /* host writer output, overlaps the copy */
    e->t_stream_ms = stats ? (gpujpeg_get_time() - t_fmt) * 1000.0 : 0.0;
    if ( gj_cuda_stream_sync(e->stream) ) {
        GJ_ERR("Encoder copy of compressed data failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( e->with_segment_info ) {
        /* the APP13 tables in front of every scan: position of every segment relative to the scan's first byte, then the
         * scan's end [ref: src/gpujpeg_writer.c:522-546, src/gpujpeg_encoder.c:575-621] */
        for ( int s = 0; s < g->scan_count; s++ ) {
            const int first = g->lay.scan_seg_begin[s], segs = g->lay.scan_seg_begin[s + 1] - first;
            const uint64_t scan_start = e->h_seg_pos[first];
            const uint64_t scan_end = s + 1 < g->scan_count ? e->h_seg_pos[g->lay.scan_seg_begin[s + 1]] - (uint64_t)e->pre_len[s + 1]
                                                            : (uint64_t)total - 2;
            uint8_t* table = e->out + scan_start - (uint64_t)e->pre_len[s];
            for ( int i = 0; i <= segs; i++ ) {
                const uint32_t pos = (uint32_t)((i < segs ? e->h_seg_pos[first + i] : scan_end) - scan_start);
                uint8_t* q = table + gj_segment_info_entry_offset(i);
                q[0] = (uint8_t)(pos >> 24);
                q[1] = (uint8_t)(pos >> 16);
                q[2] = (uint8_t)(pos >> 8);
                q[3] = (uint8_t)pos;
            }
        }
    }
    *out = e->out;
    *out_size = total;
    return 0;
}

/* [ref: src/gpujpeg_encoder.c:351-646] */
int gpujpeg_encoder_encode(struct gpujpeg_encoder* e, const struct gpujpeg_parameters* param,
                           const struct gpujpeg_image_parameters* param_image, const struct gpujpeg_encoder_input* input,
                           uint8_t** image_compressed, size_t* image_compressed_size)
{
    assert(param->comp_count <= GPUJPEG_MAX_COMPONENT_COUNT);
    assert(param->quality >= 0 && param->quality <= 100);
    assert(param->restart_interval >= RESTART_AUTO);
    assert(param->interleaved == 0 || param->interleaved == 1);
    if ( !e || !input || !image_compressed || !image_compressed_size ) return GPUJPEG_ERROR;

    const int img_changed = !e->initialised || !same_image(&e->param_image, param_image);
    struct gpujpeg_parameters a = adjust_params(e, param, param_image, img_changed);
    const int stats = a.perf_stats || a.verbose >= GPUJPEG_LL_STATUS;
    const double t_begin = stats ? gpujpeg_get_time() : 0.0;
    const int in = params_supported(&a, param_image);
    if ( !in || (e->writer_libjpeg && !libjpeg_supported(e, &a, param_image)) ) return GPUJPEG_ERROR;
    const struct gj_k1_request k1 = k1_request(e, in);

    /* quantisation tables follow the quality [ref: src/gpujpeg_encoder.c:372-380] */
    int tables_dirty = 0;
    if ( e->quality != a.quality ) {
        for ( int t = 0; t < 2; t++ ) {
            gj_quant_raw(t, a.quality, e->raw_q[t]);
            gj_quant_forward_zz(e->raw_q[t], e->h_tab.fwd_zz[t]);
        }
        e->quality = a.quality;
        tables_dirty = 1;
    }
    if ( standard_tables_back(e) ) tables_dirty = 1;
    e->counts_valid = 0;
    int geometry_dirty = 0;
    if ( img_changed || !same_param(&e->param, &a) || e->out_is_pinned != e->out_pinned || !e->out ||
         memcmp(&k1, &e->k1_req, sizeof k1) != 0 ) {
        if ( encoder_init_image(e, &a, param_image, &k1) ) return GPUJPEG_ERROR;
        geometry_dirty = 1;
    }
    e->param.quality = a.quality;
    e->param.verbose = a.verbose;
    e->param.perf_stats = a.perf_stats;
    const struct gj_geometry* g = &e->geo;

    /* an Exif header carries the time of day: composed for every frame, as the reference does for all headers */
    if ( (tables_dirty || geometry_dirty || e->header_written != e->header_type || e->extras_dirty ||
          e->header_type == GPUJPEG_HEADER_EXIF) && compose_headers(e) )
        return GPUJPEG_ERROR;

    /* input [ref: src/gpujpeg_encoder.c:402-476] */
    const uint8_t* d_raw;
    int k1_done = 0, k2_done = 0;   /* the stripe pipeline has launched them already */
    if ( input->type == GPUJPEG_ENCODER_INPUT_IMAGE ) {
        /* the reference's unit test passes a device pointer as a host image and expects it to work
         * [ref: test/unit/run_tests.c:40-79]; cudaMemcpyDefault semantics give the same result */
        if ( grow((void**)&e->d_raw, &e->d_raw_size, g->raw_size) ) {
            GJ_ERR("Encoder raw data allocation failed: %s\n", gj_cuda_last_error());
            return GPUJPEG_ERROR;
        }
        const int on_device = gj_cuda_pointer_is_device(input->image);
        if ( !on_device && !stats && stripes_usable(e) ) {
            if ( encode_striped(e, input->image, &k2_done) ) {
                GJ_ERR("Encoder raw data copy / forward DCT failed: %s\n", gj_cuda_last_error());
                return GPUJPEG_ERROR;
            }
            k1_done = 1;
        }
        else {
            if ( stats && e->timers_ok ) gj_timer_start(&e->t_to, e->stream);
            int rc = on_device ? gj_cuda_memcpy_d2d_async(e->d_raw, input->image, g->raw_size, e->stream)
                               : gj_cuda_memcpy_h2d_async(e->d_raw, input->image, g->raw_size, e->stream);
            if ( rc ) {
                GJ_ERR("Encoder raw data copy failed: %s\n", gj_cuda_last_error());
                return GPUJPEG_ERROR;
            }
            if ( stats && e->timers_ok ) gj_timer_stop(&e->t_to, e->stream);
        }
        d_raw = e->d_raw;
    }
    else if ( input->type == GPUJPEG_ENCODER_INPUT_GPU_IMAGE ) {
        d_raw = input->image;
    }
    else {
        GJ_ERR("OpenGL texture input is not supported in this build.\n");
        return GPUJPEG_ERROR;
    }

    if ( e->channel_remap ) {
        /* the permutation works in place on the encoder's own copy of the image [ref: src/gpujpeg_preprocessor.cu:516-559];
         * a caller's GPU image is copied first instead of being modified */
        struct gj_raw_layout rl;
        if ( gj_raw_layout_init(&rl, &e->param_image) ) return GPUJPEG_ERROR;
        if ( d_raw != e->d_raw ) {
            if ( grow((void**)&e->d_raw, &e->d_raw_size, g->raw_size) || gj_cuda_memcpy_d2d_async(e->d_raw, d_raw, g->raw_size, e->stream) )
                return GPUJPEG_ERROR;
            d_raw = e->d_raw;
        }
        const int rc = gj_launch_channel_remap(e->d_raw, &rl, e->param_image.pixel_format, g->width, g->height, e->channel_remap,
                                               e->stream);
        if ( rc == -2 ) GJ_ERR("Wrong channel remapping given, given %u channels but pixel format has %d!\n", e->channel_remap >> 24,
                               gpujpeg_pixel_format_get_comp_count(e->param_image.pixel_format));
        else if ( rc == -3 ) GJ_ERR("Channel remapping is not implemented for chroma-subsampled pixel formats in this build.\n");
        if ( rc ) return GPUJPEG_ERROR;
    }
    if ( stats && e->timers_ok ) {
        gj_timer_start(&e->t_gpu, e->stream);
        gj_timer_start(&e->t_pre, e->stream);
    }
    if ( !k1_done && launch_k1(e, d_raw, 0, e->k1.mcu_rows) ) {
        GJ_ERR("Forward DCT launch failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    if ( stats && e->timers_ok ) {
        gj_timer_stop(&e->t_pre, e->stream);
        gj_timer_start(&e->t_huff, e->stream);
    }
    if ( encode_tail(e, k2_done, stats, image_compressed, image_compressed_size) ) return GPUJPEG_ERROR;
    const size_t total = *image_compressed_size;

    e->stats_valid = 0;
    if ( stats && e->timers_ok ) {
        memset(&e->stats, 0, sizeof e->stats);
        e->stats.duration_memory_to = input->type == GPUJPEG_ENCODER_INPUT_IMAGE ? gj_timer_ms(&e->t_to) : 0.0;
        e->stats.duration_memory_from = gj_timer_ms(&e->t_from);
        e->stats.duration_preprocessor = 0.0; /* fused into the DCT kernel */
        e->stats.duration_dct_quantization = gj_timer_ms(&e->t_pre);
        e->stats.duration_huffman_coder = gj_timer_ms(&e->t_huff);
        e->stats.duration_stream = e->t_stream_ms;
        e->stats.duration_in_gpu = gj_timer_ms(&e->t_gpu);
        e->stats_valid = 1;
        if ( a.verbose >= GPUJPEG_LL_STATUS ) {
            /* [ref: src/gpujpeg_common.c:2169-2253] */
            fprintf(stderr, " -Copy To Device:    %10.3f ms\n", e->stats.duration_memory_to);
            fprintf(stderr, " -Preproc+DCT+Quant: %10.3f ms\n", e->stats.duration_dct_quantization);
            fprintf(stderr, " -Huffman Encoder:   %10.3f ms\n", e->stats.duration_huffman_coder);
            fprintf(stderr, " -Copy From Device:  %10.3f ms\n", e->stats.duration_memory_from);
            fprintf(stderr, " -Stream Formatter:  %10.3f ms\n", e->stats.duration_stream);
            fprintf(stderr, "Encode Image GPU:    %10.3f ms (only in-GPU processing)\n", e->stats.duration_in_gpu);
            fprintf(stderr, "Encode Image Bare:   %10.3f ms (without copy to/from GPU memory)\n",
                    (gpujpeg_get_time() - t_begin) * 1000.0 - e->stats.duration_memory_to - e->stats.duration_memory_from);
            fprintf(stderr, "Encode Image:        %10.3f ms\n", (gpujpeg_get_time() - t_begin) * 1000.0);
            fprintf(stderr, "Compressed Size:%15zu bytes %dx%d %s %s%s\n", total, e->param_image.width,
                    e->param_image.height, gpujpeg_color_space_get_name(e->param.color_space_internal),
                    gpujpeg_subsampling_get_name(e->param.comp_count, e->param.sampling_factor),
                    e->param.interleaved ? " interleaved" : " non-interleaved");
        }
    }
    return GPUJPEG_NOERR;
}

int gj_encoder_setup_coefficients(struct gpujpeg_encoder* e, const struct gpujpeg_parameters* p, int width, int height,
                                  const uint8_t comp_q[GJ_MAX_COMP][64], const uint8_t comp_tq[GJ_MAX_COMP], const uint8_t* com,
                                  size_t com_size, const struct gpujpeg_image_metadata* metadata, int16_t** d_coef,
                                  uint64_t** d_nzmask, const struct gj_geometry** geo)
{
    if ( com_size > e->com_cap ) {
        free(e->com);
        e->com_cap = 0;
        if ( !(e->com = (uint8_t*)malloc(com_size)) ) return -1;
        e->com_cap = com_size;
    }
    if ( com_size ) memcpy(e->com, com, com_size);
    memcpy(e->comp_q, comp_q, sizeof e->comp_q);
    memcpy(e->comp_tq, comp_tq, sizeof e->comp_tq);
    e->extras.comp_q = (const uint8_t(*)[64])e->comp_q;
    e->extras.comp_tq = e->comp_tq;
    e->extras.com = com_size ? e->com : (const uint8_t*)"";   /* no COM segment in the source: none in the output */
    e->extras.com_size = com_size;
    e->extras.metadata = *metadata;
    e->coef_input = 1;
    struct gpujpeg_image_parameters pi;
    gpujpeg_image_set_default_parameters(&pi);
    pi.width = width;
    pi.height = height;
    pi.color_space = p->color_space_internal;
    pi.pixel_format = p->comp_count == 1 ? GPUJPEG_U8 : p->comp_count == 4 ? GPUJPEG_4444_U8_P0123 : GPUJPEG_444_U8_P012;
    struct gpujpeg_parameters a = *p;
    if ( a.restart_interval == RESTART_AUTO )   /* what RESTART_AUTO gives gpujpeg_encoder_encode for this frame */
        a.restart_interval = gpujpeg_encoder_suggest_restart_interval(&pi, packed_sampling(&a), a.interleaved, a.verbose);
    standard_tables_back(e);
    e->counts_valid = 0;
    const struct gj_k1_request k1 = k1_request(e, GJ_IN_UNSUPPORTED);
    if ( encoder_init_image(e, &a, &pi, &k1) || compose_headers(e) ) return -1;
    *d_coef = e->d_coef;
    *d_nzmask = e->d_nzmask;
    *geo = &e->geo;
    return 0;
}

int gj_encoder_finish(struct gpujpeg_encoder* e, uint8_t** out, size_t* out_size)
{
    return encode_tail(e, 0, 0, out, out_size);
}

int gpujpeg_encoder_get_stats(struct gpujpeg_encoder* encoder, struct gpujpeg_duration_stats* stats)
{
    if ( !encoder || !stats || !encoder->stats_valid ) return -1;
    *stats = encoder->stats;
    return 0;
}

/* [ref: src/gpujpeg_encoder.c:728-733] */
void gpujpeg_encoder_set_jpeg_header(struct gpujpeg_encoder* encoder, enum gpujpeg_header_type header_type)
{
    encoder->header_type = header_type;
}

/* enc_metadata=orientation=<deg>[-]: quarter turns clockwise, '-' = mirrored afterwards [ref: src/gpujpeg_encoder.c:700-734] */
static int add_metadata(struct gpujpeg_image_metadata* metadata, const char* config)
{
    if ( strstr(config, "help") != NULL ) {
        printf(GPUJPEG_ENC_OPT_METADATA " usage:\n"
               "\t" GPUJPEG_ENC_OPT_METADATA "=orientation=<deg>[-]\n"
               "\t\t<deg> - clockwise rotation - 0, 90, 180 or 270 degrees\n"
               "\t\t'-'   - mirror the image horizontally after rotation applied\n");
        return GPUJPEG_ERROR;
    }
    static const char key[] = "orientation=";
    if ( strncmp(config, key, sizeof key - 1) != 0 ) {
        printf("Wrong metadata item: %s\n", config);
        return GPUJPEG_ERROR;
    }
    char* end = NULL;
    const long deg = strtol(config + sizeof key - 1, &end, 10);
    int flip = 0;
    if ( *end == '-' ) {
        flip = 1;
        end++;
    }
    if ( *end != '\0' || deg < 0 || deg > 270 || deg % 90 != 0 ) {
        printf("Wrong orientation value: %s\n", config);
        return GPUJPEG_ERROR;
    }
    metadata->vals[GPUJPEG_METADATA_ORIENTATION].set = 1;
    metadata->vals[GPUJPEG_METADATA_ORIENTATION].orient.rotation = (unsigned)(deg / 90);
    metadata->vals[GPUJPEG_METADATA_ORIENTATION].orient.flip = (unsigned)flip;
    return GPUJPEG_NOERR;
}

/* [ref: src/gpujpeg_encoder.c:736-800] */
int gpujpeg_encoder_set_option(struct gpujpeg_encoder* encoder, const char* opt, const char* val)
{
    if ( !encoder || !opt || !val ) return GPUJPEG_ERROR;
    if ( strcmp(opt, GPUJPEG_ENC_OPT_OUT) == 0 ) {
        if ( strcmp(val, GPUJPEG_ENC_OUT_VAL_PINNED) == 0 ) encoder->out_pinned = 1;
        else if ( strcmp(val, GPUJPEG_ENC_OUT_VAL_PAGEABLE) == 0 ) encoder->out_pinned = 0;
        else {
            GJ_ERR("Unknown encoder output type: %s\n", val);
            return GPUJPEG_ERROR;
        }
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_ENCODER_OPT_OUT_PINNED) == 0 ) {
        encoder->out_pinned = strcmp(val, GPUJPEG_VAL_TRUE) == 0;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_HDR) == 0 ) {   /* [ref: src/gpujpeg_encoder.c:759-766] */
        const enum gpujpeg_header_type t = gpujpeg_header_type_by_name(val);
        if ( t == GPUJPEG_HEADER_DEFAULT ) {
            GJ_ERR("Unknown encoder header type: %s\n", val);
            return GPUJPEG_ERROR;
        }
        encoder->header_type = t;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_FLIPPED_BOOL) == 0 ) {   /* [ref: src/gpujpeg_encoder.c:767-769] */
        const int b = gj_parse_bool(val, GPUJPEG_ENC_OPT_FLIPPED_BOOL);
        if ( b < 0 ) return GPUJPEG_ERROR;
        encoder->flipped = b;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_CHANNEL_REMAP) == 0 ) {   /* [ref: src/gpujpeg_encoder.c:770-772] */
        const unsigned m = gj_parse_channel_remap(val, GPUJPEG_ENC_OPT_CHANNEL_REMAP);
        if ( !m ) return GPUJPEG_ERROR;
        encoder->channel_remap = m;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_EXIF_TAG) == 0 ) {   /* a user tag asks for the Exif header [ref: src/gpujpeg_encoder.c:773-776] */
        encoder->header_type = GPUJPEG_HEADER_EXIF;
        encoder->extras_dirty = 1;
        return gj_exif_add_tag((struct gj_exif_tags**)&encoder->extras.exif_tags, val) == 0 ? GPUJPEG_NOERR : GPUJPEG_ERROR;
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_METADATA) == 0 ) {   /* [ref: src/gpujpeg_encoder.c:777-779] */
        encoder->extras_dirty = 1;
        return add_metadata(&encoder->extras.metadata, val);
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_HUFFMAN) == 0 ) {   /* extension: Huffman tables fitted to every frame */
        if ( strcmp(val, GPUJPEG_ENC_HUFFMAN_VAL_STANDARD) == 0 ) encoder->huff_optimized = 0;
        else if ( strcmp(val, GPUJPEG_ENC_HUFFMAN_VAL_OPTIMIZED) == 0 ) encoder->huff_optimized = 1;
        else {
            GJ_ERR("Unknown Huffman table choice: %s\n", val);
            return GPUJPEG_ERROR;
        }
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_ENC_OPT_WRITER) == 0 ) {   /* extension: whose file the encoder writes */
        if ( strcmp(val, GPUJPEG_ENC_WRITER_VAL_GPUJPEG) == 0 ) encoder->writer_libjpeg = 0;
        else if ( strcmp(val, GPUJPEG_ENC_WRITER_VAL_LIBJPEG) == 0 ) encoder->writer_libjpeg = 1;
        else {
            GJ_ERR("Unknown encoder writer: %s\n", val);
            return GPUJPEG_ERROR;
        }
        encoder->extras.libjpeg = encoder->writer_libjpeg;
        encoder->extras_dirty = 1;
        return GPUJPEG_NOERR;
    }
    GJ_ERR("Invalid encoder option: %s!\n", opt);
    return GPUJPEG_ERROR;
}

void gpujpeg_encoder_print_options(void)
{
    printf("\t" GPUJPEG_ENC_OPT_OUT "=[" GPUJPEG_ENC_OUT_VAL_PAGEABLE "|" GPUJPEG_ENC_OUT_VAL_PINNED
           "] - output buffer in pageable or pinned host memory\n");
    printf("\t" GPUJPEG_ENC_OPT_HDR "=[" GPUJPEG_ENC_HDR_VAL_JFIF "|" GPUJPEG_ENC_HDR_VAL_ADOBE "|" GPUJPEG_ENC_HDR_VAL_EXIF "|" GPUJPEG_ENC_HDR_VAL_SPIFF
           "] - output JPEG header (default: by internal colour space)\n");
    printf("\t" GPUJPEG_ENC_OPT_EXIF_TAG "=<key>=<value>|help - custom EXIF tag (use help for syntax)\n");
    printf("\t" GPUJPEG_ENC_OPT_METADATA "=<key>=<value>|help - set image metadata\n");
    printf("\t" GPUJPEG_ENC_OPT_FLIPPED_BOOL "=[" GPUJPEG_VAL_FALSE "|" GPUJPEG_VAL_TRUE
           "] - whether is the input image should be vertically flipped (prior encode)\n");
    printf("\t" GPUJPEG_ENC_OPT_CHANNEL_REMAP "=XYZ[W] - input channel mapping, eg. '210F' for GBRX,\n"
           "\t\t'210' for GBR; special placeholders 'F' and 'Z' to set a channel to all-ones or all-zeros\n");
    printf("\t" GPUJPEG_ENC_OPT_HUFFMAN "=[" GPUJPEG_ENC_HUFFMAN_VAL_STANDARD "|" GPUJPEG_ENC_HUFFMAN_VAL_OPTIMIZED
           "] - Huffman tables of T.81 Annex K (default) or fitted to every frame\n");
    printf("\t" GPUJPEG_ENC_OPT_WRITER "=[" GPUJPEG_ENC_WRITER_VAL_GPUJPEG "|" GPUJPEG_ENC_WRITER_VAL_LIBJPEG
           "] - this library's stream (default) or the file libjpeg-turbo writes with its defaults\n");
}

/* ---- extension: re-run the GPU stages of the last configured frame on device-resident data ----
 * stage_mask bit 0 = K1 (colour+FDCT+quant, the kernel of the writer chosen), bit 3 = the symbol statistics of enc_opt_huffman=optimized (kernel alone),
 * bit 1 = K2 (Huffman encode + scan assembly, with the tables the last gpujpeg_encoder_encode chose).  Nothing is
 * copied to or from the host and nothing is synchronised: the caller times the stream with CUDA events.
 * d_raw == NULL re-uses the device copy of the last host image.  Used by bench.py for the
 * "inputs already resident in HBM" number and for per-stage roofline timing. */
GPUJPEG_API int gpujpegx_encoder_run_resident(struct gpujpeg_encoder* e, const uint8_t* d_raw, int stage_mask)
{
    if ( !e || !e->initialised ) return -1;
    if ( !d_raw ) d_raw = e->d_raw;
    if ( !d_raw ) return -1;
    if ( (stage_mask & 1) && launch_k1(e, d_raw, 0, e->k1.mcu_rows) ) return -1;
    if ( (stage_mask & 8) && launch_stats(e) ) return -1;
    if ( (stage_mask & 2) && launch_k2(e) ) return -1;
    return 0;
}

/* ---- extension used by the parity tests: the symbol counts the statistics kernel found in the last frame ---- */
GPUJPEG_API int gpujpegx_encoder_get_symbol_counts(struct gpujpeg_encoder* e, uint64_t out[2][2][256])
{
    if ( !e || !e->initialised || !e->counts_valid || !out ) return -1;
    if ( gj_cuda_memcpy_d2h_async(e->h_counts, e->d_counts, GJ_HUFF_COUNTS_BYTES, e->stream) || gj_cuda_stream_sync(e->stream) )
        return -1;
    memcpy(out, e->h_counts, GJ_HUFF_COUNTS_BYTES);
    return 0;
}

/* ---- extension used by bench.py: the JPEG stream the last K2 launch produced (resident re-runs included) ---- */
GPUJPEG_API long long gpujpegx_encoder_get_stream(struct gpujpeg_encoder* e, uint8_t* out, size_t capacity)
{
    if ( !e || !e->initialised || e->with_segment_info || !e->d_info_cur ) return -1;
    if ( gj_cuda_memcpy_d2h_async(e->h_info, e->d_info_cur, 32, e->stream) || gj_cuda_stream_sync(e->stream) ) return -1;
    const size_t total = (size_t)e->h_info[0];
    if ( e->h_info[1] || total < e->header_size + 2 || total > e->d_stream_size ) return -1;
    if ( !out ) return (long long)total;
    if ( total > capacity ) return -1;
    if ( gj_cuda_memcpy_d2h_async(out + e->header_size, e->d_stream + e->header_size, total - e->header_size, e->stream) ||
         gj_cuda_stream_sync(e->stream) )
        return -1;
    memcpy(out, e->header, e->header_size);
    return (long long)total;
}

/* ---- extension used by the parity tests: quantised coefficients of the last frame, natural order ---- */
GPUJPEG_API int gpujpegx_encoder_get_coefficients(struct gpujpeg_encoder* e, int16_t* out, size_t count)
{
    if ( !e || !e->initialised || count != e->geo.coef_count ) return -1;
    return gj_coef_to_host_natural(e->d_coef, NULL, e->d_nzmask, count, out, e->stream);
}
