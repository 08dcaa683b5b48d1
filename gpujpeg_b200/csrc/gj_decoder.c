/*
 * gj_decoder.c -- the public decoder API on top of the sm_90a stage launchers.  Host C.
 *
 * Contract of the reference orchestrator (src/gpujpeg_decoder.c:94-469): lazily (re)initialises
 * from the stream, one CUDA stream, blocks until the pixels are where the output descriptor says.
 * Pipeline of this build:
 *
 *     host reader: marker segments only (headers, SOS); the file is uploaded ONCE, untouched, and the
 *                  restart markers are found by K0 on the device -- the reference walks the whole stream
 *                  with memchr and re-packs it segment by segment (src/gpujpeg_reader.c:1038-1155),
 *                  which alone costs several times the GPU time of the whole decode at 8K
 *     H2D file bytes -> K0 marker list -> (tiny D2H, sync) -> host finishes the marker walk
 *       -> K3 Huffman decode (always on the GPU: no "fewer than 32 segments => CPU" fallback,
 *          src/gpujpeg_decoder.c:254-286)
 *       -> K4 dequant + IDCT + colour transform + interleave (one launch)
 *     D2H pixels (unless a device output was requested)
 *
 * Supported: baseline 8-bit YCbCr-JPEG or grey streams, 1 or 3 components, 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0, interleaved or
 * not, any restart interval (or none), any DHT/DQT tables with ids 0..3; progressive (SOF2, Huffman) frames of the same
 * samplings through decode_progressive (one GPU thread per restart segment of a scan); output negotiated in choose_output():
 * GPUJPEG_RGB 444-u8-p012 through the fused kernel, the stream's own samples in a matching pixel format straight from
 * the IDCT, every other pixel format x colour space combination through the generic pass.
 */
#include <stdlib.h>
#include <string.h>

#include "gj_internal.h"

#define GJ_MK_OTHER_CAP 256 /* markers other than RSTn the device reports back (SOS, EOI, ...) */
#define GJ_CTA_BYTES0 (64 * 1024)   /* first size of the tile-status area behind the result block: files up to 32 MB */
#define GJ_MK_WORDS (8 + 4 * GJ_MK_OTHER_CAP)   /* K0 result block: 8 counters/flags + {rank, position, code, clean position} per marker */

#define GJ_STRIPES 8
#define GJ_STRIPE_MIN_BYTES ((size_t)8 << 20)

struct gpujpeg_decoder {
    gj_stream_t stream;
    /* stripe pipeline of host output (RGB frames of GJ_STRIPE_MIN_BYTES or more from the fused kernels): K4 runs on GJ_STRIPES pieces of the frame,
     * every finished piece leaves for the host on a copy stream while the next one is transformed */
    gj_stream_t copy_stream;
    void* ev_stripe[GJ_STRIPES]; void* ev_done;
    int stripes;                  /* GPUJPEG_B200_STRIPES (1 = off), default GJ_STRIPES */
    size_t stripe_min_bytes;      /* GPUJPEG_B200_STRIPE_MIN_BYTES (tests), default GJ_STRIPE_MIN_BYTES */
    int k3_parts;                 /* GPUJPEG_B200_STRIPES_K3 (0 = K3 on the whole frame first); -1 = not read yet */
    int device;
    int verbose, perf_stats;
    struct gpujpeg_parameters param;
    struct gpujpeg_image_parameters param_image;
    struct gj_geometry geo;
    int initialised;
    enum gpujpeg_pixel_format req_pixel_format;
    enum gpujpeg_color_space req_color_space;
    int idct_flavour;
    int flipped;                  /* dec_opt_flipped */
    unsigned channel_remap;       /* dec_opt_channel_remap: (count << 24) | selector nibbles, 0 = none */
    int huffman_req;              /* dec_opt_huffman: GJ_K3_AUTO, GJ_K3_THREAD_PER_SEGMENT or GJ_K3_SUBSEQUENCE */
    int used_subsequences;        /* the last frame's Huffman stage ran the sub-sequence kernel */
    void* d_ss_scratch; size_t d_ss_scratch_size;   /* its per-segment and per-sub-sequence state */
    int force_lanes[GJ_MAX_COMP]; /* dec_opt_huffman_lanes: lanes per restart segment by scan, 0 = chosen from the frame's segment count */
    int sm_count;
    int ff_cs_itu601_is_709;      /* [ref: libgpujpeg/gpujpeg_decoder.h:95] */
    struct gj_k4_plan k4;         /* what K4 does with the frame being / last decoded (gj_k4_choose) */
    uint8_t* d_planes; size_t d_planes_size;   /* component planes between the IDCT and the generic pass */
    struct gj_raw_layout raw;     /* the output's layout (every output but the fused kernels' uncropped RGB) */
    /* scaled decoding (dec_opt_scale): scale_req is the option, scale the divisor of the frame being / last decoded (1, 2, 4
     * or 8); the frame's output is out_w x out_h pixels, out_size bytes; scomp = the component planes at that scale (the
     * block grids of geo.comp, 8 / scale samples per block side, width / height the samples that carry image data) */
    int scale_req, scale;
    int out_w, out_h;
    size_t out_size;
    struct gj_comp_geo scomp[GJ_MAX_COMP];
    /* dec_opt_crop: crop_req = the option is set, crop_r* its rectangle in output pixels; crop = the frame being / last decoded
     * is cropped (kept apart from the option, as scale from scale_req, so that a resident re-run always works on the frame's own
     * rectangle: k4.rect, the blocks of every component it needs k4.win.blk), d_pick / h_pick the segments K3 (or every
     * progressive scan) decodes: {segment, blocks} pairs */
    int crop_req, crop_rx, crop_ry, crop_rw, crop_rh;
    int crop;
    uint32_t* d_pick; size_t d_pick_size;
    uint32_t* h_pick; size_t h_pick_size;
    /* dec_opt_orientation: orient_mode 0 = none, 1 = auto (the stream's own), 2 = orient_rot / orient_flip; orient = the frame
     * being / last decoded is turned or mirrored, by k4.map (which also maps a crop) */
    int orient_mode, orient_rot, orient_flip;
    int orient;
    /* dec_opt_pixels: pixels_req 1 = libjpeg (the option) */
    int pixels_req;
    struct gpujpeg_image_metadata metadata;

    struct gj_dev_dec_tables h_tab, h_tab_prev;
    struct gj_dev_dec_tables* d_tab;
    int tab_valid;

    uint8_t* d_file; size_t d_file_size;
    uint32_t* d_list_pos; size_t d_list_pos_size;   /* K0 marker list: positions */
    uint8_t* d_list_code; size_t d_list_code_size;  /*                  codes     */
    uint32_t* d_list_cpos; size_t d_list_cpos_size; /*                  positions in the clean stream */
    uint8_t* d_clean; size_t d_clean_size;          /* K0 clean stream: stuffing and markers removed, big-endian words */
    uint32_t* d_seg_tab; size_t d_seg_tab_size;     /* resynchronised streams only: per segment {raw start, clean start, clean end} */
    uint32_t* d_seg_off; uint32_t* h_seg_off; size_t seg_off_size;   /* streams with segment info: file offset of every segment (h: pinned) */
    int used_segment_info;                          /* the last frame's scans were split by the stream's own tables */
    int ignore_segment_info;                        /* set while a frame whose tables proved wrong is decoded again */
    unsigned long long* d_cta; size_t d_cta_size;   /* K0 scratch: tile status words, kept right behind d_mk (one allocation, one memset) */
    uint32_t* d_mk;                                 /* K0 results (layout in gpujpeg_decoder_decode) */
    uint32_t* d_k3_ctr;                             /* K3 work counters (8 words, zero between launches) */
    uint32_t* h_mk;                                 /* pinned mirror */
    int16_t* d_coef; size_t d_coef_size;
    uint8_t* d_cext; size_t d_cext_size;     /* one extent byte per block of d_coef (GJ_CEXT_FULL) */
    uint8_t* d_raw; size_t d_raw_size;
    uint8_t* h_raw; size_t h_raw_size;       /* pinned, INTERNAL_BUFFER output */

    struct gj_timer t_to, t_from, t_huff, t_dct, t_gpu;
    int timers_ok;
    struct gpujpeg_duration_stats stats;
    int stats_valid;

    struct gj_huff_dec_args last_args;  /* launch arguments of the last frame (resident re-runs) */
    size_t last_ecs_begin; uint32_t last_list_cap;
    int last_tq[GJ_MAX_COMP];
    int last_valid;

    /* progressive frames (decode_progressive): the last frame's scans and launch arguments, every scan's Huffman tables */
    int last_progressive;
    struct gj_prog_args last_prog;
    struct gj_prog_scan* prog_scans;   /* [GJ_MAX_SCANS] */
    struct gj_dec_lut* h_prog_luts;    /* [GJ_MAX_SCANS * GJ_MAX_COMP] */
    struct gj_dec_lut* d_prog_luts;

    /* gj_decoder_decode_coefficients: the frame stops after the Huffman stage with raw coefficients (no K4, no output); what
     * it hands out besides the device buffers */
    int coef_only;
    uint8_t coef_qt[GJ_MAX_COMP][64];
    int coef_tq[GJ_MAX_COMP];
    uint8_t* com; size_t com_cap;
    /* ... and the caller's window over the frame's blocks (gj_coef_window_fn; NULL: every block) */
    gj_coef_window_fn coef_window;
    void* coef_window_ctx;
};

/* ---- output descriptor helpers [ref: src/gpujpeg_decoder.c:44-92] ---- */
void gpujpeg_decoder_output_set_default(struct gpujpeg_decoder_output* output)
{
    memset(output, 0, sizeof *output);
    output->type = GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER;
}
void gpujpeg_decoder_output_set_custom(struct gpujpeg_decoder_output* output, uint8_t* custom_buffer)
{
    memset(output, 0, sizeof *output);
    output->type = GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER;
    output->data = custom_buffer;
}
void gpujpeg_decoder_output_set_texture(struct gpujpeg_decoder_output* output, struct gpujpeg_opengl_texture* texture)
{
    memset(output, 0, sizeof *output);
    output->type = GPUJPEG_DECODER_OUTPUT_OPENGL_TEXTURE;
    output->texture = texture;
}
void gpujpeg_decoder_output_set_cuda_buffer(struct gpujpeg_decoder_output* output)
{
    memset(output, 0, sizeof *output);
    output->type = GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER;
}
void gpujpeg_decoder_output_set_custom_cuda(struct gpujpeg_decoder_output* output, uint8_t* d_custom_buffer)
{
    memset(output, 0, sizeof *output);
    output->type = GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER;
    output->data = d_custom_buffer;
}

struct gpujpeg_decoder_init_parameters gpujpeg_decoder_default_init_parameters(void)
{
    struct gpujpeg_decoder_init_parameters p;
    memset(&p, 0, sizeof p);
    return p;
}

/* [ref: src/gpujpeg_decoder.c:94-181] */
struct gpujpeg_decoder* gpujpeg_decoder_create_with_params(const struct gpujpeg_decoder_init_parameters* params)
{
    struct gpujpeg_decoder* d = (struct gpujpeg_decoder*)calloc(1, sizeof *d);
    if ( !d ) return NULL;
    d->stream = (gj_stream_t)params->stream;
    d->verbose = params->verbose;
    d->perf_stats = params->perf_stats;
    d->ff_cs_itu601_is_709 = params->ff_cs_itu601_is_709;
    d->device = gj_cuda_get_device();
    d->sm_count = gj_cuda_sm_count();
    d->req_pixel_format = GPUJPEG_PIXFMT_AUTODETECT;
    d->k3_parts = -1;
    d->scale_req = d->scale = 1;
    d->req_color_space = GPUJPEG_CS_DEFAULT;
    if ( d->device < 0 || gj_cuda_malloc((void**)&d->d_tab, sizeof *d->d_tab) ||
         gj_cuda_malloc((void**)&d->d_mk, GJ_MK_WORDS * 4 + GJ_CTA_BYTES0) || gj_cuda_malloc((void**)&d->d_k3_ctr, 32) ||
         gj_cuda_memset_async(d->d_k3_ctr, 0, 32, d->stream) || gj_cuda_stream_sync(d->stream) ||
         gj_cuda_malloc_host((void**)&d->h_mk, GJ_MK_WORDS * 4) ) {
        GJ_ERR("Decoder allocation failed: %s\n", gj_cuda_last_error());
        free(d);
        return NULL;
    }
    d->timers_ok = !(gj_timer_create(&d->t_to) || gj_timer_create(&d->t_from) || gj_timer_create(&d->t_huff) ||
                     gj_timer_create(&d->t_dct) || gj_timer_create(&d->t_gpu));
    return d;
}

struct gpujpeg_decoder* gpujpeg_decoder_create(cudaStream_t stream)
{
    struct gpujpeg_decoder_init_parameters p = gpujpeg_decoder_default_init_parameters();
    p.stream = stream;
    return gpujpeg_decoder_create_with_params(&p);
}

int gpujpeg_decoder_destroy(struct gpujpeg_decoder* d)
{
    if ( !d ) return -1;
    gj_cuda_free(d->d_tab);
    gj_cuda_free(d->d_file);
    gj_cuda_free(d->d_list_pos);
    gj_cuda_free(d->d_list_code);
    gj_cuda_free(d->d_list_cpos);
    gj_cuda_free(d->d_clean);
    gj_cuda_free(d->d_seg_tab);
    gj_cuda_free(d->d_seg_off);
    if ( d->h_seg_off ) gj_cuda_free_host(d->h_seg_off);
    gj_cuda_free(d->d_mk);
    gj_cuda_free(d->d_k3_ctr);
    gj_cuda_free_host(d->h_mk);
    gj_cuda_free(d->d_coef);
    gj_cuda_free(d->d_cext);
    gj_cuda_free(d->d_planes);
    gj_cuda_free(d->d_raw);
    gj_cuda_free_host(d->h_raw);
    gj_cuda_free(d->d_prog_luts);
    gj_cuda_free(d->d_pick);
    gj_cuda_free(d->d_ss_scratch);
    free(d->com);
    free(d->h_pick);
    free(d->prog_scans);
    free(d->h_prog_luts);
    if ( d->copy_stream ) gj_cuda_stream_destroy(d->copy_stream);
    gj_cuda_event_destroy(d->ev_done);
    for ( int i = 0; i < GJ_STRIPES; i++ )
        gj_cuda_event_destroy(d->ev_stripe[i]);
    gj_timer_destroy(&d->t_to);
    gj_timer_destroy(&d->t_from);
    gj_timer_destroy(&d->t_huff);
    gj_timer_destroy(&d->t_dct);
    gj_timer_destroy(&d->t_gpu);
    free(d);
    return 0;
}

static int grow_dev(void** p, size_t* have, size_t want)
{
    if ( *have >= want ) return 0;
    gj_cuda_free(*p);
    *p = NULL;
    *have = 0;
    if ( gj_cuda_malloc(p, want) ) return -1;
    *have = want;
    return 0;
}
static int grow_host(void** p, size_t* have, size_t want)
{
    if ( *have >= want ) return 0;
    gj_cuda_free_host(*p);
    *p = NULL;
    *have = 0;
    if ( gj_cuda_malloc_host(p, want) ) return -1;
    *have = want;
    return 0;
}

/* K0's result block and its tile-status words as one allocation (nothing in it outlives a frame) */
static int grow_mk_cta(struct gpujpeg_decoder* d, size_t cta_bytes)
{
    if ( d->d_cta && cta_bytes <= d->d_cta_size ) return 0;
    if ( !d->d_cta && cta_bytes <= GJ_CTA_BYTES0 ) {
        d->d_cta = (unsigned long long*)(d->d_mk + GJ_MK_WORDS);
        d->d_cta_size = GJ_CTA_BYTES0;
        return 0;
    }
    const size_t want = cta_bytes + cta_bytes / 4;
    uint32_t* fresh = NULL;
    if ( gj_cuda_stream_sync(d->stream) || gj_cuda_malloc((void**)&fresh, GJ_MK_WORDS * 4 + want) ) return -1;
    gj_cuda_free(d->d_mk);
    d->d_mk = fresh;
    d->d_cta = (unsigned long long*)(fresh + GJ_MK_WORDS);
    d->d_cta_size = want;
    return 0;
}

/* [ref: src/gpujpeg_decoder.c:184-231] pre-allocation for a known geometry */
int gpujpeg_decoder_init(struct gpujpeg_decoder* d, const struct gpujpeg_parameters* param,
                         const struct gpujpeg_image_parameters* param_image)
{
    d->verbose = param->verbose;
    d->perf_stats = param->perf_stats || param->verbose >= GPUJPEG_LL_STATUS;
    if ( param_image->width <= 0 || param_image->height <= 0 || param->comp_count <= 0 ) return 0;
    /* stream-supplied dimensions: all index arithmetic below is sized for frames of at most 2^30 pixels */
    if ( (size_t)param_image->width * (size_t)param_image->height > ((size_t)1 << 30) ) {
        GJ_ERR("Image size %dx%d exceeds the supported maximum of 2^30 pixels.\n", param_image->width, param_image->height);
        return -1;
    }
    struct gpujpeg_parameters p = *param;
    struct gpujpeg_image_parameters pi = *param_image;
    if ( p.comp_count != 3 && p.comp_count != 1 && p.comp_count != 4 ) {
        GJ_ERR("This build decodes 1-, 3- and 4-component images only.\n");
        return -1;
    }
    if ( (int)pi.pixel_format < 0 )
        pi.pixel_format = p.comp_count == 1 ? GPUJPEG_U8 : p.comp_count == 4 ? GPUJPEG_4444_U8_P0123 : GPUJPEG_444_U8_P012;
    gj_geometry_init(&d->geo, &p, &pi);
    const struct gj_geometry* g = &d->geo;
    /* (the output of a scaled frame is smaller: gpujpeg_decoder_decode sizes d_raw for it, size_output) */
    if ( grow_dev((void**)&d->d_coef, &d->d_coef_size, g->coef_count * 2) ||
         grow_dev((void**)&d->d_cext, &d->d_cext_size, g->coef_count / 64) ||
         (d->scale == 1 && !d->coef_only && grow_dev((void**)&d->d_raw, &d->d_raw_size, g->raw_size)) ) {
        GJ_ERR("Decoder device allocation failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    d->param = p;
    d->param_image = pi;
    d->initialised = 1;
    return 0;
}

/* [ref: src/gpujpeg_decoder.c:471-483] */
void gpujpeg_decoder_set_output_format(struct gpujpeg_decoder* decoder, enum gpujpeg_color_space color_space,
                                       enum gpujpeg_pixel_format pixel_format)
{
    decoder->req_color_space = color_space;
    decoder->req_pixel_format = pixel_format;
}

/* What this build decodes to (anything else fails loudly); gj_k4_choose turns it into the frame's K4:
 *   GJ_OUT_RGB      3-component YCbCr stream -> GPUJPEG_RGB / 444-u8-p012 (the default request), any supported sampling
 *   GJ_OUT_SAMPLES  the stream's own components, no colour transform: GPUJPEG_U8 for 1-component streams; for
 *                   3-component streams colour space GPUJPEG_YCBCR_JPEG (or GPUJPEG_NONE) with a pixel format of the
 *                   stream's sampling: 444-u8-p012, 444/422/420-u8-p0p1p2, 422-u8-p1020, or the special values
 *                   GPUJPEG_PIXFMT_NATIVE / _STD resolved as the reference does [ref: src/gpujpeg_reader.c:1507-1581]
 *   GJ_OUT_GENERIC  any of those pixel formats in GPUJPEG_RGB / _YCBCR_BT601 / _YCBCR_JPEG / _YCBCR_BT709 whatever the stream's
 *                   sampling: the IDCT writes component planes, one extra pass converts them (gj_convert.cu)
 * dec_opt_pixels=libjpeg takes GPUJPEG_RGB 444-u8-p012 or GPUJPEG_U8 of these (gpujpeg_decoder_decode). */

static int choose_output(const struct gpujpeg_decoder* d, const struct gj_stream* st, struct gpujpeg_image_parameters* pi)
{
    enum gpujpeg_pixel_format pf = d->req_pixel_format;
    enum gpujpeg_color_space cs = d->req_color_space;
    const int special = (int)pf < 0;   /* GPUJPEG_PIXFMT_NONE / _AUTODETECT / _NO_ALPHA / _STD / _NATIVE */
    if ( st->comp_count == 1 ) {
        if ( !special && pf != GPUJPEG_U8 ) {
            GJ_ERR("This build decodes 1-component JPEGs to GPUJPEG_U8 only (%s requested).\n", gpujpeg_pixel_format_get_name(pf));
            return 0;
        }
        pi->pixel_format = GPUJPEG_U8;
        pi->color_space = (cs == GPUJPEG_CS_DEFAULT || cs == GPUJPEG_NONE) ? GPUJPEG_YCBCR_JPEG : cs;
        return GJ_OUT_SAMPLES;
    }
    const int lh = st->comp_hv[0] >> 4, lv = st->comp_hv[0] & 15;
    if ( cs == GPUJPEG_CS_DEFAULT ) cs = GPUJPEG_RGB;
    if ( cs == GPUJPEG_NONE ) cs = st->color_space;
    if ( special ) {
        const int planar_by_sampling = pf == GPUJPEG_PIXFMT_STD && cs != GPUJPEG_RGB;
        if ( pf == GPUJPEG_PIXFMT_NATIVE && st->comp_count == 4 ) pf = GPUJPEG_4444_U8_P0123;   /* [ref: src/gpujpeg_reader.c:1510-1512] */
        else if ( pf == GPUJPEG_PIXFMT_NATIVE || planar_by_sampling ) {
            const int il = pf == GPUJPEG_PIXFMT_NATIVE && st->scan[0].ncomp > 1;
            if ( lh == 2 && lv == 2 ) pf = GPUJPEG_420_U8_P0P1P2;
            else if ( lh == 2 && lv == 1 ) pf = il ? GPUJPEG_422_U8_P1020 : GPUJPEG_422_U8_P0P1P2;
            else pf = il ? GPUJPEG_444_U8_P012 : GPUJPEG_444_U8_P0P1P2;
        }
        else {
            /* a fourth component comes out as alpha unless the caller asked for "no alpha" [ref: src/gpujpeg_reader.c:1576-1581] */
            pf = st->comp_count == 4 && pf != GPUJPEG_PIXFMT_NO_ALPHA ? GPUJPEG_4444_U8_P0123 : GPUJPEG_444_U8_P012;
        }
    }
    pi->pixel_format = pf;
    pi->color_space = cs;
    if ( st->comp_count == 3 && cs == GPUJPEG_RGB && pf == GPUJPEG_444_U8_P012 && st->color_space == GPUJPEG_YCBCR_BT601_256LVLS )
        return GJ_OUT_RGB;
    if ( cs != GPUJPEG_RGB && cs != GPUJPEG_YCBCR_BT601 && cs != GPUJPEG_YCBCR_BT601_256LVLS && cs != GPUJPEG_YCBCR_BT709 ) {
        GJ_ERR("Colour space %s is not produced by this build.\n", gpujpeg_color_space_get_name(cs));
        return 0;
    }
    struct gj_raw_layout rl;
    if ( gj_raw_layout_init(&rl, pi) || rl.comp_count != 3 ) {
        GJ_ERR("Pixel format %s (%dx%d) is not produced by this build.\n", gpujpeg_pixel_format_get_name(pf), pi->width,
               pi->height);
        return 0;
    }
    if ( st->comp_count == 4 || cs != st->color_space || rl.sampling[0].horizontal != lh || rl.sampling[0].vertical != lv ||
         rl.alpha_off ) {
        if ( (pi->width & 1) && rl.sampling[0].horizontal == 2 && pf != GPUJPEG_420_U8_P0P1P2 ) {
            GJ_ERR("Odd widths are only produced without colour / sampling conversion for this pixel format.\n");
            return 0;
        }
        return GJ_OUT_GENERIC;
    }
    return GJ_OUT_SAMPLES;
}

/* K4 as the frame's plan says: the IDCT (the fused kernels on MCU rows [my0, my1), the per-block ones on the frame), the flip
 * of the planes, the pass from the planes to the output */
static int launch_k4(struct gpujpeg_decoder* d, const int comp_tq[GJ_MAX_COMP], uint8_t* d_out, int my0, int my1)
{
    const struct gj_geometry* g = &d->geo;
    const struct gj_k4_plan* p = &d->k4;
    if ( p->kernel == GJ_K4_FUSED )
        return gj_launch_idct_fused(p, d->d_coef, d->d_cext, g->comp, comp_tq, d_out, g->width, g->height, g->pitch, my0, my1, &d->h_tab,
                                    d->stream);
    struct gj_raw_layout pl;
    struct gj_comp_geo padded[GJ_MAX_COMP];
    if ( p->to_planes ) gj_planes_layout(&pl, padded, g->comp, g->comp_count, p->n);
    const struct gj_comp_geo* comp = p->to_planes ? padded : p->scomp ? d->scomp : g->comp;
    if ( gj_launch_idct_blocks(p, d->d_coef, d->d_cext, comp, g->comp_count, comp_tq, p->to_planes ? d->d_planes : d_out,
                               p->to_planes ? &pl : &d->raw, &d->h_tab, d->stream) )
        return -1;
    if ( p->flip == GJ_K4_FLIP_PLANES && gj_launch_flip_planes(d->d_planes, padded, g->comp_count, d->stream) ) return -1;
    const struct gj_orient_map* map = p->post_map ? &p->map : NULL;
    if ( p->post == GJ_K4_POST_CONVERT )
        return gj_launch_convert_out(d->d_planes, d_out, &d->raw, d->param_image.pixel_format, d->param_image.color_space,
                                     d->param.color_space_internal, d->out_w, d->out_h, g->comp, g->comp_count, g->max_hs, g->max_vs, p->n,
                                     map, d->stream);
    if ( p->post == GJ_K4_POST_LIBJPEG )
        return gj_launch_libjpeg_out(d->d_planes, d_out, g->comp, g->comp_count, g->max_hs, g->max_vs, d->out_w, d->out_h,
                                     d->param.color_space_internal == GPUJPEG_RGB, map, d->stream);
    return 0;
}

/* The stripe pipeline applies to what the fused RGB kernels write as they go (k4.stripes), on frames large enough */
static int stripes_usable(struct gpujpeg_decoder* d)
{
    const struct gj_geometry* g = &d->geo;
    if ( !d->k4.stripes ) return 0;
    if ( d->stripes == 0 ) {
        const char* v = getenv("GPUJPEG_B200_STRIPES");
        const char* m = getenv("GPUJPEG_B200_STRIPE_MIN_BYTES");
        d->stripe_min_bytes = m ? (size_t)strtoull(m, NULL, 0) : GJ_STRIPE_MIN_BYTES;
        d->stripes = v ? atoi(v) : GJ_STRIPES;
        if ( d->stripes < 1 ) d->stripes = 1;
        if ( d->stripes > GJ_STRIPES ) d->stripes = GJ_STRIPES;
    }
    if ( d->stripes < 2 || g->bcy / g->max_vs < 2 * d->stripes || g->raw_size < d->stripe_min_bytes ) return 0;
    if ( !d->copy_stream ) {
        if ( gj_cuda_stream_create(&d->copy_stream) || gj_cuda_event_create(&d->ev_done) ) {
            d->stripes = 1;
            return 0;
        }
        for ( int i = 0; i < GJ_STRIPES; i++ )
            if ( gj_cuda_event_create(&d->ev_stripe[i]) ) {
                d->stripes = 1;
                return 0;
            }
    }
    return 1;
}

/* K4 stripe by stripe on the coder's stream, D2H of every finished stripe on the copy stream; the coder's stream then waits
 * for the last copy, so that its next synchronisation covers the whole picture */
static int decode_striped(struct gpujpeg_decoder* d, const int comp_tq[GJ_MAX_COMP], uint8_t* d_out, uint8_t* h_dst,
                          const struct gj_huff_dec_args* k3 /* NULL: K3 has run on the whole frame */)
{
    const struct gj_geometry* g = &d->geo;
    struct gj_huff_dec_args part;
    int segs_done[GJ_MAX_COMP] = {0, 0, 0, 0};
    if ( k3 ) part = *k3;
    const int mcu_h = 8 * g->max_vs;                                  /* image rows per MCU row (4:4:4: one block row) */
    const int mcu_rows = d->k4.mcu_rows;
    for ( int i = 0; i < d->stripes; i++ ) {
        const int my0 = (int)((long long)mcu_rows * i / d->stripes), my1 = (int)((long long)mcu_rows * (i + 1) / d->stripes);
        const size_t row0 = (size_t)my0 * mcu_h, row1 = (size_t)my1 * mcu_h < (size_t)g->height ? (size_t)my1 * mcu_h : (size_t)g->height;
        const size_t off = row0 * (size_t)g->pitch;
        const size_t bytes = (i + 1 == d->stripes ? g->raw_size : row1 * (size_t)g->pitch) - off;
        if ( k3 ) {
            /* the segments that hold the blocks of the rows [0, my1), handed over at multiples of 32 segments (whole units of
             * every lane count); 4:4:4, one scan per component: block position = MCU number in every scan */
            int any = 0;
            for ( int k = 0; k < g->scan_count; k++ ) {
                const int segs = g->lay.scan_seg_begin[k + 1] - g->lay.scan_seg_begin[k];
                long long hi = i + 1 == d->stripes ? segs : (((long long)my1 * g->bcx + g->seg_mcu - 1) / g->seg_mcu + 31) / 32 * 32;
                if ( hi > segs ) hi = segs;
                part.part_seg_lo[k] = segs_done[k];
                part.part_seg_hi[k] = (int)hi;
                if ( (int)hi > segs_done[k] ) any = 1;
                segs_done[k] = (int)hi;
            }
            if ( any ) {
                for ( int k = 0; k < g->scan_count; k++ )   /* (part_seg_hi == 0 means "the whole scan": an empty range at 0 is [0, 0) of nothing) */
                    if ( part.part_seg_hi[k] == 0 ) part.part_seg_lo[k] = 0;
                if ( gj_launch_huffman_decode(&part, d->stream) ) return -1;
            }
        }
        if ( launch_k4(d, comp_tq, d_out, my0, my1) ||
             gj_cuda_event_record(d->ev_stripe[i], d->stream) || gj_cuda_stream_wait_event(d->copy_stream, d->ev_stripe[i]) ||
             gj_cuda_memcpy_d2h_async(h_dst + off, d_out + off, bytes, d->copy_stream) )
            return -1;
    }
    if ( gj_cuda_event_record(d->ev_done, d->copy_stream) || gj_cuda_stream_wait_event(d->stream, d->ev_done) ) return -1;
    return 0;
}

/* A stream whose restart markers do not count RST0..RST7 cyclically (or whose count does not fit the geometry): the
 * reference's reader ends the current segment at the offending marker, skips everything up to the next marker that
 * carries the EXPECTED number, and goes on from there with consecutive segment numbers; when no such marker follows, the
 * rest of the scan is dropped [ref: src/gpujpeg_reader.c:1038-1155].  The same walk here, over the marker list K0 built
 * (fetched from the device only on this path); the result is an explicit table {raw start, clean start, clean end} per
 * segment for K3, segments that no longer exist marked absent (their blocks decode to zero, as the reference's cleared
 * coefficient buffer gives, src/gpujpeg_decoder.c:301). */
static int resync_segments(struct gpujpeg_decoder* d, const struct gj_stream* st, const uint32_t first_rank[GJ_MAX_COMP],
                           const uint32_t end_rank[GJ_MAX_COMP], const uint32_t scan_cbegin[GJ_MAX_COMP], struct gj_huff_dec_args* ha)
{
    const struct gj_geometry* g = &d->geo;
    const uint32_t n_list = end_rank[g->scan_count - 1] + 1;
    uint8_t* code = (uint8_t*)malloc((size_t)n_list);
    uint32_t* pos = (uint32_t*)malloc((size_t)n_list * 8);
    uint32_t* tab = (uint32_t*)malloc((size_t)g->seg_count * 12);
    int rc = -1;
    if ( code && pos && tab && !gj_cuda_memcpy_d2h_async(code, d->d_list_code, n_list, d->stream) &&
         !gj_cuda_memcpy_d2h_async(pos, d->d_list_pos, (size_t)n_list * 4, d->stream) &&
         !gj_cuda_memcpy_d2h_async(pos + n_list, d->d_list_cpos, (size_t)n_list * 4, d->stream) && !gj_cuda_stream_sync(d->stream) ) {
        const uint32_t* cpos = pos + n_list;
        for ( int k = 0; k < g->scan_count; k++ ) {
            const int seg0 = g->lay.scan_seg_begin[k], segs = g->lay.scan_seg_begin[k + 1] - seg0;
            int n = 0, prev = 7;   /* "RST0 - 1" */
            uint32_t start_raw = (uint32_t)st->scan[k].begin, start_clean = scan_cbegin[k];
            uint32_t m = first_rank[k];
            while ( m < end_rank[k] && n < segs ) {   /* markers [first_rank, end_rank) are the scan's RSTn */
                const int expected = (prev + 1) & 7;
                tab[3 * (seg0 + n)] = start_raw;
                tab[3 * (seg0 + n) + 1] = start_clean;
                tab[3 * (seg0 + n) + 2] = cpos[m];
                n++;
                if ( (code[m] & 7) != expected ) {
                    GJ_ERR("Expected marker 0x%X but 0x%X was presented!\n", 0xD0 + expected, code[m]);
                    uint32_t q = m + 1;
                    while ( q < end_rank[k] && code[q] != 0xD0 + expected ) q++;
                    if ( q >= end_rank[k] ) {
                        GJ_ERR("No marker 0x%X was found until end of current scan!\n", 0xD0 + expected);
                        m = end_rank[k] + 1;   /* the rest of the scan is lost */
                        break;
                    }
                    fprintf(stderr, "[GPUJPEG] [Recovery] Skipping %u bytes of data until marker 0x%X was found!\n",
                            pos[q] - pos[m], 0xD0 + expected);
                    m = q;
                }
                prev = expected;
                start_raw = pos[m] + 2;
                start_clean = cpos[m];
                m++;
            }
            if ( m <= end_rank[k] && n < segs ) {   /* the data in front of the marker that ends the scan */
                tab[3 * (seg0 + n)] = start_raw;
                tab[3 * (seg0 + n) + 1] = start_clean;
                tab[3 * (seg0 + n) + 2] = cpos[end_rank[k]];
                n++;
            }
            for ( ; n < segs; n++ ) {
                tab[3 * (seg0 + n)] = 0xFFFFFFFFu;   /* absent */
                tab[3 * (seg0 + n) + 1] = tab[3 * (seg0 + n) + 2] = 0;
            }
        }
        if ( !grow_dev((void**)&d->d_seg_tab, &d->d_seg_tab_size, (size_t)g->seg_count * 12) &&
             !gj_cuda_memcpy_h2d_async(d->d_seg_tab, tab, (size_t)g->seg_count * 12, d->stream) &&
             !gj_cuda_memset_async(d->d_mk + 3, 0, 4, d->stream) && !gj_cuda_stream_sync(d->stream) ) {
            ha->d_seg_tab = d->d_seg_tab;
            rc = 0;
        }
    }
    if ( rc ) GJ_ERR("Restart resynchronisation failed: %s\n", gj_cuda_last_error());
    free(code);
    free(pos);
    free(tab);
    return rc;
}

/* Segment info [ref: src/gpujpeg_reader.c:1168-1215]: a stream can carry, in front of every scan, the position of every
 * restart segment.  The reference's reader then splits the scan by that table instead of searching for markers; here the
 * search is K0's job on the device, and the table only pays when K3 runs one thread per segment on the file bytes (the
 * other kernels read K0's clean stream; gj_k3_choose): then K0 and the round trip for its report are skipped altogether.
 * The table is advisory: count, order and range are checked, and anything odd sends the frame down the K0 path.
 * Walks the remaining scans on the host (extents from the tables, marker segments between scans by length), fills
 * d->h_seg_off.  Returns 1 if the frame can be decoded from the tables (st / pos / adobe advanced to the end of the
 * stream), 0 to use K0 (st / pos / adobe untouched). */
static int split_by_segment_info(struct gpujpeg_decoder* d, const uint8_t* image, size_t image_size, struct gj_stream* st,
                                 size_t* pos, int* adobe)
{
    const struct gj_geometry* g = &d->geo;
    if ( !st->seginfo[0].pieces || g->seg_mcu <= 0 || st->restart_interval <= 0 || d->ignore_segment_info ) return 0;
    if ( (size_t)g->seg_count * 4 > d->seg_off_size ) {
        gj_cuda_free(d->d_seg_off);
        if ( d->h_seg_off ) gj_cuda_free_host(d->h_seg_off);
        d->d_seg_off = NULL;
        d->h_seg_off = NULL;
        d->seg_off_size = 0;
        if ( gj_cuda_malloc((void**)&d->d_seg_off, (size_t)g->seg_count * 4) ||
             gj_cuda_malloc_host((void**)&d->h_seg_off, (size_t)g->seg_count * 4) )
            return 0;
        d->seg_off_size = (size_t)g->seg_count * 4;
    }
    struct gj_stream t = *st;
    size_t p = *pos;
    int ad = *adobe;
    struct gj_huff_dec_args k3 = {0};   /* (only the scans' bytes and the choice) */
    for ( int k = 0;; k++ ) {
        if ( k >= g->scan_count || k >= t.scan_count ) return 0;
        const struct gj_seginfo* si = &t.seginfo[k];
        const int first = g->lay.scan_seg_begin[k], segs = g->lay.scan_seg_begin[k + 1] - first;
        if ( si->bytes != ((size_t)segs + 1) * 4 ) return 0;
        /* the positions, piece by piece (a piece boundary falls on an entry boundary in the reference's writer; any other
         * cut is read byte-wise all the same).  Checked here: count, order, range; that every segment really starts behind
         * the restart marker with the right number is checked by K3 where it reads the bytes anyway (a host check costs a
         * cache miss per segment: 0.15 ms for an 8K frame) -- a frame that fails there is decoded again by marker scan. */
        const size_t begin = t.scan[k].begin;
        uint32_t prev = 0;
        int piece = 0;
        uint32_t at = 0;
        for ( int i = 0; i <= segs; i++ ) {
            uint32_t v = 0;
            if ( piece < si->pieces && at + 4 <= si->piece_bytes[piece] ) {
                const uint8_t* q = si->piece[piece] + at;
                v = (uint32_t)q[0] << 24 | (uint32_t)q[1] << 16 | (uint32_t)q[2] << 8 | q[3];
                at += 4;
            }
            else {
                for ( int b = 0; b < 4; b++ ) {
                    while ( piece < si->pieces && at >= si->piece_bytes[piece] ) {
                        piece++;
                        at = 0;
                    }
                    if ( piece >= si->pieces ) return 0;
                    v = v << 8 | si->piece[piece][at++];
                }
            }
            if ( (i == 0 && v != 0) || (i > 0 && v < prev + 2) || begin + v + 2 > image_size ) return 0;
            if ( i < segs ) d->h_seg_off[first + i] = (uint32_t)(begin + v);
            prev = v;
        }
        t.scan[k].end = begin + prev;
        if ( image[t.scan[k].end] != 0xFF ) return 0;   /* a marker follows the scan */
        k3.scan_bytes[k] = prev;
        p = t.scan[k].end;
        const int r = gj_reader_walk(image, image_size, &p, &t, &ad);
        if ( r < 0 ) return 0;
        if ( r == 0 ) {
            if ( k + 1 != g->scan_count ) return 0;
            break;
        }
    }
    if ( gj_k3_choose(g, d->huffman_req, d->force_lanes, GJ_K3_SEGMENT_INFO, d->crop, &k3) < 0 ) return 0;
    *st = t;
    *pos = p;
    *adobe = ad;
    return 1;
}

/* K0 on the uploaded file, its report back to the host, and the host's part of the marker walk: per scan from the report
 * alone (no second kernel, no walk over the entropy-coded bytes) where it ends, how many markers lie in front of it, where its
 * clean bytes start; the marker segments between scans are read by length (gj_reader_walk), so that st / pos / adobe end at
 * the end of the stream.  The rank arrays have room for every scan the reader accepts for the frame's process. */
static int k0_scan_extents(struct gpujpeg_decoder* d, const uint8_t* image, size_t image_size, size_t ecs_begin, uint32_t list_cap,
                           struct gj_stream* st, size_t* pos, int* adobe, uint32_t* first_rank, uint32_t* end_rank, uint32_t* scan_cbegin)
{
    const struct gj_geometry* g = &d->geo;
    /* d_mk: [0] total markers, [1] non-RST markers, [2] list overflow, [3] restart sequence error (K3), [5] clean bytes,
     *       [8..] {rank, position, code, clean position} of the non-RST markers */
    if ( gj_launch_marker_scan(d->d_file, ecs_begin, image_size, d->d_cta, d->d_list_pos, d->d_list_code, d->d_list_cpos,
                               list_cap, d->d_clean, d->d_mk, d->d_mk + 8, GJ_MK_OTHER_CAP, d->stream) ||
         gj_cuda_memcpy_d2h_async(d->h_mk, d->d_mk, GJ_MK_WORDS * 4, d->stream) ||
         gj_cuda_stream_sync(d->stream) ) {
        GJ_ERR("Marker scan failed: %s\n", gj_cuda_last_error());
        return -1;
    }

    /* ---- host reader, part 2: scan extents from the marker list, marker segments between scans by length ---- */
    const uint32_t n_other = d->h_mk[1];
    if ( n_other == 0 || n_other > GJ_MK_OTHER_CAP ) {
        GJ_ERR("JPEG stream has %u restart markers / %u other markers in its scan data, expected %d restart segments "
               "for a %dx%d image with restart interval %d!\n", d->h_mk[0], n_other, g->seg_count, st->width, st->height,
               st->restart_interval);
        return -1;
    }
    uint32_t* other = d->h_mk + 8; /* insertion sort by position: a handful of entries */
    for ( uint32_t i = 1; i < n_other; i++ ) {
        uint32_t t[4] = {other[4 * i], other[4 * i + 1], other[4 * i + 2], other[4 * i + 3]};
        uint32_t j = i;
        while ( j > 0 && other[4 * (j - 1) + 1] > t[1] ) {
            memcpy(other + 4 * j, other + 4 * (j - 1), 16);
            j--;
        }
        memcpy(other + 4 * j, t, 16);
    }
    /* per scan, from the marker report alone (no second kernel, no walk over the entropy-coded bytes): where it ends,
     * how many markers lie in front of it, how many restart markers it holds, where its clean bytes start */
    for ( int k = 0; k < st->scan_count; k++ ) {
        /* a scan ends at the first marker that is not RSTn: inside entropy-coded data that test is exact */
        size_t e1 = 0;
        int last_before = -1;
        for ( uint32_t i = 0; i < n_other; i++ ) {
            if ( other[4 * i + 1] >= st->scan[k].begin ) {
                e1 = other[4 * i + 1];
                end_rank[k] = other[4 * i];
                break;
            }
            last_before = (int)i;
        }
        if ( last_before >= 0 ) {
            /* the last marker in front of the scan (its SOS): everything up to the scan's first byte that K0 kept
             * belongs to the clean stream too -- the same keep rule, applied to the few header bytes */
            const uint32_t* m = other + 4 * last_before;
            first_rank[k] = m[0] + 1;
            uint32_t c = m[3];
            if ( st->scan[k].begin - m[1] > 4096 ) {
                GJ_ERR("Unsupported scan structure (no marker in front of scan %d).\n", k);
                return -1;
            }
            for ( size_t q = (size_t)m[1] + 2; q < st->scan[k].begin; q++ ) {
                const int b0 = image[q], b1 = q + 1 < image_size ? image[q + 1] : 0, prev = image[q - 1];
                if ( !((b0 == 0xFF && b1 != 0) || (prev == 0xFF && b0 != 0xFF)) ) c++;
            }
            scan_cbegin[k] = c;
        }
        if ( e1 == 0 ) {
            GJ_ERR("JPEG data unexpected ended while reading SOS marker!\n");
            return -1;
        }
        st->scan[k].end = e1;
        *pos = e1;
        const int r = gj_reader_walk(image, image_size, pos, st, adobe);
        if ( r < 0 ) return -1;
        if ( r == 0 ) break; /* EOI (or end of data) */
    }
    return 0;
}

/* upload the file once, untouched, into buffers sized for K0 (marker list of list_cap entries, clean stream, tile status) */
static int upload_file(struct gpujpeg_decoder* d, const uint8_t* image, size_t image_size, size_t ecs_begin, uint32_t list_cap, int stats)
{
    const size_t n_cta = (image_size - ecs_begin + 16) / 4096 + 2;
    if ( grow_dev((void**)&d->d_file, &d->d_file_size, image_size + 64) ||
         grow_dev((void**)&d->d_list_pos, &d->d_list_pos_size, (size_t)list_cap * 4) ||
         grow_dev((void**)&d->d_list_code, &d->d_list_code_size, (size_t)list_cap) ||
         grow_dev((void**)&d->d_list_cpos, &d->d_list_cpos_size, (size_t)list_cap * 4) ||
         grow_dev((void**)&d->d_clean, &d->d_clean_size, image_size - ecs_begin + 64) ||
         grow_mk_cta(d, n_cta * 8) ) {
        GJ_ERR("Decoder device allocation failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( stats && d->timers_ok ) gj_timer_start(&d->t_to, d->stream);
    if ( gj_cuda_memcpy_h2d_async(d->d_file, image, image_size, d->stream) ) {
        GJ_ERR("Decoder copy of compressed data failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( stats && d->timers_ok ) gj_timer_stop(&d->t_to, d->stream);
    return 0;
}

/* K4 (whole frame, or stripe by stripe with the copies to the host overlapped) straight into the buffer the caller asked for,
 * the channel remap, the copy to the host; k3_part: the Huffman decoder runs per stripe as well (decode_striped) */
static int k4_and_output(struct gpujpeg_decoder* d, struct gpujpeg_decoder_output* output, const struct gpujpeg_image_parameters* pi,
                         const int comp_tq[GJ_MAX_COMP], int striped, const struct gj_huff_dec_args* k3_part, int stats)
{
    const int to_host = output->type == GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER || output->type == GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER;
    uint8_t* d_out = d->d_raw;
    if ( output->type == GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER ) {
        if ( !output->data ) return -1;
        d_out = output->data;
    }
    else if ( output->type == GPUJPEG_DECODER_OUTPUT_OPENGL_TEXTURE ) {
        GJ_ERR("OpenGL texture output is not supported in this build.\n");
        return -1;
    }
    uint8_t* h_dst = output->data;
    if ( to_host ) {
        if ( output->type == GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER ) {
            if ( grow_host((void**)&d->h_raw, &d->h_raw_size, d->out_size) ) return -1;
            h_dst = d->h_raw;
        }
        else if ( !h_dst ) {
            return -1;
        }
    }
    int copied = 0;
    if ( striped ) {
        if ( decode_striped(d, comp_tq, d_out, h_dst, k3_part) ) {
            GJ_ERR("Inverse DCT / copy of raw data failed: %s\n", gj_cuda_last_error());
            return -1;
        }
        copied = 1;
    }
    else if ( launch_k4(d, comp_tq, d_out, 0, d->k4.mcu_rows) ) {
        GJ_ERR("Inverse DCT launch failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( d->channel_remap ) {   /* on the finished raw image, in place [ref: src/gpujpeg_postprocessor.cu:450, 493] */
        struct gj_raw_layout rl;
        if ( gj_raw_layout_init(&rl, pi) ) return -1;
        const int rc = gj_launch_channel_remap(d_out, &rl, pi->pixel_format, pi->width, pi->height, d->channel_remap, d->stream);
        if ( rc == -2 ) GJ_ERR("Wrong channel remapping given, given %u channels but pixel format has %d!\n", d->channel_remap >> 24,
                               gpujpeg_pixel_format_get_comp_count(pi->pixel_format));
        else if ( rc == -3 ) GJ_ERR("Channel remapping is not implemented for chroma-subsampled pixel formats in this build.\n");
        if ( rc ) return -1;
    }
    if ( stats && d->timers_ok ) {
        gj_timer_stop(&d->t_dct, d->stream);
        gj_timer_stop(&d->t_gpu, d->stream);
    }

    output->data_size = d->out_size;
    output->param_image = *pi;
    if ( to_host ) {
        if ( !copied ) {
            if ( stats && d->timers_ok ) gj_timer_start(&d->t_from, d->stream);
            if ( gj_cuda_memcpy_d2h_async(h_dst, d_out, d->out_size, d->stream) ) {
                GJ_ERR("Decoder copy of raw data failed: %s\n", gj_cuda_last_error());
                return -1;
            }
            if ( stats && d->timers_ok ) gj_timer_stop(&d->t_from, d->stream);
        }
        output->data = h_dst;
    }
    else {
        output->data = d_out;
    }
    return 0;
}

/* the per-stage timers of the frame just decoded (gpujpeg_decoder_get_stats) */
static void record_stats(struct gpujpeg_decoder* d, const struct gpujpeg_decoder_output* output, const struct gpujpeg_image_parameters* pi,
                         int stats, double t_reader_ms, double t_begin)
{
    d->stats_valid = 0;
    if ( stats && d->timers_ok ) {
        memset(&d->stats, 0, sizeof d->stats);
        d->stats.duration_stream = t_reader_ms;
        d->stats.duration_memory_to = gj_timer_ms(&d->t_to);
        d->stats.duration_huffman_coder = gj_timer_ms(&d->t_huff);
        d->stats.duration_dct_quantization = gj_timer_ms(&d->t_dct);
        d->stats.duration_in_gpu = gj_timer_ms(&d->t_gpu);
        if ( output->type == GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER || output->type == GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER )
            d->stats.duration_memory_from = gj_timer_ms(&d->t_from);
        d->stats_valid = 1;
        if ( d->verbose >= GPUJPEG_LL_STATUS ) {
            fprintf(stderr, " -Stream Reader:     %10.3f ms\n", d->stats.duration_stream);
            fprintf(stderr, " -Copy To Device:    %10.3f ms\n", d->stats.duration_memory_to);
            fprintf(stderr, " -Huffman Decoder:   %10.3f ms\n", d->stats.duration_huffman_coder);
            fprintf(stderr, " -DeQuant+IDCT+Post: %10.3f ms\n", d->stats.duration_dct_quantization);
            fprintf(stderr, " -Copy From Device:  %10.3f ms\n", d->stats.duration_memory_from);
            fprintf(stderr, "Decode Image GPU:    %10.3f ms (only in-GPU processing)\n", d->stats.duration_in_gpu);
            fprintf(stderr, "Decode Image:        %10.3f ms\n", (gpujpeg_get_time() - t_begin) * 1000.0);
            fprintf(stderr, "Decompressed Size:%13zu bytes %dx%d %s %s\n", output->data_size, pi->width, pi->height,
                    gpujpeg_pixel_format_get_name(pi->pixel_format), gpujpeg_color_space_get_name(pi->color_space));
        }
    }
}

/* The output buffers of the frame: pi is the output (at scaled frames ceil(W / scale) x ceil(H / scale) pixels), d->geo the
 * stream's own geometry.  A scaled component keeps its block grid; its samples that carry image data are counted as
 * gj_geometry_init counts them for an image of the output's size. */
static int size_output(struct gpujpeg_decoder* d, const struct gpujpeg_image_parameters* pi)
{
    const struct gj_geometry* g = &d->geo;
    d->out_w = pi->width;
    d->out_h = pi->height;
    d->out_size = d->scale == 1 && !d->crop ? g->raw_size : d->raw.size;
    for ( int c = 0; c < g->comp_count; c++ ) {
        const int div_h = g->max_hs / g->comp[c].hs, div_v = g->max_vs / g->comp[c].vs;
        d->scomp[c] = g->comp[c];
        d->scomp[c].width = (pi->width + div_h - 1) / div_h;
        d->scomp[c].height = (pi->height + div_v - 1) / div_v;
    }
    if ( grow_dev((void**)&d->d_raw, &d->d_raw_size, d->out_size) || grow_dev((void**)&d->d_planes, &d->d_planes_size, d->k4.planes_bytes) ) {
        GJ_ERR("Decoder device allocation failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    return 0;
}

/* dec_opt_crop: room for `pairs` {segment, blocks} pairs on the host and the device */
static int grow_pick(struct gpujpeg_decoder* d, size_t pairs)
{
    if ( pairs * 8 > d->h_pick_size ) {
        free(d->h_pick);
        d->h_pick_size = 0;
        if ( !(d->h_pick = (uint32_t*)malloc(pairs * 8)) ) return -1;
        d->h_pick_size = pairs * 8;
    }
    return grow_dev((void**)&d->d_pick, &d->d_pick_size, pairs * 8);
}

/* gj_decoder_decode_coefficients with a window: the caller's rectangle of blocks on the frame's geometry, decoded as a
 * dec_opt_crop frame decodes the blocks K4 needs (the same pick lists, the same kernels, the same extent rule) */
static int coef_window(struct gpujpeg_decoder* d, const struct gj_stream* st)
{
    if ( !d->coef_only || !d->coef_window ) return 0;
    const int r = d->coef_window(d->coef_window_ctx, &d->geo, st->progressive, &st->metadata, d->k4.win.blk);
    if ( r < 0 ) return -1;
    d->crop = r;
    return 0;
}

/* Progressive (SOF2) frames, from the first SOS on: the same upload, K0 and host marker walk as a baseline frame, then per
 * scan the parameters and Huffman tables (those in force at its SOS), one table upload, the scan kernels in stream order
 * (gj_progressive.cu) and the same K4 / output stage.  Segment-info tables and dec_opt_huffman / dec_opt_huffman_lanes do not
 * apply; a restart marker with the wrong number is refused (no resynchronisation). */
static int decode_progressive(struct gpujpeg_decoder* d, uint8_t* image, size_t image_size, struct gpujpeg_decoder_output* output,
                              struct gj_stream* st, struct gpujpeg_parameters* p, struct gpujpeg_image_parameters* pi,
                              const struct gj_k4_request* k4, size_t pos, int adobe, enum gpujpeg_color_space early_cs, int stats,
                              double t_begin)
{
    static const int comp_tq[GJ_MAX_COMP] = {0, 1, 2, 3};   /* qinv_zz[c]: the table component c latched at its first scan */
    d->last_valid = 0;
    d->used_segment_info = 0;
    d->used_subsequences = 0;
    if ( (!d->prog_scans && !(d->prog_scans = (struct gj_prog_scan*)malloc(sizeof(struct gj_prog_scan) * GJ_MAX_SCANS))) ||
         (!d->h_prog_luts && !(d->h_prog_luts = (struct gj_dec_lut*)malloc(sizeof(struct gj_dec_lut) * GJ_MAX_SCANS * GJ_MAX_COMP))) ||
         (!d->d_prog_luts && gj_cuda_malloc((void**)&d->d_prog_luts, sizeof(struct gj_dec_lut) * GJ_MAX_SCANS * GJ_MAX_COMP)) ) {
        GJ_ERR("Decoder allocation failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    /* every restart marker of every scan goes into K0's list: at most one per two bytes of entropy-coded data */
    const size_t ecs_begin = st->scan[0].begin;
    const uint32_t list_cap = (uint32_t)((image_size - ecs_begin) / 2 + 1 + GJ_MK_OTHER_CAP);
    uint32_t first_rank[GJ_MAX_SCANS], end_rank[GJ_MAX_SCANS], scan_cbegin[GJ_MAX_SCANS];
    memset(first_rank, 0, sizeof first_rank);
    memset(end_rank, 0, sizeof end_rank);
    memset(scan_cbegin, 0, sizeof scan_cbegin);
    if ( upload_file(d, image, image_size, ecs_begin, list_cap, stats) ||
         k0_scan_extents(d, image, image_size, ecs_begin, list_cap, st, &pos, &adobe, first_rank, end_rank, scan_cbegin) ||
         gj_reader_finish(st, adobe, d->verbose) )
        return GPUJPEG_ERROR;
    d->metadata = st->metadata;
    if ( d->orient ) memset(&d->metadata.vals[GPUJPEG_METADATA_ORIENTATION], 0, sizeof d->metadata.vals[0]);   /* the pixels are upright */
    if ( st->color_space != early_cs ) {
        GJ_ERR("The stream's colour space (%s) is announced after its first scan header; not supported.\n",
               gpujpeg_color_space_get_name(st->color_space));
        return GPUJPEG_ERROR;
    }
    /* the coefficient planes are padded to whole MCUs as soon as any scan interleaves (libjpeg's DC scans do) */
    int il = 0;
    for ( int k = 0; k < st->scan_count; k++ )
        il |= st->scan[k].ncomp > 1;
    if ( il != p->interleaved ) {
        struct gpujpeg_image_parameters pg = *pi;   /* the coefficient planes: the stream's own size */
        pg.width = st->width;
        pg.height = st->height;
        p->interleaved = il;
        if ( gpujpeg_decoder_init(d, p, &pg) ) return GPUJPEG_ERROR;
        gj_k4_choose(&d->geo, k4, &d->k4);   /* (the planes are padded to whole MCUs now) */
        if ( !d->coef_only && size_output(d, pi) ) return GPUJPEG_ERROR;
    }
    const struct gj_geometry* g = &d->geo;
    if ( coef_window(d, st) ) return GPUJPEG_ERROR;

    /* scans and their Huffman tables */
    int nlut = 0;
    for ( int k = 0; k < st->scan_count; k++ ) {
        struct gj_prog_scan* S = &d->prog_scans[k];
        if ( gj_prog_scan_init(g, st, k, st->restart_interval, S) ) {
            GJ_ERR("Unsupported scan structure (progressive scan %d: components out of frame order or outside the frame).\n", k);
            return GPUJPEG_ERROR;
        }
        S->first_rank = first_rank[k];
        S->cbegin = scan_cbegin[k];
        if ( end_rank[k] >= list_cap || end_rank[k] - first_rank[k] != (uint32_t)(S->seg_count - 1) ) {
            GJ_ERR("JPEG stream has a broken restart-marker structure (progressive scan %d holds %u restart markers, expected %d)!\n",
                   k, end_rank[k] - first_rank[k], S->seg_count - 1);
            return GPUJPEG_ERROR;
        }
        S->lut0 = nlut;
        const int nt = S->kind == GJ_PROG_DC_FIRST ? S->ncomp : S->kind == GJ_PROG_DC_REFINE ? 0 : 1;
        for ( int i = 0; i < nt; i++ ) {
            if ( !st->scan[k].huff_at[i] ) {
                GJ_ERR("Huffman table used by progressive scan %d is missing!\n", k);
                return GPUJPEG_ERROR;
            }
            struct gj_huff_spec spec;
            gj_huff_spec_at(image, st->scan[k].huff_at[i], &spec);
            if ( gj_dec_lut_build(&spec, &d->h_prog_luts[nlut++]) ) {
                GJ_ERR("Invalid Huffman table (progressive scan %d)!\n", k);
                return GPUJPEG_ERROR;
            }
        }
    }
    /* dequantisation by component: the table latched at the component's first scan */
    memset(&d->h_tab, 0, sizeof d->h_tab);
    for ( int c = 0; c < st->comp_count; c++ ) {
        const uint8_t* q = st->have_comp_qt[c] ? st->comp_qt[c] : st->have_qt[st->comp_tq[c]] ? st->qt[st->comp_tq[c]] : NULL;
        for ( int k = 0; q && k < 64; k++ )
            d->h_tab.qinv_zz[c][k] = q[k];
        if ( d->coef_only ) {
            d->coef_tq[c] = st->comp_tq[c];
            memset(d->coef_qt[c], 0, 64);
            if ( q ) memcpy(d->coef_qt[c], q, 64);
        }
    }
    const double t_reader_ms = (gpujpeg_get_time() - t_begin) * 1000.0;
    if ( !d->tab_valid || memcmp(&d->h_tab, &d->h_tab_prev, sizeof d->h_tab) != 0 ) {
        d->h_tab_prev = d->h_tab;
        if ( gj_cuda_memcpy_h2d_async(d->d_tab, &d->h_tab_prev, sizeof d->h_tab, d->stream) ) return GPUJPEG_ERROR;
        d->tab_valid = 1;
    }
    if ( nlut && gj_cuda_memcpy_h2d_async(d->d_prog_luts, d->h_prog_luts, sizeof(struct gj_dec_lut) * (size_t)nlut, d->stream) )
        return GPUJPEG_ERROR;

    struct gj_prog_args* a = &d->last_prog;
    memset(a, 0, sizeof *a);
    if ( d->crop ) {   /* every scan decodes the segments that hold the rectangle's blocks (gj_prog_crop_pick) */
        size_t pairs = 0;
        for ( int k = 0; k < st->scan_count; k++ )
            pairs += (size_t)d->prog_scans[k].seg_count;
        if ( grow_pick(d, pairs) ) {
            GJ_ERR("Decoder allocation failed: %s\n", gj_cuda_last_error());
            return GPUJPEG_ERROR;
        }
        int n = 0;
        for ( int k = 0; k < st->scan_count; k++ ) {
            a->pick_off[k] = n;
            a->pick_n[k] = gj_prog_crop_pick(&d->prog_scans[k], st->scan[k].comp, d->k4.win.blk, d->h_pick + 2 * n);
            n += a->pick_n[k];
        }
        if ( n && gj_cuda_memcpy_h2d_async(d->d_pick, d->h_pick, (size_t)n * 8, d->stream) ) return GPUJPEG_ERROR;
        a->d_pick = d->d_pick;
    }
    a->scans = d->prog_scans;
    a->scan_count = st->scan_count;
    a->d_luts = d->d_prog_luts;
    a->d_clean = (const uint32_t*)d->d_clean;
    a->d_list_cpos = d->d_list_cpos;
    a->d_list_code = d->d_list_code;
    a->d_error = d->d_mk + 3;
    a->d_coef = d->d_coef;
    a->d_cext = d->d_cext;
    a->coef_count = g->coef_count;
    a->dequantize = d->k4.dequantize;
    a->comp_count = g->comp_count;
    for ( int c = 0; c < g->comp_count; c++ )
        a->comp_blk_off[c] = g->comp[c].blk_off;
    a->d_tables = d->d_tab;
    d->last_args.file_size = image_size;   /* what a resident re-run of K0 needs */
    d->last_ecs_begin = ecs_begin;
    d->last_list_cap = list_cap;
    d->last_progressive = 1;
    d->last_valid = 1;
    if ( stats && d->timers_ok ) {
        gj_timer_start(&d->t_gpu, d->stream);
        gj_timer_start(&d->t_huff, d->stream);
    }
    if ( gj_launch_progressive_decode(a, d->stream) ) {
        GJ_ERR("Progressive Huffman decoder launch failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    if ( stats && d->timers_ok ) {
        gj_timer_stop(&d->t_huff, d->stream);
        gj_timer_start(&d->t_dct, d->stream);
    }
    const int to_host = output->type == GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER || output->type == GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER;
    const int striped = to_host && !stats && stripes_usable(d);
    if ( !d->coef_only && k4_and_output(d, output, pi, comp_tq, striped, NULL, stats) ) return GPUJPEG_ERROR;
    if ( gj_cuda_memcpy_d2h_async(d->h_mk, d->d_mk, 16, d->stream) || gj_cuda_stream_sync(d->stream) ) {
        GJ_ERR("Decoder failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    if ( d->h_mk[3] ) {
        GJ_ERR("Restart marker with the wrong number in a progressive scan; not supported.\n");
        d->last_valid = 0;
        return GPUJPEG_ERROR;
    }
    output->metadata = &d->metadata;
    record_stats(d, output, pi, stats, t_reader_ms, t_begin);
    return GPUJPEG_NOERR;
}

/* dec_opt_pixels=libjpeg is defined for full-range YCbCr (JFIF, Adobe transform 1), RGB-internal (Adobe transform 0) and grey
 * streams, at scale 1, with the default IDCT option, no flip and no channel remap: 1 (with a message) for anything else */
static int libjpeg_refused(const struct gpujpeg_decoder* d, const struct gj_stream* st, enum gpujpeg_color_space cs)
{
    const char* why = st->comp_count == 4                                                        ? "4-component streams"
                      : cs != GPUJPEG_YCBCR_BT601_256LVLS && cs != GPUJPEG_RGB                  ? gpujpeg_color_space_get_name(cs)
                      : d->scale_req != 1                                                       ? GPUJPEG_DEC_OPT_SCALE " other than 1"
                      : d->flipped                                                              ? GPUJPEG_DEC_OPT_FLIPPED_BOOL
                      : d->channel_remap                                                        ? GPUJPEG_DEC_OPT_CHANNEL_REMAP
                      : d->idct_flavour != 0                                                    ? GPUJPEG_DEC_OPT_IDCT " other than int"
                                                                                                : NULL;
    if ( why ) GJ_ERR("dec_opt_pixels=libjpeg is not supported for %s.\n", why);
    return why != NULL;
}

/* [ref: src/gpujpeg_decoder.c:234-469] */
int gpujpeg_decoder_decode(struct gpujpeg_decoder* d, uint8_t* image, size_t image_size,
                           struct gpujpeg_decoder_output* output)
{
    if ( !d || !image || !output ) return GPUJPEG_ERROR;
    const int stats = d->perf_stats || d->verbose >= GPUJPEG_LL_STATUS;
    const double t_begin = gpujpeg_get_time();

    /* ---- host reader, part 1: marker segments up to the first SOS (never touches entropy-coded data) ---- */
    struct gj_stream st;
    gj_reader_begin(&st, d->ff_cs_itu601_is_709);
    st.verbose = d->verbose;
    if ( image_size < 4 || image[0] != 0xFF || image[1] != 0xD8 ) {
        GJ_ERR("JPEG data should begin with SOI marker!\n");
        return GPUJPEG_ERROR;
    }
    if ( image_size >= 0xFFFFFFFFull ) {
        GJ_ERR("JPEG streams of 4 GiB or more are not supported.\n");
        return GPUJPEG_ERROR;
    }
    size_t pos = 2;
    int adobe = -1;
    if ( gj_reader_walk(image, image_size, &pos, &st, &adobe) != 1 ) {
        GJ_ERR("Decoder failed when decoding image data (no scan found)!\n");
        return GPUJPEG_ERROR;
    }
    if ( st.comp_count != 3 && st.comp_count != 1 && st.comp_count != 4 ) {
        GJ_ERR("This build decodes 1-, 3- and 4-component JPEGs only (stream has %d).\n", st.comp_count);
        return GPUJPEG_ERROR;
    }
    if ( st.comp_count == 1 ) st.comp_hv[0] = 0x11;   /* a single component is never subsampled (T.81 A.2.2) */
    /* luminance 1x1, 2x1, 1x2 or 2x2 with 1x1 chrominance (4:4:4, 4:2:2, 4:4:0, 4:2:0) */
    if ( st.comp_count >= 3 ) {   /* (a fourth component -- alpha -- with the first component's sampling) */
        const int lh = st.comp_hv[0] >> 4, lv = st.comp_hv[0] & 15;
        if ( lh < 1 || lh > 2 || lv < 1 || lv > 2 || st.comp_hv[1] != 0x11 || st.comp_hv[2] != 0x11 ||
             (st.comp_count == 4 && st.comp_hv[3] != st.comp_hv[0]) ) {
            GJ_ERR("This build decodes 4:4:4, 4:2:2, 4:2:0 and 4:4:0 only (sampling factors %dx%d %dx%d %dx%d).\n", lh, lv,
                   st.comp_hv[1] >> 4, st.comp_hv[1] & 15, st.comp_hv[2] >> 4, st.comp_hv[2] & 15);
            return GPUJPEG_ERROR;
        }
    }
    st.interleaved = st.scan[0].ncomp > 1;
    if ( !st.progressive && st.interleaved && st.scan[0].ncomp != st.comp_count ) {
        GJ_ERR("Unsupported scan structure (%d components in first scan).\n", st.scan[0].ncomp);
        return GPUJPEG_ERROR;
    }

    struct gpujpeg_parameters p;
    gpujpeg_set_default_parameters(&p);
    p.verbose = d->verbose;
    p.perf_stats = d->perf_stats;
    p.restart_interval = st.restart_interval;
    p.interleaved = st.interleaved;
    p.comp_count = st.comp_count;
    memset(p.sampling_factor, 0, sizeof p.sampling_factor);
    for ( int c = 0; c < st.comp_count; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)(st.comp_hv[c] >> 4);
        p.sampling_factor[c].vertical = (uint8_t)(st.comp_hv[c] & 15);
    }
    /* colour space of the components: SPIFF header / Adobe APP14 / component ids seen so far decide (the same rule gj_reader_finish
     * applies at the end; a stream that changes its mind after the first SOS is refused below) */
    const enum gpujpeg_color_space early_cs = gj_stream_color_space(&st, adobe);
    st.color_space = early_cs;
    p.color_space_internal = early_cs;
    /* dec_opt_scale: the output is ceil(W / scale) x ceil(H / scale) pixels, negotiated as a full-size image of that size */
    if ( d->scale_req > 1 && d->flipped ) {
        GJ_ERR("dec_opt_flipped is not supported together with dec_opt_scale.\n");
        return GPUJPEG_ERROR;
    }
    if ( d->crop_req && d->flipped ) {
        GJ_ERR("dec_opt_flipped is not supported together with dec_opt_crop.\n");
        return GPUJPEG_ERROR;
    }
    /* dec_opt_orientation: the stream's own orientation (SPIFF directory / Exif, read with the headers) or the option's */
    int rot = d->orient_rot, oflip = d->orient_flip;
    if ( d->orient_mode == 1 ) {
        const int set = st.metadata.vals[GPUJPEG_METADATA_ORIENTATION].set;
        rot = set ? (int)st.metadata.vals[GPUJPEG_METADATA_ORIENTATION].orient.rotation : 0;
        oflip = set ? (int)st.metadata.vals[GPUJPEG_METADATA_ORIENTATION].orient.flip : 0;
    }
    const int orient = d->orient_mode != 0 && (rot != 0 || oflip != 0);
    /* (the flip acts on the padded planes, which is no mirror of the image; see below) */
    if ( orient && d->flipped ) {
        GJ_ERR("dec_opt_flipped is not supported together with dec_opt_orientation.\n");
        return GPUJPEG_ERROR;
    }
    /* dec_opt_pixels=libjpeg: the streams and options it is defined for */
    const int libjpeg = d->pixels_req && !d->coef_only;
    if ( libjpeg && libjpeg_refused(d, &st, early_cs) ) return GPUJPEG_ERROR;
    /* the frame's scale, rectangle and orientation are committed to the decoder only once nothing below can refuse the frame: a
     * refused frame leaves the last frame's state, which a resident re-run may still use, untouched */
    const int scale = d->scale_req;
    int crop = 0;
    struct gpujpeg_image_parameters pi;
    gpujpeg_image_set_default_parameters(&pi);
    const int sw = (st.width + scale - 1) / scale, sh = (st.height + scale - 1) / scale;   /* the (scaled) image as stored */
    pi.width = (rot & 1) ? sh : sw;   /* the output: a quarter turn swaps the sides */
    pi.height = (rot & 1) ? sw : sh;
    /* dec_opt_crop: the output is the rectangle (of the oriented image), negotiated as an image of its size */
    if ( d->crop_req ) {
        if ( d->crop_rx >= pi.width || d->crop_ry >= pi.height || d->crop_rw > pi.width - d->crop_rx || d->crop_rh > pi.height - d->crop_ry ) {
            GJ_ERR("Crop %dx%d+%d+%d does not lie inside the %dx%d output image.\n", d->crop_rw, d->crop_rh, d->crop_rx, d->crop_ry,
                   pi.width, pi.height);
            return GPUJPEG_ERROR;
        }
        /* a rectangle that is the whole image is the plain decode (the stripe pipeline included) */
        if ( d->crop_rw < pi.width || d->crop_rh < pi.height ) crop = 1;
        pi.width = d->crop_rw;
        pi.height = d->crop_rh;
    }
    const int out = choose_output(d, &st, &pi);
    if ( !out ) return GPUJPEG_ERROR;
    if ( libjpeg ) {
        if ( st.comp_count == 3 ? pi.pixel_format != GPUJPEG_444_U8_P012 || pi.color_space != GPUJPEG_RGB
                                : pi.color_space != GPUJPEG_YCBCR_BT601_256LVLS ) {
            GJ_ERR("dec_opt_pixels=libjpeg produces GPUJPEG_RGB 444-u8-p012 (grey streams: GPUJPEG_U8) only (%s %s requested).\n",
                   gpujpeg_color_space_get_name(pi.color_space), gpujpeg_pixel_format_get_name(pi.pixel_format));
            return GPUJPEG_ERROR;
        }
    }
    /* the 2:1 chroma pairs of a turned or mirrored image of odd size are not the source's pairs turned */
    if ( orient && (pi.pixel_format == GPUJPEG_422_U8_P1020 || pi.pixel_format == GPUJPEG_422_U8_P0P1P2 ||
                    pi.pixel_format == GPUJPEG_420_U8_P0P1P2) ) {
        GJ_ERR("dec_opt_orientation is not supported for pixel format %s (chroma subsampling).\n",
               gpujpeg_pixel_format_get_name(pi.pixel_format));
        return GPUJPEG_ERROR;
    }
    /* the output rectangle's map to the (scaled) image and the rectangle of the image it shows */
    struct gj_k4_request k4 = {out, libjpeg, scale, crop, {0, 0, 0, 0}, orient, {0}, d->flipped, d->idct_flavour, d->coef_only,
                               d->channel_remap != 0};
    int ow, oh;
    const int rect[4] = {d->crop_rx, d->crop_ry, d->crop_rw, d->crop_rh};
    if ( gj_orient_frame(sw, sh, orient ? rot : 0, orient ? oflip : 0, crop ? rect : NULL, &ow, &oh, &k4.map, k4.src) ) return GPUJPEG_ERROR;
    if ( crop ) {
        struct gj_raw_layout rl;
        if ( gj_raw_layout_init(&rl, &pi) == 0 &&
             ((rl.sampling[0].horizontal == 2 && (d->crop_rx & 1)) || (rl.sampling[0].vertical == 2 && (d->crop_ry & 1))) ) {
            GJ_ERR("Crop %dx%d+%d+%d: pixel format %s needs an even %s.\n", d->crop_rw, d->crop_rh, d->crop_rx, d->crop_ry,
                   gpujpeg_pixel_format_get_name(pi.pixel_format), (d->crop_rx & 1) ? "X" : "Y");
            return GPUJPEG_ERROR;
        }
    }
    /* from here on the decoder's buffers and output state change: the last frame can no longer be re-run (a frame that
     * completes sets last_valid again) */
    d->last_valid = 0;
    d->scale = scale;
    d->crop = crop;
    d->orient = orient;
    struct gpujpeg_image_parameters pg = pi;   /* the coefficient planes: the stream's own size */
    pg.width = st.width;
    pg.height = st.height;

    if ( !d->initialised || d->param_image.width != pg.width || d->param_image.height != pg.height ||
         d->param_image.pixel_format != pg.pixel_format || d->param.comp_count != p.comp_count ||
         d->param.color_space_internal != p.color_space_internal ||
         d->param.restart_interval != p.restart_interval || d->param.interleaved != p.interleaved ||
         memcmp(d->param.sampling_factor, p.sampling_factor, sizeof p.sampling_factor) != 0 ) {
        if ( d->initialised ) GJ_VERBOSE(d->verbose, "Reinitializing decoder.\n");
        if ( gpujpeg_decoder_init(d, &p, &pg) ) return GPUJPEG_ERROR;
    }
    gj_k4_choose(&d->geo, &k4, &d->k4);
    d->param_image.color_space = pi.color_space;
    if ( !d->coef_only && (((d->k4.kernel != GJ_K4_FUSED || d->crop) && gj_raw_layout_init(&d->raw, &pi)) || size_output(d, &pi)) )
        return GPUJPEG_ERROR;
    const struct gj_geometry* g = &d->geo;
    if ( !st.progressive && coef_window(d, &st) ) return GPUJPEG_ERROR;

    if ( st.progressive ) return decode_progressive(d, image, image_size, output, &st, &p, &pi, &k4, pos, adobe, early_cs, stats, t_begin);

    /* ---- upload the file once, untouched; K0 builds the marker list on the device ---- */
    const size_t ecs_begin = st.scan[0].begin;
    /* K0 tiles the file from a 16-byte aligned base below the first scan and its tile status holds 31-bit counts; a stream
     * whose scans span 2^31 bytes or more is refused here, before any upload, whether or not it carries segment-info tables
     * (which would skip K0), so that both forms of one stream get the same answer */
    if ( image_size - (ecs_begin & ~(size_t)15) >= ((size_t)1 << 31) ) {
        GJ_ERR("JPEG entropy-coded data of %zu bytes exceeds the supported maximum of 2^31 bytes.\n", image_size - ecs_begin);
        return GPUJPEG_ERROR;
    }
    const uint32_t list_cap = (uint32_t)g->seg_count + GJ_MK_OTHER_CAP;
    if ( upload_file(d, image, image_size, ecs_begin, list_cap, stats) ) return GPUJPEG_ERROR;
    uint32_t first_rank[GJ_MAX_COMP] = {0, 0, 0, 0}, end_rank[GJ_MAX_COMP] = {0, 0, 0, 0}, scan_cbegin[GJ_MAX_COMP] = {0, 0, 0, 0};
    /* ---- scans split by the stream's own segment-info tables (no K0, no round trip), or ... ---- */
    const int by_table = split_by_segment_info(d, image, image_size, &st, &pos, &adobe);
    d->used_segment_info = by_table;
    if ( by_table ) {
        if ( gj_cuda_memcpy_h2d_async(d->d_seg_off, d->h_seg_off, (size_t)g->seg_count * 4, d->stream) ||
             gj_cuda_memset_async(d->d_mk, 0, 32, d->stream) ) {
            GJ_ERR("Decoder copy of the segment table failed: %s\n", gj_cuda_last_error());
            return GPUJPEG_ERROR;
        }
    }
    else {
    /* ---- ... K0 builds the marker list and the clean stream on the device ---- */
    if ( k0_scan_extents(d, image, image_size, ecs_begin, list_cap, &st, &pos, &adobe, first_rank, end_rank, scan_cbegin) )
        return GPUJPEG_ERROR;
    }   /* K0 path */
    if ( gj_reader_finish(&st, adobe, d->verbose) ) return GPUJPEG_ERROR;
    d->metadata = st.metadata;   /* handed out with the output [ref: src/gpujpeg_reader.c:1626-1636, src/gpujpeg_decoder.c:466] */
    if ( d->orient ) memset(&d->metadata.vals[GPUJPEG_METADATA_ORIENTATION], 0, sizeof d->metadata.vals[0]);   /* the pixels are upright */
    if ( st.color_space != early_cs ) {
        GJ_ERR("The stream's colour space (%s) is announced after its first scan header; not supported.\n",
               gpujpeg_color_space_get_name(st.color_space));
        return GPUJPEG_ERROR;
    }
    if ( st.scan_count != g->scan_count ) {
        GJ_ERR("Unsupported scan structure (%d scans, expected %d).\n", st.scan_count, g->scan_count);
        return GPUJPEG_ERROR;
    }
    for ( int c = 0; c < st.comp_count; c++ ) {
        if ( !st.have_qt[st.comp_tq[c]] ) {
            GJ_ERR("Quantization table %d is missing!\n", st.comp_tq[c]);
            return GPUJPEG_ERROR;
        }
        if ( d->coef_only ) {
            d->coef_tq[c] = st.comp_tq[c];
            memcpy(d->coef_qt[c], st.qt[st.comp_tq[c]], 64);
        }
    }

    /* tables: dequantisation (zig-zag order, by table id) and Huffman LUTs (by class and id) */
    memset(&d->h_tab, 0, sizeof d->h_tab);
    for ( int t = 0; t < 4; t++ )
        if ( st.have_qt[t] )
            for ( int k = 0; k < 64; k++ )
                d->h_tab.qinv_zz[t][k] = st.qt[t][k];
    struct gj_huff_dec_args ha;
    memset(&ha, 0, sizeof ha);
    for ( int s = 0; s < st.scan_count; s++ ) {
        if ( st.scan[s].ncomp != g->comps_per_scan ) {
            GJ_ERR("Unsupported scan structure (scan %d has %d components).\n", s, st.scan[s].ncomp);
            return GPUJPEG_ERROR;
        }
        for ( int k = 0; k < st.scan[s].ncomp; k++ ) {
            /* the block order inside an MCU follows the frame's component order (T.81 A.2.3) */
            if ( g->interleaved && st.scan[s].comp[k] != k ) {
                GJ_ERR("Unsupported scan structure (components of the interleaved scan are not in frame order).\n");
                return GPUJPEG_ERROR;
            }
        }
        /* one scan per component: scan s must code component s, so that every component is coded exactly once and
         * the segment / block counts of scan s (geometry) are those of the plane K3 writes to */
        if ( !g->interleaved && st.scan[s].comp[0] != s ) {
            GJ_ERR("Unsupported scan structure (scan %d codes component %d; scans must follow the frame's component order).\n",
                   s, st.scan[s].comp[0]);
            return GPUJPEG_ERROR;
        }
        for ( int k = 0; k < st.scan[s].ncomp; k++ ) {
            const int td = st.scan[s].td[k], ta = st.scan[s].ta[k];
            if ( !st.have_huff[0][td] || !st.have_huff[1][ta] ) {
                GJ_ERR("Huffman table (DC %d / AC %d) used by scan %d is missing!\n", td, ta, s);
                return GPUJPEG_ERROR;
            }
            ha.scan_comp[s][k] = st.scan[s].comp[k];
            ha.scan_td[s][k] = td;
            ha.scan_tq[s][k] = st.comp_tq[st.scan[s].comp[k]];
            ha.scan_ta[s][k] = ta;
        }
        ha.scan_begin[s] = (uint32_t)st.scan[s].begin;
    }
    for ( int cls = 0; cls < 2; cls++ )
        for ( int id = 0; id < 4; id++ )
            if ( st.have_huff[cls][id] ) {
                if ( gj_dec_lut_build(&st.huff[cls][id], &d->h_tab.lut[cls][id]) ) {
                    GJ_ERR("Invalid Huffman table (class %d id %d)!\n", cls, id);
                    return GPUJPEG_ERROR;
                }
                gj_dec_fast_build(&st.huff[cls][id], cls, &d->h_tab.fast[cls][id]);
            }
    const double t_reader_ms = (gpujpeg_get_time() - t_begin) * 1000.0;

    if ( !d->tab_valid || memcmp(&d->h_tab, &d->h_tab_prev, sizeof d->h_tab) != 0 ) {
        /* h_tab_prev is what the in-flight copy reads from: never modified while a frame is running */
        d->h_tab_prev = d->h_tab;
        if ( gj_cuda_memcpy_h2d_async(d->d_tab, &d->h_tab_prev, sizeof d->h_tab, d->stream) ) return GPUJPEG_ERROR;
        d->tab_valid = 1;
    }
    if ( stats && d->timers_ok ) {
        gj_timer_start(&d->t_gpu, d->stream);
        gj_timer_start(&d->t_huff, d->stream);
    }
    /* restart structure [ref: src/gpujpeg_reader.c:1038-1155]: scan k should hold one restart marker per segment boundary,
     * counting RST0..RST7 cyclically.  The count is checked here, the numbering by K3; a stream that fails either is
     * resynchronised the way the reference's reader does it (resync_segments below) and decoded from an explicit
     * segment table. */
    int resync = 0;
    for ( int k = 0; k < g->scan_count && !by_table; k++ ) {
        const int segs = g->lay.scan_seg_begin[k + 1] - g->lay.scan_seg_begin[k];
        if ( end_rank[k] >= list_cap ) {
            GJ_ERR("JPEG stream has a broken restart-marker structure (scan %d holds %u restart markers, expected %d "
                   "for a %dx%d image with restart interval %d)!\n", k, end_rank[k] - first_rank[k], segs - 1, st.width,
                   st.height, st.restart_interval);
            return GPUJPEG_ERROR;
        }
        if ( end_rank[k] - first_rank[k] != (uint32_t)(segs - 1) ) resync = 1;
    }

    /* ---- K3 ---- */
    ha.d_file = d->d_file;
    ha.file_size = image_size;
    ha.dequantize = d->k4.dequantize;
    ha.d_seg_off = by_table ? d->d_seg_off : NULL; /* segment starts: the stream's own table, or the device-built marker list */
    ha.d_seg_len = NULL;
    ha.d_list_pos = d->d_list_pos;
    ha.d_list_code = d->d_list_code;
    ha.d_error = d->d_mk + 3;
    ha.d_unit_ctr = d->d_k3_ctr;
    ha.d_clean = (const uint32_t*)d->d_clean;
    ha.d_list_cpos = d->d_list_cpos;
    for ( int k = 0; k < g->scan_count; k++ ) {
        ha.first_rank[k] = first_rank[k];
        ha.scan_cbegin[k] = scan_cbegin[k];
        ha.scan_bytes[k] = (uint32_t)(st.scan[k].end - st.scan[k].begin);
    }
    const int pick = gj_k3_choose(g, d->huffman_req, d->force_lanes,
                                  by_table ? GJ_K3_SEGMENT_INFO : resync ? GJ_K3_RESYNC_TABLE : GJ_K3_MARKER_LIST, d->crop, &ha);
    if ( pick < 0 ) return GPUJPEG_ERROR;   /* (not for a frame split_by_segment_info accepted: the same question) */
    ha.seg_count = g->seg_count;
    ha.lay = g->lay;
    ha.seg_mcu = g->seg_mcu;
    ha.d_coef = d->d_coef;
    ha.d_cext = d->d_cext;
    ha.d_tables = d->d_tab;
    if ( ha.kernel == GJ_K3_SUBSEQUENCE ) {
        const int ctas = gj_subseq_grid();
        const size_t need = ctas > 0 ? gj_subseq_scratch_bytes(g->seg_count, ha.ecs_bytes, ctas) : 0;
        if ( ctas <= 0 || grow_dev(&d->d_ss_scratch, &d->d_ss_scratch_size, need) ) {
            GJ_ERR("Decoder allocation failed: %s\n", gj_cuda_last_error());
            return GPUJPEG_ERROR;
        }
        ha.d_ss_scratch = d->d_ss_scratch;
        ha.ss_scratch_bytes = d->d_ss_scratch_size;
    }
    /* a cropped frame: K3 decodes the segments that hold the blocks K4 transforms (gj_crop_pick), unless the sub-sequence kernel
     * decodes the whole frame */
    if ( pick ) {
        if ( grow_pick(d, (size_t)g->seg_count) ) {
            GJ_ERR("Decoder allocation failed: %s\n", gj_cuda_last_error());
            return GPUJPEG_ERROR;
        }
        int n = 0;
        for ( int k = 0; k < g->scan_count; k++ )
            n += gj_crop_pick(g, k, d->k4.win.blk, d->h_pick + 2 * n);
        if ( n && gj_cuda_memcpy_h2d_async(d->d_pick, d->h_pick, (size_t)n * 8, d->stream) ) return GPUJPEG_ERROR;
        ha.d_pick = d->d_pick;
        ha.pick_count = n;
    }
    d->last_args = ha;
    d->last_ecs_begin = ecs_begin;
    d->last_list_cap = list_cap;
    memcpy(d->last_tq, st.comp_tq, sizeof d->last_tq);
    d->last_valid = 1;
    d->last_progressive = 0;
  for ( int pass = 0;; pass++ ) {
    if ( resync ) {
        if ( resync_segments(d, &st, first_rank, end_rank, scan_cbegin, &ha) ||
             gj_k3_choose(g, d->huffman_req, d->force_lanes, GJ_K3_RESYNC_TABLE, d->crop, &ha) < 0 )   /* (the same pick) */
            return GPUJPEG_ERROR;
        d->last_args = ha;
    }
    /* host output of a large frame leaves stripe by stripe (decode_striped): K4 per stripe and, where the Huffman decoder can
     * work on a part of the frame, K3 per stripe as well -- the segments the stripe's rows need, just before its K4 */
    const int to_host = output->type == GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER || output->type == GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER;
    const int striped = to_host && !stats && stripes_usable(d);
    if ( d->k3_parts < 0 ) {
        const char* v = getenv("GPUJPEG_B200_STRIPES_K3");
        d->k3_parts = !(v && v[0] == '0');
    }
    /* (part_seg_lo / part_seg_hi: the self-synchronising kernel on 4:4:4 frames with one scan per component, positions from
     * the marker list) */
    const int k3_striped = striped && d->k3_parts && ha.kernel == GJ_K3_SELF_SYNC && !resync && g->lay.simple && !g->lay.interleaved;
    /* a cropped frame leaves blocks undecoded: their extent 0 makes them read as zero (the rule of gj_internal.h) */
    if ( d->crop && gj_cuda_memset_async(d->d_cext, 0, g->coef_count / 64, d->stream) ) {
        GJ_ERR("Decoder extent clear failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    if ( !k3_striped && gj_launch_huffman_decode(&ha, d->stream) ) {
        GJ_ERR("Huffman decoder launch failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    if ( stats && d->timers_ok ) {
        gj_timer_stop(&d->t_huff, d->stream);
        gj_timer_start(&d->t_dct, d->stream);
    }

    if ( !d->coef_only && k4_and_output(d, output, &pi, st.comp_tq, striped, k3_striped ? &ha : NULL, stats) )
        return GPUJPEG_ERROR;
    if ( gj_cuda_memcpy_d2h_async(d->h_mk, d->d_mk, 16, d->stream) || gj_cuda_stream_sync(d->stream) ) {
        GJ_ERR("Decoder failed: %s\n", gj_cuda_last_error());
        return GPUJPEG_ERROR;
    }
    if ( d->h_mk[3] && by_table ) {
        /* a position of the stream's segment-info table does not lie behind the restart marker it should: forget the tables */
        GJ_VERBOSE(d->verbose, "Segment info of the stream does not match its restart markers; decoding by marker scan.\n");
        d->ignore_segment_info = 1;
        const int rc = gpujpeg_decoder_decode(d, image, image_size, output);
        d->ignore_segment_info = 0;
        return rc;
    }
    if ( d->h_mk[3] && !resync && pass == 0 ) {
        /* K3 met a restart marker with the wrong number: resynchronise [ref: src/gpujpeg_reader.c:1071-1105] and decode again */
        resync = 1;
        continue;
    }
    break;
  }
    d->used_subsequences = ha.kernel == GJ_K3_SUBSEQUENCE;
    output->metadata = &d->metadata;

    record_stats(d, output, &pi, stats, t_reader_ms, t_begin);
    return GPUJPEG_NOERR;
}

int gj_decoder_decode_coefficients(struct gpujpeg_decoder* d, const uint8_t* image, size_t image_size, gj_coef_window_fn window,
                                   void* ctx, struct gj_coef_frame* f)
{
    if ( !d || !image || !f ) return -1;
    struct gpujpeg_decoder_output output;
    gpujpeg_decoder_output_set_default(&output);
    d->coef_only = 1;
    d->coef_window = window;
    d->coef_window_ctx = ctx;
    const int rc = gpujpeg_decoder_decode(d, (uint8_t*)image, image_size, &output);
    d->coef_only = 0;
    d->coef_window = NULL;
    d->coef_window_ctx = NULL;
    d->last_valid = 0;   /* a resident re-run would take the raw coefficients for K4's */
    if ( rc ) return -1;
    const size_t com = gj_com_segments(image, image_size, NULL);
    if ( com > d->com_cap ) {
        free(d->com);
        d->com_cap = 0;
        if ( !(d->com = (uint8_t*)malloc(com)) ) return -1;
        d->com_cap = com;
    }
    memset(f, 0, sizeof *f);
    f->geo = &d->geo;
    f->d_coef = d->d_coef;
    f->d_cext = d->d_cext;
    f->progressive = d->last_progressive;
    f->color_space = d->param.color_space_internal;
    memcpy(f->qt, d->coef_qt, sizeof f->qt);
    memcpy(f->tq, d->coef_tq, sizeof f->tq);
    f->metadata = d->metadata;
    f->com_size = gj_com_segments(image, image_size, d->com);
    f->com = d->com;
    return 0;
}

int gpujpeg_decoder_get_stats(struct gpujpeg_decoder* decoder, struct gpujpeg_duration_stats* stats)
{
    if ( !decoder || !stats || !decoder->stats_valid ) return -1;
    *stats = decoder->stats;
    return 0;
}

/* [ref: src/gpujpeg_reader.c:1738-1872] */
int gpujpeg_decoder_get_image_info2(uint8_t* image, size_t image_size, struct gpujpeg_image_info* info, int verbose,
                                    unsigned flags)
{
    struct gj_stream st;
    if ( gj_reader_parse(image, image_size, &st, verbose) ) return -1;
    memset(info, 0, sizeof *info);
    gpujpeg_image_set_default_parameters(&info->param_image);
    gpujpeg_set_default_parameters(&info->param);
    info->param_image.width = st.width;
    info->param_image.height = st.height;
    info->param_image.color_space = st.color_space;
    /* the stream's native pixel format [ref: src/gpujpeg_reader.c:1507-1547, 1750] */
    info->param_image.pixel_format = st.comp_count == 1 ? GPUJPEG_U8 : st.comp_count == 4 ? GPUJPEG_4444_U8_P0123 : GPUJPEG_444_U8_P012;
    if ( st.comp_count == 3 && st.comp_hv[1] == 0x11 && st.comp_hv[2] == 0x11 ) {
        const int il = st.interleaved;
        if ( st.comp_hv[0] == 0x22 ) info->param_image.pixel_format = GPUJPEG_420_U8_P0P1P2;
        else if ( st.comp_hv[0] == 0x21 ) info->param_image.pixel_format = il ? GPUJPEG_422_U8_P1020 : GPUJPEG_422_U8_P0P1P2;
        else info->param_image.pixel_format = il ? GPUJPEG_444_U8_P012 : GPUJPEG_444_U8_P0P1P2;
    }
    info->param.comp_count = st.comp_count;
    info->param.restart_interval = st.restart_interval;
    info->param.interleaved = st.interleaved;
    info->param.color_space_internal = st.color_space;
    for ( int c = 0; c < st.comp_count; c++ ) {
        info->param.sampling_factor[c].horizontal = (uint8_t)(st.comp_hv[c] >> 4);
        info->param.sampling_factor[c].vertical = (uint8_t)(st.comp_hv[c] & 15);
    }
    info->header_type = st.header_type;
    info->metadata = st.metadata;
    info->comment = st.comment;
    info->segment_count = 0;
    if ( flags & GPUJPEG_COUNT_SEG_COUNT_REQ ) {
        int n = 0;
        for ( int s = 0; s < st.scan_count; s++ ) {
            n++;
            for ( size_t i = st.scan[s].begin; i + 1 < st.scan[s].end; i++ )
                if ( image[i] == 0xFF && image[i + 1] >= 0xD0 && image[i + 1] <= 0xD7 ) n++;
        }
        info->segment_count = n;
    }
    return 0;
}

int gpujpeg_decoder_get_image_info(uint8_t* image, size_t image_size, struct gpujpeg_image_parameters* param_image,
                                   struct gpujpeg_parameters* param, int* segment_count)
{
    struct gpujpeg_image_info info;
    if ( gpujpeg_decoder_get_image_info2(image, image_size, &info, param ? param->verbose : 0,
                                         segment_count ? GPUJPEG_COUNT_SEG_COUNT_REQ : 0) )
        return -1;
    if ( param_image ) *param_image = info.param_image;
    if ( param ) {
        const int verbose = param->verbose, perf = param->perf_stats;
        *param = info.param;
        param->verbose = verbose;
        param->perf_stats = perf;
    }
    if ( segment_count ) *segment_count = info.segment_count;
    return 0;
}

/* [ref: src/gpujpeg_decoder.c:485-531] */
int gpujpeg_decoder_set_option(struct gpujpeg_decoder* decoder, const char* opt, const char* val)
{
    if ( !decoder || !opt || !val ) return GPUJPEG_ERROR;
    if ( strcmp(opt, GPUJPEG_DEC_OPT_IDCT) == 0 ) {
        if ( strcmp(val, GPUJPEG_DEC_IDCT_VAL_INT) == 0 ) decoder->idct_flavour = 0;
        else if ( strcmp(val, GPUJPEG_DEC_IDCT_VAL_FLOAT_GPUREF) == 0 ) decoder->idct_flavour = 1;
        else {
            GJ_ERR("Unknown IDCT flavour: %s\n", val);
            return GPUJPEG_ERROR;
        }
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_HUFFMAN) == 0 ) {
        if ( strcmp(val, GPUJPEG_DEC_HUFFMAN_VAL_AUTO) == 0 ) decoder->huffman_req = GJ_K3_AUTO;
        else if ( strcmp(val, GPUJPEG_DEC_HUFFMAN_VAL_THREAD_PER_SEGMENT) == 0 ) decoder->huffman_req = GJ_K3_THREAD_PER_SEGMENT;
        else if ( strcmp(val, GPUJPEG_DEC_HUFFMAN_VAL_SUBSEQUENCE) == 0 ) decoder->huffman_req = GJ_K3_SUBSEQUENCE;
        else {
            GJ_ERR("Unknown Huffman decoder kernel: %s\n", val);
            return GPUJPEG_ERROR;
        }
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_HUFFMAN_LANES) == 0 ) {
        /* one number for every scan, or a comma-separated list by scan */
        int lanes[GJ_MAX_COMP] = {0, 0, 0, 0}, count = 0;
        const char* p = val;
        while ( *p && count < GJ_MAX_COMP ) {
            const int n = atoi(p);
            if ( n < 0 || n > 32 || (n & (n - 1)) ) {
                GJ_ERR("Lanes per restart segment must be 0 (automatic) or a power of two up to 32 (got %s).\n", val);
                return GPUJPEG_ERROR;
            }
            lanes[count++] = n;
            while ( *p && *p != ',' ) p++;
            if ( *p == ',' ) p++;
        }
        for ( int k = 0; k < GJ_MAX_COMP; k++ )
            decoder->force_lanes[k] = count == 1 ? lanes[0] : lanes[k];
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_FLIPPED_BOOL) == 0 ) {   /* [ref: src/gpujpeg_decoder.c:499-501] */
        const int b = gj_parse_bool(val, GPUJPEG_DEC_OPT_FLIPPED_BOOL);
        if ( b < 0 ) return GPUJPEG_ERROR;
        decoder->flipped = b;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_CHANNEL_REMAP) == 0 ) {   /* [ref: src/gpujpeg_decoder.c:502-504] */
        const unsigned m = gj_parse_channel_remap(val, GPUJPEG_DEC_OPT_CHANNEL_REMAP);
        if ( !m ) return GPUJPEG_ERROR;
        decoder->channel_remap = m;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_SCALE) == 0 ) {
        static const char* const vals[4] = {"1", "1/2", "1/4", "1/8"};
        for ( int i = 0; i < 4; i++ )
            if ( strcmp(val, vals[i]) == 0 ) {
                decoder->scale_req = 1 << i;
                return GPUJPEG_NOERR;
            }
        GJ_ERR("Unknown decoding scale: %s (1, 1/2, 1/4 or 1/8)\n", val);
        return GPUJPEG_ERROR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_CROP) == 0 ) {
        if ( strcmp(val, "none") == 0 ) {
            decoder->crop_req = 0;
            return GPUJPEG_NOERR;
        }
        int v[4];
        if ( gj_parse_crop(val, v) ) {
            GJ_ERR("Invalid crop: %s (WxH+X+Y with W, H >= 1, or none)\n", val);
            return GPUJPEG_ERROR;
        }
        decoder->crop_rw = v[0];
        decoder->crop_rh = v[1];
        decoder->crop_rx = v[2];
        decoder->crop_ry = v[3];
        decoder->crop_req = 1;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_ORIENTATION) == 0 ) {
        int mode, rot, flip;
        if ( gj_parse_orientation(val, &mode, &rot, &flip) ) {
            GJ_ERR("Invalid orientation: %s (none, auto, or 0, 90, 180 or 270 optionally followed by '-')\n", val);
            return GPUJPEG_ERROR;
        }
        decoder->orient_mode = mode;
        decoder->orient_rot = rot;
        decoder->orient_flip = flip;
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_PIXELS) == 0 ) {
        if ( strcmp(val, GPUJPEG_DEC_PIXELS_VAL_GPUJPEG) == 0 ) decoder->pixels_req = 0;
        else if ( strcmp(val, GPUJPEG_DEC_PIXELS_VAL_LIBJPEG) == 0 ) decoder->pixels_req = 1;
        else {
            GJ_ERR("Unknown output pixels: %s (gpujpeg or libjpeg)\n", val);
            return GPUJPEG_ERROR;
        }
        return GPUJPEG_NOERR;
    }
    if ( strcmp(opt, GPUJPEG_DEC_OPT_TGA_RLE_BOOL) == 0 || strcmp(opt, GPUJPEG_DEC_OPT_ALIGNMENT_BYTES_INT) == 0 ) {
        GJ_ERR("Decoder option %s is not implemented in this build.\n", opt);
        return GPUJPEG_ERROR;
    }
    GJ_ERR("Invalid decoder option: %s!\n", opt);
    return GPUJPEG_ERROR;
}

void gpujpeg_decoder_print_options(void)
{
    printf("\t" GPUJPEG_DEC_OPT_IDCT "=[" GPUJPEG_DEC_IDCT_VAL_INT "|" GPUJPEG_DEC_IDCT_VAL_FLOAT_GPUREF
           "] - inverse DCT flavour (default: int = gpujpeg_idct_cpu)\n");
    printf("\t" GPUJPEG_DEC_OPT_FLIPPED_BOOL "=[" GPUJPEG_VAL_FALSE "|" GPUJPEG_VAL_TRUE "] - flip the decoded image vertically\n");
    printf("\t" GPUJPEG_DEC_OPT_CHANNEL_REMAP "=XYZ[W] - output channel mapping (as the encoder option)\n");
    printf("\t" GPUJPEG_DEC_OPT_SCALE "=[1|1/2|1/4|1/8] - decode to ceil(W*scale) x ceil(H*scale) pixels with libjpeg's reduced inverse "
           "DCTs (default: 1)\n");
    printf("\t" GPUJPEG_DEC_OPT_CROP "=[WxH+X+Y|none] - decode only this rectangle of the (scaled) output image, Huffman-decoding only "
           "the restart segments it covers (default: none)\n");
    printf("\t" GPUJPEG_DEC_OPT_ORIENTATION "=[none|auto|<deg>[-]] - turn the output <deg> = 0, 90, 180 or 270 degrees clockwise, then "
           "mirror it horizontally with '-'; auto: as the stream's SPIFF or Exif orientation says (default: none)\n");
    printf("\t" GPUJPEG_DEC_OPT_PIXELS "=[" GPUJPEG_DEC_PIXELS_VAL_GPUJPEG "|" GPUJPEG_DEC_PIXELS_VAL_LIBJPEG "] - the pixels of "
           "gpujpeg's arithmetic, or those libjpeg-turbo's jpeg_read_scanlines returns with its default parameters: ISLOW IDCT, fancy "
           "upsampling, its YCbCr -> RGB (default: gpujpeg)\n");
}

GPUJPEG_API int gpujpegx_decoder_used_segment_info(const struct gpujpeg_decoder* d)
{
    return d && d->last_valid ? d->used_segment_info : -1;
}

GPUJPEG_API int gpujpegx_decoder_used_subsequences(const struct gpujpeg_decoder* d)
{
    return d && d->last_valid ? d->used_subsequences : -1;
}

GPUJPEG_API int gpujpegx_decoder_subsequence_rounds(struct gpujpeg_decoder* d)
{
    if ( !d || !d->last_valid || !d->used_subsequences ) return -1;
    return gj_subseq_rounds(d->d_ss_scratch, d->stream);
}

/* ---- extension: re-run the GPU stages of the last decoded frame on the JPEG bytes already on the device ----
 * stage_mask bit 2 = K0 (marker list + clean stream from the file bytes), bit 0 = K3 (Huffman decode), bit 1 = K4
 * (dequant+IDCT+colour).  No copies, no sync; what the host derived from K0's report for this file (scan extents,
 * ranks) is reused, so 7 = every GPU stage of a decode that starts from the JPEG bytes. */
GPUJPEG_API int gpujpegx_decoder_run_resident(struct gpujpeg_decoder* d, uint8_t* d_out, int stage_mask)
{
    if ( !d || !d->last_valid ) return -1;
    if ( d->last_progressive ) {
        /* bit 2 K0, bit 0 the zeroing, every scan and the dequantisation, bit 1 K4 */
        static const int comp_tq[GJ_MAX_COMP] = {0, 1, 2, 3};
        if ( (stage_mask & 4) &&
             gj_launch_marker_scan(d->d_file, d->last_ecs_begin, d->last_args.file_size, d->d_cta, d->d_list_pos, d->d_list_code,
                                   d->d_list_cpos, d->last_list_cap, d->d_clean, d->d_mk, d->d_mk + 8, GJ_MK_OTHER_CAP, d->stream) )
            return -1;
        if ( (stage_mask & 1) && gj_launch_progressive_decode(&d->last_prog, d->stream) ) return -1;
        if ( (stage_mask & 2) && launch_k4(d, comp_tq, d_out ? d_out : d->d_raw, 0, d->k4.mcu_rows) ) return -1;
        return 0;
    }
    if ( (stage_mask & 4) && !d->used_segment_info &&
         gj_launch_marker_scan(d->d_file, d->last_ecs_begin, d->last_args.file_size, d->d_cta, d->d_list_pos, d->d_list_code,
                               d->d_list_cpos, d->last_list_cap, d->d_clean, d->d_mk, d->d_mk + 8, GJ_MK_OTHER_CAP, d->stream) )
        return -1;
    if ( (stage_mask & 1) && d->crop && gj_cuda_memset_async(d->d_cext, 0, d->geo.coef_count / 64, d->stream) ) return -1;
    if ( (stage_mask & 1) && gj_launch_huffman_decode(&d->last_args, d->stream) ) return -1;
    if ( (stage_mask & 2) && launch_k4(d, d->last_tq, d_out ? d_out : d->d_raw, 0, d->k4.mcu_rows) ) return -1;
    return 0;
}

/* ---- extension used by the parity tests: coefficients of the last decoded frame, natural order ---- */
/* Returns 0 when the values are raw quantised coefficients, 1 when they are already multiplied by the
 * quantiser and wrapped to int16 (integer IDCT flavour: the multiply is fused into the Huffman decoder). */
GPUJPEG_API int gpujpegx_decoder_get_coefficients(struct gpujpeg_decoder* d, int16_t* out, size_t count)
{
    if ( !d || !d->initialised || !d->last_valid || count != d->geo.coef_count ) return -1;
    if ( gj_coef_to_host_natural(d->d_coef, d->d_cext, NULL, count, out, d->stream) ) return -1;
    return d->k4.dequantize;
}
