/*
 * gj_transcoder.c -- lossless JPEG-to-JPEG rewrite (gpujpegx_transcode).  Host C.
 *
 * One decoder and one encoder on the transcoder's stream, so that stream order serialises them:
 *
 *     decoder up to its raw quantised coefficients (K0, K3 or the progressive scans; gj_decoder_decode_coefficients)
 *       -> host plan: trim, output size and sampling, block maps (gj_transcode_plan); with tran_opt_crop the plan is cut to the
 *          rectangle (gj_transcode_crop) inside the decode, once the frame's geometry is known, so that the decoder Huffman-decodes
 *          only the restart segments that hold the blocks the cut plan reads (gj_transcode_window)
 *       -> k_coef_transform: the decoder's blocks -> the encoder's coefficients and non-zero masks, turned / mirrored, with
 *          the baseline range check (one synchronisation: a frame out of range is refused before anything is written)
 *       -> the encoder's work after K1 (fitted tables, K2, copies; gj_encoder_finish)
 *
 * The output is one baseline frame with the source's quantisation tables and COM segments, the source's interleaving (a
 * progressive source of several components becomes one interleaved scan), the restart interval and Huffman tables asked for.
 */
#include <stdlib.h>
#include <string.h>

#include "gj_internal.h"
#include "../../include/gpujpegx.h"

struct gpujpegx_transcoder {
    gj_stream_t stream;
    struct gpujpeg_decoder* dec;
    struct gpujpeg_encoder* enc;
    int mode, rot, flip;   /* tran_opt_transform as gj_parse_orientation gives it: 0 none, 1 auto, 2 rot / flip */
    int perfect;
    int restart;           /* RESTART_AUTO or the interval */
    int crop, crop_rect[4];   /* tran_opt_crop: set, and x, y, w, h of the transformed image */
    uint32_t* d_range;
    uint32_t* h_range;     /* pinned */
};

GPUJPEG_API struct gpujpegx_transcoder* gpujpegx_transcoder_create(cudaStream_t stream)
{
    struct gpujpegx_transcoder* t = (struct gpujpegx_transcoder*)calloc(1, sizeof *t);
    if ( !t ) return NULL;
    t->stream = (gj_stream_t)stream;
    t->restart = RESTART_AUTO;
    t->dec = gpujpeg_decoder_create(stream);
    t->enc = t->dec ? gpujpeg_encoder_create(stream) : NULL;
    if ( !t->enc || gpujpeg_encoder_set_option(t->enc, GPUJPEG_ENC_OPT_OUT, GPUJPEG_ENC_OUT_VAL_PINNED) ||
         gj_cuda_malloc((void**)&t->d_range, 4) || gj_cuda_malloc_host((void**)&t->h_range, 4) ) {
        GJ_ERR("Transcoder allocation failed: %s\n", gj_cuda_last_error());
        gpujpegx_transcoder_destroy(t);
        return NULL;
    }
    return t;
}

GPUJPEG_API void gpujpegx_transcoder_destroy(struct gpujpegx_transcoder* t)
{
    if ( !t ) return;
    gpujpeg_encoder_destroy(t->enc);
    gpujpeg_decoder_destroy(t->dec);
    gj_cuda_free(t->d_range);
    if ( t->h_range ) gj_cuda_free_host(t->h_range);
    free(t);
}

GPUJPEG_API int gpujpegx_transcoder_set_option(struct gpujpegx_transcoder* t, const char* opt, const char* val)
{
    if ( !t || !opt || !val ) return -1;
    if ( strcmp(opt, GPUJPEGX_TRAN_OPT_TRANSFORM) == 0 ) {
        int mode, rot, flip;
        if ( gj_parse_orientation(val, &mode, &rot, &flip) ) {
            GJ_ERR("Wrong " GPUJPEGX_TRAN_OPT_TRANSFORM " value: %s (none, auto or <deg>[-] with deg 0, 90, 180 or 270)\n", val);
            return -1;
        }
        t->mode = mode;
        t->rot = rot;
        t->flip = flip;
        return 0;
    }
    if ( strcmp(opt, GPUJPEGX_TRAN_OPT_PERFECT) == 0 ) {
        const int b = gj_parse_bool(val, GPUJPEGX_TRAN_OPT_PERFECT);
        if ( b < 0 ) return -1;
        t->perfect = b;
        return 0;
    }
    if ( strcmp(opt, GPUJPEGX_TRAN_OPT_RESTART) == 0 ) {
        if ( strcmp(val, "auto") == 0 ) {
            t->restart = RESTART_AUTO;
            return 0;
        }
        char* end = NULL;
        const long n = strtol(val, &end, 10);
        if ( !val[0] || *end != '\0' || n < 0 || n > 65535 ) {
            GJ_ERR("Wrong " GPUJPEGX_TRAN_OPT_RESTART " value: %s (auto or 0 to 65535)\n", val);
            return -1;
        }
        t->restart = (int)n;
        return 0;
    }
    if ( strcmp(opt, GPUJPEGX_TRAN_OPT_CROP) == 0 ) {
        if ( strcmp(val, "none") == 0 ) {
            t->crop = 0;
            return 0;
        }
        int v[4];
        if ( gj_parse_crop(val, v) ) {
            GJ_ERR("Wrong " GPUJPEGX_TRAN_OPT_CROP " value: %s (WxH+X+Y with W, H >= 1, or none)\n", val);
            return -1;
        }
        t->crop = 1;
        t->crop_rect[0] = v[2];
        t->crop_rect[1] = v[3];
        t->crop_rect[2] = v[0];
        t->crop_rect[3] = v[1];
        return 0;
    }
    if ( strcmp(opt, GPUJPEGX_TRAN_OPT_HUFFMAN) == 0 ) return gpujpeg_encoder_set_option(t->enc, GPUJPEG_ENC_OPT_HUFFMAN, val);
    GJ_ERR("Invalid transcoder option: %s!\n", opt);
    return -1;
}

/* a frame's orientation, output interleaving and plan (cut to tran_opt_crop's rectangle) */
struct frame_plan {
    const struct gpujpegx_transcoder* t;
    int transformed, out_il;
    struct gj_transcode_plan plan;
};

static int make_plan(struct frame_plan* fp, const struct gj_geometry* g, int progressive, const struct gpujpeg_image_metadata* md)
{
    const struct gpujpegx_transcoder* t = fp->t;
    const int n = g->comp_count;
    int rot = t->rot, flip = t->flip;
    if ( t->mode == 1 ) {
        const int set = md->vals[GPUJPEG_METADATA_ORIENTATION].set;
        rot = set ? (int)md->vals[GPUJPEG_METADATA_ORIENTATION].orient.rotation : 0;
        flip = set ? (int)md->vals[GPUJPEG_METADATA_ORIENTATION].orient.flip : 0;
    }
    fp->transformed = t->mode != 0 && (rot != 0 || flip != 0);
    if ( !fp->transformed ) rot = flip = 0;

    /* the output keeps the source's interleaving; a progressive frame of several components becomes one interleaved scan */
    fp->out_il = progressive ? n > 1 : g->interleaved;
    int hs[GJ_MAX_COMP], vs[GJ_MAX_COMP];
    for ( int c = 0; c < n; c++ ) {
        hs[c] = g->comp[c].hs;
        vs[c] = g->comp[c].vs;
    }
    char why[GJ_WHY_BYTES];
    if ( gj_transcode_plan(g->width, g->height, n, hs, vs, g->interleaved, fp->out_il, rot, flip, t->perfect, &fp->plan, why) ) {
        GJ_ERR("Cannot transcode: %s.\n", why);
        return -1;
    }
    if ( t->crop ) {
        const struct gj_transcode_plan full = fp->plan;
        if ( gj_transcode_crop(&full, g->width, g->height, n, fp->out_il, t->crop_rect, &fp->plan, why) ) {
            GJ_ERR("Cannot transcode: %s.\n", why);
            return -1;
        }
    }
    return 0;
}

/* the decoder's window (gj_coef_window_fn) for tran_opt_crop: the plan, and the source blocks it reads */
static int crop_window(void* ctx, const struct gj_geometry* g, int progressive, const struct gpujpeg_image_metadata* md,
                       struct gj_blk_rect win[GJ_MAX_COMP])
{
    struct frame_plan* fp = (struct frame_plan*)ctx;
    if ( make_plan(fp, g, progressive, md) ) return -1;
    gj_transcode_window(&fp->plan, g->comp_count, win);
    for ( int c = 0; c < g->comp_count; c++ )   /* a window of every block decodes as a frame without one */
        if ( win[c].bx0 > 0 || win[c].by0 > 0 || win[c].bx1 < g->comp[c].bcx || win[c].by1 < g->comp[c].bcy ) return 1;
    return 0;
}

GPUJPEG_API int gpujpegx_transcode(struct gpujpegx_transcoder* t, const uint8_t* jpeg, size_t size, uint8_t** out, size_t* out_size)
{
    if ( !t || !jpeg || !out || !out_size ) return -1;
    struct frame_plan fp;
    memset(&fp, 0, sizeof fp);
    fp.t = t;
    struct gj_coef_frame f;
    if ( gj_decoder_decode_coefficients(t->dec, jpeg, size, t->crop ? crop_window : NULL, &fp, &f) ) return -1;
    const struct gj_geometry* g = f.geo;
    const int n = g->comp_count;
    if ( f.color_space != GPUJPEG_YCBCR_BT601_256LVLS &&
         !(n >= 3 && (f.color_space == GPUJPEG_RGB || f.color_space == GPUJPEG_YCBCR_BT601 || f.color_space == GPUJPEG_YCBCR_BT709)) ) {
        GJ_ERR("Transcoding a %d-component %s stream is not supported.\n", n, gpujpeg_color_space_get_name(f.color_space));
        return -1;
    }
    /* (a cropped frame's plan was made inside the decode, on the metadata its window saw) */
    if ( !t->crop && make_plan(&fp, g, f.progressive, &f.metadata) ) return -1;
    const struct gj_transcode_plan plan = fp.plan;
    const int transformed = fp.transformed, out_il = fp.out_il;

    /* quantisation tables: the source's, transposed with the blocks; a table id that two components use with different tables
     * (a progressive frame may redefine one between the components' first scans) moves to a free id */
    uint8_t q[GJ_MAX_COMP][64], tq[GJ_MAX_COMP];
    memset(q, 0, sizeof q);
    memset(tq, 0, sizeof tq);
    unsigned used = 0;
    for ( int c = 0; c < n; c++ ) {
        for ( int k = 0; k < 64; k++ ) {
            const int nat = gj_zigzag_to_natural[k];
            const int s = plan.transpose ? gj_natural_to_zigzag[(nat & 7) * 8 + (nat >> 3)] : k;
            if ( !f.qt[c][s] ) {
                GJ_ERR("Cannot transcode: component %d has no valid quantisation table.\n", c);
                return -1;
            }
            q[c][k] = f.qt[c][s];
        }
        int id = f.tq[c] & 3;
        for ( int e = 0; e < c; e++ )
            if ( tq[e] == id && memcmp(q[e], q[c], 64) != 0 ) {
                id = -1;
                break;
            }
        if ( id < 0 ) {
            for ( id = 0; id < 4 && (used & (1u << id)); id++ ) {}
            if ( id == 4 ) {
                GJ_ERR("Cannot transcode: more than four distinct quantisation tables.\n");
                return -1;
            }
        }
        used |= 1u << id;
        tq[c] = (uint8_t)id;
    }

    struct gpujpeg_parameters p;
    gpujpeg_set_default_parameters(&p);
    p.comp_count = n;
    p.interleaved = out_il;
    p.restart_interval = t->restart;
    p.segment_info = 0;
    p.color_space_internal = f.color_space;
    memset(p.sampling_factor, 0, sizeof p.sampling_factor);
    for ( int c = 0; c < n; c++ ) {
        p.sampling_factor[c].horizontal = (uint8_t)plan.hs[c];
        p.sampling_factor[c].vertical = (uint8_t)plan.vs[c];
    }
    struct gpujpeg_image_metadata md = f.metadata;
    if ( transformed ) memset(&md.vals[GPUJPEG_METADATA_ORIENTATION], 0, sizeof md.vals[0]);   /* the pixels are upright now */
    int16_t* d_coef;
    uint64_t* d_nzmask;
    const struct gj_geometry* go;
    if ( gj_encoder_setup_coefficients(t->enc, &p, plan.width, plan.height, (const uint8_t(*)[64])q, tq, f.com, f.com_size, &md, &d_coef,
                                       &d_nzmask, &go) )
        return -1;

    struct gj_coef_transform_args a;
    memset(&a, 0, sizeof a);
    a.d_src = f.d_coef;
    a.d_cext = f.d_cext;
    a.d_dst = d_coef;
    a.d_nzmask = d_nzmask;
    a.comp_count = n;
    a.dst_blocks = (int)(go->coef_count / 64);
    a.transpose = plan.transpose;
    a.neg_x = plan.neg_x;
    a.neg_y = plan.neg_y;
    a.d_range = t->d_range;
    for ( int c = 0; c < n; c++ ) {
        a.src_blk_off[c] = g->comp[c].blk_off;
        a.dst_blk_off[c] = go->comp[c].blk_off;
        a.blk[c] = plan.blk[c];
        if ( plan.blk[c].out_bcx != go->comp[c].bcx || plan.blk[c].out_bcy != go->comp[c].bcy ) {
            GJ_ERR("Transcoder plan and encoder geometry disagree (component %d).\n", c);
            return -1;
        }
    }
    if ( gj_cuda_memset_async(t->d_range, 0, 4, t->stream) || gj_launch_coef_transform(&a, t->stream) ||
         gj_cuda_memcpy_d2h_async(t->h_range, t->d_range, 4, t->stream) || gj_cuda_stream_sync(t->stream) ) {
        GJ_ERR("Coefficient transform failed: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( *t->h_range ) {
        GJ_ERR("Cannot transcode: a coefficient lies outside the 8-bit baseline range (DC -1024..1023, AC -1023..1023).\n");
        return -1;
    }
    return gj_encoder_finish(t->enc, out, out_size);
}
