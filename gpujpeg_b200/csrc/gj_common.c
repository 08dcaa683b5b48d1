/*
 * gj_common.c -- the part of the libgpujpeg API that is not on the data path: version, defaults,
 * name tables, device selection, image-size arithmetic, raw/.tst image helpers, OpenGL stubs.
 * Behaviour follows src/gpujpeg_common.c (cited per function); file formats other than raw dumps
 * and the procedural ".tst" test images are outside the hot path and rejected loudly.
 */
#include <assert.h>
#include <errno.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <sys/time.h>

#include "gj_internal.h"

/* ---- version / time [ref: src/gpujpeg_common.c:75-104] ---- */
int gpujpeg_version(void) { return GPUJPEG_VERSION_INT; }

const char* gpujpeg_version_to_string(int version)
{
    static __thread char buf[32];
    snprintf(buf, sizeof buf, "%d.%d.%d", version >> 16, (version >> 8) & 0xFF, version & 0xFF);
    return buf;
}

double gpujpeg_get_time(void)
{
    struct timeval tv;
    gettimeofday(&tv, 0);
    return (double)tv.tv_sec + (double)tv.tv_usec * 0.000001;
}

/* ---- devices [ref: src/gpujpeg_common.c:154-288] ---- */
struct gpujpeg_devices_info gpujpeg_get_devices_info(void)
{
    struct gpujpeg_devices_info info;
    memset(&info, 0, sizeof info);
    int n = gj_cuda_device_count();
    if ( n < 0 ) {
        GJ_ERR("Cannot get number of CUDA devices: %s\n", gj_cuda_last_error());
        return info;
    }
    if ( n > GPUJPEG_MAX_DEVICE_COUNT ) {
        GJ_WARN("There are available more CUDA devices (%d) than maximum count (%d).\n", n, GPUJPEG_MAX_DEVICE_COUNT);
        n = GPUJPEG_MAX_DEVICE_COUNT;
    }
    info.device_count = n;
    for ( int i = 0; i < n; i++ )
        gj_cuda_device_props(i, &info.device[i]);
    return info;
}

int gpujpeg_print_devices_info(void)
{
    struct gpujpeg_devices_info info = gpujpeg_get_devices_info();
    if ( info.device_count == 0 ) {
        printf("There is no device supporting CUDA.\n");
        return -1;
    }
    printf("There %s %d device%s supporting CUDA:\n", info.device_count == 1 ? "is" : "are", info.device_count,
           info.device_count == 1 ? "" : "s");
    for ( int i = 0; i < info.device_count; i++ ) {
        const struct gpujpeg_device_info* d = &info.device[i];
        printf("\nDevice #%d: \"%s\"\n", d->id, d->name);
        printf("  Compute capability: %d.%d\n", d->cc_major, d->cc_minor);
        printf("  Total amount of global memory: %zu KiB\n", d->global_memory / 1024);
        printf("  Total amount of constant memory: %zu KiB\n", d->constant_memory / 1024);
        printf("  Total amount of shared memory per block: %zu KiB\n", d->shared_memory / 1024);
        printf("  Total number of registers available per block: %d\n", d->register_count);
        printf("  Multiprocessors: %d\n", d->multiprocessor_count);
    }
    return 0;
}

int gpujpeg_init_device(int device_id, int flags)
{
    const int n = gj_cuda_device_count();
    if ( n < 0 ) {
        GJ_ERR("Cannot get number of CUDA devices: %s\n", gj_cuda_last_error());
        return -1;
    }
    if ( n == 0 ) {
        GJ_ERR("No CUDA enabled device\n");
        return -1;
    }
    if ( device_id < 0 || device_id >= n ) {
        GJ_ERR("Selected device %d is out of bound. Devices on your system are in range %d - %d\n", device_id, 0, n - 1);
        return -1;
    }
    struct gpujpeg_device_info d;
    if ( gj_cuda_device_props(device_id, &d) ) {
        GJ_ERR("Can't get CUDA device properties!\n");
        return -1;
    }
    if ( d.cc_major != 9 || d.cc_minor != 0 ) {
        GJ_ERR("Device %d (%s, c.c. %d.%d) is not a c.c. 9.0 Hopper GPU: this build carries sm_90a code only.\n", device_id,
               d.name, d.cc_major, d.cc_minor);
        return -1;
    }
    if ( flags & GPUJPEG_INIT_DEV_VERBOSE )
        fprintf(stderr, "Using Device #%d:       %s (c.c. %d.%d)\n", device_id, d.name, d.cc_major, d.cc_minor);
    if ( gj_cuda_set_device(device_id) ) {
        GJ_ERR("Set CUDA device: %s\n", gj_cuda_last_error());
        return -1;
    }
    /* same readiness probe as the reference: a 1-byte allocation + copy */
    void* p = NULL;
    uint8_t one = 8;
    if ( gj_cuda_malloc(&p, 1) || gj_cuda_memcpy_h2d_async(p, &one, 1, NULL) || gj_cuda_stream_sync(NULL) ) {
        GJ_ERR("Failed to initialize CUDA device: %s\n", gj_cuda_last_error());
        gj_cuda_free(p);
        return -1;
    }
    gj_cuda_free(p);
    return 0;
}

void gpujpeg_set_device(int index) { gj_cuda_set_device(index); }
void gpujpeg_device_reset(void) { gj_cuda_device_reset(); }

/* ---- parameters [ref: src/gpujpeg_common.c:290-378] ---- */
void gpujpeg_set_default_parameters(struct gpujpeg_parameters* param)
{
    memset(param, 0, sizeof *param);
    param->verbose = GPUJPEG_LL_INFO;
    param->quality = 75;
    param->restart_interval = 8;
    for ( int c = 0; c < GPUJPEG_MAX_COMPONENT_COUNT; c++ ) {
        param->sampling_factor[c].horizontal = 1;
        param->sampling_factor[c].vertical = 1;
    }
    param->color_space_internal = GPUJPEG_YCBCR_BT601_256LVLS;
}
struct gpujpeg_parameters gpujpeg_default_parameters(void)
{
    struct gpujpeg_parameters p;
    gpujpeg_set_default_parameters(&p);
    return p;
}
void gpujpeg_image_set_default_parameters(struct gpujpeg_image_parameters* param)
{
    param->width = 0;
    param->height = 0;
    param->color_space = GPUJPEG_RGB;
    param->pixel_format = GPUJPEG_444_U8_P012;
    param->width_padding = 0;
}
struct gpujpeg_image_parameters gpujpeg_default_image_parameters(void)
{
    struct gpujpeg_image_parameters p;
    gpujpeg_image_set_default_parameters(&p);
    return p;
}

/* [ref: src/gpujpeg_common.c:309-346] packed h/v nibbles, component 1 first */
void gpujpeg_parameters_chroma_subsampling(struct gpujpeg_parameters* param, gpujpeg_sampling_factor_t subsampling)
{
    param->comp_count = 0;
    for ( int c = 0; c < GPUJPEG_MAX_COMPONENT_COUNT; c++ ) {
        const int h = (subsampling >> (28 - 8 * c)) & 0xF, v = (subsampling >> (24 - 8 * c)) & 0xF;
        param->sampling_factor[c].horizontal = (uint8_t)h;
        param->sampling_factor[c].vertical = (uint8_t)v;
        if ( h != 0 && v != 0 ) param->comp_count = c + 1;
    }
}

static gpujpeg_sampling_factor_t pack_sampling(int comp_count, const struct gpujpeg_component_sampling_factor* f)
{
    gpujpeg_sampling_factor_t r = 0;
    for ( int c = 0; c < comp_count && c < 4; c++ )
        r |= (gpujpeg_sampling_factor_t)f[c].horizontal << (28 - 8 * c) | (gpujpeg_sampling_factor_t)f[c].vertical << (24 - 8 * c);
    return r;
}

/* [ref: src/gpujpeg_common.c:1905-1950] J:a:b naming (the strings are pinned by test/unit/run_tests.c:17-36) */
const char* gpujpeg_subsampling_get_name(int comp_count, const struct gpujpeg_component_sampling_factor* f)
{
    static __thread char buf[128];
    if ( comp_count == 1 ) return strcpy(buf, "4:0:0");
    const int J = 4;
    if ( comp_count == 2 && f[0].vertical == f[1].vertical ) {
        snprintf(buf, sizeof buf, "4:0:0:%d", J / f[0].horizontal * f[1].horizontal);
        return buf;
    }
    if ( f[1].horizontal == f[2].horizontal && f[1].vertical == f[2].horizontal &&
         (comp_count == 3 || (comp_count == 4 && f[0].vertical == f[3].vertical)) ) {
        const int a = J / f[0].horizontal * f[1].horizontal;
        const int vert_change = 2 / f[0].vertical * f[1].vertical == 2;
        snprintf(buf, sizeof buf, "%d:%d:%d", J, a, a * vert_change);
        if ( comp_count == 4 )
            snprintf(buf + strlen(buf), sizeof buf - strlen(buf), ":%d", J / f[0].horizontal * f[3].horizontal);
        return buf;
    }
    if ( pack_sampling(comp_count, f) == GPUJPEG_SUBSAMPLING_442 ) return strcpy(buf, "4:4:2");
    if ( pack_sampling(comp_count, f) == GPUJPEG_SUBSAMPLING_421 ) return strcpy(buf, "4:2:1");
    buf[0] = 0;
    for ( int i = 0; i < comp_count; i++ )
        snprintf(buf + strlen(buf), sizeof buf - strlen(buf), "%s%d-%d", i ? ":" : "", f[i].horizontal, f[i].vertical);
    return buf;
}

/* [ref: src/gpujpeg_common.c:1952-2005] */
gpujpeg_sampling_factor_t gpujpeg_subsampling_from_name(const char* subsampling)
{
    int J = 0, a = 0, b = 0, alpha = 0;
    int n = sscanf(subsampling, "%d:%d:%d:%d", &J, &a, &b, &alpha);
    if ( n == 1 && (J / 1000 == 4 || J / 100 == 4) ) { /* "422" / "4444" without colons */
        if ( J / 1000 == 4 ) {
            n = 4;
            alpha = J % 10;
            J /= 10;
        }
        else {
            n = 3;
        }
        J -= 400;
        a = J / 10;
        b = J % 10;
        J = 4;
    }
    if ( n < 3 || J != 4 || (alpha != 4 && alpha != 0) ) return GPUJPEG_SUBSAMPLING_UNKNOWN;
    if ( a != b && b != 0 ) {
        if ( a == 4 && b == 2 && alpha == 0 ) return GPUJPEG_SUBSAMPLING_442;
        if ( a == 2 && b == 1 && alpha == 0 ) return GPUJPEG_SUBSAMPLING_421;
        return GPUJPEG_SUBSAMPLING_UNKNOWN;
    }
    if ( a == 0 && b == 0 && alpha == 0 ) return GPUJPEG_SUBSAMPLING_400;
    if ( a == 0 ) return GPUJPEG_SUBSAMPLING_UNKNOWN;
    struct gpujpeg_component_sampling_factor f[4];
    memset(f, 0, sizeof f);
    f[0].horizontal = (uint8_t)(4 / a);
    f[0].vertical = a == b ? 1 : 2;
    f[1].horizontal = f[2].horizontal = f[1].vertical = f[2].vertical = 1;
    if ( alpha == 0 ) return pack_sampling(3, f);
    f[3] = f[0];
    return pack_sampling(4, f);
}

/* ---- name tables [ref: src/gpujpeg_common.c:125-152, 2007-2135, 2340-2390] ---- */
static const struct {
    enum gpujpeg_pixel_format fmt;
    int planar, comps, bpp;
    const char* name;
} k_pixfmt[] = {
    {GPUJPEG_PIXFMT_STD, 0, 0, 0, "(file standard)"},   {GPUJPEG_PIXFMT_NO_ALPHA, 0, 0, 0, "(without alpha)"},
    {GPUJPEG_PIXFMT_AUTODETECT, 0, 0, 0, "(autodetect)"}, {GPUJPEG_PIXFMT_NONE, 0, 0, 0, "(unknown)"},
    {GPUJPEG_U8, 0, 1, 1, "u8"},                          {GPUJPEG_444_U8_P012, 0, 3, 3, "444-u8-p012"},
    {GPUJPEG_444_U8_P0P1P2, 1, 3, 0, "444-u8-p0p1p2"},    {GPUJPEG_422_U8_P1020, 0, 3, 2, "422-u8-p1020"},
    {GPUJPEG_422_U8_P0P1P2, 1, 3, 0, "422-u8-p0p1p2"},    {GPUJPEG_420_U8_P0P1P2, 1, 3, 0, "420-u8-p0p1p2"},
    {GPUJPEG_4444_U8_P0123, 0, 4, 4, "4444-u8-p0123"},
};
#define N_PIXFMT ((int)(sizeof k_pixfmt / sizeof k_pixfmt[0]))

const char* gpujpeg_color_space_get_name(enum gpujpeg_color_space cs)
{
    switch ( (int)cs ) {
        case GPUJPEG_NONE: return "None";
        case GPUJPEG_RGB: return "RGB";
        case GPUJPEG_YUV: return "YUV";
        case GPUJPEG_YCBCR_BT601: return "YCbCr BT.601 (limtted range)";
        case GPUJPEG_YCBCR_BT601_256LVLS: return "YCbCr BT.601 256 Levels (YCbCr JPEG)";
        case GPUJPEG_YCBCR_BT709: return "YCbCr BT.709 (limited range)";
        default: break;
    }
    return cs == GPUJPEG_CS_DEFAULT ? "(default CS)" : "Unknown";
}

void gpujpeg_print_pixel_formats(void)
{
    fprintf(stderr, "                          u8 (grayscale)          420-u8-p0p1p2 (planar 4:2:0)\n"
                    "                          422-u8-p1020 (eg. UYVY) 422-u8-p0p1p2 (planar 4:2:2)\n"
                    "                          444-u8-p012 (eg. RGB)   444-u8-p0p1p2 (planar 4:4:4)\n"
                    "                          4444-u8-p0123 (RGBA)\n");
}

enum gpujpeg_pixel_format gpujpeg_pixel_format_by_name(const char* name)
{
    for ( int i = 0; i < N_PIXFMT; i++ )
        if ( strcmp(k_pixfmt[i].name, name) == 0 ) return k_pixfmt[i].fmt;
    if ( strcmp(name, "help") == 0 ) gpujpeg_print_pixel_formats();
    return GPUJPEG_PIXFMT_NONE;
}
int gpujpeg_pixel_format_get_comp_count(enum gpujpeg_pixel_format f)
{
    for ( int i = 0; i < N_PIXFMT; i++ )
        if ( k_pixfmt[i].fmt == f ) return k_pixfmt[i].comps;
    return 0;
}
const char* gpujpeg_pixel_format_get_name(enum gpujpeg_pixel_format f)
{
    for ( int i = 0; i < N_PIXFMT; i++ )
        if ( k_pixfmt[i].fmt == f ) return k_pixfmt[i].name;
    return NULL;
}
int gpujpeg_pixel_format_is_planar(enum gpujpeg_pixel_format f)
{
    for ( int i = 0; i < N_PIXFMT; i++ )
        if ( k_pixfmt[i].fmt == f ) return k_pixfmt[i].planar;
    return 0;
}
static int pixfmt_bpp(enum gpujpeg_pixel_format f)
{
    for ( int i = 0; i < N_PIXFMT; i++ )
        if ( k_pixfmt[i].fmt == f ) return k_pixfmt[i].bpp;
    return 0;
}

enum gpujpeg_color_space gpujpeg_color_space_by_name(const char* name)
{
    if ( strcmp(name, "rgb") == 0 ) return GPUJPEG_RGB;
    if ( strcmp(name, "yuv") == 0 ) return GPUJPEG_YUV;
    if ( strcmp(name, "ycbcr") == 0 ) return GPUJPEG_YCBCR;
    if ( strcmp(name, "ycbcr-jpeg") == 0 ) return GPUJPEG_YCBCR_BT601_256LVLS;
    if ( strcmp(name, "ycbcr-bt601") == 0 ) return GPUJPEG_YCBCR_BT601;
    if ( strcmp(name, "ycbcr-bt709") == 0 ) return GPUJPEG_YCBCR_BT709;
    if ( strcmp(name, "help") == 0 )
        fprintf(stderr, "Available color spaces:\n- rgb\n- yuv (deprecated)\n- ycbcr       - same as ycbcr-bt709\n"
                        "- ycbcr-jpeg  - BT.601 full range\n- ycbcr-bt601 - limitted range\n- ycbcr-bt709 - limitted range\n");
    return GPUJPEG_NONE;
}

enum gpujpeg_header_type gpujpeg_header_type_by_name(const char* name)
{
    if ( strcasecmp(name, GPUJPEG_ENC_HDR_VAL_JFIF) == 0 ) return GPUJPEG_HEADER_JFIF;
    if ( strcasecmp(name, GPUJPEG_ENC_HDR_VAL_EXIF) == 0 ) return GPUJPEG_HEADER_EXIF;
    if ( strcasecmp(name, GPUJPEG_ENC_HDR_VAL_ADOBE) == 0 ) return GPUJPEG_HEADER_ADOBE;
    if ( strcasecmp(name, GPUJPEG_ENC_HDR_VAL_SPIFF) == 0 ) return GPUJPEG_HEADER_SPIFF;
    return GPUJPEG_HEADER_DEFAULT;
}
const char* gpujpeg_header_type_get_name(enum gpujpeg_header_type t)
{
    switch ( t ) {
        case GPUJPEG_HEADER_DEFAULT: return "undefined";
        case GPUJPEG_HEADER_JFIF: return GPUJPEG_ENC_HDR_VAL_JFIF;
        case GPUJPEG_HEADER_SPIFF: return GPUJPEG_ENC_HDR_VAL_SPIFF;
        case GPUJPEG_HEADER_ADOBE: return GPUJPEG_ENC_HDR_VAL_ADOBE;
        case GPUJPEG_HEADER_EXIF: return GPUJPEG_ENC_HDR_VAL_EXIF;
    }
    return "undefined";
}
const char* gpujpeg_orientation_get_name(struct gpujpeg_orientation o)
{
    static const char* const names[8] = {"normal",
                                         "mirror horizontal",
                                         "rotated CW 90 deg",
                                         "rotated CW 90 and mirrored horizontal",
                                         "rotated 180 deg",
                                         "flipped vertical",
                                         "rotated CW 270 deg",
                                         "rotated CW 270 deg and mirrored horizontal"};
    return names[(o.rotation << 1 | o.flip) & 7];
}

/* ---- image helpers [ref: src/gpujpeg_common.c:402-470, 1176-1330] ---- */
size_t gpujpeg_image_calculate_size(struct gpujpeg_image_parameters* param)
{
    assert(param->width > 0 && param->height > 0);
    assert(param->width <= 65535 && param->height <= 65535);
    assert(param->width_padding >= 0);
    const int bpp = pixfmt_bpp(param->pixel_format);
    if ( bpp ) return ((size_t)param->width + param->width_padding) * param->height * bpp;
    switch ( param->pixel_format ) {
        case GPUJPEG_444_U8_P0P1P2: return (size_t)param->width * param->height * 3;
        case GPUJPEG_422_U8_P0P1P2:
            return (size_t)param->width * param->height + (size_t)2 * ((param->width + 1) / 2) * param->height;
        case GPUJPEG_420_U8_P0P1P2:
            return (size_t)param->width * param->height +
                   (size_t)2 * ((param->width + 1) / 2) * ((param->height + 1) / 2);
        default: return 0;
    }
}

enum gpujpeg_image_file_format gpujpeg_image_get_file_format(const char* filename)
{
    static const struct {
        const char* ext;
        enum gpujpeg_image_file_format format;
    } ext_map[] = {
        {"raw", GPUJPEG_IMAGE_FILE_RAW},   {"rgb", GPUJPEG_IMAGE_FILE_RGB},   {"rgba", GPUJPEG_IMAGE_FILE_RGBA},
        {"yuv", GPUJPEG_IMAGE_FILE_YUV},   {"yuva", GPUJPEG_IMAGE_FILE_YUVA}, {"uyvy", GPUJPEG_IMAGE_FILE_UYVY},
        {"i420", GPUJPEG_IMAGE_FILE_I420}, {"r", GPUJPEG_IMAGE_FILE_GRAY},    {"jpg", GPUJPEG_IMAGE_FILE_JPEG},
        {"jpeg", GPUJPEG_IMAGE_FILE_JPEG}, {"jfif", GPUJPEG_IMAGE_FILE_JPEG}, {"bmp", GPUJPEG_IMAGE_FILE_BMP},
        {"gif", GPUJPEG_IMAGE_FILE_GIF},   {"png", GPUJPEG_IMAGE_FILE_PNG},   {"tga", GPUJPEG_IMAGE_FILE_TGA},
        {"pnm", GPUJPEG_IMAGE_FILE_PNM},   {"pgm", GPUJPEG_IMAGE_FILE_PGM},   {"ppm", GPUJPEG_IMAGE_FILE_PPM},
        {"pam", GPUJPEG_IMAGE_FILE_PAM},   {"y4m", GPUJPEG_IMAGE_FILE_Y4M},   {"tst", GPUJPEG_IMAGE_FILE_TST},
        {"XXX", GPUJPEG_IMAGE_FILE_RAW},
    };
    const char* ext = strrchr(filename, '.');
    if ( !ext ) return GPUJPEG_IMAGE_FILE_UNKNOWN;
    ext++;
    for ( unsigned i = 0; i < sizeof ext_map / sizeof ext_map[0]; i++ )
        if ( strcasecmp(ext, ext_map[i].ext) == 0 ) return ext_map[i].format;
    return GPUJPEG_IMAGE_FILE_UNKNOWN;
}

/* "<W>x<H>[.c_<CS>][.p_<PF>][.<pattern>].tst" procedural test images
 * [ref: src/utils/image_delegate.c:341-363 usage, :561-633 generators].  Extra pattern in this build:
 * "photo[_<seed>]" (SURVEY.md section 8d S-photo). */
enum { PAT_GRADIENT, PAT_BLANK, PAT_NOISE, PAT_RANDOM, PAT_PHOTO };
static int tst_parse(const char* filename, struct gpujpeg_image_parameters* pi, int* pattern, int* arg)
{
    char name[256];
    const char* base = strrchr(filename, '/');
    base = base ? base + 1 : filename;
    if ( strlen(base) >= sizeof name ) return -1;
    strcpy(name, base);
    char* dot = strrchr(name, '.');
    if ( !dot ) return -1;
    *dot = 0; /* drop ".tst" */
    *pattern = PAT_GRADIENT;
    *arg = 12345;
    int first = 1;
    for ( char* tok = strtok(name, "."); tok; tok = strtok(NULL, "."), first = 0 ) {
        if ( first ) {
            if ( sscanf(tok, "%dx%d", &pi->width, &pi->height) != 2 || pi->width <= 0 || pi->height <= 0 ) return -1;
        }
        else if ( strncmp(tok, "c_", 2) == 0 ) {
            pi->color_space = gpujpeg_color_space_by_name(tok + 2);
            if ( pi->color_space == GPUJPEG_NONE ) return -1;
        }
        else if ( strncmp(tok, "p_", 2) == 0 ) {
            pi->pixel_format = gpujpeg_pixel_format_by_name(tok + 2);
            if ( pi->pixel_format == GPUJPEG_PIXFMT_NONE ) return -1;
        }
        else if ( strcmp(tok, "gradient") == 0 ) {
            *pattern = PAT_GRADIENT;
        }
        else if ( strcmp(tok, "noise") == 0 ) {
            *pattern = PAT_NOISE;
        }
        else if ( strncmp(tok, "blank", 5) == 0 ) {
            *pattern = PAT_BLANK;
            *arg = tok[5] == '_' ? atoi(tok + 6) : 0;
        }
        else if ( strncmp(tok, "random", 6) == 0 ) {
            *pattern = PAT_RANDOM;
            if ( tok[6] == '_' ) *arg = atoi(tok + 7);
        }
        else if ( strncmp(tok, "photo", 5) == 0 ) {
            *pattern = PAT_PHOTO;
            if ( tok[5] == '_' ) *arg = atoi(tok + 6);
        }
        else {
            GJ_ERR("Unknown .tst option: %s\n", tok);
            return -1;
        }
    }
    return first ? -1 : 0;
}

static uint32_t lcg_next(uint32_t s) { return (1664525u * s + 1013904223u) % 2147483647u; }
static int tri512(int t)
{
    int a = t % 512 - 256;
    if ( a < 0 ) a = -a;
    return a > 255 ? 255 : a;
}

static int tst_load(const char* filename, uint8_t** image, size_t* image_size)
{
    struct gpujpeg_image_parameters pi = gpujpeg_default_image_parameters();
    int pattern, arg;
    if ( tst_parse(filename, &pi, &pattern, &arg) ) {
        GJ_ERR("Cannot parse test image name %s (<W>x<H>[.c_<CS>][.p_<PF>][.<pattern>].tst)\n", filename);
        return -1;
    }
    const size_t size = gpujpeg_image_calculate_size(&pi);
    uint8_t* data = NULL;
    if ( size == 0 || gj_cuda_malloc_host((void**)&data, size) ) {
        GJ_ERR("Could not alloc host pointer: %s\n", gj_cuda_last_error());
        return -1;
    }
    switch ( pattern ) {
        case PAT_GRADIENT: {
            const size_t line = size / pi.height;
            for ( int y = 0; y < pi.height; y++ )
                memset(data + (size_t)y * line, y * 255 / pi.height, line);
            break;
        }
        case PAT_BLANK: memset(data, arg, size); break;
        case PAT_NOISE: arg = (int)(gpujpeg_get_time() * 1e6); /* non-deterministic seed */
        /* fall through */
        case PAT_RANDOM: {
            uint32_t s = (uint32_t)arg;
            for ( size_t i = 0; i < size; i++ ) {
                s = lcg_next(s);
                data[i] = (uint8_t)(s % 256u);
            }
            break;
        }
        case PAT_PHOTO: {
            if ( pi.pixel_format != GPUJPEG_444_U8_P012 ) {
                GJ_ERR("The photo pattern is defined for 444-u8-p012 only\n");
                gj_cuda_free_host(data);
                return -1;
            }
            uint32_t s = (uint32_t)arg;
            size_t i = 0;
            for ( int y = 0; y < pi.height; y++ )
                for ( int x = 0; x < pi.width; x++ )
                    for ( int ch = 0; ch < 3; ch++ ) {
                        s = lcg_next(s);
                        const int noise = (int)((s % 256u) & 31u) - 16;
                        const int v = (tri512((int)((long long)x * 1024 / pi.width) + 85 * ch) +
                                       tri512((int)((long long)y * 768 / pi.height) + 40 * ch)) / 2 + noise;
                        data[i++] = (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v);
                    }
            break;
        }
    }
    *image = data;
    *image_size = size;
    return 0;
}

static void* pinned_alloc(size_t size)
{
    void* p = NULL;
    if ( gj_cuda_malloc_host(&p, size ? size : 1) ) {
        GJ_ERR("Could not alloc host pointer: %s\n", gj_cuda_last_error());
        return NULL;
    }
    return p;
}

/* returns a CUDA-pinned buffer, to be released with gpujpeg_image_destroy [ref: src/gpujpeg_common.c:1216-1256].
 * Netpbm and Y4M files are parsed (gj_imageio.c), .tst names are generated, everything else is read as it is. */
int gpujpeg_image_load_from_file(const char* filename, uint8_t** image, size_t* image_size)
{
    const enum gpujpeg_image_file_format format = gpujpeg_image_get_file_format(filename);
    switch ( format ) {
        case GPUJPEG_IMAGE_FILE_TST: return tst_load(filename, image, image_size);
        case GPUJPEG_IMAGE_FILE_PGM:
        case GPUJPEG_IMAGE_FILE_PPM:
        case GPUJPEG_IMAGE_FILE_PNM:
        case GPUJPEG_IMAGE_FILE_PAM:
        case GPUJPEG_IMAGE_FILE_Y4M: return gj_imgfile_load(filename, image, image_size, pinned_alloc) ? 1 : 0;
        case GPUJPEG_IMAGE_FILE_BMP:
        case GPUJPEG_IMAGE_FILE_GIF:
        case GPUJPEG_IMAGE_FILE_PNG:
        case GPUJPEG_IMAGE_FILE_TGA:
            GJ_ERR("Image file format of %s is not supported by this build (raw dumps, .jpg, .tst, PNM / PAM and Y4M only)\n",
                   filename);
            return -1;
        default: break;
    }
    FILE* f = fopen(filename, "rb");
    if ( !f ) {
        GJ_ERR("Failed open %s for reading: %s\n", filename, strerror(errno));
        return -1;
    }
    if ( *image_size == 0 ) {
        fseek(f, 0, SEEK_END);
        *image_size = (size_t)ftell(f);
        rewind(f);
    }
    uint8_t* data = NULL;
    if ( gj_cuda_malloc_host((void**)&data, *image_size ? *image_size : 1) ) {
        GJ_ERR("Initialize CUDA host buffer: %s\n", gj_cuda_last_error());
        fclose(f);
        return -1;
    }
    if ( fread(data, 1, *image_size, f) != *image_size ) {
        GJ_ERR("Failed to load image data [%zd bytes] from file %s!\n", *image_size, filename);
        fclose(f);
        gj_cuda_free_host(data);
        return -1;
    }
    fclose(f);
    *image = data;
    return 0;
}

/* "name.XXX": the extension that can hold the image is filled in (the caller's string is written to, as in the reference)
 * [ref: src/gpujpeg_common.c:1258-1275]; PNM / PAM / Y4M get their headers, other names a plain dump */
int gpujpeg_image_save_to_file(const char* filename, const uint8_t* image, size_t image_size,
                               const struct gpujpeg_image_parameters* param_image)
{
    char* dot = strrchr(filename, '.');
    if ( dot && strcmp(dot, ".XXX") == 0 && param_image ) {
        const char* ext = param_image->pixel_format != GPUJPEG_U8 && param_image->color_space != GPUJPEG_RGB ? "y4m"
                          : param_image->pixel_format == GPUJPEG_4444_U8_P0123                              ? "pam"
                                                                                                            : "pnm";
        memcpy(dot + 1, ext, 3);
    }
    const enum gpujpeg_image_file_format format = gpujpeg_image_get_file_format(filename);
    if ( param_image ) {
        switch ( format ) {
            case GPUJPEG_IMAGE_FILE_PAM: return gj_imgfile_save_pam(filename, param_image, image, 0);
            case GPUJPEG_IMAGE_FILE_PGM:
            case GPUJPEG_IMAGE_FILE_PPM:
            case GPUJPEG_IMAGE_FILE_PNM: return gj_imgfile_save_pam(filename, param_image, image, 1);
            case GPUJPEG_IMAGE_FILE_Y4M: return gj_imgfile_save_y4m(filename, param_image, image);
            case GPUJPEG_IMAGE_FILE_BMP:
            case GPUJPEG_IMAGE_FILE_GIF:
            case GPUJPEG_IMAGE_FILE_PNG:
            case GPUJPEG_IMAGE_FILE_TGA:
                GJ_ERR("Image file format of %s is not supported by this build (raw dumps, .jpg, PNM / PAM and Y4M only)\n",
                       filename);
                return -1;
            default: break;
        }
    }
    FILE* f = fopen(filename, "wb");
    if ( !f ) {
        GJ_ERR("Failed open %s for writing: %s\n", filename, strerror(errno));
        return -1;
    }
    if ( fwrite(image, 1, image_size, f) != image_size ) {
        GJ_ERR("Failed to write image data [%zd bytes] to file %s!\n", image_size, filename);
        fclose(f);
        return -1;
    }
    fclose(f);
    return 0;
}

/* What a file name (and, for formats with a header, the file) says about the image.  Return values are the reference's:
 * negative = error; raw formats return 1, PAM / PNM names of files still to be written return 1 as well
 * [ref: src/gpujpeg_common.c:1311-1371, src/utils/image_delegate.c:149-205, 253-298] */
int gpujpeg_image_get_properties(const char* filename, struct gpujpeg_image_parameters* param_image, int file_exists)
{
    const enum gpujpeg_image_file_format format = gpujpeg_image_get_file_format(filename);
    int pattern, arg;
    switch ( format ) {
        case GPUJPEG_IMAGE_FILE_TST: return tst_parse(filename, param_image, &pattern, &arg);
        case GPUJPEG_IMAGE_FILE_PGM:
        case GPUJPEG_IMAGE_FILE_PPM:
        case GPUJPEG_IMAGE_FILE_PNM:
        case GPUJPEG_IMAGE_FILE_PAM:
            if ( !file_exists ) {
                param_image->pixel_format = format == GPUJPEG_IMAGE_FILE_PGM   ? GPUJPEG_U8
                                            : format == GPUJPEG_IMAGE_FILE_PPM ? GPUJPEG_444_U8_P012
                                            : format == GPUJPEG_IMAGE_FILE_PNM ? GPUJPEG_PIXFMT_NO_ALPHA
                                                                               : GPUJPEG_PIXFMT_AUTODETECT;
                param_image->color_space = format == GPUJPEG_IMAGE_FILE_PGM ? GPUJPEG_YCBCR_JPEG : GPUJPEG_CS_DEFAULT;
                return 1;
            }
            /* fall through */
        case GPUJPEG_IMAGE_FILE_Y4M: {
            if ( !file_exists ) {
                param_image->color_space = GPUJPEG_YCBCR_BT601_256LVLS;
                param_image->pixel_format = GPUJPEG_PIXFMT_STD;
                return 0;
            }
            struct gj_imgfile f;
            if ( gj_imgfile_probe(filename, &f) ) return GPUJPEG_ERROR;
            return gj_imgfile_params(filename, &f, param_image);
        }
        case GPUJPEG_IMAGE_FILE_BMP:
        case GPUJPEG_IMAGE_FILE_GIF:
        case GPUJPEG_IMAGE_FILE_PNG:
        case GPUJPEG_IMAGE_FILE_TGA:
            GJ_ERR("Image file format of %s is not supported by this build\n", filename);
            return -1;
        case GPUJPEG_IMAGE_FILE_UNKNOWN: GJ_ERR("GPUJPEG_IMAGE_FILE_UNKNOWN should not be passed!\n"); return -1;
        case GPUJPEG_IMAGE_FILE_JPEG: GJ_ERR("GPUJPEG_IMAGE_FILE_JPEG should not be passed!\n"); return -1;
        default: break;
    }
    switch ( format ) {   /* raw dumps: the extension names colour space and pixel format */
        case GPUJPEG_IMAGE_FILE_RGB:
        case GPUJPEG_IMAGE_FILE_RGBA: param_image->color_space = GPUJPEG_RGB; break;
        case GPUJPEG_IMAGE_FILE_GRAY:
        case GPUJPEG_IMAGE_FILE_YUV:
        case GPUJPEG_IMAGE_FILE_YUVA:
        case GPUJPEG_IMAGE_FILE_UYVY:
        case GPUJPEG_IMAGE_FILE_I420: param_image->color_space = GPUJPEG_YCBCR_JPEG; break;
        default: break;
    }
    switch ( format ) {
        case GPUJPEG_IMAGE_FILE_RAW: param_image->pixel_format = GPUJPEG_PIXFMT_STD; break;
        case GPUJPEG_IMAGE_FILE_GRAY: param_image->pixel_format = GPUJPEG_U8; break;
        case GPUJPEG_IMAGE_FILE_RGBA:
        case GPUJPEG_IMAGE_FILE_YUVA: param_image->pixel_format = GPUJPEG_4444_U8_P0123; break;
        case GPUJPEG_IMAGE_FILE_UYVY: param_image->pixel_format = GPUJPEG_422_U8_P1020; break;
        case GPUJPEG_IMAGE_FILE_I420: param_image->pixel_format = GPUJPEG_420_U8_P0P1P2; break;
        default: param_image->pixel_format = GPUJPEG_444_U8_P012; break;   /* .rgb, .yuv */
    }
    return 1;
}

int gpujpeg_image_destroy(uint8_t* image) { return gj_cuda_free_host(image); }

/* smallest and largest sample of every component of a raw image file, printed to stdout; packed 4:4:4 and UYVY only, as
 * in the reference [ref: src/gpujpeg_common.c:1383-1442] */
void gpujpeg_image_range_info(const char* filename, int width, int height, enum gpujpeg_pixel_format pixel_format)
{
    uint8_t* image = NULL;
    size_t size = 0;
    if ( gpujpeg_image_load_from_file(filename, &image, &size) != 0 ) {
        GJ_ERR("Failed to load image [%s]!\n", filename);
        return;
    }
    int lo[3] = {256, 256, 256}, hi[3] = {0, 0, 0};
    const size_t pixels = (size_t)(width > 0 ? width : 0) * (size_t)(height > 0 ? height : 0);
    if ( pixel_format == GPUJPEG_444_U8_P012 && size >= pixels * 3 ) {
        for ( size_t i = 0; i < pixels * 3; i++ ) {
            const int c = (int)(i % 3), v = image[i];
            if ( v < lo[c] ) lo[c] = v;
            if ( v > hi[c] ) hi[c] = v;
        }
    }
    else if ( pixel_format == GPUJPEG_422_U8_P1020 && size >= pixels * 2 ) {
        /* U Y V Y: the odd bytes are luminance, the even ones alternate between the chrominance components; the reference
         * files the byte of an even pixel under component 3 and that of an odd pixel under component 2 */
        for ( size_t i = 0; i < pixels; i++ ) {
            const int y = image[2 * i + 1], ch = image[2 * i], c = (i & 1) ? 1 : 2;
            if ( y < lo[0] ) lo[0] = y;
            if ( y > hi[0] ) hi[0] = y;
            if ( ch < lo[c] ) lo[c] = ch;
            if ( ch > hi[c] ) hi[c] = ch;
        }
    }
    else {
        GJ_ERR("gpujpeg_image_range_info handles 444-u8-p012 and 422-u8-p1020 files of at least width x height pixels only.\n");
        gpujpeg_image_destroy(image);
        return;
    }
    printf("Image Samples Range:\n");
    for ( int c = 0; c < 3; c++ )
        printf("Component %d: %d - %d\n", c + 1, lo[c], hi[c]);
    gpujpeg_image_destroy(image);
}

/* "currently defunct" in the reference as well [ref: libgpujpeg/gpujpeg_common.h:455-470] */
int gpujpeg_image_convert(const char* input, const char* output, struct gpujpeg_image_parameters param_image_from,
                          struct gpujpeg_image_parameters param_image_to)
{
    (void)input; (void)output; (void)param_image_from; (void)param_image_to;
    GJ_ERR("gpujpeg_image_convert is defunct\n");
    return -1;
}

/* ---- OpenGL interop: same answers as the reference built without GL [ref: src/gpujpeg_common.c:1521-1887] ---- */
int gpujpeg_opengl_init(struct gpujpeg_opengl_context** ctx) { (void)ctx; return -2; }
void gpujpeg_opengl_destroy(struct gpujpeg_opengl_context* ctx) { (void)ctx; }
int gpujpeg_opengl_texture_create(int width, int height, uint8_t* data) { (void)width; (void)height; (void)data; return 0; }
int gpujpeg_opengl_texture_set_data(int texture_id, uint8_t* data) { (void)texture_id; (void)data; return -1; }
int gpujpeg_opengl_texture_get_data(int texture_id, uint8_t* data, size_t* data_size)
{
    (void)texture_id; (void)data; (void)data_size;
    return -1;
}
void gpujpeg_opengl_texture_destroy(int texture_id) { (void)texture_id; }
struct gpujpeg_opengl_texture* gpujpeg_opengl_texture_register(int texture_id, enum gpujpeg_opengl_texture_type texture_type)
{
    (void)texture_id; (void)texture_type;
    GJ_ERR("OpenGL interoperability is not supported in this build\n");
    return NULL;
}
void gpujpeg_opengl_texture_unregister(struct gpujpeg_opengl_texture* texture) { (void)texture; }
uint8_t* gpujpeg_opengl_texture_map(struct gpujpeg_opengl_texture* texture, size_t* data_size)
{
    (void)texture; (void)data_size;
    return NULL;
}
void gpujpeg_opengl_texture_unmap(struct gpujpeg_opengl_texture* texture) { (void)texture; }

/* [ref: src/gpujpeg_common.c:2325-2338] */
int gj_parse_bool(const char* val, const char* optname)
{
    if ( strcasecmp(val, GPUJPEG_VAL_TRUE) == 0 ) return 1;
    if ( strcasecmp(val, GPUJPEG_VAL_FALSE) == 0 ) return 0;
    GJ_ERR("Unknown option %s for %s\n", val, optname);
    return -1;
}

/* [ref: src/gpujpeg_encoder.c:662-698] "XYZ[W]": output channel i takes input channel <digit i>; 'F' = all ones,
 * 'Z' = all zeros */
unsigned gj_parse_channel_remap(const char* val, const char* optname)
{
    const int count = (int)strlen(val);
    if ( count < 1 || count > GPUJPEG_MAX_COMPONENT_COUNT ) {
        GJ_ERR("Mapping for more than %d channels specified!\n", GPUJPEG_MAX_COMPONENT_COUNT);
        return 0;
    }
    unsigned map = 0;
    for ( int i = count - 1; i >= 0; i-- ) {
        int src = val[i] - '0';
        if ( val[i] == 'F' ) src = 4;
        else if ( val[i] == 'Z' ) src = 5;
        else if ( src < 0 || src >= count ) {
            GJ_ERR("Invalid channel index %c for %s (mapping %d channels)!\n", val[i], optname, count);
            return 0;
        }
        map = map << 4 | (unsigned)src;
    }
    return map | (unsigned)count << 24;
}
