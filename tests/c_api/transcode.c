/* A C caller of the transcoder (include/gpujpegx.h): reads a JPEG file, rewrites it losslessly with a transform and a restart
 * interval, writes the result.
 *   transcode <in.jpg> <out.jpg> <transform> <restart>      exit 0 ok, 3 no CUDA device, 1 error */
#include <gpujpegx.h>
#include <stdio.h>
#include <stdlib.h>

int main(int argc, char** argv)
{
    if ( argc < 5 ) return 1;
    FILE* f = fopen(argv[1], "rb");
    if ( !f ) return 1;
    fseek(f, 0, SEEK_END);
    const long size = ftell(f);
    fseek(f, 0, SEEK_SET);
    uint8_t* jpeg = (uint8_t*)malloc((size_t)size);
    if ( !jpeg || fread(jpeg, 1, (size_t)size, f) != (size_t)size ) return 1;
    fclose(f);

    struct gpujpegx_transcoder* t = gpujpegx_transcoder_create(NULL);
    if ( !t ) return 3;
    uint8_t* out = NULL;
    size_t out_size = 0;
    if ( gpujpegx_transcoder_set_option(t, GPUJPEGX_TRAN_OPT_TRANSFORM, argv[3]) ||
         gpujpegx_transcoder_set_option(t, GPUJPEGX_TRAN_OPT_RESTART, argv[4]) ||
         gpujpegx_transcode(t, jpeg, (size_t)size, &out, &out_size) ) {
        gpujpegx_transcoder_destroy(t);
        return 1;
    }
    f = fopen(argv[2], "wb");
    if ( !f || fwrite(out, 1, out_size, f) != out_size ) return 1;
    fclose(f);
    printf("%zu -> %zu bytes\n", (size_t)size, out_size);
    gpujpegx_transcoder_destroy(t);
    free(jpeg);
    return 0;
}
