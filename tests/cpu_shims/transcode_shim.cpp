// The transcoder's coefficient map (gj_coef_src in gj_device.cuh) compiled for the host: tests/test_transcode_plan.py.
#include "../../gpujpeg_b200/csrc/gj_device.cuh"

extern "C" int ts_coef_src(int k, int transpose, int neg_x, int neg_y, int* negate)
{
    return gj_coef_src(k, transpose, neg_x, neg_y, negate);
}
