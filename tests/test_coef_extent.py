"""The block-extent helpers of gj_device.cuh (the decoder's format between the Huffman decoder and the IDCT), compiled for the
host: a block whose last stored coefficient has zig-zag index k has extent k // 8 + 1 chunks, at most GJ_CEXT_FULL; every
coefficient up to k lies inside it, and nothing in a chunk past it counts."""
import os
import subprocess

import numpy as np

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpujpeg_b200", "csrc")

PROGRAM = r"""
#include <stdio.h>
#include "gj_device.cuh"
int main()
{
    printf("%d\n", GJ_CEXT_FULL);
    for ( int last = 0; last < 64; last++ ) {
        printf("%d", gj_cext_of(last));
        for ( int k = 0; k < 64; k++ )
            printf(" %d", (int)gj_cext_holds(gj_cext_of(last), k));
        printf("\n");
    }
    for ( int ext = 0; ext <= GJ_CEXT_FULL; ext++ ) {
        for ( int k = 0; k < 64; k++ )
            printf("%d ", (int)gj_cext_holds(ext, k));
        printf("\n");
    }
    return 0;
}
"""


def test_extent_helpers(tmp_path):
    src, exe = tmp_path / "cext.cpp", tmp_path / "cext"
    src.write_text(PROGRAM)
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++17", "-I", CSRC, "-o", str(exe), str(src)])
    lines = subprocess.check_output([str(exe)], text=True).split("\n")
    full = int(lines[0])
    assert full == 8
    for last in range(64):
        vals = [int(x) for x in lines[1 + last].split()]
        ext, holds = vals[0], np.array(vals[1:], bool)
        assert ext == last // 8 + 1 and 1 <= ext <= full
        assert holds[:last + 1].all(), "a stored coefficient lies outside its block's extent"
        assert holds.sum() == 8 * ext
    for ext in range(full + 1):
        holds = np.array([int(x) for x in lines[65 + ext].split()], bool)
        assert np.array_equal(holds, np.arange(64) < 8 * ext)
