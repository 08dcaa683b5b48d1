"""Builds gpujpeg_b200/lib/libgpujpeg.so.0 -- the drop-in C-ABI library -- for sm_90a (H100).

Host files are C (gcc), kernels are CUDA (nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo),
the CUDA runtime is linked statically so the .so is self-contained next to torch's own runtime.
nvcc cross-compiles without a GPU, so this runs in the build container; the built .so is
git-ignored but travels to the GPU box with the repo snapshot.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
SONAME = "libgpujpeg.so.0"
LIB = os.path.join(LIBDIR, SONAME)

C_SOURCES = ["gj_tables.c", "gj_codestream.c", "gj_common.c", "gj_imageio.c", "gj_exif.c", "gj_encoder.c", "gj_decoder.c", "gj_batch.c",
             "gj_transcoder.c"]
CU_SOURCES = ["gj_cuda_util.cu", "gj_dct.cu", "gj_huffman.cu", "gj_huffdec.cu", "gj_huffscan.cu", "gj_markers.cu", "gj_convert.cu", "gj_progressive.cu",
              "gj_transcode.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _gcc():
    return "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    """Compile (if needed) and return the path of libgpujpeg.so.0."""
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(OBJDIR, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "gpujpeg_b200.h"))
    headers.append(os.path.join(os.path.dirname(HERE), "include", "gpujpegx.h"))
    have_sources = all(os.path.exists(os.path.join(CSRC, f)) for f in C_SOURCES + CU_SOURCES)
    if not have_sources:
        if os.path.exists(LIB):
            return LIB
        raise RuntimeError("gpujpeg_b200 sources missing and no prebuilt library")
    objs = []
    relink = force
    for src in C_SOURCES:
        s, o = os.path.join(CSRC, src), os.path.join(OBJDIR, src + ".o")
        if force or _stale(o, [s] + headers):
            cmd = [_gcc(), "-O2", "-std=gnu11", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wextra", "-Wno-unused-parameter",
                   "-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            subprocess.check_call(cmd)
            relink = True
        objs.append(o)
    for src in CU_SOURCES:
        s, o = os.path.join(CSRC, src), os.path.join(OBJDIR, src + ".o")
        if force or _stale(o, [s] + headers):
            cmd = [_nvcc(), "-O3", "-std=c++17", "-lineinfo", *ARCH, "-Xcompiler", "-fPIC,-fvisibility=hidden",
                   "-Xptxas", "-v" if verbose else "-warn-spills", "-c", s, "-o", o]
            if verbose:
                print(" ".join(cmd))
            subprocess.check_call(cmd)
            relink = True
        objs.append(o)
    if relink or not os.path.exists(LIB):
        cmd = [_nvcc(), "-shared", *ARCH, "-cudart", "static", "-Xlinker", "-soname=" + SONAME, "-o", LIB, *objs, "-lpthread"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
        link = os.path.join(LIBDIR, "libgpujpeg.so")
        if os.path.lexists(link):
            os.remove(link)
        os.symlink(SONAME, link)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
