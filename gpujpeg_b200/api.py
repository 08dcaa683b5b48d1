"""ctypes mirror of the libgpujpeg C API (include/gpujpeg_b200.h).

Names, argument meaning and error behaviour follow the reference interface
(libgpujpeg/gpujpeg_{common,encoder,decoder}.h): functions return 0 / -1, constructors return NULL,
diagnostics go to stderr.  The small ``Encoder`` / ``Decoder`` classes only manage lifetimes and
numpy <-> pointer conversion around ``gpujpeg_encoder_encode`` / ``gpujpeg_decoder_decode``.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

GPUJPEG_NOERR, GPUJPEG_ERROR = 0, -1
# enum gpujpeg_color_space
GPUJPEG_NONE, GPUJPEG_RGB, GPUJPEG_YCBCR_BT601, GPUJPEG_YCBCR_BT601_256LVLS, GPUJPEG_YCBCR_BT709, GPUJPEG_YUV = 0, 1, 2, 3, 4, 5
GPUJPEG_YCBCR_JPEG = GPUJPEG_YCBCR_BT601_256LVLS
# enum gpujpeg_pixel_format
GPUJPEG_PIXFMT_NONE, GPUJPEG_U8, GPUJPEG_444_U8_P012, GPUJPEG_444_U8_P0P1P2 = -1, 0, 1, 2
GPUJPEG_422_U8_P1020, GPUJPEG_422_U8_P0P1P2, GPUJPEG_420_U8_P0P1P2, GPUJPEG_4444_U8_P0123 = 3, 4, 5, 6
# enum gpujpeg_encoder_input_type / gpujpeg_decoder_output_type
GPUJPEG_ENCODER_INPUT_IMAGE, GPUJPEG_ENCODER_INPUT_OPENGL_TEXTURE, GPUJPEG_ENCODER_INPUT_GPU_IMAGE = 0, 1, 2
(GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER, GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER, GPUJPEG_DECODER_OUTPUT_OPENGL_TEXTURE,
 GPUJPEG_DECODER_OUTPUT_CUDA_BUFFER, GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER) = range(5)
RESTART_AUTO, RESTART_NONE = -1, 0


class SamplingFactor(C.Structure):
    _fields_ = [("horizontal", C.c_uint8), ("vertical", C.c_uint8)]


class Parameters(C.Structure):
    """struct gpujpeg_parameters"""
    _fields_ = [("verbose", C.c_int), ("perf_stats", C.c_int), ("quality", C.c_int), ("restart_interval", C.c_int),
                ("interleaved", C.c_int), ("segment_info", C.c_int), ("comp_count", C.c_int),
                ("sampling_factor", SamplingFactor * 4), ("color_space_internal", C.c_int)]


class ImageParameters(C.Structure):
    """struct gpujpeg_image_parameters"""
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("color_space", C.c_int), ("pixel_format", C.c_int),
                ("width_padding", C.c_int)]


class EncoderInput(C.Structure):
    _fields_ = [("type", C.c_int), ("image", C.c_void_p), ("texture", C.c_void_p)]


class DecoderOutput(C.Structure):
    _fields_ = [("type", C.c_int), ("data", C.c_void_p), ("data_size", C.c_size_t), ("param_image", ImageParameters),
                ("texture", C.c_void_p), ("metadata", C.c_void_p)]


class DurationStats(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("duration_memory_to", "duration_memory_from", "duration_memory_map",
                                          "duration_memory_unmap", "duration_preprocessor", "duration_dct_quantization",
                                          "duration_huffman_coder", "duration_stream", "duration_in_gpu")]


class GpuJpegError(RuntimeError):
    pass


def library_path():
    return _build.build_library()


def _load():
    path = library_path()
    lib_ = C.CDLL(path)
    vp, ci, cs = C.c_void_p, C.c_int, C.c_size_t
    sigs = {
        "gpujpeg_version": (ci, []),
        "gpujpeg_version_to_string": (C.c_char_p, [ci]),
        "gpujpeg_init_device": (ci, [ci, ci]),
        "gpujpeg_set_default_parameters": (None, [C.POINTER(Parameters)]),
        "gpujpeg_image_set_default_parameters": (None, [C.POINTER(ImageParameters)]),
        "gpujpeg_parameters_chroma_subsampling": (None, [C.POINTER(Parameters), C.c_uint32]),
        "gpujpeg_image_calculate_size": (cs, [C.POINTER(ImageParameters)]),
        "gpujpeg_image_load_from_file": (ci, [C.c_char_p, C.POINTER(vp), C.POINTER(cs)]),
        "gpujpeg_image_destroy": (ci, [vp]),
        "gpujpeg_encoder_create": (vp, [vp]),
        "gpujpeg_encoder_destroy": (ci, [vp]),
        "gpujpeg_encoder_encode": (ci, [vp, C.POINTER(Parameters), C.POINTER(ImageParameters), C.POINTER(EncoderInput),
                                        C.POINTER(vp), C.POINTER(cs)]),
        "gpujpeg_encoder_set_option": (ci, [vp, C.c_char_p, C.c_char_p]),
        "gpujpeg_encoder_get_stats": (ci, [vp, C.POINTER(DurationStats)]),
        "gpujpeg_encoder_suggest_restart_interval": (ci, [C.POINTER(ImageParameters), C.c_uint32, C.c_bool, ci]),
        "gpujpeg_decoder_create": (vp, [vp]),
        "gpujpeg_decoder_destroy": (ci, [vp]),
        "gpujpeg_decoder_decode": (ci, [vp, vp, cs, C.POINTER(DecoderOutput)]),
        "gpujpeg_decoder_set_option": (ci, [vp, C.c_char_p, C.c_char_p]),
        "gpujpeg_decoder_set_output_format": (None, [vp, ci, ci]),
        "gpujpeg_decoder_get_stats": (ci, [vp, C.POINTER(DurationStats)]),
        "gpujpeg_decoder_get_image_info": (ci, [vp, cs, C.POINTER(ImageParameters), C.POINTER(Parameters), C.POINTER(ci)]),
        "gpujpegx_encoder_get_coefficients": (ci, [vp, vp, cs]),
        "gpujpegx_encoder_get_stream": (C.c_longlong, [vp, vp, cs]),
        "gpujpegx_encoder_run_resident": (ci, [vp, vp, ci]),
        "gpujpegx_decoder_run_resident": (ci, [vp, vp, ci]),
        "gpujpegx_decoder_get_coefficients": (ci, [vp, vp, cs]),
        "gpujpegx_decoder_used_segment_info": (ci, [vp]),
        "gpujpegx_batch_create": (vp, [C.POINTER(ci), ci]),
        "gpujpegx_batch_destroy": (None, [vp]),
        "gpujpegx_batch_device_count": (ci, [vp]),
        "gpujpegx_batch_owner": (ci, [vp, ci]),
        "gpujpegx_batch_encode": (ci, [vp, C.POINTER(Parameters), C.POINTER(ImageParameters), C.POINTER(vp), ci, ci, C.POINTER(vp),
                                       C.POINTER(cs)]),
        "gpujpegx_batch_decode": (ci, [vp, C.POINTER(vp), C.POINTER(cs), ci, C.POINTER(vp), ci]),
        "gpujpegx_batch_last_ms": (C.c_double, [vp]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(lib_, name)
        fn.restype, fn.argtypes = res, args
    return lib_


lib = _load()


def version():
    return lib.gpujpeg_version_to_string(lib.gpujpeg_version()).decode()


SUBSAMPLING = {"4:4:4": (1, 1), "4:2:2": (2, 1), "4:2:0": (2, 2), "4:4:0": (1, 2)}


def default_parameters(quality=75, restart_interval=RESTART_AUTO, interleaved=0, subsampling="4:4:4"):
    """subsampling: a J:a:b name or the luminance sampling factors (h, v); chrominance is 1x1
    (what gpujpeg_parameters_chroma_subsampling(param, GPUJPEG_SUBSAMPLING_xxx) sets)."""
    p = Parameters()
    lib.gpujpeg_set_default_parameters(C.byref(p))
    p.quality, p.restart_interval, p.interleaved = quality, restart_interval, interleaved
    lh, lv = SUBSAMPLING[subsampling] if isinstance(subsampling, str) else subsampling
    if (lh, lv) != (1, 1):   # GPUJPEG_SUBSAMPLING_xxx packing: one nibble pair per component, first component on top
        lib.gpujpeg_parameters_chroma_subsampling(C.byref(p), lh << 28 | lv << 24 | 0x111100)
    return p


def coefficient_count(width, height, sampling=(1, 1), interleaved=0):
    """int16 coefficients the coder keeps for a 3-component frame [ref: src/gpujpeg_common.c:671-736]"""
    mh, mv = sampling
    n = 0
    for c in range(3):
        hs, vs = (mh, mv) if c == 0 else (1, 1)
        dh_, dv_ = mh // hs, mv // vs
        cw = (width + dh_ - 1) // dh_ * dh_ * hs // mh
        ch = (height + dv_ - 1) // dv_ * dv_ * vs // mv
        mx, my = (8 * hs, 8 * vs) if interleaved else (8, 8)
        n += ((cw + mx - 1) // mx * mx) * ((ch + my - 1) // my * my)
    return n


def image_parameters(width, height, width_padding=0, pixel_format=None, color_space=None):
    pi = ImageParameters()
    lib.gpujpeg_image_set_default_parameters(C.byref(pi))
    pi.width, pi.height, pi.width_padding = width, height, width_padding
    if pixel_format is not None:
        pi.pixel_format = pixel_format
    if color_space is not None:
        pi.color_space = color_space
    return pi


# enum gpujpeg_pixel_format / gpujpeg_color_space values used by the helpers below
(GPUJPEG_U8, GPUJPEG_444_U8_P012, GPUJPEG_444_U8_P0P1P2, GPUJPEG_422_U8_P1020, GPUJPEG_422_U8_P0P1P2,
 GPUJPEG_420_U8_P0P1P2, GPUJPEG_4444_U8_P0123) = range(7)
GPUJPEG_PIXFMT_AUTODETECT, GPUJPEG_PIXFMT_NO_ALPHA = -2, -3
GPUJPEG_PIXFMT_NATIVE, GPUJPEG_PIXFMT_STD = -5, -4
GPUJPEG_NONE, GPUJPEG_RGB, GPUJPEG_YCBCR_BT601, GPUJPEG_YCBCR_JPEG, GPUJPEG_YCBCR_BT709 = range(5)
GPUJPEG_CS_DEFAULT = -1


def _ptr(x):
    """host numpy array, torch tensor (host or device) or raw integer address -> (address, is_device)"""
    if isinstance(x, int):
        return x, None
    if isinstance(x, np.ndarray):
        assert x.flags["C_CONTIGUOUS"]
        return x.ctypes.data, False
    if hasattr(x, "data_ptr"):
        assert x.is_contiguous()
        return x.data_ptr(), bool(x.is_cuda)
    raise TypeError(type(x))


class Encoder:
    """gpujpeg_encoder_create / gpujpeg_encoder_encode / gpujpeg_encoder_destroy"""

    def __init__(self, stream=0, pinned_output=False):
        self._h = lib.gpujpeg_encoder_create(C.c_void_p(stream))
        if not self._h:
            raise GpuJpegError("gpujpeg_encoder_create failed (no CUDA device?)")
        if pinned_output:
            self.set_option("enc_opt_out", "enc_out_val_pinned")

    def set_option(self, key, val):
        if lib.gpujpeg_encoder_set_option(self._h, key.encode(), val.encode()) != 0:
            raise GpuJpegError("gpujpeg_encoder_set_option(%s, %s) failed" % (key, val))

    def encode_raw(self, image, param, param_image, device=None):
        """returns (address, size) of the encoder-owned JPEG buffer (valid until the next call)"""
        addr, is_dev = _ptr(image)
        if device is not None:
            is_dev = device
        inp = EncoderInput(GPUJPEG_ENCODER_INPUT_GPU_IMAGE if is_dev else GPUJPEG_ENCODER_INPUT_IMAGE, addr, None)
        out, size = C.c_void_p(), C.c_size_t()
        rc = lib.gpujpeg_encoder_encode(self._h, C.byref(param), C.byref(param_image), C.byref(inp), C.byref(out),
                                        C.byref(size))
        if rc != 0:
            raise GpuJpegError("gpujpeg_encoder_encode failed (%d)" % rc)
        return out.value, size.value

    def encode(self, image, quality=75, restart_interval=RESTART_AUTO, interleaved=0, width=None, height=None,
               width_padding=0, verbose=0, subsampling="4:4:4", segment_info=0):
        """image: HxWx3 uint8 numpy array / torch tensor (host or cuda).  Returns the JPEG as numpy uint8 (a copy)."""
        if width is None:
            height, width = image.shape[0], image.shape[1]
        p = default_parameters(quality, restart_interval, interleaved, subsampling)
        p.verbose = verbose
        p.segment_info = segment_info
        addr, size = self.encode_raw(image, p, image_parameters(width, height, width_padding))
        return np.ctypeslib.as_array((C.c_uint8 * size).from_address(addr)).copy()

    def encode_samples(self, raw, width, height, pixel_format, quality=75, restart_interval=RESTART_AUTO, interleaved=0,
                       color_space=GPUJPEG_YCBCR_JPEG, subsampling=None, alpha=False, color_space_internal=None):
        """raw: flat uint8 buffer in `pixel_format` / `color_space`.  With the JPEG colour space and subsampling=None the
        samples go into the JPEG as they are (the JPEG takes the format's sampling); other colour spaces are
        transformed, and `subsampling` ("4:2:0", ...) selects a JPEG sampling other than the format's.  Returns the
        JPEG bytes."""
        p = default_parameters(quality, restart_interval, interleaved, subsampling or "4:4:4")
        if subsampling == "4:4:4":
            lib.gpujpeg_parameters_chroma_subsampling(C.byref(p), 0x11111100)
        if alpha:   # comp_count = 4: the alpha samples of a 4444-u8-p0123 image become a fourth component (first one's sampling)
            lh, lv = SUBSAMPLING[subsampling or "4:4:4"]
            lib.gpujpeg_parameters_chroma_subsampling(C.byref(p), lh << 28 | lv << 24 | 0x111100 | lh << 4 | lv)
        if color_space_internal is not None:
            p.color_space_internal = color_space_internal
        # subsampling None: comp_count stays 0 and the sampling is derived from the pixel format
        addr, size = self.encode_raw(raw, p, image_parameters(width, height, 0, pixel_format, color_space))
        return np.ctypeslib.as_array((C.c_uint8 * size).from_address(addr)).copy()

    def run_resident(self, d_raw=None, stage_mask=3):
        """enqueue the GPU stages only (bit0 K1, bit1 K2) on device-resident data; no copies, no sync"""
        addr = _ptr(d_raw)[0] if d_raw is not None else None
        if lib.gpujpegx_encoder_run_resident(self._h, addr, stage_mask) != 0:
            raise GpuJpegError("gpujpegx_encoder_run_resident failed")

    def stream(self):
        """the JPEG bytes the last K2 launch produced (after run_resident too), as gpujpeg_encoder_encode returns them"""
        n = lib.gpujpegx_encoder_get_stream(self._h, None, 0)
        out = np.empty(max(n, 0), np.uint8)
        if n < 0 or lib.gpujpegx_encoder_get_stream(self._h, out.ctypes.data, out.size) != n:
            raise GpuJpegError("gpujpegx_encoder_get_stream failed")
        return out

    def coefficients(self, width, height, sampling=(1, 1), interleaved=0):
        """quantised coefficients of the last frame, natural order (parity tests): (3, blocks*64) int16 for 4:4:4,
        one flat array, component after component, for the subsampled modes"""
        if tuple(sampling) == (1, 1):
            dw, dh = (width + 7) // 8 * 8, (height + 7) // 8 * 8
            out = np.empty((3, dw * dh), np.int16)
        else:
            out = np.empty(coefficient_count(width, height, sampling, interleaved), np.int16)
        if lib.gpujpegx_encoder_get_coefficients(self._h, out.ctypes.data, out.size) != 0:
            raise GpuJpegError("gpujpegx_encoder_get_coefficients failed")
        return out

    def stats(self):
        s = DurationStats()
        return s if lib.gpujpeg_encoder_get_stats(self._h, C.byref(s)) == 0 else None

    def close(self):
        if self._h:
            lib.gpujpeg_encoder_destroy(self._h)
            self._h = None

    __del__ = close


class Decoder:
    """gpujpeg_decoder_create / gpujpeg_decoder_decode / gpujpeg_decoder_destroy"""

    def __init__(self, stream=0, idct="int"):
        self._h = lib.gpujpeg_decoder_create(C.c_void_p(stream))
        if not self._h:
            raise GpuJpegError("gpujpeg_decoder_create failed (no CUDA device?)")
        if idct != "int":
            self.set_option("dec_opt_idct", idct)

    def set_option(self, key, val):
        if lib.gpujpeg_decoder_set_option(self._h, key.encode(), val.encode()) != 0:
            raise GpuJpegError("gpujpeg_decoder_set_option(%s, %s) failed" % (key, val))

    def decode_raw(self, jpeg_addr, jpeg_size, out_type=GPUJPEG_DECODER_OUTPUT_INTERNAL_BUFFER, out_addr=None):
        out = DecoderOutput()
        out.type = out_type
        out.data = out_addr
        rc = lib.gpujpeg_decoder_decode(self._h, C.c_void_p(jpeg_addr), jpeg_size, C.byref(out))
        if rc != 0:
            raise GpuJpegError("gpujpeg_decoder_decode failed (%d)" % rc)
        return out

    def decode(self, jpeg, out=None):
        """jpeg: uint8 numpy array.  out: optional HxWx3 destination (numpy = custom host buffer, cuda tensor =
        custom CUDA buffer).  Returns an HxWx3 uint8 numpy array (a copy) or `out`."""
        jpeg = np.ascontiguousarray(jpeg, np.uint8)
        if out is None:
            o = self.decode_raw(jpeg.ctypes.data, jpeg.size)
            w, h = o.param_image.width, o.param_image.height
            return np.ctypeslib.as_array((C.c_uint8 * o.data_size).from_address(o.data)).reshape(h, w, 3).copy()
        addr, is_dev = _ptr(out)
        self.decode_raw(jpeg.ctypes.data, jpeg.size,
                        GPUJPEG_DECODER_OUTPUT_CUSTOM_CUDA_BUFFER if is_dev else GPUJPEG_DECODER_OUTPUT_CUSTOM_BUFFER, addr)
        return out

    def set_output_format(self, color_space, pixel_format):
        lib.gpujpeg_decoder_set_output_format(self._h, color_space, pixel_format)

    def decode_samples(self, jpeg):
        """decode with the output format set by set_output_format; returns (flat uint8 copy, ImageParameters)"""
        jpeg = np.ascontiguousarray(jpeg, np.uint8)
        o = self.decode_raw(jpeg.ctypes.data, jpeg.size)
        return np.ctypeslib.as_array((C.c_uint8 * o.data_size).from_address(o.data)).copy(), o.param_image

    def run_resident(self, d_out=None, stage_mask=3):
        """enqueue the GPU stages only (bit0 K3, bit1 K4) of the last decoded frame; no copies, no sync"""
        addr = _ptr(d_out)[0] if d_out is not None else None
        if lib.gpujpegx_decoder_run_resident(self._h, addr, stage_mask) != 0:
            raise GpuJpegError("gpujpegx_decoder_run_resident failed")

    def used_segment_info(self):
        """True if the last frame's scans were split by the stream's own segment-info tables (no marker scan on the device)"""
        return lib.gpujpegx_decoder_used_segment_info(self._h) == 1

    def coefficients(self, width, height, sampling=(1, 1), interleaved=0):
        """coefficients of the last frame, natural order: (array, dequantized) -- with the integer IDCT flavour
        the Huffman decoder already stores coefficient*quantiser wrapped to int16 (dequantized = True)"""
        if tuple(sampling) == (1, 1):
            dw, dh = (width + 7) // 8 * 8, (height + 7) // 8 * 8
            out = np.empty((3, dw * dh), np.int16)
        else:
            out = np.empty(coefficient_count(width, height, sampling, interleaved), np.int16)
        rc = lib.gpujpegx_decoder_get_coefficients(self._h, out.ctypes.data, out.size)
        if rc < 0:
            raise GpuJpegError("gpujpegx_decoder_get_coefficients failed")
        return out, bool(rc)

    def stats(self):
        s = DurationStats()
        return s if lib.gpujpeg_decoder_get_stats(self._h, C.byref(s)) == 0 else None

    def close(self):
        if self._h:
            lib.gpujpeg_decoder_destroy(self._h)
            self._h = None

    __del__ = close


GPUJPEGX_HOST, GPUJPEGX_DEVICE_OWNER, GPUJPEGX_DEVICE_FIRST = 0, 1, 2


class Batch:
    """gpujpegx_batch_*: frames sharded round-robin over the GPUs of one box, one worker (host thread + stream + coder
    pair) per device (include/gpujpegx.h).  `devices`: list of device indices (a device may appear more than once:
    several workers on one GPU); None = every visible device."""

    def __init__(self, devices=None):
        if devices is None:
            self._h = lib.gpujpegx_batch_create(None, 0)
        else:
            arr = (C.c_int * len(devices))(*devices)
            self._h = lib.gpujpegx_batch_create(arr, len(devices))
        if not self._h:
            raise GpuJpegError("gpujpegx_batch_create failed")
        self.device_count = lib.gpujpegx_batch_device_count(self._h)

    def owner(self, frame):
        return lib.gpujpegx_batch_owner(self._h, frame)

    def encode(self, images, param, param_image, where=GPUJPEGX_HOST):
        """images: list of arrays / tensors / addresses.  Returns the list of JPEG streams (numpy copies)."""
        n = len(images)
        ptrs = (C.c_void_p * n)(*[_ptr(x)[0] for x in images])
        out, sizes = (C.c_void_p * n)(), (C.c_size_t * n)()
        if lib.gpujpegx_batch_encode(self._h, C.byref(param), C.byref(param_image), ptrs, n, where, out, sizes) != 0:
            raise GpuJpegError("gpujpegx_batch_encode failed")
        return [np.ctypeslib.as_array((C.c_uint8 * sizes[f]).from_address(out[f])).copy() for f in range(n)]

    def decode(self, jpegs, outputs, where=GPUJPEGX_HOST):
        """jpegs: list of uint8 numpy arrays; outputs: list of destination arrays / tensors (filled in place)"""
        n = len(jpegs)
        jpegs = [np.ascontiguousarray(j, np.uint8) for j in jpegs]
        ptrs = (C.c_void_p * n)(*[j.ctypes.data for j in jpegs])
        sizes = (C.c_size_t * n)(*[j.size for j in jpegs])
        outs = (C.c_void_p * n)(*[_ptr(x)[0] for x in outputs])
        if lib.gpujpegx_batch_decode(self._h, ptrs, sizes, n, outs, where) != 0:
            raise GpuJpegError("gpujpegx_batch_decode failed")
        return outputs

    def last_ms(self):
        return lib.gpujpegx_batch_last_ms(self._h)

    def close(self):
        if self._h:
            lib.gpujpegx_batch_destroy(self._h)
            self._h = None

    __del__ = close
