"""ctypes binding of the C ABI in include/lilliput_b200.h + include/lp_opencv.h.

The same `Lib` class binds either library:

* ``lilliput_b200/liblilliput_b200.so`` -- the product: sm_90a CUDA kernels
  behind lilliput's cgo surface.  `load_cuda()` fails loudly if it is missing
  or no CUDA device can be initialised; there is no CPU fallback.
* ``oracle/_ref/libref_oracle.so`` -- the reference's own shims (test
  infrastructure; see oracle/Makefile).  Only tests/, __graft_entry__.smoke()
  and bench.py's CPU-baseline legs may load it.

Function names mirror the reference API they stand for (ref ops.go / opencv.go).
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_LIB = os.environ.get("LP_CUDA_LIB") or os.path.join(ROOT, "lilliput_b200", "liblilliput_b200.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_oracle.so")

# ImageOpsSizeMethod, ref ops.go:17-22
ImageOpsNoResize, ImageOpsFit, ImageOpsResize = 0, 1, 2
# encoder option keys, ref opencv.hpp:33-36 / opencv.go:62-70
JpegQuality, JpegProgressive, PngCompression, WebpQuality = 1, 2, 16, 64
# OpenCV pixel types
CV_8UC1, CV_8UC3, CV_8UC4 = 0, 16, 24
INTER_LINEAR, INTER_CUBIC, INTER_AREA = 1, 2, 3

LP_OK, LP_ERR_INVALID_IMAGE, LP_ERR_DECODING_FAILED, LP_ERR_BUF_TOO_SMALL = 0, -1, -2, -3
LP_ERR_FRAMEBUF_NO_PIXELS, LP_ERR_SKIP_NOT_SUPPORTED, LP_ERR_ENCODE_TIMEOUT, LP_ERR_EOF = -4, -5, -6, -7

LP_ERRORS = {
    0: "ok", -1: "ErrInvalidImage", -2: "ErrDecodingFailed", -3: "ErrBufTooSmall",
    -4: "ErrFrameBufNoPixels", -5: "ErrSkipNotSupported", -6: "ErrEncodeTimeout", -7: "EOF",
    -8: "unsupported", -9: "cuda", -10: "bad argument",
}


class LilliputError(RuntimeError):
    def __init__(self, code: int):
        self.code = code
        super().__init__(LP_ERRORS.get(code, f"lp_status {code}"))


class _ImageOptions(C.Structure):
    _fields_ = [
        ("file_type", C.c_char_p), ("width", C.c_int), ("height", C.c_int),
        ("resize_method", C.c_int), ("normalize_orientation", C.c_int),
        ("encode_options", C.POINTER(C.c_int)), ("encode_options_len", C.c_size_t),
        ("max_encode_frames", C.c_int), ("max_encode_duration_ns", C.c_int64),
        ("encode_timeout_ns", C.c_int64), ("disable_animated_output", C.c_int),
        ("force_sdr", C.c_int),
    ]


class _BatchConfig(C.Structure):
    _fields_ = [
        ("device", C.c_int), ("max_images", C.c_int), ("src_width", C.c_int),
        ("src_height", C.c_int), ("dst_width", C.c_int), ("dst_height", C.c_int),
        ("resize_method", C.c_int), ("jpeg_quality", C.c_int), ("max_in_bytes", C.c_size_t),
        ("out_cap", C.c_size_t), ("chunk", C.c_int),
    ]


@dataclass
class ImageOptions:
    """Mirror of lilliput.ImageOptions (ref ops.go:26-65)."""
    FileType: str = ".jpeg"
    Width: int = 0
    Height: int = 0
    ResizeMethod: int = ImageOpsNoResize
    NormalizeOrientation: bool = False
    EncodeOptions: dict = field(default_factory=dict)
    MaxEncodeFrames: int = 0
    MaxEncodeDuration_ns: int = 0
    EncodeTimeout_ns: int = 0
    DisableAnimatedOutput: bool = False
    ForceSdr: bool = False

    def _c(self):
        flat = []
        for k, v in self.EncodeOptions.items():
            flat += [int(k), int(v)]
        arr = (C.c_int * max(1, len(flat)))(*flat)
        o = _ImageOptions(self.FileType.encode(), self.Width, self.Height, self.ResizeMethod,
                          int(self.NormalizeOrientation), arr, len(flat), self.MaxEncodeFrames,
                          self.MaxEncodeDuration_ns, self.EncodeTimeout_ns,
                          int(self.DisableAnimatedOutput), int(self.ForceSdr))
        o._keep = arr
        return o


def _u8p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_uint8))


class Lib:
    def __init__(self, path: str):
        if not os.path.exists(path):
            raise FileNotFoundError(
                f"{path} is not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
        self.path = path
        self.l = C.CDLL(path, mode=getattr(os, "RTLD_LOCAL", 0) | getattr(os, "RTLD_NOW", 2))
        l = self.l
        l.lp_backend_name.restype = C.c_char_p
        l.lp_transform.restype = C.c_int
        l.lp_transform.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(_ImageOptions), C.c_void_p,
                                   C.c_size_t, C.POINTER(C.c_size_t), C.c_int]
        l.lp_decode_host.restype = C.c_int
        l.lp_decode_host.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t] + \
            [C.POINTER(C.c_int)] * 4
        l.lp_fit_host.restype = C.c_int
        l.lp_fit_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                  C.c_int]
        l.lp_resize_host.restype = C.c_int
        l.lp_resize_host.argtypes = [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p] + [C.c_int] * 3
        l.lp_encode_host.restype = C.c_int
        l.lp_encode_host.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.POINTER(C.c_int), C.c_size_t, C.c_void_p, C.c_size_t,
                                     C.POINTER(C.c_size_t)]
        l.lp_orient_host.restype = C.c_int
        l.lp_orient_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                     C.POINTER(C.c_int), C.POINTER(C.c_int)]
        self.backend = l.lp_backend_name().decode()

    # --- whole path: NewDecoder + ImageOps.Transform (ref ops.go:352) -------------------
    def transform(self, data: bytes, opt: ImageOptions, dst_cap: int = 8 << 20,
                  max_size: int = 8192) -> bytes:
        src = np.frombuffer(data, dtype=np.uint8)
        dst = np.empty(dst_cap, dtype=np.uint8)
        n = C.c_size_t(0)
        o = opt._c()
        rc = self.l.lp_transform(src.ctypes.data, src.size, C.byref(o), dst.ctypes.data, dst.size,
                                 C.byref(n), max_size)
        if rc != 0:
            raise LilliputError(rc)
        return dst[: n.value].tobytes()

    # --- stages ---------------------------------------------------------------------
    def header(self, data: bytes):
        src = np.frombuffer(data, dtype=np.uint8)
        w, h, t, o = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        rc = self.l.lp_decode_host(src.ctypes.data, src.size, None, 0, C.byref(w), C.byref(h),
                                   C.byref(t), C.byref(o))
        if rc != 0:
            raise LilliputError(rc)
        return w.value, h.value, t.value, o.value

    def decode(self, data: bytes) -> np.ndarray:
        """openCVDecoder.DecodeTo (ref opencv.go:816): packed BGR/BGRA/Gray u8."""
        w0, h0, t0, _ = self.header(data)
        if max(w0, h0) > 8192:  # the helper's framebuffer limit (lilliput_host.cpp kHelperMaxSide)
            raise LilliputError(LP_ERR_BUF_TOO_SMALL)
        src = np.frombuffer(data, dtype=np.uint8)
        ch = ((t0 >> 3) & 63) + 1
        px = np.empty(h0 * w0 * ch, dtype=np.uint8)
        w, h, t, o = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        rc = self.l.lp_decode_host(src.ctypes.data, src.size, px.ctypes.data, px.size, C.byref(w),
                                   C.byref(h), C.byref(t), C.byref(o))
        if rc != 0:
            raise LilliputError(rc)
        return px.reshape(h.value, w.value, ch) if ch > 1 else px.reshape(h.value, w.value)

    @staticmethod
    def _type_of(img: np.ndarray) -> int:
        ch = 1 if img.ndim == 2 else img.shape[2]
        return (ch - 1) << 3

    def fit(self, img: np.ndarray, w: int, h: int) -> np.ndarray:
        """Framebuffer.Fit (ref opencv.go:326)."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        ch = 1 if img.ndim == 2 else img.shape[2]
        dst = np.empty((h, w, ch) if ch > 1 else (h, w), dtype=np.uint8)
        rc = self.l.lp_fit_host(img.ctypes.data, img.shape[1], img.shape[0], self._type_of(img),
                                dst.ctypes.data, w, h)
        if rc != 0:
            raise LilliputError(rc)
        return dst

    def resize(self, img: np.ndarray, w: int, h: int, crop=None, interpolation=INTER_AREA):
        """opencv_mat_resize on an opencv_mat_crop view (ref opencv.cpp:196-215)."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        ch = 1 if img.ndim == 2 else img.shape[2]
        cx, cy, cw, chh = crop if crop else (0, 0, img.shape[1], img.shape[0])
        dst = np.empty((h, w, ch) if ch > 1 else (h, w), dtype=np.uint8)
        rc = self.l.lp_resize_host(img.ctypes.data, img.shape[1], img.shape[0], self._type_of(img),
                                   cx, cy, cw, chh, dst.ctypes.data, w, h, interpolation)
        if rc != 0:
            raise LilliputError(rc)
        return dst

    def encode(self, ext: str, img: np.ndarray, opts: dict | None = None,
               dst_cap: int = 0) -> bytes:
        """openCVEncoder.Encode (ref opencv.go:872)."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        flat = []
        for k, v in (opts or {}).items():
            flat += [int(k), int(v)]
        arr = (C.c_int * max(1, len(flat)))(*flat)
        cap = dst_cap or (img.size * 2 + (1 << 16))
        dst = np.empty(cap, dtype=np.uint8)
        n = C.c_size_t(0)
        rc = self.l.lp_encode_host(ext.encode(), img.ctypes.data, img.shape[1], img.shape[0],
                                   self._type_of(img), arr, len(flat), dst.ctypes.data, dst.size,
                                   C.byref(n))
        if rc != 0:
            raise LilliputError(rc)
        return dst[: n.value].tobytes()

    # --- GIF (ref giflib.go) -------------------------------------------------------------
    def gif_info(self, data: bytes) -> dict:
        class _Info(C.Structure):
            _fields_ = [("width", C.c_int), ("height", C.c_int), ("frame_count", C.c_int),
                        ("loop_count", C.c_int), ("duration_ms", C.c_int), ("background_color", C.c_uint)]
        src = np.frombuffer(data, dtype=np.uint8)
        info = _Info()
        self.l.lp_gif_get_info.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p]
        rc = self.l.lp_gif_get_info(src.ctypes.data, src.size, C.byref(info))
        if rc != 0:
            raise LilliputError(rc)
        return {k: getattr(info, k) for k, _ in _Info._fields_}

    def gif_frames(self, data: bytes, max_frames: int = 1 << 16):
        """gifDecoder.DecodeTo until EOF: (frames[n,h,w,4] BGRA full canvas, delays_ms, disposals, rc)."""
        info = self.gif_info(data)
        n = max(1, min(max_frames, info["frame_count"] + 1))
        src = np.frombuffer(data, dtype=np.uint8)
        frames = np.zeros((n, info["height"], info["width"], 4), dtype=np.uint8)
        delays = (C.c_int * n)()
        disp = (C.c_int * n)()
        got = C.c_int(0)
        self.l.lp_gif_decode_frames_host.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int,
                                                     C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
        rc = self.l.lp_gif_decode_frames_host(src.ctypes.data, src.size, frames.ctypes.data, frames.nbytes,
                                              n, C.byref(got), delays, disp)
        k = got.value
        return frames[:k], list(delays[:k]), list(disp[:k]), rc

    # --- WebP (ref webp.hpp) ---------------------------------------------------------------
    def webp_frames(self, data: bytes, max_frames: int = 1 << 16, decode: bool = True):
        """Raw webp_decoder_* walk: (info dict, [frame arrays], [meta dicts], rc)."""
        src = np.frombuffer(data, dtype=np.uint8)
        info = (C.c_uint * 8)()
        got = C.c_int(0)
        f = self.l.lp_webp_decode_frames_host
        f.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_int), C.c_void_p,
                      C.c_void_p]
        rc = f(src.ctypes.data, src.size, None, 0, 0, C.byref(got), None, info)
        if rc != 0:
            return None, [], [], rc
        keys = ("width", "height", "pixel_type", "num_frames", "total_duration", "loop_count", "bg_color", "icc_len")
        inf = dict(zip(keys, [int(v) for v in info]))
        if not decode:
            return inf, [], [], 0
        n = max(1, min(max_frames, inf["num_frames"]))
        buf = np.zeros(n * inf["width"] * inf["height"] * 4, dtype=np.uint8)
        meta = (C.c_int * (8 * n))()
        rc = f(src.ctypes.data, src.size, buf.ctypes.data, buf.nbytes, n, C.byref(got), meta, info)
        frames, metas, off = [], [], 0
        for i in range(got.value):
            w, h, ch, x, y, delay, dispose, blend = [int(v) for v in meta[8 * i:8 * i + 8]]
            frames.append(buf[off:off + w * h * ch].reshape(h, w, ch).copy())
            off += w * h * ch
            metas.append(dict(x=x, y=y, delay=delay, dispose=dispose, blend=blend))
        return inf, frames, metas, rc

    def tonemap(self, img: np.ndarray, transfer: int, primaries: int) -> np.ndarray:
        """Framebuffer.TonemapToSDR (ref opencv.go:791-810) on a packed BGR / BGRA frame."""
        out = np.ascontiguousarray(img).copy()
        self.l.lp_tonemap_host.restype = C.c_int
        self.l.lp_tonemap_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        rc = self.l.lp_tonemap_host(out.ctypes.data, out.shape[1], out.shape[0], self._type_of(out), transfer, primaries)
        if rc:
            raise LilliputError(rc)
        return out

    def orient(self, img: np.ndarray, orientation: int) -> np.ndarray:
        """Framebuffer.OrientationTransform (ref opencv.go:271)."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        ch = 1 if img.ndim == 2 else img.shape[2]
        dst = np.empty(img.size, dtype=np.uint8)
        ow, oh = C.c_int(), C.c_int()
        rc = self.l.lp_orient_host(img.ctypes.data, img.shape[1], img.shape[0],
                                   self._type_of(img), orientation, dst.ctypes.data,
                                   C.byref(ow), C.byref(oh))
        if rc != 0:
            raise LilliputError(rc)
        return dst.reshape(oh.value, ow.value, ch) if ch > 1 else dst.reshape(oh.value, ow.value)


_cache: dict[str, Lib] = {}


def load_cuda() -> Lib:
    """The product library.  Raises if it was not built -- never falls back."""
    if "cuda" not in _cache:
        _cache["cuda"] = Lib(CUDA_LIB)
    return _cache["cuda"]


def load_reference() -> Lib:
    """oracle/_ref (reference shims).  Test/baseline infrastructure only."""
    if "ref" not in _cache:
        _cache["ref"] = Lib(REF_LIB)
    return _cache["ref"]


# ----------------------------------------------------------------------------------------------
# Batch API (CUDA library only)
# ----------------------------------------------------------------------------------------------
STAGE_NAMES = ["huff_decode", "idct_color", "resize", "enc_transform", "enc_entropy", "total"]


class Batch:
    """lp_batch_*: N independent JPEGs -> Fit/area resize -> JPEG on one GPU."""

    def __init__(self, lib: Lib, device: int, max_images: int, src_w: int, src_h: int, dst_w: int,
                 dst_h: int, quality: int, max_in_bytes: int, out_cap: int = 65536,
                 resize_method: int = ImageOpsFit, chunk: int = 0):
        self.lib = lib
        l = lib.l
        l.lp_batch_create.restype = C.c_void_p
        l.lp_batch_create.argtypes = [C.POINTER(_BatchConfig)]
        l.lp_batch_destroy.argtypes = [C.c_void_p]
        for name in ("lp_batch_stage",):
            getattr(l, name).restype = C.c_int
        l.lp_batch_stage.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        l.lp_batch_run.restype = C.c_int
        l.lp_batch_run.argtypes = [C.c_void_p, C.c_void_p]
        l.lp_batch_fetch.restype = C.c_int
        l.lp_batch_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        l.lp_batch_transform.restype = C.c_int
        l.lp_batch_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
        l.lp_batch_last_launches.restype = C.c_int
        l.lp_batch_last_launches.argtypes = [C.c_void_p]
        l.lp_batch_chunk.restype = C.c_int
        l.lp_batch_chunk.argtypes = [C.c_void_p]
        for name in ("lp_batch_decoded_dev", "lp_batch_resized_dev"):
            getattr(l, name).restype = C.c_void_p
            getattr(l, name).argtypes = [C.c_void_p, C.POINTER(C.c_size_t)]
        l.lp_memcpy_d2h.restype = C.c_int
        l.lp_memcpy_d2h.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        cfg = _BatchConfig(device, max_images, src_w, src_h, dst_w, dst_h, resize_method, quality,
                           max_in_bytes, out_cap, chunk)
        self.h = l.lp_batch_create(C.byref(cfg))
        if not self.h:
            raise RuntimeError("lp_batch_create failed (no CUDA device / out of memory)")
        self.max_images = max_images
        self.out_cap = out_cap

    def close(self):
        if self.h:
            self.lib.l.lp_batch_destroy(self.h)
            self.h = None

    @staticmethod
    def _ptr_arrays(bufs):
        n = len(bufs)
        ptrs = (C.c_void_p * n)()
        lens = (C.c_size_t * n)()
        keep = []
        for i, b in enumerate(bufs):
            if isinstance(b, tuple):  # (address, length): already-pinned memory
                ptrs[i], lens[i] = b
            else:
                a = np.frombuffer(b, dtype=np.uint8)
                keep.append(a)
                ptrs[i], lens[i] = a.ctypes.data, a.size
        return ptrs, lens, keep

    def stage(self, bufs):
        ptrs, lens, keep = self._ptr_arrays(bufs)
        status = (C.c_int * len(bufs))()
        rc = self.lib.l.lp_batch_stage(self.h, ptrs, lens, len(bufs), status)
        if rc:
            raise LilliputError(rc)
        return list(status)

    def run(self):
        ms = (C.c_float * 6)()
        rc = self.lib.l.lp_batch_run(self.h, ms)
        if rc:
            raise LilliputError(rc)
        return dict(zip(STAGE_NAMES, list(ms)))

    def fetch(self, n):
        out = np.empty((n, self.out_cap), dtype=np.uint8)
        ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
        lens = (C.c_size_t * n)()
        status = (C.c_int * n)()
        rc = self.lib.l.lp_batch_fetch(self.h, ptrs, lens, status)
        if rc:
            raise LilliputError(rc)
        return [out[i, : lens[i]].tobytes() for i in range(n)], list(status)

    def transform_into(self, ptrs, lens, n, out_ptrs, out_lens, status):
        """Raw call for bench.py: all arrays prebuilt (no Python work in the timed region)."""
        return self.lib.l.lp_batch_transform(self.h, ptrs, lens, n, out_ptrs, out_lens, status)

    def transform(self, bufs):
        n = len(bufs)
        ptrs, lens, keep = self._ptr_arrays(bufs)
        out = np.empty((n, self.out_cap), dtype=np.uint8)
        out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
        out_lens = (C.c_size_t * n)()
        status = (C.c_int * n)()
        rc = self.lib.l.lp_batch_transform(self.h, ptrs, lens, n, out_ptrs, out_lens, status)
        if rc:
            raise LilliputError(rc)
        return [out[i, : out_lens[i]].tobytes() for i in range(n)], list(status)

    def last_launches(self):
        return self.lib.l.lp_batch_last_launches(self.h)

    def _copy_back(self, getter, n):
        stride = C.c_size_t(0)
        ptr = getter(self.h, C.byref(stride))
        buf = np.empty((n, stride.value), dtype=np.uint8)
        rc = self.lib.l.lp_memcpy_d2h(buf.ctypes.data, ptr, buf.nbytes)
        if rc:
            raise LilliputError(rc)
        return buf

    def decoded_windows(self, n: int, win_h: int) -> np.ndarray:
        """The decoded pixel windows of the last `run()`: (n, win_h, row stride in bytes), u8 BGR, rows padded as
        the decoder wrote them.  The frame buffer holds one chunk, so the staged batch must fit in one."""
        if n > self.lib.l.lp_batch_chunk(self.h):
            raise ValueError("the decoded frames of a multi-chunk batch are not kept")
        buf = self._copy_back(self.lib.l.lp_batch_decoded_dev, n)
        if buf.shape[1] % win_h:
            raise ValueError(f"frame stride {buf.shape[1]} is not a whole number of {win_h} rows")
        return buf.reshape(n, win_h, buf.shape[1] // win_h)

    def resized_frames(self, n: int, w: int, h: int) -> np.ndarray:
        """The resized frames of the last `run()`: (n, h, w, 3) u8 BGR."""
        buf = self._copy_back(self.lib.l.lp_batch_resized_dev, n)
        if buf.shape[1] != w * h * 3:
            raise ValueError(f"resized frames are {buf.shape[1]} bytes, not {w}x{h}x3")
        return buf.reshape(n, h, w, 3)


# ----------------------------------------------------------------------------------------------
class _XBatchConfig(C.Structure):
    _fields_ = [("device", C.c_int), ("arena_bytes", C.c_size_t), ("host_threads", C.c_int), ("max_size", C.c_int)]


class _XBatchStats(C.Structure):
    _fields_ = [("grid_items", C.c_int), ("fallback_items", C.c_int), ("groups", C.c_int), ("launches", C.c_int),
                ("ms_parse", C.c_double), ("ms_grid", C.c_double), ("ms_fallback", C.c_double), ("ms_total", C.c_double),
                ("ms_decode", C.c_double), ("ms_resize", C.c_double), ("ms_encode", C.c_double),
                ("h2d_bytes", C.c_size_t), ("d2h_bytes", C.c_size_t), ("ms_busy_max_lane", C.c_double)]


class XBatch:
    """lp_xbatch_*: N independent images of any supported format / size, one set of options, grouped into grid
    launches; per-item results are those of lp_transform (include/lilliput_b200.h)."""

    def __init__(self, lib: Lib, device: int = 0, arena_bytes: int = 0, host_threads: int = 0, max_size: int = 8192):
        self.lib = lib
        l = lib.l
        l.lp_xbatch_create.restype = C.c_void_p
        l.lp_xbatch_create.argtypes = [C.POINTER(_XBatchConfig)]
        l.lp_xbatch_destroy.argtypes = [C.c_void_p]
        l.lp_xbatch_transform.restype = C.c_int
        l.lp_xbatch_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(_ImageOptions),
                                          C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        l.lp_xbatch_get_stats.argtypes = [C.c_void_p, C.POINTER(_XBatchStats)]
        cfg = _XBatchConfig(device, arena_bytes, host_threads, max_size)
        self.h = l.lp_xbatch_create(C.byref(cfg))
        if not self.h:
            raise RuntimeError("lp_xbatch_create failed (no CUDA device / out of memory)")

    def close(self):
        if self.h:
            self.lib.l.lp_xbatch_destroy(self.h)
            self.h = None

    def transform_into(self, ptrs, lens, n, copt, out_ptrs, out_cap, out_lens, status):
        """Raw call for bench.py: every array prebuilt."""
        return self.lib.l.lp_xbatch_transform(self.h, ptrs, lens, n, C.byref(copt), out_ptrs, out_cap, out_lens, status)

    def transform(self, bufs, opt: ImageOptions, out_cap: int = 1 << 20):
        n = len(bufs)
        ptrs, lens, keep = Batch._ptr_arrays(bufs)
        out = np.empty((n, out_cap), dtype=np.uint8)
        out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
        out_lens = (C.c_size_t * n)()
        status = (C.c_int * n)()
        copt = opt._c()
        rc = self.lib.l.lp_xbatch_transform(self.h, ptrs, lens, n, C.byref(copt), out_ptrs, out_cap, out_lens, status)
        if rc:
            raise LilliputError(rc)
        return [out[i, : out_lens[i]].tobytes() for i in range(n)], list(status)

    def stats(self) -> dict:
        s = _XBatchStats()
        self.lib.l.lp_xbatch_get_stats(self.h, C.byref(s))
        return {k: getattr(s, k) for k, _ in _XBatchStats._fields_}


class MultiBatch:
    """lp_multi_*: one lp_xbatch per GPU behind one call, sharded by image index (contiguous blocks balanced by
    compressed bytes), no collective."""

    def __init__(self, lib: Lib, devices, arena_bytes: int = 0, host_threads: int = 0, max_size: int = 8192):
        self.lib = lib
        l = lib.l
        l.lp_multi_create.restype = C.c_void_p
        l.lp_multi_create.argtypes = [C.POINTER(C.c_int), C.c_int, C.POINTER(_XBatchConfig)]
        l.lp_multi_destroy.argtypes = [C.c_void_p]
        l.lp_multi_transform.restype = C.c_int
        l.lp_multi_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(_ImageOptions),
                                         C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        l.lp_multi_get_stats.argtypes = [C.c_void_p, C.c_int, C.POINTER(_XBatchStats)]
        devs = (C.c_int * len(devices))(*devices)
        cfg = _XBatchConfig(0, arena_bytes, host_threads, max_size)
        self.n_devices = len(devices)
        self.h = l.lp_multi_create(devs, len(devices), C.byref(cfg))
        if not self.h:
            raise RuntimeError("lp_multi_create failed")

    def close(self):
        if self.h:
            self.lib.l.lp_multi_destroy(self.h)
            self.h = None

    def transform_into(self, ptrs, lens, n, copt, out_ptrs, out_cap, out_lens, status):
        return self.lib.l.lp_multi_transform(self.h, ptrs, lens, n, C.byref(copt), out_ptrs, out_cap, out_lens, status)

    def transform(self, bufs, opt: ImageOptions, out_cap: int = 1 << 20):
        n = len(bufs)
        ptrs, lens, keep = Batch._ptr_arrays(bufs)
        out = np.empty((n, out_cap), dtype=np.uint8)
        out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
        out_lens = (C.c_size_t * n)()
        status = (C.c_int * n)()
        copt = opt._c()
        rc = self.lib.l.lp_multi_transform(self.h, ptrs, lens, n, C.byref(copt), out_ptrs, out_cap, out_lens, status)
        if rc:
            raise LilliputError(rc)
        return [out[i, : out_lens[i]].tobytes() for i in range(n)], list(status)

    def stats(self, device_index: int) -> dict:
        s = _XBatchStats()
        self.lib.l.lp_multi_get_stats(self.h, device_index, C.byref(s))
        return {k: getattr(s, k) for k, _ in _XBatchStats._fields_}
