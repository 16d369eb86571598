"""Helpers shared by the WebP tests (test infrastructure)."""
import ctypes
import os
import struct
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_BUILD = os.path.join(ROOT, "oracle", "_build")


def webp_golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "webp_golden.npz"))


def chunks_of(webp: bytes):
    """[(tag, payload)] of a RIFF/WEBP file's top-level chunks."""
    pos, out = 12, []
    while pos + 8 <= len(webp):
        n = struct.unpack("<I", webp[pos + 4:pos + 8])[0]
        out.append((webp[pos:pos + 4], webp[pos + 8:pos + 8 + n]))
        pos += 8 + n + (n & 1)
    return out


def vp8_cpu_lib():
    """oracle/oracle_webp.cpp (the device's WebP codec logic compiled for the host) as a ctypes handle."""
    os.makedirs(_BUILD, exist_ok=True)
    so = os.path.join(_BUILD, "libvp8cpu.so")
    srcs = [os.path.join(ROOT, "oracle", "oracle_webp.cpp"),
            os.path.join(ROOT, "lilliput_b200", "csrc", "vp8_core.h"),
            os.path.join(ROOT, "lilliput_b200", "csrc", "vp8_tables.h"),
            os.path.join(ROOT, "lilliput_b200", "csrc", "vp8l_core.h"),
            os.path.join(ROOT, "lilliput_b200", "csrc", "vp8_enc_core.h"),
            os.path.join(ROOT, "lilliput_b200", "csrc", "vp8l_enc_core.h")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, srcs[0]])
    return ctypes.CDLL(so)


def vp8_cpu_decode(lib, payload: bytes) -> np.ndarray:
    arr = np.frombuffer(payload, np.uint8)
    w, h = ctypes.c_int(), ctypes.c_int()
    p = arr.ctypes.data_as(ctypes.c_void_p)
    assert lib.vp8_cpu_info(p, ctypes.c_size_t(arr.size), ctypes.byref(w), ctypes.byref(h)) == 0
    out = np.zeros((h.value, w.value, 3), np.uint8)
    rc = lib.vp8_cpu_decode_bgr(p, ctypes.c_size_t(arr.size), out.ctypes.data_as(ctypes.c_void_p), w.value * 3, 0, None)
    assert rc == 0, rc
    return out


def frames_of(webp: bytes):
    """[(image_tag, image_payload, alph_payload or None)] for every frame of a still or animated file."""
    out = []
    for tag, payload in chunks_of(webp):
        if tag == b"ANMF":
            sub = chunks_of(b"\0" * 12 + payload[16:])
            alph = next((p for t, p in sub if t == b"ALPH"), None)
            img = next(((t, p) for t, p in sub if t in (b"VP8 ", b"VP8L")))
            out.append((img[0], img[1], alph))
    if not out:
        top = chunks_of(webp)
        alph = next((p for t, p in top if t == b"ALPH"), None)
        img = next(((t, p) for t, p in top if t in (b"VP8 ", b"VP8L")))
        out.append((img[0], img[1], alph))
    return out


def vp8l_cpu_decode(lib, payload: bytes, w: int, h: int, channels: int) -> np.ndarray:
    arr = np.frombuffer(payload, np.uint8)
    out = np.zeros((h, w, channels), np.uint8)
    rc = lib.vp8l_cpu_decode(arr.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(arr.size), w, h,
                             out.ctypes.data_as(ctypes.c_void_p), channels)
    assert rc == 0, rc
    return out


def alph_cpu_decode(lib, payload: bytes, w: int, h: int) -> np.ndarray:
    arr = np.frombuffer(payload, np.uint8)
    out = np.zeros((h, w), np.uint8)
    rc = lib.alph_cpu_decode(arr.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(arr.size), w, h,
                             out.ctypes.data_as(ctypes.c_void_p))
    assert rc == 0, rc
    return out


def vp8l_cpu_encode(lib, img: np.ndarray) -> bytes:
    """vp8l_enc_core.h on the host: BGR(A) frame -> "VP8L" payload, or a plane -> "ALPH" payload."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    c = 1 if img.ndim == 2 else img.shape[2]
    out = np.zeros(w * h * 8 + 65536, np.uint8)
    lib.vp8l_cpu_encode.restype = ctypes.c_long
    n = lib.vp8l_cpu_encode(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(w * c), w, h, c,
                            out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(out.size))
    assert n > 0, n
    return out[:n].tobytes()


def vp8_cpu_encode(lib, img: np.ndarray, quality: int, filter_level: int = -1, try_i4=None) -> bytes:
    """vp8_enc_core.h on the host: BGR(A) frame -> "VP8 " payload.  try_i4: None = as the device encodes, 0 / 1 = forced."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w, c = img.shape
    out = np.zeros(w * h * 4 + 65536, np.uint8)
    if try_i4 is None:
        lib.vp8_cpu_encode.restype = ctypes.c_long
        n = lib.vp8_cpu_encode(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(w * c), w, h, c, quality, filter_level,
                               out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(out.size))
    else:
        lib.vp8_cpu_encode_i4.restype = ctypes.c_long
        n = lib.vp8_cpu_encode_i4(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(w * c), w, h, c, quality, filter_level,
                                  int(try_i4), out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(out.size))
    assert n > 0, n
    return out[:n].tobytes()


def optional_reference():
    """The reference's own shims (oracle/_ref) when they are built, else None: tests check them in addition to
    libwebp_decode, never instead of it."""
    from lilliput_b200 import abi
    return abi.load_reference() if os.path.exists(abi.REF_LIB) else None


def libwebp_decode(data: bytes) -> np.ndarray:
    """A whole WebP file decoded by libwebp (OpenCV's WebP codec): BGR, or BGRA when the file has alpha -- what
    WebPDecodeBGR(A)Into gives.  An independent decoder of the device's streams."""
    import cv2
    img = cv2.imdecode(np.frombuffer(bytes(data), np.uint8), cv2.IMREAD_UNCHANGED)
    assert img is not None, "libwebp refused the stream"
    return img


def pillow_animation(data: bytes):
    """(frame count, loop count, [frame durations in ms], (width, height)) of an animated WebP, as Pillow's WebP
    reader (libwebp's demuxer) sees them."""
    import io

    from PIL import Image
    im = Image.open(io.BytesIO(bytes(data)))
    assert im.format == "WEBP"
    durations = []
    for k in range(im.n_frames):
        im.seek(k)
        im.load()  # (the reader sets a frame's duration when it decodes it)
        durations.append(im.info["duration"])
    return im.n_frames, im.info.get("loop", 0), durations, im.size


def vp8_partition_sizes(payload: bytes):
    """(first partition size, [token partition sizes]) of a "VP8 " key-frame payload, from its frame tag and the
    partition size table behind the first partition (RFC 6386 9.1 / 9.5)."""
    tag = payload[0] | (payload[1] << 8) | (payload[2] << 16)
    p0 = tag >> 5
    nparts = 1 << _log2_partitions_field(payload, p0)
    at = 10 + p0
    sizes = [int.from_bytes(payload[at + 3 * i:at + 3 * i + 3], "little") for i in range(nparts - 1)]
    rest = len(payload) - at - 3 * (nparts - 1) - sum(sizes)
    return p0, sizes + [rest]


def _log2_partitions_field(payload: bytes, p0: int) -> int:
    """The 2-bit partition-count field of the frame header, read with a boolean decoder (RFC 6386 7.3 / 9.2-9.5)."""
    data = payload[10:10 + p0]
    value, pos, rng, bits = (data[0] << 8) | data[1], 2, 255, 8

    def read_bit():
        nonlocal value, pos, rng, bits
        split = 1 + (((rng - 1) * 128) >> 8)
        big = split << 8
        if value >= big:
            bit, rng, value = 1, rng - split, value - big
        else:
            bit, rng = 0, split
        while rng < 128:
            value <<= 1
            rng <<= 1
            bits -= 1
            if bits == 0:
                value |= data[pos] if pos < len(data) else 0
                pos += 1
                bits = 8
        return bit

    def read_literal(n):
        v = 0
        for _ in range(n):
            v = (v << 1) | read_bit()
        return v
    # colour space, clamping, segmentation (this encoder writes none), filter type, level, sharpness, no deltas
    read_literal(2)
    assert read_bit() == 0, "segmentation header not parsed here"
    read_literal(1 + 6 + 3)
    assert read_bit() == 0, "loop-filter deltas not parsed here"
    return read_literal(2)


def riff(chunks) -> bytes:
    body = b"WEBP" + b"".join(t + struct.pack("<I", len(p)) + p + (b"\0" if len(p) & 1 else b"") for t, p in chunks)
    return b"RIFF" + struct.pack("<I", len(body)) + body


def psnr(a, b) -> float:
    m = ((a.astype(np.float64) - b.astype(np.float64)) ** 2).mean()
    return 99.0 if m == 0 else float(10 * np.log10(255.0 * 255.0 / m))
