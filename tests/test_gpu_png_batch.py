"""GPU: the batched PNG encoder below lp_xbatch (csrc/png_encode.cu, png_encode_batch through lp_png_encode_batch_dev)
and its device checksum arithmetic (lp_png_checksums_dev: warp_crc32 / warp_adler_partials per 32 KB piece, the
pieces folded as the pack kernel folds a file's chunks).

N frames of one geometry through one batch equal N calls of the per-image encoder, which is the same launcher with
N = 1; the CRC-32 and Adler-32 equal zlib's on buffers whose lengths leave every lane-slice remainder."""
import ctypes as C
import zlib

import numpy as np
import pytest

from lilliput_b200 import abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_lib):
    l = cuda_lib.l
    l.lp_dev_alloc.restype = C.c_void_p
    l.lp_dev_alloc.argtypes = [C.c_size_t]
    l.lp_dev_free.argtypes = [C.c_void_p]
    for f in (l.lp_memcpy_h2d, l.lp_memcpy_d2h):
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    l.lp_png_checksums_dev.restype = C.c_int
    l.lp_png_checksums_dev.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    l.lp_png_encode_batch_dev.restype = C.c_int
    l.lp_png_encode_batch_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]
    return l


def device_checksums(l, data: bytes):
    d = l.lp_dev_alloc(max(len(data), 1))
    assert d
    try:
        if data:
            buf = np.frombuffer(data, np.uint8)
            assert l.lp_memcpy_h2d(d, buf.ctypes.data, buf.size) == 0
        crc, adler = C.c_uint32(0), C.c_uint32(0)
        assert l.lp_png_checksums_dev(d, len(data), C.byref(crc), C.byref(adler)) == 0
        return crc.value, adler.value
    finally:
        l.lp_dev_free(d)


def test_device_checksums_are_zlibs(dev):
    rng = np.random.default_rng(6)
    lengths = [0, 1, 2, 31, 32, 33, 63, 64, 65, 1000, 32767, 32768, 32769, 65535, 65536, 65537]
    lengths += [32768 + r for r in range(3, 32, 4)] + [int(v) for v in rng.integers(70000, 1 << 20, 6)] + [1 << 20]
    for n in lengths:
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert device_checksums(dev, data) == (zlib.crc32(data), zlib.adler32(data)), n
    for data in (b"\xff" * 100000, bytes(100000)):
        assert device_checksums(dev, data) == (zlib.crc32(data), zlib.adler32(data))


def encode_batch(l, frames: np.ndarray, level: int, adaptive: bool, slot: int, pad: int = 0):
    """frames: (n, h, w, ch) u8.  pad: extra bytes between rows and between frames (strides the batch must honour)."""
    n, h, w, ch = frames.shape
    row = w * ch + pad
    img = row * h + 3 * pad
    host = np.zeros(n * img + 16, np.uint8)
    for i in range(n):
        view = host[i * img: i * img + row * h].reshape(h, row)
        view[:, : w * ch] = frames[i].reshape(h, w * ch)
        view[:, w * ch:] = 0xA5
    d_frames, d_files, d_len = l.lp_dev_alloc(host.size), l.lp_dev_alloc(n * slot), l.lp_dev_alloc(4 * n)
    assert d_frames and d_files and d_len
    try:
        assert l.lp_memcpy_h2d(d_frames, host.ctypes.data, host.size) == 0
        assert l.lp_png_encode_batch_dev(d_frames, img, row, w, h, ch, n, level, int(adaptive), d_files, slot, d_len) == 0
        lens = np.zeros(n, np.uint32)
        files = np.zeros(n * slot, np.uint8)
        assert l.lp_memcpy_d2h(lens.ctypes.data, d_len, 4 * n) == 0
        assert l.lp_memcpy_d2h(files.ctypes.data, d_files, n * slot) == 0
        return [files[i * slot: i * slot + int(lens[i])].tobytes() for i in range(n)]
    finally:
        for p in (d_frames, d_files, d_len):
            l.lp_dev_free(p)


@pytest.mark.parametrize("case", [(64, 48, 3, 5), (256, 256, 3, 9), (100, 70, 4, 4), (33, 17, 1, 7), (1, 1, 3, 3),
                                  (85, 128, 3, 2), (300, 400, 4, 3)])
def test_batch_equals_per_image_encoder(cuda_lib, dev, case):
    """Random smooth + noisy frames: file i of the batch is byte for byte what the per-image encoder writes for frame i,
    at stored, fast and thorough levels, with and without adaptive filters, on packed and on padded strides."""
    w, h, ch, n = case
    rng = np.random.default_rng(w * 1000 + h)
    base = np.cumsum(rng.integers(-3, 4, (n, h, w, ch)), axis=2)
    frames = ((base + rng.integers(0, 256, (n, 1, 1, ch))) % 256).astype(np.uint8)
    frames[n // 2] = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)  # incompressible: stored chunks among the others
    slot = ((w * ch + 1) * h // 32768 + 1) * 32832 + 256
    for level, adaptive, pad in [(None, False, 0), (0, True, 0), (1, True, 5), (6, True, 0), (9, True, 0)]:
        opts = {} if level is None else {abi.PngCompression: level}
        want = [cuda_lib.encode(".png", f if ch > 1 else f[:, :, 0], opts) for f in frames]
        got = encode_batch(dev, frames, 1 if level is None else level, adaptive, slot, pad)
        assert got == want, (case, level)


def test_a_file_that_does_not_fit_its_slot_gets_length_zero(cuda_lib, dev):
    rng = np.random.default_rng(9)
    frames = np.zeros((3, 64, 64, 3), np.uint8)
    frames[1] = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)  # ~12 KB of noise; the flat frames are a few hundred bytes
    got = encode_batch(dev, frames, 6, True, 4096)
    assert len(got[0]) > 0 and len(got[2]) > 0 and got[1] == b""
    assert got[0] == cuda_lib.encode(".png", frames[0], {abi.PngCompression: 6})
