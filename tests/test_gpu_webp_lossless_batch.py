"""GPU: the batched lossless WebP encoder (csrc/webp_encode.cu, webp_encode_lossless_batch through
lp_webp_lossless_encode_batch_dev): n device frames of one geometry -> n "VP8L" payloads.

Every payload equals vp8l_enc_core.h run on the host (vp8l_cpu_encode: the same stream head, one pixel after another
through the bit writer) byte for byte, and libwebp decodes it, wrapped as a still, back to the frame exactly.  The
frames cover what the tiles, the per-frame scan and the word-OR packing meet: tile edges in mid-row, one frame over many
tiles, thousands of one-tile frames, padded strides, zero pixel bits, codes at the 15-bit limit and pixels whose bits
span three words."""
import ctypes as C

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.webp_util import chunks_of, libwebp_decode, riff, vp8_cpu_lib, vp8l_cpu_encode

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_lib):
    l = cuda_lib.l
    l.lp_dev_alloc.restype = C.c_void_p
    l.lp_dev_alloc.argtypes = [C.c_size_t]
    l.lp_dev_free.argtypes = [C.c_void_p]
    l.lp_memcpy_h2d.restype = C.c_int
    l.lp_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    l.lp_webp_lossless_encode_batch_dev.restype = C.c_int
    l.lp_webp_lossless_encode_batch_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int,
                                                    C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    return l


@pytest.fixture(scope="module")
def cpu():
    return vp8_cpu_lib()


def encode_batch(l, frames, row_pad=0, img_pad=0, part_bytes=0):
    """frames: [n, h, w, c] -> the n payloads, the frames laid out on the device with padded rows and images."""
    frames = np.ascontiguousarray(frames, np.uint8)
    n, h, w, c = frames.shape
    row = w * c + row_pad
    img = h * row + img_pad
    host = np.zeros(n * img + 16, np.uint8)
    for k in range(n):
        view = host[k * img:k * img + h * row].reshape(h, row)
        view[:, :w * c] = frames[k].reshape(h, w * c)
        view[:, w * c:] = 0xA5  # padding the encoder must not read
    d = l.lp_dev_alloc(host.size)
    assert d
    try:
        assert l.lp_memcpy_h2d(d, host.ctypes.data, host.size) == 0
        cap = n * (w * h * 8 + 4096)
        out = np.empty(cap, np.uint8)
        offs, lens = (C.c_size_t * n)(), (C.c_size_t * n)()
        rc = l.lp_webp_lossless_encode_batch_dev(d, img, row, w, h, c, n, part_bytes, out.ctypes.data, cap, offs, lens)
        assert rc == 0, rc
        return [out[offs[k]:offs[k] + lens[k]].tobytes() for k in range(n)]
    finally:
        l.lp_dev_free(d)


def check(l, cpu, frames, decode=True, **kw):
    got = encode_batch(l, frames, **kw)
    for k, f in enumerate(frames):
        assert got[k] == vp8l_cpu_encode(cpu, f), f"frame {k} of {len(frames)} ({f.shape}) differs from vp8l_enc_core.h"
        if decode:
            assert np.array_equal(libwebp_decode(riff([(b"VP8L", got[k])])), f), f"frame {k}: libwebp decodes other pixels"
    return got


def residual_frame(res_g, res_r, res_b, res_a, width):
    """A BGRA frame of one row whose VP8L residuals (subtract-green, then the left prediction of row 0) are the given
    sequences, continued over further rows of the same pixels."""
    g = np.cumsum(res_g) & 255
    r = (np.cumsum(res_r) + g) & 255
    b = (np.cumsum(res_b) + g) & 255
    a = (np.cumsum(res_a) + 255) & 255  # (the first pixel is predicted from 0xff000000)
    row = np.stack([b, g, r, a], axis=-1).astype(np.uint8)[:width]
    return row[None]


def fibonacci_symbols(n_symbols, seed):
    """A sequence in which symbol k occurs F(k) times (Fibonacci): the deepest Huffman tree there is for its length, so
    plain Huffman gives codes over 15 bits and build_lengths has to flatten them."""
    f = [1, 1]
    while len(f) < n_symbols:
        f.append(f[-1] + f[-2])
    syms = np.concatenate([np.full(c, s, np.int64) for s, c in enumerate(f)])
    return syms[np.random.default_rng(seed).permutation(syms.size)]


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("w,h", [(1, 1), (1, 37), (37, 1), (2047, 1), (2049, 3), (100, 41), (333, 211), (3000, 7)],
                         ids=lambda v: str(v))
def test_geometries(dev, cpu, w, h, ch):
    """One frame and three frames per call; widths that put tile edges (2048 pixels) mid-row."""
    frames = np.stack([synth_image(10 + k, w, h, ch, noise=8.0) for k in range(3)])
    check(dev, cpu, frames[:1])
    check(dev, cpu, frames)


def test_one_frame_over_many_tiles(dev, cpu):
    """3840 x 2160 RGBA with n = 1: over 4000 tiles in one frame (the per-image path's largest calls look like this)."""
    img = synth_image(21, 3840, 2160, 4, noise=10.0)
    check(dev, cpu, img[None])


def test_thousands_of_small_frames(dev, cpu):
    """n = 2000 frames of 13 x 9, each a tile of its own, every one with its own codes."""
    frames = np.stack([synth_image(1000 + k, 13, 9, 4, noise=float(k % 50)) for k in range(2000)])
    frames[::7, :, :, 3] = 255
    check(dev, cpu, frames, decode=False)
    for k in range(0, 2000, 97):
        assert np.array_equal(libwebp_decode(riff([(b"VP8L", vp8l_cpu_encode(cpu, frames[k]))])), frames[k])


def test_mixed_content_in_one_call(dev, cpu):
    w, h = 160, 120
    flat = np.zeros((h, w, 4), np.uint8)
    flat[:] = (30, 60, 90, 255)
    noise = np.random.default_rng(3).integers(0, 256, (h, w, 4), dtype=np.uint8)
    grad = np.zeros((h, w, 4), np.uint8)
    grad[..., 0] = np.arange(w)[None, :]
    grad[..., 1] = np.arange(h)[:, None]
    grad[..., 2] = 200
    grad[..., 3] = (np.arange(w)[None, :] * 2) & 255
    art = synth_image(5, w, h, 4, noise=0.0)
    frames = np.stack([flat, noise, grad, art, noise[::-1].copy(), flat])
    check(dev, cpu, frames)


@pytest.mark.parametrize("row_pad,img_pad", [(1, 0), (13, 0), (0, 7), (29, 4099)])
def test_padded_strides(dev, cpu, row_pad, img_pad):
    for ch in (3, 4):
        frames = np.stack([synth_image(40 + k, 71, 23, ch) for k in range(4)])
        check(dev, cpu, frames, row_pad=row_pad, img_pad=img_pad)


def test_single_colour_frames_have_no_pixel_bits(dev, cpu):
    """Opaque black: every residual, the first pixel's included, is 0, so all four codes have one symbol and the
    payload is the head alone, whatever the size.  Another flat colour differs from its prediction at the first pixel."""
    lengths = []
    for w, h in [(1, 1), (64, 64), (2048, 3), (1000, 1000)]:
        for ch in (3, 4):
            img = np.zeros((h, w, ch), np.uint8)
            if ch == 4:
                img[..., 3] = 255
            (p,) = check(dev, cpu, img[None])
            lengths.append(len(p))
        img = np.zeros((h, w, 4), np.uint8)
        img[:] = (9, 200, 77, 255)
        check(dev, cpu, img[None])
    assert len(set(lengths)) == 1, lengths


def test_constant_alpha(dev, cpu):
    img = synth_image(50, 300, 200, 4, noise=12.0)
    img[..., 3] = 255
    check(dev, cpu, np.stack([img, img[::-1].copy()]))


def test_code_length_limit(dev, cpu):
    """Fibonacci-distributed residuals in every channel: Huffman depths past 15, flattened by build_lengths."""
    g = fibonacci_symbols(19, 1)  # F(1..19) sums to 10945 pixels: depth 18 before the limit
    n = g.size
    perm = np.random.default_rng(2).permutation(256)
    frame = residual_frame(g, perm[g], (g * 7) & 255, (g * 13) & 255, n)
    check(dev, cpu, frame[None])
    # the same residuals in three rows of a narrower frame (rows after the first are predicted from above as well)
    check(dev, cpu, frame[:, :3000].reshape(1, 1, 3000, 4).repeat(3, axis=1))


def test_pixels_across_three_words(dev, cpu):
    """The rarest symbol of every channel at the same pixels: those pixels cost ~60 bits, so most of them start far
    enough into a word to touch three.  Eight rotations of the sequence move them to other bit positions."""
    g = fibonacci_symbols(19, 5)
    frames = []
    for k in range(8):
        s = np.roll(g, 37 * k)
        frames.append(residual_frame(s, s, s, s, s.size)[0])
    check(dev, cpu, np.stack(frames)[:, None])


def test_parts_equal_one_call(dev, cpu):
    """A call forced into parts (a bound of one byte: a part per frame; a few frames per part) gives the same bytes."""
    frames = np.stack([synth_image(70 + k, 90, 70, 4, noise=float(3 * k)) for k in range(12)])
    whole = check(dev, cpu, frames, decode=False)
    for bound in (1, 20000, 60000):
        assert encode_batch(dev, frames, part_bytes=bound) == whole, bound


def test_per_image_encoder_is_the_batch(cuda_lib, dev):
    """webp_encoder_write's lossless branch is this encoder with n = 1: the file's only chunk is the hook's payload."""
    for seed, w, h, ch in [(80, 200, 120, 3), (81, 97, 61, 4), (82, 1, 1, 4), (83, 1920, 1080, 4)]:
        img = synth_image(seed, w, h, ch, noise=9.0)
        data = cuda_lib.encode(".webp", img, {abi.WebpQuality: 101})
        assert chunks_of(data) == [(b"VP8L", encode_batch(dev, img[None])[0])]
