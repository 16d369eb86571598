"""CPU: the lossy WebP encoder core (vp8_enc_core.h) on the content and sizes that stress its bitstream limits, built
for the host with the device's scratch sizes (vp8enc::part0_scratch_bytes / token_scratch_bytes).

  * Detailed frames must encode.  The first partition (frame header + per-macroblock modes) costs 1-28 bytes per
    macroblock; its scratch is a worst-case bound, clipped at the format's 2^19-byte limit, beyond which the frame is
    coded again with 16x16 prediction only.
  * libwebp (OpenCV's WebP codec) decodes every stream to the pixels of the device's decoder core.
  * Token partitions keep at least half of their 2 KiB-per-macroblock scratch free on adversarial content.
  * The bound covers the exact worst case, computed from the format's probability tables.
"""
import ctypes

import cv2  # noqa: F401  libwebp_decode's libwebp: a missing decoder fails these tests, it does not skip them
import numpy as np
import pytest

from lilliput_b200.synth import synth_image
from tests.webp_util import libwebp_decode, riff, vp8_cpu_decode, vp8_cpu_encode, vp8_cpu_lib, vp8_partition_sizes

PART0_LIMIT = 1 << 19


@pytest.fixture(scope="module")
def cpu():
    return vp8_cpu_lib()


def scratch_bytes(cpu, w, h):
    sizes = (ctypes.c_size_t * 2)()
    cpu.vp8_cpu_scratch_bytes(w, h, sizes)
    return sizes[0], sizes[1]


def uniform_noise(seed, w, h, ch=3):
    return np.random.default_rng(seed).integers(0, 256, (h, w, ch), dtype=np.uint8)


def alternating_rows(seed, w, h, flat_first=True):
    """Macroblock rows alternately flat grey and uniform noise."""
    img = uniform_noise(seed, w, h)
    for r in range(0 if flat_first else 16, h, 32):
        img[r:r + 16] = 128
    return img


# (name, frame maker, quality): the frames the first partition's old scratch (2 B per macroblock + 4 KiB) refused,
# and their neighbours
CASES = [
    ("synth1280x720", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 90),
    ("synth1280x720", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 95),
    ("synth1280x720", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 99),
    ("synth1280x720", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 100),
    ("alt_rows1024x512", lambda: alternating_rows(3, 1024, 512), 50),
    ("noise256", lambda: uniform_noise(4, 256, 256), 50),
    ("noise768", lambda: uniform_noise(5, 768, 768), 85),
    ("noise_odd_rows", lambda: alternating_rows(6, 512, 512, flat_first=True), 100),
    ("noise_even_rows", lambda: alternating_rows(7, 512, 512, flat_first=False), 100),
    ("checker1px", lambda: np.kron((np.indices((640, 640)).sum(0) & 1)[:, :, None] * 255, np.ones(3)).astype(np.uint8), 100),
]


@pytest.mark.parametrize("name,make,quality", CASES, ids=[f"{c[0]}-q{c[2]}" for c in CASES])
def test_detailed_frames_encode_and_decode_identically_with_libwebp(cpu, name, make, quality):
    img = make()
    h, w = img.shape[:2]
    payload = vp8_cpu_encode(cpu, img, quality)  # asserts the encoder wrote a stream
    # ... with 4x4 prediction: these first partitions are far below the format's limit, no 16x16-only retry is due
    assert payload == vp8_cpu_encode(cpu, img, quality, try_i4=1)
    p0, parts = vp8_partition_sizes(payload)
    assert p0 <= scratch_bytes(cpu, w, h)[0] and p0 < PART0_LIMIT
    mine = vp8_cpu_decode(cpu, payload)
    assert mine.shape == img.shape
    assert np.array_equal(libwebp_decode(riff([(b"VP8 ", payload)])), mine), name


@pytest.mark.parametrize("name,make,quality", CASES, ids=[f"{c[0]}-q{c[2]}" for c in CASES])
def test_token_partitions_keep_half_their_scratch_free(cpu, name, make, quality):
    """Token partition q holds macroblock rows q, q + n, ...: 2048 bytes of scratch per macroblock.  The worst content
    (noise in the rows the statistics pass does not sample, so the probabilities are fitted to flat rows) stays under
    half of that."""
    img = make()
    h, w = img.shape[:2]
    mb_w, mb_h = (w + 15) // 16, (h + 15) // 16
    payload = vp8_cpu_encode(cpu, img, quality)
    _, parts = vp8_partition_sizes(payload)
    n = len(parts)
    assert sum(parts) > 0
    for q, size in enumerate(parts):
        rows = (mb_h - q + n - 1) // n
        assert size <= rows * mb_w * 2048 // 2, (name, q, size, rows * mb_w)


def test_first_partition_bound_covers_the_exact_worst_case(cpu):
    """part0_scratch_bytes is a bound from constants; vp8_cpu_part0_worst_bits walks the format's fixed probabilities
    (every context of the sixteen sub-block modes, the skip flag at any probability, every coefficient-probability
    update) for the exact worst.  The scratch must hold that for every frame size, up to the format's limit."""
    header, per_mb = ctypes.c_double(), ctypes.c_double()
    cpu.vp8_cpu_part0_worst_bits(ctypes.byref(header), ctypes.byref(per_mb))
    assert 1000 * 8 < header.value < 9542 * 8           # 29 + 1056 * 9 + 9 booleans, < 8 bits each
    assert 150 < per_mb.value < 1216                    # 1 + 1 + 16 * 9 + 3 booleans, < 8 bits each
    for w, h in [(1, 1), (16, 16), (97, 61), (256, 256), (1280, 720), (1920, 1080), (2000, 2000), (4096, 4096),
                 (16383, 16383), (16383, 16), (16, 16383)]:
        nmb = ((w + 15) // 16) * ((h + 15) // 16)
        worst = int(np.ceil((header.value + nmb * per_mb.value) / 8)) + 4  # + the coder's flush
        part0, tokens = scratch_bytes(cpu, w, h)
        assert part0 >= min(worst, PART0_LIMIT - 1), (w, h, part0, worst)
        assert part0 <= PART0_LIMIT - 1
        assert tokens >= nmb * 2048 + 8 * 64


def test_first_partition_beyond_the_format_limit_is_coded_with_16x16_prediction(cpu):
    """4096 x 4096 uniform noise with 4x4 prediction needs ~9 bytes of modes per macroblock: 570 KB, over the 19-bit
    size field.  The encoder codes it again with 16x16 prediction only (< 1 byte per macroblock)."""
    img = uniform_noise(8, 4096, 4096)
    out = np.zeros(4096 * 4096 * 4 + 65536, np.uint8)
    cpu.vp8_cpu_encode_i4.restype = ctypes.c_long
    n = cpu.vp8_cpu_encode_i4(img.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(4096 * 3), 4096, 4096, 3, 75, -1, 1,
                              out.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(out.size))
    assert n == -1  # with 4x4 prediction: the first partition outgrows the format
    payload = vp8_cpu_encode(cpu, img, 75)
    assert payload == vp8_cpu_encode(cpu, img, 75, try_i4=0)
    p0, _ = vp8_partition_sizes(payload)
    assert p0 < 64 * 1024
    assert np.array_equal(libwebp_decode(riff([(b"VP8 ", payload)])), vp8_cpu_decode(cpu, payload))
