"""Inputs for the baseline JPEG encoder tests, all generated from seeds, and the reference they are held to.

The reference is what OpenCV's JPEG writer makes of a frame: cv2.imencode(".jpg", img, [IMWRITE_JPEG_QUALITY, q]) over
libjpeg-turbo's defaults (4:2:0, Annex K tables, ISLOW, no restarts).  A case is (content, w, h, ch, q, seed); q None
means no JpegQuality option at all (OpenCV's default, 95).

- `edge_matrix()`: every width 1..33 against heights on both sides of the 8- and 16-row block and MCU edges, gray, BGR
  and BGRA, with the content and the quality rotating per case: every W mod 16 and H mod 16 class, so right, bottom and
  corner dummy luma blocks, partial chroma blocks and replicated edges at every offset.
- `quality_sweep()`: every quality 0..100 and the out-of-range / absent option, colour and gray.
- `launch_shapes()`: what the entropy kernel does in rounds -- MCU counts on both sides of its 256-MCU scan chunks and
  of 512, a 1080p frame of saturated noise (about 4.7 MB, over a thousand 4,096-byte stuffing rounds), a file whose
  1-padded last byte is 0xFF (so the padding is stuffed) and one whose bits fill the last byte exactly (no padding).
"""
import numpy as np

from lilliput_b200.synth import synth_image
from tests import jpeg_progressive_cases

CONTENTS = ["noise", "binary", "checker", "gradient", "flat", "sparse", "photo"]
WIDTHS = list(range(1, 34))
HEIGHTS = [1, 2, 7, 8, 9, 15, 16, 17, 24, 31, 32, 33]
CHANNELS = [1, 3, 4]
QUALITIES = [1, 10, 25, 50, 75, 85, 90, 95, 98, 100]

# zig-zag position -> natural index (T.81 Figure A.6)
ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
          21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
          61, 54, 47, 55, 62, 63]
# late zig-zag positions for the sparse content: a run of 32+ zeros before them (two or three ZRLs), 63 ends a block
# without EOB
SPARSE_POSITIONS = [63, 62, 33, 48, 63, 40, 55, 47]

# The first seeds among noise(40, 24, 3, q 75) frames whose scan ends in a 1-padded byte equal to 0xFF (so stuffed), and
# whose bit total is a multiple of 8 (no padding); tests/test_oracle_jpeg_encode.py checks both on libjpeg-turbo's files.
PAD_FF_SEED = 1466
NO_PAD_SEED = 4


def _basis(u: int, v: int) -> np.ndarray:
    """The 8x8 DCT basis image of natural coefficient (v, u) (row v, column u), peak 1."""
    k = np.arange(8)
    cu, cv = np.cos((2 * k + 1) * u * np.pi / 16), np.cos((2 * k + 1) * v * np.pi / 16)
    return cv[:, None] * cu[None, :]


def image(content: str, w: int, h: int, ch: int, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed + 7919 * w + 104729 * h + 31 * ch)
    shape = (h, w, ch) if ch > 1 else (h, w)
    if content == "noise":
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if content == "binary":  # saturated: dense 0xFF in the scan, the largest files
        return (rng.integers(0, 2, shape, dtype=np.uint8) * 255).astype(np.uint8)
    if content == "checker":
        y, x = np.mgrid[0:h, 0:w]
        if ch == 1:  # 8x8 cells of 0 / 255: luma DC differences of +-2040, category 11 where Q(DC) is 1 (q >= 98)
            return (((x // 8 + y // 8) & 1) * 255).astype(np.uint8)
        # 16x16 cells (one per MCU) of blue / yellow: Cb 255 / 0, so chroma DC differences of +-2040 too, and luma
        # differences of +-1576 (category 11)
        cell = ((x // 16 + y // 16) & 1).astype(bool)
        img = np.empty(shape, np.uint8)
        img[..., 0] = np.where(cell, 255, 0)
        img[..., 1] = np.where(cell, 0, 255)
        img[..., 2] = np.where(cell, 0, 255)
        if ch == 4:
            img[..., 3] = rng.integers(0, 256, (h, w), dtype=np.uint8)
        return img
    if content in ("gradient", "flat"):
        if content == "flat":
            return np.full(shape, int(rng.integers(0, 256)), dtype=np.uint8)
        return jpeg_progressive_cases.image(content, w, h, ch, seed)
    if content == "sparse":
        # each 8x8 block: mid-grey plus one DCT basis image of a late zig-zag position, so the quantised block holds
        # one large AC coefficient after a long zero run (ZRLs) -- at 63, no EOB.  Grey in colour, so Y carries it.
        plane = np.full((-(-h // 8) * 8, -(-w // 8) * 8), 128.0)
        for by in range(plane.shape[0] // 8):
            for bx in range(plane.shape[1] // 8):
                nat = ZIGZAG[SPARSE_POSITIONS[(bx + 3 * by + seed) % len(SPARSE_POSITIONS)]]
                amp = float(rng.uniform(40, 120)) * (1 if rng.integers(0, 2) else -1)
                plane[by * 8:by * 8 + 8, bx * 8:bx * 8 + 8] += amp * _basis(nat % 8, nat // 8)
        y = np.clip(np.round(plane[:h, :w]), 0, 255).astype(np.uint8)
        if ch == 1:
            return y
        img = np.repeat(y[:, :, None], ch, axis=2)
        if ch == 4:
            img[..., 3] = rng.integers(0, 256, (h, w), dtype=np.uint8)
        return img
    if content == "photo":
        img = synth_image(seed + 1000 * ch + 7 * w + 13 * h, w, h, ch, noise=6.0)
        return img.reshape(h, w) if ch == 1 else img.reshape(h, w, ch)
    raise ValueError(content)


def case_image(case) -> np.ndarray:
    content, w, h, ch, _, seed = case
    return image(content, w, h, ch, seed)


def edge_matrix():
    """Every (w, h, ch) of the edge grid once; content and quality rotate with the case index (7 contents against 10
    qualities, so every content meets every quality)."""
    out = []
    for i, (w, h, ch) in enumerate((w, h, ch) for h in HEIGHTS for w in WIDTHS for ch in CHANNELS):
        out.append((CONTENTS[i % len(CONTENTS)], w, h, ch, QUALITIES[(i // len(CONTENTS)) % len(QUALITIES)], i))
    return out


def quality_sweep():
    """Every quality 0..100, -5 and 101 (clamped to 0 and 100; 0 codes as 1) and no option (95), colour and gray."""
    out = []
    for q in [None, -5, *range(101), 101]:
        out.append(("photo", 45, 37, 3, q, 1))
        out.append(("photo", 37, 45, 1, q, 2))
    return out


def launch_shapes():
    out = []
    for n in (255, 256, 257, 511, 512, 513):
        out.append(("noise", 16 * n, 16, 3, 75, n))    # colour strip: n MCUs of 16x16
        out.append(("photo", 8 * n, 8, 1, 90, n))      # gray strip: n MCUs of 8x8
    out.append(("noise", 16, 16 * 257, 4, 50, 3))     # a column of 257 MCUs
    out.append(("binary", 1920, 1080, 3, 100, 0))
    out.append(("noise", 40, 24, 3, 75, PAD_FF_SEED))
    out.append(("noise", 40, 24, 3, 75, NO_PAD_SEED))
    return out


def reference(img: np.ndarray, q) -> bytes:
    """OpenCV's JPEG file of img at quality q (None: no quality option)."""
    import cv2
    ok, enc = cv2.imencode(".jpg", img, [] if q is None else [cv2.IMWRITE_JPEG_QUALITY, q])
    assert ok
    return enc.tobytes()


def encode_options(q) -> dict:
    from lilliput_b200 import abi
    return {} if q is None else {abi.JpegQuality: q}
