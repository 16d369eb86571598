"""JPEG decode cases that reach every tile edge of jpeg_idct_color_kernel, shared by the CPU reference check and the
GPU tests.

The kernel runs one CTA per tile of an image (lilliput_b200/csrc/jpeg_decode.cu):
  spans    as many MCU columns as fit in the shared-memory budget, evened out over the region of interest;
           neighbouring spans rebuild each other's halo column;
  bands    four bands of MCU rows; a band IDCTs the row above it into a three-row chroma ring;
  windows  the batch path decodes only the Fit crop window plus a chroma margin, into a strided frame.
`window()` restates jpeg_item_set_window + tile_layout so that the geometries below can be picked from it, and
`check_coverage()` asserts that the list reaches every such edge in every sampling layout.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from lilliput_b200.synth import synth_image

# Dynamic shared memory of one jpeg_idct_color_kernel CTA (kTileSmemBytes in jpeg_decode.cu).  The span widths, and so
# the geometries that reach two and three spans, follow from it.
TILE_SMEM_BYTES = 24 * 1024

# name -> (cv2.IMWRITE_JPEG_SAMPLING_FACTOR, (h, v) of each component); gray is a one-component file
SAMPLINGS = {
    "444": (0x111111, ((1, 1), (1, 1), (1, 1))),
    "422": (0x211111, ((2, 1), (1, 1), (1, 1))),
    "420": (0x221111, ((2, 2), (1, 1), (1, 1))),
    "411": (0x411111, ((4, 1), (1, 1), (1, 1))),
    "440": (0x121111, ((1, 2), (1, 1), (1, 1))),
    "gray": (None, ((1, 1),)),
}
COLOR_SAMPLINGS = ("444", "422", "420", "411", "440")
CONTENTS = ("noise", "smooth", "blocks")
# plain = Huffman tables of Annex K, optimized = per-file tables, rstN = a restart interval of N MCUs, rstrow = one
# MCU row; per image, progressive and restart files go through the multi-scan decoder
MODES = ("plain", "optimized", "rst1", "rst3", "rstrow", "progressive")


def mcu_size(sampling: str):
    comps = SAMPLINGS[sampling][1]
    return 8 * max(h for h, _ in comps), 8 * max(v for _, v in comps)


def tile_layout_bytes(sampling: str, cols: int) -> int:
    """tile_layout(): shared memory of a span `cols` MCU columns wide.  Every component keeps rows of cols + 2 MCU
    columns; those upsampled with the rows above and below keep three MCU rows, the others one."""
    comps = SAMPLINGS[sampling][1]
    maxh, maxv = max(h for h, _ in comps), max(v for _, v in comps)
    total = 0
    for h, v in comps:
        hr, vr = maxh // h, maxv // v
        rows = (3 if vr == 2 and hr <= 2 else 1) * 8 * v
        total += (((cols + 2) * 8 * h + 15) & ~15) * rows
    return total


@dataclass(frozen=True)
class Window:
    x0: int
    y0: int
    w: int
    h: int
    row_stride: int  # bytes between rows of the decoded frame
    roi_mcx: int
    roi_mcy: int
    tile_mcx: int
    tiles_x: int
    bands: int

    @property
    def uneven_last_span(self) -> bool:
        return self.roi_mcx % self.tile_mcx != 0


def window(sampling: str, W: int, H: int, x0: int, y0: int, x1: int, y1: int, align16: bool) -> Window:
    """jpeg_item_set_window(): the decoded pixel window [x0, x1) x [y0, y1), its row stride, and the tiles of its
    region of interest (the window plus one chroma sample on every side, in whole MCUs)."""
    mw, mh = mcu_size(sampling)
    maxh, maxv = mw // 8, mh // 8
    x0, y0, x1, y1 = max(x0, 0), max(y0, 0), min(x1, W), min(y1, H)
    if align16:
        x0 &= ~15
        x1 = min((x1 + 15) & ~15, W)
    ch = 1 if sampling == "gray" else 3
    stride = W * ch if (x0 == 0 and x1 == W) else ((x1 - x0) * ch + 15) // 16 * 16
    px0, px1 = max(x0 - 2 * maxh, 0), min(x1 - 1 + 2 * maxh, W - 1)
    py0, py1 = max(y0 - 2 * maxv, 0), min(y1 - 1 + 2 * maxv, H - 1)
    mcx = px1 // mw - px0 // mw + 1
    mcy = py1 // mh - py0 // mh + 1
    span = mcx
    while span > 1 and tile_layout_bytes(sampling, span) > TILE_SMEM_BYTES:
        span -= 1
    nspans = -(-mcx // span)
    tile_mcx = -(-mcx // nspans)
    tile_mcy = (mcy + 3) // 4
    return Window(x0, y0, x1 - x0, y1 - y0, stride, mcx, mcy, tile_mcx, -(-mcx // tile_mcx), -(-mcy // tile_mcy))


def full_window(sampling: str, W: int, H: int) -> Window:
    """What the per-image decoder (opencv_decoder_read_data) decodes: the whole image, rows packed."""
    return window(sampling, W, H, 0, 0, W, H, False)


def max_span(sampling: str) -> int:
    """Widest span in MCU columns."""
    span = 1
    while tile_layout_bytes(sampling, span + 1) <= TILE_SMEM_BYTES:
        span += 1
    return span


# ---------------------------------------------------------------------------------------------------- per-image cases

@dataclass(frozen=True)
class Case:
    sampling: str
    w: int
    h: int
    content: str
    mode: str
    quality: int

    @property
    def label(self) -> str:
        return f"{self.sampling}-{self.w}x{self.h}-{self.content}-{self.mode}-q{self.quality}"


def _geometries(sampling: str):
    """(w, h, mode) per sampling: widths 1 to 4, one span with widths on and off the 16-pixel grid, two spans, three
    or more with an uneven last span; heights of 1, 2, 3, 4, 5 and 9 or more MCU rows.  Restart and progressive files
    are among the multi-span ones."""
    mw, mh = mcu_size(sampling)
    span = max_span(sampling)
    # three or more spans, uneven: the smallest width past two spans whose last span comes out short
    mcx3 = 2 * span + 1
    while -(-mcx3 // 3) * 3 == mcx3:
        mcx3 += 1
    return [
        (1, 1, "plain"),
        (2, 3 * mh - 5, "rst1"),
        (3, mh + 1, "progressive"),
        (4, 5 * mh, "optimized"),
        (4, 9 * mh + 3, "rst3"),
        (96, 4 * mh - 1, "plain"),                       # one span, a multiple of 16
        (37, 11 * mh - 2, "rstrow"),                     # one span, off the 16-pixel grid
        ((span * mw + mw + 15) // 16 * 16, 5 * mh, "plain"),   # two spans, a multiple of 16
        (span * mw + 2 * mw + 5, 2 * mh, "rstrow"),      # two spans, off the grid
        (span * mw + 3 * mw + 16, 9 * mh + 1, "progressive"),  # two spans, nine bands' worth of rows
        (mcx3 * mw - 3, 3 * mh - 2, "rst3"),             # three spans, uneven
        (mcx3 * mw + 2 * mw, 8, "optimized"),
        ((mcx3 * mw) // 16 * 16, 2, "progressive"),
    ]


def cases() -> list[Case]:
    rng = np.random.default_rng(20261015)
    out = []
    for s in SAMPLINGS:
        for k, (w, h, mode) in enumerate(_geometries(s)):
            out.append(Case(s, w, max(h, 1), CONTENTS[k % 3], mode, int(rng.integers(1, 101))))
    # the 4:2:0 headline sampling: the 16-pixel colour path over several spans and many bands, restart and not
    out.append(Case("420", 1280, 150, "smooth", "plain", 90))
    out.append(Case("420", 1280, 150, "noise", "rstrow", 75))
    out.append(Case("420", 1600, 33, "blocks", "progressive", 85))
    return out


def narrow_cases() -> list[Case]:
    """Every sampling at widths 1 to 8 and heights 1 to 40: where chroma upsampling switches filters."""
    rng = np.random.default_rng(8)
    out = []
    for s in SAMPLINGS:
        for w in range(1, 9):
            for h in range(1, 41):
                mode = MODES[(w + h) % len(MODES)]
                out.append(Case(s, w, h, CONTENTS[(w * 3 + h) % 3], mode, int(rng.integers(1, 101))))
    return out


def image(content: str, w: int, h: int, ch: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if content == "noise":  # white noise: every tap matters
        img = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)
    elif content == "smooth":  # smooth field + edges
        img = synth_image(seed, w, h, ch, noise=3.0).reshape(h, w, ch)
    else:  # saturated blocks: rounding at 0 / 255
        img = (rng.integers(0, 2, (h // 3 + 1, w // 3 + 1, ch), dtype=np.uint8) * 255).repeat(3, 0).repeat(3, 1)[:h, :w]
    return np.ascontiguousarray(img if ch > 1 else img.reshape(h, w))


def mcus(case: Case) -> int:
    mw, mh = mcu_size(case.sampling)
    return -(-case.w // mw) * -(-case.h // mh)


def restart_interval(case: Case) -> int:
    """MCUs per restart interval of an rst case."""
    return -(-case.w // mcu_size(case.sampling)[0]) if case.mode == "rstrow" else int(case.mode[3:])


def encode(case: Case, seed: int = 0) -> bytes:
    import cv2

    sf, _ = SAMPLINGS[case.sampling]
    img = image(case.content, case.w, case.h, 1 if sf is None else 3, seed + 7919 * case.w + 104729 * case.h)
    opts = [cv2.IMWRITE_JPEG_QUALITY, case.quality]
    if sf is not None:
        opts += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf]
    if case.mode == "optimized":
        opts += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    elif case.mode == "progressive":
        opts += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    elif case.mode.startswith("rst"):
        opts += [cv2.IMWRITE_JPEG_RST_INTERVAL, restart_interval(case)]
    ok, enc = cv2.imencode(".jpg", img, opts)
    assert ok, case
    return enc.tobytes()


def check_coverage(case_list: list[Case]) -> None:
    """Every sampling reaches one, two and three or more spans (one of them with a short last span), 1, 2, 3, 4, 5
    and 9 or more MCU rows (at 5 the fourth band is empty), widths on and off the 16-pixel grid (the 4:2:0 16-pixel
    colour path on and off), widths 1 to 4, and multi-span restart and progressive files."""
    for s in SAMPLINGS:
        mine = [c for c in case_list if c.sampling == s]
        wins = [(c, full_window(s, c.w, c.h)) for c in mine]
        tiles = {min(wn.tiles_x, 3) for _, wn in wins}
        assert tiles == {1, 2, 3}, (s, tiles)
        assert any(wn.tiles_x >= 3 and wn.uneven_last_span for _, wn in wins), s
        rows = {wn.roi_mcy for _, wn in wins}
        assert {1, 2, 3, 4, 5} <= rows and max(rows) >= 9, (s, sorted(rows))
        assert any(wn.roi_mcy == 5 and wn.bands == 3 for _, wn in wins), s
        assert any(c.w % 16 == 0 for c in mine) and any(c.w % 16 for c in mine), s
        assert {1, 2, 3, 4} <= {c.w for c in mine}, s
        multi = {c.mode for c, wn in wins if wn.tiles_x >= 2}
        assert {"plain", "progressive"} <= multi and any(m.startswith("rst") for m in multi), (s, multi)
    fast = [c for c in case_list if c.sampling == "420" and c.w % 16 == 0 and full_window("420", c.w, c.h).tiles_x >= 2]
    assert fast, "no multi-span 4:2:0 frame takes the 16-pixel colour path"


# ---------------------------------------------------------------------------------------------------- batch windows

# (source w, source h, requested w, requested h, ImageOpsFit / ImageOpsResize): what each one reaches
BATCH_GEOMETRIES = [
    (1010, 200, 64, 64, "fit"),      # wide source cut left and right, crop_x = 405 off the 16-pixel grid
    (240, 900, 50, 50, "fit"),       # tall source cut top and bottom: the window starts mid-image
    (230, 200, 64, 64, "fit"),       # the window starts at column 0 but stops short of the right edge
    (203, 200, 64, 64, "fit"),       # the window reaches the right edge of a width off the grid: whole rows
    (96, 64, 96, 64, "fit"),         # the same-size copy
    (333, 217, 100, 60, "resize"),   # ImageOpsResize: the full frame, rows packed
    (1600, 700, 64, 64, "fit"),      # multi-span windows on the 16-pixel grid (the 4:2:0 16-pixel path)
    (4600, 40, 1000, 10, "fit"),     # windows of two or more spans in every sampling
]


def batch_window(sampling: str, W: int, H: int, crop) -> Window:
    """The window the batch path decodes for the Fit crop (x, y, w, h): the crop, its x range rounded out to 16
    pixels (kernels.cuh: align16)."""
    cx, cy, cw, chh = crop
    return window(sampling, W, H, cx, cy, cx + cw, cy + chh, True)
