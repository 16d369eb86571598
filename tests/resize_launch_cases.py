"""INTER_AREA resize launches as the batches shape them: which kernel `resize_launch` (csrc/resize.cu) picks for a case
and how it bands it, a seeded catalogue of multi-image launches, and an fp64 reference of the area mean.

The batches call resize_launch with many images at once (lp_batch: a whole chunk; lp_xbatch: every run of equal
geometry in a task, every frame of a GIF task), so the general area kernel runs with 16-row bands there, while a
per-image call runs it with 1- or 2-row bands.  The catalogue reaches every kernel the launcher has, every band height,
ragged last tiles and bands, unaligned rows and images (row padding, image padding and a base offset put each image's
first staged byte on a different residue mod 16), crops at every edge, and the headline shape itself.

The mirror below restates the launcher's choices in plain Python with the tap tables of the oracle
(oracle_area_taps); tests/test_resize_launch_cases.py pins its constants on resize.cu.  It assumes the tuning
variables LP_RESIZE_RPB and LP_RESIZE_VARIANT are unset, as they are in production.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import functools

import numpy as np

from oracle import oracle

PADS = (2, 3, 4, 6, 8, 12, 16)  # pad_taps: the unrolled tap counts of resize_area_kernel
TILE = 256                      # kAreaTile: destination pixels per CTA
MAX_BAND = 16                   # kAreaMaxBand: destination rows per CTA
MAX_Y_TAPS = 16                 # kAreaMaxYTaps
SLOTS = 4                       # kAreaSlots: ring depth
NUM_SMS = 132                   # kNumSMs
SMEM_LIMIT = 200 * 1024         # above this the launcher takes the generic kernel
MAX_GRID_Z = 65535              # images per launch (gridDim.z)
DBL_EPSILON = 2.220446049250313e-16


def pad_taps(maxt: int) -> int:
    return next((p for p in PADS if maxt <= p), maxt)


@functools.lru_cache(maxsize=None)
def area_taps(ssize: int, dsize: int):
    """oracle_area_taps for one axis: (first, count, weights [dsize][maxt], maxt)."""
    cap = -(-ssize // dsize) + 2
    first, count, w = (C.c_int * dsize)(), (C.c_int * dsize)(), (C.c_float * (dsize * cap))()
    maxt = oracle.lib().oracle_area_taps(ssize, dsize, first, count, w, cap)
    if maxt < 1:
        raise RuntimeError(f"oracle_area_taps({ssize}, {dsize}) = {maxt}")
    weights = np.frombuffer(w, dtype=np.float32).reshape(dsize, cap)[:, :maxt].copy()
    return np.frombuffer(first, dtype=np.int32).copy(), np.frombuffer(count, dtype=np.int32).copy(), weights, maxt


def rows_per_band(dw: int, dh: int, n: int) -> int:
    """Destination rows per CTA: 16, halved while fewer than 4 CTAs per SM would be in flight."""
    ctas = -(-dw // TILE) * n
    rpb = MAX_BAND
    while rpb > 1 and ctas * -(-dh // rpb) < 4 * NUM_SMS:
        rpb >>= 1
    return rpb


@dataclasses.dataclass(frozen=True)
class Launch:
    kernel: str      # copy | box | area | area_sorted (the C=3, 6-tap tap-sorted variant) | generic | bilinear
    padt: int = 0    # x taps per destination pixel as laid out (area kernels)
    ypadt: int = 0   # y taps, likewise
    rpb: int = 0     # rows per band (area and area_sorted)
    why: str = ""    # generic: "x" (x taps > 16), "y" (y taps > 16) or "smem" (a staged row too wide)
    k: tuple = ()    # box: (kx, ky)

    @property
    def tma(self) -> bool:
        return self.kernel in ("area", "area_sorted")


def dispatch(C: int, cw: int, ch: int, dw: int, dh: int, n: int) -> Launch:
    """The kernel resize_launch(INTER_AREA) launches for a crop of cw x ch -> dw x dh, n images of C channels (n at
    most MAX_GRID_Z: a larger call is launched in slices of that many images)."""
    if cw == dw and ch == dh:
        return Launch("copy")
    sx, sy = 1.0 / (dw / cw), 1.0 / (dh / ch)
    ix, iy = round(sx), round(sy)  # lrint: half to even, as round()
    if sx >= 1 and sy >= 1:
        if abs(sx - ix) < DBL_EPSILON and abs(sy - iy) < DBL_EPSILON:
            return Launch("box", k=(ix, iy))
        xf, xc, _, mx = area_taps(cw, dw)
        my = area_taps(ch, dh)[3]
        padt, ypadt = pad_taps(mx), pad_taps(my)
        if padt > 16:
            return Launch("generic", padt, ypadt, why="x")
        span = max(int(xf[min(x0 + TILE, dw) - 1] + xc[min(x0 + TILE, dw) - 1] - xf[x0]) for x0 in range(0, dw, TILE))
        slot = -(-(span * C + 16 + padt * C + 8) // 128) * 128
        if 256 + MAX_BAND * MAX_Y_TAPS * 4 + SLOTS * slot > SMEM_LIMIT:
            return Launch("generic", padt, ypadt, why="smem")
        if ypadt > MAX_Y_TAPS:
            return Launch("generic", padt, ypadt, why="y")
        kernel = "area_sorted" if C == 3 and padt == 6 else "area"
        return Launch(kernel, padt, ypadt, rows_per_band(dw, dh, n))
    return Launch("bilinear")


# ------------------------------------------------------------------ cases

CONTENTS = ("noise", "extremes", "const", "ramp")


@dataclasses.dataclass(frozen=True)
class Case:
    label: str
    C: int
    sw: int
    sh: int
    crop: tuple      # (x, y, w, h) inside sw x sh
    dw: int
    dh: int
    n: int
    src_row_pad: int = 0   # bytes after each source row
    src_img_pad: int = 0   # bytes after each source image
    base: int = 0          # offset of image 0 in the (256-byte aligned) source allocation
    dst_row_pad: int = 0
    dst_img_pad: int = 0
    content: str = "noise"
    seed: int = 0

    @property
    def src_row_stride(self) -> int:
        return self.sw * self.C + self.src_row_pad

    @property
    def src_img_stride(self) -> int:
        return self.sh * self.src_row_stride + self.src_img_pad

    @property
    def dst_row_stride(self) -> int:
        return self.dw * self.C + self.dst_row_pad

    @property
    def dst_img_stride(self) -> int:
        return self.dh * self.dst_row_stride + self.dst_img_pad

    @property
    def src_bytes(self) -> int:
        return self.base + self.n * self.src_img_stride

    @property
    def dst_bytes(self) -> int:
        return self.n * self.dst_img_stride

    @property
    def downscale(self) -> bool:
        return self.crop[2] >= self.dw and self.crop[3] >= self.dh

    def launch(self) -> Launch:
        return dispatch(self.C, self.crop[2], self.crop[3], self.dw, self.dh, min(self.n, MAX_GRID_Z))

    def shape(self, h: int, w: int) -> tuple:
        return (h, w) if self.C == 1 else (h, w, self.C)

    def image(self, i: int) -> np.ndarray:
        """Source image i (sh x sw), different for every index."""
        rng = np.random.default_rng((self.seed, i))
        shp = self.shape(self.sh, self.sw)
        if self.content == "noise":
            return rng.integers(0, 256, shp, dtype=np.uint8)
        if self.content == "extremes":
            return (rng.integers(0, 2, shp, dtype=np.uint8) * 255).astype(np.uint8)
        if self.content == "const":
            return np.full(shp, (self.seed * 7 + 37 * i) % 256, dtype=np.uint8)
        if self.content == "ramp":  # neighbours differ by 0 or 1: box means land on .5
            y, x = np.mgrid[0:self.sh, 0:self.sw]
            v = ((self.seed + 29 * i) % 256 + (x + y + i) // 2) % 256
            return np.broadcast_to(v.reshape(self.sh, self.sw, *([1] if self.C > 1 else [])), shp).astype(np.uint8)
        raise ValueError(self.content)

    def images(self) -> np.ndarray:
        return np.stack([self.image(i) for i in range(self.n)])

    def pack(self, images: np.ndarray) -> np.ndarray:
        """The source allocation: the images at their strides and offset, every padding byte random (a padding byte
        read with a non-zero weight changes the output)."""
        buf = np.random.default_rng((self.seed, 1 << 20)).integers(0, 256, self.src_bytes, dtype=np.uint8)
        src_view(buf, self)[:] = images.reshape(self.n, self.sh, self.sw * self.C)
        return buf

    def seg0_residues(self) -> set:
        """Residues mod 16 of the first source byte every CTA of the area kernel stages (`seg0` in
        resize_area_kernel), over every image, band and tile; the allocation is 256-byte aligned."""
        L = self.launch()
        assert L.tma, self
        cx, cy, cw, chh = self.crop
        xf = area_taps(cw, self.dw)[0]
        yf = area_taps(chh, self.dh)[0]
        rows = (cy + yf[0:self.dh:L.rpb].astype(np.int64)) * self.src_row_stride
        cols = (cx + xf[0:self.dw:TILE].astype(np.int64)) * self.C
        imgs = self.base + np.arange(self.n, dtype=np.int64) * self.src_img_stride
        return set(np.unique((imgs[:, None, None] + rows[None, :, None] + cols[None, None, :]) % 16).tolist())

    def expected(self, images: np.ndarray) -> list:
        return [oracle.resize(im, self.dw, self.dh, crop=self.crop) for im in images]


def src_view(buf: np.ndarray, case: Case) -> np.ndarray:
    """(n, sh, sw*C) view of the images in a packed source allocation."""
    return np.lib.stride_tricks.as_strided(buf[case.base:], shape=(case.n, case.sh, case.sw * case.C),
                                           strides=(case.src_img_stride, case.src_row_stride, 1), writeable=True)


def dst_view(buf: np.ndarray, case: Case) -> np.ndarray:
    """(n, dh, dw*C) view of the images in a destination allocation."""
    return np.lib.stride_tricks.as_strided(buf, shape=(case.n, case.dh, case.dw * case.C),
                                           strides=(case.dst_img_stride, case.dst_row_stride, 1), writeable=True)


# ------------------------------------------------------------------ fp64 reference


def area_weights64(ssize: int, dsize: int) -> np.ndarray:
    """[dsize][ssize]: overlap of source cell k with [d*s/dsize, (d+1)*s/dsize), normalised to sum 1, in float64."""
    sc = ssize / dsize
    lo = np.arange(dsize, dtype=np.float64)[:, None] * sc
    k = np.arange(ssize, dtype=np.float64)[None, :]
    w = np.clip(np.minimum(lo + sc, k + 1) - np.maximum(lo, k), 0.0, None)
    return w / w.sum(axis=1, keepdims=True)


def area_mean64(images: np.ndarray, crop, dw: int, dh: int) -> np.ndarray:
    """The exact area mean of the crop of each image (n, h, w[, C]) -> (n, dh, dw, C) float64, separably."""
    cx, cy, cw, chh = crop
    x = images[:, cy:cy + chh, cx:cx + cw].astype(np.float64)
    if x.ndim == 3:
        x = x[..., None]
    n, _, _, c = x.shape
    t = area_weights64(chh, dh) @ x.reshape(n, chh, cw * c)                # (n, dh, cw*C)
    t = t.reshape(n, dh, cw, c).transpose(0, 1, 3, 2) @ area_weights64(cw, dw).T  # (n, dh, C, dw)
    return t.transpose(0, 1, 3, 2)


AREA_TOLERANCE = 0.5 + 1e-4  # a rounded fp32 chain against the exact mean: half an LSB plus the fp32 error


# ------------------------------------------------------------------ the catalogue


def _n_for_rpb(rng, dw: int, dh: int, rpb: int, extra: int = 16) -> int:
    """A number of images (2 or more) that gets `rpb` rows per band (the smallest few such counts)."""
    ns = [n for n in range(2, 4 * 4 * NUM_SMS + 1) if rows_per_band(dw, dh, n) == rpb]
    assert ns, (dw, dh, rpb)
    return int(rng.choice(ns[:extra]))


def _width_for_padt(rng, C: int, dw: int, padt: int) -> int:
    """A crop width whose x tap table pads to `padt`, at a scale that is not an integer."""
    prev = max([p for p in PADS if p < padt], default=0)
    lo, hi = int(dw * max(1.0, prev - 1.5)) + 1, int(dw * (padt + 0.5))
    ok = [cw for cw in range(lo, hi) if cw % dw and pad_taps(area_taps.__wrapped__(cw, dw)[3]) == padt]
    assert ok, f"no crop width for dw={dw} padt={padt}"
    return int(rng.choice(ok))


def _make(rng, label, C, cw, chh, dw, dh, n, *, content=None, right=None, bottom=None, pad=True, seed=None) -> Case:
    """A case with a crop of cw x chh at a random place in a larger source (or touching its right / bottom edge)."""
    ex, ey = int(rng.integers(0, 9)), int(rng.integers(0, 6))
    right = rng.random() < 0.3 if right is None else right
    bottom = rng.random() < 0.3 if bottom is None else bottom
    cx = ex if right else int(rng.integers(0, ex + 1))
    cy = ey if bottom else int(rng.integers(0, ey + 1))
    return Case(label, C, cw + ex, chh + ey, (cx, cy, cw, chh), dw, dh, n,
                src_row_pad=int(rng.integers(0, 18)) if pad else 0,
                src_img_pad=int(rng.integers(0, 300)) if pad else 0,
                base=int(rng.integers(0, 16)) if pad else 0,
                dst_row_pad=int(rng.integers(0, 10)) if pad else 0,
                dst_img_pad=int(rng.integers(0, 40)) if pad else 0,
                content=content or str(rng.choice(CONTENTS, p=[0.55, 0.15, 0.1, 0.2])),
                seed=int(rng.integers(1 << 30)) if seed is None else seed)


@functools.lru_cache(maxsize=None)
def catalogue() -> tuple:
    rng = np.random.default_rng(20261016)
    cases = []
    # every (C, padt) cell of the area kernel: 16-row bands with a ragged last band, and 1-row bands
    for C in (1, 3, 4):
        for padt in PADS:
            dw = int(rng.integers(14, 28))
            dh = int(rng.choice([17, 23, 33, 45]))
            ys = rng.uniform(1.05, 1.95) if padt % 4 == 2 else rng.uniform(1.05, 2.6)
            cases.append(_make(rng, f"cell-C{C}-t{padt}-rpb16", C, _width_for_padt(rng, C, dw, padt), int(round(dh * ys)),
                               dw, dh, _n_for_rpb(rng, dw, dh, 16)))
            dw, dh = int(rng.integers(9, 40)), int(rng.integers(5, 30))
            cases.append(_make(rng, f"cell-C{C}-t{padt}-rpb1", C, _width_for_padt(rng, C, dw, padt),
                               int(round(dh * rng.uniform(1.05, 3.5))), dw, dh, _n_for_rpb(rng, dw, dh, 1, extra=4)))
    # the band heights between, for each C (y scale in (1, 2) on half of them: most rows share a boundary row)
    for C in (1, 3, 4):
        for rpb in (2, 4, 8, 16):
            dw, dh = int(rng.integers(12, 60)), int(rng.integers(16, 70))
            padt = int(rng.choice(PADS[:5]))
            ys = rng.uniform(1.05, 1.95) if rpb % 4 == 0 else rng.uniform(2.05, 4.5)
            cases.append(_make(rng, f"band-C{C}-rpb{rpb}", C, _width_for_padt(rng, C, dw, padt), int(round(dh * ys)),
                               dw, dh, _n_for_rpb(rng, dw, dh, rpb)))
    # destination widths at the 256-pixel tile edges (the tap sort works per tile): the tap-sorted kernel and another
    for dw in (1, 255, 256, 257, 513):
        dh = int(rng.integers(3, 12))
        for C, padt in ((3, 6), (int(rng.choice([1, 4])), int(rng.choice([2, 3, 4])))):
            cw = _width_for_padt(rng, C, dw, padt) if dw > 1 else int(rng.integers(2, 15))
            cases.append(_make(rng, f"width{dw}-C{C}", C, cw, int(round(dh * rng.uniform(1.1, 2.9))) | 1, dw, dh,
                               int(rng.integers(2, 9))))
    # two tiles, the second ragged, at 16-row bands
    for C, padt in ((3, 6), (4, 4), (1, 12)):
        dw, dh = int(rng.integers(257, 300)), int(rng.choice([17, 19]))
        cases.append(_make(rng, f"tiles2-C{C}-rpb16", C, _width_for_padt(rng, C, dw, padt),
                           int(round(dh * rng.uniform(1.05, 1.6))), dw, dh, _n_for_rpb(rng, dw, dh, 16)))
    # the 6-tap 3-channel kernel over many image offsets: every residue of its first staged byte
    for k in range(3):
        dw, dh = int(rng.integers(20, 90)), int(rng.integers(8, 40))
        cases.append(_make(rng, f"residues-{k}", 3, _width_for_padt(rng, 3, dw, 6), int(round(dh * rng.uniform(1.2, 3.0))),
                           dw, dh, int(rng.integers(17, 60)), content="noise"))
    # the other kernels, each with several images and padded strides
    for C in (1, 3, 4):
        dw, dh = int(rng.integers(5, 40)), int(rng.integers(4, 30))
        cases.append(_make(rng, f"box2x2-C{C}", C, 2 * dw, 2 * dh, dw, dh, int(rng.integers(3, 40))))
        kx, ky = (3, 3) if C == 1 else (4, 2) if C == 3 else (5, 7)
        cases.append(_make(rng, f"box{kx}x{ky}-C{C}", C, kx * dw, ky * dh, dw, dh, int(rng.integers(3, 40))))
        dw, dh = int(rng.integers(3, 12)), int(rng.integers(3, 12))
        cases.append(_make(rng, f"generic-x-C{C}", C, int(round(dw * rng.uniform(17.2, 22.0))) | 1,
                           int(round(dh * rng.uniform(1.1, 3.0))), dw, dh, int(rng.integers(3, 30))))
        cases.append(_make(rng, f"generic-y-C{C}", C, int(round(dw * rng.uniform(1.1, 5.0))) | 1,
                           int(round(dh * rng.uniform(17.2, 22.0))) | 1, dw, dh, int(rng.integers(3, 30))))
        for k, (xs, ys) in enumerate(((0.4, 0.7), (0.6, 1.7), (2.3, 0.5))):
            dw, dh = int(rng.integers(8, 40)), int(rng.integers(8, 30))
            cases.append(_make(rng, f"bilinear{k}-C{C}", C, max(1, int(dw * xs)), max(1, int(dh * ys)), dw, dh,
                               int(rng.integers(3, 30))))
        dw, dh = int(rng.integers(3, 50)), int(rng.integers(3, 30))
        cases.append(_make(rng, f"copy-C{C}", C, dw, dh, dw, dh, int(rng.integers(3, 30))))
    # the headline: 1080p, the Fit crop, 256 x 256, one lp_batch chunk of distinct frames
    cases.append(Case("headline-1080p", 3, 1920, 1080, (420, 0, 1080, 1080), 256, 256, 40, content="noise", seed=1080))
    return tuple(cases)


def huge_cases() -> tuple:
    """More images than one launch takes (MAX_GRID_Z + 37), tiny, one case per kernel; distinct noise images."""
    n = MAX_GRID_Z + 37
    rng = np.random.default_rng(65572)
    mk = functools.partial(_make, rng, content="noise")
    return (mk("huge-box", 3, 6, 4, 3, 2, n),
            mk("huge-area", 3, 9, 7, 4, 3, n),
            mk("huge-generic", 1, 41, 4, 2, 3, n),
            mk("huge-bilinear", 4, 4, 3, 7, 5, n),
            mk("huge-copy", 1, 5, 3, 5, 3, n))
