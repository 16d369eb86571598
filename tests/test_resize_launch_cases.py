"""CPU: the resize launch catalogue (tests/resize_launch_cases.py) reaches every launch shape it is meant to, its mirror
of the launcher is pinned on csrc/resize.cu, and the oracle it is checked against agrees with the exact area mean.

tests/test_gpu_resize_launches.py runs the same catalogue on the device."""
import os
import re

import numpy as np
import pytest

from tests import resize_launch_cases as rlc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = rlc.catalogue()
DOWN = [c for c in CASES if c.launch().kernel != "bilinear"]


def _src(name):
    with open(os.path.join(ROOT, "lilliput_b200", "csrc", name)) as f:
        return f.read()


def test_mirror_constants_are_the_launchers():
    src = _src("resize.cu")
    opts = re.search(r"const int opts\[\] = \{([^}]*)\}", src).group(1)
    assert tuple(int(v) for v in opts.split(",")) == rlc.PADS
    for name, want in (("kAreaTile", rlc.TILE), ("kAreaSlots", rlc.SLOTS), ("kAreaMaxBand", rlc.MAX_BAND),
                       ("kAreaMaxYTaps", rlc.MAX_Y_TAPS), ("kMaxImagesPerLaunch", rlc.MAX_GRID_Z)):
        assert int(re.search(rf"constexpr int {name} = (\d+);", src).group(1)) == want, name
    assert int(re.search(r"constexpr int kNumSMs = (\d+);", _src("common.cuh")).group(1)) == rlc.NUM_SMS
    assert "area_smem_bytes(p.slot_bytes) > 200 * 1024" in src
    assert "while (rpb > 1 && ctas_per_row_group * ceil_div(a.dst_h, rpb) < 4L * kNumSMs) rpb >>= 1;" in src
    # one unrolled kernel per tap count, and the tap-sorted one is the default for 3 channels, 6 taps
    cases = re.search(r"switch \(padt\) \{(.*?)\}", src, re.S).group(1)
    assert tuple(int(v) for v in re.findall(r"case (\d+): return launch_area<C, \1,", cases)) == rlc.PADS
    assert "default: return launch_area<3, 6, 2, 2, true>(p, n, st);" in src


def _coverage():
    """Every cell the catalogue must reach -> whether it does."""
    cells = {}
    tma = [(c, c.launch()) for c in CASES if c.launch().tma]
    for C in (1, 3, 4):
        for padt in rlc.PADS:
            cells[f"C={C} padt={padt} rpb=16 ragged last band"] = any(
                c.C == C and L.padt == padt and L.rpb == 16 and c.dh % 16 for c, L in tma)
            cells[f"C={C} padt={padt} rpb=1"] = any(c.C == C and L.padt == padt and L.rpb == 1 for c, L in tma)
        for rpb in (1, 2, 4, 8, 16):
            cells[f"C={C} rpb={rpb}"] = any(c.C == C and L.rpb == rpb for c, L in tma)
        cells[f"C={C} y scale in (1, 2) with bands of 2+ rows"] = any(
            c.C == C and L.rpb > 1 and 1 < c.crop[3] / c.dh < 2 for c, L in tma)
        cells[f"C={C} odd source row stride"] = any(c.C == C and c.src_row_stride % 2 for c, L in tma)
    cells["C=3 padt=6 is the tap-sorted kernel"] = all(L.kernel == "area_sorted" for c, L in tma if c.C == 3 and L.padt == 6)
    for dw in (1, 255, 256, 257, 513):
        cells[f"dw={dw}"] = any(c.dw == dw for c, L in tma)
        if dw > 1:
            cells[f"dw={dw} tap-sorted"] = any(c.dw == dw and L.kernel == "area_sorted" for c, L in tma)
    cells["two tiles at rpb=16"] = any(c.dw > rlc.TILE and L.rpb == 16 for c, L in tma)
    residues = set()
    for c, L in tma:
        if L.kernel == "area_sorted":
            residues |= c.seg0_residues()
    for r in range(16):
        cells[f"tap-sorted kernel, seg0 % 16 == {r}"] = r in residues
    cells["crop at the right edge"] = any(c.crop[0] > 0 and c.crop[0] + c.crop[2] == c.sw for c, L in tma)
    cells["crop at the bottom edge"] = any(c.crop[1] > 0 and c.crop[1] + c.crop[3] == c.sh for c, L in tma)
    padded = [(c, c.launch()) for c in CASES if c.n > 1 and c.src_row_pad and c.src_img_pad and c.dst_row_pad]
    cells["box 2x2"] = any(L.kernel == "box" and L.k == (2, 2) for c, L in padded)
    cells["box k x k"] = any(L.kernel == "box" and L.k != (2, 2) for c, L in padded)
    cells["generic by x taps"] = any(L.kernel == "generic" and L.why == "x" for c, L in padded)
    cells["generic by y taps"] = any(L.kernel == "generic" and L.why == "y" for c, L in padded)
    cells["area-mode bilinear"] = any(L.kernel == "bilinear" for c, L in padded)
    cells["same-size copy"] = any(L.kernel == "copy" for c, L in padded)
    cells["headline 1920x1080 crop (420, 0, 1080, 1080) -> 256x256, C=3, n=40, rpb=16"] = any(
        (c.C, c.sw, c.sh, c.crop, c.dw, c.dh, c.n) == (3, 1920, 1080, (420, 0, 1080, 1080), 256, 256, 40)
        and L.kernel == "area_sorted" and L.rpb == 16 and c.content == "noise" for c, L in tma)
    cells["headline gets rpb=16 from n=33"] = rlc.rows_per_band(256, 256, 33) == 16 > rlc.rows_per_band(256, 256, 32)
    huge = {h.launch().kernel for h in rlc.huge_cases() if h.n > rlc.MAX_GRID_Z}
    for k in ("box", "area", "generic", "bilinear", "copy"):
        cells[f"more than {rlc.MAX_GRID_Z} images: {k}"] = k in huge
    return cells


def test_catalogue_reaches_every_cell():
    cells = _coverage()
    assert len(cells) > 80
    assert [k for k, v in cells.items() if not v] == []


def test_catalogue_stays_small():
    assert len({c.label for c in CASES}) == len(CASES)
    assert sum(c.src_bytes + c.dst_bytes for c in CASES) < 512 << 20
    assert all(c.src_bytes < 256 << 20 for c in CASES + rlc.huge_cases())


def _axes():
    ax = set()
    for c in CASES:
        L = c.launch()
        if L.tma or L.kernel == "generic":
            ax |= {(c.crop[2], c.dw), (c.crop[3], c.dh)}
    return sorted(ax)


@pytest.mark.parametrize("ssize,dsize", _axes())
def test_tap_tables_are_the_area_overlaps(ssize, dsize):
    """oracle_area_taps (which the mirror pads and the device table restates) against the overlaps in fp64: the taps
    cover the cells that overlap the destination interval by more than 1e-3 (OpenCV drops slivers), weighted by the
    overlap over the cell, and the mirror's padding holds them."""
    first, count, w, maxt = rlc.area_taps(ssize, dsize)
    assert maxt == count.max()
    padt = rlc.pad_taps(maxt)
    assert padt >= maxt and (padt in rlc.PADS or padt > 16)
    sc = ssize / dsize
    for d in range(dsize):
        f1 = d * sc
        cell = min(sc, ssize - f1)
        k = np.arange(ssize)
        ov = np.clip(np.minimum(f1 + sc, k + 1) - np.maximum(f1, k), 0.0, None)
        support = np.nonzero(ov > 1e-3)[0]
        assert (first[d], count[d]) == (support[0], len(support)), d
        np.testing.assert_allclose(w[d, :count[d]], ov[support] / cell, rtol=2e-7, atol=0)
        assert np.all(w[d, count[d]:] == 0)


@pytest.mark.parametrize("case", DOWN, ids=[c.label for c in DOWN])
def test_oracle_is_within_half_of_the_exact_mean(case):
    """The oracle's area resize against the fp64 area mean of the same crop: within half an LSB (+1e-4 for the fp32
    chain), and a constant image comes out as the same constant."""
    images = case.images()
    got = np.stack(case.expected(images)).reshape(case.n, case.dh, case.dw, case.C).astype(np.float64)
    err = np.abs(got - rlc.area_mean64(images, case.crop, case.dw, case.dh))
    assert err.max() <= rlc.AREA_TOLERANCE, (err.max(), np.unravel_index(err.argmax(), err.shape))
    for v in (0, 1, 127, 128, 254, 255):
        out = rlc.oracle.resize(np.full(case.shape(case.sh, case.sw), v, np.uint8), case.dw, case.dh, crop=case.crop)
        assert (out == v).all(), v
