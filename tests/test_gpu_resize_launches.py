"""GPU: INTER_AREA resize launches as the batches shape them, bit-exact against the oracle.

Every case of tests/resize_launch_cases.py goes through lp_resize_area_dev as one launch of n images: every kernel the
launcher has, 1- to 16-row bands with ragged last bands and tiles, unaligned rows and images, crops at the edges and
the 1080p headline shape.  Each image must equal the oracle bit for bit and (downscales) lie within half an LSB of the
exact area mean; no byte of destination padding may be written.  Calls with more images than one launch takes
(gridDim.z <= 65535) are checked on either side of the split.  Then the product paths that launch 16-row bands: an
lp_batch chunk of 40 1080p JPEGs, and lp_xbatch runs of RGBA PNGs.
"""
import ctypes as C
import struct
import zlib

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests import resize_launch_cases as rlc
from tests.test_gpu_xbatch import T, check_against_per_image

pytestmark = pytest.mark.gpu
SENTINEL = 0xA7
CASES = rlc.catalogue()
HUGE = rlc.huge_cases()


@pytest.fixture(scope="module")
def dev(cuda_lib):
    l = cuda_lib.l
    l.lp_dev_alloc.restype = C.c_void_p
    l.lp_dev_alloc.argtypes = [C.c_size_t]
    l.lp_dev_free.argtypes = [C.c_void_p]
    for f in (l.lp_memcpy_h2d, l.lp_memcpy_d2h):
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    l.lp_dev_synchronize.restype = C.c_int
    l.lp_resize_area_dev.restype = C.c_int
    l.lp_resize_area_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return l


def resize_on_device(l, case, src):
    """One lp_resize_area_dev call on the packed source allocation `src`; the whole destination allocation (filled
    with SENTINEL before the call) comes back."""
    dst = np.full(case.dst_bytes, SENTINEL, dtype=np.uint8)
    d_src, d_dst = l.lp_dev_alloc(src.size), l.lp_dev_alloc(dst.size)
    try:
        assert d_src and d_dst
        assert l.lp_memcpy_h2d(d_src, src.ctypes.data, src.size) == 0
        assert l.lp_memcpy_h2d(d_dst, dst.ctypes.data, dst.size) == 0
        cx, cy, cw, chh = case.crop
        rc = l.lp_resize_area_dev(d_src + case.base, case.src_img_stride, case.src_row_stride, case.C, cx, cy, cw, chh,
                                  d_dst, case.dst_img_stride, case.dst_row_stride, case.dw, case.dh, case.n, None)
        assert l.lp_dev_synchronize() == 0
        assert l.lp_memcpy_d2h(dst.ctypes.data, d_dst, dst.size) == 0
    finally:
        l.lp_dev_free(d_src)
        l.lp_dev_free(d_dst)
    return rc, dst


def check_images(case, images, got, idx):
    """got[k] (dh, dw*C) is the device's image idx[k] of `images`."""
    want = [rlc.oracle.resize(images[i], case.dw, case.dh, crop=case.crop).reshape(case.dh, -1) for i in idx]
    bad = [i for i, g, w in zip(idx, got, want) if not np.array_equal(g, w)]
    if bad:
        k = idx.index(bad[0])
        d = np.abs(got[k].astype(int) - want[k].astype(int))
        y, x = np.unravel_index(d.argmax(), d.shape)
        pytest.fail(f"{case.label} ({case.launch()}): {len(bad)} of {len(idx)} images differ from the oracle; image "
                    f"{bad[0]}: {int((d > 0).sum())} bytes, up to {d.max()}, first worst at row {y} byte {x}")
    if case.downscale:
        exact = rlc.area_mean64(images[idx], case.crop, case.dw, case.dh).reshape(len(idx), case.dh, -1)
        err = np.abs(np.asarray(got, dtype=np.float64) - exact).max()
        assert err <= rlc.AREA_TOLERANCE, f"{case.label}: {err} from the exact area mean"


def check_padding(case, dst):
    mask = np.ones(dst.size, dtype=bool)
    rlc.dst_view(mask, case)[:] = False
    written = np.nonzero(dst[mask] != SENTINEL)[0]
    assert written.size == 0, f"{case.label}: {written.size} destination padding bytes written"


@pytest.mark.parametrize("case", CASES, ids=[c.label for c in CASES])
def test_launch_matches_oracle(dev, case):
    images = case.images()
    rc, dst = resize_on_device(dev, case, case.pack(images))
    assert rc == 0, f"{case.label}: lp_resize_area_dev returned {rc}"
    check_images(case, images, list(rlc.dst_view(dst, case)), list(range(case.n)))
    check_padding(case, dst)


@pytest.mark.parametrize("case", HUGE, ids=[c.label for c in HUGE])
def test_more_images_than_one_launch(dev, case):
    """65535 + 37 distinct images in one call: the launcher splits it into launches of at most 65535 images.  Every
    image from 65500 on (both sides of the split) and a seeded sample of the rest against the oracle."""
    assert case.n > rlc.MAX_GRID_Z
    src = np.random.default_rng(case.seed).integers(0, 256, case.src_bytes, dtype=np.uint8)
    images = rlc.src_view(src, case).reshape(case.n, *case.shape(case.sh, case.sw))
    rc, dst = resize_on_device(dev, case, src)
    assert rc == 0, f"{case.label}: lp_resize_area_dev returned {rc}"
    idx = sorted(set(np.random.default_rng(7).choice(65500, 300, replace=False).tolist()) | set(range(65500, case.n)))
    crops = {images[i, case.crop[1]:case.crop[1] + case.crop[3], case.crop[0]:case.crop[0] + case.crop[2]].tobytes()
             for i in idx}
    assert len(crops) == len(idx)  # a wrong image offset cannot give the right answer
    out = rlc.dst_view(dst, case)
    check_images(case, images, [out[i] for i in idx], idx)
    check_padding(case, dst)


def test_lp_batch_chunk_of_40_1080p_frames(cuda_lib, oracle):
    """The headline chunk: 40 distinct 1920x1080 JPEGs, Fit 256x256, one chunk -> one resize launch at 16-row bands
    (from 33 images on); the resized frames against the oracle's Fit of the oracle's decode."""
    n, w, h = 40, 1920, 1080
    crop = oracle.fit_rect(w, h, 256, 256)
    assert crop == (420, 0, 1080, 1080)
    assert rlc.dispatch(3, crop[2], crop[3], 256, 256, n) == rlc.Launch("area_sorted", 6, 6, 16)
    base = synth_image(3000, w, h, 3, noise=0.0)
    rng = np.random.default_rng(3000)
    files = [oracle.jpeg_encode(np.roll(base, 7 * i, axis=1) ^ rng.integers(0, 8, base.shape, dtype=np.uint8), 90)
             for i in range(n)]
    b = abi.Batch(cuda_lib, 0, n, w, h, 256, 256, 85, max_in_bytes=sum(map(len, files)) + 4096, chunk=n)
    try:
        assert b.stage(files) == [0] * n
        b.run()
        resized = b.resized_frames(n, 256, 256)
    finally:
        b.close()
    bad = [i for i, f in enumerate(files) if not np.array_equal(resized[i], oracle.fit(oracle.jpeg_decode(f)[0], 256, 256))]
    assert bad == []


def rgba_png(img):
    """BGRA frame -> 8-bit RGBA PNG, filter None, one IDAT (tests/png_writer.py covers the filters; this is fast)."""
    h, w, _ = img.shape
    rows = np.concatenate([np.zeros((h, 1), np.uint8), img[:, :, [2, 1, 0, 3]].reshape(h, -1)], axis=1)

    def chunk(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d))
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(rows.tobytes(), 1)) + chunk(b"IEND", b""))


def smallest_png_launch(files, w, h):
    """A lower bound on the images of one resize launch when lp_xbatch takes `files` (PNGs of one geometry, w x h RGBA).

    lp_xbatch puts every PNG of a call in one list and cuts it into tasks at half the list's device bytes
    (split_by_memory in csrc/xbatch.cu); run_png resizes each run of equal geometry in a task's frame window with one
    launch, and here the window holds the whole task.  An item's bytes are twice its file size plus more than its
    inflated scanlines, (4w + 1) * h.  The first task closes past half the total, so each of the two holds at least
    total / (2 * largest item) - 1 images."""
    need = [2 * len(f) + (4 * w + 1) * h for f in files]
    return int(sum(need) // (2 * max(need))) - 1


@pytest.mark.parametrize("w,h", [(384, 216), (385, 217)])  # the second: 1540-byte rows, 4 mod 16
def test_lp_xbatch_png_runs_at_16_row_bands(cuda_lib, w, h):
    """BASELINE config 3 geometry (RGBA PNG -> Fit 128x128 -> WebP), 160 images in one call: each of the two tasks
    resizes its ~80 frames in one launch, 4 channels at 16-row bands (from 66 images on).  Bytes == lp_transform of
    each file (whose resize runs one image at 1-row bands), every item through the grid path."""
    n = 160
    base = synth_image(4000 + w, w, h, 4, noise=0.0)
    rng = np.random.default_rng(w)
    files = [rgba_png(np.roll(base, 5 * k, axis=1) ^ rng.integers(0, 8, base.shape, dtype=np.uint8)) for k in range(n)]
    per_launch = smallest_png_launch(files, w, h)
    crop = rlc.oracle.fit_rect(w, h, 128, 128)
    assert crop == ((w - h) // 2, 0, h, h)
    L = rlc.dispatch(4, h, h, 128, 128, per_launch)
    assert L.kernel == "area" and L.rpb == 16, (per_launch, L)
    opt = abi.ImageOptions(FileType=".webp", Width=128, Height=128, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.WebpQuality: 85}, EncodeTimeout_ns=T)
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    try:
        _, status = check_against_per_image(cuda_lib, xb, files, opt)
        st = xb.stats()
    finally:
        xb.close()
    assert status == [0] * n
    assert st["grid_items"] == n and st["fallback_items"] == 0
