"""GPU: several renditions of every file in one heterogeneous batch call (lp_xbatch_transform_renditions,
csrc/xbatch.cu).  Each file is uploaded and decoded once; every (item, rendition) pair is resized and encoded with that
rendition's options.

Every pair is compared with per-image lp_transform of the same library (status and bytes).  The pair counts are asserted
exactly against a routing oracle made of calls that already exist: the pairs a renditions call runs on the grid are the
sum over r of grid_items of lp_xbatch_transform(files, opts[r]).  So a pair silently handed to the per-image path, or
a rendition that changed which pairs take the grid, cannot pass."""
import ctypes as C
import io

import cv2
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch import per_image, rgb_png
from tests.test_gpu_xbatch_hdr_png import hdr_png, png_file, source, with_cicp
from tests.test_gpu_xbatch_jpeg_webp import cv2_jpeg, png_profile, webp_still_with_icc, with_exif_orientation, with_iccp

pytestmark = pytest.mark.gpu
T = 10**12
CAP = 1 << 22
FIT, RESIZE = abi.ImageOpsFit, abi.ImageOpsResize
PAIR_STATS = ("grid_items", "fallback_items", "groups", "launches", "h2d_bytes", "d2h_bytes")


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def jpeg(w, h, method, q=85, progressive=False, **kw):
    enc = {abi.JpegQuality: q}
    if progressive:
        enc[abi.JpegProgressive] = 1
    return abi.ImageOptions(FileType=".jpeg", Width=w, Height=h, ResizeMethod=method, EncodeOptions=enc, EncodeTimeout_ns=T, **kw)


def webp(w, h, method, q=85, **kw):
    kw.setdefault("EncodeTimeout_ns", T)
    return abi.ImageOptions(FileType=".webp", Width=w, Height=h, ResizeMethod=method, EncodeOptions={abi.WebpQuality: q}, **kw)


def png(w, h, method, level=None, **kw):
    enc = {} if level is None else {abi.PngCompression: level}
    return abi.ImageOptions(FileType=".png", Width=w, Height=h, ResizeMethod=method, EncodeOptions=enc, EncodeTimeout_ns=T, **kw)


def gif(w, h, method):
    return abi.ImageOptions(FileType=".gif", Width=w, Height=h, ResizeMethod=method, EncodeTimeout_ns=T)


def pil_gif(seed, w, h, n):
    from PIL import Image
    frames = [Image.fromarray(synth_image(seed + k, w, h, 3)[:, :, ::-1].copy()).quantize(64) for k in range(n)]
    bio = io.BytesIO()
    frames[0].save(bio, "GIF", save_all=True, append_images=frames[1:], duration=40, loop=0)
    return bio.getvalue()


def pil_webp_animation(seed, w, h, n, lossless):
    from PIL import Image
    frames = [Image.fromarray(synth_image(seed + k, w, h, 4)[:, :, [2, 1, 0, 3]].copy(), "RGBA") for k in range(n)]
    bio = io.BytesIO()
    frames[0].save(bio, "WEBP", save_all=True, append_images=frames[1:], duration=50, loop=0, lossless=lossless, quality=80)
    return bio.getvalue()


def cv2_webp(img, q):
    ok, b = cv2.imencode(".webp", img, [cv2.IMWRITE_WEBP_QUALITY, q])
    assert ok
    return bytes(b)


def corpus():
    """(name, file): every source kind the grid takes, the ones routed per image, and damaged files"""
    s420, s422, s444 = (cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444)
    base = cv2_jpeg(synth_image(1, 640, 360, 3), 90, sampling=s420)
    files = [
        ("jpeg_420", base),
        ("jpeg_420_same_size", cv2_jpeg(synth_image(2, 640, 360, 3), 70, sampling=s420)),
        ("jpeg_rst", cv2_jpeg(synth_image(3, 320, 240, 3), 85, rst=4)),
        ("jpeg_progressive", cv2_jpeg(synth_image(4, 300, 200, 3), 80, progressive=True)),
        ("jpeg_422_odd", cv2_jpeg(synth_image(5, 203, 117, 3), 90, sampling=s422)),
        ("jpeg_444_odd", cv2_jpeg(synth_image(6, 161, 97, 3), 95, sampling=s444)),
        ("jpeg_1x1", cv2_jpeg(synth_image(7, 1, 1, 3), 90)),
        ("jpeg_gray", cv2_jpeg(synth_image(8, 120, 90, 1), 90)),
        ("jpeg_rotated", with_exif_orientation(cv2_jpeg(synth_image(9, 200, 120, 3), 90), 6)),
        ("png_rgb", rgb_png(synth_image(10, 300, 200, 3))),
        ("png_rgba", rgb_png(synth_image(11, 256, 256, 4))),
        ("png_16bit", png_file(source(12, 130, 70, "rgb", 16)[1], 2, 16)),
        ("png_adam7", rgb_png(synth_image(13, 97, 61, 3), interlace=True)),
        ("png_pq", hdr_png(14, 101, 75, "rgb", 16, 16, 9)),
        ("png_hlg", hdr_png(15, 64, 48, "rgba", 16, 18, 12)),
        ("png_gray", png_file(synth_image(16, 50, 40, 1).reshape(40, 50, 1), 0, 8)),
        ("webp_lossy", cv2_webp(synth_image(17, 240, 160, 3), 80)),
        ("webp_lossy_alpha", cv2_webp(synth_image(18, 120, 100, 4), 80)),
        ("webp_lossless", cv2_webp(synth_image(19, 90, 70, 4), 101)),
        ("webp_anim_lossy", pil_webp_animation(20, 96, 64, 3, lossless=False)),
        ("webp_anim_lossless", pil_webp_animation(24, 64, 48, 2, lossless=True)),
        ("gif_anim", pil_gif(30, 80, 60, 3)),
        ("gif_one_frame", pil_gif(34, 50, 50, 1)),
        ("jpeg_truncated", base[: len(base) // 2]),
        ("jpeg_damaged_scan", base[:600] + bytes(200) + base[800:]),
        ("png_truncated", rgb_png(synth_image(35, 60, 40, 3))[:-40]),
        ("gif_truncated", pil_gif(36, 40, 40, 2)[:-30]),
        ("garbage", bytes(range(256)) * 4),
    ]
    return files


@pytest.fixture(scope="module")
def files():
    return corpus()


RENDITION_SETS = {
    # the avatar / thumbnail set the benchmark runs
    "thumbnails": [jpeg(256, 256, FIT), webp(512, 512, FIT), png(96, 96, FIT)],
    # every sink, wide / tall / square / larger than the source, Fit and Resize
    "every_sink": [jpeg(300, 60, FIT, progressive=True), webp(60, 300, FIT, q=101), png(100, 100, RESIZE, level=9),
                   png(2000, 1500, FIT, level=1), gif(64, 64, FIT), webp(50, 23, RESIZE, q=60), jpeg(1000, 1000, FIT, q=95)],
    # renditions whose gates differ: GIF output takes GIF sources only, lossless WebP no JPEG or WebP source, a negative
    # MaxEncodeDuration sends every PNG output per image, DisableAnimatedOutput writes stills of animations
    "gates": [gif(48, 48, FIT), webp(64, 64, FIT, q=101), png(32, 32, FIT, MaxEncodeDuration_ns=-1), jpeg(80, 40, FIT),
              webp(64, 64, FIT, DisableAnimatedOutput=True)],
}


def check_renditions(lib, xb, files, opts, cap=CAP):
    """Every pair against lp_transform and against the call with its options alone, and the pair counts against those
    calls; returns the outputs"""
    outs, status = xb.transform_renditions(files, opts, out_cap=cap)
    st = xb.stats()
    for i, f in enumerate(files):
        for r, o in enumerate(opts):
            want, code = per_image(lib, f, o, cap)
            assert status[i][r] == code, f"item {i} rendition {r}: batch status {status[i][r]}, lp_transform {code}"
            assert outs[i][r] == want, f"item {i} rendition {r}: bytes differ from lp_transform ({len(outs[i][r])} vs {len(want)} B)"
    grid = 0
    for r, o in enumerate(opts):
        alone, alone_status = xb.transform(files, o, out_cap=cap)
        assert [s[r] for s in status] == alone_status and [b[r] for b in outs] == alone
        grid += xb.stats()["grid_items"]
    assert st["grid_items"] == grid and st["fallback_items"] == len(files) * len(opts) - grid, (st, grid)
    return outs, status, st


@pytest.mark.parametrize("name", list(RENDITION_SETS))
def test_mixed_corpus_every_pair_is_lp_transform(cuda_lib, xb, files, name):
    check_renditions(cuda_lib, xb, [d for _, d in files], RENDITION_SETS[name])


def test_one_rendition_is_lp_xbatch_transform(cuda_lib, xb, files):
    data = [d for _, d in files]
    for o in RENDITION_SETS["every_sink"] + RENDITION_SETS["thumbnails"]:
        outs, status = xb.transform(data, o, out_cap=CAP)
        single = xb.stats()
        routs, rstatus = xb.transform_renditions(data, [o], out_cap=CAP)
        st = xb.stats()
        assert [s[0] for s in rstatus] == status
        assert [b[0] for b in routs] == outs
        assert {k: st[k] for k in PAIR_STATS} == {k: single[k] for k in PAIR_STATS}, o.FileType


def grid_files():
    """files every rendition of the thumbnail set takes on the grid: JPEGs of three geometries, RGB / RGBA PNGs, WebP stills"""
    out = [cv2_jpeg(synth_image(100 + k, 640, 360, 3), 85) for k in range(4)]
    out += [cv2_jpeg(synth_image(110 + k, 333, 500, 3), 90, sampling=cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444) for k in range(3)]
    out += [cv2_jpeg(synth_image(120, 1920, 1080, 3), 90, progressive=True)]
    out += [rgb_png(synth_image(130 + k, 300, 200, 3 + k % 2)) for k in range(4)]
    out += [cv2_webp(synth_image(140 + k, 240, 160, 3), 80) for k in range(3)]
    return out


def test_each_file_is_uploaded_once(cuda_lib, xb):
    data = grid_files()
    opts = RENDITION_SETS["thumbnails"]
    _, _, st = check_renditions(cuda_lib, xb, data, opts)
    assert st["grid_items"] == len(data) * len(opts) and st["fallback_items"] == 0, st
    xb.transform(data, opts[0], out_cap=CAP)
    assert st["h2d_bytes"] == xb.stats()["h2d_bytes"]


def test_duplicate_renditions_give_the_same_bytes(cuda_lib, xb, files):
    data = [d for _, d in files]
    o = webp(120, 120, FIT, q=70)
    outs, status, _ = check_renditions(cuda_lib, xb, data, [o, jpeg(64, 64, FIT), o])
    for i in range(len(data)):
        assert outs[i][0] == outs[i][2] and status[i][0] == status[i][2]


def test_gates_that_differ_per_rendition(cuda_lib, xb):
    """A zero encode budget and MaxEncodeFrames 1 send JPEGs and PNGs with a profile to WebP per image (Transform decides
    them after the frame); the same files' middle rendition stays on the grid"""
    profile = png_profile()
    data = [d for d in grid_files() if d[:2] == b"\xff\xd8"]
    data += [with_iccp(rgb_png(synth_image(150 + k, 200, 150, 3 + k % 2)), profile) for k in range(3)]
    opts = [webp(64, 64, FIT, EncodeTimeout_ns=0), webp(64, 64, FIT), webp(64, 64, FIT, MaxEncodeFrames=1)]
    _, status, st = check_renditions(cuda_lib, xb, data, opts)
    assert st["grid_items"] == len(data) and st["fallback_items"] == 2 * len(data), st
    assert all(s[1] == 0 and s[0] != 0 and s[2] != 0 for s in status), status


@pytest.mark.parametrize("kind", ["png", "webp"])
def test_rendition_skipping_an_item_between_equal_geometries(cuda_lib, xb, kind):
    """Four files of one geometry, the second of which one rendition sends per image (an SDR cICP chunk keeps a PNG's
    PNG output per image, an ICC profile a WebP still's WebP output under a zero encode budget); the first three share
    a task.  The third file is resized from its own decoded frame, not from the second's."""
    if kind == "png":
        a, b, c, d = (rgb_png(synth_image(500 + k, 200, 150, 3)) for k in range(4))
        data, opts = [a, with_cicp(b, 1, 13), c, d], [png(64, 64, FIT), jpeg(64, 64, FIT)]
        _, _, st = check_renditions(cuda_lib, xb, data, opts)
    else:
        # (under a zero budget the grid writes a plain lossy still where lp_transform reports ErrEncodeTimeout, so each
        # rendition is held against a call with its options alone, whose task has no file in between)
        a, c, d = (cv2_webp(synth_image(510 + k, 200, 150, 3), 80) for k in range(3))
        data = [a, webp_still_with_icc(png_profile(), 200, 150, 513), c, d]
        opts = [webp(64, 64, FIT, EncodeTimeout_ns=0), jpeg(64, 64, FIT)]
        outs, status = xb.transform_renditions(data, opts, out_cap=CAP)
        st = xb.stats()
        for r, o in enumerate(opts):
            alone, alone_status = xb.transform(data, o, out_cap=CAP)
            assert [s[r] for s in status] == alone_status and [b[r] for b in outs] == alone, r
    assert st["grid_items"] == 7 and st["fallback_items"] == 1, st


@pytest.mark.parametrize("src", [(640, 360), (360, 640), (257, 255), (1920, 1080)], ids=["wide", "tall", "odd", "1080p"])
def test_jpeg_window_union(cuda_lib, xb, src):
    """A wide and a tall Fit crop different parts of the frame; Resize and a same-aspect Fit reach every edge.  The
    decoded window is the bounding box of them all; each rendition's bytes equal a call with that rendition alone."""
    w, h = src
    data = [cv2_jpeg(synth_image(200 + k, w, h, 3), 88) for k in range(3)]
    opts = [jpeg(400, 40, FIT), webp(40, 400, FIT), png(w // 3, h // 3, FIT), jpeg(100, 30, RESIZE, progressive=True),
            webp(17, 200, RESIZE)]
    outs, status, st = check_renditions(cuda_lib, xb, data, opts)
    assert st["fallback_items"] == 0, st
    for r, o in enumerate(opts):
        alone, alone_status = xb.transform_renditions(data, [o], out_cap=CAP)
        assert [s[r] for s in status] == [s[0] for s in alone_status]
        assert [b[r] for b in outs] == [b[0] for b in alone]


@pytest.mark.parametrize("cap", [700, 1000, 1024])
def test_small_buffers(cuda_lib, xb, files, cap):
    """Buffer sizes inside and on a 256-byte unit: a JPEG file of a group with several renditions leaves the grid exactly
    where it leaves the pipelined path of a call with its options alone"""
    data = [d for _, d in files] + grid_files()
    _, status, _ = check_renditions(cuda_lib, xb, data, RENDITION_SETS["thumbnails"], cap=cap)
    assert any(abi.LP_ERR_BUF_TOO_SMALL in s for s in status)


@pytest.mark.parametrize("order", ["still_first", "animation_first"])
def test_animated_webp_as_still_and_as_animation(cuda_lib, xb, order):
    """An animated WebP whose renditions want frame 0 as a still (DisableAnimatedOutput) and the whole animation: each
    rendition gets its own result whatever the order"""
    data = [pil_webp_animation(300, 96, 64, 4, lossless=False), pil_webp_animation(310, 64, 48, 3, lossless=True),
            pil_webp_animation(320, 96, 64, 2, lossless=False), cv2_webp(synth_image(330, 96, 64, 3), 80)]
    still, anim = webp(48, 48, FIT, DisableAnimatedOutput=True), webp(40, 30, FIT, q=70)
    opts = [still, anim] if order == "still_first" else [anim, still]
    outs, status, st = check_renditions(cuda_lib, xb, data, opts)
    assert st["fallback_items"] == 0, st
    r_anim = opts.index(anim)
    for i in range(3):  # the animations' full outputs carry one ANMF chunk per frame, the stills none
        assert outs[i][r_anim].count(b"ANMF") >= 2 and outs[i][1 - r_anim].count(b"ANMF") == 0


def test_jpeg_sink_parts_fit_a_small_arena(cuda_lib):
    """A group of several renditions with a JPEG one, more frames than the lane's arena holds JPEG slots for at a large
    buffer size: the JPEG sink encodes in parts and every pair stays where separate calls put it"""
    distinct = [cv2_jpeg(synth_image(400 + k, 320, 240, 3), 85) for k in range(8)]
    data = [distinct[k % 8] for k in range(1200)]  # (two tasks of 600: more than the 512 frames the sink's room is kept for)
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        _, status, st = check_renditions(cuda_lib, small, data, [jpeg(256, 256, FIT), webp(64, 64, FIT)])
    finally:
        small.close()
    assert st["grid_items"] == 2 * len(data) and st["fallback_items"] == 0, st


def test_small_arena_gives_the_same_bytes(cuda_lib, xb, files):
    data = [d for _, d in files] + grid_files() * 6
    opts = RENDITION_SETS["thumbnails"] + [gif(48, 48, FIT)]
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        got = small.transform_renditions(data, opts, out_cap=CAP)
    finally:
        small.close()
    assert got == xb.transform_renditions(data, opts, out_cap=CAP)


def test_multi_gpu_call_equals_the_single_gpu_call(cuda_lib, xb, files):
    data = [d for _, d in files] + grid_files()
    opts = RENDITION_SETS["every_sink"]
    m = abi.MultiBatch(cuda_lib, [0], arena_bytes=4 << 30)
    try:
        got = m.transform_renditions(data, opts, out_cap=CAP)
    finally:
        m.close()
    assert got == xb.transform_renditions(data, opts, out_cap=CAP)


def test_bad_arguments_are_refused(cuda_lib, xb, files):
    l = cuda_lib.l
    data = [files[0][1]]
    ptrs, lens, keep = abi.Batch._ptr_arrays(data)
    buf = np.zeros((17, 1024), np.uint8)
    out_ptrs = (C.c_void_p * 17)(*[buf[p].ctypes.data for p in range(17)])
    out_lens = (C.c_size_t * 17)(*([12345] * 17))
    status = (C.c_int * 17)(*([77] * 17))
    cs = [jpeg(32, 32, FIT)._c() for _ in range(17)]
    copts = (abi._ImageOptions * 17)(*cs)
    for fn, h in ((l.lp_xbatch_transform_renditions, xb.h),):
        for k, o in ((0, copts), (17, copts), (-1, copts), (1, None)):
            assert fn(h, ptrs, lens, 1, o, k, out_ptrs, 1024, out_lens, status) == -10
    m = abi.MultiBatch(cuda_lib, [0], arena_bytes=1 << 30)
    try:
        for k, o in ((0, copts), (17, copts), (1, None)):
            assert l.lp_multi_transform_renditions(m.h, ptrs, lens, 1, o, k, out_ptrs, 1024, out_lens, status) == -10
    finally:
        m.close()
    assert list(status) == [77] * 17 and list(out_lens) == [12345] * 17
    # sixteen renditions is the most a call takes
    outs, st = xb.transform_renditions(data, [jpeg(16 + r, 16, FIT) for r in range(16)], out_cap=1 << 16)
    assert st == [[0] * 16]
