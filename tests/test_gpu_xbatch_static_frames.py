"""GPU: DisableAnimatedOutput in the heterogeneous batch (lp_xbatch_transform, csrc/xbatch.cu): frame 0 of every GIF and
animated WebP written as a still WebP or a one-frame GIF on the device, and one-frame GIFs to WebP without the flag.

Every item is compared with per-image lp_transform of the same library, status and bytes, and grid_items /
fallback_items are asserted exactly, so a silent hand-over to the per-image path cannot pass.  Independently of the
library, the WebP outputs decoded by libwebp must match the oracle's frame 0 (oracle_gif.c compositor, or the per-frame
WebP decode composited in numpy) fitted by the oracle, and a GIF output of a palette the writer maps exactly must decode
(Pillow, giflib's format) to frame 0 itself."""
import io

import numpy as np
import pytest

from lilliput_b200 import abi
from oracle import oracle
from tests.gif_streams import app, comment, gcb, lzw_literals, write_gif
from tests.test_gpu_xbatch import check_against_per_image
from tests.test_gpu_xbatch_webp import (_plane, animation, anmf, composite, icc_profile, lossless_frame, lossy_frame)
from tests import vp8l_streams as vs
from tests.webp_util import chunks_of, frames_of, libwebp_decode, psnr, vp8_cpu_encode, vp8_cpu_lib

pytestmark = pytest.mark.gpu
T = 10**12
W, H = 72, 54


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def opts(ext, q=85, **kw):
    kw.setdefault("EncodeTimeout_ns", T)
    kw.setdefault("DisableAnimatedOutput", True)
    kw.setdefault("Width", 40)
    kw.setdefault("Height", 40)
    kw.setdefault("ResizeMethod", abi.ImageOpsFit)
    if ext == ".webp":
        kw.setdefault("EncodeOptions", {abi.WebpQuality: q})
    elif ext == ".jpeg":
        kw.setdefault("EncodeOptions", {abi.JpegQuality: q})
    return abi.ImageOptions(FileType=ext, **kw)


def expect_counts(xb, grid, fallback):
    st = xb.stats()
    assert (st["grid_items"], st["fallback_items"]) == (grid, fallback), st


def _pal(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n * 3, dtype=np.uint8).tobytes()


def _idx(seed, h, w, n):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = ((x * n) // max(w, 1) + (y // 4) * 3 + rng.integers(0, n)) % n
    return np.where(rng.random((h, w)) < 0.2, rng.integers(0, n, (h, w)), base).astype(np.uint8)


def later(k0, n=3, pal=16):
    return [dict(idx=_idx(k0 + k, H, W, pal), gcb=gcb(1, 4)) for k in range(n)]


def synthetic_gifs():
    """Each file steers one feature of frame 0 and of what the per-image decoder has seen when it stops there."""
    g16, g64 = _pal(1, 16), _pal(2, 64)
    c = {}
    c["partial_offset"] = write_gif(W, H, [dict(idx=_idx(10, 20, 33, 64), left=7, top=9)] + later(11, pal=64), gct=g64)
    c["partial_offset_transparent"] = write_gif(W, H, [dict(idx=_idx(12, 17, 25, 16), left=40, top=30, gcb=gcb(1, 3, 5))]
                                                + later(13), gct=g16, bg=2)
    c["transparent_gcb"] = write_gif(W, H, [dict(idx=_idx(14, H, W, 16), gcb=gcb(0, 4, 3))] + later(15), gct=g16, bg=3)
    c["transparent_no_gcb"] = write_gif(W, H, [dict(idx=_idx(16, 30, 30, 16), left=4, top=4, gcb=None)] + later(17), gct=g16)
    c["background_drop"] = write_gif(W, H, [dict(idx=_idx(18, H, W, 16), gcb=gcb(1, 4, 6))] + later(19), gct=g16, bg=6)
    c["interlaced"] = write_gif(W, H, [dict(idx=_idx(20, 37, 50, 64), left=5, top=3, interlace=True)] + later(21, pal=64),
                                gct=g64)
    c["local_palette"] = write_gif(W, H, [dict(idx=_idx(22, H, W, 32), local=_pal(23, 32))] + later(24), gct=g16)
    c["no_global_table"] = write_gif(W, H, [dict(idx=_idx(25 + k, H, W, 8), local=_pal(26 + k, 8)) for k in range(3)])
    c["dispose2"] = write_gif(W, H, [dict(idx=_idx(30, 30, 40, 16), left=10, top=8, gcb=gcb(2, 4, 3))] + later(31), gct=g16)
    c["dispose3"] = write_gif(W, H, [dict(idx=_idx(32, 20, 20, 16), left=40, top=20, gcb=gcb(3, 4, 5))] + later(33), gct=g16)
    c["extensions_after"] = write_gif(W, H, [
        dict(idx=_idx(34, H, W, 16), pre=comment(b"first frame") + app(b"XMP DataXMP", b"<x/>" * 40), gcb=gcb(0, 7, 2)),
        dict(idx=_idx(35, H, W, 16), pre=app(b"XMP DataXMP", b"<y/>" * 80) + comment(b"between" * 50))],
        gct=g16, trailer_ext=comment(b"after the last frame") + app(b"TRAILER1.00", b"\x01\x02\x03"))
    c["one_frame"] = write_gif(W, H, [dict(idx=_idx(36, H, W, 64), gcb=gcb(0, 0, 9))], gct=g64, loop=False)
    c["one_frame_trailer"] = write_gif(W, H, [dict(idx=_idx(37, 30, 20, 16), left=3, top=2)], gct=g16,
                                       trailer_ext=comment(b"behind the only frame"))
    # 128 frames, each later frame the whole canvas while frame 0 is a small rectangle
    c["reel_128"] = write_gif(W, H, [dict(idx=_idx(38, 8, 8, 16), left=30, top=20)] + later(40, n=127), gct=g16)
    return c


def damaged_gifs():
    """{name: (file, whether frame 0 decodes)}: damage behind frame 0 is never read with the flag; damage inside it is."""
    g16 = _pal(3, 16)
    f0 = dict(idx=_idx(50, H, W, 16))
    head = write_gif(W, H, [f0], gct=g16)[:-1]  # through frame 0's image data
    good = write_gif(W, H, [f0] + later(51), gct=g16)
    assert good.startswith(head)
    out = {"cut_in_frame1": (good[:len(head) + 40], True), "no_trailer": (good[:-1], True),
           "bad_record_after_frame0": (head + b"\x77" + good[len(head):], True)}
    idx = _idx(52, H, W, 16)
    short = lzw_literals(idx[:H // 3], 4)  # the code stream ends a third of the way into the frame
    out["short_stream_frame0"] = (write_gif(W, H, [dict(idx=idx, stream=(4, short))] + later(53), gct=g16), False)
    return out


# ---------------------------------------------------------------- GIF sources

GEOMETRIES = [dict(Width=40, Height=40, ResizeMethod=abi.ImageOpsFit), dict(Width=64, Height=24, ResizeMethod=abi.ImageOpsFit),
              dict(Width=20, Height=50, ResizeMethod=abi.ImageOpsFit), dict(Width=40, Height=40, ResizeMethod=abi.ImageOpsResize),
              dict(Width=64, Height=24, ResizeMethod=abi.ImageOpsResize), dict(Width=20, Height=50, ResizeMethod=abi.ImageOpsResize)]
SINKS = [(".webp", 1), (".webp", 50), (".webp", 85), (".webp", 100), (".gif", 0)]


@pytest.mark.parametrize("sink,q", SINKS)
def test_golden_gif_fixtures(cuda_lib, xb, golden, sink, q):
    files = [golden[k].tobytes() for k in sorted(golden.files) if k.startswith("gif_") and golden[k].ndim == 1]
    for geo in GEOMETRIES:
        _, status = check_against_per_image(cuda_lib, xb, files, opts(sink, q, **geo))
        assert status == [0] * len(files)
        expect_counts(xb, len(files), 0)


@pytest.mark.parametrize("sink,q", SINKS)
def test_synthetic_gifs(cuda_lib, xb, sink, q):
    cases = synthetic_gifs()
    files = list(cases.values())
    for geo in GEOMETRIES[:1] + GEOMETRIES[4:5]:
        _, status = check_against_per_image(cuda_lib, xb, files, opts(sink, q, **geo))
        assert status == [0] * len(files), dict(zip(cases, status))
        expect_counts(xb, len(files), 0)


def test_damaged_gifs(cuda_lib, xb):
    cases = damaged_gifs()
    files = [f for f, _ in cases.values()]
    for sink in (".webp", ".gif"):
        _, status = check_against_per_image(cuda_lib, xb, files, opts(sink))
        for (name, (_, ok)), s in zip(cases.items(), status):
            assert (s == 0) == ok, (sink, name, s)
        bad = sum(not ok for _, ok in cases.values())
        expect_counts(xb, len(files) - bad, bad)


def test_one_frame_gif_to_webp_without_the_flag(cuda_lib, xb):
    cases = synthetic_gifs()
    ones = [cases["one_frame"], cases["one_frame_trailer"]]
    anims = [cases["partial_offset"], cases["extensions_after"]]
    check_against_per_image(cuda_lib, xb, ones + anims, opts(".webp", DisableAnimatedOutput=False))
    expect_counts(xb, 4, 0)
    # no time to encode: the deadline check after the frame decides, per image
    _, status = check_against_per_image(cuda_lib, xb, ones, opts(".webp", DisableAnimatedOutput=False, EncodeTimeout_ns=0))
    assert all(s != 0 for s in status)
    expect_counts(xb, 0, 2)


def test_prefix_upload(cuda_lib, xb):
    reel = synthetic_gifs()["reel_128"]
    files = [reel] * 8
    for sink in (".webp", ".gif"):
        check_against_per_image(cuda_lib, xb, files, opts(sink))
        expect_counts(xb, len(files), 0)
        h2d = xb.stats()["h2d_bytes"]
        assert h2d < sum(map(len, files)) / 50, (h2d, sum(map(len, files)))


# ---------------------------------------------------------------- animated WebP sources

@pytest.fixture(scope="module")
def cpu():
    return vp8_cpu_lib()


def webp_animations(cpu):
    Wd, Hd = 64, 48
    full = lambda s: anmf(0, 0, Wd, Hd, lossy_frame(Wd, Hd, s, _plane(s, Wd, Hd, 128)))  # noqa: E731
    c = {}
    c["subrect_blend"] = animation(Wd, Hd, [anmf(10, 6, 30, 24, lossy_frame(30, 24, 1, _plane(1, 30, 24))), full(2)])
    c["subrect_no_blend"] = animation(Wd, Hd, [anmf(8, 4, 40, 30, lossy_frame(40, 30, 3, _plane(3, 40, 30)), blend=False,
                                                    dispose=True), full(4)])
    c["alph_full"] = animation(Wd, Hd, [full(5), full(6), full(7)])
    c["lossless_first"] = animation(Wd, Hd, [anmf(0, 0, Wd, Hd, lossless_frame(cpu, Wd, Hd, 8)), full(9)])
    c["lossless_subrect"] = animation(Wd, Hd, [anmf(4, 2, 40, 30, lossless_frame(cpu, 40, 30, 10), blend=False), full(11)])
    c["opaque_3ch"] = animation(Wd, Hd, [anmf(0, 0, Wd, Hd, lossy_frame(Wd, Hd, 12)), anmf(8, 8, 30, 20, lossy_frame(30, 20, 13))],
                                alpha=False)
    c["icc"] = animation(Wd, Hd, [full(14), full(15)], icc=icc_profile())
    junk = b"\x01" + np.random.default_rng(3).integers(0, 256, 24, dtype=np.uint8).tobytes()
    c["damaged_later_frame"] = animation(Wd, Hd, [full(16), anmf(4, 4, 20, 20, vs.chunk(b"ALPH", junk)
                                                                   + vs.chunk(b"VP8 ", vs.lossy_payload(20, 20, 17))), full(18)])
    return c


def test_animated_webp(cuda_lib, xb, cpu):
    cases = webp_animations(cpu)
    files = list(cases.values())
    for q in (1, 50, 85, 100):
        for geo in (GEOMETRIES[0], GEOMETRIES[4], dict(Width=64, Height=48, ResizeMethod=abi.ImageOpsResize)):
            outs, status = check_against_per_image(cuda_lib, xb, files, opts(".webp", q, **geo))
            assert status == [0] * len(files), dict(zip(cases, status))
            expect_counts(xb, len(files), 0)
    for name, out in zip(cases, outs):
        tags = [t for t, _ in chunks_of(out)]
        assert b"ANIM" not in tags and b"ANMF" not in tags, name
        assert (b"ICCP" in tags) == (name == "icc") and (b"VP8X" in tags) == (b"ICCP" in tags or b"ALPH" in tags), (name, tags)
    assert dict(chunks_of(outs[list(cases).index("icc")]))[b"ICCP"] == icc_profile()
    # the flag takes only frame 0 across PCIe
    check_against_per_image(cuda_lib, xb, files, opts(".webp"))
    assert xb.stats()["h2d_bytes"] < sum(map(len, files))


# ---------------------------------------------------------------- option gates

def test_option_gates(cuda_lib, xb, cpu):
    gifs = synthetic_gifs()
    webps = webp_animations(cpu)
    files = [gifs["partial_offset"], gifs["one_frame"], webps["subrect_blend"], webps["icc"]]
    check_against_per_image(cuda_lib, xb, files, opts(".webp", EncodeTimeout_ns=0))
    expect_counts(xb, 4, 0)
    check_against_per_image(cuda_lib, xb, files[:2], opts(".gif", EncodeTimeout_ns=0))
    expect_counts(xb, 2, 0)
    for kw in (dict(MaxEncodeFrames=1), dict(MaxEncodeFrames=2), dict(MaxEncodeDuration_ns=1), dict(MaxEncodeDuration_ns=-1)):
        check_against_per_image(cuda_lib, xb, files, opts(".webp", **kw))
        expect_counts(xb, 0, 4)
        check_against_per_image(cuda_lib, xb, files[:2], opts(".gif", **kw))
        expect_counts(xb, 0, 2)
    # JPEG and PNG sinks: the flag moves nothing
    for ext in (".jpeg", ".png"):
        counts = []
        for flag in (False, True):
            check_against_per_image(cuda_lib, xb, files, opts(ext, DisableAnimatedOutput=flag))
            st = xb.stats()
            counts.append((st["grid_items"], st["fallback_items"]))
        assert counts[0] == counts[1] == (0, 4), (ext, counts)


# ---------------------------------------------------------------- against the oracle

def smooth_gifs():
    """Frame 0 features of synthetic_gifs() over smooth content (a colour ramp), which lossy WebP keeps within its
    usual tolerance."""
    ramp = np.stack([np.arange(64) * 4, 255 - np.arange(64) * 4, np.full(64, 128)], 1).astype(np.uint8).tobytes()

    def grad(h, w, hole=False):
        y, x = np.mgrid[0:h, 0:w]
        idx = ((x * 10) // max(w - 1, 1) + (y * 5) // max(h - 1, 1)).astype(np.uint8)
        if hole:  # index 63 is the transparent one
            idx[h // 4:h // 2, w // 4:w // 2] = 63
        return idx
    return {"partial_offset": write_gif(W, H, [dict(idx=grad(20, 33), left=7, top=9)] + later(70, pal=64), gct=ramp),
            "transparent_gcb": write_gif(W, H, [dict(idx=grad(H, W, True), gcb=gcb(0, 4, 63))] + later(71, pal=64), gct=ramp, bg=63),
            "interlaced": write_gif(W, H, [dict(idx=grad(37, 50), left=5, top=3, interlace=True)] + later(72, pal=64), gct=ramp),
            "dispose3": write_gif(W, H, [dict(idx=grad(20, 20), left=40, top=20, gcb=gcb(3, 4, 5))] + later(73, pal=64), gct=ramp),
            "reel_128": write_gif(W, H, [dict(idx=grad(8, 8), left=30, top=20)] + later(74, n=127, pal=64), gct=ramp)}


def test_webp_pixels_against_the_oracle(cuda_lib, xb, cpu):
    """Frame 0 composited by the oracle (oracle_gif.c; the per-frame WebP decodes blended in numpy), fitted by the oracle
    and encoded by the host build of the VP8 encoder gives the batch's payload; libwebp reads the batch's alpha as the
    composite's, and the colour of the smooth GIFs within the lossy tolerance."""
    gifs = smooth_gifs()
    webps = webp_animations(cpu)
    names = list(gifs)
    wnames = ["subrect_blend", "subrect_no_blend", "lossless_first", "opaque_3ch"]
    files = [gifs[k] for k in names] + [webps[k] for k in wnames]
    q = 100
    outs, status = xb.transform(files, opts(".webp", q), out_cap=1 << 22)
    assert status == [0] * len(files)
    expect_counts(xb, len(files), 0)
    want = [oracle.fit(oracle.gif_frames(gifs[k], max_frames=1)[0][0], 40, 40) for k in names]
    want += [composite(cuda_lib, webps[k], 40, 40)[0] for k in wnames]
    for name, out, fit in zip(names + wnames, outs, want):
        (tag, vp8, alph), = frames_of(out)
        assert tag == b"VP8 " and vp8 == vp8_cpu_encode(cpu, fit, q), f"{name}: VP8 payload"
        got = libwebp_decode(out)
        opaque = fit.shape[2] == 3 or (fit[:, :, 3] == 255).all()
        assert got.shape[2] == (3 if opaque else 4) and (alph is None) == opaque, name
        seen = np.ones(fit.shape[:2], bool)
        if not opaque:
            assert np.array_equal(got[:, :, 3], fit[:, :, 3]), f"{name}: alpha"
            seen = fit[:, :, 3] == 255  # (colour under transparent pixels is the encoder's to choose)
        if name in gifs:  # (the hand-built WebP frames are noise: their payload check above is the exact one)
            assert psnr(got[seen][:, :3], fit[seen][:, :3]) > 28.0, name


def test_gif_pixels_exact(cuda_lib, xb):
    """A palette of bucket midpoints (every channel 8k + 4): the writer maps each colour to itself, so the one-frame GIF,
    at the canvas size, decodes to the oracle's frame 0 exactly (transparent where frame 0 is)."""
    pytest.importorskip("PIL")
    from PIL import Image
    rng = np.random.default_rng(7)
    pal = (rng.choice(32, (16, 3), replace=True) * 8 + 4).astype(np.uint8)
    pal[:, 0] = np.arange(16) * 8 + 4  # distinct entries
    g = pal.tobytes()
    files = [write_gif(W, H, [dict(idx=_idx(60, H, W, 16), gcb=gcb(1, 4))] + later(61), gct=g),
             write_gif(W, H, [dict(idx=_idx(62, 20, 30, 16), left=9, top=7, gcb=gcb(1, 4, 3))] + later(63), gct=g, bg=3)]
    outs, status = check_against_per_image(cuda_lib, xb, files, opts(".gif", Width=W, Height=H, ResizeMethod=abi.ImageOpsResize))
    assert status == [0, 0]
    expect_counts(xb, 2, 0)
    for f, out in zip(files, outs):
        frame0 = oracle.gif_frames(f, max_frames=1)[0][0]  # BGRA
        im = Image.open(io.BytesIO(out))
        assert getattr(im, "n_frames", 1) == 1
        got = np.asarray(im.convert("RGBA"))
        seen = frame0[:, :, 3] == 255
        assert np.array_equal(got[:, :, 3] == 255, seen)
        assert np.array_equal(got[seen][:, :3], frame0[seen][:, [2, 1, 0]])


# ---------------------------------------------------------------- several GPUs

def test_multi_gpu_equals_single(cuda_lib, xb, cpu):
    import torch
    ndev = max(1, torch.cuda.device_count())
    devices = list(range(ndev)) if ndev > 1 else [0, 0]
    gifs, webps = synthetic_gifs(), webp_animations(cpu)
    files = list(gifs.values())[:6] + list(webps.values())[:4]
    opt = opts(".webp")
    want, wst = xb.transform(files, opt)
    m = abi.MultiBatch(cuda_lib, devices, arena_bytes=4 << 30)
    try:
        outs, status = m.transform(files, opt)
        assert status == wst == [0] * len(files) and outs == want
        assert sum(m.stats(g)["grid_items"] for g in range(len(devices))) == len(files)
    finally:
        m.close()
