"""GPU: lp_xbatch_decode_clips -- up to T frames of every item, spread over the animation, in a caller's device tensor.

Every expectation comes from outside the call:
  - T = 1 is lp_xbatch_decode_frames, byte for byte, over its mixed corpus;
  - sampling and timing: animations built with Pillow whose frame k is a solid colour that names k, with chosen delays;
    the colour of every slot must name the frame the rule floor(t * F / T) selects, and frame_index / start_ms / nframes
    must follow from the delays written;
  - pixels: lp_transform to lossless animated WebP with no limits, whose every frame is an exact copy of the frame
    Transform handed its encoder, decoded by the per-image WebP decoder (U8 equal, float dtypes within one ulp);
  - routing is asserted exactly (grid_items / fallback_items)."""
import ctypes as C
import io

import cv2
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch import rgb_png
from tests.test_gpu_xbatch_frames import BIAS, DTYPES, SCALE, assert_slice, corpus, expected_slice, tensor
from tests.test_gpu_xbatch_hdr_png import png_file, source
from tests.test_gpu_xbatch_jpeg_webp import cv2_jpeg
from tests.test_gpu_xbatch_renditions import pil_webp_animation

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
TIMEOUT = 10**12
FIT, RESIZE = abi.ImageOpsFit, abi.ImageOpsResize
BAD_ARGUMENT = -10  # LP_ERR_BAD_ARGUMENT


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def opts(w, h, method, **kw):
    return abi.ImageOptions(FileType=".jpeg", Width=w, Height=h, ResizeMethod=method, EncodeOptions={abi.JpegQuality: 50},
                            EncodeTimeout_ns=TIMEOUT, **kw)


def clips(xb, files, opt, T, H, W, ch=4, nchw=False, rgb=False, dtype="u8", fill=0x5A):
    """(tensor on the host as n x T x slice, width, height, nframes, frame_index, start_ms, status)"""
    n = len(files)
    t = tensor(n * T, H, W, ch, dtype, nchw, fill)
    out = xb.decode_clips(files, opt, T, t.data_ptr(), t.numel() * t.element_size(), H, W, ch, nchw, rgb, dtype, SCALE, BIAS)
    return (t.cpu().reshape(n, T, *t.shape[1:]),) + out


def selected(F, T):
    return list(range(F)) if F <= T else [t * F // T for t in range(T)]


# ------------------------------------------------------------------ T = 1 is lp_xbatch_decode_frames

@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("nchw", [False, True])
def test_one_frame_is_decode_frames(xb, dtype, ch, nchw):
    files = [f for _, f in corpus()]
    n, H, W = len(files), 72, 128
    for opt in (opts(64, 64, FIT), opts(40, 120, RESIZE, NormalizeOrientation=True)):
        a = tensor(n, H, W, ch, dtype, nchw)
        w0, h0, st0 = xb.decode_frames(files, opt, a.data_ptr(), a.numel() * a.element_size(), H, W, ch, nchw, True, dtype,
                                       SCALE, BIAS)
        got, w, h, nf, index, start, st = clips(xb, files, opt, 1, H, W, ch, nchw, True, dtype)
        assert (w, h, st) == (w0, h0, st0)
        assert torch.equal(got[:, 0].contiguous().view(torch.uint8), a.cpu().view(torch.uint8))
        assert index == [0 if s == 0 else -1 for s in st] and start == [0] * n
        assert all((f >= 1) == (s == 0) for f, s in zip(nf, st))


# ------------------------------------------------------------------ sampling and timing

def colour(k):
    """B, G, R of frame k: two channels name it, 24 / 20 apart"""
    return (90, 16 + (k // 10) * 20, 16 + (k % 10) * 24)


def frame_of(px):
    """the frame whose colour is nearest the pixel (B, G, R), and the distance"""
    d = [max(abs(int(px[c]) - colour(k)[c]) for c in range(3)) for k in range(110)]
    k = int(np.argmin(d))
    return k, d[k]


def gif_delays(F):
    """centiseconds: 0 and 1 included, and one frame of 655 s"""
    return [[0, 1, 65500][k] if k < 3 else 2 + (k * 7) % 40 for k in range(F)]


def solid_gif(F, w=40, h=30):
    from PIL import Image
    ims = [Image.new("RGB", (w, h), colour(k)[::-1]) for k in range(F)]
    bio = io.BytesIO()
    ims[0].save(bio, "GIF", save_all=True, append_images=ims[1:], duration=[10 * d for d in gif_delays(F)], loop=0,
                optimize=False, disposal=1)
    return bio.getvalue(), [10 * d for d in gif_delays(F)]


def solid_webp(F, w=40, h=30):
    from PIL import Image
    ims = [Image.new("RGBA", (w, h), colour(k)[::-1] + (255,)) for k in range(F)]
    durs = [10 + (k * 13) % 90 for k in range(F)]
    bio = io.BytesIO()
    ims[0].save(bio, "WEBP", save_all=True, append_images=ims[1:], duration=durs, loop=0, lossless=True)
    return bio.getvalue(), durs


@pytest.mark.parametrize("route", ["grid", "per_image"])
@pytest.mark.parametrize("T", [1, 3, 8])
def test_sampling_and_timing(xb, T, route):
    """the grid (Resize to 20 x 15), and the per-image route's ClipEncoder (NoResize: animations go per image)"""
    from PIL import Image
    counts = sorted({F for F in (1, 2, T - 1, T, T + 1, 2 * T, 3 * T + 1, 100) if F >= 1})
    files, durs, Fs = [], [], []
    for F in counts:
        for make in (solid_gif, solid_webp):
            data, d = make(F)
            assert Image.open(io.BytesIO(data)).n_frames == F  # (Pillow kept every frame)
            files.append(data)
            durs.append(d)
            Fs.append(F)
    grid = route == "grid"
    opt, H, W, fw, fh = (opts(20, 15, RESIZE), 16, 24, 20, 15) if grid else (opts(0, 0, abi.ImageOpsNoResize), 32, 48, 40, 30)
    got, w, h, nf, index, start, st = clips(xb, files, opt, T, H, W, ch=3)
    assert st == [0] * len(files) and nf == Fs
    assert xb.stats()["grid_items" if grid else "fallback_items"] == len(files)
    for i, F in enumerate(Fs):
        sel = selected(F, T)
        assert index[i * T:(i + 1) * T] == sel + [-1] * (T - len(sel)), f"item {i} (F {F})"
        assert start[i * T:(i + 1) * T] == [sum(durs[i][:k]) for k in sel] + [0] * (T - len(sel)), f"item {i} (F {F})"
        assert (w[i], h[i]) == (fw, fh)
        for t in range(T):
            s = got[i, t].numpy()
            if t >= len(sel):
                assert not s.any(), f"item {i} slot {t}: unused but not zero"
                continue
            k, d = frame_of(s[7, 10])
            assert (k, d <= 3) == (sel[t], True), f"item {i} (F {F}) slot {t}: frame {k} at distance {d}, want {sel[t]}"
            assert not s[fh:].any() and not s[:, fw:].any()


# ------------------------------------------------------------------ pixels against lp_transform to lossless WebP

def webp_frames_of_transform(lib, data, opt):
    """(status, frames): every frame lp_transform(data, opt with lossless ".webp", no limits) hands its encoder"""
    o = abi.ImageOptions(**{**opt.__dict__, "FileType": ".webp", "EncodeOptions": {abi.WebpQuality: 101}, "MaxEncodeFrames": 0,
                            "MaxEncodeDuration_ns": 0, "DisableAnimatedOutput": False, "EncodeTimeout_ns": 10**15})
    try:
        out = lib.transform(data, o, dst_cap=1 << 27)
    except abi.LilliputError as e:
        return e.code, []
    _, frames, metas, rc = lib.webp_frames(out)
    assert rc == 0
    for f, m in zip(frames, metas):
        assert (m["x"], m["y"]) == (0, 0) and f.shape[:2] == frames[0].shape[:2]  # (full-canvas frames)
    return 0, frames


def gif_disposals(seed, w, h, n):
    """local palettes, a transparent index, every disposal"""
    from PIL import Image
    ims = [Image.fromarray(synth_image(seed + k, w, h, 3)[:, :, ::-1].copy()).quantize(32 + 8 * k) for k in range(n)]
    bio = io.BytesIO()
    ims[0].save(bio, "GIF", save_all=True, append_images=ims[1:], duration=[30 + 10 * k for k in range(n)], loop=0,
                transparency=0, disposal=[k % 4 for k in range(n)], optimize=False)
    return bio.getvalue()


def scrolling_gif(seed, w, h, n, step=4):
    """config 4 in miniature: one global palette, the field scrolled `step` px per frame"""
    from PIL import Image
    base = Image.fromarray(synth_image(seed, w, h, 3, noise=0.0)[:, :, ::-1].copy()).quantize(64)
    idx = np.asarray(base)
    ims = []
    for k in range(n):
        im = Image.fromarray(np.roll(idx, step * k, axis=1), "P")
        im.putpalette(base.getpalette())
        ims.append(im)
    bio = io.BytesIO()
    ims[0].save(bio, "GIF", save_all=True, append_images=ims[1:], duration=40, loop=0)
    return bio.getvalue()


def animations():
    return [
        ("gif_disposals", gif_disposals(40, 90, 70, 11)),
        ("gif_scrolling", scrolling_gif(41, 320, 180, 24)),
        ("webp_lossy", pil_webp_animation(42, 96, 64, 9, lossless=False)),
        ("webp_lossless", pil_webp_animation(51, 64, 48, 7, lossless=True)),
        ("jpeg_still", cv2_jpeg(synth_image(60, 200, 150, 3), 90)),
        ("png_still", rgb_png(synth_image(61, 120, 90, 4))),
    ]


def riff_chunks(data, at=12):
    """[(fourcc, payload)] of a RIFF body from `at`"""
    out = []
    while at + 8 <= len(data):
        n = int.from_bytes(data[at + 4:at + 8], "little")
        out.append((data[at:at + 4], data[at + 8:at + 8 + n]))
        at += 8 + n + (n & 1)
    return out


def chunk(tag, payload):
    return tag + len(payload).to_bytes(4, "little") + payload + (b"\0" if len(payload) & 1 else b"")


def anmf_webp(w, h, frames):
    """An animated WebP written chunk by chunk: frames are (BGRA pixels, x, y, lossless, blend, dispose, ms), x and y
    even; blend: alpha-blend onto the canvas (else copy), dispose: clear the rectangle to transparent afterwards"""
    from PIL import Image
    body = b""
    for px, x, y, lossless, blend, dispose, ms in frames:
        bio = io.BytesIO()
        Image.fromarray(px[:, :, [2, 1, 0, 3]].copy(), "RGBA").save(bio, "WEBP", lossless=lossless, quality=80)
        image = b"".join(chunk(t, p) for t, p in riff_chunks(bio.getvalue()) if t in (b"ALPH", b"VP8 ", b"VP8L"))
        fh, fw = px.shape[:2]
        head = b"".join(v.to_bytes(3, "little") for v in (x // 2, y // 2, fw - 1, fh - 1, ms))
        body += chunk(b"ANMF", head + bytes([(0 if blend else 2) | (1 if dispose else 0)]) + image)
    vp8x = chunk(b"VP8X", bytes([0x12, 0, 0, 0]) + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little"))
    data = b"WEBP" + vp8x + chunk(b"ANIM", bytes([0, 0, 0, 0, 0, 0])) + body
    return b"RIFF" + len(data).to_bytes(4, "little") + data


def anmf_headers(data):
    """(x, y, w, h, blend, dispose, image chunks) of every ANMF chunk, parsed back from the file"""
    out = []
    for tag, p in riff_chunks(data):
        if tag == b"ANMF":
            v = [int.from_bytes(p[k:k + 3], "little") for k in range(0, 15, 3)]
            out.append((2 * v[0], 2 * v[1], v[2] + 1, v[3] + 1, not p[15] & 2, bool(p[15] & 1),
                        [t for t, _ in riff_chunks(p, 16)]))
    return out


def sprite_animation(seed, w=96, h=64):
    """A lossy opaque background, then eight translucent sprites (lossless and lossy + ALPH) moving over it, most blended,
    some copied, some disposed to background"""
    rng = np.random.default_rng(seed)
    bg = np.concatenate([synth_image(seed, w, h, 3), np.full((h, w, 1), 255, np.uint8)], 2)
    frames = [(bg, 0, 0, False, False, False, 40)]
    for k in range(1, 9):
        sw, sh = (40, 30) if k % 4 == 0 else (24, 18)
        px = rng.integers(0, 256, (sh, sw, 4), dtype=np.uint8)
        px[:, :, 3] = np.linspace(40, 220, sw, dtype=np.uint8)[None, :]  # translucent, varying across the sprite
        x, y = (6 * k) % (w - sw) // 2 * 2, (4 * k) % (h - sh) // 2 * 2
        frames.append((px, x, y, k % 2 == 1, k % 3 != 2, k in (2, 5, 7), 20 + 10 * k))
    return anmf_webp(w, h, frames)


@pytest.mark.parametrize("T", [2, 3, 4])
def test_frames_composited_but_not_stored(cuda_lib, xb, T):
    """WebP animations whose sub-rectangles blend over and dispose from the canvas state that unstored frames built"""
    files = [sprite_animation(100), sprite_animation(101)]
    for data in files:
        heads = anmf_headers(data)
        assert len(heads) == 9
        assert any(hw < 96 or hh < 64 for _, _, hw, hh, *_ in heads), "no sub-rectangle"
        assert any(b for *_, b, _, _ in heads) and any(not b for *_, b, _, _ in heads), "not both blend methods"
        assert any(d for *_, d, _ in heads), "no dispose to background"
        assert any(b"ALPH" in c for *_, c in heads) and any(b"VP8L" in c for *_, c in heads), "no ALPH or no VP8L frame"
    opt = opts(80, 60, RESIZE)
    got, w, h, nf, index, start, st = clips(xb, files, opt, T, 64, 80, ch=4)
    assert st == [0, 0] and nf == [9, 9] and xb.stats()["grid_items"] == 2
    for i, data in enumerate(files):
        code, frames = webp_frames_of_transform(cuda_lib, data, opt)
        assert code == 0 and len(frames) == 9
        sel = selected(9, T)
        assert index[i * T:(i + 1) * T] == sel
        for t, f in enumerate(sel):
            assert_slice(got[i, t], expected_slice(frames[f], 64, 80, 4, False, False, "u8", SCALE, BIAS), "u8",
                         f"item {i} slot {t} (frame {f})")


@pytest.mark.parametrize("T,opt,dtype,nchw", [
    (8, opts(96, 96, FIT), "u8", False),
    (3, opts(64, 48, RESIZE), "f16", True),
    (5, opts(50, 80, FIT), "f32", False),
])
def test_frames_equal_transform(cuda_lib, xb, T, opt, dtype, nchw):
    named = animations()
    files = [f for _, f in named]
    H, W, ch = 96, 96, 4
    got, w, h, nf, index, start, st = clips(xb, files, opt, T, H, W, ch, nchw, True, dtype)
    assert xb.stats()["grid_items"] == len(files)
    for i, (name, data) in enumerate(named):
        code, frames = webp_frames_of_transform(cuda_lib, data, opt)
        assert st[i] == code == 0, name
        sel = selected(len(frames), T)
        assert nf[i] == len(frames) and index[i * T:(i + 1) * T] == sel + [-1] * (T - len(sel)), name
        assert (w[i], h[i]) == (frames[0].shape[1], frames[0].shape[0]), name
        for t in range(T):
            want = expected_slice(frames[sel[t]] if t < len(sel) else None, H, W, ch, nchw, True, dtype, SCALE, BIAS)
            assert_slice(got[i, t], want, dtype, f"{name} slot {t}")


# ------------------------------------------------------------------ routing

def gif_frame_data(data):
    """[(start, end)] of every frame's sub-block run (behind the LZW minimum code size)"""
    p = 13 + ((3 << ((data[10] & 7) + 1)) if data[10] & 0x80 else 0)
    out = []
    while data[p] != 0x3B:
        image = data[p] == 0x2C
        if image:
            flags = data[p + 9]
            p += 10 + ((3 << ((flags & 7) + 1)) if flags & 0x80 else 0) + 1
        else:  # an extension: introducer, label
            p += 2
        s = p
        while data[p]:
            p += data[p] + 1
        p += 1
        if image:
            out.append((s, p))
    return out


def damaged(data, frame):
    """every code-stream byte of one frame set to 0xFF, sub-block lengths kept"""
    b = bytearray(data)
    s, e = gif_frame_data(data)[frame]
    p = s
    while b[p]:
        b[p + 1:p + 1 + b[p]] = b"\xff" * b[p]
        p += b[p] + 1
    return bytes(b)


def test_routing(cuda_lib, xb):
    T = 4
    anim = scrolling_gif(70, 64, 48, 20)  # frames 0, 5, 10, 15 selected: L = 15
    assert len(gif_frame_data(anim)) == 20
    behind, at_l, before = damaged(anim, 18), damaged(anim, 15), damaged(anim, 7)
    opt = opts(32, 32, FIT)
    well = [anim, pil_webp_animation(71, 48, 40, 6, lossless=False), gif_disposals(72, 50, 40, 5)]
    *_, st = clips(xb, well, opt, T, 32, 32)
    assert st == [0, 0, 0] and xb.stats()["grid_items"] == 3
    # damage behind L is never read, on either route
    got, *_, st = clips(xb, [behind, anim], opt, T, 32, 32)
    assert st == [0, 0] and xb.stats()["grid_items"] == 2
    assert torch.equal(got[0], got[1])
    # at or before L: Transform's error (lossless WebP output decodes every frame, and fails at the same one)
    for bad in (at_l, before):
        got, w, h, nf, index, start, st = clips(xb, [bad], opt, T, 32, 32)
        code, _ = webp_frames_of_transform(cuda_lib, bad, opt)
        assert st == [code] and code != 0
        assert (w, h, nf, index, start) == ([0], [0], [0], [-1] * T, [0] * T) and not got.any()
        assert xb.stats()["fallback_items"] == 1
    # NoResize, gray PNGs and eXIf-rotated PNGs: per image
    *_, st = clips(xb, [anim], opts(0, 0, abi.ImageOpsNoResize), T, 64, 64)
    assert st == [0] and xb.stats()["fallback_items"] == 1
    gray = png_file(synth_image(73, 50, 40, 1).reshape(40, 50, 1), 0, 8)
    exif = png_file(source(74, 70, 50, "rgb", 8)[1], 2, 8, orientation=6)
    got, w, h, nf, index, start, st = clips(xb, [gray, exif], opt, T, 32, 32)
    assert st == [0, 0] and nf == [1, 1] and index == [0, -1, -1, -1] * 2 and xb.stats()["fallback_items"] == 2
    assert not got[:, 1:].any()


# ------------------------------------------------------------------ memory per task

def test_long_animations_share_a_small_arena(cuda_lib):
    """32 animations of 400 frames of 320 x 240: 123 MB of canvases each and as much again resized, more than a lane of
    this context (half its arena) holds; eight canvases each fit, so every item takes the grid"""
    distinct = [scrolling_gif(80 + k, 320, 240, 400, step=3) for k in range(2)]
    files = distinct * 16
    x = abi.XBatch(cuda_lib, 0, arena_bytes=384 << 20)
    try:
        T, opt = 8, opts(64, 64, FIT)
        got, w, h, nf, index, start, st = clips(x, files, opt, T, 64, 64)
        assert st == [0] * 32 and x.stats()["grid_items"] == 32 and nf == [400] * 32
    finally:
        x.close()
    for k, data in enumerate(distinct):
        _, frames = webp_frames_of_transform(cuda_lib, data, opt)
        for t, f in enumerate(selected(400, T)):
            want = expected_slice(frames[f], 64, 64, 4, False, False, "u8", SCALE, BIAS)
            for i in (k, k + 2 * 15):
                assert_slice(got[i, t], want, "u8", f"item {i} slot {t}")


# ------------------------------------------------------------------ arguments

def test_bad_arguments_write_nothing(cuda_lib, xb):
    files = [scrolling_gif(90, 40, 30, 6), cv2_jpeg(synth_image(91, 60, 40, 3), 90)]
    n, H, W = len(files), 32, 32
    opt = opts(32, 32, FIT)
    t = tensor(n * 4, H, W, 3, "u8", False, fill=0xA5)
    nbytes = t.numel()
    for T, size in ((0, nbytes), (4097, nbytes), (4, nbytes - 1), (5, nbytes)):
        with pytest.raises(abi.LilliputError) as e:
            xb.decode_clips(files, opt, T, t.data_ptr(), size, H, W, 3)
        assert e.value.code == BAD_ARGUMENT, (T, size)
    l = cuda_lib.l
    ptrs, lens, keep = abi.Batch._ptr_arrays(files)
    arrays = [(C.c_int * n)() for _ in range(4)] + [(C.c_int * (n * 4))(), (C.c_int64 * (n * 4))()]
    ft = abi._FrameTensor(t.data_ptr(), nbytes, H, W, 3, 0, 1, 0, (C.c_float * 4)(1, 1, 1, 1), (C.c_float * 4)())
    copt = opt._c()
    for k in range(6):  # width, height, nframes, status, frame_index, start_ms: each null in turn
        a = list(arrays)
        a[k] = None
        w, h, nf, status, index, start = a
        assert l.lp_xbatch_decode_clips(xb.h, ptrs, lens, n, C.byref(copt), 4, C.byref(ft), w, h, nf, index, start, status) == \
            BAD_ARGUMENT
    assert bool((t.cpu() == 0xA5).all()), "a refused call wrote into the tensor"
    assert xb.decode_clips([], opt, 4, t.data_ptr(), nbytes, H, W, 3) == ([], [], [], [], [], [])
    assert bool((t.cpu() == 0xA5).all())
