"""GPU: lp_xbatch_encode_clips -- animations written from clips in a caller's device tensor.

An item of nframes >= 2 must answer as lp_transform(A_i, opt) does, where A_i is an animated WebP this test builds chunk
by chunk: VP8X (animation flag, alpha flag exactly for four channels), ANIM (background 0xFFFFFFFF, the loop count) and
one full-canvas ANMF per frame with no blending, no disposal and the caller's duration, whose image is Pillow's exact
lossless VP8L encoding of the u8 frame the numpy restatement of the conversion gives.  Before any comparison the per-image
WebP decoder must read A_i back as exactly those frames, durations, loop count and background.  An item of one frame must
answer as lp_xbatch_encode_frames does for its first slice, i.e. as lp_transform of a PNG of the frame.

Which items take the grid is asserted exactly, against the gates written down in xbatch.cu and DESIGN.md (predicted_grid).
"""
import ctypes as C
import io

import numpy as np
import pytest

from lilliput_b200 import abi
from tests.test_gpu_xbatch_clips import chunk, riff_chunks, scrolling_gif, gif_disposals, sprite_animation
from tests.test_gpu_xbatch_encode_frames import DTYPES, LBIAS, LSCALE, device_tensor, restate
from tests.test_gpu_xbatch_encode_frames import reference as png_reference
from tests.test_gpu_xbatch_renditions import pil_webp_animation

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
TIMEOUT = 10**12
FIT, RESIZE, NO_RESIZE = abi.ImageOpsFit, abi.ImageOpsResize, abi.ImageOpsNoResize
BAD = -10  # LP_ERR_BAD_ARGUMENT
CV_8UC3, CV_8UC4 = 16, 24


# ---------------------------------------------------------------- A_i, the file each clip item stands for

def vp8l(frame):
    """Pillow's exact lossless encoding of a u8 BGR / BGRA frame: the VP8L chunk alone"""
    from PIL import Image
    rgb = frame[:, :, [2, 1, 0, 3][:frame.shape[2]]].copy()
    bio = io.BytesIO()
    Image.fromarray(rgb, "RGBA" if frame.shape[2] == 4 else "RGB").save(bio, "WEBP", lossless=True, exact=True, quality=0,
                                                                          method=0)
    chunks = riff_chunks(bio.getvalue())
    assert [t for t, _ in chunks] == [b"VP8L"], [t for t, _ in chunks]
    return chunk(b"VP8L", chunks[0][1])


def clip_webp(frames, durations, loops):
    """A_i: frames (u8 BGR / BGRA, one size) as full-canvas, no-blend, no-dispose ANMF frames"""
    h, w, ch = frames[0].shape
    body = b""
    for f, ms in zip(frames, durations):
        head = b"".join(v.to_bytes(3, "little") for v in (0, 0, w - 1, h - 1, ms))
        body += chunk(b"ANMF", head + bytes([2]) + vp8l(f))
    vp8x = chunk(b"VP8X", bytes([0x02 | (0x10 if ch == 4 else 0), 0, 0, 0]) + (w - 1).to_bytes(3, "little") +
                 (h - 1).to_bytes(3, "little"))
    anim = chunk(b"ANIM", (0xFFFFFFFF).to_bytes(4, "little") + loops.to_bytes(2, "little"))
    data = b"WEBP" + vp8x + anim + body
    return b"RIFF" + len(data).to_bytes(4, "little") + data


def check_oracle_file(lib, data, frames, durations, loops):
    """the per-image decoder reads A_i back exactly as built"""
    info, got, metas, rc = lib.webp_frames(data)
    h, w, ch = frames[0].shape
    assert rc == 0 and len(got) == len(frames)
    assert (info["width"], info["height"], info["num_frames"]) == (w, h, len(frames))
    assert info["pixel_type"] == (CV_8UC4 if ch == 4 else CV_8UC3)
    assert (info["loop_count"], info["bg_color"]) == (loops, 0xFFFFFFFF)
    for k, (f, m) in enumerate(zip(got, metas)):
        assert f.shape == frames[k].shape and np.array_equal(f, frames[k]), f"frame {k} is not exact"
        assert (m["x"], m["y"], m["delay"], m["blend"], m["dispose"]) == (0, 0, durations[k], 1, 0), f"frame {k}: {m}"


def clip_reference(lib, frames, durations, loops, opt, out_cap, max_size=8192):
    """(status, bytes) an item must have: lp_transform(A_i) for several frames, encode_frames' (a PNG's) for one"""
    if len(frames) == 1:
        return png_reference(lib, frames[0], opt, out_cap, max_size)
    data = clip_webp(frames, durations, loops)
    check_oracle_file(lib, data, frames, durations, loops)
    try:
        return 0, lib.transform(data, opt, dst_cap=out_cap, max_size=max_size)
    except abi.LilliputError as e:
        return e.code, b""


def predicted_grid(opt, nframes):
    """the gates of xbatch.cu (parse_frame_pair, clip_gates) for items of valid arguments within max_size"""
    webp = opt.FileType == ".webp"
    n = 0
    for nf in nframes:
        if nf == 1:
            n += not (opt.MaxEncodeDuration_ns < 0 or opt.FileType == ".gif" or
                      (webp and (opt.EncodeTimeout_ns <= 0 or opt.MaxEncodeFrames == 1)))
        else:
            n += (opt.FileType != ".gif" and opt.MaxEncodeDuration_ns == 0 and
                  (not webp or (opt.MaxEncodeFrames == 0 and (opt.DisableAnimatedOutput or opt.EncodeTimeout_ns > 0))))
    return n


# ---------------------------------------------------------------- designed clips

def clip_frames(seed, w, h, ch, nf):
    """nf u8 frames: random colours, every alpha class (0, 127, 128, 255 and ramps), colour kept under alpha 0, and a
    moving block so no two frames are equal"""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(nf):
        f = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)
        if w > 4 and h > 4:
            y, x = np.mgrid[0:h, 0:w]
            f[..., 0] = np.where((x - k) % w < w // 3, (x * 7 + y * 3 + k) % 256, f[..., 0])
        if ch == 4:
            cls = (np.arange(w)[None, :] + np.arange(h)[:, None] + k) % 5
            f[..., 3] = np.choose(cls, [0, 127, 128, 255, (np.arange(w)[None, :] * 37 + k) % 256 + 0 * cls])
        out.append(f)
    return out


DURATION_CLASSES = [0, 1, 65535, 0xFFFFFF]


def durations_for(seed, nf):
    """every duration class, and others between"""
    rng = np.random.default_rng(seed)
    return [DURATION_CLASSES[(seed + k // 2) % 4] if k % 2 == 0 else int(rng.integers(0, 400)) for k in range(nf)]


BOX_H, BOX_W = 32, 40


def clip_batch(T, ch, seed=0, sizes=None):
    """items of nframes 2, T - 1, T and 1 (sizes 1x1, odd, box-sized), each (frames, durations)"""
    sizes = sizes or [(1, 1), (37, 23), (BOX_W, BOX_H), (13, 29)]
    counts = [2, max(T - 1, 1), T, 1]
    return [(clip_frames(seed + 10 * k, w, h, ch, nf), durations_for(seed + k, nf)) for k, ((w, h), nf) in enumerate(zip(sizes, counts))]


def clip_tensor(items, T, H, W, ch, dtype="u8", nchw=False, rgb=False, scale=None, offset=0):
    """the device tensor of items (n * T slices, unused slots filled with 0x5A-ish noise), widths, heights, nframes and
    durations (unused slots -1)"""
    n = len(items)
    a = np.full((n * T, H, W, ch), 90.0, np.float64)
    ms = []
    for i, (frames, durs) in enumerate(items):
        for t, f in enumerate(frames):
            v = f.astype(np.float64)
            a[i * T + t, :f.shape[0], :f.shape[1]] = v[..., [2, 1, 0, 3][:ch]] if rgb else v
        ms += list(durs) + [-1] * (T - len(durs))
    if scale is not None:
        a = a / scale
    if nchw:
        a = a.transpose(0, 3, 1, 2)
    t, keep = device_tensor(a, dtype, offset)
    w = [f[0].shape[1] for f, _ in items]
    h = [f[0].shape[0] for f, _ in items]
    return t, keep, w, h, [len(f) for f, _ in items], ms


def encode(xb, t, T, nf, w, h, ms, opt, ch, loops=0, nchw=False, rgb=False, dtype="u8", scale=None, bias=None, out_cap=1 << 22):
    H, W = (t.shape[2], t.shape[3]) if nchw else (t.shape[1], t.shape[2])
    return xb.encode_clips(t.data_ptr(), t.numel() * t.element_size(), T, nf, w, h, ms, opt, H, W, loops, ch, nchw, rgb, dtype,
                           scale, bias, out_cap)


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def check_items(lib, items, loops, opt, outs, st, out_cap=1 << 22, max_size=8192):
    for i, (frames, durs) in enumerate(items):
        code, want = clip_reference(lib, frames, durs, loops, opt, out_cap, max_size)
        what = f"item {i} ({len(frames)} frames of {frames[0].shape})"
        assert st[i] == code, f"{what}: status {st[i]}, lp_transform {code}"
        assert outs[i] == want, f"{what}: {len(outs[i])} bytes differ from lp_transform's {len(want)}"


# ---------------------------------------------------------------- the contract

SINKS = {
    "webp_q1": (".webp", {abi.WebpQuality: 1}),
    "webp_q50": (".webp", {abi.WebpQuality: 50}),
    "webp_q85": (".webp", {abi.WebpQuality: 85}),
    "webp_q100": (".webp", {abi.WebpQuality: 100}),
    "webp_q101": (".webp", {abi.WebpQuality: 101}),
    "jpeg": (".jpeg", {abi.JpegQuality: 85}),
    "png": (".png", {}),
    "gif": (".gif", {}),
}
GEOMETRIES = {"fit": (24, 20, FIT), "resize": (30, 18, RESIZE), "no_resize": (0, 0, NO_RESIZE)}


def options(sink, geometry, **kw):
    ext, eo = SINKS[sink]
    w, h, m = GEOMETRIES[geometry]
    return abi.ImageOptions(FileType=ext, Width=w, Height=h, ResizeMethod=m, EncodeOptions=dict(eo),
                            **{"EncodeTimeout_ns": TIMEOUT, **kw})


@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("sink", list(SINKS))
def test_contract(cuda_lib, xb, sink, geometry):
    """nframes 2, T - 1, T and 1 for T in 2, 8, 33, three and four channels (u8 NHWC BGR, and f16 NCHW RGB at scale 255),
    durations 0, 1, 65535 and 0xFFFFFF, loop counts 0, 1 and 65535: every item's status and bytes, and the exact split"""
    opt = options(sink, geometry)
    for T, loops in ((2, 0), (8, 1), (33, 65535)):
        for ch in (3, 4):
            items = clip_batch(T, ch, seed=T + ch)
            if ch == 3:
                t, keep, w, h, nf, ms = clip_tensor(items, T, BOX_H, BOX_W, 3)
                outs, st = encode(xb, t, T, nf, w, h, ms, opt, 3, loops)
            else:
                t, keep, w, h, nf, ms = clip_tensor(items, T, BOX_H, BOX_W, 4, "f16", True, True, 255.0)
                got, amb = restate(t, "f16", 4, True, True, [255.0] * 4, [0.0] * 4)  # (the frames come back exactly)
                assert not amb.any()
                for i, (frames, _) in enumerate(items):
                    for k, f in enumerate(frames):
                        assert np.array_equal(got[i * T + k, :f.shape[0], :f.shape[1]], f)
                outs, st = encode(xb, t, T, nf, w, h, ms, opt, 4, loops, True, True, "f16", [255.0] * 4)
            s = xb.stats()
            check_items(cuda_lib, items, loops, opt, outs, st)
            want = predicted_grid(opt, nf)
            assert (s["grid_items"], s["fallback_items"]) == (want, len(items) - want), (T, ch)
            if sink != "gif":
                assert want == len(items)


@pytest.mark.parametrize("sink", ["webp_q85", "webp_q101", "png"])
def test_small_out_cap(cuda_lib, xb, sink):
    """a buffer too small for some files: the status lp_transform gives, where it gives it"""
    T = 8
    items = clip_batch(T, 4, seed=5)
    t, keep, w, h, nf, ms = clip_tensor(items, T, BOX_H, BOX_W, 4)
    opt = options(sink, "fit")
    outs, st = encode(xb, t, T, nf, w, h, ms, opt, 4, out_cap=600)
    assert any(s != 0 for s in st), st
    check_items(cuda_lib, items, 0, opt, outs, st, out_cap=600)


@pytest.mark.parametrize("geometry", ["fit", "no_resize"])
def test_frames_over_max_size(cuda_lib, geometry):
    """a context with max_size 32: clips over it in either side answer as lp_transform(A_i, ..., max_size 32) does"""
    T = 3
    items = clip_batch(T, 3, seed=9, sizes=[(40, 20), (20, 30), (33, 33), (32, 32)])
    opt = options("webp_q85", geometry)
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30, max_size=32)
    try:
        t, keep, w, h, nf, ms = clip_tensor(items, T, 40, 40, 3)
        outs, st = encode(small, t, T, nf, w, h, ms, opt, 3)
        assert small.stats()["grid_items"] == 2  # (20 x 30 and 32 x 32)
    finally:
        small.close()
    check_items(cuda_lib, items, 0, opt, outs, st, max_size=32)


# ---------------------------------------------------------------- options

NF = 5
OPTIONS = {
    "disable_animated": {"DisableAnimatedOutput": True},
    "disable_animated_timeout_0": {"DisableAnimatedOutput": True, "EncodeTimeout_ns": 0},
    "max_frames_1": {"MaxEncodeFrames": 1},
    "max_frames_nf_minus_1": {"MaxEncodeFrames": NF - 1},
    "max_frames_nf": {"MaxEncodeFrames": NF},
    "max_frames_nf_plus_1": {"MaxEncodeFrames": NF + 1},
    "max_duration_neg": {"MaxEncodeDuration_ns": -1},
    "max_duration_below": {"MaxEncodeDuration_ns": 250 * 10**6},
    "max_duration_above": {"MaxEncodeDuration_ns": 10**10},
    "timeout_0": {"EncodeTimeout_ns": 0},
    "timeout_positive": {"EncodeTimeout_ns": 10**11},
}


@pytest.mark.parametrize("option", list(OPTIONS))
@pytest.mark.parametrize("sink", ["webp_q85", "webp_q101", "jpeg", "png", "gif"])
def test_options(cuda_lib, xb, sink, option):
    """clips of 5 frames of 100 ms (and one of one frame): status, bytes and the exact split under every option class"""
    T = 6
    sizes = [(40, 32), (17, 9), (1, 1), (25, 31)]
    items = [(clip_frames(70 + k, w, h, 4, NF if k < 3 else 1), [100] * (NF if k < 3 else 1)) for k, (w, h) in enumerate(sizes)]
    t, keep, w, h, nf, ms = clip_tensor(items, T, BOX_H + 8, BOX_W, 4)
    opt = options(sink, "fit", **OPTIONS[option])
    outs, st = encode(xb, t, T, nf, w, h, ms, opt, 4, loops=3)
    s = xb.stats()
    check_items(cuda_lib, items, 3, opt, outs, st)
    want = predicted_grid(opt, nf)
    assert (s["grid_items"], s["fallback_items"]) == (want, len(items) - want)


# ---------------------------------------------------------------- T = 1 and one-frame items are encode_frames

L_H, L_W = 19, 37
L_SIZES = [(37, 19), (23, 11), (1, 1)]


def designed_values(seed, dtype, ch, nchw, n):
    rng = np.random.default_rng(seed)
    if dtype == "u8":
        a = rng.integers(0, 256, (n, L_H, L_W, ch)).astype(np.float64)
    else:
        v = rng.uniform(-40, 300, (n, L_H, L_W, ch))
        ties = rng.integers(-3, 258, (n, L_H, L_W, ch)) + 0.5
        v = np.where(rng.random((n, L_H, L_W, ch)) < 0.3, ties, v)
        a = (v - np.array(LBIAS[:ch])) / np.array(LSCALE[:ch])
        special = rng.random((n, L_H, L_W, ch))
        a = np.where(special < 0.02, np.nan, a)
        a = np.where((special >= 0.02) & (special < 0.04), np.inf, a)
    return a.transpose(0, 3, 1, 2) if nchw else a


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("rgb", [False, True])
@pytest.mark.parametrize("nchw", [False, True])
def test_one_frame_items_are_encode_frames(xb, dtype, ch, rgb, nchw):
    """T = 1, and one-frame items of T = 3 (slice 3i): the bytes, statuses and split of lp_xbatch_encode_frames over the
    same slices, to .png under NoResize and to .webp under Fit.  RGB tensors start one element past a 16-byte boundary."""
    n, T = len(L_SIZES), 3
    t, keep = device_tensor(designed_values(len(dtype) + 2 * ch + 5 * rgb + 11 * nchw, dtype, ch, nchw, n * T), dtype,
                            offset=1 if rgb else 0)
    assert (t.data_ptr() % 16 != 0) == rgb
    w, h = [s[0] for s in L_SIZES], [s[1] for s in L_SIZES]
    H, W = L_H, L_W
    nbytes = t.numel() * t.element_size()
    for opt in (abi.ImageOptions(FileType=".png", ResizeMethod=NO_RESIZE, EncodeTimeout_ns=TIMEOUT),
                abi.ImageOptions(FileType=".webp", Width=16, Height=16, ResizeMethod=FIT, EncodeOptions={abi.WebpQuality: 85},
                                 EncodeTimeout_ns=TIMEOUT)):
        args = (H, W, ch, nchw, rgb, dtype, LSCALE, LBIAS)
        # every slice an encode_frames item, slice s of size L_SIZES[s // 3]; item i of the clips is slice i (T = 1) or
        # slice 3i (T = 3)
        ws, hs = [w[s // T] for s in range(n * T)], [h[s // T] for s in range(n * T)]
        frames_out, frames_st = xb.encode_frames(t.data_ptr(), nbytes, ws, hs, opt, *args)
        frames_stats = xb.stats()
        one, one_st = xb.encode_clips(t.data_ptr(), nbytes, 1, [1] * n, ws[:n], hs[:n], [-1] * n, opt, H, W, 0, *args[2:])
        s = xb.stats()
        assert (one, one_st) == (frames_out[:n], frames_st[:n])
        assert s["grid_items"] == n and frames_stats["grid_items"] == n * T
        three, three_st = xb.encode_clips(t.data_ptr(), nbytes, T, [1] * n, w, h, [-5] * (n * T), opt, H, W, 7, *args[2:])
        assert (three, three_st) == (frames_out[::T], frames_st[::T])
        assert xb.stats()["grid_items"] == n
        assert all(x == 0 for x in frames_st)


# ---------------------------------------------------------------- round trip with decode_clips

def last_duration(lib, data):
    if data[:4] == b"GIF8":
        _, delays, _, rc = lib.gif_frames(data)
        assert rc == 0
        return delays
    _, _, metas, rc = lib.webp_frames(data)
    assert rc == 0
    return [m["delay"] for m in metas]


def test_round_trip_with_decode_clips(cuda_lib, xb):
    """GIFs and animated WebPs (sprite_animation's blended, copied and disposed sub-rectangles included) through
    decode_clips (T >= F, u8), encode_clips to lossless .webp under NoResize with the start_ms differences as durations,
    and decode_clips again: the same tensor, frame indices and start times"""
    files = [scrolling_gif(31, 64, 48, 12), gif_disposals(32, 50, 40, 7), sprite_animation(33),
             pil_webp_animation(34, 48, 40, 5, lossless=False), pil_webp_animation(35, 30, 20, 3, lossless=True)]
    T, H, W, ch = 12, 64, 96, 4
    opt = abi.ImageOptions(FileType=".png", ResizeMethod=NO_RESIZE, EncodeTimeout_ns=TIMEOUT)
    n = len(files)

    def decode(bufs):
        t = torch.full((len(bufs) * T, H, W, ch), 0x33, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        w, h, nf, index, start, st = xb.decode_clips(bufs, opt, T, t.data_ptr(), t.numel(), H, W, ch, False, False, "u8")
        assert st == [0] * len(bufs)
        return t, w, h, nf, index, start

    t, w, h, nf, index, start = decode(files)
    assert all(f <= T for f in nf)
    ms = []
    for i, data in enumerate(files):
        s = start[i * T:i * T + nf[i]]
        d = [b - a for a, b in zip(s, s[1:])] + [last_duration(cuda_lib, data)[nf[i] - 1]]
        assert d[:-1] == last_duration(cuda_lib, data)[:nf[i] - 1]
        ms += d + [0] * (T - nf[i])
    webp = abi.ImageOptions(FileType=".webp", ResizeMethod=NO_RESIZE, EncodeOptions={abi.WebpQuality: 101},
                            EncodeTimeout_ns=TIMEOUT)
    outs, st = encode(xb, t, T, nf, w, h, ms, webp, ch, out_cap=1 << 22)
    assert st == [0] * n and xb.stats()["grid_items"] == n
    t2, w2, h2, nf2, index2, start2 = decode(outs)
    assert (w2, h2, nf2, index2, start2) == (w, h, nf, index, start)
    assert torch.equal(t2, t)


# ---------------------------------------------------------------- scale, memory and schedules

def test_more_than_65535_slots(cuda_lib):
    """4200 clips of T = 16: 67200 slots in one call; items of four distinct clips, each equal to its reference"""
    T, n = 16, 4200
    distinct = [(clip_frames(200 + k, 3, 2, 3, [16, 2, 9, 1][k]), durations_for(k, [16, 2, 9, 1][k])) for k in range(4)]
    items = [distinct[i % 4] for i in range(n)]
    t, keep, w, h, nf, ms = clip_tensor(items, T, 2, 4, 3)
    opt = abi.ImageOptions(FileType=".webp", ResizeMethod=NO_RESIZE, EncodeOptions={abi.WebpQuality: 101}, EncodeTimeout_ns=TIMEOUT)
    x = abi.XBatch(cuda_lib, 0, arena_bytes=2 << 30)
    try:
        outs, st = encode(x, t, T, nf, w, h, ms, opt, 3, loops=2, out_cap=1 << 14)
        assert x.stats()["grid_items"] == n
    finally:
        x.close()
    for k, (frames, durs) in enumerate(distinct):
        want = clip_reference(cuda_lib, frames, durs, 2, opt, 1 << 14)
        for i in range(k, n, 4):
            assert (st[i], outs[i]) == want, f"item {i}"


def test_long_clips_split_across_tasks(cuda_lib):
    """three clips of 256 frames of 1280 x 720 from a 2 GiB arena (one clip per lane task): every item on the grid, and
    the bytes of a roomy context and of lp_transform(A_0)"""
    T, n, H, W = 256, 3, 720, 1280
    g = torch.Generator(device="cuda").manual_seed(5)
    base = torch.randint(0, 256, (n, 1, H // 8, W // 8, 3), dtype=torch.uint8, device="cuda", generator=g)
    shift = torch.arange(T, device="cuda").view(1, T, 1, 1, 1)
    big = base.repeat_interleave(8, 2).repeat_interleave(8, 3)  # (n, 1, H, W, 3)
    t = torch.empty((n, T, H, W, 3), dtype=torch.uint8, device="cuda")
    for i in range(n):  # (uint8 sums wrap: frame k is the pattern plus 3k mod 256)
        t[i] = big[i] + (shift[0] * 3 % 256).to(torch.uint8)
    t = t.view(n * T, H, W, 3)
    torch.cuda.synchronize()
    nf, w, h = [T, T - 1, 200], [W, 1279, 641], [H, 719, 360]
    ms = [40] * (n * T)
    opt = abi.ImageOptions(FileType=".webp", Width=160, Height=160, ResizeMethod=FIT, EncodeOptions={abi.WebpQuality: 85},
                           EncodeTimeout_ns=TIMEOUT)
    small = abi.XBatch(cuda_lib, 0, arena_bytes=2 << 30)
    try:
        outs, st = encode(small, t, T, nf, w, h, ms, opt, 3, out_cap=1 << 23)
        s = small.stats()
        assert st == [0] * n and s["grid_items"] == n, (st, s)
    finally:
        small.close()
    roomy = abi.XBatch(cuda_lib, 0, arena_bytes=16 << 30)
    try:
        again, st2 = encode(roomy, t, T, nf, w, h, ms, opt, 3, out_cap=1 << 23)
        assert st2 == st and again == outs and roomy.stats()["grid_items"] == n
    finally:
        roomy.close()
    frames = [f.cpu().numpy() for f in t[:T]]
    data = clip_webp(frames, ms[:T], 0)
    assert cuda_lib.transform(data, opt, dst_cap=1 << 23) == outs[0]


@pytest.mark.parametrize("threads", [1, 8])
def test_schedule_independence(cuda_lib, xb, threads):
    """the same bytes alone and in a shared call, with host_threads 1 or many"""
    T = 8
    items = clip_batch(T, 4, seed=40) + clip_batch(T, 4, seed=41, sizes=[(40, 32), (9, 5), (40, 32), (2, 3)])
    t, keep, w, h, nf, ms = clip_tensor(items, T, BOX_H, BOX_W, 4)
    opt = options("webp_q85", "resize")
    x = abi.XBatch(cuda_lib, 0, arena_bytes=2 << 30, host_threads=threads)
    try:
        whole, st = encode(x, t, T, nf, w, h, ms, opt, 4, loops=9)
        assert st == [0] * len(items) and x.stats()["grid_items"] == len(items)
    finally:
        x.close()
    for i in range(len(items)):
        alone, sa = encode(xb, t[i * T:(i + 1) * T], T, nf[i:i + 1], w[i:i + 1], h[i:i + 1], ms[i * T:(i + 1) * T], opt, 4, loops=9)
        assert sa == [0] and alone[0] == whole[i], f"item {i} differs alone"


def test_transfers(xb):
    """no pixel crosses PCIe on the way in (the item table only); the files come home (every frame's payload: the
    container around the frames, at most 48 bytes per frame and 64 per file, is written on the host)"""
    T, n = 12, 16
    t = torch.randint(0, 256, (n * T, 64, 64, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    opt = options("webp_q85", "fit")
    nf = [T - k % 3 for k in range(n)]
    outs, st = encode(xb, t, T, nf, [64 - k for k in range(n)], [64] * n, [30] * (n * T), opt, 4)
    s = xb.stats()
    assert st == [0] * n and s["grid_items"] == n
    assert s["h2d_bytes"] <= 24 * n * T + 4096
    files = sum(len(o) for o in outs)
    assert files - 48 * sum(nf) - 64 * n <= s["d2h_bytes"] <= files


# ---------------------------------------------------------------- arguments

def test_bad_item_arguments(cuda_lib, xb):
    """nframes outside 1..T, a size outside 1..box, a used duration outside 0..0xFFFFFF: that item alone fails"""
    T = 4
    items = [(clip_frames(300 + k, 20, 16, 3, 3), [50, 60, 70]) for k in range(10)]
    t, keep, w, h, nf, ms = clip_tensor(items, T, BOX_H, BOX_W, 3)
    nf[0], nf[1], w[2], h[3] = 0, T + 1, 0, BOX_H + 1
    ms[4 * T + 1], ms[5 * T + 2] = -1, 0x1000000
    ms[6 * T + 3] = -7  # an unused slot: not read
    nf[7], ms[7 * T] = 1, 0x7FFFFFFF  # a one-frame item: its duration is not read
    opt = options("webp_q85", "fit")
    outs, st = encode(xb, t, T, nf, w, h, ms, opt, 3)
    for i in range(10):
        if i < 6:
            assert (st[i], outs[i]) == (BAD, b""), f"item {i}"
        elif i == 7:
            assert (st[i], outs[i]) == png_reference(cuda_lib, items[i][0][0], opt, 1 << 22), f"item {i}"
        else:
            assert (st[i], outs[i]) == clip_reference(cuda_lib, *items[i], 0, opt, 1 << 22), f"item {i}"


def test_bad_arguments_write_nothing(xb):
    T, n, H, W = 3, 2, BOX_H, BOX_W
    items = [(clip_frames(400 + k, 20, 16, 3, 2), [10, 20]) for k in range(n)]
    t, keep, w, h, nf, ms = clip_tensor(items, T, H, W, 3)
    before = t.cpu().clone()
    nbytes = t.numel()
    host = np.zeros(nbytes, np.uint8)
    l = xb.lib.l
    opt = options("webp_q85", "fit")._c()
    out = np.full((n, 4096), 0xA5, np.uint8)
    out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
    out_lens = (C.c_size_t * n)(*([12345] * n))
    status = (C.c_int * n)(*([77] * n))
    nfs, ws, hs, mss = (C.c_int * n)(*nf), (C.c_int * n)(*w), (C.c_int * n)(*h), (C.c_int * (n * T))(*ms)

    def tensor(**kw):
        a = dict(data=t.data_ptr(), bytes=nbytes, height=H, width=W, channels=3, nchw=0, rgb=0, dtype=0)
        a.update(kw)
        return abi._FrameTensor(a["data"], a["bytes"], a["height"], a["width"], a["channels"], a["nchw"], a["rgb"],
                                a["dtype"], (C.c_float * 4)(1, 1, 1, 1), (C.c_float * 4)())

    good = tensor()
    base = dict(src=C.byref(good), n=n, T=T, nf=nfs, w=ws, h=hs, ms=mss, loops=0, opt=C.byref(opt), out=out_ptrs, ol=out_lens,
                st=status)
    cases = {
        "undersized for n * T": dict(src=C.byref(tensor(bytes=nbytes - 1))),
        "n slices only": dict(src=C.byref(tensor(bytes=nbytes // T))),
        "host memory": dict(src=C.byref(tensor(data=host.ctypes.data))),
        "channels 5": dict(src=C.byref(tensor(channels=5))),
        "unknown dtype": dict(src=C.byref(tensor(dtype=7))),
        "null tensor": dict(src=None),
        "T 0": dict(T=0), "T 4097": dict(T=4097), "T past the tensor": dict(T=T + 1),
        "loop -1": dict(loops=-1), "loop 65536": dict(loops=65536),
        "negative n": dict(n=-1),
        "null opt": dict(opt=None), "null nframes": dict(nf=None), "null width": dict(w=None), "null height": dict(h=None),
        "null durations": dict(ms=None), "null out": dict(out=None), "null out_len": dict(ol=None), "null status": dict(st=None),
    }
    for what, kw in cases.items():
        a = {**base, **kw}
        rc = l.lp_xbatch_encode_clips(xb.h, a["src"], a["n"], a["T"], a["nf"], a["w"], a["h"], a["ms"], a["loops"], a["opt"],
                                      a["out"], 4096, a["ol"], a["st"])
        assert rc == BAD, what
    assert not host.any()
    assert bool((out == 0xA5).all()), "a refused call wrote into out"
    assert list(out_lens) == [12345] * n and list(status) == [77] * n, "a refused call wrote out_len or status"
    assert torch.equal(t.cpu(), before), "a refused call wrote into the tensor"
    assert xb.encode_clips(t.data_ptr(), nbytes, T, [], [], [], [], options("webp_q85", "fit"), H, W) == ([], [])

