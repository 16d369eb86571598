"""GPU: lp_xbatch_encode_frames -- files written from a caller's device tensor.

Item i's reference is the same library's lp_transform of cv2.imencode(".png", frame_i) with the call's options, where
frame_i is the u8 BGR / BGRA frame a numpy restatement of the conversion makes of slice i: status and bytes must be
equal.  The restatement works in float64 (x * scale + bias, round half to even, clamp, NaN as 0); a float element whose
float64 value lies within one fp32 ulp of a half-integer, without being an fp32 value itself, may round either way on
the device (its fmaf rounds to fp32 first) and is not compared.

Which items take the grid is asserted exactly: what lp_xbatch_transform counts for the same PNGs and options, except
under NoResize, where the tensor items take the grid as the PNGs would under Resize."""
import ctypes as C

import cv2
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch import rgb_png
from tests.test_gpu_xbatch_jpeg_webp import cv2_jpeg
from tests.test_gpu_xbatch_renditions import cv2_webp

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
T = 10**12
FIT, RESIZE, NO_RESIZE = abi.ImageOpsFit, abi.ImageOpsResize, abi.ImageOpsNoResize
DTYPES = {"u8": torch.uint8, "f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
BAD = -10  # LP_ERR_BAD_ARGUMENT
BGR = [2, 1, 0, 3]  # RGB(A) <-> BGR(A)


# ---------------------------------------------------------------- frames, tensors and the restatement

def design_frame(seed, w, h, ch, content, alpha):
    """u8 BGR / BGRA frame: `content` flat, gradient or synth (photo-like); `alpha` opaque, partial or clear"""
    rng = np.random.default_rng(seed)
    if content == "flat":
        f = np.broadcast_to(rng.integers(0, 256, ch, dtype=np.uint8), (h, w, ch)).copy()
    elif content == "gradient":
        y, x = np.mgrid[0:h, 0:w]
        f = np.stack([(x * (c + 1) * 255 // max(w, 1) + y * (3 - c) * 255 // max(h, 1) + 40 * c) % 256 for c in range(ch)], -1)
        f = f.astype(np.uint8)
    else:
        f = synth_image(seed, w, h, ch)
    if ch == 4:
        f[..., 3] = {"opaque": 255, "clear": 0}.get(alpha, 0)
        if alpha == "partial":
            f[..., 3] = (np.arange(w)[None, :] * 251 // max(w - 1, 1) + np.arange(h)[:, None]) % 256
    return np.ascontiguousarray(f)


# (w, h, content, alpha) in a 96 x 128 box: 1x1, odd sizes, box-sized, and narrow ones Fit and Resize upscale
BOX_H, BOX_W = 96, 128
FRAMES = [(1, 1, "flat", "opaque"), (37, 23, "gradient", "partial"), (20, 60, "synth", "opaque"),
          (BOX_W, BOX_H, "synth", "partial"), (101, 67, "flat", "clear"), (64, 64, "gradient", "opaque"),
          (13, 90, "gradient", "clear")]


def frames_for(ch):
    return [design_frame(100 + k, w, h, ch, c, a) for k, (w, h, c, a) in enumerate(FRAMES)]


def device_tensor(a, dtype, offset=0):
    """(tensor, keep): the float64 / u8 numpy array `a` stored as dtype on the device, its base `offset` elements past
    an allocation's start (an element-aligned base that is not 16-byte aligned when offset is odd)"""
    src = torch.from_numpy(np.ascontiguousarray(a)).to(DTYPES[dtype])
    keep = torch.zeros(src.numel() + offset, dtype=DTYPES[dtype], device="cuda")
    t = keep[offset:].view(src.shape)
    t.copy_(src.cuda())
    torch.cuda.synchronize()  # (the library's streams do not wait for torch's)
    return t, keep


def layout(frames, H, W, ch, rgb, nchw, fill=0.0):
    """float64 N x H x W x C (or N x C x H x W) array, frames[i] (BGR order) at slice i's top-left in tensor order"""
    a = np.full((len(frames), H, W, ch), fill, np.float64)
    for i, f in enumerate(frames):
        v = f.astype(np.float64)
        a[i, : f.shape[0], : f.shape[1]] = v[..., BGR[:ch]] if rgb else v
    return a.transpose(0, 3, 1, 2) if nchw else a


def restate(t, dtype, ch, nchw, rgb, scale, bias):
    """numpy restatement of the conversion: (u8 N x H x W x C in BGR(A) order, mask of elements that may round either
    way)"""
    a = t.detach().cpu().to(torch.float64).numpy()
    if nchw:
        a = a.transpose(0, 2, 3, 1)
    if dtype == "u8":
        v, amb = a, np.zeros(a.shape, bool)
    else:
        s = np.float32(scale[:ch]).astype(np.float64)
        b = np.float32(bias[:ch]).astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            v = a * s + b
            v32 = v.astype(np.float32)
            exact = v32.astype(np.float64) == v
            ulp = np.spacing(np.abs(v32)).astype(np.float64)
            amb = np.isfinite(v) & ~exact & (np.abs(v - np.floor(v) - 0.5) <= ulp)
            v = np.where(np.isnan(v), 0.0, np.clip(np.rint(v), 0, 255))
    if rgb:
        v, amb = v[..., BGR[:ch]], amb[..., BGR[:ch]]
    return v.astype(np.uint8), amb


def png_of(frame):
    ok, b = cv2.imencode(".png", frame)
    assert ok
    b = bytes(b)
    off, chunks = 8, []
    while off + 8 <= len(b):
        n = int.from_bytes(b[off:off + 4], "big")
        chunks.append(b[off + 4:off + 8])
        off += n + 12
    assert chunks == [b"IHDR"] + [b"IDAT"] * (len(chunks) - 2) + [b"IEND"], chunks  # no ancillary chunks
    assert b[25] == (6 if frame.shape[2] == 4 else 2) and b[24] == 8  # colour type 2 / 6, 8 bits
    return b


def reference(lib, frame, opt, out_cap, max_size=8192):
    """(status, bytes) of lp_transform(PNG of frame, opt)"""
    try:
        return 0, lib.transform(png_of(frame), opt, dst_cap=out_cap, max_size=max_size)
    except abi.LilliputError as e:
        return e.code, b""


def encode(xb, t, widths, heights, opt, ch, nchw=False, rgb=False, dtype="u8", scale=None, bias=None, out_cap=1 << 22):
    H, W = (t.shape[2], t.shape[3]) if nchw else (t.shape[1], t.shape[2])
    return xb.encode_frames(t.data_ptr(), t.numel() * t.element_size(), widths, heights, opt, H, W, ch, nchw, rgb, dtype,
                            scale, bias, out_cap)


def sizes(frames):
    return [f.shape[1] for f in frames], [f.shape[0] for f in frames]


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def check_contract(lib, xb, frames, opt, outs, st, out_cap=1 << 22, names=None):
    for i, f in enumerate(frames):
        code, want = reference(lib, f, opt, out_cap)
        what = f"item {i} {f.shape}{' ' + names[i] if names else ''}"
        assert st[i] == code, f"{what}: status {st[i]}, lp_transform {code}"
        assert outs[i] == want, f"{what}: {len(outs[i])} bytes differ from lp_transform's {len(want)}"


def expected_grid(xb, frames, opt, out_cap=1 << 22):
    """grid items of lp_xbatch_transform over the frames' PNGs (under NoResize: as under Resize, which the PNGs' gates
    let through where NoResize does not).  A negative MaxEncodeDuration, and to .webp a zero encode budget or
    MaxEncodeFrames 1, send every tensor item per image: lp_transform fails those, where lp_xbatch_transform keeps
    ICC-less PNGs on the grid."""
    if opt.MaxEncodeDuration_ns < 0 or (opt.FileType == ".webp" and (opt.EncodeTimeout_ns <= 0 or opt.MaxEncodeFrames == 1)):
        return 0
    o = abi.ImageOptions(**opt.__dict__)
    if o.ResizeMethod == NO_RESIZE:
        o.ResizeMethod, o.Width, o.Height = RESIZE, 16, 16
    xb.transform([png_of(f) for f in frames], o, out_cap=out_cap)
    return xb.stats()["grid_items"]


# ---------------------------------------------------------------- the contract

SINKS = {
    "jpeg_q1": (".jpeg", {abi.JpegQuality: 1}),
    "jpeg_q50": (".jpeg", {abi.JpegQuality: 50}),
    "jpeg_q85": (".jpeg", {abi.JpegQuality: 85}),
    "jpeg_q100": (".jpeg", {abi.JpegQuality: 100}),
    "jpeg_progressive": (".jpeg", {abi.JpegQuality: 85, abi.JpegProgressive: 1}),
    "png": (".png", {}),
    "png_0": (".png", {abi.PngCompression: 0}),
    "png_1": (".png", {abi.PngCompression: 1}),
    "png_6": (".png", {abi.PngCompression: 6}),
    "png_9": (".png", {abi.PngCompression: 9}),
    "webp_q1": (".webp", {abi.WebpQuality: 1}),
    "webp_q85": (".webp", {abi.WebpQuality: 85}),
    "webp_q100": (".webp", {abi.WebpQuality: 100}),
    "webp_q101": (".webp", {abi.WebpQuality: 101}),
    "gif": (".gif", {}),
}
GEOMETRIES = {"fit": (48, 40, FIT), "resize": (50, 30, RESIZE), "no_resize": (0, 0, NO_RESIZE)}


def options(sink, geometry, **kw):
    ext, eo = SINKS[sink]
    w, h, m = GEOMETRIES[geometry]
    return abi.ImageOptions(FileType=ext, Width=w, Height=h, ResizeMethod=m, EncodeOptions=dict(eo),
                            **{"EncodeTimeout_ns": T, **kw})


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
@pytest.mark.parametrize("sink", list(SINKS))
def test_contract(cuda_lib, xb, sink, geometry, ch):
    """Every item's status and bytes are lp_transform's of its PNG; the grid / per-image split is exact.  Three channels
    come from a u8 NHWC BGR tensor, four from an f16 NCHW RGB one stored as v / 255 and read back with scale 255."""
    frames = frames_for(ch)
    opt = options(sink, geometry)
    w, h = sizes(frames)
    if ch == 3:
        t, keep = device_tensor(layout(frames, BOX_H, BOX_W, 3, False, False), "u8")
        outs, st = encode(xb, t, w, h, opt, 3)
    else:
        t, keep = device_tensor(layout(frames, BOX_H, BOX_W, 4, True, True) / 255.0, "f16")
        got, amb = restate(t, "f16", 4, True, True, [255.0] * 4, [0.0] * 4)
        assert not amb.any()
        for i, f in enumerate(frames):
            assert np.array_equal(got[i, : f.shape[0], : f.shape[1]], f)
        outs, st = encode(xb, t, w, h, opt, 4, nchw=True, rgb=True, dtype="f16", scale=[255.0] * 4)
    s = xb.stats()
    check_contract(cuda_lib, xb, frames, opt, outs, st)
    want = expected_grid(xb, frames, opt)
    assert (s["grid_items"], s["fallback_items"]) == (want, len(frames) - want)
    if geometry == "no_resize" and sink != "gif":
        assert want == len(frames)


@pytest.mark.parametrize("geometry", ["fit", "no_resize"])
@pytest.mark.parametrize("option", ["timeout_0", "max_frames_1", "max_duration_1", "max_duration_neg"])
@pytest.mark.parametrize("sink", ["jpeg_q85", "png", "webp_q85", "webp_q101", "gif"])
def test_options(cuda_lib, xb, sink, option, geometry):
    """EncodeTimeout 0, MaxEncodeFrames 1 and MaxEncodeDuration +-1: the status and bytes of lp_transform, the split of
    lp_xbatch_transform"""
    kw = {"timeout_0": {"EncodeTimeout_ns": 0}, "max_frames_1": {"MaxEncodeFrames": 1},
          "max_duration_1": {"MaxEncodeDuration_ns": 1}, "max_duration_neg": {"MaxEncodeDuration_ns": -1}}[option]
    frames = frames_for(4)
    opt = options(sink, geometry, **kw)
    t, keep = device_tensor(layout(frames, BOX_H, BOX_W, 4, False, False), "u8")
    w, h = sizes(frames)
    outs, st = encode(xb, t, w, h, opt, 4)
    s = xb.stats()
    check_contract(cuda_lib, xb, frames, opt, outs, st)
    want = expected_grid(xb, frames, opt)
    assert (s["grid_items"], s["fallback_items"]) == (want, len(frames) - want)


@pytest.mark.parametrize("sink", ["jpeg_q85", "png_0", "webp_q85", "webp_q101"])
def test_small_out_cap(cuda_lib, xb, sink):
    """A buffer too small for some files: ErrBufTooSmall (or the sink's own refusal) exactly where lp_transform gives it"""
    frames = frames_for(3)
    out_cap = 400
    opt = options(sink, "fit")
    t, keep = device_tensor(layout(frames, BOX_H, BOX_W, 3, False, False), "u8")
    w, h = sizes(frames)
    outs, st = encode(xb, t, w, h, opt, 3, out_cap=out_cap)
    assert any(s != 0 for s in st), st
    check_contract(cuda_lib, xb, frames, opt, outs, st, out_cap=out_cap)


@pytest.mark.parametrize("geometry", ["fit", "no_resize"])
def test_frames_over_max_size(cuda_lib, geometry):
    """A context with max_size 64: frames over it in either side answer as lp_transform(..., max_size 64) does"""
    frames = [design_frame(7, 100, 40, 3, "synth", ""), design_frame(8, 40, 30, 3, "gradient", ""),
              design_frame(9, 30, 160, 3, "flat", ""), design_frame(10, 64, 64, 3, "synth", "")]
    opt = options("jpeg_q85", geometry)
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30, max_size=64)
    try:
        t, keep = device_tensor(layout(frames, 160, 100, 3, False, False), "u8")
        w, h = sizes(frames)
        outs, st = encode(small, t, w, h, opt, 3)
    finally:
        small.close()
    for i, f in enumerate(frames):
        assert (st[i], outs[i]) == reference(cuda_lib, f, opt, 1 << 22, max_size=64), f"item {i} {f.shape}"


# ---------------------------------------------------------------- layouts and the conversion

LSCALE = [1.0, 0.5, 2.0, 4.0]
LBIAS = [0.0, 0.25, -1.0, 0.5]
L_H, L_W = 19, 37  # (a row of 37 x C elements is no whole number of 16-byte pieces)
L_SIZES = [(37, 19), (23, 11), (1, 1)]


def designed_values(seed, dtype, ch, nchw):
    """float64 tensor (before the dtype's rounding) of len(L_SIZES) slices: random values around 0..255 after the
    conversion, exact k + 0.5 ties, negatives, values over 255, and for float dtypes NaN and +-inf"""
    rng = np.random.default_rng(seed)
    n = len(L_SIZES)
    if dtype == "u8":
        a = rng.integers(0, 256, (n, L_H, L_W, ch)).astype(np.float64)
    else:
        v = rng.uniform(-40, 300, (n, L_H, L_W, ch))
        ties = rng.integers(-3, 258, (n, L_H, L_W, ch)) + 0.5
        pick = rng.random((n, L_H, L_W, ch))
        v = np.where(pick < 0.3, ties, v)
        a = (v - np.array(LBIAS[:ch])) / np.array(LSCALE[:ch])
        special = rng.random((n, L_H, L_W, ch))
        a = np.where(special < 0.02, np.nan, a)
        a = np.where((special >= 0.02) & (special < 0.04), np.inf, a)
        a = np.where((special >= 0.04) & (special < 0.06), -np.inf, a)
        a = np.where((special >= 0.06) & (special < 0.07), 1e30, a)
    return a.transpose(0, 3, 1, 2) if nchw else a


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("rgb", [False, True])
@pytest.mark.parametrize("nchw", [False, True])
def test_layouts(xb, dtype, ch, rgb, nchw):
    """Every dtype, layout, channel order and count, seen through NoResize .png files decoded by cv2, against the
    numpy restatement.  RGB tensors start one element past a 16-byte boundary."""
    t, keep = device_tensor(designed_values(len(dtype) + 2 * ch + 5 * rgb + 11 * nchw, dtype, ch, nchw), dtype,
                            offset=1 if rgb else 0)
    assert (t.data_ptr() % 16 != 0) == rgb
    want, amb = restate(t, dtype, ch, nchw, rgb, LSCALE, LBIAS)
    opt = abi.ImageOptions(FileType=".png", ResizeMethod=NO_RESIZE, EncodeTimeout_ns=T)
    w, h = [s[0] for s in L_SIZES], [s[1] for s in L_SIZES]
    outs, st = encode(xb, t, w, h, opt, ch, nchw, rgb, dtype, LSCALE, LBIAS)
    assert st == [0] * len(L_SIZES) and xb.stats()["grid_items"] == len(L_SIZES)
    for i, (fw, fh) in enumerate(L_SIZES):
        got = cv2.imdecode(np.frombuffer(outs[i], np.uint8), cv2.IMREAD_UNCHANGED)
        got = got.reshape(fh, fw, -1)
        assert got.shape == (fh, fw, ch)
        sel = ~amb[i, :fh, :fw]
        bad = (got != want[i, :fh, :fw]) & sel
        assert not bad.any(), f"item {i}: {int(bad.sum())} elements differ, e.g. {got[bad][:4]} vs {want[i, :fh, :fw][bad][:4]}"
        if dtype == "u8":
            assert sel.all()


# ---------------------------------------------------------------- with decode_frames, schedules, transfers

def round_trip_sources():
    return [cv2_jpeg(synth_image(1, 320, 200, 3), 90), cv2_jpeg(synth_image(2, 97, 131, 3), 75, progressive=True),
            rgb_png(synth_image(3, 180, 120, 3)), rgb_png(synth_image(4, 61, 45, 3)),
            cv2_webp(synth_image(5, 240, 160, 3), 80), cv2_webp(synth_image(6, 33, 77, 3), 60)]


@pytest.mark.parametrize("dtype", ["u8", "f16"])
def test_round_trip_with_decode_frames(xb, dtype):
    """decode_frames, then encode_frames of the same tensor under NoResize to .png, writes lp_xbatch_transform's .png
    files: u8 NHWC BGR as is, and f16 NCHW RGB stored with scale 1/255 and read back with scale 255"""
    files = round_trip_sources()
    opt = abi.ImageOptions(FileType=".png", Width=96, Height=72, ResizeMethod=FIT, EncodeOptions={abi.PngCompression: 1},
                           EncodeTimeout_ns=T)
    want, want_st = xb.transform(files, opt, out_cap=1 << 22)
    assert want_st == [0] * len(files)
    nchw, rgb = dtype == "f16", dtype == "f16"
    shape = (len(files), 3, 72, 96) if nchw else (len(files), 72, 96, 3)
    t = torch.zeros(shape, dtype=DTYPES[dtype], device="cuda")
    torch.cuda.synchronize()
    w, h, st = xb.decode_frames(files, opt, t.data_ptr(), t.numel() * t.element_size(), 72, 96, 3, nchw, rgb, dtype,
                                [1 / 255] * 4, [0.0] * 4)
    assert st == [0] * len(files)
    back = abi.ImageOptions(**{**opt.__dict__, "ResizeMethod": NO_RESIZE, "Width": 0, "Height": 0})
    outs, st = encode(xb, t, w, h, back, 3, nchw, rgb, dtype, [255.0] * 4, [0.0] * 4)
    assert st == [0] * len(files)
    assert outs == want


def test_u8_survives_fp16_and_bf16_at_scale_one_255th():
    """Every u8 value stored as fp16 or bf16 with scale 1/255 comes back with scale 255 (what the round trip relies on)"""
    v = torch.arange(256, dtype=torch.float32)
    for dt in (torch.float16, torch.bfloat16):
        x = (v * np.float32(1 / 255)).to(dt).to(torch.float32)
        back = torch.round(x * 255)
        assert torch.equal(back, v), dt
        assert float((x * 255 - v).abs().max()) < 0.5


def test_schedule_independence(cuda_lib, xb):
    """The same files alone, in the full batch, and from a 1 GiB arena whose lanes hold a fraction of the items"""
    n, H, W = 128, 1536, 2048
    g = torch.Generator(device="cuda").manual_seed(3)
    t = torch.randint(0, 256, (n, H, W, 4), dtype=torch.uint8, device="cuda", generator=g)
    torch.cuda.synchronize()
    rng = np.random.default_rng(4)
    w = [int(x) for x in rng.integers(700, W + 1, n)]
    h = [int(x) for x in rng.integers(500, H + 1, n)]
    opt = abi.ImageOptions(FileType=".jpeg", Width=256, Height=192, ResizeMethod=FIT, EncodeOptions={abi.JpegQuality: 85},
                           EncodeTimeout_ns=T)
    whole, st = encode(xb, t, w, h, opt, 4, out_cap=1 << 20)
    assert st == [0] * n
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        chunked, st2 = encode(small, t, w, h, opt, 4, out_cap=1 << 20)
    finally:
        small.close()
    assert st2 == st
    for i in range(n):
        assert chunked[i] == whole[i], f"item {i} differs in the 1 GiB arena"
    for i in (0, 1, 57, n - 1):
        alone, sa = encode(xb, t[i:i + 1], [w[i]], [h[i]], opt, 4, out_cap=1 << 20)
        assert sa == [0] and alone[0] == whole[i], f"item {i} differs alone"


def test_transfers(xb):
    """No pixel crosses PCIe on the way in (the item table only); the files come home"""
    n = 64
    t = torch.randint(0, 256, (n, 256, 256, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    opt = abi.ImageOptions(FileType=".jpeg", Width=128, Height=128, ResizeMethod=FIT, EncodeOptions={abi.JpegQuality: 85},
                           EncodeTimeout_ns=T)
    outs, st = encode(xb, t, [256 - k for k in range(n)], [256] * n, opt, 4)
    s = xb.stats()
    assert st == [0] * n and s["grid_items"] == n
    assert s["h2d_bytes"] <= 64 * n + 4096
    assert s["d2h_bytes"] >= sum(len(o) for o in outs)


# ---------------------------------------------------------------- arguments and state

def test_bad_item_sizes(cuda_lib, xb):
    """A width or height outside 1..box fails that item alone with LP_ERR_BAD_ARGUMENT"""
    frames = frames_for(3)
    t, keep = device_tensor(layout(frames, BOX_H, BOX_W, 3, False, False), "u8")
    w, h = sizes(frames)
    bad = {1: (0, h[1]), 2: (w[2], BOX_H + 1), 4: (-5, h[4]), 5: (BOX_W + 1, h[5])}
    for i, (bw, bh) in bad.items():
        w[i], h[i] = bw, bh
    opt = options("jpeg_q85", "fit")
    outs, st = encode(xb, t, w, h, opt, 3)
    for i, f in enumerate(frames):
        if i in bad:
            assert (st[i], outs[i]) == (BAD, b""), f"item {i}"
        else:
            assert (st[i], outs[i]) == reference(cuda_lib, f, opt, 1 << 22), f"item {i}"


def test_bad_arguments_write_nothing(xb):
    frames = frames_for(3)[:4]
    n, H, W = len(frames), BOX_H, BOX_W
    t, keep = device_tensor(layout(frames, H, W, 3, False, False), "u8")
    nbytes = t.numel()
    host = np.zeros(nbytes, np.uint8)
    w, h = sizes(frames)
    l = xb.lib.l
    opt = options("jpeg_q85", "fit")._c()
    out = np.full((n, 4096), 0xA5, np.uint8)
    out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
    out_lens = (C.c_size_t * n)(*([12345] * n))
    status = (C.c_int * n)(*([77] * n))
    ws, hs = (C.c_int * n)(*w), (C.c_int * n)(*h)

    def tensor(**kw):
        a = dict(data=t.data_ptr(), bytes=nbytes, height=H, width=W, channels=3, nchw=0, rgb=0, dtype=0)
        a.update(kw)
        return abi._FrameTensor(a["data"], a["bytes"], a["height"], a["width"], a["channels"], a["nchw"], a["rgb"],
                                a["dtype"], (C.c_float * 4)(1, 1, 1, 1), (C.c_float * 4)())

    tensor_cases = {
        "undersized": dict(bytes=nbytes - 1), "host memory": dict(data=host.ctypes.data), "null data": dict(data=0),
        "channels 2": dict(channels=2), "channels 5": dict(channels=5), "unknown dtype": dict(dtype=7),
        "empty box": dict(height=0), "misaligned f32": dict(data=t.data_ptr() + 2, dtype=3, bytes=nbytes - 2),
    }
    for what, kw in tensor_cases.items():
        rc = l.lp_xbatch_encode_frames(xb.h, C.byref(tensor(**kw)), n, ws, hs, C.byref(opt), out_ptrs, 4096, out_lens, status)
        assert rc == BAD, what
    good = tensor()
    calls = {
        "null tensor": (None, n, ws, hs, C.byref(opt), out_ptrs, out_lens, status),
        "negative n": (C.byref(good), -1, ws, hs, C.byref(opt), out_ptrs, out_lens, status),
        "null opt": (C.byref(good), n, ws, hs, None, out_ptrs, out_lens, status),
        "null width": (C.byref(good), n, None, hs, C.byref(opt), out_ptrs, out_lens, status),
        "null height": (C.byref(good), n, ws, None, C.byref(opt), out_ptrs, out_lens, status),
        "null out": (C.byref(good), n, ws, hs, C.byref(opt), None, out_lens, status),
        "null out_len": (C.byref(good), n, ws, hs, C.byref(opt), out_ptrs, None, status),
        "null status": (C.byref(good), n, ws, hs, C.byref(opt), out_ptrs, out_lens, None),
    }
    for what, (tp, nn, a, b, o, op, ol, s) in calls.items():
        assert l.lp_xbatch_encode_frames(xb.h, tp, nn, a, b, o, op, 4096, ol, s) == BAD, what
    assert not host.any()
    assert bool((out == 0xA5).all()), "a refused call wrote into out"
    assert list(out_lens) == [12345] * n and list(status) == [77] * n, "a refused call wrote out_len or status"


def test_no_leaked_state(cuda_lib, xb):
    """lp_xbatch_transform and decode_frames on the same context answer the same before and after encode_frames"""
    files = round_trip_sources()
    jopt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=FIT, EncodeOptions={abi.JpegQuality: 85},
                            EncodeTimeout_ns=T)

    def others():
        outs = xb.transform(files, jopt, out_cap=1 << 22)
        s = {k: xb.stats()[k] for k in ("grid_items", "fallback_items", "d2h_bytes", "h2d_bytes")}
        d = torch.zeros((len(files), 64, 64, 4), dtype=torch.float16, device="cuda")
        torch.cuda.synchronize()
        r = xb.decode_frames(files, jopt, d.data_ptr(), d.numel() * 2, 64, 64, 4, False, True, "f16", [1 / 255] * 4, [0.0] * 4)
        return outs, s, r, d.cpu()

    before = others()
    frames = frames_for(4)
    t, keep = device_tensor(layout(frames, BOX_H, BOX_W, 4, False, False), "u8")
    w, h = sizes(frames)
    encode(xb, t, w, h, options("png_1", "no_resize"), 4)
    after = others()
    assert before[:3] == after[:3]
    assert torch.equal(before[3], after[3])
