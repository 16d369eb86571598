"""GPU: lp_xbatch_decode_frames -- the frame every item would be encoded from, written into a caller's device tensor.

The reference for item i is the same library's lp_transform(in[i], opt with ".png", PngCompression 0) decoded by cv2
(IMREAD_UNCHANGED) and laid out in numpy: U8 must be equal, float dtypes within one unit in the last place of the dtype
(the expectation is computed in float64 and rounded to the dtype).  Status and frame size are lp_transform's.

Which items take the grid is asserted exactly: an item whose source the other sinks already route the same way is
counted by a call of lp_xbatch_transform with those options (".png" for stills, ".webp" with DisableAnimatedOutput for
GIFs and animated WebPs, whose first-frame plans this call shares); the well-formed rotated and gray JPEGs and SDR-cICP
PNGs, which only this call takes on the grid, count one each; gray and eXIf-rotated PNGs, NoResize and MaxEncodeDuration
count none."""
import ctypes as C

import cv2
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch import rgb_png
from tests.test_gpu_xbatch_hdr_png import hdr_png, png_file, source, with_cicp
from tests.test_gpu_xbatch_jpeg_webp import cv2_jpeg, with_exif_orientation
from tests.test_gpu_xbatch_renditions import cv2_webp, pil_gif, pil_webp_animation

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
T = 10**12
FIT, RESIZE = abi.ImageOpsFit, abi.ImageOpsResize
DTYPES = {"u8": torch.uint8, "f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
BITS = {"u8": torch.uint8, "f16": torch.int16, "bf16": torch.int16, "f32": torch.int32}
SCALE = [1 / (255 * 0.229), 1 / (255 * 0.224), 1 / (255 * 0.225), 1 / 255]
BIAS = [-0.485 / 0.229, -0.456 / 0.224, -0.406 / 0.225, 0.25]
# well-formed sources only this call takes on the grid; sources it sends per image whatever the options
FRAMES_ONLY_GRID = {"jpeg_gray", "jpeg_gray_progressive", "png_sdr_cicp"} | {f"jpeg_rot{o}" for o in range(2, 9)}
PER_IMAGE = {"png_gray", "png_exif"}
ANIMATED = {"webp_anim_lossy", "webp_anim_lossless", "gif_anim", "gif_one_frame", "gif_truncated"}


def corpus():
    s420, s422, s444 = (cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                        cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444)
    base = cv2_jpeg(synth_image(1, 640, 360, 3), 90, sampling=s420)
    files = [
        ("jpeg_420", base),
        ("jpeg_rst", cv2_jpeg(synth_image(3, 320, 240, 3), 85, rst=4)),
        ("jpeg_progressive", cv2_jpeg(synth_image(4, 300, 200, 3), 80, progressive=True)),
        ("jpeg_422_odd", cv2_jpeg(synth_image(5, 203, 117, 3), 90, sampling=s422)),
        ("jpeg_444_odd", cv2_jpeg(synth_image(6, 161, 97, 3), 95, sampling=s444)),
        ("jpeg_1x1", cv2_jpeg(synth_image(7, 1, 1, 3), 90)),
        ("jpeg_gray", cv2_jpeg(synth_image(8, 120, 90, 1), 90)),
        ("jpeg_gray_progressive", cv2_jpeg(synth_image(9, 75, 131, 1), 85, progressive=True)),
    ]
    rot = cv2_jpeg(synth_image(10, 200, 120, 3), 90)
    files += [(f"jpeg_rot{o}", with_exif_orientation(rot, o)) for o in range(2, 9)]
    files += [
        ("png_rgb", rgb_png(synth_image(11, 300, 200, 3))),
        ("png_rgba", rgb_png(synth_image(12, 256, 256, 4))),
        ("png_16bit", png_file(source(13, 130, 70, "rgb", 16)[1], 2, 16)),
        ("png_16bit_rgba", png_file(source(14, 90, 66, "rgba", 16)[1], 6, 16)),
        ("png_pq", hdr_png(15, 101, 75, "rgb", 16, 16, 9)),
        ("png_hlg", hdr_png(16, 64, 48, "rgba", 16, 18, 12)),
        ("png_sdr_cicp", with_cicp(rgb_png(synth_image(17, 80, 60, 3)), 1, 13)),
        ("png_gray", png_file(synth_image(18, 50, 40, 1).reshape(40, 50, 1), 0, 8)),
        ("png_exif", png_file(source(19, 70, 50, "rgb", 8)[1], 2, 8, orientation=6)),
        ("webp_lossy", cv2_webp(synth_image(20, 240, 160, 3), 80)),
        ("webp_lossy_alpha", cv2_webp(synth_image(21, 120, 100, 4), 80)),
        ("webp_lossless", cv2_webp(synth_image(22, 90, 70, 4), 101)),
        ("webp_anim_lossy", pil_webp_animation(23, 96, 64, 3, lossless=False)),
        ("webp_anim_lossless", pil_webp_animation(27, 64, 48, 2, lossless=True)),
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


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def opts(w, h, method, **kw):
    return abi.ImageOptions(FileType=".jpeg", Width=w, Height=h, ResizeMethod=method, EncodeOptions={abi.JpegQuality: 50},
                            EncodeTimeout_ns=T, **kw)


def reference_frame(lib, data, opt):
    """(status, frame): lp_transform to an uncompressed PNG, decoded by cv2 (gray 2-D, BGR or BGRA)"""
    o = abi.ImageOptions(**{**opt.__dict__, "FileType": ".png", "EncodeOptions": {abi.PngCompression: 0}})
    try:
        png = lib.transform(data, o, dst_cap=1 << 26)
    except abi.LilliputError as e:
        return e.code, None
    return 0, cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)


def expected_slice(frame, H, W, ch, nchw, rgb, dtype, scale, bias):
    """float64 slice (H x W x C, or C x H x W) of one frame, zero outside it"""
    out = np.zeros((H, W, ch), np.float64)
    if frame is not None:
        f = frame[..., None] if frame.ndim == 2 else frame
        h, w, c = f.shape
        for k in range(ch):
            if k == 3:
                v = f[..., 3] if c == 4 else np.full((h, w), 255)
            else:
                v = f[..., 0] if c == 1 else f[..., 2 - k if rgb else k]
            v = v.astype(np.float64)
            out[:h, :w, k] = v if dtype == "u8" else v * np.float64(np.float32(scale[k])) + np.float64(np.float32(bias[k]))
    return out.transpose(2, 0, 1) if nchw else out


def assert_slice(got, want, dtype, what):
    """got: the device slice (torch, on the host); want: float64 numpy.  U8 exact, floats within one ulp"""
    exp = torch.from_numpy(np.ascontiguousarray(want)).to(DTYPES[dtype])
    if dtype == "u8":
        assert torch.equal(got, exp), f"{what}: {int((got != exp).sum())} elements differ"
        return
    a, b = got.view(BITS[dtype]).to(torch.int64), exp.view(BITS[dtype]).to(torch.int64)
    bad = ((a - b).abs() > 1) & (got.to(torch.float64) != exp.to(torch.float64))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements beyond one ulp, e.g. {got[bad][:4]} vs {exp[bad][:4]}"


def tensor(n, H, W, ch, dtype, nchw, fill=0x5A):
    shape = (n, ch, H, W) if nchw else (n, H, W, ch)
    t = torch.empty(shape, dtype=DTYPES[dtype], device="cuda")
    t.view(torch.uint8).fill_(fill)
    torch.cuda.synchronize()  # (the library's streams do not wait for torch's)
    return t


def decode(xb, files, opt, H, W, ch=4, nchw=False, rgb=False, dtype="u8", scale=SCALE, bias=BIAS, fill=0x5A):
    t = tensor(len(files), H, W, ch, dtype, nchw, fill)
    w, h, st = xb.decode_frames(files, opt, t.data_ptr(), t.numel() * t.element_size(), H, W, ch, nchw, rgb, dtype, scale, bias)
    return t.cpu(), w, h, st


def check_items(lib, files, opt, got, w, h, st, H, W, ch=4, nchw=False, rgb=False, dtype="u8", names=None):
    for i, f in enumerate(files):
        what = f"item {i} ({names[i] if names else ''})"
        code, frame = reference_frame(lib, f, opt)
        if code == 0 and (frame.shape[0] > H or frame.shape[1] > W):
            code, frame = abi.LP_ERR_BUF_TOO_SMALL, None
        assert st[i] == code, f"{what}: status {st[i]}, lp_transform {code}"
        size = (frame.shape[1], frame.shape[0]) if code == 0 else (0, 0)
        assert (w[i], h[i]) == size, f"{what}: size {w[i]} x {h[i]}, lp_transform {size}"
        assert_slice(got[i], expected_slice(frame if code == 0 else None, H, W, ch, nchw, rgb, dtype, SCALE, BIAS), dtype, what)


def expected_grid(xb, name, data, opt):
    if name in FRAMES_ONLY_GRID:
        return 1
    if name in PER_IMAGE:
        return 0
    o = abi.ImageOptions(**opt.__dict__)
    o.FileType, o.EncodeOptions = (".webp", {abi.WebpQuality: 80}) if name in ANIMATED else (".png", {abi.PngCompression: 1})
    o.DisableAnimatedOutput = name in ANIMATED
    xb.transform([data], o, out_cap=1 << 25)
    return xb.stats()["grid_items"]


MODES = {
    "fit_square": opts(64, 64, FIT),
    "fit_wide_normalized": opts(120, 40, FIT, NormalizeOrientation=True),
    "resize_tall": opts(40, 120, RESIZE),
    "fit_oversized_normalized": opts(2000, 1500, FIT, NormalizeOrientation=True),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_mixed_corpus(cuda_lib, xb, files, mode):
    """Every status, size and slice against lp_transform; the grid / per-image split exact; no pixel comes home"""
    opt = MODES[mode]
    names, data = [n for n, _ in files], [f for _, f in files]
    H, W = opt.Height, opt.Width
    got, w, h, st = decode(xb, data, opt, H, W)
    s = xb.stats()
    check_items(cuda_lib, data, opt, got, w, h, st, H, W, names=names)
    want = sum(expected_grid(xb, n, f, opt) for n, f in files)
    assert (s["grid_items"], s["fallback_items"]) == (want, len(files) - want)
    assert s["d2h_bytes"] == 0


def test_per_image_options(cuda_lib, xb, files):
    """NoResize and a MaxEncodeDuration send every item per image, still with lp_transform's frame"""
    data = [f for n, f in files if not n.startswith("jpeg_rot")][:12]
    for opt in (abi.ImageOptions(FileType=".webp", ResizeMethod=abi.ImageOpsNoResize, EncodeTimeout_ns=T),
                opts(48, 48, FIT, MaxEncodeDuration_ns=10**9)):
        got, w, h, st = decode(xb, data, opt, 400, 700)
        assert xb.stats()["grid_items"] == 0
        check_items(cuda_lib, data, opt, got, w, h, st, 400, 700)


LAYOUT_FILES = ("jpeg_420", "jpeg_gray", "jpeg_rot6", "png_rgba", "png_gray", "webp_lossy_alpha", "gif_anim", "png_pq")


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("rgb", [False, True])
@pytest.mark.parametrize("nchw", [False, True])
def test_layouts(cuda_lib, xb, files, dtype, ch, rgb, nchw):
    """Every layout, channel order, channel count and dtype, with scale and bias, in a box larger than every frame (its
    odd sizes put slice boundaries inside 16-byte pieces)"""
    sel = dict(files)
    data = [sel[n] for n in LAYOUT_FILES]
    opt = opts(48, 40, FIT, NormalizeOrientation=True)
    got, w, h, st = decode(xb, data, opt, 43, 51, ch, nchw, rgb, dtype)
    assert all(s == 0 for s in st)
    check_items(cuda_lib, data, opt, got, w, h, st, 43, 51, ch, nchw, rgb, dtype, names=list(LAYOUT_FILES))


def test_box_smaller_than_some_frames(cuda_lib, xb, files):
    """A frame over the box in either dimension: LP_ERR_BUF_TOO_SMALL, zero slice, 0 x 0; the items around it intact"""
    data = [f for _, f in files] + [cv2_jpeg(synth_image(50, 24, 30, 3), 90), rgb_png(synth_image(51, 30, 20, 4))]
    opt = opts(64, 64, FIT)
    got, w, h, st = decode(xb, data, opt, 30, 40, 3, True, True, "f16")
    assert abi.LP_ERR_BUF_TOO_SMALL in st and st.count(0) >= 3
    check_items(cuda_lib, data, opt, got, w, h, st, 30, 40, 3, True, True, "f16")


def test_schedule_independence(cuda_lib, xb, files):
    """The same slice alone, in the batch, with both lanes busy, and from a 1 GiB arena that splits the work in chunks"""
    data = [f for _, f in files]
    opt = opts(96, 72, FIT)
    H, W = 72, 96
    whole, w0, h0, st0 = decode(xb, data, opt, H, W, 3, True, True, "bf16")
    many = data * 12
    rng = np.random.default_rng(5)
    order = rng.permutation(len(many))
    busy, w1, h1, st1 = decode(xb, [many[k] for k in order], opt, H, W, 3, True, True, "bf16")
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        chunked, w2, h2, st2 = decode(small, [many[k] for k in order], opt, H, W, 3, True, True, "bf16")
    finally:
        small.close()
    for i in range(len(data)):
        alone, wa, ha, sa = decode(xb, [data[i]], opt, H, W, 3, True, True, "bf16")
        assert (sa[0], wa[0], ha[0]) == (st0[i], w0[i], h0[i])
        assert torch.equal(alone[0], whole[i]), f"item {i}: alone differs from in the batch"
    for j, k in enumerate(order):
        i = k % len(data)
        assert (st1[j], w1[j], h1[j]) == (st0[i], w0[i], h0[i]) == (st2[j], w2[j], h2[j])
        assert torch.equal(busy[j], whole[i]) and torch.equal(chunked[j], whole[i]), f"position {j} (item {i}) differs"


def test_bad_arguments_write_nothing(cuda_lib, xb, files):
    data = [f for _, f in files][:6]
    n, H, W = len(data), 32, 32
    opt = opts(32, 32, FIT)
    t = tensor(n, H, W, 3, "u8", False)
    nbytes = t.numel()
    host = np.zeros(nbytes, np.uint8)
    cases = {
        "undersized": dict(bytes=nbytes - 1),
        "host memory": dict(data_ptr=host.ctypes.data),
        "channels 2": dict(channels=2),
        "channels 5": dict(channels=5),
        "unknown dtype": dict(dtype=7),
        "empty box": dict(height=0),
        "misaligned f32": dict(data_ptr=t.data_ptr() + 2, dtype="f32", bytes=nbytes - 2),
    }
    for what, kw in cases.items():
        a = dict(data_ptr=t.data_ptr(), bytes=nbytes, height=H, width=W, channels=3, dtype="u8")
        a.update(kw)
        with pytest.raises(abi.LilliputError) as e:
            xb.decode_frames(data, opt, **a)
        assert e.value.code == -10, what
    l = cuda_lib.l
    ptrs, lens, keep = abi.Batch._ptr_arrays(data)
    ints = [(C.c_int * n)() for _ in range(3)]
    copt = opt._c()
    good = abi._FrameTensor(t.data_ptr(), nbytes, H, W, 3, 0, 1, 0)
    assert l.lp_xbatch_decode_frames(xb.h, ptrs, lens, n, C.byref(copt), None, *ints) == -10  # null dst
    assert l.lp_xbatch_decode_frames(xb.h, ptrs, lens, -1, C.byref(copt), C.byref(good), *ints) == -10  # negative n
    assert not host.any()
    assert bool((t.view(torch.uint8) == 0x5A).all()), "a refused call wrote into the tensor"


def test_transform_unaffected(cuda_lib, xb, files):
    """lp_xbatch_transform on the same context returns the same bytes before and after a decode_frames call"""
    data = [f for _, f in files]
    for o in (abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=FIT, EncodeOptions={abi.JpegQuality: 85}),
              abi.ImageOptions(FileType=".webp", Width=80, Height=80, ResizeMethod=FIT, EncodeOptions={abi.WebpQuality: 80},
                               EncodeTimeout_ns=T, DisableAnimatedOutput=True)):
        before = xb.transform(data, o, out_cap=1 << 22)
        s_before = {k: xb.stats()[k] for k in ("grid_items", "fallback_items", "d2h_bytes")}
        decode(xb, data, opts(64, 64, FIT), 64, 64)
        assert xb.transform(data, o, out_cap=1 << 22) == before
        assert {k: xb.stats()[k] for k in ("grid_items", "fallback_items", "d2h_bytes")} == s_before
