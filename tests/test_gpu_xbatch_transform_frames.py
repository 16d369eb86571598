"""GPU: lp_xbatch_transform_frames -- file renditions and frame renditions of the same uploads in one call.

The yardsticks are the two calls it replaces, on the same context: every file pair must equal what
lp_xbatch_transform_renditions writes (status and bytes), and every frame rendition's tensor, sizes and statuses what
lp_xbatch_decode_frames writes, bit for bit, with the same sentinel in both tensors and guard bytes behind the last
slice that must stay untouched.  The routing is asserted exactly against the same calls: the pairs the mixed call runs
on the grid are the renditions call's plus each decode_frames call's."""
import ctypes as C

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch_frames import BIAS, DTYPES, SCALE, corpus
from tests.test_gpu_xbatch_jpeg_webp import cv2_jpeg, with_exif_orientation
from tests.test_gpu_xbatch_renditions import RENDITION_SETS, grid_files

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
T = 10**12
CAP = 1 << 22
FIT, RESIZE = abi.ImageOpsFit, abi.ImageOpsResize
FILL, GUARD = 0x5A, 4096  # sentinel byte; guard bytes behind the n slices
BAD_ARGUMENT = -10  # LP_ERR_BAD_ARGUMENT
PACK_ENTRY = 32  # sizeof(FramePackItem): one per packed frame, the only bytes a frame rendition uploads


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


@pytest.fixture(scope="module")
def files():
    return corpus()


def file_opts(w, h, method, norm):
    def o(ext, enc, **kw):
        return abi.ImageOptions(FileType=ext, Width=w, Height=h, ResizeMethod=method, NormalizeOrientation=norm,
                                EncodeOptions=enc, EncodeTimeout_ns=T, **kw)
    return [o(".jpeg", {abi.JpegQuality: 85}), o(".webp", {abi.WebpQuality: 80}), o(".png", {abi.PngCompression: 1})]


class Frame:
    """A frame rendition: its options and tensor layout, and a device buffer of n slices + GUARD bytes, prefilled"""

    def __init__(self, opt, H, W, ch, nchw, rgb, dtype, scaled):
        self.opt, self.H, self.W, self.ch, self.nchw, self.rgb, self.dtype = opt, H, W, ch, nchw, rgb, dtype
        self.scale, self.bias = (SCALE, BIAS) if scaled else (None, None)

    def slice_bytes(self):
        return self.H * self.W * self.ch * torch.empty((), dtype=DTYPES[self.dtype]).element_size()

    def buffer(self, n):
        b = torch.full((n * self.slice_bytes() + GUARD,), FILL, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()  # (the library's streams do not wait for torch's)
        return b

    def spec(self, buf, n, **kw):
        s = dict(opt=self.opt, data_ptr=buf.data_ptr(), bytes=n * self.slice_bytes(), height=self.H, width=self.W,
                 channels=self.ch, nchw=self.nchw, rgb=self.rgb, dtype=self.dtype, scale=self.scale, bias=self.bias)
        s.update(kw)
        return s

    def decode_frames(self, xb, data):
        buf = self.buffer(len(data))
        s = self.spec(buf, len(data))
        w, h, st = xb.decode_frames(data, s["opt"], s["data_ptr"], s["bytes"], self.H, self.W, self.ch, self.nchw, self.rgb,
                                    self.dtype, self.scale, self.bias)
        return buf.cpu(), (w, h, st), xb.stats()


def frame_renditions(norm, method=FIT):
    def o(w, h):
        return abi.ImageOptions(FileType=".png", Width=w, Height=h, ResizeMethod=method, NormalizeOrientation=norm)
    return [Frame(o(224, 224), 224, 224, 3, True, True, "f16", True), Frame(o(96, 96), 96, 96, 4, False, False, "u8", False)]


def mixed(xb, data, opts, frames):
    bufs = [f.buffer(len(data)) for f in frames]
    outs, status, sizes = xb.transform_frames(data, opts, [f.spec(b, len(data)) for f, b in zip(frames, bufs)], out_cap=CAP)
    return outs, status, [b.cpu() for b in bufs], sizes, xb.stats()


def check_against_separate_calls(xb, data, opts, frames, names=None):
    """The mixed call against transform_renditions + one decode_frames per frame rendition; returns the mixed stats"""
    outs, status, tensors, sizes, s = mixed(xb, data, opts, frames)
    grid = fallback = 0
    if opts:
        r_outs, r_status = xb.transform_renditions(data, opts, out_cap=CAP)
        rs = xb.stats()
        grid, fallback = rs["grid_items"], rs["fallback_items"]
        for i in range(len(data)):
            what = f"item {i} ({names[i] if names else ''})"
            assert status[i] == r_status[i], f"{what}: status {status[i]}, transform_renditions {r_status[i]}"
            assert outs[i] == r_outs[i], f"{what}: file bytes differ from transform_renditions"
    for j, f in enumerate(frames):
        want, want_sizes, fs = f.decode_frames(xb, data)
        grid += fs["grid_items"]
        fallback += fs["fallback_items"]
        assert sizes[j] == want_sizes, f"frame rendition {j}: sizes / statuses differ from decode_frames"
        assert bool((tensors[j][-GUARD:] == FILL).all()), f"frame rendition {j}: a guard byte past the last slice was written"
        if not torch.equal(tensors[j], want):
            per = f.slice_bytes()
            bad = sorted({int(b) // per for b in torch.nonzero(tensors[j] != want).flatten()[:1000]})
            raise AssertionError(f"frame rendition {j}: slices {bad[:10]} differ from decode_frames")
    assert (s["grid_items"], s["fallback_items"]) == (grid, fallback), (s, grid, fallback)
    assert s["grid_items"] + s["fallback_items"] == len(data) * (len(opts) + len(frames))
    return s


MODES = {
    "fit_normalized": (FIT, True),
    "resize": (RESIZE, False),
    "fit": (FIT, False),
    "resize_normalized": (RESIZE, True),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_equal_to_separate_calls(xb, files, mode):
    """k = 3 file renditions and m = 2 frame renditions over every source kind, damaged files included"""
    method, norm = MODES[mode]
    names, data = [n for n, _ in files], [f for _, f in files]
    check_against_separate_calls(xb, data, file_opts(200, 150, method, norm), frame_renditions(norm, method), names)


def test_each_file_is_uploaded_once(xb):
    """Frame renditions beside file renditions on the grid upload nothing but their pack tables"""
    data = grid_files()
    opts, frames = RENDITION_SETS["thumbnails"], frame_renditions(True)
    s = check_against_separate_calls(xb, data, opts, frames)
    assert s["fallback_items"] == 0, s
    xb.transform_renditions(data, opts, out_cap=CAP)
    files_only = xb.stats()
    assert s["h2d_bytes"] - files_only["h2d_bytes"] == len(frames) * len(data) * PACK_ENTRY, (s, files_only)
    assert s["d2h_bytes"] == files_only["d2h_bytes"]


def test_jpeg_decode_time_is_not_doubled(xb):
    """On JPEGs, the mixed call's decode stage is the files-only call's, not the sum of two calls'"""
    data = [cv2_jpeg(synth_image(200 + k, 1920, 1080, 3), 90) for k in range(8)] * 24
    # (two file renditions: the files-only call decodes through the same resize-only context, whose stage times it reports)
    opts, frames = file_opts(256, 256, FIT, True)[:2], frame_renditions(True)[:1]
    bufs = [f.buffer(len(data)) for f in frames]
    specs = [f.spec(b, len(data)) for f, b in zip(frames, bufs)]
    both, files_only, decode_only = [], [], []
    for _ in range(4):
        xb.transform_frames(data, opts, specs, out_cap=CAP)
        both.append(xb.stats()["ms_decode"])
        xb.transform_renditions(data, opts, out_cap=CAP)
        files_only.append(xb.stats()["ms_decode"])
        frames[0].decode_frames(xb, data)
        decode_only.append(xb.stats()["ms_decode"])
    m_both, m_files, m_frames = min(both[1:]), min(files_only[1:]), min(decode_only[1:])
    assert m_both < 0.5 * (m_files + m_frames) + 0.25 * m_files, (both, files_only, decode_only)


def test_one_frame_rendition_alone_is_decode_frames(cuda_lib, xb, files):
    data = [f for _, f in files]
    f = frame_renditions(True)[0]
    _, _, tensors, sizes, s = mixed(xb, data, [], [f])
    want, want_sizes, ws = f.decode_frames(xb, data)
    assert torch.equal(tensors[0], want) and sizes[0] == want_sizes
    keys = ("grid_items", "fallback_items", "groups", "launches", "h2d_bytes", "d2h_bytes")
    assert {k: s[k] for k in keys} == {k: ws[k] for k in keys}


def test_file_renditions_alone_are_transform_renditions(xb, files):
    data = [f for _, f in files]
    opts = file_opts(100, 100, FIT, True)
    outs, status, _, sizes, s = mixed(xb, data, opts, [])
    assert sizes == []
    assert (outs, status) == xb.transform_renditions(data, opts, out_cap=CAP)
    rs = xb.stats()
    keys = ("grid_items", "fallback_items", "groups", "launches", "h2d_bytes", "d2h_bytes")
    assert {k: s[k] for k in keys} == {k: rs[k] for k in keys}


def test_box_too_small_in_one_rendition_only(xb, files):
    """A frame over one tensor's box is LP_ERR_BUF_TOO_SMALL there and nowhere else"""
    data = [f for _, f in files]
    norm = True
    o = abi.ImageOptions(FileType=".png", Width=160, Height=160, ResizeMethod=FIT, NormalizeOrientation=norm)
    frames = [Frame(o, 120, 120, 3, False, True, "u8", False), Frame(o, 160, 160, 3, True, True, "bf16", True)]
    check_against_separate_calls(xb, data, file_opts(160, 160, FIT, norm)[:1], frames)
    _, _, _, sizes, _ = mixed(xb, data, file_opts(160, 160, FIT, norm)[:1], frames)
    assert abi.LP_ERR_BUF_TOO_SMALL in sizes[0][2] and abi.LP_ERR_BUF_TOO_SMALL not in sizes[1][2]


def test_no_resize_frames_beside_grid_files(xb, files):
    """A NoResize frame rendition (every item per image) beside file renditions on the grid"""
    data = [f for _, f in files][:14]
    nr = abi.ImageOptions(FileType=".png", ResizeMethod=abi.ImageOpsNoResize)
    frames = [Frame(nr, 400, 700, 4, False, False, "u8", False)]
    s = check_against_separate_calls(xb, data, file_opts(64, 64, FIT, True), frames)
    assert s["grid_items"] > 0


def test_two_frame_renditions_over_rotated_and_gray_jpegs(xb):
    rot = cv2_jpeg(synth_image(300, 200, 120, 3), 90)
    data = [with_exif_orientation(rot, o) for o in range(1, 9)]
    data += [cv2_jpeg(synth_image(301, 120, 90, 1), 90), cv2_jpeg(synth_image(302, 75, 131, 1), 85, progressive=True)]
    data += [cv2_jpeg(synth_image(303, 200, 120, 3), 80)] * 3  # upright files of the rotated ones' geometry
    for norm in (True, False):
        frames = frame_renditions(norm)
        s = check_against_separate_calls(xb, data, file_opts(64, 48, FIT, norm), frames)
        assert s["grid_items"] >= len(data) * len(frames)
        check_against_separate_calls(xb, data, [], frames)


def test_many_1080p_jpegs(xb):
    """Enough files for several decode chunks on both lanes"""
    data = [cv2_jpeg(synth_image(400 + k, 1920, 1080, 3), 90) for k in range(8)] * 80
    data[::7] = [with_exif_orientation(d, 6) for d in data[::7]]
    frames = [Frame(abi.ImageOptions(FileType=".png", Width=224, Height=224, ResizeMethod=FIT, NormalizeOrientation=True),
                    224, 224, 3, True, True, "f16", True)]
    s = check_against_separate_calls(xb, data, file_opts(256, 256, FIT, True)[:2], frames)
    assert s["fallback_items"] == 2 * len(data[::7]), s


def test_bad_arguments_write_nothing(cuda_lib, xb, files):
    l = cuda_lib.l
    data = [f for _, f in files][:5]
    n = len(data)
    ptrs, lens, keep = abi.Batch._ptr_arrays(data)
    fr = frame_renditions(True)
    bufs = [f.buffer(n) for f in fr]
    cs = [o._c() for o in file_opts(64, 64, FIT, True)]
    copts = (abi._ImageOptions * 3)(*cs)
    outbuf = np.zeros((n * 3, 1 << 16), np.uint8)
    out_ptrs = (C.c_void_p * (n * 3))(*[outbuf[p].ctypes.data for p in range(n * 3)])
    out_lens = (C.c_size_t * (n * 3))(*([777] * (n * 3)))
    status = (C.c_int * (n * 3))(*([555] * (n * 3)))
    sizes = [[(C.c_int * n)(*([333] * n)) for _ in range(3)] for _ in fr]
    fcs = [f.opt._c() for f in fr]
    host = np.zeros(fr[1].slice_bytes() * n, np.uint8)

    def frs(mutate=None):
        arr = []
        for j, f in enumerate(fr):
            s = f.spec(bufs[j], n)
            if mutate:
                mutate(j, s)
            t = abi._frame_tensor(**{a: s[a] for a in ("data_ptr", "bytes", "height", "width", "channels", "nchw", "rgb",
                                                       "dtype", "scale", "bias")})
            arr.append(abi._FrameRendition(fcs[j], t, *[C.cast(z, C.c_void_p) for z in sizes[j]]))
        return (abi._FrameRendition * len(arr))(*arr)

    def call(k=3, m=2, opts=copts, out=out_ptrs, olen=out_lens, st=status, frames=None, nn=n):
        f = frs() if frames is None else frames
        return l.lp_xbatch_transform_frames(xb.h, ptrs, lens, nn, opts, k, out, 1 << 16, olen, st, f, m)

    def set_(key, value, only=None):
        def mutate(j, s):
            if only is None or j == only:
                s[key] = value
        return frs(mutate)

    many = (abi._FrameRendition * 16)(*([frs()[0]] * 16))
    cases = {
        "k + m = 0": lambda: call(k=0, m=0),
        "k + m = 17": lambda: call(k=3, m=14, frames=many),
        "negative k": lambda: call(k=-1, m=2),
        "negative m": lambda: call(k=3, m=-1),
        "negative n": lambda: call(nn=-1),
        "null opts": lambda: call(opts=None),
        "null out": lambda: call(out=None),
        "null out_len": lambda: call(olen=None),
        "null status": lambda: call(st=None),
        "null frames": lambda: l.lp_xbatch_transform_frames(xb.h, ptrs, lens, n, copts, 3, out_ptrs, 1 << 16, out_lens, status,
                                                            None, 2),
        "null in": lambda: l.lp_xbatch_transform_frames(xb.h, None, lens, n, copts, 3, out_ptrs, 1 << 16, out_lens, status, frs(), 2),
        "host memory": lambda: call(frames=set_("data_ptr", host.ctypes.data, only=1)),
        "undersized second": lambda: call(frames=set_("bytes", n * fr[1].slice_bytes() - 1, only=1)),
        "bad dtype in the second only": lambda: call(frames=set_("dtype", 7, only=1)),
        "overlapping tensors": lambda: call(frames=set_("data_ptr", bufs[0].data_ptr() + 64, only=1)),
        "same tensor twice": lambda: call(frames=set_("data_ptr", bufs[0].data_ptr(), only=1)),
    }

    def null_size(j, what):
        arr = frs()
        setattr(arr[j], what, None)
        return arr
    for what in ("width", "height", "status"):
        cases[f"null {what} of the second"] = (lambda w: lambda: call(frames=null_size(1, w)))(what)
    if torch.cuda.device_count() > 1:
        other = torch.full((n * fr[1].slice_bytes(),), FILL, dtype=torch.uint8, device="cuda:1")
        cases["another device's memory"] = lambda: call(frames=set_("data_ptr", other.data_ptr(), only=1))
    for what, fn in cases.items():
        assert fn() == BAD_ARGUMENT, what
    torch.cuda.synchronize()
    assert list(out_lens) == [777] * (n * 3) and list(status) == [555] * (n * 3)
    assert all(list(z) == [333] * n for s in sizes for z in s)
    assert not outbuf.any() and not host.any()
    for b in bufs:
        assert bool((b == FILL).all()), "a refused call wrote into a tensor"
    # the same arrays in a good call: written
    assert call() == 0
    assert 555 not in list(status) and all(333 not in list(z) for s in sizes for z in s)
