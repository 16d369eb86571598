"""GPU: the GIF encoder kernels of csrc/gif_decode.cu (palette-run owner election, bucket resolution, mapping with
previous-frame substitution, one-lane LZW) against the oracle's serial encoder, byte for byte, on the catalogue of
tests/gif_encode_cases.py:
  per image  the exported giflib_* surface (include/lp_giflib.h) driven through ctypes with the designed BGRA frames,
             and with destinations cut around frame boundaries (success or failure as the oracle);
  batch      lp_xbatch_transform with .gif output: ImageOpsResize to the source size (a plain copy, so the encoder gets
             the designed composites) and Fit downscales, against the oracle and per-image lp_transform, with
             grid_items asserted so a hand-over to the per-image path cannot pass."""
import ctypes as C
import os
import time

import numpy as np
import pytest

from lilliput_b200 import abi
from tests import gif_encode_cases as ec
from tests.golden.make_golden_gif_encode import TIMEOUT_NS
from tests.test_gif_encode_cases import FITS, given_frames, transcode
from tests.test_gpu_xbatch import check_against_per_image
from tests.test_gpu_xbatch_gif import W as SW, H as SH, synthetic_gifs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ec.cases()


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


class Cgo:
    """giflib_decoder_* / giflib_encoder_* as lilliput's giflib.go calls them."""

    def __init__(self, lib):
        l = self.l = lib.l
        vp = C.c_void_p
        for name, res, args in (("opencv_mat_create_from_data", vp, [C.c_int, C.c_int, C.c_int, vp, C.c_size_t]),
                                ("opencv_mat_release", None, [vp]),
                                ("giflib_decoder_create", vp, [vp]), ("giflib_decoder_release", None, [vp]),
                                ("giflib_decoder_decode_frame_header", C.c_int, [vp]),
                                ("giflib_decoder_decode_frame", C.c_bool, [vp, vp]),
                                ("giflib_encoder_create", vp, [vp, C.c_size_t]),
                                ("giflib_encoder_init", C.c_bool, [vp, vp, C.c_int, C.c_int]),
                                ("giflib_encoder_encode_frame", C.c_bool, [vp, vp, vp]),
                                ("giflib_encoder_flush", C.c_bool, [vp, vp]), ("giflib_encoder_release", None, [vp]),
                                ("giflib_encoder_get_output_length", C.c_int, [vp])):
            f = getattr(l, name)
            f.restype, f.argtypes = res, args

    def mat(self, a):
        h, w = a.shape[:2]
        m = self.l.opencv_mat_create_from_data(w, h, abi.CV_8UC4 if a.ndim == 3 else 0, a.ctypes.data, a.size)
        assert m
        return m

    def transcode(self, gif: bytes, frames, cap: int):
        """Decode every frame, encode frames[k] in its place, flush: (the file or None when a call fails, the number
        of frames encoded)."""
        src = np.frombuffer(gif, np.uint8).copy()
        l = self.l
        bm = l.opencv_mat_create_from_data(src.size, 1, 0, src.ctypes.data, src.size)
        d = l.giflib_decoder_create(bm)
        assert d
        dst = np.zeros(cap, np.uint8)
        e = l.giflib_encoder_create(dst.ctypes.data, cap)
        keep, ok, done = [], True, 0
        try:
            canvas = None
            for k, f in enumerate(frames):
                assert l.giflib_decoder_decode_frame_header(d) == 0
                if canvas is None:
                    h, w = given_frames_shape(gif)
                    canvas = np.zeros((h, w, 4), np.uint8)
                    cm = self.mat(canvas)
                    keep.append(cm)
                assert l.giflib_decoder_decode_frame(d, cm)
                f = np.ascontiguousarray(f)
                fm = self.mat(f)
                keep.append(fm)
                if k == 0:
                    l.giflib_encoder_init(e, d, f.shape[1], f.shape[0])
                if not l.giflib_encoder_encode_frame(e, d, fm):
                    ok = False
                    break
                done += 1
            assert ok is False or l.giflib_decoder_decode_frame_header(d) == 1
            ok = ok and l.giflib_encoder_flush(e, d)
            n = l.giflib_encoder_get_output_length(e)
            return (dst[:n].tobytes() if ok else None), done
        finally:
            l.giflib_encoder_release(e)
            l.giflib_decoder_release(d)
            for m in keep + [bm]:
                l.opencv_mat_release(m)


def given_frames_shape(gif: bytes):
    return int.from_bytes(gif[8:10], "little"), int.from_bytes(gif[6:8], "little")


@pytest.fixture(scope="module")
def cgo(cuda_lib):
    return Cgo(cuda_lib)


def oracle_or_none(oracle, case, frames, cap):
    it = iter(frames)
    try:
        out = oracle.gif_transcode(case.gif, lambda f: next(it), cap=cap)
    except RuntimeError:
        return None
    return out or None


def record_ends(out: bytes):
    """Offsets just behind each extension block and each frame's code stream, and which of them end a frame."""
    ends, p = [], 13 + (3 << ((out[10] & 7) + 1) if out[10] & 0x80 else 0)
    while out[p] != 0x3B:
        image = out[p] == 0x2C
        if image:
            flags = out[p + 9]
            p += 10 + (3 << ((flags & 7) + 1) if flags & 0x80 else 0) + 1
        else:
            p += 2
        while out[p]:
            p += out[p] + 1
        p += 1
        ends.append((p, image))
    return ends


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_per_image_encoder(cgo, oracle, case):
    frames = given_frames(oracle, case)
    want = transcode(oracle, case, frames)
    assert cgo.transcode(case.gif, frames, 16 << 20) == (want, len(frames))
    # destinations cut around the first records' ends and the file's end: success or failure as the oracle, and the
    # frame that fails is the first one whose records do not fit
    ends = record_ends(want)
    cuts = [e for e, _ in ends[:4] + ends[-2:]] + [len(want)]
    for cap in sorted({c for e in cuts for c in (e - 1, e, e + 1)}):
        exp = oracle_or_none(oracle, case, frames, cap)
        got, done = cgo.transcode(case.gif, frames, cap)
        assert (got is None) == (exp is None), f"cap {cap} of {len(want)}: device {got is not None}, oracle {exp is not None}"
        assert done == sum(e <= cap for e, image in ends if image), f"cap {cap}: {done} frames written"
        if got is not None:
            assert got == exp == want


def _goldens(golden):
    return [golden[k].tobytes() for k in sorted(golden.files) if k.startswith("gif_") and golden[k].ndim == 1]


def _batch(cuda_lib, xb, oracle, files, opt, per_frame):
    outs, status = check_against_per_image(cuda_lib, xb, files, opt, cap=16 << 20)
    st = xb.stats()
    assert status == [0] * len(files) and st["grid_items"] == len(files) and st["fallback_items"] == 0, st
    for i, (f, out) in enumerate(zip(files, outs)):
        assert out == oracle.gif_transcode(f, per_frame(f), cap=16 << 20), f"item {i}"
    return outs


def _palette_runs(out: bytes):
    runs, last = [], None
    for f in ec.read_gif(out)["frames"]:
        c = bytes(f["colors"])
        if c == last:
            runs[-1] += 1
        else:
            runs.append(1)
        last = c
    return runs


def test_batch_palette_cases_resize_to_source(cuda_lib, xb, oracle, golden):
    """The W x H file cases interleaved with the golden fixtures in one call: the cases' frames reach the encoder
    unchanged, the fixtures are resized onto the same grid."""
    cases, gold = [c.gif for c in ec.palette_cases()], _goldens(golden)
    files = []
    for i in range(max(len(cases), len(gold))):
        files += cases[i:i + 1] + gold[i:i + 1]
    opt = abi.ImageOptions(FileType=".gif", Width=ec.W, Height=ec.H, ResizeMethod=abi.ImageOpsResize,
                           EncodeTimeout_ns=TIMEOUT_NS)
    outs = _batch(cuda_lib, xb, oracle, files, opt,
                  lambda f: None if f in cases else (lambda fr: oracle.resize(fr, ec.W, ec.H)))
    runs = [n for o in outs for n in _palette_runs(o)]
    assert len(runs) >= 50 and 1 in runs and max(runs) >= 8, runs


@pytest.mark.parametrize("size", FITS, ids=lambda s: f"fit{s[0]}x{s[1]}")
def test_batch_palette_cases_fit(cuda_lib, xb, oracle, golden, size):
    """Fit downscales: alpha averages to 127 / 128 and colours land on bucket edges."""
    files = [c.gif for c in ec.palette_cases()] + _goldens(golden)
    opt = abi.ImageOptions(FileType=".gif", Width=size[0], Height=size[1], ResizeMethod=abi.ImageOpsFit,
                           EncodeTimeout_ns=TIMEOUT_NS)

    def fit(f):
        h, w = oracle.gif_frames(f, max_frames=1)[0][0].shape[:2]
        ow, oh = oracle.expected_size(w, h, *size)
        return lambda fr: oracle.fit(fr, ow, oh)
    _batch(cuda_lib, xb, oracle, files, opt, fit)


def test_batch_lzw_cases(cuda_lib, xb, oracle):
    """Every code size filling the table three times and more, stream lengths on and next to 255 k, 1 x 1, 1 x N,
    N x 1 and interlaced frames of heights 1..17: one call per canvas size, each resized to its own size."""
    groups = {}
    for c in ec.lzw_cases():
        groups.setdefault(given_frames_shape(c.gif), []).append(c.gif)
    for (h, w), files in groups.items():
        opt = abi.ImageOptions(FileType=".gif", Width=w, Height=h, ResizeMethod=abi.ImageOpsResize,
                               EncodeTimeout_ns=TIMEOUT_NS)
        _batch(cuda_lib, xb, oracle, files, opt, lambda f: None)


@pytest.mark.parametrize("case", ec.big_cases(), ids=lambda c: c.name)
def test_large_frames(cuda_lib, xb, oracle, cgo, case):
    """Frames that fill the string table dozens of times, per image and in the batch; the wall time of each path is
    printed (the LZW kernel is one lane per frame)."""
    h, w = given_frames_shape(case.gif)
    want = oracle.gif_transcode(case.gif, cap=16 << 20)
    frames = given_frames(oracle, case)
    t = time.perf_counter()
    assert cgo.transcode(case.gif, frames, 16 << 20) == (want, len(frames))
    t_img = time.perf_counter() - t
    opt = abi.ImageOptions(FileType=".gif", Width=w, Height=h, ResizeMethod=abi.ImageOpsResize,
                           EncodeTimeout_ns=TIMEOUT_NS)
    t = time.perf_counter()
    outs, status = xb.transform([case.gif], opt, out_cap=16 << 20)
    t_batch = time.perf_counter() - t
    assert status == [0] and xb.stats()["grid_items"] == 1 and outs[0] == want
    assert min(f["full_clears"] for f in ec.read_gif(want)["frames"]) >= 10
    print(f"{case.name}: per image {t_img * 1e3:.0f} ms, batch {t_batch * 1e3:.0f} ms for {len(frames)} frames")


@pytest.mark.parametrize("kw", [dict(Width=40, Height=40, ResizeMethod=abi.ImageOpsFit),
                                dict(Width=50, Height=23, ResizeMethod=abi.ImageOpsResize),
                                dict(Width=SW, Height=SH, ResizeMethod=abi.ImageOpsResize)],
                         ids=["fit40", "resize50x23", "resize_to_source"])
def test_synthetic_animations_against_the_oracle(cuda_lib, xb, oracle, kw):
    """The designed animations of test_gpu_xbatch_gif.py, which otherwise meet only the per-image path."""
    files = list(synthetic_gifs().values())
    opt = abi.ImageOptions(FileType=".gif", EncodeTimeout_ns=TIMEOUT_NS, **kw)
    w, h = kw["Width"], kw["Height"]
    if kw["ResizeMethod"] == abi.ImageOpsFit:
        ow, oh = oracle.expected_size(SW, SH, w, h)
        per_frame = lambda f: (lambda fr: oracle.fit(fr, ow, oh))   # noqa: E731
    elif (w, h) == (SW, SH):
        per_frame = lambda f: None   # noqa: E731
    else:
        per_frame = lambda f: (lambda fr: oracle.resize(fr, w, h))   # noqa: E731
    _batch(cuda_lib, xb, oracle, files, opt, per_frame)
