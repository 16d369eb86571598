"""GPU: JPEG sources to lossy WebP in the heterogeneous batch (lp_xbatch_transform, csrc/xbatch.cu): the lp_batch
pipeline of a JPEG group stops after the resize and its frames go to the batched WebP encoder; JPEG, PNG and WebP
sources carry their ICC profiles into the file as WebpEncoder does.

Every item is compared with per-image lp_transform of the same library (status and bytes), and grid_items /
fallback_items are asserted exactly, so a silent hand-over to the per-image path cannot pass.  Outside ourselves:
libwebp decodes every output as our decoder does, and the pixels are close to the oracle's decode + Fit."""
import struct
import zlib

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests import jpeg_scan_streams as js
from tests import vp8l_streams as vs
from tests.test_gpu_xbatch import check_against_per_image, rgb_png
from tests.webp_util import chunks_of, libwebp_decode, optional_reference, psnr

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
T = 10**12

FIT = dict(Width=256, Height=256, ResizeMethod=abi.ImageOpsFit)
RESIZE = dict(Width=300, Height=170, ResizeMethod=abi.ImageOpsResize)


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def webp_opt(q=85, **kw):
    kw.setdefault("EncodeTimeout_ns", T)
    return abi.ImageOptions(FileType=".webp", EncodeOptions={abi.WebpQuality: q}, **kw)


def cv2_jpeg(img, q=90, sampling=None, optimize=False, rst=0, progressive=False):
    flags = [cv2.IMWRITE_JPEG_QUALITY, q]
    if sampling is not None:
        flags += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sampling]
    if optimize:
        flags += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if rst:
        flags += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if progressive:
        flags += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, b = cv2.imencode(".jpg", img, flags)
    assert ok
    return bytes(b)


def after_app0(jpeg: bytes, *segments: bytes) -> bytes:
    """Segments inserted behind SOI and the JFIF APP0 segment cv2 writes."""
    at = 2
    if jpeg[2:4] == b"\xff\xe0":
        at = 4 + struct.unpack(">H", jpeg[4:6])[0]
    return jpeg[:at] + b"".join(segments) + jpeg[at:]


def app2(seq, cnt, body):
    payload = b"ICC_PROFILE\0" + bytes([seq, cnt]) + body
    return b"\xff\xe2" + struct.pack(">H", len(payload) + 2) + payload


def icc_profile(n, seed=7, declared=None):
    """Bytes shaped like an ICC profile as far as the WebP writer looks: the big-endian size field (= n unless given)."""
    b = bytearray(np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes())
    b[0:4] = (n if declared is None else declared).to_bytes(4, "big")
    return bytes(b)


def png_profile(n=532, seed=3):
    """A profile libpng's png_get_iCCP accepts: an RGB display-class v4 header (D50, acsp, no tags) + a seeded tail."""
    p = bytearray(np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes())
    p[0:132] = bytes(132)
    p[0:4] = struct.pack(">I", n)
    p[8] = 4
    p[12:16], p[16:20], p[20:24], p[36:40] = b"mntr", b"RGB ", b"XYZ ", b"acsp"
    p[68:80] = bytes([0, 0, 0xf6, 0xd6, 0, 1, 0, 0, 0, 0, 0xd3, 0x2d])
    return bytes(p)


def with_iccp(png: bytes, profile: bytes) -> bytes:
    body = b"icc\0\0" + zlib.compress(profile, 6)
    chunk = struct.pack(">I", len(body)) + b"iCCP" + body + struct.pack(">I", zlib.crc32(b"iCCP" + body))
    return png[:33] + chunk + png[33:]  # behind IHDR


def with_exif_orientation(jpeg: bytes, orientation: int) -> bytes:
    tiff = b"II*\x00\x08\x00\x00\x00" + b"\x01\x00" + b"\x12\x01\x03\x00\x01\x00\x00\x00" + bytes([orientation, 0, 0, 0]) + b"\x00\x00\x00\x00"
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + jpeg[2:]


def webp_still_with_icc(icc, w=40, h=30, seed=42):
    return vs.riff(vs.vp8x(w, h, 0x20) + vs.chunk(b"ICCP", icc) + vs.chunk(b"VP8 ", vs.lossy_payload(w, h, seed)))


# ---------------------------------------------------------------- every JPEG kind on the grid

SIZES = [(854, 480), (1280, 720), (500, 333), (17, 9)]
KINDS = ["420", "422", "444", "optimize", "rst", "progressive", "per_component"]


def jpeg_kinds():
    """(name, file): every kind at every size, source qualities spread over 1..100, and one 3840x2160."""
    samp = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}
    out, k = [], 0
    for w, h in SIZES:
        for kind in KINDS:
            q = [1, 100, 37, 64, 12, 88, 50][k % 7] if k < 7 else 1 + (k * 37) % 100
            seed = 4000 + k
            if kind == "per_component":  # one scan per component, from the stream writer (its own quantisation)
                data = js.write(js.frame("420", w, h, seed), js.sequential_per_component(), progressive=False)
                out.append((f"{kind}_{w}x{h}", data))
            else:
                img = synth_image(seed, w, h, 3, noise=3.0 + k % 5)
                data = cv2_jpeg(img, q, sampling=samp.get(kind), optimize=kind == "optimize", rst=5 if kind == "rst" else 0,
                                progressive=kind == "progressive")
                out.append((f"{kind}_{w}x{h}_q{q}", data))
            k += 1
    out.append(("420_3840x2160_q90", cv2_jpeg(synth_image(4100, 3840, 2160, 3), 90)))
    return out


@pytest.fixture(scope="module")
def kinds():
    return jpeg_kinds()


@pytest.mark.parametrize("geom", [FIT, RESIZE], ids=["fit", "resize"])
def test_every_jpeg_kind_on_the_grid(cuda_lib, xb, kinds, geom):
    files = [d for _, d in kinds]
    for q in (1, 50, 85, 100):
        _, status = check_against_per_image(cuda_lib, xb, files, webp_opt(q, **geom))
        assert status == [0] * len(files), dict(zip([n for n, _ in kinds], status))
        st = xb.stats()
        assert st["grid_items"] == len(files) and st["fallback_items"] == 0, (q, st)
        assert st["ms_decode"] > 0 and st["ms_resize"] > 0 and st["ms_encode"] > 0, st


def test_against_libwebp_and_the_oracle(cuda_lib, xb, kinds, oracle):
    names = [n for n, _ in kinds]
    files = [d for _, d in kinds]
    outs, status = xb.transform(files, webp_opt(85, **FIT), out_cap=1 << 22)
    assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
    ref_lib = optional_reference()
    for name, f, out in zip(names, files, outs):
        got = libwebp_decode(out)
        _, mine, _, rc = cuda_lib.webp_frames(out)
        assert rc == 0 and np.array_equal(mine[0], got), name
        if ref_lib:
            _, frames, _, rc = ref_lib.webp_frames(out)
            assert rc == 0 and np.array_equal(frames[0], got), name
        dec, _ = oracle.jpeg_decode(f)
        ew, eh = oracle.expected_size(dec.shape[1], dec.shape[0], 256, 256)
        fit = oracle.fit(dec, ew, eh)
        assert got.shape == fit.shape, name
        # (a 9x9 frame is all block edges, and the stream writer's frames are random coefficients -- noise to a lossy
        # encoder: for those, libwebp's decode above is the check)
        if min(ew, eh) >= 64 and not name.startswith("per_component"):
            assert psnr(got, fit) > 28.0, name


# ---------------------------------------------------------------- ICC profiles

def test_icc_profiles_travel_into_the_webp(cuda_lib, xb):
    base = cv2_jpeg(synth_image(4200, 640, 360, 3), 85)
    prof = icc_profile(3000)
    big = icc_profile(40000, seed=8)
    good_png = png_profile()
    cases = {
        "jpeg_one_segment": (after_app0(base, app2(1, 1, prof)), prof),
        "jpeg_three_segments": (after_app0(base, app2(1, 3, prof[:1000]), app2(2, 3, prof[1000:2200]), app2(3, 3, prof[2200:])), prof),
        "jpeg_three_out_of_order": (after_app0(base, app2(3, 3, prof[2200:]), app2(1, 3, prof[:1000]), app2(2, 3, prof[1000:2200])), prof),
        "jpeg_missing_segment": (after_app0(base, app2(1, 3, prof[:1000]), app2(3, 3, prof[2200:])), None),
        "jpeg_declared_size_disagrees": (after_app0(base, app2(1, 1, icc_profile(3000, declared=3001))), None),
        "jpeg_shorter_than_header": (after_app0(base, app2(1, 1, icc_profile(100))), None),
        "jpeg_over_32k": (after_app0(base, app2(1, 2, big[:20000]), app2(2, 2, big[20000:])), None),
        "jpeg_no_profile": (base, None),
        "png_valid_iccp": (with_iccp(rgb_png(synth_image(4201, 300, 200, 3)), good_png), good_png),
        "png_rgba_valid_iccp": (with_iccp(rgb_png(synth_image(4202, 300, 200, 4)), good_png), good_png),
        "png_iccp_libpng_refuses": (with_iccp(rgb_png(synth_image(4203, 300, 200, 3)), bytes(range(200)) * 3), None),
        "webp_with_icc": (webp_still_with_icc(icc_profile(400, seed=9)), icc_profile(400, seed=9)),
        "webp_icc_size_disagrees": (webp_still_with_icc(icc_profile(400, seed=9, declared=5)), None),
    }
    files = [f for f, _ in cases.values()]
    for geom in (FIT, RESIZE):
        outs, status = check_against_per_image(cuda_lib, xb, files, webp_opt(85, **geom))
        assert status == [0] * len(files), dict(zip(cases, status))
        st = xb.stats()
        assert st["grid_items"] == len(files) and st["fallback_items"] == 0, st
        for (name, (_, want)), out in zip(cases.items(), outs):
            got = dict(chunks_of(out)).get(b"ICCP")
            assert got == want, name


# ---------------------------------------------------------------- what stays per image

def test_per_image_routing(cuda_lib, xb):
    good = [cv2_jpeg(synth_image(4300 + k, 320 + 32 * k, 240, 3), 80) for k in range(3)]
    gray = cv2_jpeg(synth_image(4310, 320, 240, 1), 80)
    rotated = with_exif_orientation(good[0], 6)
    damaged = b"\xff\xd8\xff\xe0 not a jpeg at all"
    truncated = good[1][: len(good[1]) // 2]
    after = cv2_jpeg(synth_image(4320, 352, 240, 3), 80)  # good[1]'s geometry: the truncated file sits inside its group
    files = good + [gray, rotated, damaged, truncated, after]
    _, status = check_against_per_image(cuda_lib, xb, files, webp_opt(85, NormalizeOrientation=True, **FIT))
    # (the gray file fails per image too: the WebP writer takes BGR or BGRA frames only)
    assert status[:3] == [0] * 3 and status[3] == abi.LP_ERR_INVALID_IMAGE and status[4] == 0 and status[5] != 0
    assert status[7] == 0
    st = xb.stats()
    # the truncated file passes the header parser; the device decode refuses it (the stream ends before the last MCU)
    # and it is handed over, its group's other files encoded on either side of it
    assert st["grid_items"] == 4 and st["fallback_items"] == 4, st
    for opt in (webp_opt(85, EncodeTimeout_ns=0, **FIT), webp_opt(101, **FIT)):
        check_against_per_image(cuda_lib, xb, good, opt)
        st = xb.stats()
        assert st["grid_items"] == 0 and st["fallback_items"] == len(good), (opt, st)


def test_options(cuda_lib, xb):
    files = [cv2_jpeg(synth_image(4400 + k, 400, 300, 3), 85) for k in range(4)]
    files.append(after_app0(files[0], app2(1, 1, icc_profile(2000))))
    # a PNG with a profile: under MaxEncodeFrames 1 and a negative MaxEncodeDuration the per-image path fails it (the
    # PNG decoder cannot skip to the end either), so it stays there as the JPEGs do
    files.append(with_iccp(rgb_png(synth_image(4410, 400, 300, 3)), png_profile()))
    n = len(files)
    for kw, grid in [(dict(DisableAnimatedOutput=True), n),
                     (dict(MaxEncodeFrames=1), 0),
                     (dict(MaxEncodeFrames=2), n),
                     (dict(MaxEncodeDuration_ns=1), n),
                     (dict(MaxEncodeDuration_ns=-1), 0)]:
        _, status = check_against_per_image(cuda_lib, xb, files, webp_opt(85, **kw, **FIT))
        st = xb.stats()
        assert st["grid_items"] == grid and st["fallback_items"] == n - grid, (kw, st)
        if grid:
            assert status == [0] * n, (kw, status)
    # an output buffer too small for the file: ErrInvalidImage, as per image (the WebP writer returns no bytes)
    _, status = check_against_per_image(cuda_lib, xb, files, webp_opt(85, **FIT), cap=700)
    assert status == [abi.LP_ERR_INVALID_IMAGE] * n and xb.stats()["grid_items"] == n


# ---------------------------------------------------------------- config 5 in miniature, to WebP

def config5_to_webp_files(cuda_lib):
    files = []
    for k, (w, h) in enumerate([(854, 480), (1280, 720), (854, 480), (640, 360)]):
        files.append(cv2_jpeg(synth_image(4500 + k, w, h, 3), 90))
    files.append(after_app0(files[0], app2(1, 1, icc_profile(3000, seed=11))))
    files.append(rgb_png(synth_image(4510, 854, 480, 3)))
    files.append(rgb_png(synth_image(4511, 640, 360, 4)))
    files.append(with_iccp(rgb_png(synth_image(4512, 640, 360, 3)), png_profile()))
    files.append(cuda_lib.encode(".webp", synth_image(4520, 854, 480, 3), {abi.WebpQuality: 85}))
    files.append(cuda_lib.encode(".webp", synth_image(4521, 1280, 720, 3), {abi.WebpQuality: 85}))
    return files


def test_config5_miniature_to_webp(cuda_lib, xb):
    files = config5_to_webp_files(cuda_lib)
    opt = webp_opt(85, NormalizeOrientation=True, **FIT)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt)
    assert status == [0] * len(files)
    st = xb.stats()
    assert st["grid_items"] == len(files) and st["fallback_items"] == 0, st
    m = abi.MultiBatch(cuda_lib, [0, 0], arena_bytes=4 << 30)
    try:
        m_outs, m_status = m.transform(files, opt, out_cap=1 << 22)
        assert m_status == status and m_outs == outs
        assert sum(m.stats(g)["grid_items"] for g in range(2)) == len(files)
        assert sum(m.stats(g)["fallback_items"] for g in range(2)) == 0
    finally:
        m.close()
