"""GPU: PNG output in the heterogeneous batch (lp_xbatch_transform, csrc/xbatch.cu): JPEG, PNG and WebP stills are
decoded and resized on the grid path and every run of resized frames goes through png_encode_batch (csrc/png_encode.cu:
filter, DEFLATE, checksums and container on the device, whole files in device slots).

Every item is compared with per-image lp_transform of the same library (status and bytes), and grid_items /
fallback_items are asserted exactly, so a silent hand-over to the per-image path cannot pass.  Outside ourselves: cv2 and
Pillow (libpng: both chunk CRCs and the Adler-32 are verified on read) decode every output to the resized pixels."""
import io
import struct
import zlib

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch import check_against_per_image, per_image, rgb_png

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
T = 10**12

FIT = dict(Width=256, Height=256, ResizeMethod=abi.ImageOpsFit)
RESIZE = dict(Width=300, Height=170, ResizeMethod=abi.ImageOpsResize)
LEVELS = [None, 0, 1, 3, 6, 9]


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def png_opt(level=3, **kw):
    kw.setdefault("EncodeTimeout_ns", T)
    return abi.ImageOptions(FileType=".png", EncodeOptions={} if level is None else {abi.PngCompression: level}, **kw)


def cv2_jpeg(img, q=90, *flags):
    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, *flags])
    assert ok
    return bytes(b)


def with_exif_orientation(jpeg: bytes, orientation: int) -> bytes:
    tiff = b"II*\x00\x08\x00\x00\x00" + b"\x01\x00" + b"\x12\x01\x03\x00\x01\x00\x00\x00" + bytes([orientation, 0, 0, 0]) + b"\x00\x00\x00\x00"
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + jpeg[2:]


def with_cicp(png: bytes, primaries=1, transfer=13) -> bytes:
    body = bytes([primaries, transfer, 0, 1])
    chunk = struct.pack(">I", 4) + b"cICP" + body + struct.pack(">I", zlib.crc32(b"cICP" + body))
    return png[:33] + chunk + png[33:]  # behind IHDR


def pillow_animation(w=48, h=32, n=3):
    from PIL import Image
    ims = [Image.fromarray(synth_image(5900 + k, w, h, 3)[:, :, ::-1].copy()) for k in range(n)]
    buf = io.BytesIO()
    ims[0].save(buf, "WEBP", save_all=True, append_images=ims[1:], duration=40, quality=70)
    return buf.getvalue()


def mixed_files(cuda_lib):
    """(name, file): the formats and kinds the grid path takes to PNG."""
    out = []
    for k, (w, h) in enumerate([(854, 480), (500, 333), (1280, 720), (17, 9)]):
        out.append((f"jpeg_baseline_{w}x{h}", cv2_jpeg(synth_image(5000 + k, w, h, 3, noise=3.0), 85)))
    out.append(("jpeg_progressive", cv2_jpeg(synth_image(5010, 854, 480, 3), 80, cv2.IMWRITE_JPEG_PROGRESSIVE, 1)))
    out.append(("jpeg_444", cv2_jpeg(synth_image(5011, 640, 360, 3), 92, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                     cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444)))
    out.append(("jpeg_rst", cv2_jpeg(synth_image(5012, 640, 360, 3), 70, cv2.IMWRITE_JPEG_RST_INTERVAL, 5)))
    out.append(("png_rgb", rgb_png(synth_image(5020, 640, 360, 3))))
    out.append(("png_rgb_same_size", rgb_png(synth_image(5021, 640, 360, 3, noise=12.0))))
    out.append(("png_rgba", rgb_png(synth_image(5022, 300, 200, 4))))
    out.append(("png_rgba_interlaced", rgb_png(synth_image(5023, 300, 200, 4), interlace=True)))
    out.append(("webp_lossy", cuda_lib.encode(".webp", synth_image(5030, 512, 288, 3), {abi.WebpQuality: 85})))
    out.append(("webp_lossy_alph", cuda_lib.encode(".webp", synth_image(5031, 320, 240, 4), {abi.WebpQuality: 80})))
    out.append(("webp_lossless", cuda_lib.encode(".webp", synth_image(5032, 200, 100, 3), {abi.WebpQuality: 101})))
    out.append(("webp_lossless_alpha", cuda_lib.encode(".webp", synth_image(5033, 200, 100, 4), {abi.WebpQuality: 101})))
    return out


@pytest.fixture(scope="module")
def mixed(cuda_lib):
    return mixed_files(cuda_lib)


def png_ihdr(data: bytes):
    assert data[:8] == b"\x89PNG\r\n\x1a\n" and data[12:16] == b"IHDR"
    w, h, depth, ctype, _, _, interlace = struct.unpack(">IIBBBBB", data[16:29])
    return w, h, depth, ctype, interlace


# ---------------------------------------------------------------- the mixed batch at every level

@pytest.mark.parametrize("geom", [FIT, RESIZE], ids=["fit", "resize"])
def test_mixed_batch_every_level(cuda_lib, xb, mixed, geom):
    names = [n for n, _ in mixed]
    files = [d for _, d in mixed]
    for level in LEVELS:
        outs, status = check_against_per_image(cuda_lib, xb, files, png_opt(level, **geom))
        assert status == [0] * len(files), (level, dict(zip(names, status)))
        st = xb.stats()
        assert st["grid_items"] == len(files) and st["fallback_items"] == 0, (level, st)
        assert st["ms_encode"] > 0, st
        for name, out in zip(names, outs):
            _, _, depth, ctype, interlace = png_ihdr(out)
            assert (depth, interlace) == (8, 0) and ctype in (2, 6), (name, level)
            if name.startswith("png_rgba"):
                assert ctype == 6, (name, level)  # RGBA in -> colour type 6 out
            elif name.startswith(("jpeg_", "png_rgb")):
                assert ctype == 2, (name, level)


def test_outputs_decode_outside_the_library(cuda_lib, xb, mixed):
    """cv2 and Pillow read every file (libpng checks the IHDR / IDAT / IEND CRCs and the Adler-32) and agree; PNG and JPEG
    sources decode to the resize of the decoded source; RGBA sources keep their alpha."""
    from PIL import Image
    names = [n for n, _ in mixed]
    files = [d for _, d in mixed]
    for level in (None, 0, 6):
        outs, status = xb.transform(files, png_opt(level, **RESIZE), out_cap=1 << 22)
        assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
        for name, f, out in zip(names, files, outs):
            got = cv2.imdecode(np.frombuffer(out, np.uint8), cv2.IMREAD_UNCHANGED)
            assert got is not None and got.shape[:2] == (170, 300), name
            pil = np.array(Image.open(io.BytesIO(out)))
            assert np.array_equal(pil[:, :, [2, 1, 0, 3]] if pil.shape[2] == 4 else pil[:, :, ::-1], got), name
            assert np.array_equal(cuda_lib.decode(out), got), name
            if name.startswith(("png_", "jpeg_")):
                src = cuda_lib.decode(f)
                assert np.array_equal(got, cuda_lib.resize(src, 300, 170)), (name, level)
            if name.startswith("png_rgba"):
                assert got.shape[2] == 4, name  # (its alpha plane equals the resized source's, compared above)


def test_size_against_libpng(cuda_lib, xb, mixed, ref_lib):
    """DESIGN.md's bound for the PNG encoder: within 1.10 x (+ 256 B) of the reference's file at the same level."""
    files = [d for _, d in mixed]
    for level in (1, 6, 9):
        outs, status = xb.transform(files, png_opt(level, **FIT), out_cap=1 << 22)
        assert status == [0] * len(files)
        for out in outs:
            img = cuda_lib.decode(out)
            if img.shape[0] * img.shape[1] > 4096:
                ref = ref_lib.encode(".png", img, {abi.PngCompression: level})
                assert len(out) <= 1.10 * len(ref) + 256, (level, len(out), len(ref))


# ---------------------------------------------------------------- geometry edges

EDGES = [(1, 1), (1, 300), (300, 1), (257, 64), (85, 128), (341, 64), (10, 1057), (2, 3641)]


@pytest.mark.parametrize("level", [None, 0, 6])
def test_geometry_edges(cuda_lib, xb, level):
    """Rows of one pixel, 257-wide rows, and filtered sizes at chunk boundaries: (85 * 3 + 1) * 128 = 32768 and
    (341 * 3 + 1) * 64 = 65536 exactly, (10 * 3 + 1) * 1057 = 32767, (2 * 4 + 1) * 3641 = 32769 (RGBA)."""
    rgb = [rgb_png(synth_image(5100 + k, 120 + k, 90, 3, noise=5.0)) for k in range(3)]
    rgba = [rgb_png(synth_image(5110 + k, 120 + k, 90, 4, noise=5.0)) for k in range(2)]
    jpeg = [cv2_jpeg(synth_image(5120, 160, 120, 3), 85)]
    files = rgb + rgba + jpeg
    for w, h in EDGES:
        outs, status = check_against_per_image(cuda_lib, xb, files, png_opt(level, Width=w, Height=h, ResizeMethod=abi.ImageOpsResize))
        assert status == [0] * len(files), (w, h, status)
        st = xb.stats()
        assert st["grid_items"] == len(files) and st["fallback_items"] == 0, (w, h, st)
        for out in outs:
            assert png_ihdr(out)[:2] == (w, h)
            got = cv2.imdecode(np.frombuffer(out, np.uint8), cv2.IMREAD_UNCHANGED)
            assert got is not None and got.shape[:2] == (h, w)


def test_output_of_several_hundred_chunks(cuda_lib, xb):
    """2048 x 2048 RGBA: 513 chunks per file, the pack kernel's offsets and checksum folds over more chunks than it has
    threads."""
    files = [rgb_png(synth_image(5200 + k, 96, 64, 4, noise=20.0)) for k in range(2)]
    files.append(rgb_png(synth_image(5202, 96, 64, 3, noise=20.0)))
    opt = png_opt(1, Width=2048, Height=2048, ResizeMethod=abi.ImageOpsResize)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt, cap=20 << 20)
    assert status == [0] * 3
    st = xb.stats()
    assert st["grid_items"] == 3 and st["fallback_items"] == 0, st
    got = cv2.imdecode(np.frombuffer(outs[0], np.uint8), cv2.IMREAD_UNCHANGED)
    assert got.shape == (2048, 2048, 4)
    assert np.array_equal(got, cuda_lib.resize(cuda_lib.decode(files[0]), 2048, 2048))


# ---------------------------------------------------------------- what stays per image

def test_per_image_routing(cuda_lib, xb, golden):
    good = [cv2_jpeg(synth_image(5300 + k, 320 + 32 * k, 240, 3), 80) for k in range(3)]
    good.append(rgb_png(synth_image(5303, 200, 150, 4)))
    good.append(cuda_lib.encode(".webp", synth_image(5304, 200, 150, 3), {abi.WebpQuality: 85}))
    after = cv2_jpeg(synth_image(5320, 352, 240, 3), 80)  # good[1]'s geometry: the truncated file sits inside its group
    per_image_files = {
        "gray_png": golden["png_gray"].tobytes(),
        "gray_jpeg": cv2_jpeg(synth_image(5310, 320, 240, 1), 80),
        "animated_webp": pillow_animation(),
        "gif": golden["gif_party-discord"].tobytes(),
        "rotated_jpeg": with_exif_orientation(good[0], 6),
        "png_cicp": with_cicp(rgb_png(synth_image(5311, 200, 150, 3))),
        "damaged": b"\xff\xd8\xff\xe0 not a jpeg at all",
        "truncated_jpeg": good[1][: len(good[1]) // 2],
        "truncated_png": good[3][: len(good[3]) // 2],
    }
    files = good + list(per_image_files.values()) + [after]
    outs, status = check_against_per_image(cuda_lib, xb, files, png_opt(3, NormalizeOrientation=True, **FIT))
    assert status[: len(good)] == [0] * len(good) and status[-1] == 0
    by_name = dict(zip(per_image_files, status[len(good):]))
    assert by_name["gray_png"] == 0 and by_name["rotated_jpeg"] == 0 and by_name["png_cicp"] == 0, by_name
    assert by_name["damaged"] != 0 and by_name["truncated_jpeg"] != 0, by_name
    st = xb.stats()
    assert st["grid_items"] == len(good) + 1 and st["fallback_items"] == len(per_image_files), st
    # the cICP chunk rides into the output, as Transform re-attaches it
    assert b"cICP" in outs[len(good) + list(per_image_files).index("png_cicp")][:64]
    # NoResize: everything per image
    check_against_per_image(cuda_lib, xb, good, png_opt(3, ResizeMethod=abi.ImageOpsNoResize))
    st = xb.stats()
    assert st["grid_items"] == 0 and st["fallback_items"] == len(good), st


def test_options(cuda_lib, xb):
    """The OpenCV encoder returns its file from the first Encode call, so MaxEncodeFrames, DisableAnimatedOutput and
    the deadline never come into play; a negative MaxEncodeDuration is exceeded before the frame is encoded and no
    still decoder can skip to the end, so lp_transform fails those and they stay with it, as WebP stills (whose frame
    has a duration) do under any MaxEncodeDuration."""
    files = [cv2_jpeg(synth_image(5400 + k, 400, 300, 3), 85) for k in range(3)]
    files.append(rgb_png(synth_image(5410, 400, 300, 3)))
    files.append(rgb_png(synth_image(5411, 400, 300, 4)))
    files.append(cuda_lib.encode(".webp", synth_image(5412, 400, 300, 3), {abi.WebpQuality: 85}))
    files.append(cuda_lib.encode(".webp", synth_image(5413, 400, 300, 4), {abi.WebpQuality: 101}))
    n = len(files)
    for kw, grid in [(dict(DisableAnimatedOutput=True), n),
                     (dict(MaxEncodeFrames=1), n),
                     (dict(MaxEncodeFrames=2), n),
                     (dict(MaxEncodeDuration_ns=1), n - 2),  # (a WebP still's frame has a duration: lp_transform decides)
                     (dict(MaxEncodeDuration_ns=-1), 0),
                     (dict(EncodeTimeout_ns=0), n)]:
        _, status = check_against_per_image(cuda_lib, xb, files, png_opt(3, **kw, **FIT))
        st = xb.stats()
        assert st["grid_items"] == grid and st["fallback_items"] == n - grid, (kw, st)
        if grid == n:
            assert status == [0] * n, (kw, status)
        elif grid == 0:
            assert all(s != 0 for s in status), (kw, status)
    # the extension is matched as NewEncoder matches it
    _, status = check_against_per_image(cuda_lib, xb, files, abi.ImageOptions(FileType=".PNG", EncodeTimeout_ns=T, **FIT))
    assert status == [0] * n and xb.stats()["grid_items"] == n


def test_small_output_buffers(cuda_lib, xb, mixed):
    files = [d for _, d in mixed]
    opt = png_opt(3, **FIT)
    sizes = sorted(len(per_image(cuda_lib, f, opt)[0]) for f in files)
    for cap in (10, sizes[0] - 1, sizes[len(sizes) // 2], sizes[-1]):
        _, status = check_against_per_image(cuda_lib, xb, files, opt, cap=cap)
        refused = [s for s in status if s != 0]
        assert len(refused) == sum(1 for s in sizes if s > cap), (cap, status)
        assert all(s == abi.LP_ERR_BUF_TOO_SMALL for s in refused), (cap, status)
        st = xb.stats()  # a file that does not fit is handed to lp_transform, which reports it
        assert st["fallback_items"] == len(refused) and st["grid_items"] == len(files) - len(refused), (cap, st)


def test_multi_gpu_dispatcher(cuda_lib, xb, mixed):
    files = [d for _, d in mixed]
    opt = png_opt(6, NormalizeOrientation=True, **FIT)
    outs, status = xb.transform(files, opt, out_cap=1 << 22)
    assert status == [0] * len(files)
    m = abi.MultiBatch(cuda_lib, [0, 0], arena_bytes=4 << 30)
    try:
        m_outs, m_status = m.transform(files, opt, out_cap=1 << 22)
        assert m_status == status and m_outs == outs
        assert sum(m.stats(g)["grid_items"] for g in range(2)) == len(files)
        assert sum(m.stats(g)["fallback_items"] for g in range(2)) == 0
    finally:
        m.close()
