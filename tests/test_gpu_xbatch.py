"""GPU: the heterogeneous batch entry point (lp_xbatch_*, csrc/xbatch.cu) against per-image Transform.

The contract of lp_xbatch_transform is "status and bytes of every item are what lp_transform returns for it", so
every test compares the batch with lp_transform of the SAME library item by item (which the other GPU suites pin on
the oracle / the live reference), and the measured BASELINE shapes additionally against the reference itself:
  config 5 in miniature  mixed JPEG / PNG / WebP (+ things the grid path must hand to the per-image path) -> JPEG
  config 3               PNG RGBA -> Fit -> lossy WebP + alpha, incl. ONE full-size 3840x2160 -> 512x512 image
  config 4               animated GIF -> Fit -> animated WebP, incl. a 1280x720 animation -> 256x256
"""
import io

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.png_writer import write_png
from tests.webp_util import frames_of, libwebp_decode, optional_reference, pillow_animation, psnr, riff

pytestmark = pytest.mark.gpu
T = 10**12


def per_image(lib, data, opt, cap=1 << 22):
    try:
        return lib.transform(data, opt, dst_cap=cap), 0
    except abi.LilliputError as e:
        return b"", e.code


def check_against_per_image(lib, xb, files, opt, cap=1 << 22):
    outs, status = xb.transform(files, opt, out_cap=cap)
    for i, f in enumerate(files):
        want, code = per_image(lib, f, opt, cap)
        assert status[i] == code, f"item {i}: batch status {status[i]}, lp_transform {code}"
        assert outs[i] == want, f"item {i}: batch bytes differ from lp_transform ({len(outs[i])} vs {len(want)} B)"
    return outs, status


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=12 << 30)
    yield x
    x.close()


def rgb_png(img, **kw):
    ch = img.shape[2]
    return write_png(img[:, :, [2, 1, 0, 3]] if ch == 4 else img[:, :, ::-1], 6 if ch == 4 else 2, 8, **kw)


def test_mixed_batch_to_jpeg(cuda_lib, xb, oracle, golden):
    """BASELINE config 5 in miniature: formats x sizes in one call, outputs byte-identical to lp_transform."""
    files = []
    for k, (w, h) in enumerate([(320, 180), (427, 240), (320, 180), (640, 360)]):
        files.append(oracle.jpeg_encode(synth_image(100 + k, w, h, 3), 90))                  # JPEG groups (2 sizes share one)
    files.append(rgb_png(synth_image(200, 300, 200, 3)))                                     # PNG RGB, two IDAT chunks
    files.append(rgb_png(synth_image(201, 300, 200, 4), ftypes=(4,)))                        # PNG RGBA, Paeth
    files.append(rgb_png(synth_image(202, 300, 200, 3), interlace=True))                     # Adam7
    files.append(cuda_lib.encode(".webp", synth_image(300, 256, 144, 3), {abi.WebpQuality: 85}))  # lossy WebP
    files.append(cuda_lib.encode(".webp", synth_image(301, 256, 144, 3), {abi.WebpQuality: 70}))
    files.append(cuda_lib.encode(".webp", synth_image(302, 200, 100, 3), {abi.WebpQuality: 101}))  # lossless: per image
    files.append(golden["gif_party-discord"].tobytes())                                      # GIF -> JPEG: per image
    files.append(b"\xff\xd8\xff\xe0 not a jpeg at all")                                      # error item
    files.append(files[0][: len(files[0]) // 2])                                             # truncated JPEG
    files.append(golden["png_gray"].tobytes())                                               # gray PNG: per image
    opt = abi.ImageOptions(FileType=".jpeg", Width=96, Height=96, ResizeMethod=abi.ImageOpsFit,
                           NormalizeOrientation=True, EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt)
    st = xb.stats()
    assert st["grid_items"] >= 9 and st["launches"] > 0
    assert status[:9] == [0] * 9
    # and the grid-decoded items against the oracle / reference pixels, not only against ourselves
    dec, _ = oracle.jpeg_decode(files[0])
    assert outs[0] == oracle.jpeg_encode(oracle.fit(dec, 96, 96), 85)
    src = oracle.png_decode(files[4])
    src = src[0] if isinstance(src, tuple) else src
    assert outs[4] == oracle.jpeg_encode(oracle.fit(src, 96, 96), 85)


def test_mixed_batch_resize_method_and_quality(cuda_lib, xb, oracle):
    files = [oracle.jpeg_encode(synth_image(400 + k, 200 + 40 * k, 150, 3), 85) for k in range(3)]
    files.append(rgb_png(synth_image(410, 222, 133, 4)))
    opt = abi.ImageOptions(FileType=".jpeg", Width=80, Height=50, ResizeMethod=abi.ImageOpsResize,
                           EncodeOptions={abi.JpegQuality: 60}, EncodeTimeout_ns=T)
    check_against_per_image(cuda_lib, xb, files, opt)
    # a request larger than the source: calculateExpectedSize rules (ops.go:243-255)
    opt = abi.ImageOptions(FileType=".jpeg", Width=4000, Height=4000, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 75}, EncodeTimeout_ns=T)
    check_against_per_image(cuda_lib, xb, files, opt)


def test_png_to_webp_config3_miniature(cuda_lib, xb, oracle):
    files = [rgb_png(synth_image(500 + k, 384, 216, 4, noise=8.0)) for k in range(5)]
    files.append(rgb_png(synth_image(510, 384, 216, 3)))            # opaque RGB: no ALPH, simple file
    opaque = synth_image(511, 384, 216, 4)
    opaque[:, :, 3] = 255
    files.append(rgb_png(opaque))                                   # RGBA but fully opaque: libwebp drops the alpha plane
    opt = abi.ImageOptions(FileType=".webp", Width=128, Height=128, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.WebpQuality: 85}, EncodeTimeout_ns=T)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt)
    assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
    # against libwebp (and the reference's shims where built): it decodes our stream; alpha exact, colour close to the
    # fitted source
    ref_lib = optional_reference()
    for k in (0, 5, 6):
        src = oracle.png_decode(files[k])
        src = src[0] if isinstance(src, tuple) else src
        fit = oracle.fit(src, 128, 128)
        got = libwebp_decode(outs[k])
        _, mine, _, rc = cuda_lib.webp_frames(outs[k])
        assert rc == 0 and np.array_equal(mine[0], got)
        if ref_lib:
            info, frames, _, rc = ref_lib.webp_frames(outs[k])
            assert rc == 0 and np.array_equal(frames[0], got)
        if k == 0:
            assert got.shape[2] == 4 and np.array_equal(got[:, :, 3], fit[:, :, 3])
        else:
            assert got.shape[2] == 3
        assert psnr(got[:, :, :3], fit[:, :, :3]) > 28.0


def test_png_to_webp_config3_full_size(cuda_lib, xb, oracle):
    """One BASELINE config 3 image at full size: 3840x2160 RGBA PNG (zlib level 6, Paeth) -> Fit 512x512 -> WebP
    q85 + alpha, through the batch call; == lp_transform, and the reference's decoder reads it back."""
    import struct
    import zlib
    img = synth_image(2000, 3840, 2160, 4)
    rgb = np.ascontiguousarray(img[:, :, [2, 1, 0, 3]]).astype(np.int16)
    f = rgb.copy()
    f[:, 1:] -= rgb[:, :-1]                                         # Sub filter (vectorised; Paeth is covered in miniature)
    rows = np.concatenate([np.full((2160, 1), 1, np.uint8), (f & 255).astype(np.uint8).reshape(2160, -1)], axis=1).tobytes()

    def ch(t, d):
        return struct.pack(">I", len(d)) + t + d + struct.pack(">I", zlib.crc32(t + d) & 0xffffffff)
    z = zlib.compress(rows, 6)
    png = b"\x89PNG\r\n\x1a\n" + ch(b"IHDR", struct.pack(">IIBBBBB", 3840, 2160, 8, 6, 0, 0, 0))
    for o in range(0, len(z), 1 << 20):                             # 1 MiB IDAT chunks: the device gathers them
        png += ch(b"IDAT", z[o:o + (1 << 20)])
    png += ch(b"IEND", b"")
    opt = abi.ImageOptions(FileType=".webp", Width=512, Height=512, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.WebpQuality: 85}, EncodeTimeout_ns=T)
    outs, status = check_against_per_image(cuda_lib, xb, [png, png], opt)
    assert status == [0, 0] and xb.stats()["grid_items"] == 2
    fit = oracle.fit(img, 512, 512)
    got = libwebp_decode(outs[0])
    assert np.array_equal(got[:, :, 3], fit[:, :, 3])
    assert psnr(got[:, :, :3], fit[:, :, :3]) > 30.0
    ref_lib = optional_reference()
    if ref_lib:
        info, frames, _, rc = ref_lib.webp_frames(outs[0])
        assert rc == 0 and np.array_equal(frames[0], got)


def _gif(frames, duration=40, loop=0, **kw):
    from PIL import Image
    ims = [Image.fromarray(f[:, :, ::-1].copy()).quantize(kw.pop("colors", 64)) if f.ndim == 3 else f for f in frames]
    bio = io.BytesIO()
    ims[0].save(bio, "GIF", save_all=True, append_images=ims[1:], duration=duration, loop=loop, **kw)
    return bio.getvalue()


def test_gif_to_animated_webp_config4(cuda_lib, xb, golden):
    pytest.importorskip("PIL")
    files = [golden[k].tobytes() for k in golden.files if k.startswith("gif_") and golden[k].ndim == 1][:6]
    base = synth_image(700, 1280, 720, 3, noise=0.0)
    big = [np.roll(base, 8 * k, axis=1) for k in range(6)]         # BASELINE config 4 canvas, a few frames
    files.append(_gif(big, duration=40))
    files.append(_gif([synth_image(710 + k, 200, 120, 3, noise=0.0) for k in range(3)], duration=[20, 70, 130], loop=3))
    opt = abi.ImageOptions(FileType=".webp", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.WebpQuality: 85}, EncodeTimeout_ns=T)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt, cap=1 << 24)
    assert xb.stats()["grid_items"] >= 2
    # libwebp reads the animation back: frame count, delays, loop count; every frame, rewrapped as a still, decodes to
    # the device's frame
    k = len(files) - 1
    assert pillow_animation(outs[k])[:3] == (3, 3, [20, 70, 130])
    assert pillow_animation(outs[k - 1])[0] == 6 and pillow_animation(outs[k - 1])[3] == (256, 256)
    for out in outs:
        _, mine, _, rc = cuda_lib.webp_frames(out)
        assert rc == 0 and len(mine) == len(frames_of(out))
        for f, (tag, payload, alph) in zip(mine, frames_of(out)):
            chunks = [(b"VP8 ", payload)] if alph is None else [
                (b"VP8X", bytes([0x10, 0, 0, 0]) + (f.shape[1] - 1).to_bytes(3, "little") + (f.shape[0] - 1).to_bytes(3, "little")),
                (b"ALPH", alph), (tag, payload)]
            got = libwebp_decode(riff(chunks))
            assert np.array_equal(f[:, :, :got.shape[2]], got)
            assert got.shape[2] == 4 or f.shape[2] == 3 or (f[:, :, 3] == 255).all()
    ref_lib = optional_reference()
    if ref_lib:
        info, frames, metas, rc = ref_lib.webp_frames(outs[k])
        assert rc == 0 and info["num_frames"] == 3 and info["loop_count"] == 3
        assert [m["delay"] for m in metas] == [20, 70, 130]
        info, frames, metas, rc = ref_lib.webp_frames(outs[k - 1])
        assert rc == 0 and info["num_frames"] == 6 and frames[0].shape[:2] == (256, 256)


def test_xbatch_empty_and_small_buffers(cuda_lib, xb, oracle):
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    outs, status = xb.transform([], opt)
    assert outs == [] and status == []
    files = [oracle.jpeg_encode(synth_image(800 + k, 256, 256, 3), 90) for k in range(3)]
    check_against_per_image(cuda_lib, xb, files, opt, cap=700)       # too small for the output: same error per item


def test_multi_gpu_dispatcher_matches_per_image(cuda_lib, oracle):
    """lp_multi_*: the library-level sharding by image index.  Runs on however many GPUs the box has (1 is enough to
    exercise the dispatcher; the same device twice exercises two contexts side by side)."""
    import torch
    ndev = max(1, torch.cuda.device_count())
    devices = list(range(ndev)) if ndev > 1 else [0, 0]
    m = abi.MultiBatch(cuda_lib, devices, arena_bytes=6 << 30)
    try:
        files = [oracle.jpeg_encode(synth_image(950 + k, 320, 200, 3), 90) for k in range(9)]
        files += [rgb_png(synth_image(960 + k, 160 + 16 * k, 120, 4)) for k in range(4)]
        opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                               EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
        outs, status = m.transform(files, opt)
        assert status == [0] * len(files)
        for f, o in zip(files, outs):
            assert o == cuda_lib.transform(f, opt)
        assert sum(m.stats(g)["grid_items"] + m.stats(g)["fallback_items"] for g in range(len(devices))) == len(files)
    finally:
        m.close()


def test_many_distinct_huffman_table_sets(cuda_lib, xb):
    """Per-image OPTIMISED Huffman tables (every file its own DHT): more distinct table sets than the 64 the batch
    context used to hold, three sizes, one call -- all taken by the grid path, bytes == lp_transform."""
    cv2 = pytest.importorskip("cv2")
    files = []
    for k in range(75):
        w, h = [(320, 240), (400, 300), (512, 288)][k % 3]
        ok, b = cv2.imencode(".jpg", synth_image(1200 + k, w, h, 3, noise=4.0 + (k % 7)), [cv2.IMWRITE_JPEG_QUALITY, 70 + (k % 25),
                                                                                           cv2.IMWRITE_JPEG_OPTIMIZE, 1])
        assert ok
        files.append(bytes(b))
    opt = abi.ImageOptions(FileType=".jpeg", Width=100, Height=100, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 80}, EncodeTimeout_ns=T)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt)
    assert status == [0] * len(files)
    st = xb.stats()
    assert st["grid_items"] == len(files) and st["fallback_items"] == 0


def _with_exif_orientation(jpeg: bytes, orientation: int) -> bytes:
    """APP1 / EXIF with one IFD entry (0x0112 orientation) right behind SOI."""
    tiff = b"II*\x00\x08\x00\x00\x00" + b"\x01\x00" + b"\x12\x01\x03\x00\x01\x00\x00\x00" + bytes([orientation, 0, 0, 0]) + b"\x00\x00\x00\x00"
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + jpeg[2:]


def test_jpeg_share_of_config5_every_kind_in_one_call(cuda_lib, xb):
    """The JPEG share of BASELINE config 5 as real corpora have it: five sizes, per-image optimised Huffman tables, 4:2:0 /
    4:2:2 / 4:4:4 / gray, restart intervals, progressive files and EXIF-rotated ones in ONE call.  Every item comes back
    LP_OK with the bytes lp_transform gives it, whichever path (grid or per-image hand-over) the batch chose for it."""
    cv2 = pytest.importorskip("cv2")
    sizes = [(854, 480), (1280, 720), (640, 360), (1024, 768), (500, 333)]
    samp = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
    files = []
    for k in range(60):
        w, h = sizes[k % 5]
        flags = [cv2.IMWRITE_JPEG_QUALITY, 60 + (k * 7) % 38, cv2.IMWRITE_JPEG_OPTIMIZE, 1,
                 cv2.IMWRITE_JPEG_SAMPLING_FACTOR, samp[(k // 5) % 3]]
        if k % 11 == 3:
            flags += [cv2.IMWRITE_JPEG_RST_INTERVAL, 7]
        if k % 13 == 5:
            flags += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
        img = synth_image(1500 + k, w, h, 1 if k % 17 == 9 else 3, noise=3.0 + (k % 5))
        ok, b = cv2.imencode(".jpg", img, flags)
        assert ok
        b = bytes(b)
        if k % 7 == 2:
            b = _with_exif_orientation(b, 2 + (k // 7) % 7)
        files.append(b)
    opt = abi.ImageOptions(FileType=".jpeg", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit, NormalizeOrientation=True,
                           EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt)
    assert status == [0] * len(files)
    st = xb.stats()
    assert st["grid_items"] + st["fallback_items"] == len(files)
    assert st["grid_items"] >= 40  # the baseline colour files; progressive / rotated / gray ones may be handed over
