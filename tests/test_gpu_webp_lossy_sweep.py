"""GPU: lossy WebP output across every quality, frame geometry and content class, checked against libwebp.

For every case the device's VP8 payload (webp_encoder_write -> webp_encode_lossy_batch) is byte-identical to the
host build of the same core (vp8_enc_core.h through oracle_webp.cpp, sized like the device), and three decoders agree
on its pixels: libwebp (OpenCV's WebP codec, an independent implementation), the device's decoder and the decoder
core on the host.  BGRA frames keep their alpha exactly; an all-opaque frame carries no ALPH chunk.  The large and
detailed frames are those whose first partition (frame header + per-macroblock modes) used to outgrow its scratch, and
one whose first partition exceeds the format's 2^19-byte limit with 4x4 prediction (coded with 16x16 prediction only).
The batch paths must give every such item status 0 and the bytes lp_transform gives it."""
import io

import cv2  # noqa: F401  libwebp_decode's libwebp: a missing decoder fails these tests, it does not skip them
import numpy as np
import pytest
from PIL import Image

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.png_writer import write_png
from tests.webp_util import (chunks_of, frames_of, libwebp_decode, pillow_animation, riff, vp8_cpu_decode, vp8_cpu_encode,
                             vp8_cpu_lib, vp8_partition_sizes)

pytestmark = pytest.mark.gpu
T = 10**12


@pytest.fixture(scope="module")
def cpu():
    return vp8_cpu_lib()


def uniform_noise(seed, w, h, ch=3):
    return np.random.default_rng(seed).integers(0, 256, (h, w, ch), dtype=np.uint8)


def alternating_rows(seed, w, h, ch=3):
    img = uniform_noise(seed, w, h, ch)
    for r in range(0, h, 32):
        img[r:r + 16, :, :3] = 128
    return img


def with_random_alpha(img, seed):
    out = np.concatenate([img[:, :, :3], np.zeros(img.shape[:2] + (1,), np.uint8)], axis=2)
    out[:, :, 3] = np.random.default_rng(seed).integers(0, 256, img.shape[:2], dtype=np.uint8)
    return out


def device_decode(cuda_lib, data, w, h):
    """The device decoder's pixels for a WebP file.  The stage helper behind webp_frames sizes its framebuffer like an
    ImageOps of 8192 and refuses larger frames (ErrBufTooSmall); those go through Transform with framebuffers of the
    frame's size, unresized and written losslessly, so libwebp reads back exactly what the device decoded."""
    if max(w, h) <= 8192:
        _, frames, _, rc = cuda_lib.webp_frames(data)
        assert rc == 0, rc
        return frames[0]
    _, frames, _, rc = cuda_lib.webp_frames(data)
    assert rc == abi.LP_ERR_BUF_TOO_SMALL and frames == []
    opt = abi.ImageOptions(FileType=".webp", Width=0, Height=0, ResizeMethod=abi.ImageOpsNoResize,
                           EncodeOptions={abi.WebpQuality: 101}, EncodeTimeout_ns=T)
    out = cuda_lib.transform(data, opt, dst_cap=w * h * 8 + (1 << 20), max_size=max(w, h))
    assert [t for t, _ in chunks_of(out)] == [b"VP8L"]
    return libwebp_decode(out)


def check_lossy(cuda_lib, cpu, img, quality):
    """One still through the device; returns the VP8 payload."""
    h, w, ch = img.shape
    data = cuda_lib.encode(".webp", img, {abi.WebpQuality: quality}, dst_cap=img.size * 4 + (1 << 20))
    transparent = ch == 4 and bool((img[:, :, 3] != 255).any())
    assert [t for t, _ in chunks_of(data)] == ([b"VP8X", b"ALPH", b"VP8 "] if transparent else [b"VP8 "]), (w, h, quality)
    payload = dict(chunks_of(data))[b"VP8 "]
    # (the encoder option reads quality 0 as 1, as the reference's webp.cpp does)
    assert bytes(payload) == vp8_cpu_encode(cpu, img, max(quality, 1)), ("device and host core differ", w, h, quality)
    assert vp8_partition_sizes(payload)[0] < 1 << 19
    theirs = libwebp_decode(data)
    assert theirs.shape == (h, w, 4 if transparent else 3)
    assert np.array_equal(theirs[:, :, :3], vp8_cpu_decode(cpu, payload)), (w, h, quality)
    if transparent:
        assert np.array_equal(theirs[:, :, 3], img[:, :, 3]), (w, h, quality)
    assert np.array_equal(device_decode(cuda_lib, data, w, h), theirs), (w, h, quality)
    return payload


@pytest.mark.parametrize("quality", range(0, 101))
def test_every_quality(cuda_lib, cpu, quality):
    check_lossy(cuda_lib, cpu, synth_image(900, 97, 61, 3, noise=30.0), quality)
    check_lossy(cuda_lib, cpu, with_random_alpha(synth_image(901, 256, 144, 3, noise=8.0), 902), quality)


def test_quality_101_is_lossless(cuda_lib):
    for img in (synth_image(900, 97, 61, 3, noise=30.0), with_random_alpha(synth_image(901, 256, 144, 3), 902)):
        data = cuda_lib.encode(".webp", img, {abi.WebpQuality: 101})
        assert [t for t, _ in chunks_of(data)] == [b"VP8L"]
        assert np.array_equal(libwebp_decode(data), img)


GEOMETRY = [(1, 1), (1, 2), (2, 1), (1, 300), (300, 1), (15, 15), (16, 16), (17, 17), (31, 33), (16383, 16), (16383, 17),
            (16, 4096)]


@pytest.mark.parametrize("w,h", GEOMETRY, ids=[f"{w}x{h}" for w, h in GEOMETRY])
def test_geometry(cuda_lib, cpu, w, h):
    img = synth_image(w * 7 + h, w, h, 3, noise=12.0)
    for quality in (0, 50, 85, 100):
        check_lossy(cuda_lib, cpu, img, quality)
    opaque = np.concatenate([img, np.full((h, w, 1), 255, np.uint8)], axis=2)
    check_lossy(cuda_lib, cpu, opaque, 85)            # BGRA, all opaque: no ALPH
    check_lossy(cuda_lib, cpu, with_random_alpha(img, w + h), 85)


def _checkerboard(w, h):
    return np.kron((np.indices((h, w)).sum(0) & 1)[:, :, None] * 255, np.ones(3)).astype(np.uint8)


def _hard_edges(w, h):
    img = np.zeros((h, w, 3), np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(77)
    for _ in range(12):
        a, b = rng.normal(size=2)
        img[(a * (xx - w / 2) + b * (yy - h / 2)) > rng.normal() * 20] = rng.integers(0, 256, 3)
    return img


CONTENT = {
    "smooth": lambda: synth_image(910, 256, 256, 3, noise=0.0),
    "sensor_noise": lambda: synth_image(911, 256, 256, 3, noise=12.0),
    "uniform_noise": lambda: uniform_noise(912, 256, 256),
    "checkerboard": lambda: _checkerboard(256, 256),
    "flat": lambda: np.full((256, 256, 3), (40, 180, 90), np.uint8),
    "hard_edges": lambda: _hard_edges(256, 256),
    "alternating_rows": lambda: alternating_rows(913, 256, 256),
}


@pytest.mark.parametrize("name", list(CONTENT))
def test_content_classes(cuda_lib, cpu, name):
    img = CONTENT[name]()
    for quality in (0, 50, 85, 100):
        check_lossy(cuda_lib, cpu, img, quality)


LARGE = [
    ("synth1280x720-q90", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 90),
    ("synth1280x720-q95", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 95),
    ("synth1280x720-q100", lambda: synth_image(7, 1280, 720, 3, noise=6.0), 100),
    ("synth1920x1080-q100", lambda: synth_image(8, 1920, 1080, 3, noise=6.0), 100),
    ("synth3840x2160-q85", lambda: synth_image(9, 3840, 2160, 3, noise=6.0), 85),
    ("synth3840x2160-q100", lambda: synth_image(9, 3840, 2160, 3, noise=6.0), 100),
    ("synth3840x2160-bgra-q85", lambda: with_random_alpha(synth_image(10, 3840, 2160, 3, noise=6.0), 11), 85),
    ("synth3840x2160-bgra-q100", lambda: with_random_alpha(synth_image(10, 3840, 2160, 3, noise=6.0), 11), 100),
    ("alt_rows1024x512-q50", lambda: alternating_rows(3, 1024, 512), 50),
]


@pytest.mark.parametrize("name,make,quality", LARGE, ids=[c[0] for c in LARGE])
def test_large_detailed_frames(cuda_lib, cpu, name, make, quality):
    payload = check_lossy(cuda_lib, cpu, make(), quality)
    # 4x4 prediction kept: these are far below the format's limit, no 16x16-only retry is due
    assert payload == vp8_cpu_encode(cpu, make(), quality, try_i4=1)


def test_first_partition_beyond_the_format_limit_is_retried_with_16x16_prediction(cuda_lib, cpu):
    img = uniform_noise(8, 4096, 4096)
    payload = check_lossy(cuda_lib, cpu, img, 75)
    assert payload == vp8_cpu_encode(cpu, img, 75, try_i4=0)


# ---- the batch paths ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=12 << 30)
    yield x
    x.close()


def _all_ok_and_per_image(cuda_lib, xb, files, opt, cap):
    outs, status = xb.transform(files, opt, out_cap=cap)
    assert status == [0] * len(files), status
    for i, f in enumerate(files):
        assert outs[i] == cuda_lib.transform(f, opt, dst_cap=cap), f"item {i}: batch bytes differ from lp_transform"
    return outs


def _png(img):
    ch = img.shape[2]
    return write_png(img[:, :, [2, 1, 0, 3]] if ch == 4 else img[:, :, ::-1], 6 if ch == 4 else 2, 8)


def test_xbatch_png_to_webp_detailed_frames(cuda_lib, xb):
    """PNG -> Fit 1280x720 -> WebP q100 in one heterogeneous call: sources at the output size (detail passes through
    untouched), larger, and smaller ones (which keep their own size), RGB and RGBA."""
    files = [_png(synth_image(920, 1280, 720, 3, noise=6.0)),
             _png(alternating_rows(921, 1280, 720)),
             _png(with_random_alpha(synth_image(922, 1280, 720, 3, noise=6.0), 923)),
             _png(synth_image(924, 1920, 1080, 3, noise=12.0)),
             _png(synth_image(925, 640, 360, 3, noise=12.0)),
             _png(with_random_alpha(uniform_noise(926, 500, 300), 927))]
    opt = abi.ImageOptions(FileType=".webp", Width=1280, Height=720, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.WebpQuality: 100}, EncodeTimeout_ns=T)
    outs = _all_ok_and_per_image(cuda_lib, xb, files, opt, 1 << 24)
    assert len({libwebp_decode(o).shape[:2] for o in outs}) >= 2  # mixed geometry
    for o in outs:
        theirs = libwebp_decode(o)
        _, mine, _, rc = cuda_lib.webp_frames(o)
        assert rc == 0 and np.array_equal(mine[0], theirs)


def _gif(frames, durations, loop):
    ims = [Image.fromarray(f[:, :, ::-1].copy()).quantize(64) for f in frames]
    bio = io.BytesIO()
    ims[0].save(bio, "GIF", save_all=True, append_images=ims[1:], duration=durations, loop=loop)
    return bio.getvalue()


def test_xbatch_gif_to_animated_webp_detailed_canvas(cuda_lib, xb):
    """GIF -> animated WebP q95 with a 1280x720 canvas of detailed frames: every frame is a valid lossy still that
    libwebp decodes to the device's frame; frame count, delays and loop count read back with Pillow's WebP reader."""
    base = synth_image(930, 1280, 720, 3, noise=12.0)
    durations = [40, 70, 130]
    files = [_gif([np.roll(base, 24 * k, axis=1) for k in range(3)], durations, 2),
             _gif([synth_image(931 + k, 320, 200, 3, noise=12.0) for k in range(2)], [50, 60], 0)]
    opt = abi.ImageOptions(FileType=".webp", Width=0, Height=0, ResizeMethod=abi.ImageOpsNoResize,
                           EncodeOptions={abi.WebpQuality: 95}, EncodeTimeout_ns=T)
    outs = _all_ok_and_per_image(cuda_lib, xb, files, opt, 1 << 25)
    for out, n, want_delays, loop, size in [(outs[0], 3, durations, 2, (1280, 720)), (outs[1], 2, [50, 60], 0, (320, 200))]:
        _, mine, _, rc = cuda_lib.webp_frames(out)
        assert rc == 0 and len(mine) == n
        parts = frames_of(out)
        assert len(parts) == n
        for k, (tag, payload, alph) in enumerate(parts):
            assert tag == b"VP8 " and alph is None  # GIF frames without transparency: opaque canvas, no ALPH
            theirs = libwebp_decode(riff([(b"VP8 ", payload)]))
            assert theirs.shape == (size[1], size[0], 3)
            assert np.array_equal(mine[k][:, :, :3], theirs), k
            assert mine[k].shape[2] == 3 or (mine[k][:, :, 3] == 255).all()
        assert pillow_animation(out) == (n, loop, want_delays, size)
