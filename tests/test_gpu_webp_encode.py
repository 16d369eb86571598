"""GPU: WebP encode through the webp_encoder_* ABI (webp.go's Encode -> write / flush).
  lossless (quality > 100): decoded pixels == input pixels, with the device decoder and with libwebp (OpenCV's
                            WebP codec; the reference's own shims too where oracle/_ref is built);
  lossy:  valid VP8 -- device decoder and libwebp agree bit for bit on the stream -- and
          PSNR within 1 dB of libwebp's at the same quality; BGRA adds an exact ALPH plane;
  container: VP8X / ICCP / ANIM / ANMF as libwebp and Pillow's WebP reader read them back;
  whole Transform calls: PNG -> WebP, GIF -> animated WebP."""
import cv2
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.webp_util import chunks_of, frames_of, libwebp_decode, optional_reference, pillow_animation, psnr, riff

pytestmark = pytest.mark.gpu
LOSSLESS = {abi.WebpQuality: 101}


@pytest.mark.parametrize("seed,w,h,ch,noise", [(5, 200, 120, 3, 6.0), (6, 97, 61, 4, 40.0), (7, 1, 1, 3, 6.0),
                                               (8, 513, 3, 4, 6.0), (9, 2, 300, 3, 20.0), (10, 1920, 1080, 3, 6.0)])
def test_lossless_webp_round_trip(cuda_lib, seed, w, h, ch, noise):
    img = synth_image(seed, w, h, ch, noise=noise)
    data = cuda_lib.encode(".webp", img, LOSSLESS)
    assert [t for t, _ in chunks_of(data)] == [b"VP8L"]  # simple file format: no VP8X needed
    _, frames, _, rc = cuda_lib.webp_frames(data)
    assert rc == 0 and np.array_equal(frames[0], img)


def test_lossless_webp_decodes_with_the_reference(cuda_lib):
    ref_lib = optional_reference()
    for seed, w, h, ch in [(11, 333, 211, 3), (12, 120, 90, 4)]:
        img = synth_image(seed, w, h, ch, noise=15.0)
        data = cuda_lib.encode(".webp", img, LOSSLESS)
        assert np.array_equal(libwebp_decode(data), img)
        if ref_lib:
            _, frames, _, rc = ref_lib.webp_frames(data)
            assert rc == 0 and np.array_equal(frames[0], img)


@pytest.mark.parametrize("quality", [30, 75, 90])
def test_lossy_webp_is_valid_and_of_libwebp_quality(cuda_lib, quality):
    ref_lib = optional_reference()
    for seed, w, h, noise in [(31, 512, 512, 6.0), (32, 97, 61, 30.0), (33, 33, 65, 12.0)]:
        img = synth_image(seed, w, h, 3, noise=noise)
        data = cuda_lib.encode(".webp", img, {abi.WebpQuality: quality})
        assert [t for t, _ in chunks_of(data)] == [b"VP8 "]
        _, mine, _, rc1 = cuda_lib.webp_frames(data)
        theirs = libwebp_decode(data)
        assert rc1 == 0 and np.array_equal(mine[0], theirs)
        if ref_lib:
            _, ref, _, rc2 = ref_lib.webp_frames(data)
            assert rc2 == 0 and np.array_equal(mine[0], ref[0])
        ok, lw = cv2.imencode(".webp", img, [cv2.IMWRITE_WEBP_QUALITY, quality])
        assert psnr(theirs, img) > psnr(cv2.imdecode(lw, cv2.IMREAD_COLOR), img) - 1.0


def test_lossy_webp_with_alpha_keeps_alpha_exact(cuda_lib):
    img = synth_image(41, 160, 120, 4, noise=10.0)
    data = cuda_lib.encode(".webp", img, {abi.WebpQuality: 80})
    assert [t for t, _ in chunks_of(data)] == [b"VP8X", b"ALPH", b"VP8 "]
    theirs = libwebp_decode(data)
    assert theirs.shape == img.shape
    assert np.array_equal(theirs[:, :, 3], img[:, :, 3])
    assert psnr(theirs[:, :, :3], img[:, :, :3]) > 25.0  # noisy content at q80
    _, mine, _, _ = cuda_lib.webp_frames(data)
    assert np.array_equal(mine[0], theirs)
    ref_lib = optional_reference()
    if ref_lib:
        info, frames, _, rc = ref_lib.webp_frames(data)
        assert rc == 0 and info["pixel_type"] == abi.CV_8UC4 and np.array_equal(mine[0], frames[0])


def test_png_to_webp_transform(cuda_lib, golden, oracle):
    """BASELINE config 3 in miniature: PNG RGBA -> Fit -> WebP lossy + alpha through lp_transform."""
    data = golden["png_rgba"].tobytes()
    src = oracle.png_decode(data)
    src = src[0] if isinstance(src, tuple) else src
    out = cuda_lib.transform(data, abi.ImageOptions(FileType=".webp", Width=32, Height=32, ResizeMethod=abi.ImageOpsFit,
                                                    EncodeOptions={abi.WebpQuality: 101}, EncodeTimeout_ns=10**12))
    assert np.array_equal(libwebp_decode(out), oracle.fit(src, 32, 32))  # lossless: the fitted pixels, exactly
    ref_lib = optional_reference()
    if ref_lib:
        _, frames, _, rc = ref_lib.webp_frames(out)
        assert rc == 0 and np.array_equal(frames[0], oracle.fit(src, 32, 32))


def test_gif_to_animated_webp_transform(cuda_lib, golden):
    """BASELINE config 4 in miniature: animated GIF -> Fit -> animated WebP; frame count, durations,
    loop count and background survive, and the (lossless) frames are the composited GIF frames."""
    data = golden["gif_party-discord"].tobytes()
    out = cuda_lib.transform(data, abi.ImageOptions(FileType=".webp", Width=0, Height=0, ResizeMethod=abi.ImageOpsNoResize,
                                                    EncodeOptions={abi.WebpQuality: 101}, EncodeTimeout_ns=10**12))
    gif_frames, delays, _, _ = cuda_lib.gif_frames(data)
    # every ANMF frame is a full canvas (no blending): rewrapped as a still, libwebp decodes it to the GIF frame
    parts = frames_of(out)
    assert len(parts) == len(gif_frames) == 16
    for (tag, payload, _), want in zip(parts, gif_frames):
        got = libwebp_decode(riff([(tag, payload)]))
        if got.shape[2] == 3:  # a frame without transparency: libwebp returns BGR
            got = np.concatenate([got, np.full(got.shape[:2] + (1,), 255, np.uint8)], axis=2)
        assert np.array_equal(got, want)
    assert pillow_animation(out)[:3] == (16, 0, list(delays))
    ref_lib = optional_reference()
    if ref_lib:
        info, frames, metas, rc = ref_lib.webp_frames(out)
        assert rc == 0 and info["num_frames"] == len(gif_frames) == 16
        assert info["loop_count"] == 0 and info["total_duration"] == sum(delays)
        assert [m["delay"] for m in metas] == delays
        for a, b in zip(frames, gif_frames):
            assert np.array_equal(a, b)


def test_webp_encoder_reports_a_full_destination(cuda_lib):
    img = synth_image(51, 200, 200, 3)
    with pytest.raises(abi.LilliputError):
        cuda_lib.encode(".webp", img, {abi.WebpQuality: 90}, dst_cap=500)


def test_device_lossy_stream_is_byte_identical_to_the_serial_core(cuda_lib):
    """The device analyses a macroblock with the whole warp (webp_encode.cu: vp8_analyse_warp); the host build of the
    same core (oracle/_build/libvp8cpu.so, vp8enc::analyse_and_reconstruct) walks it on one thread.  Same
    arithmetic, same decisions: the VP8 payloads must be the same bytes."""
    from tests.webp_util import chunks_of, vp8_cpu_encode, vp8_cpu_lib
    cpu = vp8_cpu_lib()
    for seed, w, h, q, noise in [(71, 256, 256, 85, 6.0), (72, 97, 61, 40, 25.0), (73, 16, 16, 90, 3.0), (74, 333, 35, 75, 12.0)]:
        img = synth_image(seed, w, h, 3, noise=noise)
        data = cuda_lib.encode(".webp", img, {abi.WebpQuality: q})
        payload = dict(chunks_of(data))[b"VP8 "]
        assert bytes(payload) == bytes(vp8_cpu_encode(cpu, img, q)), (seed, w, h, q)
