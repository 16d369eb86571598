"""CPU: the WebP ENCODER cores the device runs (vp8l_enc_core.h lossless, vp8_enc_core.h lossy),
compiled for the host by oracle/oracle_webp.cpp.
  lossless: the stream decodes (with the device's own decoder core, and with libwebp -- OpenCV's WebP codec, and
            the reference's shims where oracle/_ref is present) to exactly the input pixels;
  lossy:    the stream is a valid VP8 key frame -- both decoders agree bit for bit on its pixels --
            and its PSNR against the source is within 1 dB of (in practice above) what libwebp
            reaches at the same `quality` on the committed golden streams' sources."""
import numpy as np
import pytest

from lilliput_b200.synth import synth_image
from tests.webp_util import (alph_cpu_decode, libwebp_decode, optional_reference, psnr, riff, vp8_cpu_decode, vp8_cpu_encode,
                             vp8_cpu_lib, vp8l_cpu_decode, vp8l_cpu_encode)


@pytest.fixture(scope="module")
def cpu():
    return vp8_cpu_lib()


IMAGES = [(5, 200, 120, 3, 6.0), (6, 97, 61, 4, 40.0), (7, 1, 1, 3, 6.0), (8, 513, 3, 4, 6.0), (9, 2, 300, 3, 20.0)]


@pytest.mark.parametrize("seed,w,h,ch,noise", IMAGES)
def test_lossless_encoder_round_trips(cpu, seed, w, h, ch, noise):
    img = synth_image(seed, w, h, ch, noise=noise)
    payload = vp8l_cpu_encode(cpu, img)
    assert np.array_equal(vp8l_cpu_decode(cpu, payload, w, h, ch), img)


def test_lossless_encoder_flat_and_random_images(cpu):
    flat = np.zeros((40, 40, 3), np.uint8)
    flat[:] = (10, 200, 30)  # single-symbol prefix codes everywhere
    rnd = np.random.default_rng(5).integers(0, 256, (50, 70, 4), dtype=np.uint8)
    for img in (flat, rnd):
        h, w, ch = img.shape
        assert np.array_equal(vp8l_cpu_decode(cpu, vp8l_cpu_encode(cpu, img), w, h, ch), img)


def test_alpha_plane_round_trips_through_alph(cpu):
    a = np.clip(synth_image(3, 96, 64, 1, noise=20.0).reshape(64, 96).astype(int) * 2 - 128, 0, 255).astype(np.uint8)
    payload = vp8l_cpu_encode(cpu, a)
    assert payload[0] == 1  # ALPH header: VP8L-compressed, unfiltered
    assert np.array_equal(alph_cpu_decode(cpu, payload, 96, 64), a)


def test_lossless_and_alpha_streams_decode_with_the_reference(cpu):
    ref_lib = optional_reference()
    img = synth_image(11, 120, 90, 4, noise=15.0)
    lossless = riff([(b"VP8L", vp8l_cpu_encode(cpu, img))])
    assert np.array_equal(libwebp_decode(lossless), img)
    # lossy colour + lossless alpha in a VP8X container
    vp8x = bytes([0x10, 0, 0, 0]) + (119).to_bytes(3, "little") + (89).to_bytes(3, "little")
    payload = vp8_cpu_encode(cpu, img, 80)
    data = riff([(b"VP8X", vp8x), (b"ALPH", vp8l_cpu_encode(cpu, img[:, :, 3])), (b"VP8 ", payload)])
    got = libwebp_decode(data)
    assert np.array_equal(got[:, :, 3], img[:, :, 3]) and np.array_equal(got[:, :, :3], vp8_cpu_decode(cpu, payload))
    if ref_lib:
        _, frames, _, rc = ref_lib.webp_frames(lossless)
        assert rc == 0 and np.array_equal(frames[0], img)
        _, frames, _, rc = ref_lib.webp_frames(data)
        assert rc == 0 and np.array_equal(frames[0][:, :, 3], img[:, :, 3])


@pytest.mark.parametrize("quality", [20, 50, 75, 90, 100])
@pytest.mark.parametrize("seed,w,h,noise", [(21, 256, 256, 6.0), (22, 97, 61, 30.0), (23, 17, 33, 6.0), (24, 1, 1, 6.0)])
def test_lossy_encoder_writes_valid_streams_of_sane_quality(cpu, quality, seed, w, h, noise):
    img = synth_image(seed, w, h, 3, noise=noise)
    payload = vp8_cpu_encode(cpu, img, quality)
    got = vp8_cpu_decode(cpu, payload)
    assert got.shape == img.shape
    if w >= 64 and noise < 10:
        assert psnr(got, img) > 27.0 + quality / 25.0  # smooth synthetic content: 28-31 dB across the range


def test_lossy_stream_decodes_identically_with_the_reference_and_matches_libwebp_quality(cpu):
    import cv2
    ref_lib = optional_reference()
    for seed, w, h, noise in [(31, 320, 200, 6.0), (32, 97, 61, 30.0), (33, 33, 65, 12.0)]:
        img = synth_image(seed, w, h, 3, noise=noise)
        for quality in (30, 75, 90):
            payload = vp8_cpu_encode(cpu, img, quality)
            theirs = libwebp_decode(riff([(b"VP8 ", payload)]))
            assert np.array_equal(theirs, vp8_cpu_decode(cpu, payload))
            if ref_lib:
                _, frames, _, rc = ref_lib.webp_frames(riff([(b"VP8 ", payload)]))
                assert rc == 0 and np.array_equal(frames[0], theirs)
            ok, lw = cv2.imencode(".webp", img, [cv2.IMWRITE_WEBP_QUALITY, quality])
            assert psnr(theirs, img) > psnr(cv2.imdecode(lw, cv2.IMREAD_COLOR), img) - 1.0


@pytest.mark.parametrize("quality", [50, 75, 85, 95])
def test_lossy_encoder_size_bound_against_libwebp(cpu, quality):
    """SURVEY 7's acceptance rule for the lossy encoder: at libwebp's PSNR (within 0.25 dB), at most 1.10 x libwebp's
    bytes -- on the content class of BASELINE config 3 (synthetic fields + edges + sensor-like noise).  The stream codes
    its coefficients with per-frame probabilities and per-macroblock skip flags (RFC 6386 13.4 / 9.11) and chooses per
    macroblock between one 16x16 prediction and sixteen 4x4 ones; on the reference's own sample photographs (not
    shippable, numbers in DESIGN.md) the files are 0.92-1.06 x libwebp's."""
    cv2 = pytest.importorskip("cv2")
    for seed, w, h, noise in [(21, 512, 512, 6.0), (51, 512, 512, 3.0), (52, 256, 256, 6.0), (53, 512, 512, 12.0),
                              (55, 384, 256, 25.0)]:
        img = synth_image(seed, w, h, 3, noise=noise)
        payload = vp8_cpu_encode(cpu, img, quality)
        ok, lw = cv2.imencode(".webp", img, [cv2.IMWRITE_WEBP_QUALITY, quality])
        assert ok
        mine, theirs = psnr(vp8_cpu_decode(cpu, payload), img), psnr(cv2.imdecode(lw, cv2.IMREAD_COLOR), img)
        assert mine >= theirs - 0.25, (seed, quality, mine, theirs)
        assert len(payload) + 20 <= 1.10 * len(lw), (seed, quality, len(payload), len(lw))  # + RIFF / chunk headers


def test_4x4_prediction_pays_on_detail_and_both_forms_are_valid(cpu):
    """The 16x16-versus-4x4 choice (RFC 6386 8.3 / 12.3): textured content comes out smaller with it than without at
    about the same PSNR, and either way libwebp and the device's decoder core agree on the pixels."""
    ref_lib = optional_reference()
    for t, (w, h) in enumerate([(256, 256), (200, 120), (97, 61)]):
        rng = np.random.default_rng(9 + t)
        # smooth field cut by straight edges at arbitrary angles: the structure sub-block modes predict and the four
        # 16x16 modes cannot
        yy, xx = np.mgrid[0:h, 0:w]
        img = synth_image(60 + t, w, h, 3, noise=1.0).astype(np.int32)
        for _ in range(14):
            a, b, c = rng.normal(size=3)
            img += ((a * xx + b * yy + c * 20 - (a * w + b * h) / 2) > 0)[:, :, None] * rng.integers(-70, 70, 3)
        img = np.clip(img, 0, 255).astype(np.uint8)
        sizes, quals = [], []
        for i4 in (0, 1):
            payload = vp8_cpu_encode(cpu, img, 80, try_i4=i4)
            mine = vp8_cpu_decode(cpu, payload)
            assert np.array_equal(libwebp_decode(riff([(b"VP8 ", payload)])), mine)
            if ref_lib:
                _, frames, _, rc = ref_lib.webp_frames(riff([(b"VP8 ", payload)]))
                assert rc == 0 and np.array_equal(frames[0], mine)
            sizes.append(len(payload))
            quals.append(psnr(mine, img))
        assert sizes[1] < 0.92 * sizes[0], sizes  # measured 0.81 / 0.81 / 0.89
        assert quals[1] > quals[0] - 0.35, quals


def test_data_forms_of_the_4x4_predictors_equal_the_code_forms(cpu):
    """The device tries the ten sub-block modes through a table (kVp8Pred4, generated by tools/gen_vp8_pred4_table.py from
    vp8::pred_4x4's source) and prices them through a path table: both must be the functions they replace."""
    import ctypes
    cpu.vp8_cpu_check_pred4_tables.restype = ctypes.c_long
    assert cpu.vp8_cpu_check_pred4_tables(ctypes.c_long(30000), ctypes.c_uint(11)) == 0
