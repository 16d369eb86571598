"""Randomised differential tests: the CPU restatement in oracle/ against the reference's own shims
(oracle/_ref, compiled in place from /root/reference) on inputs that are in no golden file.  They
run where oracle/_ref exists (the build container) and skip elsewhere; bit-exact throughout.

What is compared, with the reference entry point each side goes through:
  resize / Fit      opencv_mat_crop + opencv_mat_resize (ref opencv.cpp:196-215, opencv.go:326-374)
  orientation       opencv_mat_orientation_transform     (ref opencv.cpp:217-221)
  JPEG decode       opencv_decoder_read_data             (ref opencv.cpp:134-171): sampling factors,
                    restart intervals, gray, odd sizes, optimised tables, progressive
  JPEG encode       opencv_encoder_write                 (ref opencv.cpp:173-194): bytes
  PNG decode        the same decoder: colour types, bit depths, interlace, compression levels
  GIF decode        giflib_decoder_* + the compositor    (ref giflib.cpp:349-568)
"""
import io

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image

cv2 = pytest.importorskip("cv2")
PIL_Image = pytest.importorskip("PIL.Image")


def _rand_img(rng, h, w, ch):
    kind = int(rng.integers(0, 3))
    if kind == 0:  # white noise: every tap matters
        img = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)
    elif kind == 1:  # smooth field + edges
        img = synth_image(int(rng.integers(0, 1 << 30)), w, h, ch, noise=float(rng.uniform(0, 20)))
        img = img.reshape(h, w, ch)
    else:  # saturated blocks: rounding at 0 / 255
        img = (rng.integers(0, 2, (h // 3 + 1, w // 3 + 1, ch), dtype=np.uint8) * 255).repeat(3, 0).repeat(3, 1)[:h, :w]
    return np.ascontiguousarray(img if ch > 1 else img.reshape(h, w))


def test_resize_random_shapes(oracle, ref_lib):
    rng = np.random.default_rng(20260922)
    cases = []
    for _ in range(60):
        cases.append((int(rng.integers(1, 500)), int(rng.integers(1, 500)),
                      int(rng.integers(1, 300)), int(rng.integers(1, 300))))
    # integer-scale fast paths, identity, one-pixel outputs, pure upscales, mixed axes
    cases += [(512, 256, 256, 128), (300, 300, 100, 100), (256, 128, 64, 32), (90, 60, 90, 60), (333, 77, 1, 1),
              (5, 7, 50, 70), (64, 64, 128, 32), (641, 479, 320, 240), (1000, 3, 10, 3), (2, 2, 1, 1)]
    for sw, sh, dw, dh in cases:
        ch = int(rng.choice([1, 3, 4]))
        img = _rand_img(rng, sh, sw, ch)
        for interp in (abi.INTER_AREA, 1):
            got = oracle.resize(img, dw, dh, interpolation=interp)
            exp = ref_lib.resize(img, dw, dh, interpolation=interp)
            assert np.array_equal(got, exp), (sw, sh, dw, dh, ch, interp)


def test_fit_random_shapes(oracle, ref_lib):
    rng = np.random.default_rng(7)
    for _ in range(60):
        sw, sh = int(rng.integers(1, 900)), int(rng.integers(1, 600))
        dw, dh = int(rng.integers(1, min(sw, 400) + 1)), int(rng.integers(1, min(sh, 400) + 1))
        ch = int(rng.choice([1, 3, 4]))
        img = _rand_img(rng, sh, sw, ch)
        assert np.array_equal(oracle.fit(img, dw, dh), ref_lib.fit(img, dw, dh)), (sw, sh, dw, dh, ch)


def test_orientation_all_codes(oracle, ref_lib):
    rng = np.random.default_rng(8)
    for _ in range(6):
        w, h, ch = int(rng.integers(1, 70)), int(rng.integers(1, 70)), int(rng.choice([1, 3, 4]))
        img = _rand_img(rng, h, w, ch)
        for o in range(1, 9):
            assert np.array_equal(oracle.orient(img, o), ref_lib.orient(img, o)), (w, h, ch, o)


def _jpeg_files(rng):
    out = []
    samplings = [0x111111, 0x211111, 0x221111, 0x411111, 0x121111]
    for i in range(42):
        w, h = int(rng.integers(1, 420)), int(rng.integers(1, 320))
        gray = i % 5 == 4
        img = _rand_img(rng, h, w, 1 if gray else 3)
        opts = [cv2.IMWRITE_JPEG_QUALITY, int(rng.integers(1, 101))]
        if not gray:
            opts += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, int(samplings[i % len(samplings)])]
        if i % 3 == 0:
            opts += [cv2.IMWRITE_JPEG_RST_INTERVAL, int(rng.integers(1, 9))]
        if i % 4 == 1:
            opts += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
        if i % 7 == 6:
            opts += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
        ok, enc = cv2.imencode(".jpg", img, opts)
        assert ok
        out.append((f"{w}x{h} gray={gray} opts={opts}", enc.tobytes()))
    # frames 4 px wide or less, where libjpeg-turbo replicates 4:2:0 / 4:2:2 chroma instead of filtering it; their own
    # generator, so the draws above stay as they were
    narrow = np.random.default_rng(91)
    for w in (1, 2, 3, 4):
        for sf in (0x221111, 0x211111):
            h = int(narrow.integers(1, 40))
            img = _rand_img(narrow, h, w, 3)
            opts = [cv2.IMWRITE_JPEG_QUALITY, int(narrow.integers(1, 101)), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf]
            ok, enc = cv2.imencode(".jpg", img, opts)
            assert ok
            out.append((f"{w}x{h} opts={opts}", enc.tobytes()))
    return out


def test_jpeg_decode_random_files(oracle, ref_lib):
    rng = np.random.default_rng(9)
    for label, data in _jpeg_files(rng):
        got, _ = oracle.jpeg_decode(data)
        assert np.array_equal(got, ref_lib.decode(data)), label


def test_jpeg_encode_random_images(oracle, ref_lib):
    rng = np.random.default_rng(10)
    for _ in range(30):
        w, h, ch = int(rng.integers(1, 400)), int(rng.integers(1, 300)), int(rng.choice([1, 3, 4]))
        img = _rand_img(rng, h, w, ch)
        q = int(rng.integers(1, 101))
        assert oracle.jpeg_encode(img, q) == ref_lib.encode(".jpeg", img, {abi.JpegQuality: q}), (w, h, ch, q)


def _png_files(rng):
    out = []
    for i in range(24):
        w, h = int(rng.integers(1, 200)), int(rng.integers(1, 150))
        ch = [1, 3, 4][i % 3]
        img = _rand_img(rng, h, w, ch)
        ok, enc = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, int(rng.integers(0, 10))])
        assert ok
        out.append((f"cv2 {w}x{h}c{ch}", enc.tobytes()))
    rgb = _rand_img(rng, 57, 83, 3)
    pil_cases = [("P", {}), ("L", {}), ("LA", {}), ("RGBA", {}), ("1", {}), ("I;16", {}), ("RGB", {"optimize": True})]
    for mode, kw in pil_cases:
        if mode == "I;16":
            im = PIL_Image.fromarray(rng.integers(0, 65536, (41, 67), dtype=np.uint16))
        else:
            im = PIL_Image.fromarray(rgb).convert(mode)
        bio = io.BytesIO()
        im.save(bio, "PNG", **kw)
        out.append((f"pil {mode}", bio.getvalue()))
    return out


def test_png_decode_random_files(oracle, ref_lib):
    rng = np.random.default_rng(11)
    for label, data in _png_files(rng):
        assert np.array_equal(oracle.png_decode(data), ref_lib.decode(data)), label


def _gif_files(rng):
    out = []
    for i in range(12):
        w, h, n = int(rng.integers(8, 90)), int(rng.integers(8, 70)), int(rng.integers(1, 6))
        frames = []
        for k in range(n):
            a = _rand_img(rng, h, w, 3)
            if i % 2:  # a moving opaque patch on a flat background: partial frames after PIL's optimiser
                a[:] = 40
                a[(3 * k) % h:(3 * k) % h + 5, (5 * k) % w:(5 * k) % w + 7] = 200
            frames.append(PIL_Image.fromarray(a).quantize(int(rng.choice([2, 16, 255]))))
        bio = io.BytesIO()
        frames[0].save(bio, "GIF", save_all=True, append_images=frames[1:], duration=40 + 10 * i, loop=i,
                       disposal=int(rng.integers(0, 4)), optimize=bool(i % 2))
        out.append((f"gif {w}x{h}x{n}", bio.getvalue()))
    return out


def test_gif_decode_random_files(oracle, ref_lib):
    rng = np.random.default_rng(12)
    for label, data in _gif_files(rng):
        gf, gd, gp, grc = oracle.gif_frames(data)
        ef, ed, ep, erc = ref_lib.gif_frames(data)
        assert len(gf) == len(ef) and len(gf) >= 1, label
        assert [d * 10 for d in gd] == list(ed), (label, gd, ed)  # centiseconds -> ms (ref giflib.go:212)
        # giflib disposal 2 -> GIF_DISPOSE_BACKGROUND (1), 3 -> GIF_DISPOSE_PREVIOUS (2), else none (ref giflib.cpp:187-199)
        assert [{2: 1, 3: 2}.get(d, 0) for d in gp] == list(ep), label
        for k in range(len(gf)):
            assert np.array_equal(gf[k], ef[k]), (label, k)
