"""GPU: HDR (PQ / HLG cICP) and 16-bit PNG sources in the heterogeneous batch (lp_xbatch_transform, csrc/xbatch.cu).

A PNG whose cICP chunk carries a PQ (16) or HLG (18) transfer is tone-mapped to SDR BT.709 right after the decode, as
Transform does (ops.go:154-165): the grid path runs one batched tone map (csrc/tonemap.cu) over the HDR frames of every
frame window, between the defilter and the resize.  16-bit PNGs keep the high byte of every sample, as the per-image
decoder does.  Every item is compared with per-image lp_transform of the same library (status and bytes), with
grid_items / fallback_items asserted exactly; outside ourselves, PNG output at the source size is held against the
oracle's tone map of the oracle's (or the golden file's) decoded pixels."""
import struct
import zlib

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.test_gpu_xbatch import check_against_per_image, rgb_png

pytestmark = pytest.mark.gpu
T = 10**12
FIT = dict(Width=64, Height=64, ResizeMethod=abi.ImageOpsFit)
RESIZE = dict(Width=40, Height=27, ResizeMethod=abi.ImageOpsResize)
PRIMARIES = [9, 11, 12, 6, 10, 1, 77]  # BT.2020, P3 (DCI, Display), BT.601, XYZ, BT.709 and a code point with no matrix
LAYOUTS = {"rgb": (2, 3), "rgba": (6, 4), "ga": (4, 2)}  # colour type, samples per pixel
SIZES = [(1, 1), (3, 2), (33, 17), (64, 48), (101, 75)]
SINKS = {
    "jpeg": (".jpeg", {abi.JpegQuality: 85}),
    "webp": (".webp", {abi.WebpQuality: 85}),
    "webp_lossless": (".webp", {abi.WebpQuality: 101}),
    "png": (".png", {abi.PngCompression: 3}),
}
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]


def close_enough(a, b, frac=2e-3):  # the tone map's tolerance (tests/test_gpu_tonemap.py)
    d = np.abs(a.astype(int) - b.astype(int))
    return d.max() <= 1 and (d > 0).mean() <= frac


def chunk(tag, data):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def exif_block(orientation):
    return b"II*\x00\x08\x00\x00\x00" + b"\x01\x00" + b"\x12\x01\x03\x00\x01\x00\x00\x00" + bytes([orientation, 0, 0, 0]) + b"\x00" * 4


def png_file(samples, color_type, bit_depth, interlace=False, cicp=None, orientation=None, level=6):
    """samples: [h, w, channels] at full precision, in file order.  Every row Sub-filtered (numpy: any size is quick).
    cicp: (primaries, transfer) written right behind IHDR; orientation: an eXIf chunk in front of the IDATs."""
    h, w, c = samples.shape
    bpp = c * bit_depth // 8

    def rows(sub):
        a = np.ascontiguousarray(sub.astype(">u2" if bit_depth == 16 else np.uint8)).view(np.uint8).reshape(sub.shape[0], -1)
        f = a.copy()
        f[:, bpp:] = a[:, bpp:] - a[:, :-bpp]  # (uint8: modulo 256)
        return np.concatenate([np.ones((a.shape[0], 1), np.uint8), f], axis=1).tobytes()
    raw = b"".join(rows(samples[y0::dy, x0::dx]) for x0, y0, dx, dy in (ADAM7 if interlace else [(0, 0, 1, 1)])
                   if samples[y0::dy, x0::dx].size)
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, bit_depth, color_type, 0, 0, int(interlace)))
    if cicp is not None:
        out += chunk(b"cICP", bytes([cicp[0], cicp[1], 0, 1]))
    if orientation is not None:
        out += chunk(b"eXIf", exif_block(orientation))
    z = zlib.compress(raw, level)
    return out + chunk(b"IDAT", z[: len(z) // 2]) + chunk(b"IDAT", z[len(z) // 2:]) + chunk(b"IEND", b"")


def with_cicp(png, primaries, transfer):
    return png[:33] + chunk(b"cICP", bytes([primaries, transfer, 0, 1])) + png[33:]  # behind IHDR


def source(seed, w, h, layout, bits, noise=8.0):
    """(colour type, samples) of a synthetic PNG: 16-bit samples carry a random low byte under the 8-bit picture"""
    ct, c = LAYOUTS[layout]
    img = synth_image(seed, w, h, 4 if c != 3 else 3, noise=noise)
    s = {"rgb": lambda: img[..., ::-1], "rgba": lambda: img[..., [2, 1, 0, 3]], "ga": lambda: img[..., [1, 3]]}[layout]()
    s = s.astype(np.uint16)
    if bits == 16:
        s = s * 256 + np.random.default_rng(seed).integers(0, 256, s.shape, dtype=np.uint16)
    return ct, s


def hdr_png(seed, w, h, layout="rgb", bits=16, transfer=16, primaries=9, interlace=False, noise=8.0, **kw):
    ct, s = source(seed, w, h, layout, bits, noise)
    return png_file(s, ct, bits, interlace, cicp=(primaries, transfer), **kw)


def hdr_matrix():
    """PQ and HLG x every primaries code x RGB / RGBA / gray+alpha x 8 / 16 bits x Adam7 or not, at sizes from 1x1 up"""
    files, k = [], 0
    for transfer in (16, 18):
        for primaries in PRIMARIES:
            for layout in LAYOUTS:
                for bits in (8, 16):
                    for interlace in (False, True):
                        w, h = SIZES[k % len(SIZES)]
                        files.append(hdr_png(7000 + k, w, h, layout, bits, transfer, primaries, interlace))
                        k += 1
    return files


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


@pytest.fixture(scope="module")
def neighbours(cuda_lib, oracle):
    """(grid files, SDR-cICP PNGs): the other sources that share a call with the HDR files"""
    plain = [rgb_png(synth_image(7500, 120, 80, 3)), rgb_png(synth_image(7501, 77, 50, 4), interlace=True),
             png_file(source(7502, 90, 61, "rgb", 16)[1], 2, 16), png_file(source(7503, 64, 48, "rgba", 16)[1], 6, 16)]
    jpegs = [oracle.jpeg_encode(synth_image(7510 + k, 160, 90 + 10 * k, 3), 90) for k in range(2)]
    webps = [cuda_lib.encode(".webp", synth_image(7520 + k, 96, 64, 3), {abi.WebpQuality: 80}) for k in range(2)]
    sdr = [with_cicp(rgb_png(synth_image(7530, 100, 70, 3)), 1, 13),
           png_file(source(7531, 50, 40, "rgba", 16)[1], 6, 16, cicp=(9, 14))]
    return dict(plain=plain, jpeg=jpegs, webp=webps, sdr=sdr)


def options(sink, geom, **kw):
    ft, enc = SINKS[sink]
    kw.setdefault("EncodeTimeout_ns", T)
    return abi.ImageOptions(FileType=ft, EncodeOptions=enc, **geom, **kw)


# ---------------------------------------------------------------- the tone map itself

@pytest.mark.parametrize("transfer", [16, 18])
def test_per_image_tone_map_against_the_oracle(cuda_lib, oracle, transfer):
    """The batched tone map with one frame (Framebuffer.TonemapToSDR): the oracle's result within the tolerance, the
    same bytes on a second call, alpha untouched.  Sizes below, at and across one 4096-pixel block and a 1080p frame."""
    for seed, (w, h, c) in enumerate([(3, 2, 3), (64, 64, 4), (4097, 2, 3), (97, 61, 4), (1920, 1080, 3)]):
        img = synth_image(7400 + seed, w, h, c, noise=10.0)
        for pr in PRIMARIES:
            got = cuda_lib.tonemap(img, transfer, pr)
            assert close_enough(got, oracle.tonemap_to_sdr(img, transfer, pr)), (w, h, c, pr)
            assert np.array_equal(cuda_lib.tonemap(img, transfer, pr), got)
            if c == 4:
                assert np.array_equal(got[..., 3], img[..., 3])


# ---------------------------------------------------------------- same result as lp_transform

@pytest.mark.parametrize("geom", [FIT, RESIZE], ids=["fit", "resize"])
@pytest.mark.parametrize("sink", list(SINKS))
def test_same_result_as_lp_transform(cuda_lib, xb, neighbours, sink, geom):
    hdr = hdr_matrix()
    nb = neighbours
    files = hdr[:40] + nb["sdr"] + nb["jpeg"] + hdr[40:100] + nb["plain"] + nb["webp"] + hdr[100:]
    outs, status = check_against_per_image(cuda_lib, xb, files, options(sink, geom))
    assert all(status[files.index(f)] == 0 for f in hdr)
    # per image: SDR-cICP PNGs to PNG (Transform re-attaches the chunk); JPEG and WebP sources to lossless WebP
    per_image = {"png": len(nb["sdr"]), "webp_lossless": len(nb["jpeg"]) + len(nb["webp"])}.get(sink, 0)
    st = xb.stats()
    assert st["fallback_items"] == per_image and st["grid_items"] == len(files) - per_image, st
    if sink == "png":  # (Transform writes the chunk right behind IHDR) an HDR tag never, an SDR tag always
        assert not any(b"cICP" in outs[files.index(f)][:64] for f in hdr)
        assert all(b"cICP" in outs[files.index(f)][:64] for f in nb["sdr"])


def test_batch_composition_does_not_matter(cuda_lib, xb, neighbours):
    """A frame's tone map depends on that frame only: alone, among many different neighbours, and in a second identical
    call, the same HDR file gives the same bytes, and those are lp_transform's."""
    probes = [hdr_png(7600, 301, 203, "rgba", 16, 16, 9), hdr_png(7601, 257, 129, "rgb", 8, 18, 12, interlace=True)]
    crowd = hdr_matrix() + [f for v in neighbours.values() for f in v]
    for sink in ("png", "jpeg"):
        opt = options(sink, RESIZE)
        alone = [xb.transform([p], opt, out_cap=1 << 22)[0][0] for p in probes]
        mixed = crowd[:50] + [probes[0]] + crowd[50:] + [probes[1]]
        for _ in range(2):
            outs, status = xb.transform(mixed, opt, out_cap=1 << 22)
            assert status[50] == status[-1] == 0
            assert [outs[50], outs[-1]] == alone
        assert xb.stats()["grid_items"] == len(mixed) - (len(neighbours["sdr"]) if sink == "png" else 0)
        assert alone == [cuda_lib.transform(p, opt, dst_cap=1 << 22) for p in probes]


# ---------------------------------------------------------------- against the oracle

def test_png_output_against_the_oracle(cuda_lib, xb, oracle, golden):
    """PNG output at the source size (a plain copy in the resize): the decoded output is the oracle's tone map of the
    source's decoded pixels, within the tone map's tolerance; 16-bit golden files use the golden decoded pixels."""
    cases = []  # (file, 8-bit decoded pixels, transfer, primaries)
    for k, (w, h, layout, bits, transfer, primaries, interlace) in enumerate([
            (97, 61, "rgb", 16, 16, 9, False), (97, 61, "rgba", 8, 18, 12, True), (97, 61, "ga", 16, 18, 10, False),
            (160, 120, "rgb", 8, 16, 6, True), (160, 120, "rgba", 16, 18, 1, False), (160, 120, "rgb", 16, 16, 77, True)]):
        f = hdr_png(7700 + k, w, h, layout, bits, transfer, primaries, interlace)
        cases.append((f, oracle.png_decode(f), transfer, primaries))
    for k, name in enumerate(["rgba16", "fixture_16bit_alpha"]):
        f = with_cicp(golden[f"png_{name}"].tobytes(), (9, 12)[k], (16, 18)[k])
        cases.append((f, golden[f"pngdec_{name}"], (16, 18)[k], (9, 12)[k]))
    by_size = {}
    for c in cases:
        by_size.setdefault(c[1].shape[:2], []).append(c)
    for (h, w), group in by_size.items():
        files = [c[0] for c in group]
        outs, status = check_against_per_image(cuda_lib, xb, files, options("png", dict(Width=w, Height=h, ResizeMethod=abi.ImageOpsResize)))
        assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
        for out, (_, src, transfer, primaries) in zip(outs, group):
            got = oracle.png_decode(out)
            want = oracle.tonemap_to_sdr(src, transfer, primaries)
            assert got.shape == want.shape
            assert close_enough(got, want), (w, h, transfer, primaries)
            assert not np.array_equal(got, src)
            if src.shape[2] == 4:
                assert np.array_equal(got[..., 3], src[..., 3])


# ---------------------------------------------------------------- arena

def test_small_arena_gives_the_same_bytes(cuda_lib, xb):
    """1 GiB: each lane's frame window (a fifth of its half) holds two 4000x3000 RGBA frames, so the HDR frames of a
    task are tone-mapped window by window; the bytes are those of the large arena and of lp_transform."""
    files = []
    for k in range(4):
        ct, s = source(7800 + k, 1000, 750, "rgba", 8, noise=0.0)
        files.append(png_file(np.tile(s, (4, 4, 1)), ct, 8, cicp=((9, 12)[k % 2], (16, 18)[k % 2]), level=1))
    files += [hdr_png(7810 + k, 2000, 1500, "rgb", 16, 16, 9, level=1) for k in range(2)]
    files += hdr_matrix()[:24]
    opt = options("jpeg", FIT)
    big, big_status = xb.transform(files, opt, out_cap=1 << 22)
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        outs, status = check_against_per_image(cuda_lib, small, files, opt)
        assert small.stats()["grid_items"] == len(files) and small.stats()["fallback_items"] == 0, small.stats()
        assert status == big_status == [0] * len(files) and outs == big
    finally:
        small.close()


# ---------------------------------------------------------------- routing

def test_routing(cuda_lib, xb, golden):
    grid = [hdr_png(7900, 120, 90, "rgb", 16, 16, 9), hdr_png(7901, 90, 120, "ga", 8, 18, 12),
            png_file(source(7902, 100, 60, "rgb", 16)[1], 2, 16)]
    per_image = {
        "sdr_cicp": with_cicp(rgb_png(synth_image(7910, 100, 70, 3)), 1, 13),
        "gray16": png_file(source(7911, 80, 60, "ga", 16)[1][..., :1], 0, 16),
        "gray16_hdr": png_file(source(7912, 80, 60, "ga", 16)[1][..., :1], 0, 16, cicp=(9, 16)),
        "hdr_exif_rotated": hdr_png(7913, 120, 90, "rgb", 16, 16, 9, orientation=6),
    }
    files = grid[:1] + list(per_image.values()) + grid[1:]
    outs, status = check_against_per_image(cuda_lib, xb, files, options("png", FIT))
    assert status == [0] * len(files)
    st = xb.stats()
    assert st["grid_items"] == len(grid) and st["fallback_items"] == len(per_image), st
    assert b"cICP" in outs[1][:64]  # the SDR tag rides into the output
    # the same files to JPEG: the SDR tag changes no pixel, so that file joins the grid
    check_against_per_image(cuda_lib, xb, files, options("jpeg", FIT))
    st = xb.stats()
    assert st["grid_items"] == len(grid) + 1 and st["fallback_items"] == len(per_image) - 1, st
    # NoResize, and the lossless sink's gate on a zero encode budget (every PNG per image): nothing on the grid
    for opt in (options("jpeg", dict(Width=0, Height=0, ResizeMethod=abi.ImageOpsNoResize)),
                options("webp_lossless", FIT, EncodeTimeout_ns=0)):
        check_against_per_image(cuda_lib, xb, files, opt)
        st = xb.stats()
        assert st["grid_items"] == 0 and st["fallback_items"] == len(files), st
