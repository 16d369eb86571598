"""GPU: lossless WebP output (WebpQuality above 100) in the heterogeneous batch (lp_xbatch_transform, csrc/xbatch.cu):
PNG stills and GIF animations are decoded and resized on the grid path and every run of resized frames goes through
webp_encode_lossless_batch (csrc/webp_encode.cu); JPEG and WebP sources stay with the per-image path.

Every item is compared with per-image lp_transform of the same library (status and bytes), and grid_items /
fallback_items are asserted exactly, so a silent hand-over to the per-image path cannot pass.  Outside ourselves: libwebp
(OpenCV) decodes PNG items to the oracle's Fit of the decoded source, and Pillow reads every frame of an animation back
as the oracle's composited GIF frame, fitted."""
import io

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.png_writer import write_png
from tests.test_gpu_xbatch import check_against_per_image, rgb_png
from tests.test_gpu_xbatch_gif import synthetic_gifs
from tests.test_gpu_xbatch_jpeg_webp import cv2_jpeg, png_profile, with_iccp
from tests.webp_util import chunks_of, frames_of, libwebp_decode

pytestmark = pytest.mark.gpu
T = 10**12
FIT = dict(Width=96, Height=96, ResizeMethod=abi.ImageOpsFit)
RESIZE = dict(Width=50, Height=23, ResizeMethod=abi.ImageOpsResize)
ONE = dict(Width=1, Height=1, ResizeMethod=abi.ImageOpsResize)


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def opt(quality=101, **kw):
    kw.setdefault("EncodeTimeout_ns", T)
    return abi.ImageOptions(FileType=".webp", EncodeOptions={abi.WebpQuality: quality}, **kw)


def opaque(img):
    img = img.copy()
    img[..., 3] = 255
    return img


def png_kinds():
    """(name, PNG): every colour type the grid path decodes to BGR or BGRA, at several geometries."""
    rng = np.random.default_rng(11)
    gray_alpha = np.stack([synth_image(601, 120, 90, 1), synth_image(602, 120, 90, 1)], axis=-1)
    idx = (synth_image(603, 110, 70, 1)[..., None] // 16).astype(np.uint8)
    palette = rng.integers(0, 256, (16, 3))
    trns = bytes(int(v) for v in rng.integers(0, 256, 10))
    return [
        ("rgb", rgb_png(synth_image(600, 300, 200, 3))),
        ("rgb_same_size", rgb_png(synth_image(604, 300, 200, 3, noise=20.0))),
        ("rgba", rgb_png(synth_image(605, 256, 256, 4))),
        ("rgba_opaque", rgb_png(opaque(synth_image(606, 256, 256, 4)))),
        ("gray_alpha", write_png(gray_alpha, 4, 8)),
        ("palette_trns", write_png(idx, 3, 8, palette=palette, trns=trns)),
        ("adam7_rgb", rgb_png(synth_image(607, 97, 61, 3), interlace=True)),
        ("adam7_rgba", rgb_png(synth_image(608, 97, 61, 4), interlace=True)),
        ("small", rgb_png(synth_image(609, 5, 3, 4))),
    ]


@pytest.fixture(scope="module")
def pngs():
    return png_kinds()


@pytest.mark.parametrize("geom", [FIT, RESIZE, ONE], ids=["fit", "resize", "one_pixel"])
def test_png_sources_on_the_grid(cuda_lib, xb, pngs, geom):
    names = [n for n, _ in pngs]
    files = [d for _, d in pngs]
    outs, status = check_against_per_image(cuda_lib, xb, files, opt(**geom))
    assert status == [0] * len(files), dict(zip(names, status))
    st = xb.stats()
    assert st["grid_items"] == len(files) and st["fallback_items"] == 0, st
    for name, out in zip(names, outs):
        assert [t for t, _ in chunks_of(out)] == [b"VP8L"], name


def test_png_profile_travels_into_the_webp(cuda_lib, xb):
    prof = png_profile()
    files = [with_iccp(rgb_png(synth_image(620, 300, 200, 3)), prof), with_iccp(rgb_png(synth_image(621, 200, 300, 4)), prof),
             rgb_png(synth_image(622, 300, 200, 3))]
    outs, status = check_against_per_image(cuda_lib, xb, files, opt(**FIT))
    assert status == [0, 0, 0] and xb.stats()["grid_items"] == 3
    for k in (0, 1):
        ch = dict(chunks_of(outs[k]))
        assert ch[b"ICCP"] == prof and b"VP8L" in ch
        assert outs[k][20] & 0x20  # VP8X: ICC flag
    assert b"ICCP" not in dict(chunks_of(outs[2]))


def test_png_pixels_against_the_oracle(cuda_lib, xb, pngs, oracle):
    """libwebp decodes each PNG item to the oracle's Fit of the oracle's decode of the source, exactly."""
    files = [d for _, d in pngs]
    outs, status = xb.transform(files, opt(**FIT), out_cap=1 << 22)
    assert status == [0] * len(files)
    for (name, src), out in zip(pngs, outs):
        dec = oracle.png_decode(src)
        dec = dec[0] if isinstance(dec, tuple) else dec
        ow, oh = oracle.expected_size(dec.shape[1], dec.shape[0], FIT["Width"], FIT["Height"])
        assert np.array_equal(libwebp_decode(out), oracle.fit(dec, ow, oh)), name


def gif_files(golden):
    fixtures = [golden[k].tobytes() for k in sorted(golden.files) if k.startswith("gif_") and golden[k].ndim == 1]
    return fixtures + list(synthetic_gifs().values())


def test_gif_sources_on_the_grid(cuda_lib, xb, golden):
    """The golden GIF fixtures and the synthetic animations: every item as per image; the grid takes exactly what it
    takes for lossy output, and every synthetic animation."""
    files = gif_files(golden)
    syn = len(synthetic_gifs())
    for geom in (FIT, RESIZE):
        outs, status = check_against_per_image(cuda_lib, xb, files, opt(**geom), cap=1 << 23)
        st = xb.stats()
        xb.transform(files, opt(85, **geom), out_cap=1 << 23)
        assert st["grid_items"] == xb.stats()["grid_items"], (st, xb.stats())
        assert st["grid_items"] >= syn and all(s == 0 for s in status[-syn:]), st
        for out, s in zip(outs, status):
            if s == 0:
                assert all(tag == b"VP8L" for tag, _, _ in frames_of(out))


def test_one_frame_gifs_and_stills(cuda_lib, xb):
    """One-frame GIFs, and DisableAnimatedOutput: frame 0 of every animation written as a lossless still."""
    cases = synthetic_gifs()
    files = list(cases.values())
    outs, status = check_against_per_image(cuda_lib, xb, [cases["one_frame"]] * 3, opt(**FIT))
    assert status == [0] * 3 and xb.stats()["grid_items"] == 3
    assert [t for t, _ in chunks_of(outs[0])][-1:] == [b"VP8L"] and b"ANIM" not in dict(chunks_of(outs[0]))
    outs, status = check_against_per_image(cuda_lib, xb, files, opt(DisableAnimatedOutput=True, **FIT))
    assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
    for out in outs:
        assert b"ANIM" not in dict(chunks_of(out)) and len(frames_of(out)) == 1
    # (with no time to encode, a still still gets its frame 0 written)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt(DisableAnimatedOutput=True, EncodeTimeout_ns=0, **FIT))
    assert xb.stats()["grid_items"] == len(files)


def test_animation_frames_against_the_oracle(cuda_lib, xb, oracle):
    """Pillow (libwebp's demuxer and decoder) reads every frame of each animated output back as the oracle's composited
    GIF frame, fitted, exactly."""
    Image = pytest.importorskip("PIL.Image")
    cases = synthetic_gifs()
    names = ["local_every_frame", "palette_changes_back", "partial_offsets", "interlaced", "no_gcb"]
    files = [cases[n] for n in names]
    outs, status = xb.transform(files, opt(**FIT), out_cap=1 << 22)
    assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
    for name, src, out in zip(names, files, outs):
        frames, _, _, _ = oracle.gif_frames(src)
        h, w = frames[0].shape[:2]
        ow, oh = oracle.expected_size(w, h, FIT["Width"], FIT["Height"])
        im = Image.open(io.BytesIO(out))
        assert im.n_frames == len(frames), name
        for k, f in enumerate(frames):
            im.seek(k)
            got = np.asarray(im.convert("RGBA"))[:, :, [2, 1, 0, 3]]
            assert np.array_equal(got, oracle.fit(f, ow, oh)), (name, k)


def test_routing(cuda_lib, xb, golden):
    """JPEG and WebP sources, one-channel gray PNGs, damaged files and NoResize stay per image; the option gates are
    those of the lossy sink, with every PNG under the rule the lossy sink keeps for PNGs with a profile."""
    cases = synthetic_gifs()
    png_rgb, png_rgba = rgb_png(synth_image(640, 200, 150, 3)), rgb_png(synth_image(641, 150, 200, 4))
    gif_anim, gif_one = cases["transparency_disposal"], cases["one_frame"]
    png_icc = with_iccp(rgb_png(synth_image(642, 120, 80, 3)), png_profile())
    per_image = [cv2_jpeg(synth_image(643, 320, 240, 3), 85),
                 cuda_lib.encode(".webp", synth_image(644, 120, 90, 3), {abi.WebpQuality: 80}),
                 cuda_lib.encode(".webp", synth_image(645, 120, 90, 4), {abi.WebpQuality: 101}),
                 write_png(synth_image(646, 90, 60, 1)[..., None], 0, 8),
                 b"\x89PNG\r\n\x1a\n" + b"\0" * 40,
                 b"GIF89a" + b"\1" * 30]
    grid = [png_rgb, png_rgba, png_icc, gif_anim, gif_one]
    files = per_image[:3] + grid[:2] + per_image[3:] + grid[2:]
    outs, status = check_against_per_image(cuda_lib, xb, files, opt(**FIT))
    st = xb.stats()
    assert st["grid_items"] == len(grid) and st["fallback_items"] == len(per_image), st
    assert status[3] == status[4] == 0 and status[-3:] == [0, 0, 0]
    # (option, grid items): the gates of the lossy sink, except that under the options whose result the per-image path
    # decides after the frame (no time to encode, MaxEncodeFrames 1, a negative MaxEncodeDuration) every PNG stays per
    # image -- the lossy sink keeps only PNGs with a profile there
    gates = [(dict(), 5), (dict(ResizeMethod=abi.ImageOpsNoResize, Width=96, Height=96), 0), (dict(MaxEncodeFrames=1), 0),
             (dict(MaxEncodeFrames=2), 3), (dict(MaxEncodeDuration_ns=-1), 0), (dict(MaxEncodeDuration_ns=10**9), 3),
             (dict(EncodeTimeout_ns=0), 0), (dict(EncodeTimeout_ns=0, DisableAnimatedOutput=True), 2),
             (dict(DisableAnimatedOutput=True), 5)]
    for g, grid in gates:
        kw = dict(FIT)
        kw.update(g)
        check_against_per_image(cuda_lib, xb, files, opt(**kw))
        assert xb.stats()["grid_items"] == grid, (g, xb.stats())


def test_small_destination_buffers(cuda_lib, xb):
    cases = synthetic_gifs()
    files = [rgb_png(synth_image(660, 300, 200, 4)), cases["late_buckets"], cases["one_frame"], rgb_png(synth_image(661, 64, 64, 3))]
    sizes = [len(cuda_lib.transform(f, opt(**FIT))) for f in files]
    for cap in (min(sizes) - 1, sorted(sizes)[1], sorted(sizes)[2] + 1, 100):
        outs, status = check_against_per_image(cuda_lib, xb, files, opt(**FIT), cap=cap)
        assert xb.stats()["grid_items"] == len(files)
        assert [s != 0 for s in status] == [n > cap for n in sizes], (cap, sizes, status)
        assert all(s in (0, abi.LP_ERR_INVALID_IMAGE) for s in status), status


def test_small_arena_gives_the_same_bytes(cuda_lib, xb, pngs, golden):
    files = [d for _, d in pngs] + list(synthetic_gifs().values())
    big, big_status = xb.transform(files, opt(**FIT), out_cap=1 << 22)
    small = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        outs, status = small.transform(files, opt(**FIT), out_cap=1 << 22)
        assert status == big_status and outs == big
        assert small.stats()["grid_items"] > 0
    finally:
        small.close()


def test_multi_transform(cuda_lib, pngs):
    import torch
    ndev = max(1, torch.cuda.device_count())
    devices = list(range(ndev)) if ndev > 1 else [0, 0]
    m = abi.MultiBatch(cuda_lib, devices, arena_bytes=4 << 30)
    x = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    try:
        files = [d for _, d in pngs] + list(synthetic_gifs().values())
        outs, status = m.transform(files, opt(**FIT))
        one, one_status = x.transform(files, opt(**FIT))
        assert status == one_status == [0] * len(files) and outs == one
        assert sum(m.stats(g)["grid_items"] for g in range(len(devices))) == len(files)
    finally:
        m.close()
        x.close()
