"""GPU: GIF output in the heterogeneous batch (lp_xbatch_transform with FileType ".gif", csrc/xbatch.cu + the job-list
encoder kernels of csrc/gif_decode.cu) against per-image lp_transform of the same library, item by item: status and
bytes.  grid_items is asserted so that a silent hand-over to the per-image path cannot pass.  The reference's own
GIF -> GIF bytes (tests/golden/gif_encode_golden.npz) pin the batch too.

The synthetic animations are written byte by byte (literal-code LZW, tests/gif_streams.py), so each one has exactly the container features
it is meant to cover: local colour tables, palette changes, transparency and disposal, partial frames, interlace,
frames without a graphic control block, comment / application extensions between frames and behind the last one."""
import hashlib
import os

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.gif_streams import app, comment, gcb, write_gif
from tests.golden.make_golden_gif_encode import CASES, TIMEOUT_NS
from tests.test_gpu_xbatch import check_against_per_image, rgb_png

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "gif_encode_golden.npz"))


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


def _pal(seed, n):
    return np.random.default_rng(seed).integers(0, 256, n * 3, dtype=np.uint8).tobytes()


def _idx(seed, h, w, n):
    """Smooth-ish index pattern (blocks + gradient) so that the resize produces in-between colours."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = ((x * n) // max(w, 1) + (y // 4) * 3 + rng.integers(0, n)) % n
    noise = rng.integers(0, n, (h, w))
    return np.where(rng.random((h, w)) < 0.2, noise, base).astype(np.uint8)


W, H = 72, 54


def synthetic_gifs():
    g16, g64 = _pal(1, 16), _pal(2, 64)
    cases = {}
    cases["local_every_frame"] = write_gif(W, H, [dict(idx=_idx(10 + k, H, W, 32), local=_pal(20 + k, 32)) for k in range(4)],
                                           gct=g16)
    cases["palette_changes_back"] = write_gif(W, H, [
        dict(idx=_idx(30, H, W, 64)), dict(idx=_idx(31, H, W, 64)),
        dict(idx=_idx(32, H, W, 16), local=_pal(33, 16)),
        dict(idx=_idx(34, H, W, 64)), dict(idx=_idx(35, H, W, 64))], gct=g64)
    # frame 0 uses four colours; later frames bring in buckets nobody has consulted yet
    f0 = np.zeros((H, W), np.uint8) + (np.arange(W) // 18).astype(np.uint8)[None, :]
    cases["late_buckets"] = write_gif(W, H, [dict(idx=f0), dict(idx=_idx(40, H, W, 64)), dict(idx=(_idx(41, H, W, 64) // 2) * 2)],
                                      gct=g64)
    cases["transparency_disposal"] = write_gif(W, H, [
        dict(idx=_idx(50, H, W, 16), gcb=gcb(1, 4, 3)),
        dict(idx=_idx(51, 30, 40, 16), left=10, top=8, gcb=gcb(2, 4, 3)),
        dict(idx=_idx(52, 20, 20, 16), left=40, top=20, gcb=gcb(3, 4, 5)),
        dict(idx=_idx(53, H, W, 16), gcb=gcb(1, 4, 0)),
        dict(idx=_idx(54, 24, 30, 16), left=5, top=25, gcb=gcb(0, 4, 7))], gct=g16, bg=3)
    # opaque background (first frame without transparency), later frames whose transparent index IS the background
    cases["background_drop"] = write_gif(W, H, [
        dict(idx=_idx(55, H, W, 16), gcb=gcb(1, 4)),
        dict(idx=_idx(56, H, W, 16), gcb=gcb(1, 4, 6)),
        dict(idx=_idx(57, 20, 30, 16), left=4, top=4, gcb=gcb(0, 4, 6))], gct=g16, bg=6)
    cases["partial_offsets"] = write_gif(W, H, [
        dict(idx=_idx(60, H, W, 64)),
        dict(idx=_idx(61, 20, 33, 64), left=7, top=9),                    # no transparent index: one is forced
        dict(idx=_idx(62, 17, 25, 64), left=40, top=30, gcb=gcb(1, 3, 12)),
        dict(idx=_idx(63, 40, 10, 64), left=60, top=10, gcb=gcb(2, 3))], gct=g64)
    cases["interlaced"] = write_gif(W, H, [dict(idx=_idx(70 + k, H, W, 64), interlace=True) for k in range(3)]
                                    + [dict(idx=_idx(73, 19, 23, 64), left=3, top=4, interlace=True)], gct=g64)
    cases["no_gcb"] = write_gif(W, H, [dict(idx=_idx(80 + k, H, W, 16), gcb=None) for k in range(3)], gct=g16)
    cases["extensions"] = write_gif(W, H, [
        dict(idx=_idx(90, H, W, 16), pre=comment(b"first frame")),
        dict(idx=_idx(91, H, W, 16), pre=app(b"XMP DataXMP", b"<x/>" * 80) + comment(b"between" * 50)),
        dict(idx=_idx(92, H, W, 16), pre=gcb(2, 9, 4) + comment(b"c"), gcb=gcb(1, 7))],
        gct=g16, trailer_ext=comment(b"after the last frame") + app(b"TRAILER1.00", b"\x01\x02\x03"))
    cases["one_frame"] = write_gif(W, H, [dict(idx=_idx(95, H, W, 64), gcb=gcb(0, 0, 9))], gct=g64, loop=False)
    cases["no_global_table"] = write_gif(W, H, [dict(idx=_idx(96 + k, H, W, 8), local=_pal(97, 8)) for k in range(3)])
    return cases


# ---------------------------------------------------------------- tests

def opts(**kw):
    kw.setdefault("EncodeTimeout_ns", TIMEOUT_NS)
    return abi.ImageOptions(FileType=".gif", **kw)


def test_golden_cases_in_the_batch(cuda_lib, xb, golden):
    """Every gif_encode_golden case: all GIF fixtures in one batch call per option set; each item == lp_transform, and
    the case's own fixture == the reference's bytes.  NoResize and MaxEncodeFrames stay per image."""
    fixtures = sorted({c[0] for c in CASES} | {k[4:] for k in golden.files if k.startswith("gif_") and golden[k].ndim == 1})
    files = [golden[f"gif_{f}"].tobytes() for f in fixtures]
    for fixture, label, kw in CASES:
        outs, status = check_against_per_image(cuda_lib, xb, files, opts(**kw), cap=1 << 22)
        got = outs[fixtures.index(fixture)]
        assert hashlib.sha256(got).hexdigest() == str(G[f"sha_{fixture}__{label}"]), f"{fixture}__{label}"
        st = xb.stats()
        if kw.get("ResizeMethod") == abi.ImageOpsNoResize or kw.get("MaxEncodeFrames"):
            assert st["grid_items"] == 0
        else:
            assert st["grid_items"] >= len(files) - 2, st


def test_synthetic_animations(cuda_lib, xb):
    cases = synthetic_gifs()
    files = list(cases.values())
    for kw in (dict(Width=40, Height=40, ResizeMethod=abi.ImageOpsFit),
               dict(Width=50, Height=23, ResizeMethod=abi.ImageOpsResize),
               dict(Width=W, Height=H, ResizeMethod=abi.ImageOpsResize)):
        outs, status = check_against_per_image(cuda_lib, xb, files, opts(**kw))
        assert status == [0] * len(files), dict(zip(cases, status))
        assert xb.stats()["grid_items"] == len(files) and xb.stats()["fallback_items"] == 0


def test_config4_shape(cuda_lib, xb):
    """A 1280x720 animation of several frames -> Fit 256x256 (bench config 4 with GIF output)."""
    pytest.importorskip("PIL")
    from tests.test_gpu_xbatch import _gif
    base = synth_image(700, 1280, 720, 3, noise=0.0)
    files = [_gif([np.roll(base, 8 * k, axis=1) for k in range(6)], duration=40),
             _gif([synth_image(710 + k, 200, 120, 3, noise=0.0) for k in range(3)], duration=[20, 70, 130], loop=3)]
    outs, status = check_against_per_image(cuda_lib, xb, files, opts(Width=256, Height=256, ResizeMethod=abi.ImageOpsFit),
                                           cap=1 << 24)
    assert status == [0, 0] and xb.stats()["grid_items"] == 2
    assert outs[0][:6] == b"GIF89a" and int.from_bytes(outs[0][6:8], "little") == 256


def test_mixed_sources_timeout_and_small_buffers(cuda_lib, xb, oracle):
    """Non-GIF sources with GIF output and a zero EncodeTimeout take the per-image path and get its errors; a
    destination too small for some files gives the per-image encoder's status for exactly those."""
    cases = synthetic_gifs()
    gifs = [cases["late_buckets"], cases["one_frame"], cases["extensions"]]
    files = gifs + [oracle.jpeg_encode(synth_image(900, 120, 90, 3), 90), rgb_png(synth_image(901, 100, 80, 4))]
    fit = dict(Width=40, Height=40, ResizeMethod=abi.ImageOpsFit)
    outs, status = check_against_per_image(cuda_lib, xb, files, opts(**fit))
    assert status[:3] == [0] * 3 and status[3] != 0 and status[4] != 0
    assert xb.stats()["grid_items"] == 3
    outs, status = check_against_per_image(cuda_lib, xb, gifs, opts(EncodeTimeout_ns=0, **fit))
    assert all(s != 0 for s in status) and xb.stats()["grid_items"] == 0
    sizes = [len(cuda_lib.transform(g, opts(**fit))) for g in gifs]
    for cap in (min(sizes) - 1, sorted(sizes)[1], 10, 800):
        outs, status = check_against_per_image(cuda_lib, xb, gifs, opts(**fit), cap=cap)
        assert xb.stats()["grid_items"] == 3
    assert any(s != 0 for s in status)


def test_multi_transform_gif_output(cuda_lib):
    import torch
    ndev = max(1, torch.cuda.device_count())
    devices = list(range(ndev)) if ndev > 1 else [0, 0]
    m = abi.MultiBatch(cuda_lib, devices, arena_bytes=4 << 30)
    try:
        files = list(synthetic_gifs().values())
        opt = opts(Width=40, Height=40, ResizeMethod=abi.ImageOpsFit)
        outs, status = m.transform(files, opt)
        for f, o, s in zip(files, outs, status):
            assert s == 0 and o == cuda_lib.transform(f, opt)
        assert sum(m.stats(g)["grid_items"] for g in range(len(devices))) == len(files)
    finally:
        m.close()
