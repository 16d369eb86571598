"""GPU: WebP sources in the heterogeneous batch (lp_xbatch_transform, csrc/xbatch.cu + webp_decode_batch of
csrc/webp_decode.cu): stills of every kind and animations, every frame of every file decoded and composited on the device.

Every item is compared with per-image lp_transform of the same library (status and bytes), and grid_items is asserted
exactly, so a silent hand-over to the per-image path cannot pass.  One check is made against something other than
ourselves: the per-frame decodes composited in numpy with the oracle's blend and Fit, then encoded by the host build of
the same VP8 encoder, must give the batch's VP8 payloads, and libwebp must read the batch's alpha as the composite's."""
import io
import struct

import numpy as np
import pytest

from lilliput_b200 import abi
from oracle import oracle
from tests import vp8l_streams as vs
from tests.test_gpu_xbatch import check_against_per_image
from tests.webp_util import chunks_of, frames_of, libwebp_decode, pillow_animation, vp8_cpu_encode, vp8_cpu_lib, vp8l_cpu_encode

pytestmark = pytest.mark.gpu
T = 10**12
Q = 80


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


@pytest.fixture(scope="module")
def cpu():
    return vp8_cpu_lib()


def webp_opt(**kw):
    kw.setdefault("EncodeTimeout_ns", T)
    kw.setdefault("EncodeOptions", {abi.WebpQuality: Q})
    return abi.ImageOptions(FileType=".webp", **kw)


def jpeg_opt(**kw):
    return abi.ImageOptions(FileType=".jpeg", EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T, **kw)


FIT = dict(Width=40, Height=40, ResizeMethod=abi.ImageOpsFit)
RESIZE = dict(Width=50, Height=23, ResizeMethod=abi.ImageOpsResize)


# ---------------------------------------------------------------- hand-built containers

def u24(v):
    return int(v).to_bytes(3, "little")


def lossy_frame(w, h, seed, alpha=None):
    """ALPH? + VP8 chunks of one w x h frame; alpha: None, or a w x h plane stored raw."""
    out = b""
    if alpha is not None:
        out += vs.chunk(b"ALPH", b"\x00" + np.ascontiguousarray(alpha, np.uint8).tobytes())
    return out + vs.chunk(b"VP8 ", vs.lossy_payload(w, h, seed))


def lossless_frame(cpu, w, h, seed, opaque=False):
    rng = np.random.default_rng(seed)
    img = (rng.integers(0, 256, (h, w, 4)) // 48 * 48).astype(np.uint8)
    if opaque:  # three channels: no alpha hint in the VP8L header
        img = img[:, :, :3]
    return vs.chunk(b"VP8L", vp8l_cpu_encode(cpu, img))


def anmf(x, y, w, h, image_chunks, duration=50, dispose=False, blend=True):
    flags = (1 if dispose else 0) | (0 if blend else 2)
    return vs.chunk(b"ANMF", u24(x // 2) + u24(y // 2) + u24(w - 1) + u24(h - 1) + u24(duration) + bytes([flags]) + image_chunks)


def animation(cw, ch, frames, alpha=True, bg=0xFF204080, loops=0, icc=None):
    flags = 0x02 | (0x10 if alpha else 0) | (0x20 if icc is not None else 0)
    body = vs.vp8x(cw, ch, flags)
    if icc is not None:
        body += vs.chunk(b"ICCP", icc)
    body += vs.chunk(b"ANIM", struct.pack("<IH", bg, loops))
    return vs.riff(body + b"".join(frames))


def icc_profile(n=400, seed=5):
    """Bytes shaped like an ICC profile as far as the WebP writer looks: the big-endian size field matches."""
    b = bytearray(np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes())
    b[0:4] = n.to_bytes(4, "big")
    return bytes(b)


def _plane(seed, w, h, lo=0):
    return np.random.default_rng(seed).integers(lo, 256, (h, w), dtype=np.uint8)


def hand_built(cpu):
    W, H = 64, 48
    full = lambda s, a=True: anmf(0, 0, W, H, lossy_frame(W, H, s, _plane(s, W, H, 128) if a else None))  # noqa: E731
    cases = {}
    # frames touching the right and bottom edges (even offsets: the container stores x / 2, y / 2)
    cases["edges"] = animation(W, H, [full(1), anmf(W - 18, H - 14, 18, 14, lossy_frame(18, 14, 2, _plane(2, 18, 14))),
                                      anmf(W - 16, 0, 16, H, lossy_frame(16, H, 3), dispose=True),
                                      anmf(0, H - 6, W, 6, lossless_frame(cpu, W, 6, 4))])
    cases["one_pixel_frames"] = animation(W, H, [full(5), anmf(0, 0, 1, 1, lossy_frame(1, 1, 6, _plane(6, 1, 1))),
                                                 anmf(W - 2, H - 2, 1, 1, lossless_frame(cpu, 1, 1, 7)),
                                                 anmf(30, 20, 1, 1, lossy_frame(1, 1, 8), dispose=True, blend=False),
                                                 anmf(W - 1 - 1, H - 1 - 1, 1, 1, lossless_frame(cpu, 1, 1, 9), dispose=True)])
    combos = []
    for k, (d, b) in enumerate([(False, True), (True, True), (False, False), (True, False)]):
        combos.append(anmf(8 + 4 * k, 6 + 2 * k, 30, 24, lossy_frame(30, 24, 20 + k, _plane(20 + k, 30, 24)), dispose=d, blend=b))
        combos.append(anmf(2 * k, 4, 40, 30, lossless_frame(cpu, 40, 30, 30 + k), dispose=d, blend=b))
    cases["blend_dispose"] = animation(W, H, [full(10)] + combos)
    clear = np.zeros((24, 32), np.uint8)
    cases["transparent_over_opaque"] = animation(W, H, [full(11, a=False), anmf(10, 10, 32, 24, lossy_frame(32, 24, 12, clear)),
                                                        anmf(10, 10, 32, 24, lossy_frame(32, 24, 13, clear), blend=False),
                                                        full(14, a=False)])
    cases["durations"] = animation(W, H, [anmf(0, 0, W, H, lossy_frame(W, H, 15), duration=0),
                                          anmf(4, 4, 20, 20, lossy_frame(20, 20, 16), duration=0xFFFFFF),
                                          anmf(0, 0, W, H, lossy_frame(W, H, 17), duration=1)], alpha=False)
    cases["loops_bg"] = animation(W, H, [full(18), anmf(6, 6, 20, 20, lossy_frame(20, 20, 19, _plane(19, 20, 20)))],
                                  bg=0x80FF0000, loops=7)
    cases["loops_max"] = animation(W, H, [full(21), full(22)], bg=0x00000000, loops=65535)
    cases["opaque_3ch"] = animation(W, H, [anmf(0, 0, W, H, lossy_frame(W, H, 23)), anmf(8, 8, 30, 20, lossy_frame(30, 20, 24)),
                                           anmf(16, 0, 20, 20, lossless_frame(cpu, 20, 20, 25, opaque=True), dispose=True),
                                           anmf(0, 10, W, 20, lossy_frame(W, 20, 26), blend=False)], alpha=False)
    cases["icc"] = animation(W, H, [full(27), full(28)], icc=icc_profile())
    return cases


def test_hand_built_animations(cuda_lib, xb, cpu):
    cases = hand_built(cpu)
    files = list(cases.values())
    for f in files:  # the per-image decoder takes every one of them
        assert cuda_lib.webp_frames(f, decode=False)[3] == 0
    for kw in (FIT, RESIZE, dict(Width=64, Height=48, ResizeMethod=abi.ImageOpsResize)):
        outs, status = check_against_per_image(cuda_lib, xb, files, webp_opt(**kw))
        assert status == [0] * len(files), dict(zip(cases, status))
        st = xb.stats()
        assert st["grid_items"] == len(files) and st["fallback_items"] == 0, st
        k = list(cases).index("icc")
        assert dict(chunks_of(outs[k]))[b"ICCP"] == icc_profile()
        k = list(cases).index("loops_bg")
        assert dict(chunks_of(outs[k]))[b"ANIM"] == struct.pack("<IH", 0x80FF0000, 7)


def test_hand_built_stills_with_profile(cuda_lib, xb, cpu):
    """Stills carrying an ICC profile, lossless or lossy + ALPH: to WebP the profile travels into the output."""
    icc = icc_profile(300, 9)
    alpha = vs.riff(vs.vp8x(33, 21, 0x30) + vs.chunk(b"ICCP", icc) + lossy_frame(33, 21, 40, _plane(40, 33, 21)))
    lossless = vs.riff(vs.vp8x(40, 30, 0x30) + vs.chunk(b"ICCP", icc) + lossless_frame(cpu, 40, 30, 41))
    bad_icc = vs.riff(vs.vp8x(40, 30, 0x20) + vs.chunk(b"ICCP", b"\0\0\0\5" + icc[4:]) + vs.chunk(b"VP8 ", vs.lossy_payload(40, 30, 42)))
    files = [alpha, lossless, bad_icc]
    for opt in (webp_opt(**FIT), jpeg_opt(**FIT)):
        outs, status = check_against_per_image(cuda_lib, xb, files, opt)
        assert status == [0, 0, 0] and xb.stats()["grid_items"] == 3
        if opt.FileType == ".webp":
            assert dict(chunks_of(outs[0]))[b"ICCP"] == icc and dict(chunks_of(outs[1]))[b"ICCP"] == icc
            assert b"ICCP" not in dict(chunks_of(outs[2]))


# ---------------------------------------------------------------- Pillow (libwebp's WebPAnimEncoder: sub-rectangle frames)

def _frames(seed, w, h, n, alpha):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    out = []
    for k in range(n):
        img = np.zeros((h, w, 4), np.uint8)
        img[:, :, 0] = (x * 255 // max(w - 1, 1)).astype(np.uint8)
        img[:, :, 1] = (y * 255 // max(h - 1, 1)).astype(np.uint8)
        img[:, :, 2] = 90
        img[:, :, 3] = 255
        cx, cy = int(rng.integers(0, w)), int(rng.integers(0, h))
        m = (x - cx) ** 2 + (y - cy) ** 2 < (min(w, h) // 4) ** 2
        img[m, :3] = rng.integers(0, 256, 3)
        if alpha:
            img[:, :, 3] = np.where(m, 255, 60 + 40 * (k % 3)).astype(np.uint8)
        out.append(img)
    return out


def pillow_webp(frames, **kw):
    from PIL import Image
    ims = [Image.fromarray(np.ascontiguousarray(f[:, :, [2, 1, 0, 3]])) for f in frames]
    buf = io.BytesIO()
    ims[0].save(buf, "WEBP", save_all=True, append_images=ims[1:], duration=kw.pop("duration", 40), loop=kw.pop("loop", 0), **kw)
    return buf.getvalue()


def pillow_corpus():
    pytest.importorskip("PIL")
    files = {}
    for k, (w, h) in enumerate([(96, 64), (70, 50), (33, 47)]):
        files[f"lossy_alpha_{w}x{h}"] = pillow_webp(_frames(100 + k, w, h, 5, True), quality=70)
        files[f"lossless_{w}x{h}"] = pillow_webp(_frames(200 + k, w, h, 4, True), lossless=True)
        files[f"mixed_{w}x{h}"] = pillow_webp(_frames(300 + k, w, h, 5, True), allow_mixed=True, quality=60)
        from PIL import Image
        rgb = [Image.fromarray(np.ascontiguousarray(f[:, :, 2::-1])) for f in _frames(400 + k, w, h, 4, False)]
        buf = io.BytesIO()
        rgb[0].save(buf, "WEBP", save_all=True, append_images=rgb[1:], duration=[30, 60, 90, 120], loop=2, quality=75)
        files[f"opaque_{w}x{h}"] = buf.getvalue()
    return files


def test_pillow_animations(cuda_lib, xb):
    files = pillow_corpus()
    data = list(files.values())
    for f in data:
        n, _, _, _ = pillow_animation(f)
        assert n >= 4
    for kw in (FIT, RESIZE):
        outs, status = check_against_per_image(cuda_lib, xb, data, webp_opt(**kw))
        assert status == [0] * len(data), dict(zip(files, status))
        st = xb.stats()
        assert st["grid_items"] == len(data) and st["fallback_items"] == 0, st
    # the output is an animation libwebp reads back with the source's frame count, loop count and durations
    k = list(files).index("opaque_70x50")
    n, loop, durations, size = pillow_animation(outs[k])
    assert (n, loop, durations, size) == (4, 2, [30, 60, 90, 120], (50, 23))


# ---------------------------------------------------------------- stills

def test_still_catalogue_both_sinks(cuda_lib, xb):
    """The well-formed VP8L / ALPH catalogue (lossless stills, lossy + ALPH stills, one-frame animations)."""
    files = [c.data for c in vs.cases()]
    for opt in (jpeg_opt(Width=16, Height=16, ResizeMethod=abi.ImageOpsFit), webp_opt(Width=24, Height=12, ResizeMethod=abi.ImageOpsResize)):
        _, status = check_against_per_image(cuda_lib, xb, files, opt)
        assert status == [0] * len(files)
        st = xb.stats()
        assert st["grid_items"] == len(files) and st["fallback_items"] == 0, st


def test_routing_gates(cuda_lib, xb, cpu):
    """What stays per image: animations to JPEG, NoResize, MaxEncodeFrames, a zero encode budget (animations, and
    stills beyond the simple lossy ones to WebP), lossless WebP output."""
    anim = hand_built(cpu)["blend_dispose"]
    alpha_still = vs.alpha_still(33, 17, b"\x00" + _plane(1, 33, 17).tobytes(), vs.lossy_payload(33, 17, 3))
    simple = vs.riff(vs.chunk(b"VP8 ", vs.lossy_payload(40, 30, 4)))
    files = [anim, alpha_still, simple]
    for opt, grid in [(jpeg_opt(**FIT), 2),
                      (webp_opt(Width=40, Height=40, ResizeMethod=abi.ImageOpsNoResize), 0),
                      (webp_opt(MaxEncodeFrames=2, **FIT), 2),
                      (webp_opt(EncodeOptions={abi.WebpQuality: 101}, **FIT), 0),
                      (webp_opt(**FIT), 3)]:
        check_against_per_image(cuda_lib, xb, files, opt)
        assert xb.stats()["grid_items"] == grid, (opt, xb.stats())
    # (the simple lossy still keeps its earlier routing under a zero budget: not compared here)
    check_against_per_image(cuda_lib, xb, files[:2], webp_opt(EncodeTimeout_ns=0, **FIT))
    assert xb.stats()["grid_items"] == 0


# ---------------------------------------------------------------- damaged files

def _refused(cuda_lib, f):
    return cuda_lib.webp_frames(f)[3] != 0


def test_damaged_frames_hand_over_only_their_file(cuda_lib, xb, cpu):
    W, H = 64, 48
    good = hand_built(cpu)
    # a truncated middle frame: a lossy payload cut inside its token partition (the container stays well-formed)
    truncated = None
    for d in vs.damaged_cases():
        if d.group not in ("trunc_vp8", "trunc_vp8_partitions") or not _refused(cuda_lib, d.data):
            continue
        tag, payload, _ = frames_of(d.data)[0]
        if tag != b"VP8 " or len(payload) < 10:
            continue
        w, h = (payload[6] | (payload[7] << 8)) & 0x3FFF, (payload[8] | (payload[9] << 8)) & 0x3FFF
        if w > W or h > H:
            continue
        f = animation(W, H, [anmf(0, 0, W, H, lossy_frame(W, H, 50)), anmf(0, 0, w, h, vs.chunk(b"VP8 ", payload)),
                             anmf(0, 0, W, H, lossy_frame(W, H, 51))])
        if _refused(cuda_lib, f) and cuda_lib.webp_frames(f, decode=False)[3] == 0:
            truncated = f
            break
    assert truncated is not None
    # a bad ALPH in a middle frame: a VP8L-coded plane whose stream is garbage (a failed LAST frame reads as the end of
    # the animation per image: lp_transform writes the frames before it)
    bad_alph = None
    for seed in range(20):
        junk = b"\x01" + np.random.default_rng(seed).integers(0, 256, 24, dtype=np.uint8).tobytes()
        f = animation(W, H, [anmf(0, 0, W, H, lossy_frame(W, H, 52)),
                             anmf(4, 4, 20, 20, vs.chunk(b"ALPH", junk) + vs.chunk(b"VP8 ", vs.lossy_payload(20, 20, 53))),
                             anmf(0, 0, W, H, lossy_frame(W, H, 54))])
        if _refused(cuda_lib, f):
            bad_alph = f
            break
    assert bad_alph is not None
    files = list(good.values()) + [truncated, bad_alph]
    _, status = check_against_per_image(cuda_lib, xb, files, webp_opt(**FIT))
    assert status[:-2] == [0] * (len(files) - 2) and status[-2] != 0 and status[-1] != 0
    st = xb.stats()
    assert st["grid_items"] == len(files) - 2 and st["fallback_items"] == 2, st


# ---------------------------------------------------------------- against the oracle

def composite(cuda_lib, data, ow, oh):
    """The per-frame device decodes (webp_decoder_*) composited in numpy as ImageOps does (blend over / copy, Fit,
    clear), with the oracle's blend and resize."""
    info, frames, metas, rc = cuda_lib.webp_frames(data)
    assert rc == 0
    ch = 4 if info["pixel_type"] == abi.CV_8UC4 else 3
    canvas = np.zeros((info["height"], info["width"], ch), np.uint8)
    out = []
    for f, m in zip(frames, metas):
        x, y, h, w = m["x"], m["y"], f.shape[0], f.shape[1]
        region = canvas[y:y + h, x:x + w]
        canvas[y:y + h, x:x + w] = oracle.blend_over(f, region) if m["blend"] == 0 else f
        out.append(oracle.fit(canvas, ow, oh))
        if m["dispose"] == 1:
            canvas[y:y + h, x:x + w] = 0
    return out


def test_frames_against_the_oracle(cuda_lib, xb, cpu):
    cases = hand_built(cpu)
    names = ["blend_dispose", "edges", "transparent_over_opaque", "opaque_3ch"]
    files = [cases[k] for k in names]
    outs, status = xb.transform(files, webp_opt(**FIT), out_cap=1 << 22)
    assert status == [0] * len(files) and xb.stats()["grid_items"] == len(files)
    for name, f, out in zip(names, files, outs):
        want = composite(cuda_lib, f, 40, 40)
        got = frames_of(out)
        assert len(got) == len(want), name
        for k, ((tag, vp8, alph), fit) in enumerate(zip(got, want)):
            assert tag == b"VP8 " and vp8 == vp8_cpu_encode(cpu, fit, Q), f"{name} frame {k}: VP8 payload"
            if fit.shape[2] == 4 and alph is not None:
                dec = libwebp_decode(vs.alpha_still(40, 40, alph, vp8))
                assert np.array_equal(dec[:, :, 3], fit[:, :, 3]), f"{name} frame {k}: alpha"
            elif fit.shape[2] == 4:
                assert (fit[:, :, 3] == 255).all(), f"{name} frame {k}: no ALPH for a frame with transparency"
