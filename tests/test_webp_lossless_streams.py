"""WebP lossless (VP8L) and ALPH decoding of hand-built streams (tests/vp8l_streams.py) and of Pillow's lossless
encoder, by the host build of the decoder cores (oracle/oracle_webp.cpp over vp8l_core.h / vp8_core.h), against
libwebp (OpenCV's WebP codec) and, where it is built, the reference's own decoder: pixel for pixel where libwebp
decodes, and accept / refuse exactly where libwebp does for damaged and truncated streams."""
import ctypes
import io

import numpy as np
import pytest

from tests import vp8l_streams as vs
from tests.webp_util import frames_of, optional_reference, vp8_cpu_lib, webp_golden


@pytest.fixture(scope="module")
def lib():
    return vp8_cpu_lib()


def libwebp(data: bytes):
    """libwebp's decode of a whole file (BGR / BGRA), None when it refuses."""
    import cv2
    return cv2.imdecode(np.frombuffer(bytes(data), np.uint8), cv2.IMREAD_UNCHANGED)


def _span(payload: bytes) -> bytes:
    """The bytes the product decodes an image chunk from: the payload and its padding byte (webp_decode.cu
    image_span) -- libwebp reads on into the padding."""
    return payload + b"\0" if len(payload) & 1 else payload


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def core_decode(lib, data: bytes):
    """(status, BGR / BGRA frame) of the first frame of a file through the host cores: what the device computes."""
    tag, img, alph = frames_of(data)[0]
    if tag == b"VP8L":
        if len(img) < 5:
            return 1, None
        bits = int.from_bytes(img[1:5], "little")
        w, h = (bits & 0x3FFF) + 1, ((bits >> 14) & 0x3FFF) + 1
        arr = np.frombuffer(_span(img), np.uint8)
        out = np.zeros((h, w, 4), np.uint8)
        rc = lib.vp8l_cpu_decode(_ptr(arr), ctypes.c_size_t(arr.size), w, h, _ptr(out), 4)
        return rc, out
    arr = np.frombuffer(_span(img), np.uint8)
    w, h = ctypes.c_int(), ctypes.c_int()
    if lib.vp8_cpu_info(_ptr(arr), ctypes.c_size_t(len(img)), ctypes.byref(w), ctypes.byref(h)):
        return 1, None
    w, h = w.value, h.value
    bgr = np.zeros((h, w, 3), np.uint8)
    rc = lib.vp8_cpu_decode_bgr(_ptr(arr), ctypes.c_size_t(arr.size), _ptr(bgr), w * 3, 0, None)
    if rc or alph is None:
        return rc, bgr
    a = np.frombuffer(alph, np.uint8)
    plane = np.zeros((h, w), np.uint8)
    rc = lib.alph_cpu_decode(_ptr(a), ctypes.c_size_t(a.size), w, h, _ptr(plane))
    return rc, np.dstack([bgr, plane])


CASES = vs.cases()


def test_catalogue_reaches_every_feature():
    cov = vs.coverage()
    missing = [f for f in vs.FEATURES if not cov[f]]
    assert not missing, missing


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_stream_decodes_as_libwebp(lib, case):
    want = libwebp(case.data)
    assert want is not None, "libwebp refuses a well-formed stream"
    rc, got = core_decode(lib, case.data)
    assert rc == 0
    assert got.shape == want.shape and np.array_equal(got, want)


def test_streams_match_the_reference_decoder(lib):
    ref = optional_reference()
    if ref is None:
        pytest.skip("oracle/_ref is not built")
    for case in CASES:
        if case.kind != "vp8l":
            continue
        want = ref.decode(case.data)
        rc, got = core_decode(lib, case.data)
        assert rc == 0 and np.array_equal(got[:, :, :want.shape[2]], want), case.name


DAMAGED = vs.damaged_cases()


@pytest.mark.parametrize("group", sorted({d.group for d in DAMAGED}))
def test_damaged_streams_accepted_or_refused_as_libwebp(lib, group):
    bad = []
    for d in DAMAGED:
        if d.group != group:
            continue
        lw = libwebp(d.data) is not None
        rc, _ = core_decode(lib, d.data)
        if lw != (rc == 0):
            bad.append(f"{d.name}: libwebp {'accepts' if lw else 'refuses'}, core rc {rc}")
    assert not bad, bad[:20]


def _pillow_streams():
    from PIL import Image
    rng = np.random.default_rng(5)
    out = []
    shapes = [(1, 37), (41, 1), (17, 13), (64, 48)]
    for k, (w, h) in enumerate(shapes):
        for ncol in (2, 7, 16, 17, 256):
            pal = rng.integers(0, 256, (ncol, 4), dtype=np.uint8)
            idx = rng.integers(0, ncol, (h, w))
            out.append((f"pal{ncol}_{w}x{h}", pal[idx]))
        gx = np.linspace(0, 255, w)[None, :, None]
        gy = np.linspace(0, 255, h)[:, None, None]
        grad = np.concatenate([np.broadcast_to(gx, (h, w, 1)), np.broadcast_to(gy, (h, w, 1)),
                               np.broadcast_to((gx + gy) / 2, (h, w, 1)), np.full((h, w, 1), 200.0)], 2)
        out.append((f"gradient_{w}x{h}", grad.astype(np.uint8)))
    files = []
    for name, rgba in out:
        for q in (0, 50, 100):
            for m in (0, 3, 6):
                buf = io.BytesIO()
                Image.fromarray(rgba, "RGBA").save(buf, "WEBP", lossless=True, quality=q, method=m, exact=True)
                files.append((f"{name}_q{q}_m{m}", buf.getvalue()))
    return files


def test_pillow_lossless_sweep(lib):
    """Pillow's lossless encoder (libwebp) at quality 0 / 50 / 100 and method 0 / 3 / 6, exact, on palettes of 2 to
    256 colours and gradients, 1xN and Nx1 included: every stream decodes to libwebp's pixels."""
    bad = []
    for name, data in _pillow_streams():
        want = libwebp(data)
        rc, got = core_decode(lib, data)
        if rc or got.shape != want.shape or not np.array_equal(got, want):
            bad.append(name)
    assert not bad, bad
