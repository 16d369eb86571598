"""CPU: progressive JPEG output (lilliput_b200/csrc/jpeg_prog_core.h), compiled for the host by
tests/native/jpeg_prog_sim.cpp and fed with the quantised coefficients that oracle/oracle_jpeg_enc.c codes (read back
from its baseline file).

The contract is byte identity with what the reference writes for JpegProgressive: OpenCV's JPEG writer with
IMWRITE_JPEG_PROGRESSIVE, i.e. libjpeg-turbo's jpeg_simple_progression script with optimize_coding.  The cv2 wheel
bundles libjpeg-turbo, whose output is compared live; tests/golden/jpeg_progressive_golden.npz pins a small set of
its files so that a change in that library shows up as a fixture mismatch."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.jpeg_progressive_cases import image, matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "jpeg_progressive_golden.npz")


@pytest.fixture(scope="module")
def progressive(tmp_path_factory, oracle):
    so = str(tmp_path_factory.mktemp("jprog") / "libjprog.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "native", "jpeg_prog_sim.cpp")])
    l = C.CDLL(so)
    l.jprog_encode.restype = C.c_long
    l.jprog_encode.argtypes = [C.c_char_p, C.c_long, C.c_void_p, C.c_long]

    def encode(img: np.ndarray, q: int) -> bytes:
        base = oracle.jpeg_encode(img, q)
        cap = 2 * len(base) + (1 << 16)
        out = (C.c_uint8 * cap)()
        n = l.jprog_encode(base, len(base), out, cap)
        assert n > 0
        return bytes(out[:n])
    return encode


def _cv2_progressive(img, q):
    cv2 = pytest.importorskip("cv2")
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    assert ok
    return enc.tobytes()


def _first_diff(a: bytes, b: bytes):
    return next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))


@pytest.mark.parametrize("w,h", sorted({(c[1], c[2]) for c in matrix()}))
def test_matches_libjpeg_turbo(progressive, w, h):
    for content, cw, chh, ch, q in matrix():
        if (cw, chh) != (w, h):
            continue
        img = image(content, w, h, ch)
        want, got = _cv2_progressive(img, q), progressive(img, q)
        assert got == want, (content, w, h, ch, q, len(got), len(want), _first_diff(got, want))


def test_markers_follow_the_scan_script(progressive):
    """SOF2, one DHT per table a scan uses (none for DC refinement), the scan parameters of jpeg_simple_progression."""
    for ch, script in [(3, [(3, 0, 0, 0, 1), (1, 1, 5, 0, 2), (1, 1, 63, 0, 1), (1, 1, 63, 0, 1), (1, 6, 63, 0, 2),
                            (1, 1, 63, 2, 1), (3, 0, 0, 1, 0), (1, 1, 63, 1, 0), (1, 1, 63, 1, 0), (1, 1, 63, 1, 0)]),
                       (1, [(1, 0, 0, 0, 1), (1, 1, 5, 0, 2), (1, 6, 63, 0, 2), (1, 1, 63, 2, 1), (1, 0, 0, 1, 0),
                            (1, 1, 63, 1, 0)])]:
        data = progressive(image("noise", 40, 24, ch), 80)
        o, scans, dht_before, dhts = 2, [], [], 0
        while data[o + 1] != 0xDA or len(scans) < len(script):
            m, ln = data[o + 1], int.from_bytes(data[o + 2:o + 4], "big")
            if m == 0xC0:
                pytest.fail("baseline SOF in a progressive file")
            if m == 0xC4:
                dhts += 1
            if m == 0xDA:
                ns = data[o + 4]
                ss, se, a = data[o + 5 + 2 * ns:o + 8 + 2 * ns]
                scans.append((ns, ss, se, a >> 4, a & 15))
                dht_before.append(dhts)
                dhts = 0
                o += 2 + ln
                while not (data[o] == 0xFF and data[o + 1] not in (0x00,) and not 0xD0 <= data[o + 1] <= 0xD7):
                    o += 1
                if data[o + 1] == 0xD9:
                    break
                continue
            o += 2 + ln
        assert scans == script
        want = [2 if s[0] == 3 and s[3] == 0 else 0 if s[1] == 0 and s[3] else 1 for s in script]
        assert dht_before == want


def test_golden_fixture(progressive):
    """Files libjpeg-turbo wrote when the fixture was made: this coder still gives them, and so does the cv2 here."""
    g = np.load(GOLDEN)
    names = sorted(k[:-4] for k in g.files if k.endswith("_img"))
    assert names
    try:
        import cv2  # noqa: F401
    except ImportError:
        cv2 = None
    for name in names:
        img, want, q = g[name + "_img"], g[name + "_jpg"].tobytes(), int(g[name + "_q"])
        assert progressive(img, q) == want, name
        if cv2 is not None:
            assert _cv2_progressive(img, q) == want, f"{name}: cv2's libjpeg-turbo no longer writes the fixture's bytes"


def test_reference_library_agrees(progressive, ref_lib):
    """Where oracle/_ref is built: the reference's own encoder (libjpeg-turbo 3.1.0) writes the same bytes."""
    from lilliput_b200 import abi
    for content, w, h, ch, q in matrix()[::7]:
        if w * h > 300 * 300:
            continue
        img = image(content, w, h, ch)
        want = ref_lib.encode(".jpg", img, {abi.JpegQuality: q, abi.JpegProgressive: 1})
        assert progressive(img, q) == want, (content, w, h, ch, q)
