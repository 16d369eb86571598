"""CPU: the multi-scan JPEG streams of tests/jpeg_scan_streams.py against libjpeg-turbo (cv2) and the oracle, and the
host build of the shared multi-scan decode core (lilliput_b200/csrc/jpeg_scan_core.h, via
tests/native/jpeg_scan_sim.cpp): a decode restricted to a region of interest, with nonzero masks outside it, must
give exactly the region's coefficients of the whole-frame decode."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import jpeg_scan_streams as js

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
STREAMS = js.cases()

# what each damaged file does: (libjpeg-turbo decodes it, the oracle decodes it).  The oracle stops at the first
# corrupt Huffman code or truncated scan; libjpeg-turbo warns and fills in zeros where its whole-file read allows.
DAMAGED = {
    **{"truncated_scan%d" % s: (False, s not in (5, 7, 8, 9)) for s in range(10)},
    "missing_code": (True, False),
    "undefined_table": (False, False),
    "missing_code_sequential": (True, False),
}


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    if not shutil.which("g++") or not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("needs g++ and the CUDA headers")
    so = str(tmp_path_factory.mktemp("jscan") / "libjscan.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"),
                           "-I" + CUDA_INC, "-o", so, os.path.join(ROOT, "tests", "native", "jpeg_scan_sim.cpp"),
                           os.path.join(ROOT, "lilliput_b200", "csrc", "jpeg_parse.cpp")])
    l = C.CDLL(so)
    l.jscan_decode.restype = C.c_int
    l.jscan_decode.argtypes = [C.c_char_p, C.c_long, C.POINTER(C.c_int), C.c_void_p, C.c_long, C.POINTER(C.c_int)]

    def decode(data: bytes, roi=(0, 0, 0, 0)):
        cap = 1 << 24
        out = np.zeros(cap, dtype=np.int16)
        info = (C.c_int * 4)()
        rc = l.jscan_decode(data, len(data), (C.c_int * 4)(*roi), out.ctypes.data, cap, info)
        mx, my, nb, visits = list(info)
        mcx, mcy = (roi[2], roi[3]) if roi[2] else (mx, my)
        return rc, out[:mcx * mcy * nb * 64].reshape(mcy, mcx, nb, 64), (mx, my, nb, visits)
    return decode


def _scan_order(stream):
    """expected() in the decoder's scan order: (mcus_y, mcus_x, blocks per MCU, 64 natural)."""
    fr = stream.fr
    exp = js.expected(fr, stream.script, progressive=stream.name.split("_")[1] != "sequential" and
                      "sequential" not in stream.name)
    mx, my = fr.mcus
    parts = []
    for c, (hc, vc) in enumerate(fr.factors):
        e = exp[c].reshape(my, vc, mx, hc, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, vc * hc, 64)
        parts.append(e)
    return np.concatenate(parts, axis=2)


def test_catalogue_reaches_every_feature():
    js.check_coverage(STREAMS)


@pytest.mark.parametrize("stream", STREAMS, ids=[s.name for s in STREAMS])
def test_stream_decodes_like_libjpeg_turbo(oracle, stream):
    cv2 = pytest.importorskip("cv2")
    want = cv2.imdecode(np.frombuffer(stream.data, np.uint8), cv2.IMREAD_COLOR)
    got, _ = oracle.jpeg_decode(stream.data)
    assert want is not None and np.array_equal(got, want)


@pytest.mark.parametrize("stream", STREAMS, ids=[s.name for s in STREAMS])
def test_core_whole_frame_and_windows(sim, stream):
    rc, full, (mx, my, nb, _) = sim(stream.data)
    assert rc == 0
    assert np.array_equal(full, _scan_order(stream).astype(np.int16))
    rng = np.random.default_rng(len(stream.data))
    rois = [(0, 0, 1, 1), (mx - 1, my - 1, 1, 1), (0, 0, mx, 1), (0, my - 1, mx, 1)]
    for _ in range(4):
        x0, y0 = int(rng.integers(0, mx)), int(rng.integers(0, my))
        rois.append((x0, y0, int(rng.integers(1, mx - x0 + 1)), int(rng.integers(1, my - y0 + 1))))
    for x0, y0, w, h in rois:
        rc, part, _ = sim(stream.data, (x0, y0, w, h))
        assert rc == 0 and np.array_equal(part, full[y0:y0 + h, x0:x0 + w]), (x0, y0, w, h)


@pytest.mark.parametrize("name,data", js.damaged(), ids=[d[0] for d in js.damaged()])
def test_damaged_streams(oracle, name, data):
    cv2 = pytest.importorskip("cv2")
    ref = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR) is not None
    try:
        oracle.jpeg_decode(data)
        mine = True
    except RuntimeError:
        mine = False
    assert (ref, mine) == DAMAGED[name]


def test_over_budget_file_counts_its_block_visits(sim):
    rc, _, (_, _, _, visits) = sim(js.over_budget(), (0, 0, 1, 1))
    assert rc == 0 and visits > 1 << 26
