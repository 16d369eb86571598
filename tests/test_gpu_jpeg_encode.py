"""GPU: baseline JPEG output of the device encoder (csrc/jpeg_encode.cu: jpeg_fdct_quant_kernel, jpeg_entropy_kernel),
byte-identical to what the reference writes -- OpenCV's JPEG writer over libjpeg-turbo, compared live through the cv2
here -- in every way the project launches it:

- per image (lp_encode), over the whole case matrix of tests/jpeg_encode_cases.py;
- many frames per launch (lp_jpeg_encode_dev): padded row and image strides, an out_cap that fits the largest file
  exactly and one a byte short of it;
- lp_batch's encode launches: one per (channel count, output size) of a chunk, in slot order or through its image map;
- lp_xbatch's JPEG sink, gray and colour;
- the encoder constants past their cache bound (built per call, freed in stream order)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests import jpeg_encode_cases as jc

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 10**12


def _first_diff(a, b):
    return next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))


def _check_cases(lib, cases):
    for case in cases:
        img = jc.case_image(case)
        got, want = lib.encode(".jpg", img, jc.encode_options(case[4])), jc.reference(img, case[4])
        assert got == want, (case, len(got), len(want), _first_diff(got, want))


@pytest.mark.parametrize("h", jc.HEIGHTS)
def test_edge_matrix(cuda_lib, h):
    _check_cases(cuda_lib, [c for c in jc.edge_matrix() if c[2] == h])


def test_quality_sweep(cuda_lib):
    _check_cases(cuda_lib, jc.quality_sweep())


def test_launch_shapes(cuda_lib):
    _check_cases(cuda_lib, jc.launch_shapes())


# ---------------------------------------------------------------- many frames per launch


@pytest.fixture(scope="module")
def dev(cuda_lib):
    l = cuda_lib.l
    l.lp_dev_alloc.restype = C.c_void_p
    l.lp_dev_alloc.argtypes = [C.c_size_t]
    l.lp_dev_free.argtypes = [C.c_void_p]
    for f in (l.lp_memcpy_h2d, l.lp_memcpy_d2h):
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    l.lp_jpeg_encode_dev.restype = C.c_int
    l.lp_jpeg_encode_dev.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                     C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    return l


def encode_dev(l, frames, q, out_cap, row_pad=0, img_pad=0):
    """frames: n arrays of one (h, w[, ch]).  row_pad / img_pad: bytes of 0xA5 after every row / frame, strides the
    encoder must honour.  Returns the n files (b"" where out_len is 0)."""
    n = len(frames)
    h, w = frames[0].shape[:2]
    ch = 1 if frames[0].ndim == 2 else frames[0].shape[2]
    row = w * ch + row_pad
    img = row * h + img_pad
    host = np.full(n * img, 0xA5, np.uint8)
    for i, f in enumerate(frames):
        host[i * img: i * img + row * h].reshape(h, row)[:, : w * ch] = f.reshape(h, w * ch)
    d_frames, d_out, d_len = l.lp_dev_alloc(host.size), l.lp_dev_alloc(n * out_cap), l.lp_dev_alloc(4 * n)
    assert d_frames and d_out and d_len
    try:
        assert l.lp_memcpy_h2d(d_frames, host.ctypes.data, host.size) == 0
        assert l.lp_jpeg_encode_dev(d_frames, img, row, w, h, ch, q, n, d_out, out_cap, d_len, None) == 0
        lens = np.zeros(n, np.uint32)
        out = np.zeros(n * out_cap, np.uint8)
        assert l.lp_memcpy_d2h(lens.ctypes.data, d_len, 4 * n) == 0
        assert l.lp_memcpy_d2h(out.ctypes.data, d_out, out.size) == 0
        return [out[i * out_cap: i * out_cap + int(lens[i])].tobytes() for i in range(n)]
    finally:
        for p in (d_frames, d_out, d_len):
            l.lp_dev_free(p)


LAUNCHES = [  # (w, h, ch, n, q)
    (37, 29, 3, 1, 85),
    (64, 48, 1, 2, 50),
    (33, 17, 4, 33, 95),
    (272, 256, 3, 64, 75),   # 272 MCUs per image: a second 256-MCU scan chunk
    (136, 136, 1, 33, 100),  # 289 MCUs
    (1, 1, 3, 64, 100),
]


@pytest.mark.parametrize("case", LAUNCHES, ids=lambda c: "x".join(map(str, c)))
def test_many_frames_per_launch(dev, case):
    """Distinct frames of every content in one launch: each file is cv2's, on packed and on padded strides, with an
    out_cap that fits the largest file exactly.  One byte less: the largest files get out_len 0, the others their
    bytes."""
    w, h, ch, n, q = case
    frames = [jc.image(jc.CONTENTS[i % len(jc.CONTENTS)], w, h, ch, seed=i) for i in range(n)]
    want = [jc.reference(f, q) for f in frames]
    cap = max(map(len, want))
    assert encode_dev(dev, frames, q, cap) == want
    assert encode_dev(dev, frames, q, cap, row_pad=13, img_pad=77) == want
    short = encode_dev(dev, frames, q, cap - 1, row_pad=3, img_pad=5)
    assert short == [b"" if len(x) == cap else x for x in want]


def test_stuffed_files_at_exact_and_short_caps(dev):
    """Saturated noise (a stuffed 0xFF every few bytes): the stuffed length, not the packed one, decides the fit."""
    frames = [jc.image("binary", 160, 96, 3, seed=s) for s in range(5)]
    want = [jc.reference(f, 100) for f in frames]
    for i, x in enumerate(want):
        got = encode_dev(dev, frames, 100, len(x))
        assert got[i] == x
        assert all(g == (v if len(v) <= len(x) else b"") for g, v in zip(got, want))
        got = encode_dev(dev, frames, 100, len(x) - 1)
        assert got[i] == b""
        assert all(g == (v if len(v) < len(x) else b"") for g, v in zip(got, want))


# ---------------------------------------------------------------- lp_batch

Q_BATCH = 77


def _sof(data: bytes):
    """(width, height, components) of a file's frame header."""
    pos = 2
    while True:
        m, seg = data[pos + 1], int.from_bytes(data[pos + 2:pos + 4], "big")
        if m == 0xC0:
            return int.from_bytes(data[pos + 7:pos + 9], "big"), int.from_bytes(data[pos + 5:pos + 7], "big"), data[pos + 9]
        pos += 2 + seg


def _batch_files(kinds, orients, w, h, seed0):
    from tests.test_gpu_batch_gray import jpeg
    return [jpeg(seed0 + k, w, h, s, orientation=o) for k, (s, o) in enumerate(zip(kinds, orients))]


@pytest.mark.parametrize("mix", ["colour", "gray", "mixed"])
def test_batch_encodes_are_cv2s_of_its_frames(cuda_lib, mix):
    """One chunk.  All colour or all gray, unrotated: one encode launch in slot order.  Colour, gray and transposed
    (orientation 5-8, another output size under a Fit above the source) mixed: four launches through the image map.
    Every output is cv2's file of the resized frame the batch holds for that item."""
    w, h, dw, dh = 200, 120, 300, 150
    if mix == "mixed":
        kinds = ["gray", "420", "gray", "gray", "444", "gray", "420", "gray", "420", "444"]
        orients = [1, 6, 6, 8, 1, 5, 7, 2, 1, 3]
    else:
        kinds = ["420" if mix == "colour" else "gray"] * 7
        orients = [1] * 7
    files = _batch_files(kinds, orients, w, h, 900)
    b = abi.Batch(cuda_lib, 0, len(files), w, h, dw, dh, Q_BATCH, max_in_bytes=sum(map(len, files)) + (1 << 20),
                  out_cap=1 << 18, resize_method=abi.ImageOpsFit, normalize_orientation=True)
    try:
        b.stage(files)
        b.run()
        outs, status = b.fetch(len(files))
        assert status == [0] * len(files)
        slots = b.frame_slots(len(files), resized=True)
        sizes = set()
        for i, o in enumerate(outs):
            ow, oh, nc = _sof(o)
            assert nc == b.item_channels(i) == (1 if kinds[i] == "gray" else 3)
            frame = slots[i, : ow * oh * nc].reshape((oh, ow, nc) if nc == 3 else (oh, ow))
            assert o == jc.reference(frame, Q_BATCH), (i, kinds[i], orients[i], _first_diff(o, jc.reference(frame, Q_BATCH)))
            sizes.add((ow, oh, nc))
        assert len(sizes) == (4 if mix == "mixed" else 1), sizes
    finally:
        b.close()


# ---------------------------------------------------------------- lp_xbatch


def test_xbatch_jpeg_sink(cuda_lib, oracle):
    """Colour sources of two sizes that Fit to one geometry (the grid path's encode group), gray sources among them:
    each output is cv2's encode of the frame the oracle makes."""
    sizes = [(320, 240), (427, 240)] * 3
    files = [oracle.jpeg_encode(synth_image(700 + k, w, h, 3), 90) for k, (w, h) in enumerate(sizes)]
    for k in range(3):
        ok, g = cv2.imencode(".jpg", synth_image(750 + k, 300, 200, 1), [cv2.IMWRITE_JPEG_QUALITY, 90])
        files.insert(2 * k + 1, g.tobytes())
    for q in (85, 100):
        opt = abi.ImageOptions(FileType=".jpeg", Width=96, Height=96, ResizeMethod=abi.ImageOpsFit,
                               EncodeOptions={abi.JpegQuality: q}, EncodeTimeout_ns=T)
        xb = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
        try:
            outs, status = xb.transform(files, opt)
            assert status == [0] * len(files)
            assert xb.stats()["grid_items"] >= 6
        finally:
            xb.close()
        for i, (f, o) in enumerate(zip(files, outs)):
            frame = oracle.fit(oracle.jpeg_decode(f)[0], 96, 96)
            assert o == jc.reference(frame, q), (i, q)


# ---------------------------------------------------------------- constants past the cache bound

CHILD = r"""
from lilliput_b200 import abi
from tests import jpeg_encode_cases as jc
lib = abi.load_cuda()
keys = [(5 + 13 * k, 3 + 11 * k, k % 2 == 0, 1 + 5 * k) for k in range(20)]
for _ in range(2):
    for w, h, gray, q in keys:
        img = jc.image("photo", w, h, 1 if gray else 3, seed=q)
        assert lib.encode(".jpg", img, {abi.JpegQuality: q}) == jc.reference(img, q), (w, h, gray, q)
print("const-cap child ok")
"""


def test_constants_past_the_cache_bound():
    """LP_JPEG_ENC_CONST_CAP=1 (read once per process, so a child of its own): 20 distinct (size, gray, quality) keys
    twice each; all but the first take transient constants, and every file is still cv2's."""
    env = dict(os.environ, LP_JPEG_ENC_CONST_CAP="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "const-cap child ok" in r.stdout
