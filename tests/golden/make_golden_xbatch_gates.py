"""Generates tests/golden/xbatch_gates_golden.npz: the heterogeneous batch's gate table (tests/test_xbatch_gates.py) over
a corpus x option grid -- the files' bytes, the calls, and the table the harness printed for them, each compressed with
lzma (its window spans the whole corpus, so the files cut from one another cost little).  The files are stored, not
rebuilt, so the test does not depend on the encoders installed.

Every sink (.jpeg, .png, .webp at quality 85 and 101, .gif), lp_xbatch_decode_frames and lp_xbatch_decode_clips at
T = 1, 3 and 8, each over Fit (with and without NormalizeOrientation), Resize and NoResize x a zero and a non-zero
EncodeTimeout x MaxEncodeFrames 0 and 1 x MaxEncodeDuration < 0, 0 and > 0 x DisableAnimatedOutput off and on; three
renditions of mixed sinks over the same option classes; tensor items of lp_xbatch_encode_frames, sizes outside the box
included; and a small max_size.

Run in the build container, after make -C lilliput_b200/csrc:  python tests/golden/make_golden_xbatch_gates.py
"""
import lzma
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from lilliput_b200 import abi  # noqa: E402
from lilliput_b200.synth import synth_image  # noqa: E402
from tests.test_gpu_xbatch import rgb_png  # noqa: E402
from tests.test_gpu_xbatch_frames import corpus  # noqa: E402
from tests.test_gpu_xbatch_jpeg_webp import after_app0, app2, icc_profile, png_profile, with_iccp  # noqa: E402
from tests.test_xbatch_gates import build_sim, gate_table  # noqa: E402

T = 10**12
METHODS = [(abi.ImageOpsFit, 64, 48, 0), (abi.ImageOpsFit, 48, 64, 1), (abi.ImageOpsResize, 50, 40, 0),
           (abi.ImageOpsNoResize, 0, 0, 0)]
TIMING = [(timeout, frames, duration, dao) for timeout in (0, T) for frames in (0, 1) for duration in (-1, 0, T)
          for dao in (0, 1)]
SINKS = {"jpeg": (".jpeg", {abi.JpegQuality: 85}), "png": (".png", {}), "webp85": (".webp", {abi.WebpQuality: 85}),
         "webp101": (".webp", {abi.WebpQuality: 101}), "gif": (".gif", {})}
MIXED = [("jpeg", "webp85", "png"), ("gif", "webp101", "png"), ("webp85", "gif", "webp85"), ("png", "jpeg", "webp101")]
MIXED_SIZES = [(abi.ImageOpsFit, 64, 48), (abi.ImageOpsFit, 120, 90), (abi.ImageOpsResize, 30, 30)]
TENSOR_SIZES = [(1, 1), (64, 48), (100, 80), (101, 80), (100, 81), (0, 5), (50, 0)]


def files():
    # (the frames test's 300x200 RGB and 256x256 RGBA PNGs are most of its bytes; the golden PNGs below are the same kinds)
    out = [(n, b) for n, b in corpus() if n not in ("png_rgb", "png_rgba")]
    out += [("png_iccp", with_iccp(rgb_png(synth_image(40, 40, 30, 3)), png_profile())),
            ("jpeg_icc", after_app0(out[1][1], app2(1, 1, icc_profile(700))))]
    for npz in ("golden.npz", "webp_golden.npz"):
        g = np.load(os.path.join(ROOT, "tests", "golden", npz))
        out += [("golden_" + k, g[k].tobytes()) for k in g.files
                if k.startswith(("gif_", "png_", "webp_")) and g[k].dtype == np.uint8 and g[k].ndim == 1 and g[k].size < 8000]
    return out


def rend(sink, method, w, h, norm, timeout, frames, duration, dao):
    ext, eo = SINKS[sink]
    kv = " ".join(f"{k} {v}" for k, v in eo.items())
    return f"rend {ext} {method} {w} {h} {norm} {timeout} {frames} {duration} {dao} {kv}".rstrip()


def spec(names):
    items = "items " + " ".join(str(i) for i in range(len(names)))
    lines = [f"file {n}" for n in names]

    def call(mode, t, max_size, *body):
        lines.extend([f"call {mode} {t} {max_size}", *body, "run"])

    for m in METHODS:
        for tm in TIMING:
            for sink in SINKS:
                call("files", 0, 0, items, rend(sink, *m, *tm))
            for t in (0, 1, 3, 8):  # (frames: the options' sink is ignored, its fields too)
                call("frames", t, 0, items, rend("webp101", *m, *tm))
            for sink in SINKS:
                call("tensor", 0, 0, "box 100 80 3", "sizes " + " ".join(f"{w} {h}" for w, h in TENSOR_SIZES), rend(sink, *m, *tm))
    for mix in MIXED:
        for tm in TIMING:
            call("files", 0, 0, items, *[rend(s, *sz, 0, *tm) for s, sz in zip(mix, MIXED_SIZES)])
    for sink in SINKS:  # a small max_size, and four channels
        call("files", 0, 100, items, rend(sink, *METHODS[0], T, 0, 0, 0))
        call("tensor", 0, 60, "box 100 80 4", "sizes " + " ".join(f"{w} {h}" for w, h in TENSOR_SIZES), rend(sink, *METHODS[0], T, 0, 0, 0))
    for t in (0, 3):
        call("frames", t, 100, items, rend("jpeg", *METHODS[0], T, 0, 0, 0))
    return "\n".join(lines) + "\n"


def main():
    fs = files()
    names = [n for n, _ in fs]
    assert len(set(names)) == len(names)
    s = spec(names)
    with tempfile.TemporaryDirectory() as d:
        table = gate_table(build_sim(d), d, names, [b for _, b in fs], s)
    text = "\n".join(table) + "\n"
    path = os.path.join(ROOT, "tests", "golden", "xbatch_gates_golden.npz")
    def packed(b):
        return np.frombuffer(lzma.compress(b, preset=9), np.uint8)

    np.savez(path, names=np.array(names), lengths=np.array([len(b) for _, b in fs], np.int64),
             files=packed(b"".join(b for _, b in fs)), spec=packed(s.encode()), table=packed(text.encode()))
    print(f"{path}: {len(fs)} files, {sum(l.startswith('call ') for l in table)} calls, {len(table)} lines, "
          f"{os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
