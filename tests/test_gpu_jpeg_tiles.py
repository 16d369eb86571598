"""GPU: decoded JPEG pixels, bit-exact against the oracle, at the tile edges of jpeg_idct_color_kernel.

Per image (opencv_decoder_read_data), every case of tests/jpeg_decode_cases.py: one, two and three spans, one to
ten bands, widths 1 to 4, in every sampling, through both entropy decoders of the per-image path (the parallel decoder
for plain files, the multi-scan decoder for restart and progressive files).

Batch (lp_batch_stage + lp_batch_run): the decoded Fit crop windows themselves, each against the oracle's full
decode cut to that window, and the resized frames against the oracle's Fit, over crops that cut left / right and
top / bottom, windows off the 16-pixel grid, at the image edges, the same-size copy, ImageOpsResize and windows of
several spans, with every sampling and restart files next to plain ones in one chunk.
"""
import numpy as np
import pytest

from lilliput_b200 import abi
from tests import jpeg_decode_cases as jc

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")

CASES = jc.cases()


def _diff(got, want):
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    d = np.abs(got.astype(int) - want.astype(int))
    ys, xs = np.nonzero(d.reshape(d.shape[0], d.shape[1], -1).max(axis=2))
    return f"{len(ys)} pixels differ, by up to {d.max()}, first at (x={xs[0]}, y={ys[0]})"


@pytest.mark.parametrize("case", CASES, ids=[c.label for c in CASES])
def test_decode_matches_oracle(cuda_lib, oracle, case):
    data = jc.encode(case)
    want, _ = oracle.jpeg_decode(data)
    got = cuda_lib.decode(data)
    assert got.shape == want.shape and np.array_equal(got, want), _diff(got, want)


def _batch_files(W, H, seed):
    """Every colour sampling twice, plain and with restart markers, interleaved: one chunk mixes them all."""
    rng = np.random.default_rng(seed)
    rst = ("rst1", "rst3", "rstrow")
    cases = []
    for k, s in enumerate(jc.COLOR_SAMPLINGS):
        for mode in ("plain", rst[k % 3]):
            cases.append(jc.Case(s, W, H, jc.CONTENTS[len(cases) % 3], mode, int(rng.integers(30, 101))))
    return cases, [jc.encode(c, seed) for c in cases]


@pytest.mark.parametrize("geom", jc.BATCH_GEOMETRIES, ids=[f"{g[0]}x{g[1]}-{g[4]}-{g[2]}x{g[3]}" for g in jc.BATCH_GEOMETRIES])
def test_batch_decoded_windows_and_resized_frames(cuda_lib, oracle, geom):
    W, H, dw, dh, method = geom
    cases, files = _batch_files(W, H, W * 31 + H)
    n = len(files)
    if method == "fit":
        ew, eh = oracle.expected_size(W, H, dw, dh)
        crop = oracle.fit_rect(W, H, ew, eh)
    else:
        ew, eh, crop = dw, dh, (0, 0, W, H)
    win = jc.batch_window("444", W, H, crop)  # the window does not depend on the sampling, its tiles do
    # lp_batch sizes its restart-marker scratch from max_in_bytes (one entry per 64 bytes) and refuses a file whose
    # restart intervals no longer fit; leave room for one entry per interval, so that no file is refused
    intervals = sum(-(-jc.mcus(c) // jc.restart_interval(c)) for c in cases if c.mode.startswith("rst"))
    b = abi.Batch(cuda_lib, 0, n, W, H, dw, dh, 85, max_in_bytes=sum(map(len, files)) + 64 * intervals + 4096,
                  resize_method=abi.ImageOpsFit if method == "fit" else abi.ImageOpsResize)
    try:
        assert b.stage(files) == [0] * n
        b.run()
        frames = b.decoded_windows(n, win.h)
        resized = b.resized_frames(n, ew, eh)
    finally:
        b.close()
    # rows of a window are padded to 16 bytes; a window of whole rows is packed
    assert frames.shape[2] == win.row_stride, (frames.shape, win)
    assert win.row_stride == (W * 3 if win.w == W else -(-win.w * 3 // 16) * 16)
    bad = []
    for i, (case, data) in enumerate(zip(cases, files)):
        dec, _ = oracle.jpeg_decode(data)
        got = frames[i, :, :win.w * 3].reshape(win.h, win.w, 3)
        want = dec[win.y0:win.y0 + win.h, win.x0:win.x0 + win.w]
        if not np.array_equal(got, want):
            bad.append(f"{case.label} window {win}: {_diff(got, want)}")
        want_r = oracle.fit(dec, ew, eh) if method == "fit" else oracle.resize(dec, ew, eh)
        if not np.array_equal(resized[i], want_r):
            bad.append(f"{case.label} resized: {_diff(resized[i], want_r)}")
    assert bad == []
