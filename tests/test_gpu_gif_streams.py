"""GPU: the LZW decode kernel and the compositor of csrc/gif_decode.cu on the hand-built code streams of
tests/gif_streams.py (table full with no clear behind it, clear codes at every width, KwKwK chains, every minimum code
size, strings of thousands of pixels, frames that fill inside a round, damaged streams, odd sub-block layouts,
interlaced and off-canvas frames), through both callers of the kernels:
  per image  cuda_lib.gif_frames (lp_gif_decode_frames_host) against the oracle and the numpy ground truth;
  batch      lp_xbatch_transform with GIF and animated lossy WebP output against lp_transform, and the GIF bytes
             against the oracle's GIF -> GIF transcode."""
import numpy as np
import pytest

from lilliput_b200 import abi
from tests import gif_streams as gs
from tests.golden.make_golden_gif_encode import TIMEOUT_NS
from tests.test_gpu_xbatch import check_against_per_image
from tests.test_oracle_gif_streams import disposal_modes

pytestmark = pytest.mark.gpu
CASES = gs.cases()
FIT = 64


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=8 << 30)
    yield x
    x.close()


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_per_image_decode(cuda_lib, oracle, case):
    gf, gd, gp, grc = oracle.gif_frames(case.gif)
    ef, ed, ep, erc = cuda_lib.gif_frames(case.gif)
    assert (erc != 0) == (grc != 0) == bool(case.damage)
    assert len(ef) == len(gf) == len(case.frames)
    assert list(ed) == [d * 10 for d in gd] and list(ep) == disposal_modes(gp)
    for k in range(len(gf)):
        assert np.array_equal(ef[k], gf[k]), f"frame {k} differs from the oracle"
        assert np.array_equal(ef[k], case.frames[k]), f"frame {k} differs from the ground truth"
    if not case.damage:
        assert cuda_lib.gif_info(case.gif)["frame_count"] == len(gf)


@pytest.mark.parametrize("sink", [".gif", ".webp"])
def test_batch_decode(cuda_lib, xb, oracle, sink):
    """Every case in one call: each canvas size is one group, ~350 frames in all.  Well-formed files stay in the batch
    (grid_items); a file with a damaged stream falls back to the per-image path and gets its status."""
    files = [c.gif for c in CASES]
    if sink == ".gif":
        opt = abi.ImageOptions(FileType=".gif", Width=FIT, Height=FIT, ResizeMethod=abi.ImageOpsFit,
                               EncodeTimeout_ns=TIMEOUT_NS)
    else:
        opt = abi.ImageOptions(FileType=".webp", Width=FIT, Height=FIT, ResizeMethod=abi.ImageOpsFit,
                               EncodeOptions={abi.WebpQuality: 80}, EncodeTimeout_ns=10**12)
    outs, status = check_against_per_image(cuda_lib, xb, files, opt, cap=1 << 22)
    st = xb.stats()
    well_formed = [not c.damage for c in CASES]
    assert st["grid_items"] == sum(well_formed) and st["fallback_items"] == len(files) - sum(well_formed), st
    assert sum(len(c.frames) for c in CASES if not c.damage) >= 250
    assert all(s == 0 for s, ok in zip(status, well_formed) if ok)
    if sink != ".gif":
        return
    for c, out in zip(CASES, outs):
        if c.damage:
            continue
        ch, cw = c.frames[0].shape[:2]
        w, h = oracle.expected_size(cw, ch, FIT, FIT)
        assert out == oracle.gif_transcode(c.gif, lambda f: oracle.fit(f, w, h)), c.name
