"""GPU: the hand-built VP8 catalogue (tests/vp8_streams.py) and its coefficients past a real encoder's range through the
device decoder, per image (webp_decoder_*) and in the heterogeneous batch (lp_xbatch_transform): pixels as libwebp and
as the host build of the same cores; and an animation whose frames are such streams at unaligned offsets, some with
an ALPH plane."""
import numpy as np
import pytest

from lilliput_b200 import abi
from tests import vp8_streams as vs
from tests.test_gpu_xbatch import check_against_per_image
from tests.test_gpu_xbatch_webp import FIT, animation, anmf, webp_opt
from tests.test_webp_lossless_streams import core_decode, libwebp
from tests.webp_util import vp8_cpu_lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return vp8_cpu_lib()


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    yield x
    x.close()


def _all_cases():
    return list(vs.cases()) + [c for _, c in vs.large_coefficient_cases()]


def test_catalogue_on_the_device(cuda_lib, lib):
    bad = []
    for case in _all_cases():
        want = libwebp(case.data)
        _, frames, _, rc = cuda_lib.webp_frames(case.data)
        crc, host = core_decode(lib, case.data)
        if rc != 0 or not frames:
            bad.append(f"{case.name}: device rc {rc}")
        elif frames[0].shape != want.shape or not np.array_equal(frames[0], want):
            bad.append(f"{case.name}: pixels differ from libwebp")
        elif crc != 0 or not np.array_equal(frames[0], host):
            bad.append(f"{case.name}: pixels differ from the host cores")
    assert not bad, bad[:20]


def test_catalogue_in_the_batch(cuda_lib, xb):
    """The batch decodes lossy stills in one grid launch: every stream to PNG (lossless output, so a decode difference
    cannot hide in the encoder) exactly as per image."""
    files = [c.data for c in _all_cases()]
    opt = abi.ImageOptions(FileType=".png", Width=40, Height=40, ResizeMethod=abi.ImageOpsResize,
                           EncodeOptions={abi.PngCompression: 1}, EncodeTimeout_ns=10**12)
    _, status = check_against_per_image(cuda_lib, xb, files, opt)
    assert status == [0] * len(files)
    st = xb.stats()
    assert st["grid_items"] == len(files) and st["fallback_items"] == 0, st


def _frames():
    """(x, y, w, h, VP8 payload, ALPH payload or None) of a 96 x 80 animation: stored offsets odd (x / 2, y / 2), so
    no frame sits on the canvas's macroblock grid; every other frame carries a raw ALPH plane."""
    rng = np.random.default_rng(41)
    specs = [(0, 0, vs.Spec(96, 80, level=20)),
             (6, 10, vs.Spec(33, 21, seg=vs.Segmentation(1, 1, 0, (-10, 5, None, 20), (3, -7, 12, None),
                                                         (100, None, 30)))),
             (2, 2, vs.Spec(17, 45, simple=1, level=40, sharp=3, update=0.3)),
             (50, 30, vs.Spec(45, 49, parts=3, lf_delta=((10, -3, 7, None), (-63, 5, None, 2)), level=50)),
             (10, 70, vs.Spec(1, 9, level=5)),
             (78, 14, vs.Spec(17, 33, qi=127, limit=None, vmax=vs.MAX_LEVEL, zero_frac=0.8, level=0))]
    out = []
    for k, (x, y, sp) in enumerate(specs):
        payload, _ = vs.write_frame(sp, 7000 + k)
        alph = None
        if k % 2:
            alph = b"\x00" + rng.integers(0, 256, sp.w * sp.h, dtype=np.uint8).tobytes()
        out.append((x, y, sp.w, sp.h, payload, alph))
    return out


def _anim():
    frames = []
    for x, y, w, h, payload, alph in _frames():
        body = (vs.chunk(b"ALPH", alph) if alph is not None else b"") + vs.chunk(b"VP8 ", payload)
        frames.append(anmf(x, y, w, h, body, blend=bool(x % 4)))
    return animation(96, 80, frames)


def _still(w, h, payload, alph):
    if alph is None:
        return vs.still(payload)
    vp8x = vs.chunk(b"VP8X", bytes([0x10, 0, 0, 0]) + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little"))
    return vs.riff(vp8x + vs.chunk(b"ALPH", alph) + vs.chunk(b"VP8 ", payload))


def test_animation_of_hand_built_frames(cuda_lib, lib, xb):
    data = _anim()
    built = _frames()
    _, frames, metas, rc = cuda_lib.webp_frames(data)
    assert rc == 0 and len(frames) == len(built)
    for k, ((x, y, w, h, payload, alph), got, m) in enumerate(zip(built, frames, metas)):
        assert (m["x"], m["y"]) == (x, y), k
        still = _still(w, h, payload, alph)
        want = libwebp(still)
        crc, host = core_decode(lib, still)
        assert crc == 0 and np.array_equal(host, want), f"frame {k}: host cores differ from libwebp"
        got = got if alph is not None else got[:, :, :3]
        assert got.shape == want.shape and np.array_equal(got, want), f"frame {k}: device differs from libwebp"
    outs, status = check_against_per_image(cuda_lib, xb, [data], webp_opt(**FIT))
    assert status == [0]
    st = xb.stats()
    assert st["grid_items"] == 1 and st["fallback_items"] == 0, st
