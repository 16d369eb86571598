"""WebP lossy (VP8 key frame) decoding of hand-built streams (tests/vp8_streams.py) by the host build of the decoder
cores (oracle/oracle_webp.cpp over vp8_core.h), against libwebp twice (OpenCV's and Pillow's builds) and, where it is
built, the reference's own decoder: pixel for pixel, on streams that reach the parts of the format libwebp's encoder
never writes, and on coefficients past the range any encoder writes, where libwebp's x86 build chooses a 16-bit
inverse transform per block."""
import io

import numpy as np
import pytest

from tests import vp8_streams as vs
from tests.test_webp_lossless_streams import core_decode, libwebp
from tests.webp_util import optional_reference, vp8_cpu_lib


@pytest.fixture(scope="module")
def lib():
    return vp8_cpu_lib()


def pillow(data: bytes):
    """Pillow's libwebp decode of a still, as BGR."""
    from PIL import Image
    im = Image.open(io.BytesIO(bytes(data)))
    return np.asarray(im.convert("RGB"))[:, :, ::-1]


def _check(lib, case):
    want = libwebp(case.data)
    assert want is not None, f"{case.name}: libwebp refuses a well-formed stream"
    rc, got = core_decode(lib, case.data)
    assert rc == 0, f"{case.name}: core rc {rc}"
    assert got.shape == want.shape, case.name
    bad = np.argwhere(got != want)
    assert not len(bad), f"{case.name}: {len(bad)} samples differ from libwebp, first at {bad[:3].tolist()}"
    assert np.array_equal(pillow(case.data), want), f"{case.name}: Pillow's libwebp and OpenCV's disagree"


CASES = vs.cases()


def test_catalogue_reaches_every_feature():
    cov = vs.coverage()
    missing = [f for f in vs.FEATURES if not cov[f]]
    assert not missing, missing


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_stream_decodes_as_libwebp(lib, case):
    _check(lib, case)


def test_streams_match_the_reference_decoder(lib):
    ref = optional_reference()
    if ref is None:
        pytest.skip("oracle/_ref is not built")
    for case in CASES + tuple(c for _, c in vs.large_coefficient_cases()):
        _, frames, _, rc = ref.webp_frames(case.data)
        crc, got = core_decode(lib, case.data)
        assert rc == 0 and crc == 0 and np.array_equal(got, frames[0]), case.name


LARGE = vs.large_coefficient_cases()


@pytest.mark.parametrize("group", sorted({g for g, _ in LARGE}))
def test_large_coefficients_decode_as_libwebp(lib, group):
    """Dequantised coefficients up to the int16 range: libwebp's x86 build runs its 16-bit SSE2 transform on blocks
    with a token past zigzag position 2 (and on all four blocks of a chroma plane where one has AC), its int AC3 / DC
    transforms elsewhere; Y2 blocks take the int WHT."""
    for g, case in LARGE:
        if g == group:
            _check(lib, case)
