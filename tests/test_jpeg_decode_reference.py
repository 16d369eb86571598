"""The oracle's JPEG decoder against libjpeg-turbo (OpenCV's build, through cv2.imdecode), bit-exact, over the tile
cases of tests/jpeg_decode_cases.py and a sweep of narrow frames.  The GPU decode tests compare against the oracle, so
this is what lets them trust it at sizes the live-reference test seldom draws."""
import numpy as np
import pytest

from tests import jpeg_decode_cases as jc

cv2 = pytest.importorskip("cv2")


def test_case_list_reaches_every_tile_edge(oracle):
    jc.check_coverage(jc.cases())
    # the multi-span batch geometry gives windows of two or more spans in every sampling
    W, H, dw, dh, _ = jc.BATCH_GEOMETRIES[-1]
    crop = oracle.fit_rect(W, H, *oracle.expected_size(W, H, dw, dh))
    for s in jc.COLOR_SAMPLINGS:
        assert jc.batch_window(s, W, H, crop).tiles_x >= 2, s


def _mismatches(oracle, case_list):
    bad = []
    for case in case_list:
        data = jc.encode(case)
        got, _ = oracle.jpeg_decode(data)
        want = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)
        if got.shape != want.shape or not np.array_equal(got, want):
            bad.append(case.label)
    return bad


def test_tile_cases_match_libjpeg_turbo(oracle):
    assert _mismatches(oracle, jc.cases()) == []


@pytest.mark.parametrize("sampling", list(jc.SAMPLINGS))
def test_narrow_frames_match_libjpeg_turbo(oracle, sampling):
    """Widths 1 to 8: libjpeg-turbo replicates h2v1 / h2v2 chroma that is two samples wide or less."""
    assert _mismatches(oracle, [c for c in jc.narrow_cases() if c.sampling == sampling]) == []
