"""CPU: the baseline JPEG streams of tests/jpeg_baseline_streams.py against libjpeg-turbo (cv2) and the oracle.  Every
catalogue file decodes bit-exact alike in both; the damaged files are pinned to what each of them does."""
import numpy as np
import pytest

from tests import jpeg_baseline_streams as jb

STREAMS = jb.cases()
DAMAGED = jb.damaged()

# what each damaged file does: (libjpeg-turbo decodes it, the oracle decodes it).  libjpeg-turbo refuses a table with
# an all-ones code when the scan starts, and (through OpenCV's memory source) a scan that ends early or has no EOI
# behind it; it warns and carries on over a bad Huffman code, a run past coefficient 63 and restart markers out of
# order or missing.  The oracle takes an all-ones code, reads zeros past the end of the data, ignores the restart
# markers' numbers, and stops at a bad Huffman code, a run past 63 or a missing restart marker.
EXPECTED_DAMAGED = {
    "all_ones_code": (False, True),
    "ac_run_past_63": (True, False),
    "rst_wrong_number": (True, True),
    "rst_missing": (True, False),
    "truncated": (False, True),
    "truncated_rst": (False, False),
    "no_eoi": (False, True),
    "no_eoi_rst": (False, True),
    "missing_code": (True, False),
    "missing_code_rst": (True, False),
}


def _cv2_decode(data):
    cv2 = pytest.importorskip("cv2")
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)


def _oracle_decode(oracle, data):
    try:
        return oracle.jpeg_decode(data)[0]
    except RuntimeError:
        return None


def test_catalogue_reaches_every_feature():
    jb.check_coverage(STREAMS)


def test_parallel_decoder_constants():
    """sub_bits restates jpeg_huff_sync_kernel's subsequence length: 1024 bits below 64 KiB, then growing so that one
    subsequence per thread covers the scan."""
    assert jb.sub_bits(1) == jb.sub_bits(65536) == 1024
    assert jb.sub_bits(65537) == 1056
    assert jb.sub_bits(1 << 20) == 16384


def test_tables_are_what_they_claim():
    assert len(jb.long_prefixes(jb.LONG_AC)) >= 20
    assert sorted(jb.LONG_AC[1]) == sorted([0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)])
    for t in (jb.LONG_AC, jb.LONG_DC, jb.SINGLE_DC, jb.SINGLE_AC, jb.DENSE_AC, *jb.ANNEX_K.values()):
        assert sum(t[0]) == len(t[1]) and not jb.has_all_ones_code(t[0])
    assert max(n for _, n in jb.codes_of(*jb.LONG_DC).values()) > jb.DC_LOOK_BITS


@pytest.mark.parametrize("stream", STREAMS, ids=[s.name for s in STREAMS])
def test_stream_decodes_like_libjpeg_turbo(oracle, stream):
    want = _cv2_decode(stream.data)
    got = _oracle_decode(oracle, stream.data)
    assert want is not None and got is not None
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.parametrize("name,data,restart", DAMAGED, ids=[d[0] for d in DAMAGED])
def test_damaged_streams(oracle, name, data, restart):
    ref = _cv2_decode(data) is not None
    mine = _oracle_decode(oracle, data) is not None
    assert (ref, mine) == EXPECTED_DAMAGED[name]


@pytest.mark.xfail(strict=True, reason="libjpeg-turbo writes a value whose run passes coefficient 63 to coefficient 63; "
                                       "the oracle (and the device decoders) refuse the block")
def test_ac_run_past_63_decodes_like_libjpeg_turbo(oracle):
    data = dict((n, d) for n, d, _ in DAMAGED)["ac_run_past_63"]
    want = _cv2_decode(data)
    got = _oracle_decode(oracle, data)
    assert want is not None and got is not None and np.array_equal(got, want)
