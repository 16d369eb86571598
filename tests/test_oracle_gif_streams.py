"""CPU: the LZW stream generator of tests/gif_streams.py checked on the C oracle (giflib's decoder restated in
oracle/oracle_gif.c).  Every well-formed case decodes to the frames composited in numpy from the encoded indices, every
damaged one to the frames in front of its damaged frame and an error; the feature counts show that the catalogue
reaches each corner of the LZW decoder.  Where the reference library is built, giflib itself gives the same frames,
delays, disposals and error-versus-success."""
import functools

import numpy as np
import pytest

from tests import gif_streams as gs
from tests.webp_util import optional_reference

CASES = gs.cases()


def disposal_modes(disposals):
    """giflib disposal 2 -> GIF_DISPOSE_BACKGROUND (1), 3 -> GIF_DISPOSE_PREVIOUS (2), else none (ref giflib.cpp:187-199)"""
    return [{2: 1, 3: 2}.get(d, 0) for d in disposals]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_oracle_decodes_generated_streams(oracle, case):
    frames, delays, disposals, rc = oracle.gif_frames(case.gif)
    assert rc == (-1 if case.damage else 0)
    assert len(frames) == len(case.frames)
    for k, (got, want) in enumerate(zip(frames, case.frames)):
        assert np.array_equal(got, want), f"frame {k}"
    assert delays == [5] * len(frames) and disposals == [0] * len(frames)


@pytest.mark.parametrize("min_code", range(9))
def test_code_widths_follow_the_next_free_entry(min_code):
    """Code k of a segment is read at the bit length of the entry it creates (clear + 1 + k), at most 12 bits; at
    minimum code size 0 the first code is read at 1 bit.  The table fills and freezes at 12 bits."""
    idx = np.random.default_rng(min_code).integers(0, 1 << min_code, 60000)
    _, stats, codes = gs.lzw_encode(idx, min_code, clear="deferred")
    clear = 1 << min_code
    assert codes[0].code == clear and codes[-1].code == clear + 1
    want = [min(12, (clear + 1 + k).bit_length()) for k in range(len(codes) - 1)]
    if min_code == 0:
        want[0] = 1
    assert [c.width for c in codes[1:]] == want
    if min_code:  # a flat run at code size 0 needs 8.4 million pixels to fill the table (see flat_mc0_2900x2900)
        assert stats.frozen > 0 and stats.max_width == 12


def test_catalogue_reaches_every_corner():
    """The cases meant to cover each corner of the decoder do: a later change to the generator cannot quietly stop
    covering one."""
    good = {c.name: c for c in CASES if not c.damage}
    total = functools.reduce(gs.LzwStats.merge, (c.stats for c in good.values()))
    assert good["noise_deferred_2000x1500"].stats.frozen > 1000
    assert good["frozen_4100_wide"].stats.frozen > 0.9 * good["frozen_4100_wide"].stats.codes
    assert good["clear_every_width"].stats.clear_widths >= set(range(3, 13))
    assert good["flat_mc0_2900x2900"].stats.max_string >= 4000
    assert good["flat_mc0_2900x2900"].stats.kwkwk_lane0 > 0 and good["flat_mc0_2900x2900"].stats.kwkwk_chain == 32
    assert good["flat_mc1"].stats.kwkwk_lane0 > 0 and good["flat_mc1"].stats.kwkwk_chain == 32
    assert good["fill_then_more_codes"].overrun > 0
    assert total.near > 1000 and total.kwkwk > 4000
    assert set().union(*(c.min_codes for c in good.values())) >= set(range(9))
    assert good["interlaced_heights_1_17"].interlaced_heights >= set(range(1, 18))
    assert {c.damage for c in CASES if c.damage} == {"truncated", "eof_early", "above_top", "kwkwk_after_clear",
                                                     "empty_stream"}


def test_reference_agrees_with_oracle(oracle):
    """giflib (through the reference's own decoder) against the oracle on every case, damaged ones included."""
    ref = optional_reference()
    if ref is None:
        pytest.skip("oracle/_ref (the reference library) is not built")
    for case in CASES:
        frames, delays, disposals, rc = oracle.gif_frames(case.gif)
        rf, rd, rp, rrc = ref.gif_frames(case.gif)
        assert (rrc != 0) == (rc != 0), case.name
        assert len(rf) == len(frames), case.name
        assert [d * 10 for d in delays] == list(rd) and disposal_modes(disposals) == list(rp), case.name
        for k in range(len(frames)):
            assert np.array_equal(rf[k], frames[k]), (case.name, k)
