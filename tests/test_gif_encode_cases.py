"""CPU: the GIF encoder catalogue of tests/gif_encode_cases.py reaches what it is built for.  Every case goes through
the oracle's encoder (oracle/oracle_gif.c); its output is read back with a Python code-stream reader and its palette
indices are replayed by a serial Python model of the reference's mapping, which must agree pixel for pixel and counts
the corners met: thresholds, straddled buckets, ties, alpha 127 / 128, memo order across palette runs, previous-frame
substitution; clear codes, code widths, sub-block lengths, interlace and frame shapes on the LZW side.  Where the
reference's own library is built, the file cases give the same bytes through it."""
import functools
from collections import Counter

import numpy as np
import pytest

from lilliput_b200 import abi
from tests import gif_encode_cases as ec
from tests.golden.make_golden_gif_encode import TIMEOUT_NS

FITS = ((40, 30), (23, 17))   # the Fit sizes the batch test uses


def given_frames(oracle, case):
    return case.frames if case.frames is not None else oracle.gif_frames(case.gif)[0]


def transcode(oracle, case, frames=None):
    """The oracle's output for `case` with `frames` (the case's own by default) given to the encoder."""
    it = iter(frames if frames is not None else given_frames(oracle, case))
    return oracle.gif_transcode(case.gif, lambda f: next(it))


@functools.lru_cache(maxsize=None)
def _survey():
    from oracle import oracle
    oracle.build()
    feats, outs = Counter(), {}
    for c in ec.cases():
        out = ec.read_gif(transcode(oracle, c))
        outs[c.name] = out
        if c.palette_model:
            feats += ec.map_frames(given_frames(oracle, c), out)
    return feats, outs


def test_palette_indices_follow_the_serial_model_and_reach_every_corner(oracle):
    feats, _ = _survey()
    for f in ("extreme_owner", "two_channels_extreme", "threshold_owner", "straddle_exact", "straddle_midpoint",
              "straddle_choice_differs", "tie_duplicate_entry", "tie_equidistant", "transparent_entry_nearest",
              "transparent_ge_ncolors", "transparent_ge_ncolors_pixel", "alpha127_transparent", "alpha128_transparent",
              "alpha127_opaque", "alpha128_opaque", "late_bucket_later_frame", "bucket_other_colour_earlier_frame",
              "palette_changes_back", "local_equal_to_global", "equal_bytes_other_count", "memo_carried",
              "prev_equal_least", "prev_least_minus_1", "owner_distances_disagree", "prev_substituted",
              "prev_disposal_01", "prev_disposal_23", "first_frame_with_transparent", "no_transparent_index"):
        assert feats[f] > 0, f"no case reaches {f}"


def test_designed_threshold_pixels_are_present(oracle):
    """Channels at 14 / 15 / 16 and 239 / 240 / 241, on all three channels and with only two qualifying."""
    for c in ec.cases():
        if c.name in ("thresholds", "designed_thresholds"):
            px = np.concatenate([f[..., :3].reshape(-1, 3)[:, ::-1] for f in given_frames(oracle, c)])
            have = {tuple(int(v) for v in p) for p in px}
            for t in ec.LOW + ec.HIGH:
                assert (t, t, t) in have, (c.name, t)
            assert any(sum(v < 15 for v in p) == 2 for p in have) and any(sum(v > 240 for v in p) == 2 for p in have)


def test_code_streams_reach_every_lzw_corner():
    _, outs = _survey()
    frames = [(name, f) for name, o in outs.items() for f in o["frames"]]
    for mc in range(2, 9):
        assert any(f["min_code"] == mc and f["full_clears"] >= 3 for _, f in frames), f"code size {mc}: < 3 clear cycles"
    assert any(f["min_code"] == 2 and len(f["colors"]) == 6 and f["full_clears"] >= 3 for _, f in frames)  # 2 colours
    assert any(f["last_fill"] for _, f in frames)
    assert {f["data_len"] % 255 for _, f in frames if len(f["blocks"]) > 1} >= {0, 1, 254}
    for _, f in frames:   # sub-blocks: full ones, then the rest
        assert all(n == 255 for n in f["blocks"][:-1]) and 0 < f["blocks"][-1] <= 255 and f["eoi"]
        assert f["clear_widths"] <= {f["min_code"] + 1, 12} and max(f["widths"]) <= 12
    assert any(f["max_string"] >= 256 for name, f in frames if name == "flat")
    assert any(f["max_string"] >= 64 for name, f in frames if name == "period")
    shapes = {(f["width"], f["height"]) for _, f in frames}
    assert (1, 1) in shapes and any(w == 1 and h > 1 for w, h in shapes) and any(h == 1 and w > 1 for w, h in shapes)
    for group in (("interlaced_h",), ("designed_smaller_interlaced",)):
        heights = {f["height"] for name, f in frames if name.startswith(group) and f["interlace"]}
        assert heights >= set(range(1, 18)), (group, heights)
    o = outs["designed_smaller_interlaced"]
    assert any(f["width"] < o["width"] and f["height"] < o["height"] for f in o["frames"])
    runs = [len(o["frames"]) for name, o in outs.items() if name.startswith("noise_fill")]
    assert runs and all(n >= 2 for n in runs)


def test_fit_averages_alpha_to_127_and_128(oracle):
    """The Fit sizes of the batch test turn transparent / opaque edges into alpha 127 and 128, on frames that keep a
    transparent index, and colours onto the thresholds."""
    c = next(c for c in ec.palette_cases() if c.name == "alpha_edges")
    seen = set()
    for w, h in FITS:
        frames = oracle.gif_frames(c.gif)[0]
        ow, oh = oracle.expected_size(frames[0].shape[1], frames[0].shape[0], w, h)
        for f in frames:
            g = oracle.fit(f, ow, oh)
            seen |= set(np.unique(g[..., 3]).tolist()) | set(np.unique(g[..., :3]).tolist())
    assert {127, 128, 15, 240, 241} <= seen, sorted(seen)


@pytest.mark.parametrize("case", [c for c in ec.cases() if c.frames is None], ids=lambda c: c.name)
def test_file_cases_match_the_reference(oracle, ref_lib, case):
    """The reference's own ImageOps.Transform, resizing to the source size, against the oracle's plain transcode."""
    frames = oracle.gif_frames(case.gif)[0]
    h, w = frames[0].shape[:2]
    opt = abi.ImageOptions(FileType=".gif", Width=w, Height=h, ResizeMethod=abi.ImageOpsResize,
                           EncodeTimeout_ns=TIMEOUT_NS)
    assert ref_lib.transform(case.gif, opt, dst_cap=16 << 20) == oracle.gif_transcode(case.gif, cap=16 << 20)
