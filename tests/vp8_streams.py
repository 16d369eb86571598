"""Test infrastructure: a WebP lossy (VP8 key frame) writer whose every choice the caller steers -- the frame header
(colour space, clamping, segmentation in absolute or delta mode with or without a map, loop-filter type, level,
sharpness and deltas, token partitions, the five quantizer deltas, coefficient-probability updates, skip), and per
macroblock the segment id, skip flag, 16x16 / 4x4 / chroma modes and the coefficient levels of every block -- plus
counts of the decoder corners each stream reaches.

The writer models the entropy coding exactly as a decoder reads it (RFC 6386 7.3 boolean coder; libwebp's mode trees
and mode-probability contexts; the band / context / category token trees, with the top / left non-zero flags carried
as the decoder carries them), and the quantizer, so that it can bound dequantised coefficients.  It does not model
reconstruction: libwebp decides what the pixels are.  Probability tables are read from the product's vp8_tables.h;
libwebp decodes the streams, so a wrong entry there still fails the tests.

`cases()` is the catalogue tests/test_webp_lossy_streams.py and the device test use, `FEATURES` what it must reach.
Every catalogue coefficient stays within +-2048 after dequantisation (int16, as the decoder stores it), the range a
real encoder writes.  `large_coefficient_cases()` goes past that on purpose, one group per inverse-transform class."""
import functools
import os
import re
import struct
from collections import Counter
from dataclasses import dataclass, field
from typing import Callable, Optional

import numpy as np

_TABLES = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "lilliput_b200", "csrc",
                       "vp8_tables.h")


def _table(name, n):
    txt = open(_TABLES).read()
    m = re.search(name + r"[^=]*=\s*\{(.*?)\};", txt, re.S)
    body = re.sub(r"//[^\n]*", "", m.group(1))
    v = [int(x, 0) for x in re.findall(r"-?(?:0x[0-9a-fA-F]+|\d+)", body)]
    assert len(v) == n, (name, len(v))
    return v


COEFF_PROBA0 = np.array(_table("kVp8CoeffProba0", 1056)).reshape(4, 8, 3, 11)
COEFF_UPDATE = np.array(_table("kVp8CoeffUpdateProba", 1056)).reshape(4, 8, 3, 11)
BMODES_PROBA = np.array(_table("kVp8BModesProba", 900)).reshape(10, 10, 9)
YMODES_TREE = _table("kVp8YModesIntra4", 18)
DC_TABLE = _table("kVp8DcTable", 128)
AC_TABLE = _table("kVp8AcTable", 128)
BANDS = [0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0]
ZIGZAG = [0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15]
CAT_PROBS = [(11, [173, 148, 140]), (19, [176, 155, 140, 135]), (35, [180, 157, 141, 134, 130]),
             (67, [254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129])]
MAX_LEVEL = 67 + 2047  # the largest DCT_CAT6 value, 2048 + 66
B_MODES = ("dc", "tm", "ve", "he", "rd", "vr", "ld", "vl", "hd", "hu")  # libwebp's enum order
Y_MODES = ("dc", "tm", "v", "h")
POSITIONS = ("top", "left", "corner", "right", "inner")


def wrap16(v):
    """The int16 a dequantised coefficient is stored as (libwebp and vp8_core.h both store level * dq to int16)."""
    return ((int(v) + 32768) & 0xFFFF) - 32768


def token_name(v):
    if v <= 4:
        return ("one", "two", "three", "four")[v - 1]
    if v <= 6:
        return "cat1"
    if v <= 10:
        return "cat2"
    return "cat%d" % (3 + next(k for k, (base, p) in enumerate(CAT_PROBS) if v < base + (1 << len(p))))


# ---------------------------------------------------------------- boolean encoder (RFC 6386 7.3)


class BoolEncoder:
    def __init__(self):
        self.out, self.rng, self.bottom, self.cnt = bytearray(), 255, 0, 24

    def _carry(self):
        i = len(self.out) - 1
        while i >= 0 and self.out[i] == 255:
            self.out[i] = 0
            i -= 1
        self.out[i] += 1

    def put(self, bit, prob):
        split = 1 + (((self.rng - 1) * prob) >> 8)
        if bit:
            self.bottom += split
            self.rng -= split
        else:
            self.rng = split
        while self.rng < 128:
            self.rng <<= 1
            if self.bottom & (1 << 31):
                self._carry()
            self.bottom = (self.bottom << 1) & 0xFFFFFFFF
            self.cnt -= 1
            if self.cnt == 0:
                self.out.append((self.bottom >> 24) & 255)
                self.bottom &= (1 << 24) - 1
                self.cnt = 8

    def literal(self, v, n):
        for i in range(n - 1, -1, -1):
            self.put((v >> i) & 1, 128)

    def signed(self, v, n):
        self.literal(abs(v), n)
        self.put(int(v < 0), 128)

    def optional_signed(self, v, n):
        """A flag, then (when v is not None) magnitude and sign: the header's optional fields."""
        self.put(int(v is not None), 128)
        if v is not None:
            self.signed(v, n)

    def finish(self):
        for _ in range(32):
            self.put(0, 128)
        return bytes(self.out)


def _tree_path(sym):
    """[(probability index, bit)] reaching sub-block mode `sym` in libwebp's kVp8YModesIntra4 tree."""
    def walk(node, path):
        for b in (0, 1):
            t = YMODES_TREE[2 * node + b] if node else YMODES_TREE[b]
            if t <= 0:
                if -t == sym:
                    return path + [(node, b)]
            else:
                r = walk(t, path + [(node, b)])
                if r:
                    return r
        return None
    return walk(0, [])


_BMODE_PATHS = [_tree_path(m) for m in range(10)]


# ---------------------------------------------------------------- frame description


@dataclass
class Segmentation:
    update_map: int
    update_data: int
    absolute: int = 1
    quant: tuple = (None,) * 4    # per segment, None = not sent
    level: tuple = (None,) * 4
    proba: tuple = (None,) * 3    # segment-tree probabilities, None = not sent (255)


@dataclass
class MbPlan:
    """What one macroblock carries.  levels(k) gives block k's 16 levels in zigzag order (k = -1 Y2, 0..15 Y,
    16..19 U, 20..23 V), or None for the frame's random content."""
    segment: int = 0
    skip: int = 0
    i4: bool = False
    ymode: int = 0
    bmodes: tuple = (0,) * 16
    uvmode: int = 0
    levels: Optional[Callable] = None


@dataclass
class Spec:
    w: int
    h: int
    profile: int = 0
    colorspace: int = 0
    clamp: int = 0
    scale: tuple = (0, 0)
    simple: int = 0
    level: int = 20
    sharp: int = 0
    lf_delta: Optional[tuple] = None  # (ref deltas[4], mode deltas[4]), None entries not sent
    seg: Optional[Segmentation] = None
    qi: int = 40
    dq: tuple = (None,) * 5           # y1_dc, y2_dc, y2_ac, uv_dc, uv_ac
    parts: int = 0                    # log2 of the token partition count
    use_skip: int = 1
    skip_p: int = 200
    update: float = 0.0               # share of coefficient probabilities given a new value
    # random content, used where plan() leaves a choice to the frame
    i4_frac: float = 0.5
    skip_frac: float = 0.2
    empty_frac: float = 0.0           # share of coded macroblocks whose blocks are all zero
    zero_frac: float = 0.6            # share of zero levels in a random block
    vmax: int = 40                    # largest random level
    limit: Optional[int] = 2048       # bound on |dequantised coefficient|, None = none
    run_to_end: int = 0               # every n-th coded block ends on a zero run to position 16 instead of end-of-block
    plan: Optional[Callable] = None   # plan(rng, mx, my, mb_w, mb_h) -> MbPlan, None = random


def quant_of(sp: Spec):
    """[(y1, y2, uv) dq pairs] per segment, and the features the clips reach, as the decoder derives them."""
    st = Counter()
    seg = sp.seg
    y1d, y2d, y2a, uvd, uva = [d or 0 for d in sp.dq]

    def clip(v, hi=127):
        if v < 0:
            st["q:clip_0"] += 1
        if v > hi:
            st["q:clip_127" if hi == 127 else "q:uv_dc_clip_117"] += 1
        return min(max(v, 0), hi)
    out = []
    for s in range(4):
        if seg is not None:  # a map without data: every segment at q 0 (libwebp's reset segment header)
            q = (seg.quant[s] or 0) if seg.update_data else 0
            if not (seg.absolute if seg.update_data else 1):
                q += sp.qi
        else:
            q = sp.qi
        y2ac = AC_TABLE[clip(q + y2a)] * 101581 >> 16
        if y2ac < 8:
            st["q:y2_ac_floor_8"] += 1
        out.append(((DC_TABLE[clip(q + y1d)], AC_TABLE[clip(q)]), (2 * DC_TABLE[clip(q + y2d)], max(y2ac, 8)),
                    (DC_TABLE[clip(q + uvd, 117)], AC_TABLE[clip(q + uva)])))
    return out, st


def filter_levels(sp: Spec):
    """{(segment, i4): loop-filter level} as the decoder derives it (intra frame: reference delta 0, mode delta 0 for
    4x4 macroblocks), and the features the clips reach."""
    st = Counter()
    out = {}
    for s in range(4):
        base = sp.level
        if sp.seg is not None:
            seg = sp.seg
            base = (seg.level[s] or 0) if seg.update_data else 0
            if not (seg.absolute if seg.update_data else 1):
                base += sp.level
        for i4 in (0, 1):
            lv = base
            if sp.lf_delta is not None:
                lv += sp.lf_delta[0][0] or 0
                if i4:
                    lv += sp.lf_delta[1][0] or 0
            if lv < 0:
                st["lf:clip_0"] += 1
            if lv > 63:
                st["lf:clip_63"] += 1
            out[s, i4] = min(max(lv, 0), 63)
    return out, st


def _where(x, y, nx, ny):
    if x == 0 and y == 0:
        return "corner"
    if y == 0:
        return "top"
    if x == 0:
        return "left"
    if x == nx - 1:
        return "right"
    return "inner"


def inverse_wht(inp):
    """RFC 6386 14.3 on 16 raster-order int16 inputs: the 16 luma DCs (int16)."""
    t = [0] * 16
    for i in range(4):
        a0, a1 = inp[i] + inp[12 + i], inp[4 + i] + inp[8 + i]
        a2, a3 = inp[4 + i] - inp[8 + i], inp[i] - inp[12 + i]
        t[i], t[8 + i], t[4 + i], t[12 + i] = a0 + a1, a0 - a1, a3 + a2, a3 - a2
    out = [0] * 16
    for i in range(4):
        dc = t[4 * i] + 3
        a0, a1 = dc + t[4 * i + 3], t[4 * i + 1] + t[4 * i + 2]
        a2, a3 = t[4 * i + 1] - t[4 * i + 2], dc - t[4 * i + 3]
        out[i], out[4 + i], out[8 + i], out[12 + i] = [wrap16(v >> 3) for v in (a0 + a1, a3 + a2, a0 - a1, a3 - a2)]
    return out


# ---------------------------------------------------------------- tokens (RFC 6386 13)


def _write_large(e, v, p, st):
    st["tok:" + token_name(v)] += 1
    if v == MAX_LEVEL:
        st["tok:cat6_max"] += 1
    if v <= 4:
        e.put(0, p[3])
        if v == 2:
            e.put(0, p[4])
        else:
            e.put(1, p[4])
            e.put(v - 3, p[5])
        return
    e.put(1, p[3])
    if v <= 10:
        e.put(0, p[6])
        if v <= 6:
            e.put(0, p[7])
            e.put(v - 5, 159)
        else:
            e.put(1, p[7])
            e.put((v - 7) >> 1, 165)
            e.put((v - 7) & 1, 145)
        return
    e.put(1, p[6])
    for cat, (base, probs) in enumerate(CAT_PROBS):
        if v < base + (1 << len(probs)):
            e.put(cat >> 1, p[8])
            e.put(cat & 1, p[9 + (cat >> 1)])
            for i, pr in enumerate(probs):
                e.put(((v - base) >> (len(probs) - 1 - i)) & 1, pr)
            return
    raise ValueError(v)


def write_block(e, proba, typ, ctx, first, lv, st, run_to_end=False):
    """One block's tokens; lv = 16 levels in zigzag order.  Returns the decoder's return value: the position after
    the last token (16 after a zero run to the end)."""
    tp = proba[typ]
    nzpos = [i for i in range(first, 16) if lv[i]]
    last = nzpos[-1] + 1 if nzpos else first
    n, p = first, tp[BANDS[first]][ctx]
    while n < 16:
        if n >= last and not run_to_end:
            e.put(0, p[0])
            return n
        e.put(1, p[0])
        while n < 16 and lv[n] == 0:
            e.put(0, p[1])
            n += 1
            if n == 16:
                st["tok:zero_run_to_16"] += 1
                return 16
            p = tp[BANDS[n]][0]
        e.put(1, p[1])
        v = abs(int(lv[n]))
        if v == 1:
            st["tok:one"] += 1
            e.put(0, p[2])
            nc = 1
        else:
            e.put(1, p[2])
            _write_large(e, v, p, st)
            nc = 2
        e.put(int(lv[n] < 0), 128)
        n += 1
        p = tp[BANDS[n]][nc]
    return 16


def _random_magnitude(rng, vmax):
    if rng.random() < 0.7:
        return int(min(rng.geometric(0.4), vmax))
    lo, hi = [(1, 1), (2, 2), (3, 3), (4, 4), (5, 6), (7, 10), (11, 18), (19, 34), (35, 66), (67, MAX_LEVEL)][
        int(rng.integers(0, 10))]
    lo = min(lo, vmax)
    return int(rng.integers(lo, min(hi, vmax) + 1))


def random_levels(rng, first, dq, zero_frac, vmax, limit):
    """16 zigzag levels with about `zero_frac` zeros, |level * dq| (as int16) within `limit`."""
    lv = np.zeros(16, int)
    for i in range(first, 16):
        if rng.random() < zero_frac:
            continue
        v = _random_magnitude(rng, vmax)
        d = dq[i > 0]
        if limit is not None and abs(wrap16(v * d)) > limit:
            v = int(rng.integers(1, max(1, limit // d) + 1))
        lv[i] = v if rng.random() < 0.5 else -v
    return lv


# ---------------------------------------------------------------- the frame writer


def random_plan(rng, sp: Spec):
    i4 = bool(rng.random() < sp.i4_frac)
    return MbPlan(segment=int(rng.integers(0, 4)), skip=int(rng.random() < sp.skip_frac), i4=i4,
                  ymode=int(rng.integers(0, 4)), bmodes=tuple(int(m) for m in rng.integers(0, 10, 16)),
                  uvmode=int(rng.integers(0, 4)),
                  levels=(lambda k: np.zeros(16, int)) if rng.random() < sp.empty_frac else None)


def write_frame(sp: Spec, seed: int):
    """(VP8 payload, Counter of the features it reaches)."""
    rng = np.random.default_rng(seed)
    st = Counter()
    mb_w, mb_h = (sp.w + 15) // 16, (sp.h + 15) // 16
    st[f"size:w{sp.w}"] += 1
    st[f"size:h{sp.h}"] += 1
    if mb_w >= 40 and mb_h >= 30:
        st["size:40x30_mb"] += 1
    e = BoolEncoder()
    e.put(sp.colorspace, 128)
    e.put(sp.clamp, 128)
    seg = sp.seg
    if seg is None:
        e.put(0, 128)
    else:
        e.put(1, 128)
        e.put(seg.update_map, 128)
        e.put(seg.update_data, 128)
        if seg.update_data:
            e.put(seg.absolute, 128)
            for v in seg.quant:
                e.optional_signed(v, 7)
            for v in seg.level:
                e.optional_signed(v, 6)
            st["seg:absolute" if seg.absolute else "seg:delta"] += 1
        if seg.update_map:
            for pr in seg.proba:
                e.put(int(pr is not None), 128)
                if pr is not None:
                    e.literal(pr, 8)
                else:
                    st["seg:proba_absent"] += 1
        if seg.update_map and not seg.update_data:
            st["seg:map_without_data"] += 1
        if seg.update_data and not seg.update_map:
            st["seg:data_without_map"] += 1
    e.put(sp.simple, 128)
    e.literal(sp.level, 6)
    e.literal(sp.sharp, 3)
    if sp.lf_delta is None:
        e.put(0, 128)
    else:
        e.put(1, 128)
        e.put(1, 128)  # update the deltas
        for v in list(sp.lf_delta[0]) + list(sp.lf_delta[1]):
            e.optional_signed(v, 6)
        st["lf:deltas"] += 1
    e.literal(sp.parts, 2)
    e.literal(sp.qi, 7)
    for k, v in enumerate(sp.dq):
        e.optional_signed(v, 4)
        if v:
            st["q:delta_" + ("y1_dc", "y2_dc", "y2_ac", "uv_dc", "uv_ac")[k]] += 1
    e.put(0, 128)  # refresh_entropy_probs
    proba = COEFF_PROBA0.copy()
    updated = 0
    for idx in np.ndindex(4, 8, 3, 11):
        if rng.random() < sp.update:
            e.put(1, int(COEFF_UPDATE[idx]))
            v = int(rng.integers(0, 256))
            e.literal(v, 8)
            proba[idx] = v
            updated += 1
        else:
            e.put(0, int(COEFF_UPDATE[idx]))
    if updated == proba.size:
        st["proba:all_updated"] += 1
    e.put(sp.use_skip, 128)
    if sp.use_skip:
        e.literal(sp.skip_p, 8)
    for v, k in ((sp.colorspace, "colorspace"), (sp.clamp, "clamp"), (sp.scale != (0, 0), "scale")):
        if v:
            st["hdr:" + k] += 1
    if sp.profile:
        st[f"hdr:profile{sp.profile}"] += 1

    quant, qst = quant_of(sp)
    levels, fst = filter_levels(sp)
    filter_type = 0 if sp.level == 0 else 1 if sp.simple else 2
    used = set()
    nparts = 1 << sp.parts
    toks = [BoolEncoder() for _ in range(nparts)]
    top_modes = [0] * (mb_w * 4)
    top_nz = [0] * (mb_w * 9)
    block_no = 0
    for my in range(mb_h):
        t = toks[my & (nparts - 1)]
        left_modes, left_nz = [0] * 4, [0] * 9
        for mx in range(mb_w):
            mb = sp.plan(rng, mx, my, mb_w, mb_h) if sp.plan else random_plan(rng, sp)
            segment = mb.segment if seg is not None and seg.update_map else 0
            if seg is not None and seg.update_map:
                pr = [255 if q is None else q for q in seg.proba]
                if segment < 2:
                    e.put(0, pr[0])
                    e.put(segment, pr[1])
                else:
                    e.put(1, pr[0])
                    e.put(segment - 2, pr[2])
                st[f"seg:id{segment}"] += 1
            skip = mb.skip if sp.use_skip else 0
            if sp.use_skip:
                e.put(skip, sp.skip_p)
            e.put(0 if mb.i4 else 1, 145)
            where = _where(mx, my, mb_w, mb_h)
            tm = top_modes[mx * 4:mx * 4 + 4]
            if not mb.i4:
                ym = mb.ymode
                if ym in (0, 2):
                    e.put(0, 156)
                    e.put(int(ym == 2), 163)
                else:
                    e.put(1, 156)
                    e.put(int(ym == 1), 128)
                tm = [ym] * 4
                left_modes = [ym] * 4
                st[f"ymode:{Y_MODES[ym]}:{where}"] += 1
            else:
                for by in range(4):
                    lm = left_modes[by]
                    for bx in range(4):
                        m = mb.bmodes[by * 4 + bx]
                        prob = BMODES_PROBA[tm[bx]][lm]
                        for node, b in _BMODE_PATHS[m]:
                            e.put(b, int(prob[node]))
                        lm = tm[bx] = m
                        st[f"bmode:{B_MODES[m]}:{_where(mx * 4 + bx, my * 4 + by, mb_w * 4, mb_h * 4)}"] += 1
                    left_modes[by] = lm
            top_modes[mx * 4:mx * 4 + 4] = tm
            uv = mb.uvmode
            if uv == 0:
                e.put(0, 142)
            elif uv == 2:
                e.put(1, 142)
                e.put(0, 114)
            else:
                e.put(1, 142)
                e.put(1, 114)
                e.put(int(uv == 1), 183)
            st[f"uvmode:{Y_MODES[uv]}:{where}"] += 1
            used.add((segment, int(mb.i4)))
            tnz = top_nz[mx * 9:mx * 9 + 9]
            if skip:
                st["skip:i4" if mb.i4 else "skip:i16"] += 1
                for i in range(8):
                    tnz[i] = left_nz[i] = 0
                if not mb.i4:
                    tnz[8] = left_nz[8] = 0
                top_nz[mx * 9:mx * 9 + 9] = tnz
                continue
            y1, y2, uvq = quant[segment]
            blocks = []
            if not mb.i4:
                blocks.append((-1, 1, 8, 8, 0, y2))
            for k in range(16):
                blocks.append((k, 3 if mb.i4 else 0, k & 3, k >> 2, int(not mb.i4), y1))
            for c in range(8):
                blocks.append((16 + c, 2, 4 + (c >> 2) * 2 + (c & 1), 4 + (c >> 2) * 2 + ((c >> 1) & 1), 0, uvq))
            any_nz, y2_in = False, None
            for k, typ, ti, li, first, dq in blocks:
                lv = mb.levels(k) if mb.levels else None
                if lv is None:
                    lv = random_levels(rng, first, dq, sp.zero_frac, sp.vmax, sp.limit)
                lv = np.asarray(lv, int)
                lv[:first] = 0
                for i in range(first, 16):
                    if sp.limit is not None and abs(wrap16(lv[i] * dq[i > 0])) > sp.limit:
                        raise ValueError(f"level {lv[i]} x dq {dq[i > 0]} past the catalogue's bound")
                block_no += 1
                run = bool(sp.run_to_end and block_no % sp.run_to_end == 0 and not lv[15])
                nz = write_block(t, proba, typ, tnz[ti] + left_nz[li], first, lv, st, run)
                tnz[ti] = left_nz[li] = int(nz > first)
                any_nz |= bool(lv.any()) or run
                if k < 0:
                    y2_in = [0] * 16
                    for i in range(16):
                        y2_in[ZIGZAG[i]] = wrap16(lv[i] * dq[i > 0])
                    y2_lv = lv
            top_nz[mx * 9:mx * 9 + 9] = tnz
            if not any_nz and not sp.use_skip:
                st["noskip:all_zero_mb"] += 1
            if y2_in is not None and y2_lv.any() and not any(inverse_wht(y2_in)):
                st["y2:nonzero_wht_zero"] += 1
    payload_parts = [tk.finish() for tk in toks]
    for p in range(mb_h, nparts - 1):  # partitions no row uses: empty, but the last one must hold a byte
        payload_parts[p] = b""
        st["parts:empty_middle"] += 1
    st[f"parts:{nparts}"] += 1
    if nparts > mb_h:
        st["parts:more_than_rows"] += 1
    # features that depend on which segments / macroblock kinds the frame used
    for k in qst:
        st[k] += qst[k]
    for s, i4 in used:
        if filter_type:
            lv = levels[s, i4]
            st[f"lf:level{lv}"] += 1
            if lv:
                st[f"lf:sharp{sp.sharp}:{'simple' if sp.simple else 'normal'}"] += 1
        elif levels[s, i4]:
            st["lf:frame_level0_segment_level"] += 1
    for k in fst:
        st[k] += fst[k]
    first_part = e.finish()
    assert len(first_part) < (1 << 19)
    tag = (len(first_part) << 5) | (1 << 4) | (sp.profile << 1)
    hdr = struct.pack("<I", tag)[:3] + b"\x9d\x01\x2a" + struct.pack("<HH", sp.w | (sp.scale[0] << 14),
                                                                      sp.h | (sp.scale[1] << 14))
    sizes = b"".join(struct.pack("<I", len(x))[:3] for x in payload_parts[:-1])
    return hdr + first_part + sizes + b"".join(payload_parts), st


# ---------------------------------------------------------------- containers


def chunk(tag, payload):
    return tag + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) & 1 else b"")


def riff(chunks: bytes) -> bytes:
    body = b"WEBP" + chunks
    return b"RIFF" + struct.pack("<I", len(body)) + body


def still(payload) -> bytes:
    return riff(chunk(b"VP8 ", payload))


# ---------------------------------------------------------------- the catalogue


@dataclass
class Case:
    name: str
    data: bytes      # a whole WebP file
    payload: bytes   # its VP8 payload
    stats: Counter = field(default_factory=Counter)


def _case(name, sp: Spec, seed) -> Case:
    payload, st = write_frame(sp, seed)
    return Case(name, still(payload), payload, st)


def _systematic_modes(k, i4):
    """Every mode at every frame edge over a few frames: mode = (x + 3 y + k) mod count."""
    def plan(rng, mx, my, mb_w, mb_h):
        bm = tuple((mx * 4 + bx + 3 * (my * 4 + by) + k) % 10 for by in range(4) for bx in range(4))
        return MbPlan(segment=0, skip=0, i4=i4, ymode=(mx + 3 * my + k) % 4, bmodes=bm,
                      uvmode=(mx + 3 * my + k + 1) % 4)
    return plan


def _find_dq(v, limit):
    """(q index, 'dc' / 'ac') where v * dq, stored as int16, falls within +-limit."""
    for q in range(128):
        if abs(wrap16(v * AC_TABLE[q])) <= limit:
            return q, "ac"
        if abs(wrap16(v * DC_TABLE[q])) <= limit:
            return q, "dc"
    raise AssertionError(v)


def _catalogue():
    out = []
    seed = 1000
    # every width and height from 1 to 33 (odd ones included), each under another filter type / sharpness / level
    for n in range(1, 34):
        sp = Spec(n, 34 - n, simple=(n // 8) % 2, sharp=n % 8, level=1 + (n * 23) % 63, i4_frac=0.5,
                  profile=n % 4, vmax=80, parts=n % 4 if n % 3 == 0 else 0)
        out.append(_case(f"size_{n}x{34 - n}", sp, seed + n))
    # the 10 sub-block modes, 4 luma and 4 chroma modes at the top row, left column, corner, right column, interior
    for k in range(10):
        out.append(_case(f"bmodes_k{k}", Spec(37, 35, plan=_systematic_modes(k, True)), seed + 100 + k))
    for k in range(4):
        out.append(_case(f"ymodes_k{k}", Spec(77, 71, plan=_systematic_modes(k, False)), seed + 120 + k))
    # tokens: every category at q 0 (|level| up to 512 stays within 2048), the largest CAT6 value where its
    # dequantised int16 is small, blocks that end on a zero run to position 16
    out.append(_case("tokens_q0", Spec(48, 40, qi=0, vmax=512, zero_frac=0.3, level=10), seed + 200))
    q, which = _find_dq(MAX_LEVEL, 2048)

    def cat6_max(rng, mx, my, mb_w, mb_h):
        def levels(k):
            lv = np.zeros(16, int)
            if 0 <= k < 16:
                lv[0 if which == "dc" else 1 + (k % 15)] = MAX_LEVEL * (1 if k & 1 else -1)
            return lv
        return MbPlan(i4=True, bmodes=tuple(rng.integers(0, 10, 16)), uvmode=int(rng.integers(0, 4)), levels=levels)
    out.append(_case("tokens_cat6_max", Spec(32, 32, qi=q, plan=cat6_max), seed + 201))
    out.append(_case("tokens_zero_run_to_16", Spec(40, 40, run_to_end=3, zero_frac=0.8, level=30), seed + 202))
    # coefficient probabilities: all 1056 given new values (0 to 255), then a random third
    out.append(_case("proba_all_updated", Spec(48, 48, update=1.0, zero_frac=0.4), seed + 210))
    out.append(_case("proba_some_updated", Spec(33, 31, update=0.3), seed + 211))
    # skip: on 16x16 and 4x4 macroblocks; no skip flag at all with all-zero macroblocks
    out.append(_case("skip_i16_i4", Spec(64, 48, skip_frac=0.5, level=25), seed + 220))
    out.append(_case("no_skip_flag_zero_mbs", Spec(64, 48, use_skip=0, empty_frac=0.5, level=25), seed + 221))
    # a Y2 block whose coefficients dequantise (int16) to a value the WHT turns into all-zero DCs: the macroblock
    # counts as zero, so the inner edges are not filtered
    y2q, y2v = next((q, v) for q in range(128) for v in range(1, MAX_LEVEL + 1)
                    if wrap16(v * 2 * DC_TABLE[q]) != 0 and -3 <= wrap16(v * 2 * DC_TABLE[q]) <= 4)

    def y2_zero(rng, mx, my, mb_w, mb_h):
        if (mx + my) % 2:
            return random_plan(rng, Spec(0, 0, i4_frac=0.3, skip_frac=0))

        def levels(k):
            lv = np.zeros(16, int)
            if k == -1:
                lv[0] = y2v
            return lv
        return MbPlan(ymode=int(rng.integers(0, 4)), uvmode=int(rng.integers(0, 4)), levels=levels)
    out.append(_case("y2_wht_zero", Spec(64, 64, qi=y2q, level=40, sharp=0, plan=y2_zero), seed + 230))
    # segmentation: delta and absolute data, a map without data and data without a map, absent tree probabilities
    out.append(_case("seg_delta", Spec(64, 48, seg=Segmentation(1, 1, 0, (-10, 5, None, 20), (3, -7, 12, None),
                                                                (100, None, 30))), seed + 240))
    out.append(_case("seg_absolute", Spec(64, 48, seg=Segmentation(1, 1, 1, (0, 127, 64, 5), (0, 63, 20, 40),
                                                                   (200, 50, 128))), seed + 241))
    out.append(_case("seg_map_only", Spec(48, 48, seg=Segmentation(1, 0, proba=(128, 128, 128))), seed + 242))
    out.append(_case("seg_data_only", Spec(48, 48, seg=Segmentation(0, 1, 1, (90, 10, 10, 10), (50, 1, 1, 1))),
                     seed + 243))
    out.append(_case("seg_proba_absent", Spec(48, 48, seg=Segmentation(1, 1, 0, (4, -4, 8, -8), (None,) * 4,
                                                                       (None, None, None))), seed + 244))
    out.append(_case("seg_proba_partial", Spec(48, 48, seg=Segmentation(1, 0, proba=(None, 20, 230))), seed + 245))
    # loop filter: the high-edge-variance steps 14/15 and 39/40 (one segment each), deltas clipping to 0 and 63, a
    # segment level under a frame level of 0 (no filtering at all)
    for simple in (0, 1):
        out.append(_case(f"lf_hev_steps_{'simple' if simple else 'normal'}",
                         Spec(64, 64, simple=simple, level=30, seg=Segmentation(1, 1, 1, (None,) * 4, (14, 15, 39, 40),
                                                                                 (128, 128, 128))), seed + 250 + simple))
    out.append(_case("lf_hev_steps_delta", Spec(64, 64, level=14, lf_delta=((1, None, None, None), (25, 4, -5, None)),
                                                seg=Segmentation(1, 1, 0, (None,) * 4, (0, -1, 0, 0), (128, 128, 128))),
                     seed + 252))
    out.append(_case("lf_delta_clip_63", Spec(48, 48, level=60, lf_delta=((10, -3, 7, None), (-63, 5, None, 2))),
                     seed + 253))
    out.append(_case("lf_delta_clip_0", Spec(48, 48, level=5, sharp=5, lf_delta=((-10, 0, 0, 0), (30, 0, 0, 0))),
                     seed + 254))
    out.append(_case("lf_frame_level0_segments", Spec(48, 48, level=0, seg=Segmentation(1, 1, 1, (30, 40, 50, 60),
                                                                                       (20, 40, 63, 1), (128, 128, 128))),
                     seed + 255))
    for sharp in range(8):
        for simple in (0, 1):
            out.append(_case(f"lf_sharp{sharp}_{'simple' if simple else 'normal'}",
                             Spec(40, 24, simple=simple, sharp=sharp, level=8 + 7 * sharp), seed + 260 + 2 * sharp + simple))
    # quantizer: every delta, the clips at 0 and 127, chroma DC's clip at 117, Y2 AC's floor of 8
    out.append(_case("q_deltas", Spec(48, 48, qi=60, dq=(-15, 15, -8, 7, -15)), seed + 280))
    out.append(_case("q0_clipped", Spec(48, 48, qi=0, dq=(-15, -15, -15, -15, -15), vmax=400), seed + 281))
    out.append(_case("q127_clipped", Spec(48, 48, qi=127, dq=(15, 15, 15, 15, 15), vmax=12), seed + 282))
    out.append(_case("q_uv_dc_117", Spec(48, 48, qi=110, dq=(None, None, None, 12, None), vmax=12), seed + 283))
    # token partitions: 1, 2, 4, 8; more partitions than macroblock rows, with empty unused ones
    for parts, h in ((0, 48), (1, 80), (2, 150), (3, 140), (3, 40), (2, 17)):
        out.append(_case(f"parts{1 << parts}_h{h}", Spec(33, h, parts=parts, level=20), seed + 290 + parts * 7 + h))
    # header bits the decoder reads and ignores
    out.append(_case("header_bits", Spec(35, 21, colorspace=1, clamp=1, scale=(3, 2), profile=3), seed + 300))
    # one large frame: 40 x 30 macroblocks, odd size, mostly skipped
    out.append(_case("big_631x473", Spec(631, 473, skip_frac=0.85, zero_frac=0.9, parts=2, level=32, sharp=3),
                     seed + 310))
    return out


@functools.lru_cache(maxsize=None)
def cases() -> tuple:
    return tuple(_catalogue())


def coverage() -> Counter:
    total = Counter()
    for c in cases():
        total.update(c.stats)
    return total


FEATURES = (
    [f"bmode:{m}:{p}" for m in B_MODES for p in POSITIONS]
    + [f"ymode:{m}:{p}" for m in Y_MODES for p in POSITIONS]
    + [f"uvmode:{m}:{p}" for m in Y_MODES for p in POSITIONS]
    + [f"tok:{t}" for t in ("one", "two", "three", "four", "cat1", "cat2", "cat3", "cat4", "cat5", "cat6")]
    + ["tok:cat6_max", "tok:zero_run_to_16", "proba:all_updated"]
    + ["skip:i16", "skip:i4", "noskip:all_zero_mb", "y2:nonzero_wht_zero"]
    + [f"seg:id{s}" for s in range(4)]
    + ["seg:proba_absent", "seg:delta", "seg:absolute", "seg:map_without_data", "seg:data_without_map"]
    + [f"lf:level{v}" for v in (0, 14, 15, 39, 40, 63)] + ["lf:clip_0", "lf:clip_63", "lf:deltas",
                                                           "lf:frame_level0_segment_level"]
    + [f"lf:sharp{s}:{t}" for s in range(8) for t in ("simple", "normal")]
    + ["q:clip_0", "q:clip_127", "q:uv_dc_clip_117", "q:y2_ac_floor_8"]
    + [f"q:delta_{d}" for d in ("y1_dc", "y2_dc", "y2_ac", "uv_dc", "uv_ac")]
    + [f"parts:{n}" for n in (1, 2, 4, 8)] + ["parts:more_than_rows", "parts:empty_middle"]
    + [f"size:w{n}" for n in range(1, 34)] + [f"size:h{n}" for n in range(1, 34)] + ["size:40x30_mb"]
    + ["hdr:colorspace", "hdr:clamp", "hdr:scale"] + [f"hdr:profile{p}" for p in (1, 2, 3)]
)


# ---------------------------------------------------------------- coefficients past a real encoder's range


def _one_block_plan(pattern, i4=True, uv=False):
    """Each macroblock: one block (a random luma block, or with uv a chroma pair) carries `pattern(rng)` levels."""
    def plan(rng, mx, my, mb_w, mb_h):
        pick = int(rng.integers(0, 16))
        lvs = {}
        if uv:
            for base in (16, 20):
                a, b = rng.choice(4, 2, replace=False)
                lvs[base + int(a)], lvs[base + int(b)] = pattern(rng)
        else:
            lvs[pick] = pattern(rng)
        zero = np.zeros(16, int)
        return MbPlan(i4=i4, ymode=int(rng.integers(0, 4)), bmodes=tuple(int(m) for m in rng.integers(0, 10, 16)),
                      uvmode=int(rng.integers(0, 4)), levels=lambda k: lvs.get(k, zero))
    return plan


def _big(rng, n):
    return (rng.integers(MAX_LEVEL // 3, MAX_LEVEL + 1, n) * rng.choice([-1, 1], n)).astype(int)


def _full_pattern(rng):
    lv = np.zeros(16, int)
    pos = rng.choice(16, int(rng.integers(4, 17)), replace=False)
    lv[pos] = _big(rng, len(pos))
    lv[int(rng.integers(3, 16))] = _big(rng, 1)[0]  # a token past zigzag position 2: libwebp's full transform
    return lv


def _ac3_pattern(rng):
    lv = np.zeros(16, int)
    lv[:3] = _big(rng, 3)
    return lv


def _dc_pattern(rng):
    lv = np.zeros(16, int)
    lv[0] = _big(rng, 1)[0]
    return lv


def _uv_dc_near_limit(dq_dc):
    """Chroma DC levels whose int16 dequantised value lies within 3 of +-32767 for this dq (where libwebp's 16-bit
    +4 rounding wraps), or the largest levels when there is none."""
    vs = [v for v in range(1, MAX_LEVEL + 1) if abs(wrap16(v * dq_dc)) >= 32764]
    return vs or [MAX_LEVEL]


def large_coefficient_cases():
    """[(group, Case)]: coefficients far past +-2048, one group per libwebp inverse-transform class -- full (a token
    past zigzag position 2), AC3 (tokens at zigzag 0..2 only), DC only, chroma planes mixing a DC-only block with
    one that has AC (all four take the full transform), Y2 only -- then random blocks everywhere."""
    out = []
    big = dict(limit=None, level=0)
    groups = [("full", lambda: _one_block_plan(_full_pattern)), ("ac3", lambda: _one_block_plan(_ac3_pattern)),
              ("dc", lambda: _one_block_plan(_dc_pattern))]
    for g, mk in groups:
        for j, (q, w, h) in enumerate([(127, 32, 32), (100, 48, 33), (60, 31, 17), (127, 64, 48)]):
            sp = Spec(w, h, qi=q, plan=mk(), **big)
            if j == 3:
                sp.level = 30
            out.append((g, _case(f"large_{g}_q{q}_{w}x{h}", sp, 5000 + 17 * len(out))))
    for j, q in enumerate((34, 47, 92, 127)):
        dcs = _uv_dc_near_limit(DC_TABLE[min(q, 117)])

        def pair(rng, dcs=dcs):
            a = np.zeros(16, int)
            a[int(rng.integers(1, 16))] = int(rng.integers(1, 4)) * int(rng.choice([-1, 1]))
            b = np.zeros(16, int)
            b[0] = int(rng.choice(dcs)) * int(rng.choice([-1, 1]))
            return a, b
        out.append(("uv_mixed", _case(f"large_uv_mixed_q{q}", Spec(48, 32, qi=q, plan=_one_block_plan(pair, uv=True),
                                                                   **big), 5200 + j)))
    for j, (q, w, h) in enumerate([(127, 32, 32), (80, 48, 48), (20, 33, 17), (127, 64, 32)]):
        def y2only(rng, mx, my, mb_w, mb_h):
            y2 = np.zeros(16, int)
            pos = rng.choice(16, int(rng.integers(1, 17)), replace=False)
            y2[pos] = _big(rng, len(pos))
            zero = np.zeros(16, int)
            return MbPlan(ymode=int(rng.integers(0, 4)), uvmode=int(rng.integers(0, 4)),
                          levels=lambda k: y2 if k == -1 else zero)
        out.append(("y2_only", _case(f"large_y2_only_q{q}_{w}x{h}", Spec(w, h, qi=q, plan=y2only, level=20 * (j % 2),
                                                                          limit=None), 5300 + j)))
    for j, (q, i4) in enumerate([(127, 1.0), (127, 0.0), (90, 0.5), (40, 0.5), (127, 0.5), (10, 0.5)]):
        sp = Spec(48, 48, qi=q, i4_frac=i4, zero_frac=0.85, vmax=MAX_LEVEL, skip_frac=0.0, limit=None,
                  level=0 if j < 3 else 25)
        out.append(("random", _case(f"large_random_q{q}_i4_{i4}", sp, 5400 + j)))
    return out
