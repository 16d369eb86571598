"""Test infrastructure: baseline JPEG files (one interleaved scan, Huffman coded) whose every entropy-coding choice the
caller steers -- the Huffman table of each component and class as (bits, vals), the table ids each component names,
the padding bit value, FF fill bytes before markers, a restart interval, a COM segment that moves the scan's start
offset, a missing EOI or bytes after it -- and the symbols themselves: any block can carry a hand-written list of AC
tokens (runs of ZRL, a ZRL past coefficient 64, a run past 63) instead of the ones its coefficients give.

Built on tests/jpeg_scan_streams.py (its Frame / frame(), Bits, optimal_table and codes_of).  The writer knows the
bit offset of every block in the unstuffed scan, so the catalogue can say where blocks fall against the parallel
decoder's subsequences (lilliput_b200/csrc/jpeg_huff_parallel.cu) and assert that it reaches what libjpeg-turbo-written
files never do: long AC codes past the decoder's second-level tables, DC codes past its 9-bit lookahead, per-block
table lookup, DC and AC sizes up to 15, long synchronisation, dense byte stuffing, every scan alignment.

`cases()` is the catalogue (tests/test_jpeg_baseline_streams.py checks it against libjpeg-turbo and the oracle,
tests/test_gpu_jpeg_baseline_streams.py the device decoders against the oracle); `damaged()` the damaged files."""
import functools
import os
import re
from dataclasses import dataclass, field

import numpy as np

from tests.jpeg_decode_cases import SAMPLINGS
from tests.jpeg_scan_streams import ZIGZAG, Bits, Frame, codes_of, frame, optimal_table

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASELINE_SAMPLINGS = ("420", "422", "444", "gray")

# Parallel decoder constants (jpeg_huff_parallel.cu): subsequences of kSubBits bits, at least 1024; the AC lookahead
# is 11 bits and kHuffLongPrefixes (kernels.cuh) 11-bit prefixes of longer AC codes get a second-level table; the DC
# lookahead is 9 bits; the unstuffer reads 16-byte vectors in tiles of 512 of them.
MIN_SUB_BITS = 1024
HUFF_THREADS = 512
AC_LOOK_BITS = 11
LONG_PREFIXES = 16
DC_LOOK_BITS = 9
UNSTUFF_TILE = HUFF_THREADS * 16


def sub_bits(clean_len: int) -> int:
    """kSubBits of jpeg_huff_sync_kernel for an unstuffed scan of clean_len bytes (one subsequence per thread)."""
    total = clean_len * 8
    k = -(-total // HUFF_THREADS)
    return max(MIN_SUB_BITS, (k + 31) & ~31)


# ---------------------------------------------------------------- tables


def _annex_k():
    """The Annex K tables (bits[1..16], vals) as lilliput_b200/csrc/jpeg_std_tables.h holds them."""
    src = open(os.path.join(ROOT, "lilliput_b200", "csrc", "jpeg_std_tables.h")).read()
    arr = {m.group(1): [int(x, 0) for x in m.group(2).replace("\n", " ").split(",") if x.strip()]
           for m in re.finditer(r"static const uint8_t (\w+)\[\d+\] = \{([^}]*)\}", src)}
    return {"dc_luma": (arr["kDcLBits"][1:], arr["kDcVals"]), "dc_chroma": (arr["kDcCBits"][1:], arr["kDcVals"]),
            "ac_luma": (arr["kAcLBits"][1:], arr["kAcLVals"]), "ac_chroma": (arr["kAcCBits"][1:], arr["kAcCVals"])}


ANNEX_K = _annex_k()


def _bits(d):
    """bits[1..16] from {length: count}."""
    return [d.get(n, 0) for n in range(1, 17)]


# Every AC symbol (runs 0-15, sizes 1-15, EOB, ZRL): nine short codes of 2-10 bits, the other 233 of 12-16 bits
# under 39 distinct 11-bit prefixes, so prefixes past the 16th take the canonical walk, down to 16-bit codes.
_SHORT_AC = [0x00, 0x01, 0x02, 0x11, 0x03, 0x21, 0x12, 0x04, 0x31]
LONG_AC = (_bits({**{n: 1 for n in range(2, 11)}, 12: 40, 13: 40, 14: 40, 15: 40, 16: 73}),
           _SHORT_AC + [s for s in [0xF0] + [(r << 4) | z for z in range(1, 16) for r in range(16)] if s not in _SHORT_AC])
# DC categories 0-15, categories 12-15 on codes of 10-13 bits (past the 9-bit lookahead)
LONG_DC = (_bits({2: 2, 3: 2, 4: 2, 5: 2, 6: 2, 7: 1, 8: 1, 10: 1, 11: 1, 12: 1, 13: 1}), list(range(16)))
# one code: a flat frame's DC difference (always category 0) and its EOB
SINGLE_DC = (_bits({1: 1}), [0])
SINGLE_AC = (_bits({1: 1}), [0x00])
# ones-heavy codes: EOB is "0", a size-15 value right after the previous one is "11111110"; 32767 (fifteen 1 bits) on
# every coefficient makes most scan bytes FF
DENSE_AC = (_bits({n: 1 for n in range(1, 9)}), [0x00, 0x01, 0x11, 0x21, 0x02, 0xF0, 0x31, 0x0F])


def has_all_ones_code(bits) -> bool:
    """jdhuff.c jpeg_make_d_derived_tbl: no code may be all ones."""
    code, last = 0, max([n for n in range(1, 17) if bits[n - 1]], default=0)
    for n in range(1, last + 1):
        code += bits[n - 1]
        if code >= 1 << n:
            return True
        code <<= 1
    return False


def long_prefixes(table):
    """The distinct 11-bit prefixes of a table's AC codes longer than 11 bits, in canonical order."""
    out = []
    for code, n in sorted(codes_of(*table).values(), key=lambda cn: (cn[1], cn[0])):
        if n > AC_LOOK_BITS and code >> (n - AC_LOOK_BITS) not in out:
            out.append(code >> (n - AC_LOOK_BITS))
    return out


# ---------------------------------------------------------------- symbols

EOB, ZRL = (0, 0, 0), (15, 0, 0)


def _nbits(v):
    return int(abs(int(v))).bit_length()


def ac_tokens(z):
    """jchuff.c encode_one_block's AC symbols of a zigzag-ordered block: (run, size, value), ZRL, EOB."""
    out, r = [], 0
    for k in range(1, 64):
        v = int(z[k])
        if v == 0:
            r += 1
            continue
        while r > 15:
            out.append(ZRL)
            r -= 16
        out.append((r, _nbits(v), v))
        r = 0
    if r:
        out.append(EOB)
    return out


def scan_blocks(fr: Frame, c: int):
    """(Y, X) of component c's blocks in the order an interleaved scan codes them."""
    hc, vc = fr.factors[c]
    return [(my * vc + y, mx * hc + x) for my in range(fr.mcus[1]) for mx in range(fr.mcus[0])
            for y in range(vc) for x in range(hc)]


class _Bits(Bits):
    """Bits with a bit counter and a chosen padding bit."""

    def __init__(self):
        super().__init__()
        self.n = 0

    def put(self, v, n):
        super().put(v, n)
        self.n += n

    def flush_raw(self, pad: int) -> bytes:
        s = "".join(self.parts)
        self.parts = []
        s += str(pad) * (-len(s) % 8)
        self.n = len(s)
        return int(s, 2).to_bytes(len(s) // 8, "big") if s else b""


def _stuff(raw: bytes) -> bytes:
    return raw.replace(b"\xff", b"\xff\x00")


def _seg(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


@dataclass
class Info:
    """What the writer knows about the file it wrote."""
    scan_offset: int = 0
    scan_len: int = 0                       # entropy-coded bytes (stuffed, RST markers and fill included)
    clean_len: int = 0                      # unstuffed bytes of a scan without restart markers
    block_bits: list = field(default_factory=list)   # (start, end) bit offsets of every block, unstuffed
    used: dict = field(default_factory=dict)         # (class, id) -> symbols used
    intervals: int = 1
    stuffed: int = 0                        # 00 bytes of FF00 pairs
    tile_cross: bool = False                # an FF00 pair across an unstuffer tile edge (scan offset 8191 mod 8192),
    vector_cross: bool = False              # ... across a 16-byte vector edge (both for the per-image upload)


def write(fr: Frame, tables: dict, ids, *, restart=0, pad=1, fill_eoi=0, fill_rst=0, com_residue=None, eoi=True,
          trailer=b"", ac=None, rst_numbers=None, drop_rst=None, truncate=None, dht=None):
    """The baseline file of `fr`: one interleaved scan.  tables: (class, id) -> (bits, vals), or "optimal" for
    jchuff.c's optimal table of the symbols the components naming that id code; ids: (dc id, ac id) per component;
    ac: {(c, Y, X): AC tokens} in place of the block's own.  Damage: dht = tables written to the DHT in place of those
    the scan is coded with; rst_numbers = the n of each RSTn in order (default
    0..7 repeating); drop_rst = index of an RST marker left out; truncate = fraction of the scan's bytes kept, after
    which the file ends.  Returns (file, Info)."""
    ac = ac or {}
    nc = len(fr.factors)
    # ---- symbol stream: per MCU, per block (component, DC difference, AC tokens); restarts between MCUs
    events = []
    pred = [0] * nc
    order = [scan_blocks(fr, c) for c in range(nc)]
    pos = [0] * nc
    mcus = fr.mcus[0] * fr.mcus[1]
    for m in range(mcus):
        if restart and m and m % restart == 0:
            events.append(None)
            pred = [0] * nc
        for c, (hc, vc) in enumerate(fr.factors):
            for _ in range(hc * vc):
                Y, X = order[c][pos[c]]
                pos[c] += 1
                dc = int(fr.coef[c][Y, X, 0])
                toks = ac.get((c, Y, X))
                if toks is None:
                    toks = ac_tokens(fr.coef[c][Y, X][ZIGZAG])
                events.append((c, dc - pred[c], toks))
                pred[c] = dc
    # ---- tables
    used = {}
    for e in events:
        if e is None:
            continue
        c, d, toks = e
        used.setdefault((0, ids[c][0]), []).append(_nbits(d))
        for r, s, _ in toks:
            used.setdefault((1, ids[c][1]), []).append((r << 4) | s)
    tabs = {}
    for key in sorted(set(tables) | set(used)):
        t = tables.get(key, "optimal")
        if t == "optimal":
            freq = [0] * 256
            for s in used.get(key, []):
                freq[s] += 1
            t = optimal_table(freq)
        tabs[key] = (list(t[0]), list(t[1]))
    codes = {k: codes_of(*t) for k, t in tabs.items()}
    # ---- entropy-coded segment
    bw = _Bits()
    raw_parts, block_bits = [], []
    base = 0
    rst_k = 0
    for e in events:
        if e is None:
            raw_parts.append(bw.flush_raw(pad))
            base += bw.n
            bw.n = 0
            raw_parts.append(None)
            continue
        c, d, toks = e
        start = base + bw.n
        code, n = codes[(0, ids[c][0])][_nbits(d)]
        bw.put(code, n)
        s = _nbits(d)
        bw.put(d if d >= 0 else d - 1, s)
        for r, s, v in toks:
            code, n = codes[(1, ids[c][1])][(r << 4) | s]
            bw.put(code, n)
            bw.put(v if v >= 0 else v - 1, s)
        block_bits.append((start, base + bw.n))
    raw_parts.append(bw.flush_raw(pad))
    data = bytearray()
    for part in raw_parts:
        if part is None:
            n = rst_numbers[rst_k] if rst_numbers else rst_k & 7
            if drop_rst != rst_k:
                data += b"\xff" * fill_rst + bytes([0xFF, 0xD0 + n])
            rst_k += 1
        else:
            data += _stuff(part)
    info = Info(block_bits=block_bits, intervals=rst_k + 1,
                used={k: set(v) for k, v in used.items()})
    info.clean_len = sum(len(p) for p in raw_parts if p is not None)
    info.stuffed = sum(p.count(b"\xff") for p in raw_parts if p is not None)
    # (offsets from the scan's first byte: the unstuffer's vectors and tiles as the per-image path lays them out, where
    # the scan is uploaded on its own at a 256-byte boundary; in lp_batch they shift with the scan's place in the upload)
    ffs = [i for i in range(len(data) - 1) if data[i] == 0xFF and data[i + 1] == 0]
    info.tile_cross = any((i + 1) % UNSTUFF_TILE == 0 for i in ffs)
    info.vector_cross = any((i + 1) % 16 == 0 for i in ffs)
    if truncate is not None:
        data = data[:int(len(data) * truncate)]
    # ---- headers
    ext = any(i > 1 for p in ids for i in p) or len({p[0] for p in ids}) > 2 or len({p[1] for p in ids}) > 2 or any(
        s > 11 for (k, _), t in tabs.items() if k == 0 for s in t[1]) or any(
        s & 15 > 10 for (k, _), t in tabs.items() if k == 1 for s in t[1])
    head = bytearray()
    head += _seg(0xDB, b"".join(bytes([q]) + bytes(fr.qt[q][ZIGZAG].astype(np.uint8)) for q in range(min(nc, 2))))
    sof = bytes([8]) + fr.h.to_bytes(2, "big") + fr.w.to_bytes(2, "big") + bytes([nc])
    for c, (hc, vc) in enumerate(fr.factors):
        sof += bytes([c + 1, (hc << 4) | vc, min(c, 1)])
    head += _seg(0xC1 if ext else 0xC0, sof)
    tabs_out = {**tabs, **(dht or {})}
    head += _seg(0xC4, b"".join(bytes([(k << 4) | i]) + bytes(t[0]) + bytes(t[1]) for (k, i), t in sorted(tabs_out.items())))
    if restart:
        head += _seg(0xDD, restart.to_bytes(2, "big"))
    sos = bytes([nc]) + b"".join(bytes([c + 1, (ids[c][0] << 4) | ids[c][1]]) for c in range(nc)) + bytes([0, 63, 0])
    head += _seg(0xDA, sos)
    com = b""
    if com_residue is not None:
        n = (com_residue - (2 + len(head) + 4)) % 16
        com = _seg(0xFE, b"\x20" * n)
    out = b"\xff\xd8" + com + bytes(head)
    info.scan_offset = len(out)
    info.scan_len = len(data)
    out += bytes(data)
    if truncate is None:
        out += b"\xff" * fill_eoi + (b"\xff\xd9" if eoi else b"")
        out += trailer
    return out, info


# ---------------------------------------------------------------- content helpers


def annex_k_tables(nc):
    t = {(0, 0): ANNEX_K["dc_luma"], (1, 0): ANNEX_K["ac_luma"]}
    if nc > 1:
        t.update({(0, 1): ANNEX_K["dc_chroma"], (1, 1): ANNEX_K["ac_chroma"]})
    return t


def std_ids(nc):
    return [(0, 0)] + [(1, 1)] * (nc - 1)


def _value(rng, s):
    """A value of size category s, either sign."""
    v = int(rng.integers(1 << (s - 1), 1 << s)) if s else 0
    return v if rng.integers(0, 2) else -v


# Values past what an 8-bit encoder makes (DC categories 12-15, AC sizes 11-15) sit where the quantiser is WRAP_Q and
# are near multiples of 65536 / WRAP_Q: the decoders' 16-bit wrapping dequantisation (libjpeg-turbo's SIMD IDCT,
# restated by the oracle) brings them back to small products, so the IDCT stays in range and the pixels compare exactly.
WRAP_Q = 32
WRAP = 65536 // WRAP_Q


def wrap_quant(fr: Frame):
    """Quantisers of 1, WRAP_Q at the DC and at coefficient 63, for every table of the frame."""
    for q in fr.qt:
        q[:] = 1
        q[0] = q[63] = WRAP_Q


def _wrap_value(rng, s):
    """A value of size s >= 11 whose product with WRAP_Q is at most 96 in 16 bits."""
    t = int(rng.integers(0, 3))
    v = WRAP - 1 - t if s == 11 else WRAP * int(rng.integers(1 << (s - 12), 1 << (s - 11))) + t
    return v if rng.integers(0, 2) else -v


def all_symbol_blocks(fr: Frame, table, comps, rng):
    """AC tokens that use every symbol of an AC table at least once, over the blocks of `comps` in scan order: the
    sizes up to 5 packed into blocks (a ZRL in every third, EOB where a block stops short of coefficient 63), sizes 6
    to 10 one per block, each size of 11 or more alone at coefficient 63 of a block of its own (for wrap_quant)."""
    syms = [s for s in table[1] if s not in (0x00, 0xF0)]
    blocks = iter([(c, Y, X) for c in comps for Y, X in scan_blocks(fr, c)])
    out, k, toks, b = {}, 1, [], 0
    for s in [s for s in syms if s & 15 <= 5] + [None]:
        r, z = (s >> 4, s & 15) if s is not None else (0, 0)
        if s is None or k + r > 63:
            if k <= 63:
                toks.append(EOB)
            out[next(blocks)] = toks
            b, k, toks = b + 1, 1, []
            if s is None:
                break
        if k == 1 and r == 0 and b % 3 == 0:
            toks.append(ZRL)
            k = 17
        toks.append((r, z, _value(rng, z)))
        k += r + 1
    for s in [s for s in syms if 5 < s & 15 <= 10]:  # one per block: several would overflow the IDCT at quantiser 1
        out[next(blocks)] = [(s >> 4, s & 15, _value(rng, s & 15)), EOB]
    for s in sorted([s for s in syms if s & 15 > 10], key=lambda s: (s >> 4, s & 15)):
        r, z = s >> 4, s & 15
        out[next(blocks)] = [(0, 1, 1 if i % 2 else -1) for i in range(62 - r)] + [(r, z, _wrap_value(rng, z))]
    return out


def dc_categories(fr: Frame, c, cats, rng, restart=0, limit=32767):
    """DC values for component c (under wrap_quant) whose differences in scan order take the categories `cats` in
    turn: every value lies within 63 of a multiple of WRAP, and inside +-limit.  The running value restarts at 0 with
    every restart interval.  A category no value can reach from the previous one is coded as category 0."""
    order = scan_blocks(fr, c)
    hc, vc = fr.factors[c]
    v = 0
    for i, (Y, X) in enumerate(order):
        if restart and i % (restart * hc * vc) == 0:
            v = 0
        cat = cats[i % len(cats)]
        for _ in range(4000):
            d = _value(rng, cat)
            w = v + d
            if abs(w) <= limit and abs(w - WRAP * round(w / WRAP)) <= 63:
                v = w
                break
        fr.coef[c][Y, X, 0] = v


def tune_length(fr: Frame, tables, ids, target_bytes, **kw):
    """Sets AC tokens of the last blocks in scan order (values +-1 and +-2 from coefficient 1 on) so that the
    unstuffed scan is exactly target_bytes long.  Fixed tables only."""
    nc = len(fr.factors)
    last = []
    order = [scan_blocks(fr, c) for c in range(nc)]
    seq = []
    pos = [0] * nc
    for _ in range(fr.mcus[0] * fr.mcus[1]):
        for c, (hc, vc) in enumerate(fr.factors):
            for _ in range(hc * vc):
                seq.append((c,) + order[c][pos[c]])
                pos[c] += 1
    codes = {k: codes_of(*t) for k, t in tables.items()}

    def cost(c, toks):
        return sum(codes[(1, ids[c][1])][(r << 4) | s][1] + s for r, s, _ in toks)

    def toks_of(m, n2):
        t = [(0, 2, 2 if i % 2 else -2) if i < n2 else (0, 1, 1 if i % 2 else -1) for i in range(m)]
        return t + ([EOB] if m < 63 else [])

    ac = {}
    _, info = write(fr, tables, ids, ac=ac, **kw)
    bits = info.block_bits[-1][1]
    lo, hi = 8 * (target_bytes - 1) + 1, 8 * target_bytes
    for c, Y, X in reversed(seq):
        rest = bits - cost(c, ac_tokens(fr.coef[c][Y, X][ZIGZAG]))
        c1, c2, ce = cost(c, [(0, 1, 1)]), cost(c, [(0, 2, 2)]), cost(c, [EOB])
        for m in range(64):
            for n2 in range(m + 1):
                if lo <= rest + n2 * c2 + (m - n2) * c1 + (ce if m < 63 else 0) <= hi:
                    ac[(c, Y, X)] = toks_of(m, n2)
                    return ac
        ac[(c, Y, X)] = toks_of(63, 0)
        bits = rest + cost(c, ac[(c, Y, X)])
    raise ValueError("scan cannot reach %d bytes" % target_bytes)


# ---------------------------------------------------------------- catalogue


@dataclass
class Stream:
    name: str
    data: bytes
    sampling: str
    restart: int = 0
    features: set = field(default_factory=set)
    info: Info = None


def _table_features(fr, tabs_used, ids, info):
    f = set()
    nc = len(fr.factors)
    pairs = {tuple(p) for p in ids}
    if len(pairs) >= 3:
        f.add("three_table_pairs")
    if ids[0] == (1, 1) and all(p == (0, 0) for p in ids[1:]):
        f.add("luma_id1_chroma_id0")
    if any(i in (2, 3) for p in ids for i in p):
        if {2, 3} <= {i for p in ids for i in p}:
            f.add("table_ids_2_3")
    for (k, i), t in tabs_used.items():
        used = info.used.get((k, i), set())
        if not used:
            continue
        if sum(t[0]) == 1:
            f.add("single_code_table")
        if k == 1:
            pfx = long_prefixes(t)
            cd = codes_of(*t)
            hit = {cd[s][0] >> (cd[s][1] - AC_LOOK_BITS) for s in used if cd[s][1] > AC_LOOK_BITS}
            if len(pfx) >= 20 and len(hit) > LONG_PREFIXES:
                f.add("ac_long_prefixes")
            if {11, 12, 13, 14, 15} <= {s & 15 for s in used}:
                f.add("ac_sizes_11_15")
        else:
            if {12, 13, 14, 15} <= used:
                f.add("dc_symbols_12_15")
            if 11 in used:
                f.add("dc_category_11")
            cd = codes_of(*t)
            if i == ids[0][0] and any(cd[s][1] > DC_LOOK_BITS for s in used):
                f.add("luma_dc_long_codes")
    return f


def _stream_features(fr, info, restart, pad, fill_eoi, fill_rst, eoi, trailer):
    f = {"pad%d" % pad}
    if fr.mcus == (1, 1):
        f.add("one_mcu")
    f.add("scan_offset_mod16_%d" % (info.scan_offset % 16))
    if fill_eoi:
        f.add("fill_before_eoi")
    if fill_rst and restart:
        f.add("fill_before_rst")
    if not eoi:
        f.add("no_eoi")
    if trailer:
        f.add("bytes_after_eoi")
    if not restart:
        sb = sub_bits(info.clean_len)
        unit = sb // 8
        r = info.clean_len % unit
        if info.clean_len >= unit:
            f.add({0: "len_multiple_of_sub", 1: "len_multiple_of_sub_plus1", unit - 1: "len_multiple_of_sub_minus1"}
                  .get(r, "len_other"))
        starts = {s for s, _ in info.block_bits}
        if any(s and s % sb == 0 for s in starts):
            f.add("block_on_sub_boundary")
        if any(s // sb != (e - 1) // sb for s, e in info.block_bits):
            f.add("block_straddles_sub")
        if info.stuffed * 10 >= 3 * info.scan_len and info.tile_cross and info.vector_cross:
            f.add("dense_stuffing")
    else:
        mcus = fr.mcus[0] * fr.mcus[1]
        if restart == 1:
            f.add("dri_1")
        if restart > mcus:
            f.add("dri_over_mcus")
        if mcus % restart:
            f.add("dri_uneven")
        if info.intervals > 8:
            f.add("rst_wraps")
    return f


def _symbol_features(fr, ac, ids, info):
    """Features of the AC tokens and DC values the blocks carry."""
    f = set()
    nc = len(fr.factors)
    for c in range(nc):
        vals = [int(fr.coef[c][Y, X, 0]) for Y, X in scan_blocks(fr, c)]
        if any(v > 32767 or v < -32768 for v in vals):
            f.add("dc_sum_out_of_int16")
        for Y, X in scan_blocks(fr, c):
            toks = ac.get((c, Y, X))
            if toks is None:
                toks = ac_tokens(fr.coef[c][Y, X][ZIGZAG])
            k = 1
            for i, (r, s, _) in enumerate(toks):
                if (r, s) == (0, 0):
                    if i == 0:
                        f.add("eob_after_dc")
                    break
                k += 16 if (r, s) == (15, 0) else r + 1
                if (r, s) == (15, 0) and k == 64 and i > 0 and toks[i - 1] == ZRL:
                    f.add("zrl_run_to_63")
                if (r, s) == (15, 0) and k > 64:
                    f.add("zrl_past_64")
                if s and k == 64 and i == len(toks) - 1:
                    f.add("value_at_63_no_eob")
    return f


def _make(name, sampling, fr, tables, ids, *, restart=0, pad=1, fill_eoi=0, fill_rst=0, com=0, eoi=True, trailer=b"",
          ac=None, extra=()):
    data, info = write(fr, tables, ids, restart=restart, pad=pad, fill_eoi=fill_eoi, fill_rst=fill_rst,
                       com_residue=com, eoi=eoi, trailer=trailer, ac=ac)
    written = _dht_of(data)
    f = _table_features(fr, written, ids, info) | _stream_features(fr, info, restart, pad, fill_eoi, fill_rst, eoi,
                                                                   trailer)
    f |= _symbol_features(fr, ac or {}, ids, info) | set(extra)
    annex = [tuple(map(list, t)) for t in ANNEX_K.values()]
    if all(t in annex for t in written.values()):
        f.add("annex_k")
    if all(k not in tables for k in written):
        f.add("optimal")
    return Stream("%s_%s_%dx%d" % (sampling, name, fr.w, fr.h), data, sampling, restart, f, info)


def _dht_of(data):
    """(class, id) -> (bits, vals) of the file's DHT segments."""
    out, pos = {}, 2
    while pos + 4 <= len(data) and data[pos] == 0xFF and data[pos + 1] != 0xDA:
        n = int.from_bytes(data[pos + 2:pos + 4], "big")
        if data[pos + 1] == 0xC4:
            p, end = pos + 4, pos + 2 + n
            while p < end:
                bits = list(data[p + 1:p + 17])
                out[(data[p] >> 4, data[p] & 15)] = (bits, list(data[p + 17:p + 17 + sum(bits)]))
                p += 17 + sum(bits)
        pos += 2 + n
    return out


def _trailer():
    """A small restart-coded JPEG of its own, as cameras append after EOI (a preview, a second frame)."""
    fr = frame("420", 48, 32, seed=77, quality=80)
    data, _ = write(fr, annex_k_tables(3), std_ids(3), restart=1)
    return data


def _dims(sampling, mcx, mcy):
    mw = 8 * max(h for h, _ in SAMPLINGS[sampling][1])
    mh = 8 * max(v for _, v in SAMPLINGS[sampling][1])
    return mw * mcx, mh * mcy


@functools.lru_cache(maxsize=None)
def cases():
    out = []
    for si, s in enumerate(BASELINE_SAMPLINGS):
        nc = len(SAMPLINGS[s][1])
        colour = nc > 1
        seed = 1000 * si
        streams = []

        def add(*a, **kw):
            kw.setdefault("com", len(streams) % 16)
            streams.append(_make(*a, **kw))

        # Annex K and optimal tables on natural content, off the MCU grid
        w, h = _dims(s, 5, 3)
        fr = frame(s, w - 3, h - 5, seed + 1, quality=90)
        add("annexk_noise", s, fr, annex_k_tables(nc), std_ids(nc))
        fr = frame(s, w + 7, h + 2, seed + 2, quality=75, content="smooth")
        add("optimal_smooth", s, fr, {}, std_ids(nc), pad=0, fill_eoi=3)
        # one MCU, Annex K and optimal
        fr = frame(s, 7, 5, seed + 3, quality=95)
        add("one_mcu", s, fr, annex_k_tables(nc), std_ids(nc))
        fr = frame(s, *_dims(s, 1, 1), seed + 4, quality=60)
        add("one_mcu_opt", s, fr, {}, std_ids(nc), pad=0)
        # every AC symbol (sizes up to 15, 12-16-bit codes past the second-level tables) and every DC category (12-15
        # on codes past the 9-bit lookahead), with and without restarts
        rng = np.random.default_rng(seed + 5)
        cats = list(range(8)) + list(range(11, 16))
        big = {"gray": (16, 12), "444": (12, 10)}.get(s, (8, 6))
        fr = frame(s, *_dims(s, *big), seed + 5, quality=85)
        wrap_quant(fr)
        ac = all_symbol_blocks(fr, LONG_AC, range(nc), rng)
        for c in range(nc):
            dc_categories(fr, c, cats, rng)
        tabs = {(0, 0): LONG_DC, (1, 0): LONG_AC}
        if colour:
            tabs.update({(0, 1): LONG_DC, (1, 1): LONG_AC})
        add("long_codes", s, fr, tabs, std_ids(nc), ac=ac)
        fr = frame(s, *_dims(s, *big), seed + 6, quality=85)
        wrap_quant(fr)
        ac = all_symbol_blocks(fr, LONG_AC, range(nc), rng)
        for c in range(nc):
            dc_categories(fr, c, cats, rng, restart=5)
        add("long_codes_rst5", s, fr, tabs, std_ids(nc), ac=ac, restart=5, fill_rst=2)
        # table ids: three pairs (per-block lookup), luma on 1 and chroma on 0, ids 2 and 3
        fr = frame(s, *_dims(s, 3, 2), seed + 7, quality=80)
        if colour:
            add("three_pairs", s, fr, {}, [(0, 0), (1, 1), (2, 2)])
            add("three_pairs_rst", s, fr, {}, [(0, 0), (1, 1), (2, 2)], restart=2)
            add("swapped_ids", s, fr, annex_k_tables(nc) | {(0, 1): ANNEX_K["dc_luma"], (1, 1): ANNEX_K["ac_luma"],
                                                           (0, 0): ANNEX_K["dc_chroma"], (1, 0): ANNEX_K["ac_chroma"]},
                [(1, 1), (0, 0), (0, 0)])
            add("ids_2_3", s, fr, {}, [(2, 3), (3, 2), (3, 2)], restart=4)
            add("ids_2_3_parallel", s, fr, {}, [(3, 2), (2, 3), (2, 3)])
        else:
            add("luma_id1", s, fr, {(0, 1): ANNEX_K["dc_luma"], (1, 1): ANNEX_K["ac_luma"]}, [(1, 1)])
            add("ids_2_3", s, fr, {}, [(2, 3)], restart=4)
            add("ids_2_3_parallel", s, fr, {}, [(2, 3)])
        # flat frames: a single-code table (long synchronisation: every bit is a symbol boundary), and Annex K's
        # periodic MCU pattern, whose blocks fall on subsequence boundaries
        fr = frame(s, *_dims(s, 32, 20), seed + 8, content="flat")
        single = {(0, 0): SINGLE_DC, (1, 0): SINGLE_AC}
        if colour:
            single.update({(0, 1): SINGLE_DC, (1, 1): SINGLE_AC})
        add("flat_single_code", s, fr, single, std_ids(nc), extra={"periodic"})
        add("flat_single_code_rst", s, fr, single, std_ids(nc), restart=7, pad=0)
        fr = frame(s, 256, 160, seed + 9, content="flat")
        add("flat_annexk", s, fr, annex_k_tables(nc), std_ids(nc), extra={"periodic"}, pad=0)
        # symbols: ZRL runs to 63, a ZRL past 64, a value at 63 without EOB, EOB right after the DC, DC categories 11
        # and running DC sums outside int16
        fr = frame(s, *_dims(s, 3, 3), seed + 10, quality=70, content="smooth")
        blocks = scan_blocks(fr, 0)
        ac = {(0,) + blocks[0]: [(0, 3, 5), (13, 1, -1), ZRL, ZRL, ZRL],          # value at 15, ZRLs to 63
              (0,) + blocks[1]: [(3, 2, 3)] * 12 + [(0, 4, -9), (0, 1, 1), ZRL],   # values to 50, ZRL to 66
              (0,) + blocks[2]: [(15, 1, 1), (15, 1, -1), (15, 2, 2), (14, 5, 17)],  # value at 63, no EOB
              (0,) + blocks[3]: [EOB],
              (0,) + blocks[4]: [ZRL, ZRL, (14, 3, -4), ZRL]}                        # value at 47, ZRL to 64
        fr.qt[0][0] = WRAP_Q
        vals = [0, WRAP - 8, 2 * WRAP, 15 * WRAP, 30 * WRAP, 45 * WRAP + 3, 32 * WRAP, 20 * WRAP, 10 * WRAP, 0,
                -12 * WRAP, -24 * WRAP - 5, -15 * WRAP]
        for i, (Y, X) in enumerate(blocks):
            fr.coef[0][Y, X, 0] = vals[i % len(vals)]
        add("symbols", s, fr, {}, std_ids(nc), ac=ac)
        # the same symbols through the restart decoders: the DC sums restart, so they stay in int16 there
        fr2 = frame(s, *_dims(s, 3, 3), seed + 10, quality=70, content="smooth")
        fr2.qt[0][0] = WRAP_Q
        for i, (Y, X) in enumerate(blocks):
            fr2.coef[0][Y, X, 0] = [0, WRAP - 8, 8, WRAP, -WRAP + 8][i % 5]
        add("symbols_dri1", s, fr2, {}, std_ids(nc), ac=ac, restart=1, fill_rst=1)
        # dense byte stuffing across the unstuffer's vectors and tiles
        fr = frame(s, *_dims(s, {"420": 4, "422": 6, "444": 6, "gray": 12}[s], {"420": 3, "422": 3, "444": 4,
                                                                                 "gray": 6}[s]), seed + 11, content="flat")
        for q in fr.qt:
            q[:] = 2  # 32767 * 2 wraps to -2
        ac = {(c, Y, X): [(0, 15, 32767)] * 63 for c in range(nc) for Y, X in scan_blocks(fr, c)}
        dense = {(0, 0): SINGLE_DC, (1, 0): DENSE_AC}
        if colour:
            dense.update({(0, 1): SINGLE_DC, (1, 1): DENSE_AC})
        add("dense_ff", s, fr, dense, std_ids(nc), ac=ac)
        # scan lengths at a multiple of the subsequence length and one byte either side
        for d, tag in ((-1, "m1"), (0, "0"), (1, "p1")):
            fr = frame(s, *_dims(s, 12, 6), seed + 12, content="flat")
            tabs = annex_k_tables(nc)
            target = 128 * (3 + si) + d
            ac = tune_length(fr, tabs, std_ids(nc), target)
            add("length_" + tag, s, fr, tabs, std_ids(nc), ac=ac)
        # restart intervals: 1 (with fill bytes), longer than the frame, not dividing it; bytes after EOI
        fr = frame(s, *_dims(s, 5, 2), seed + 13, quality=85)
        add("dri1", s, fr, annex_k_tables(nc), std_ids(nc), restart=1, fill_rst=3, fill_eoi=1)
        add("dri_over", s, fr, {}, std_ids(nc), restart=11)
        fr = frame(s, *_dims(s, 7, 5), seed + 14, quality=85)
        add("dri_uneven", s, fr, {}, std_ids(nc), restart=3, pad=0)
        add("dri_trailer", s, fr, annex_k_tables(nc), std_ids(nc), restart=4, trailer=_trailer())
        add("trailer", s, fr, {}, std_ids(nc), trailer=_trailer())
        out += streams
    return out


# ---------------------------------------------------------------- damaged files


def damaged():
    """(name, file, restart interval): damage the decoders are meant to refuse or ride over, and a file without EOI."""
    out = []
    s = "420"
    fr = frame(s, 61, 45, seed=4242, quality=85)
    nc = 3
    # a DHT whose luma AC table has the all-ones code (the optimal table with its reserved code point given out)
    _, info = write(fr, {}, std_ids(nc))
    bits, vals = optimal_table([2 + 3 * (k % 5) if k in info.used[(1, 0)] else 0 for k in range(256)])
    n = max(k for k in range(16) if bits[k])
    bits = list(bits)
    bits[n] += 1
    spare = next(v for v in range(1, 256) if v not in vals and v & 15)
    vals = vals + [spare]
    assert has_all_ones_code(bits)
    out.append(("all_ones_code", write(fr, {(1, 0): (bits, vals)}, std_ids(nc))[0], 0))
    # an AC run past coefficient 63 in the third block: values at 16, 32 and 48, then a run of 15 that puts the last
    # value at 64 (libjpeg-turbo writes it to 63 and goes on with the next block)
    blocks = scan_blocks(fr, 0)
    run = [(15, 1, 1)] * 3 + [(15, 2, 3)]
    assert sum(r + 1 for r, _, _ in run) == 64
    out.append(("ac_run_past_63", write(fr, {}, std_ids(nc), ac={(0,) + blocks[2]: run})[0], 0))
    # restart markers: a wrong number, a missing one
    out.append(("rst_wrong_number", write(fr, {}, std_ids(nc), restart=2, rst_numbers=[0, 1, 5, 3, 4, 5, 6, 7, 0, 1,
                                                                                       2, 3, 4, 5])[0], 2))
    out.append(("rst_missing", write(fr, {}, std_ids(nc), restart=2, drop_rst=3)[0], 2))
    # truncated inside an MCU, with and without restarts
    out.append(("truncated", write(fr, {}, std_ids(nc), truncate=0.6)[0], 0))
    out.append(("truncated_rst", write(fr, {}, std_ids(nc), restart=3, truncate=0.6)[0], 3))
    # the whole scan, but no EOI: libjpeg-turbo's memory source suspends when the entropy decoder reads on for its
    # lookahead, and OpenCV gives up
    out.append(("no_eoi", write(fr, {}, std_ids(nc), eoi=False)[0], 0))
    out.append(("no_eoi_rst", write(fr, {}, std_ids(nc), restart=2, eoi=False)[0], 2))
    # a code the content uses missing from its table (the longest luma AC code)
    bits, vals = optimal_table([2 + 3 * (k % 5) if k in info.used[(1, 0)] else 0 for k in range(256)])
    bits = list(bits)
    n = max(k for k in range(16) if bits[k])
    bits[n] -= 1
    gone = vals[sum(bits[:n + 1])]
    vals = [v for v in vals if v != gone]
    full = optimal_table([2 + 3 * (k % 5) if k in info.used[(1, 0)] else 0 for k in range(256)])
    out.append(("missing_code", write(fr, {(1, 0): full}, std_ids(nc), dht={(1, 0): (bits, vals)})[0], 0))
    out.append(("missing_code_rst", write(fr, {(1, 0): full}, std_ids(nc), restart=2, dht={(1, 0): (bits, vals)})[0], 2))
    return out


# ---------------------------------------------------------------- coverage

FEATURES = ({"annex_k", "optimal", "ac_long_prefixes", "luma_dc_long_codes", "table_ids_2_3", "single_code_table",
             "dc_symbols_12_15", "ac_sizes_11_15", "zrl_run_to_63", "zrl_past_64", "value_at_63_no_eob",
             "eob_after_dc", "dc_category_11", "dc_sum_out_of_int16", "one_mcu", "len_multiple_of_sub",
             "len_multiple_of_sub_plus1", "len_multiple_of_sub_minus1", "block_on_sub_boundary", "block_straddles_sub",
             "periodic", "dense_stuffing", "pad0", "pad1", "fill_before_eoi", "fill_before_rst",
             "bytes_after_eoi", "dri_1", "dri_over_mcus", "dri_uneven", "rst_wraps"} |
            {"scan_offset_mod16_%d" % r for r in range(16)})
# A missing EOI is not a catalogue feature: OpenCV's libjpeg-turbo source gives up on such a file (its entropy decoder
# reads on past the data for its lookahead and the memory source has nothing more), so the oracle and the device, which
# decode the complete scan, cannot be compared with it there.  damaged() carries files without EOI instead.
# what a one-component frame cannot have
COLOUR_ONLY = {"three_table_pairs", "luma_id1_chroma_id0"}


def check_coverage(streams):
    """Every feature in every sampling of BASELINE_SAMPLINGS (the table-pair ones in the colour samplings)."""
    for s in BASELINE_SAMPLINGS:
        seen = set().union(*(st.features for st in streams if st.sampling == s))
        want = FEATURES | (COLOUR_ONLY if s != "gray" else set())
        missing = want - seen
        assert not missing, (s, sorted(missing))
