"""Test infrastructure: a WebP lossless (VP8L) bitstream writer whose every choice the caller steers -- prefix code
shapes (simple / normal, code-length repeats, max_symbol), the symbols of each entropy-coded image (literals, colour
cache indices, LZ77 copies by their plane distance code), the four transforms with caller-given sub-images and
palettes, meta prefix images, and ALPH chunks -- plus damaged variants of its streams and counts of the decoder
corners each stream reaches.

The writer does not model the transforms: pixels are random residuals and the reference decoder (libwebp) decides
what they decode to.  It does model the entropy-coded image itself (which ARGB value each symbol yields and the colour
cache), so that it can aim cache indices and copies.

`cases()` is the catalogue the CPU test (tests/test_webp_lossless_streams.py) and the device test use; `FEATURES` is
what the catalogue must reach, `damaged_cases()` the refusal list."""
import functools
import struct
from collections import Counter
from dataclasses import dataclass, field

import numpy as np

# ---------------------------------------------------------------- bits and prefix codes


class BitWriter:
    """LSB-first bit writer (spec section 2)."""

    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def put(self, v, n):
        assert 0 <= v < (1 << n) or n == 0
        self.acc |= v << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255)
            self.acc >>= 8
            self.n -= 8

    def bytes(self) -> bytes:
        return bytes(self.out) + (bytes([self.acc]) if self.n else b"")


def canonical(lens):
    """Canonical codes (deflate order: by length, then symbol) of code lengths <= 15: {symbol: (code, length)}."""
    count = Counter(l for l in lens if l)
    code, nxt = 0, {}
    for l in range(1, 16):
        code = (code + count.get(l - 1, 0)) << 1 if l > 1 else 0
        nxt[l] = code
    out = {}
    for s, l in enumerate(lens):
        if l:
            out[s] = (nxt[l], l)
            nxt[l] += 1
    return out


def flat_lengths(syms, alphabet, skew=False):
    """Code lengths of a complete code over `syms` (sorted, distinct).  Balanced, or `skew`: 1, 2, ..., 7 bits for the
    first seven, the rest balanced in the last 1/128 of the code space (so up to 15 bits for 256 of them)."""
    lens = [0] * alphabet
    syms = sorted(syms)
    k = len(syms)
    if k == 1:
        lens[syms[0]] = 1
        return lens
    if skew:
        d = min(k - 1, 7)
        for i in range(d):
            lens[syms[i]] = i + 1
        rest = syms[d:]  # share the last 2^-d of the code space
        sub = flat_lengths(list(range(len(rest))), len(rest)) if len(rest) > 1 else [0]
        for j, s in enumerate(rest):
            lens[s] = d + (sub[j] if len(rest) > 1 else 0)
        assert max(lens) <= 15
        return lens
    L = max(1, (k - 1).bit_length())
    x = (1 << L) - k  # x codes of L - 1 bits, the rest L bits
    for i, s in enumerate(syms):
        lens[s] = L - 1 if i < x else L
    return lens


@dataclass
class CodeStyle:
    """How one prefix code is written.  kind: 'auto' (simple when it fits, else normal), 'normal', 'simple'.
    Normal codes: `rle` uses 16/17/18, `max_symbol` stops the length list early with `length_nbits` = 2 + 2 * k
    (k None: the smallest that fits), `ncodes` forces the count of code-length code lengths, `skew` makes long codes.
    Simple codes: `first8` writes the first symbol with 8 bits, `twice` writes the one symbol twice."""
    kind: str = "auto"
    rle: bool = True
    max_symbol: bool = False
    nbits_k: int | None = None
    ncodes: int | None = None
    skew: bool = False
    first8: bool | None = None
    twice: bool = False
    rep16_first: bool = False
    lens: list | None = None  # explicit code lengths (damaged codes)
    raw_simple: tuple | None = None  # explicit simple code (nsym, first8, s0, s1): symbols may lie past the alphabet


ORDER = [17, 18, 0, 1, 2, 3, 4, 5, 16, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15]


def _rle_tokens(lens, rle, rep16_first):
    """(token, extra, extra bits) list of a code-length sequence."""
    toks, i, prev = [], 0, 8
    n = len(lens)
    while i < n:
        v = lens[i]
        run = 1
        while i + run < n and lens[i + run] == v:
            run += 1
        if rle and v == 0 and run >= 3:
            r = min(run, 138)
            toks.append((17, r - 3, 3) if r <= 10 else (18, r - 11, 7))
            i += r
            continue
        if rle and v != 0 and v == prev and run >= 3 and (i > 0 or rep16_first):
            r = min(run, 6)
            toks.append((16, r - 3, 2))
            i += r
            continue
        toks.append((v, 0, 0))
        if v:
            prev = v
        i += 1
    return toks


def write_code(bw, alphabet, used, st: CodeStyle, stats: Counter):
    """Writes a prefix code over the `used` symbols; returns {symbol: (code, length)} ({s: (0, 0)} for one symbol)."""
    if st.raw_simple is not None:
        nsym, first8, s0, s1 = st.raw_simple
        bw.put(1, 1)
        bw.put(nsym - 1, 1)
        bw.put(first8, 1)
        bw.put(s0, 8 if first8 else 1)
        if nsym == 2:
            bw.put(s1, 8)
        return {}
    used = sorted(set(used)) or [0]
    simple_ok = len(used) <= 2 and used[-1] < 256
    kind = st.kind if st.kind != "auto" else ("simple" if simple_ok and st.lens is None else "normal")
    if kind == "simple":
        assert simple_ok
        first8 = st.first8 if st.first8 is not None else used[0] > 1
        bw.put(1, 1)
        two = len(used) == 2 or st.twice
        bw.put(int(two), 1)
        bw.put(int(first8), 1)
        bw.put(used[0], 8 if first8 else 1)
        stats["code:simple1_8bit" if first8 else "code:simple1_1bit"] += len(used) == 1 and not st.twice
        if two:
            bw.put(used[-1], 8)
            stats["code:simple_same" if st.twice else "code:simple2"] += 1
        if len(used) == 1:
            return {used[0]: (0, 0)}
        return {used[0]: (0, 1), used[1]: (1, 1)}
    lens = st.lens if st.lens is not None else flat_lengths(used, alphabet, st.skew)
    toks = _rle_tokens(lens, st.rle, st.rep16_first)
    if st.max_symbol:
        while toks and toks[-1][0] in (0, 17, 18):
            toks.pop()
        toks = toks or [(0, 0, 0)]
    hist = sorted({t[0] for t in toks})
    cl = flat_lengths(hist, 19)
    assert max(cl) <= 7
    ccode = canonical(cl)
    last = max(i for i, s in enumerate(ORDER) if cl[s]) + 1
    ncodes = max(4, last, st.ncodes or 0)
    bw.put(0, 1)
    bw.put(ncodes - 4, 4)
    for i in range(ncodes):
        bw.put(cl[ORDER[i]], 3)
    stats[f"code:ncodes{ncodes}"] += 1
    if st.max_symbol:
        ms = len(toks)
        k = st.nbits_k if st.nbits_k is not None else next(k for k in range(8) if ms - 2 < (1 << (2 + 2 * k)))
        bw.put(1, 1)
        bw.put(k, 3)
        bw.put(ms - 2, 2 + 2 * k)
        stats["code:max_symbol"] += 1
    else:
        bw.put(0, 1)
    single_cl = len(hist) == 1
    for t, extra, nb in toks:
        if not single_cl:
            c, l = ccode[t]
            for b in range(l - 1, -1, -1):
                bw.put((c >> b) & 1, 1)
        if nb:
            bw.put(extra, nb)
        stats[f"code:rep{t}"] += t >= 16
    if st.rep16_first and toks[0][0] == 16:
        stats["code:rep16_first"] += 1
    nz = [s for s, l in enumerate(lens) if l]
    stats["code:normal_single"] += len(nz) == 1
    stats["code:long"] += max(lens) > 8
    if len(nz) == 1:
        return {nz[0]: (0, 0)}
    return canonical(lens)


def put_symbol(bw, code, s):
    c, l = code.get(s, (0, 1))  # (a damaged code need not hold the symbol: the decoder stops before it)
    for b in range(l - 1, -1, -1):
        bw.put((c >> b) & 1, 1)


# ---------------------------------------------------------------- entropy-coded images


def prefix_encode(v):
    """(symbol, extra bits, extra value) of an LZ77 length or distance code v >= 1 (spec 5.2.2)."""
    d = v - 1
    if d < 4:
        return d, 0, 0
    h = d.bit_length() - 1
    second = (d >> (h - 1)) & 1
    return 2 * h + second, h - 1, d & ((1 << (h - 1)) - 1)


def dist_map():
    pts = [(dx, dy) for dy in range(8) for dx in range(-7, 9) if not (dy == 0 and dx <= 0)]
    pts.sort(key=lambda p: (p[0] * p[0] + p[1] * p[1], abs(p[0]), p[0] < 0))
    return pts


DMAP = dist_map()


def plane_distance(xsize, code):
    if code > 120:
        return code - 120
    dx, dy = DMAP[code - 1]
    return max(1, dy * xsize + dx)


def cache_index(px, bits):
    return ((px * 0x1E35A7BD) & 0xFFFFFFFF) >> (32 - bits)


@dataclass
class Image:
    """Symbols of one entropy-coded image: ('lit', argb), ('cache', index), ('copy', length, plane_code).
    `groups`: meta prefix image (main image only) as (bits, 2-D array of group numbers); every group gets its own
    codes.  `styles`: {(group, k): CodeStyle} for k = 0 green, 1 red, 2 blue, 3 alpha, 4 distance."""
    syms: list
    cache_bits: int = 0
    groups: tuple | None = None
    styles: dict = field(default_factory=dict)
    cache_field: int | None = None  # the 4-bit cache size field when it differs from cache_bits (damaged)


def write_image(bw, xs, ys, im: Image, stats: Counter, tag: str, main: bool, meta_im=None):
    """Writes an entropy-coded image of xs x ys (spec 5, 6); returns its decoded ARGB values (before transforms)."""
    npix = xs * ys
    cb = im.cache_bits
    if cb or im.cache_field is not None:
        bw.put(1, 1)
        bw.put(im.cache_field if im.cache_field is not None else cb, 4)
        stats[f"cache:bits{cb}"] += cb > 0
        stats["cache:sub_image"] += cb > 0 and not main
    else:
        bw.put(0, 1)
    gmap, mbits, ngroups = None, 0, 1
    if main:
        if im.groups is None:
            bw.put(0, 1)
        else:
            mbits, gmap = im.groups
            bw.put(1, 1)
            bw.put(mbits - 2, 3)
            mxs, mys = -(-xs // (1 << mbits)), -(-ys // (1 << mbits))
            assert gmap.shape == (mys, mxs)
            g = gmap.reshape(-1).astype(np.int64)
            meta_syms = [("lit", 0xFF000000 | (int(v >> 8) << 16) | (int(v & 255) << 8)) for v in g]
            write_image(bw, mxs, mys, meta_im or Image(meta_syms), stats, tag + ".meta", False)
            ngroups = int(g.max()) + 1
            stats[f"meta:bits{mbits}"] += 1
            stats["meta:red_group"] += int(g.max()) >= 256
            stats["meta:unused_groups"] += ngroups - len(set(g.tolist())) >= 100
    # simulate the pixels to learn which symbols each group codes
    data = np.zeros(npix, np.uint64)
    cache = [0] * (1 << cb) if cb else None
    cache_from_copy = [False] * (1 << cb) if cb else None
    used = [[set() for _ in range(5)] for _ in range(ngroups)]
    plan = []
    src = 0
    for s in im.syms:
        gi = 0 if gmap is None else int(gmap[(src // xs) >> mbits, (src % xs) >> mbits])
        if s[0] == "lit":
            px = s[1]
            used[gi][0].add((px >> 8) & 255)
            used[gi][1].add((px >> 16) & 255)
            used[gi][2].add(px & 255)
            used[gi][3].add(px >> 24)
            plan.append((gi, s))
            if src < npix:
                data[src] = px
            if cb:
                cache[cache_index(px, cb)] = px
                cache_from_copy[cache_index(px, cb)] = False
            src += 1
        elif s[0] == "cache":
            k = s[1]
            used[gi][0].add(256 + 24 + k)
            plan.append((gi, s))
            if cb and k < (1 << cb):
                stats["cache:hit_from_copy"] += cache_from_copy[k]
                px = cache[k]
                if src < npix:
                    data[src] = px
                cache[cache_index(px, cb)] = px
                cache_from_copy[cache_index(px, cb)] = False
            src += 1
        else:
            _, length, pcode = s
            lsym = prefix_encode(length)[0]
            dsym = prefix_encode(pcode)[0]
            used[gi][0].add(256 + lsym)
            used[gi][4].add(dsym)
            plan.append((gi, s))
            dist = plane_distance(xs, pcode)
            if pcode <= 120:
                stats[f"lz:plane{pcode}"] += 1
                dx, dy = DMAP[pcode - 1]
                stats[f"lz:clamp_w{xs}"] += dy * xs + dx < 1
            else:
                stats["lz:code_gt120"] += 1
            stats[f"lz:len_sym{lsym}"] += 1
            stats[f"lz:dist_sym{dsym}"] += 1
            stats["lz:overlap"] += dist < length
            stats["lz:wrap_row"] += (src % xs) + length > xs
            for _ in range(length):
                if 0 <= src - dist and src < npix:
                    px = int(data[src - dist])
                    data[src] = px
                    if cb:
                        cache[cache_index(px, cb)] = px
                        cache_from_copy[cache_index(px, cb)] = True
                src += 1
    green_alpha = 256 + 24 + ((1 << cb) if cb else 0)
    alph = [green_alpha, 256, 256, 256, 40]
    codes = []
    for gi in range(ngroups):
        cs = []
        for k in range(5):
            st = im.styles.get((gi, k), im.styles.get(("*", k), CodeStyle()))
            cs.append(write_code(bw, alph[k], used[gi][k], st, stats))
        codes.append(cs)
    for gi, s in plan:
        c = codes[gi]
        if s[0] == "lit":
            px = s[1]
            for k, v in ((0, (px >> 8) & 255), (1, (px >> 16) & 255), (2, px & 255), (3, px >> 24)):
                put_symbol(bw, c[k], v)
        elif s[0] == "cache":
            put_symbol(bw, c[0], 256 + 24 + s[1])
        else:
            _, length, pcode = s
            ls, lnb, lv = prefix_encode(length)
            put_symbol(bw, c[0], 256 + ls)
            bw.put(lv, lnb)
            ds, dnb, dv = prefix_encode(pcode)
            put_symbol(bw, c[4], ds)
            bw.put(dv, dnb)
    return data.astype(np.uint32)


def literals(rng, n, alpha=None, channels=4, lo=0, hi=256):
    """n random literal symbols (alpha fixed when given)."""
    v = rng.integers(lo, hi, (n, 4), dtype=np.int64)
    if alpha is not None:
        v[:, 3] = alpha
    return [("lit", int((a << 24) | (r << 16) | (g << 8) | b)) for b, g, r, a in v]


# ---------------------------------------------------------------- transforms and the whole stream


def sub_size(n, bits):
    return -(-n // (1 << bits))


@dataclass
class Tr:
    """One transform: kind 'pred' (bits, modes 2-D), 'cc' (bits, (g2r, g2b, r2b) arrays), 'sg', 'ci' (palette:
    the delta-coded entries as written)."""
    kind: str
    bits: int = 0
    data: object = None
    image: Image | None = None  # how the sub-image / palette is coded (default: its values as literals)


def _pred_stats(stats, modes, bits, xs, ys):
    stats[f"pred:bits{bits}"] += 1
    stats["pred:tile_wider"] += (1 << bits) > xs
    stats[f"pred:width{xs}"] += xs <= 2
    ty_n, tx_n = modes.shape
    for ty in range(ty_n):
        for tx in range(tx_n):
            m = int(modes[ty, tx])
            x0, x1 = tx << bits, min(xs, (tx + 1) << bits)
            y0, y1 = ty << bits, min(ys, (ty + 1) << bits)
            stats[f"pred:m{m}:top"] += y0 == 0
            stats[f"pred:m{m}:left"] += x0 == 0 and y1 > 1
            stats[f"pred:m{m}:last"] += x1 == xs and xs > 1 and y1 > 1
            stats[f"pred:m{m}:inner"] += y1 > 1 and max(x0, 1) < min(x1, xs - 1)


def write_vp8l(w, h, transforms, main: Image, stats: Counter, header=True, alpha_hint=1, version=0) -> bytes:
    """A VP8L stream: the 5-byte header (unless `header` is False: an ALPH payload) + transforms + main image."""
    bw = BitWriter()
    if header:
        bw.put(0x2F, 8)
        bw.put(w - 1, 14)
        bw.put(h - 1, 14)
        bw.put(alpha_hint, 1)
        bw.put(version, 3)
        stats["hdr:version"] += version != 0
    xs = w
    kinds = []
    for t in transforms:
        bw.put(1, 1)
        typ = {"pred": 0, "cc": 1, "sg": 2, "ci": 3}[t.kind]
        bw.put(typ, 2)
        kinds.append(t.kind)
        if t.kind in ("pred", "cc"):
            bw.put(t.bits - 2, 3)
            sx, sy = sub_size(xs, t.bits), sub_size(h, t.bits)
            if t.kind == "pred":
                modes = np.asarray(t.data)
                assert modes.shape == (sy, sx)
                vals = [0xFF000000 | (int(m) << 8) for m in modes.reshape(-1)]
                _pred_stats(stats, modes, t.bits, xs, h)
            else:
                g2r, g2b, r2b = (np.asarray(a, np.int64).reshape(-1) & 255 for a in t.data)
                vals = [0xFF000000 | (int(c) << 16) | (int(b) << 8) | int(a) for a, b, c in zip(g2r, g2b, r2b)]
                allv = np.concatenate([np.asarray(a).reshape(-1) for a in t.data])
                stats[f"cc:bits{t.bits}"] += 1
                stats["cc:neg"] += bool((allv < 0).any())
                stats["cc:pos"] += bool((allv > 0).any())
            write_image(bw, sx, sy, t.image or Image([("lit", v) for v in vals]), stats, t.kind, False)
        elif t.kind == "ci":
            pal = list(t.data)
            n = len(pal)
            bw.put(n - 1, 8)
            write_image(bw, n, 1, t.image or Image([("lit", v) for v in pal]), stats, "ci", False)
            bits = 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3
            stats[f"ci:n{n}"] += 1
            acc, wrap = [0, 0, 0, 0], False
            for v in pal:
                for c in range(4):
                    s = acc[c] + ((v >> (8 * c)) & 255)
                    wrap |= s > 255
                    acc[c] = s & 255
            stats["ci:wrap"] += wrap
            stats["ci:ragged"] += bits > 0 and xs % (1 << bits) != 0
            t.packed_from = xs
            xs = sub_size(xs, bits)
            t.xbits = bits
        else:
            stats["sg"] += 1
    bw.put(0, 1)
    if "ci" in kinds and "pred" in kinds and kinds.index("pred") > kinds.index("ci"):
        stats["order:pred_after_ci"] += 1
    stats["order:all4"] += len(set(kinds)) == 4
    if len(kinds) >= 2:
        stats["order:" + ",".join(kinds)] += 1
    data = write_image(bw, xs, h, main, stats, "main", True)
    ci = next((t for t in transforms if t.kind == "ci"), None)
    if ci is not None:
        n, bits = len(ci.data), ci.xbits
        idx = (data.astype(np.int64) >> 8) & 255
        if bits:
            # indices of the packed pixels at or past the palette (only those inside the image count)
            per = 1 << bits
            bpp = 8 >> bits
            width = ci.packed_from
            rows = idx.reshape(h, xs)
            oob = False
            for x in range(width):
                sub = (rows[:, x // per] >> (bpp * (x % per))) & ((1 << bpp) - 1)
                oob |= bool((sub >= n).any())
            stats[f"ci:oob_b{bits}"] += oob
        else:
            stats["ci:oob_b0"] += bool((idx >= n).any())
    return bw.bytes()


# ---------------------------------------------------------------- containers


def chunk(tag, payload):
    return tag + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) & 1 else b"")


def riff(chunks: bytes) -> bytes:
    body = b"WEBP" + chunks
    return b"RIFF" + struct.pack("<I", len(body)) + body


def vp8x(w, h, flags):
    return chunk(b"VP8X", bytes([flags, 0, 0, 0]) + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little"))


def lossless_file(payload) -> bytes:
    return riff(chunk(b"VP8L", payload))


def alpha_still(w, h, alph, vp8) -> bytes:
    return riff(vp8x(w, h, 0x10) + chunk(b"ALPH", alph) + chunk(b"VP8 ", vp8))


def alpha_anmf(w, h, alph, vp8) -> bytes:
    """A one-frame animation whose frame covers the canvas and is not blended: it decodes to the frame itself."""
    frame = (0).to_bytes(3, "little") * 2 + (w - 1).to_bytes(3, "little") + (h - 1).to_bytes(3, "little")
    frame += (100).to_bytes(3, "little") + bytes([0x02])
    frame += chunk(b"ALPH", alph) + chunk(b"VP8 ", vp8)
    return riff(vp8x(w, h, 0x12) + chunk(b"ANIM", b"\0\0\0\0\0\0") + chunk(b"ANMF", frame))


@functools.lru_cache(maxsize=None)
def lossy_payload(w, h, seed) -> bytes:
    """A lossy VP8 payload of w x h from libwebp's encoder (the ALPH cases' colour)."""
    import cv2
    rng = np.random.default_rng(seed)
    img = (rng.integers(0, 256, (h, w, 3)) // 32 * 32).astype(np.uint8)
    ok, buf = cv2.imencode(".webp", img, [cv2.IMWRITE_WEBP_QUALITY, 80])
    assert ok
    from tests.webp_util import chunks_of
    return dict(chunks_of(buf.tobytes()))[b"VP8 "]


# ---------------------------------------------------------------- the catalogue


@dataclass
class Case:
    name: str
    data: bytes   # a whole WebP file
    kind: str     # "vp8l", "alph_still", "alph_anmf"
    stats: Counter


def _lossless(name, w, h, transforms, main, **kw) -> Case:
    st = Counter()
    return Case(name, lossless_file(write_vp8l(w, h, transforms, main, st, **kw)), "vp8l", st)


def _rand_main(rng, xs, h, **kw) -> Image:
    return Image(literals(rng, xs * h), **kw)


def _copies_image(rng, xs, h, copies, cache_bits=0, lead=None):
    """Literals for the first `lead` pixels, then the given (length, plane code) copies, then literals to the end."""
    npix = xs * h
    lead = lead if lead is not None else min(npix, 8 * xs + 8)
    syms = literals(rng, lead)
    src = lead
    for length, code in copies:
        length = min(length, npix - src)
        if length <= 0:
            break
        syms.append(("copy", length, code))
        src += length
    syms += literals(rng, npix - src)
    return Image(syms, cache_bits=cache_bits)


def _pred_modes(rng, xs, h, bits, systematic=False):
    sx, sy = sub_size(xs, bits), sub_size(h, bits)
    m = rng.integers(0, 16, (sy, sx))
    if systematic:
        m[0, :] = np.arange(sx) % 16
        m[:, 0] = np.arange(sy) % 16
        m[:, -1] = (np.arange(sy) + 5) % 16
    return m


def _cc_data(rng, xs, h, bits):
    sx, sy = sub_size(xs, bits), sub_size(h, bits)
    return tuple(rng.integers(-128, 128, (sy, sx)) for _ in range(3))


def _lossless_cases():
    out = []
    rng = np.random.default_rng(2024)
    # predictor: every mode at the top row, the left and the last column (64 x 68 at 4x4 tiles), tile bits 2..9,
    # tiles wider than the image, widths 1 and 2
    out.append(_lossless("pred_all_modes", 64, 68, [Tr("pred", 2, _pred_modes(rng, 64, 68, 2, True))],
                         _rand_main(rng, 64, 68)))
    out.append(_lossless("pred_all_modes_odd", 61, 67, [Tr("pred", 2, _pred_modes(rng, 61, 67, 2, True))],
                         _rand_main(rng, 61, 67)))
    for bits, (w, h) in zip(range(3, 10), [(45, 31), (77, 40), (100, 67), (130, 70), (300, 129), (257, 260),
                                          (100, 520)]):
        out.append(_lossless(f"pred_bits{bits}", w, h, [Tr("pred", bits, _pred_modes(rng, w, h, bits))],
                             _rand_main(rng, w, h)))
    for w, h in ((1, 37), (2, 33)):
        out.append(_lossless(f"pred_width{w}", w, h, [Tr("pred", 2, _pred_modes(rng, w, h, 2, True))],
                             _rand_main(rng, w, h)))
    # cross-colour at every tile size, subtract-green
    for bits in range(2, 10):
        w, h = 40 + 13 * bits, 30 + 7 * bits
        out.append(_lossless(f"cc_bits{bits}", w, h, [Tr("cc", bits, _cc_data(rng, w, h, bits))], _rand_main(rng, w, h)))
    out.append(_lossless("subtract_green", 33, 21, [Tr("sg")], _rand_main(rng, 33, 21)))
    # colour indexing: palette sizes across every bundling, ragged widths, indices past the palette
    for n, w in ((1, 13), (2, 21), (3, 23), (4, 15), (5, 17), (16, 19), (17, 23), (256, 31)):
        pal = [int(v) for v in rng.integers(0, 1 << 32, n, dtype=np.uint64)]
        bits = 0 if n > 16 else 1 if n > 4 else 2 if n > 2 else 3
        xs = sub_size(w, bits)
        out.append(_lossless(f"ci_n{n}", w, 11, [Tr("ci", data=pal)], Image(literals(rng, xs * 11))))
    # transform orders, predictor on the packed width, all four at once
    w, h = 50, 23
    pal = [int(v) for v in rng.integers(0, 1 << 32, 5, dtype=np.uint64)]
    out.append(_lossless("order_ci_pred", w, h, [Tr("ci", data=pal), Tr("pred", 2, _pred_modes(rng, 25, h, 2, True))],
                         Image(literals(rng, 25 * h))))
    out.append(_lossless("order_pred_cc_sg", w, h, [Tr("pred", 3, _pred_modes(rng, w, h, 3)), Tr("cc", 2, _cc_data(rng, w, h, 2)),
                                                    Tr("sg")], _rand_main(rng, w, h)))
    out.append(_lossless("order_sg_cc_pred_ci", w, h, [Tr("sg"), Tr("cc", 3, _cc_data(rng, w, h, 3)),
                                                       Tr("pred", 2, _pred_modes(rng, w, h, 2)), Tr("ci", data=pal)],
                         Image(literals(rng, 25 * h))))
    out.append(_lossless("order_ci_sg_pred_cc", w, h, [Tr("ci", data=pal[:3]), Tr("sg"), Tr("pred", 2, _pred_modes(rng, 13, h, 2)),
                                                       Tr("cc", 2, _cc_data(rng, 13, h, 2))], Image(literals(rng, 13 * h))))
    # colour cache of every size: literals, copies, hits on what a copy inserted; a cache on a sub-image
    for cb in range(1, 12):
        w, h = 40, 20
        syms = literals(rng, 60, alpha=255, hi=4)
        syms.append(("copy", 30, 1 + (cb % 4)))
        for k in range(w * h - 90):
            syms.append(("cache", int(rng.integers(0, 1 << cb))) if k % 3 else literals(rng, 1)[0])
        out.append(_lossless(f"cache_bits{cb}", w, h, [], Image(syms, cache_bits=cb)))
    modes = _pred_modes(rng, 64, 64, 2)
    sub = [0xFF000000 | (int(m) << 8) for m in modes.reshape(-1)]
    sub_syms = [("lit", v) for v in sub[:40]] + [("cache", cache_index(sub[i % 40], 4)) for i in range(40, len(sub))]
    out.append(_lossless("cache_on_sub_image", 64, 64, [Tr("pred", 2, modes, image=Image(sub_syms, cache_bits=4))],
                         _rand_main(rng, 64, 64)))
    # meta prefix codes at every tile size, group numbers that need the red byte, hundreds of unused groups
    for mb in range(2, 10):
        w, h = 30 + 20 * mb, 20 + 9 * mb
        g = rng.integers(0, 4, (sub_size(h, mb), sub_size(w, mb)))
        out.append(_lossless(f"meta_bits{mb}", w, h, [], Image(literals(rng, w * h), groups=(mb, g))))
    g = rng.choice([0, 150, 299], (sub_size(40, 2), sub_size(48, 2)))
    out.append(_lossless("meta_sparse_300", 48, 40, [], Image(literals(rng, 48 * 40), groups=(2, g))))
    g = rng.choice([3, 256, 700], (sub_size(40, 3), sub_size(40, 3)))
    out.append(_lossless("meta_red_byte", 40, 40, [], Image(literals(rng, 1600), groups=(3, g))))
    # LZ77: every plane code, codes past 120, narrow images where the distance clamps, overlaps, row wraps,
    # every length symbol up to 4096
    out.append(_lossless("lz_plane_codes", 64, 40, [], _copies_image(rng, 64, 40, [(3 + c % 9, c) for c in range(1, 121)])))
    out.append(_lossless("lz_codes_past_120", 57, 30, [], _copies_image(rng, 57, 30, [(5, 120 + d) for d in (1, 2, 7, 57, 300, 500)], lead=600)))
    for w in range(1, 9):
        codes = [c for c in range(1, 121)]
        out.append(_lossless(f"lz_width{w}", w, 120, [], _copies_image(rng, w, 120, [(2, c) for c in codes], lead=16)))
    out.append(_lossless("lz_lengths", 128, 300, [], _copies_image(
        rng, 128, 300, [(L, 1 + (L % 3)) for L in [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385,
                                                   513, 769, 1025, 1537, 2049, 3073, 4096, 4096]])))
    # the largest distance symbols: copies from more than 786 000 pixels back
    big = _copies_image(rng, 1024, 800, [(4096, 121)] * 192 + [(4096, 120 + 600000), (4096, 120 + 786500)], lead=1024)
    out.append(_lossless("lz_far_1024x800", 1024, 800, [], big))
    # prefix codes: long codes (skewed lengths), single-symbol normal codes, code-length code shapes
    out.append(_lossless("codes_long", 70, 40, [], Image(literals(rng, 2800), styles={("*", 0): CodeStyle(kind="normal", skew=True),
                                                                                       ("*", 1): CodeStyle(kind="normal", skew=True)})))
    out.append(_lossless("codes_normal_single", 20, 10, [], Image(literals(rng, 200, alpha=255, hi=1),
                                                                  styles={("*", k): CodeStyle(kind="normal") for k in range(5)})))
    out.append(_lossless("codes_max_symbol", 30, 20, [], Image(literals(rng, 600, lo=0, hi=9),
                                                               styles={("*", k): CodeStyle(kind="normal", max_symbol=True, ncodes=19, nbits_k=k + 1) for k in range(4)})))
    out.append(_lossless("codes_no_rle", 30, 20, [], Image(literals(rng, 600),
                                                           styles={("*", k): CodeStyle(kind="normal", rle=False) for k in range(4)})))
    flat256 = CodeStyle(kind="normal", lens=[8] * 256, rep16_first=True)
    out.append(_lossless("codes_rep16_first", 30, 20, [], Image(literals(rng, 600), styles={("*", 1): flat256, ("*", 2): flat256})))
    out.append(_lossless("codes_simple_shapes", 24, 10, [], Image(
        [("lit", 0xFF000000 | (200 << 16) | (1 << 8) | 7)] * 240,
        styles={("*", 0): CodeStyle(kind="simple", first8=False), ("*", 1): CodeStyle(kind="simple", first8=True),
                ("*", 2): CodeStyle(kind="simple", twice=True)})))
    return out


def alph_payload(w, h, method, filt, pre, rng, transforms=()):
    """An ALPH chunk payload: raw plane or a headerless VP8L stream, filtered residuals at random."""
    hdr = bytes([method | (filt << 2) | (pre << 4)])
    if method == 0:
        return hdr + rng.integers(0, 256, w * h, dtype=np.uint8).tobytes()
    st = Counter()
    if transforms == "ci":
        pal = [0xFF000000 | (int(v) << 8) for v in rng.integers(0, 256, 6)]
        main = Image(literals(rng, sub_size(w, 1) * h, alpha=255, hi=256))
        return hdr + write_vp8l(w, h, [Tr("ci", data=pal)], main, st, header=False)
    main = Image([("lit", 0xFF000000 | (int(g) << 8)) for g in rng.integers(0, 256, w * h)])
    return hdr + write_vp8l(w, h, [], main, st, header=False)


def _alpha_cases():
    out = []
    rng = np.random.default_rng(77)
    k = 0
    for method in (0, 1):
        for filt in range(4):
            for pre in (0, 1):
                w, h = [(1, 7), (13, 9), (33, 17), (2, 5)][k % 4]
                k += 1
                alph = alph_payload(w, h, method, filt, pre, rng, "ci" if k % 3 == 0 else ())
                vp8 = lossy_payload(w, h, k)
                st = Counter({f"alph:m{method}:f{filt}:p{pre}": 1, f"alph:w{w}": 1, "alph:odd_h": h & 1})
                out.append(Case(f"alph_still_m{method}_f{filt}_p{pre}_{w}x{h}", alpha_still(w, h, alph, vp8), "alph_still",
                                st + Counter({"alph:still": 1})))
                out.append(Case(f"alph_anmf_m{method}_f{filt}_p{pre}_{w}x{h}", alpha_anmf(w, h, alph, vp8), "alph_anmf",
                                st + Counter({"alph:anmf": 1})))
    return out


@functools.lru_cache(maxsize=None)
def cases() -> tuple:
    return tuple(_lossless_cases() + _alpha_cases())


def coverage() -> Counter:
    total = Counter()
    for c in cases():
        total.update(c.stats)
    return total


FEATURES = (
    [f"pred:m{m}:{p}" for m in range(16) for p in ("top", "left", "last", "inner")]
    + [f"pred:bits{b}" for b in range(2, 10)] + ["pred:tile_wider", "pred:width1", "pred:width2"]
    + ["cc:neg", "cc:pos"] + [f"cc:bits{b}" for b in range(2, 10)] + ["sg"]
    + [f"ci:n{n}" for n in (1, 2, 3, 4, 5, 16, 17, 256)] + ["ci:ragged", "ci:wrap"] + [f"ci:oob_b{b}" for b in range(4)]
    + ["order:pred_after_ci", "order:all4"]
    + [f"cache:bits{b}" for b in range(1, 12)] + ["cache:sub_image", "cache:hit_from_copy"]
    + [f"meta:bits{b}" for b in range(2, 10)] + ["meta:red_group", "meta:unused_groups"]
    + [f"lz:plane{c}" for c in range(1, 121)] + ["lz:code_gt120", "lz:overlap", "lz:wrap_row"]
    + [f"lz:clamp_w{w}" for w in range(1, 8)] + [f"lz:len_sym{s}" for s in range(24)] + ["lz:dist_sym38", "lz:dist_sym39"]
    + ["code:long", "code:normal_single", "code:max_symbol", "code:rep16", "code:rep17", "code:rep18", "code:rep16_first",
       "code:simple1_1bit", "code:simple1_8bit", "code:simple2", "code:simple_same", "code:ncodes4", "code:ncodes19"]
    + [f"alph:m{m}:f{f}:p{p}" for m in (0, 1) for f in range(4) for p in (0, 1)]
    + ["alph:w1", "alph:odd_h", "alph:still", "alph:anmf"]
)


# ---------------------------------------------------------------- damaged streams


@dataclass
class Damaged:
    name: str
    data: bytes
    group: str


def _cuts(n, every_tail=None, stride=1):
    """Lengths to cut a payload of n bytes to: all of them, or every one in the last `every_tail` bytes and every
    `stride`-th before."""
    if every_tail is None:
        return list(range(n))
    return sorted(set(range(max(0, n - every_tail), n)) | set(range(0, n, stride)))


def _one_image(w, h, st, main, transforms=(), **kw):
    return lossless_file(write_vp8l(w, h, list(transforms), main, Counter(), **kw))


def damaged_cases() -> list:
    from tests.webp_util import chunks_of, webp_golden
    out = []
    by_name = {c.name: c for c in cases()}
    # truncation at every byte of small VP8L payloads, VP8L ALPH payloads (one coded through a palette), and
    # lossy VP8 payloads of 1, 2, 4 and 8 token partitions (the last bytes of each, a stride through the rest)
    for name in ("pred_width2", "cache_bits5", "meta_bits2", "order_ci_pred", "lz_width3"):
        payload = dict(chunks_of(by_name[name].data))[b"VP8L"]
        cuts = _cuts(len(payload)) if len(payload) <= 500 else _cuts(len(payload), 120, len(payload) // 30)
        out += [Damaged(f"{name}_cut{k}", lossless_file(payload[:k]), "trunc_vp8l") for k in cuts]
    rng = np.random.default_rng(9)
    for w, h, tr in ((13, 9, ()), (33, 17, "ci"), (1, 7, "ci")):
        alph = alph_payload(w, h, 1, 1, 0, rng, tr)
        vp8 = lossy_payload(w, h, w)
        cuts = _cuts(len(alph)) if len(alph) <= 300 else _cuts(len(alph), 120, 23)
        out += [Damaged(f"alph_{w}x{h}_cut{k}", alpha_still(w, h, alph[:k], vp8), "trunc_alph") for k in cuts]
    vp8 = lossy_payload(64, 48, 3)
    out += [Damaged(f"vp8_64x48_cut{k}", riff(chunk(b"VP8 ", vp8[:k])), "trunc_vp8") for k in _cuts(len(vp8))]
    g = webp_golden()
    for name in ("lossy111", "lossy112", "lossy113"):
        vp8 = dict(chunks_of(g[f"webp_{name}"].tobytes()))[b"VP8 "]
        out += [Damaged(f"{name}_cut{k}", riff(chunk(b"VP8 ", vp8[:k])), "trunc_vp8_partitions")
                for k in _cuts(len(vp8), 160, 89)]
    # ALPH header byte: reserved bits, pre-processing and method values the format does not define
    w, h = 13, 9
    vp8 = lossy_payload(w, h, 13)
    for method in (0, 1):
        body = alph_payload(w, h, method, 0, 0, rng)[1:]
        for rsrv in (1, 2, 3):
            out.append(Damaged(f"alph_m{method}_rsrv{rsrv}", alpha_still(w, h, bytes([method | rsrv << 6]) + body, vp8), "alph_header"))
        for pre in (2, 3):
            out.append(Damaged(f"alph_m{method}_pre{pre}", alpha_still(w, h, bytes([method | pre << 4]) + body, vp8), "alph_header"))
    for method in (2, 3):
        out.append(Damaged(f"alph_method{method}", alpha_still(w, h, bytes([method]) + bytes(w * h), vp8), "alph_header"))
    # prefix codes: simple symbols past the distance alphabet (40), incomplete, over-subscribed and empty codes
    lits = literals(rng, 40 * 8)
    copy = Image(lits[:100] + [("copy", 20, 1)] + lits[120:])

    def code_case(name, k, style):
        im = Image(copy.syms, styles={("*", k): style})
        out.append(Damaged(name, _one_image(40, 8, None, im), "codes"))
    code_case("simple_one_past_alphabet", 4, CodeStyle(raw_simple=(1, 1, 45, 0)))
    code_case("simple_second_past_alphabet", 4, CodeStyle(raw_simple=(2, 1, prefix_encode(1)[0], 45)))
    code_case("simple_first_past_alphabet", 4, CodeStyle(raw_simple=(2, 1, 45, prefix_encode(1)[0])))
    code_case("simple_one_last_in_alphabet", 4, CodeStyle(raw_simple=(2, 1, prefix_encode(1)[0], 39)))
    code_case("incomplete", 4, CodeStyle(kind="normal", lens=[1, 2] + [0] * 38))
    code_case("over_subscribed", 4, CodeStyle(kind="normal", lens=[1, 1, 1] + [0] * 37))
    code_case("zero_symbols", 4, CodeStyle(kind="normal", lens=[0] * 40))
    code_case("green_incomplete", 0, CodeStyle(kind="normal", lens=[2] * 3 + [0] * 277))
    # colour cache size fields outside 1..11 (an index past the cache cannot be coded: the green alphabet ends there)
    for bits in (0, 12, 13, 14, 15):
        out.append(Damaged(f"cache_field{bits}", _one_image(20, 4, None, Image(literals(rng, 80), cache_field=bits)), "cache"))
    # back-references before the first pixel and past the last
    lits = literals(rng, 30 * 6)
    out.append(Damaged("copy_before_first", _one_image(30, 6, None, Image(lits[:5] + [("copy", 3, 120 + 6)] + lits[8:])), "lz"))
    out.append(Damaged("copy_at_first", _one_image(30, 6, None, Image([("copy", 3, 121)] + lits[3:])), "lz"))
    out.append(Damaged("copy_past_last", _one_image(30, 6, None, Image(lits[:170] + [("copy", 20, 121)])), "lz"))
    out.append(Damaged("copy_to_last", _one_image(30, 6, None, Image(lits[:170] + [("copy", 10, 121)])), "lz"))
    # a transform twice, the header's version bits
    for kind, tr in (("sg", Tr("sg")), ("pred", Tr("pred", 2, np.zeros((2, 8), np.int64)))):
        data = _one_image(30, 6, None, Image(literals(rng, 180)), [tr, tr])
        out.append(Damaged(f"transform_twice_{kind}", data, "transforms"))
    for v in (1, 4, 7):
        out.append(Damaged(f"version{v}", _one_image(10, 3, None, Image(literals(rng, 30)), version=v), "header"))
    return out
