"""Test infrastructure: a minimal GIF writer and an LZW encoder whose every choice the caller steers (minimum code size,
where clear codes go, EOF code or not, what follows it, sub-block layout), damaged variants of its streams, and
counts of the decoder corners each stream reaches.

The encoder keeps giflib's decoder state (DGifDecompressInput) as it writes: `running` counts the codes since the last
clear (+ clear + 2) and the width grows by one bit, at most once per code, when `running` passes 1 << bits, up to 12
bits.  So a code is as wide as the bit length of the largest entry it may name (the next free entry - 1), except the
first code after a clear at minimum code size 0, which is read at 1 bit.  Growing one entry early instead decodes to
garbage, which tests/test_oracle_gif_streams.py would catch.

`cases()` is the catalogue both the CPU check of this generator (against the C oracle) and the device tests use.  Every
file is an animation of at least two frames; a well-formed one carries its composited frames, built here in numpy from
the encoded indices."""
import functools
from dataclasses import dataclass, field

import numpy as np

# ---------------------------------------------------------------- container


def sub_blocks(data: bytes, size=255, seed=0) -> bytes:
    """`data` as sub-blocks of `size` bytes (255, 1, or "random" for 1..255 drawn from `seed`) + the terminator."""
    rng = np.random.default_rng(seed)
    out = bytearray()
    o = 0
    while o < len(data):
        n = int(rng.integers(1, 256)) if size == "random" else size
        out += bytes([len(data[o:o + n])]) + data[o:o + n]
        o += n
    return bytes(out) + b"\x00"


def lzw_literals(idx: np.ndarray, bpp: int) -> bytes:
    """Every pixel as a literal code; a clear code before the table would widen the codes."""
    clear, eoi, width = 1 << bpp, (1 << bpp) + 1, bpp + 1
    codes = []
    flat = idx.reshape(-1).tolist()
    run = (1 << bpp) - 2
    for o in range(0, len(flat), run):
        codes.append(clear)
        codes += flat[o:o + run]
    codes.append(eoi)
    return pack([(c, width) for c in codes])


def table_bits(pal) -> int:
    n = len(pal) // 3
    b = 1
    while (1 << b) < n:
        b += 1
    return b


def gcb(disposal=0, delay=5, transparent=None) -> bytes:
    return bytes([0x21, 0xF9, 4, (disposal << 2) | (transparent is not None), delay & 255, delay >> 8,
                  transparent or 0, 0])


def comment(text: bytes) -> bytes:
    return b"\x21\xFE" + sub_blocks(text)


def app(ident: bytes, payload: bytes) -> bytes:
    return b"\x21\xFF\x0b" + ident[:11] + sub_blocks(payload)


NETSCAPE = b"\x21\xFF\x0bNETSCAPE2.0\x03\x01\x00\x00\x00"


def interlace_rows(idx: np.ndarray) -> np.ndarray:
    """The rows of a frame in the order an interlaced frame stores them."""
    return np.concatenate([idx[0::8], idx[4::8], idx[2::4], idx[1::2]])


def write_gif(w, h, frames, gct=None, bg=0, trailer_ext=b"", loop=True) -> bytes:
    """frames: dicts with idx (rows x cols palette indices), and optionally left, top, local (RGB bytes), interlace,
    gcb (bytes or None for none), pre (extension bytes in front of the frame).  The code stream is every pixel as a
    literal unless the frame has `stream` = (minimum code size, code stream bytes), cut into sub-blocks of `block`
    bytes (see sub_blocks)."""
    out = bytearray(b"GIF89a" + w.to_bytes(2, "little") + h.to_bytes(2, "little"))
    if gct is not None:
        out += bytes([0x80 | 0x70 | (table_bits(gct) - 1), bg, 0]) + gct
    else:
        out += bytes([0x70, bg, 0])
    if loop:
        out += NETSCAPE
    for k, f in enumerate(frames):
        idx = np.asarray(f["idx"], np.uint8)
        fh, fw = idx.shape
        out += f.get("pre", b"")
        if f.get("gcb", b"") is not None:
            out += f.get("gcb") or gcb()
        local = f.get("local")
        flags = (0x80 | (table_bits(local) - 1) if local is not None else 0) | (0x40 if f.get("interlace") else 0)
        out += b"\x2C" + f.get("left", 0).to_bytes(2, "little") + f.get("top", 0).to_bytes(2, "little")
        out += fw.to_bytes(2, "little") + fh.to_bytes(2, "little") + bytes([flags])
        if local is not None:
            out += local
        if "stream" in f:
            min_code, data = f["stream"]
        else:
            min_code = max(2, table_bits(local if local is not None else gct))
            data = lzw_literals(interlace_rows(idx) if f.get("interlace") else idx, min_code)
        out += bytes([min_code]) + sub_blocks(data, f.get("block", 255), seed=k)
    out += trailer_ext + b";"
    return bytes(out)


# ---------------------------------------------------------------- LZW encoder


@dataclass
class LzwStats:
    """What a code stream makes the decoder do.  A lane is a code's place in the device decoder's rounds of 32 codes,
    which start after every clear code (and, at minimum code size 0, after the first code behind it)."""
    codes: int = 0          # data codes (not clear / EOF)
    kwkwk: int = 0          # codes equal to the entry they create
    kwkwk_lane0: int = 0    # ... read in lane 0, whose previous string comes from the round before
    kwkwk_chain: int = 0    # longest run of KwKwK codes in consecutive lanes of one round
    near: int = 0           # codes naming an entry created fewer than 32 codes earlier (KwKwK included)
    max_width: int = 0
    frozen: int = 0         # data codes read while the table is full
    clear_widths: set = field(default_factory=set)
    max_string: int = 0

    def merge(self, o: "LzwStats") -> "LzwStats":
        return LzwStats(self.codes + o.codes, self.kwkwk + o.kwkwk, self.kwkwk_lane0 + o.kwkwk_lane0,
                        max(self.kwkwk_chain, o.kwkwk_chain), self.near + o.near, max(self.max_width, o.max_width),
                        self.frozen + o.frozen, self.clear_widths | o.clear_widths,
                        max(self.max_string, o.max_string))


@dataclass
class Code:
    code: int
    width: int
    top: int        # the entry this code creates if it names a string and follows one; 4096 = the table is full
    pixels: int     # pixels decoded in front of it
    data: bool = False  # names a string (not a clear or EOF code)


class _Stream:
    """The codes written so far, and the decoder state behind them."""

    def __init__(self, min_code):
        self.mc, self.clear, self.eof = min_code, 1 << min_code, (1 << min_code) + 1
        self.codes: list[Code] = []
        self.stats = LzwStats()
        self.pixels = 0
        self._reset()

    def _reset(self):
        self.bits, self.running, self.top = self.mc + 1, self.clear + 2, self.clear + 2
        self.prev_len = 0   # 0: no previous string in this segment
        self.seg = 0        # data codes since the clear
        self.born, self.lens = {}, {}
        self.chain = 0

    def _put(self, code):
        self.codes.append(Code(code, self.bits, min(self.top, 4096), self.pixels, code not in (self.clear, self.eof)))
        self.stats.max_width = max(self.stats.max_width, self.bits)
        if self.running < 4097:
            self.running += 1
            if self.running > (1 << self.bits) and self.bits < 12:
                self.bits += 1

    def put_clear(self):
        self.stats.clear_widths.add(self.bits)
        self._put(self.clear)
        self._reset()

    def put_eof(self):
        self._put(self.eof)

    def put_data(self, code):
        s = self.stats
        lane = self.seg % 32 if self.mc else (0 if self.seg == 0 else (self.seg - 1) % 32)
        creates = self.prev_len > 0 and self.top < 4096
        kwkwk = creates and code == self.top
        if code < self.clear:
            n = 1
        elif kwkwk:
            n = self.prev_len + 1
        else:
            n = self.lens[code]
        if code > self.eof and self.seg - self.born.get(code, self.seg) < 32:
            s.near += 1
        self.chain = (self.chain + 1 if lane > 0 else 1) if kwkwk else 0
        s.kwkwk += kwkwk
        s.kwkwk_lane0 += kwkwk and lane == 0
        s.kwkwk_chain = max(s.kwkwk_chain, self.chain)
        s.frozen += self.prev_len > 0 and self.top >= 4096
        s.max_string = max(s.max_string, n)
        s.codes += 1
        self._put(code)
        if creates:
            self.born[self.top], self.lens[self.top] = self.seg, self.prev_len + 1
            self.top += 1
        self.prev_len = n
        self.pixels += n
        self.seg += 1


def pack(codes) -> bytes:
    """(code, width) pairs, LSB first."""
    acc = nb = 0
    out = bytearray()
    for c, w in codes:
        acc |= c << nb
        nb += w
        while nb >= 8:
            out.append(acc & 255)
            acc >>= 8
            nb -= 8
    if nb:
        out.append(acc & 255)
    return bytes(out)


def _pack(codes: list[Code]) -> bytes:
    return pack([(c.code, c.width) for c in codes])


def lzw_encode(idx, min_code, clear="full", initial_clear=True, double_clear=False, eof=True, tail=b""):
    """Palette indices (all < 1 << min_code) -> (code stream, LzwStats, [Code]).

    clear: "full"      a clear code when the next free entry would be 4095 (giflib's encoder);
           "deferred"  never: once the table is full every code is 12 bits wide against the frozen table;
           K or [K..]  a clear code behind every K data codes of a segment (a list is used in turn).
    initial_clear: start with a clear code; double_clear: every clear code twice; eof: end with the EOF code;
    tail: bytes behind the last code (garbage the decoder must not read)."""
    flat = np.asarray(idx, np.uint8).reshape(-1).tolist()
    assert max(flat, default=0) < 1 << min_code, "a palette index would read as a control code"
    s = _Stream(min_code)
    ks = None if isinstance(clear, str) else ([clear] if isinstance(clear, int) else list(clear))
    nclear = 0

    def put_clear():
        nonlocal nclear
        s.put_clear()
        if double_clear:
            s.put_clear()
        nclear += 1

    if initial_clear:
        put_clear()
    table = {}
    w = -1
    for p in flat:
        if w < 0:
            w = p
            continue
        e = table.get(w << 8 | p)
        if e is not None:
            w = e
            continue
        s.put_data(w)
        if (clear == "full" and s.top >= 4095) or (ks is not None and s.seg >= ks[(nclear - initial_clear) % len(ks)]):
            put_clear()
            table = {}
        elif s.top < 4096:
            table[w << 8 | p] = s.top
        w = p
    if w >= 0:
        s.put_data(w)
    if eof:
        s.put_eof()
    return _pack(s.codes) + tail, s.stats, s.codes


# ---------------------------------------------------------------- damaged streams: each cuts an otherwise valid stream
# at (or from) code index `at`


def truncate_in_code(codes: list[Code], at: int) -> bytes:
    """The data ends inside a code: the first code from `at` on that a byte boundary splits keeps only its low bits."""
    start = [0]
    for c in codes:
        start.append(start[-1] + c.width)
    for i in range(at, len(codes)):
        nbytes = -(-start[i] // 8)
        if start[i] < 8 * nbytes < start[i + 1]:
            return _pack(codes)[:nbytes]
    raise ValueError("no code from `at` on can be cut inside")


def eof_early(codes: list[Code], at: int, eof: int) -> bytes:
    """The EOF code in place of code `at`, before the frame is full."""
    return _pack(codes[:at] + [Code(eof, codes[at].width, 0, 0)])


def above_top(codes: list[Code], at: int) -> bytes:
    """The first data code from `at` on that has room for it becomes top + 1, an entry nobody has made; the codes
    behind stay."""
    for i in range(at, len(codes)):
        c = codes[i]
        if c.data and c.top < 4095 and c.top + 1 < 1 << c.width:
            return _pack(codes[:i] + [Code(c.top + 1, c.width, 0, 0)] + codes[i + 1:])
    raise ValueError("no room for a code above top")


def kwkwk_after_clear(codes: list[Code], at: int, min_code: int) -> bytes:
    """A clear code in front of code `at`, then the code of the entry the next code would make: KwKwK with no previous
    string.  (At minimum code size 0 the first code after a clear is 1 bit wide and cannot be that code.)"""
    assert min_code > 0
    clear = 1 << min_code
    return _pack(codes[:at] + [Code(clear, codes[at].width, 0, 0), Code(clear + 2, min_code + 1, 0, 0)]
                 + codes[at:])


# ---------------------------------------------------------------- content


def palette(seed, n) -> bytes:
    return np.random.default_rng(seed).integers(0, 256, n * 3, dtype=np.uint8).tobytes()


def content(kind, h, w, n, seed=0) -> np.ndarray:
    """h x w indices below n: flat, noise, period (a short repeating run: strings name entries made a few codes
    earlier), gradient."""
    rng = np.random.default_rng(seed)
    if kind == "flat":
        return np.full((h, w), min(1, n - 1) if n > 1 else 0, np.uint8)
    if kind == "noise":
        return rng.integers(0, n, (h, w)).astype(np.uint8)
    if kind == "period":
        p = int(rng.integers(2, 6))
        return (np.arange(h * w).reshape(h, w) % p * (n - 1) // max(p - 1, 1)).astype(np.uint8)
    if kind == "gradient":
        y, x = np.mgrid[0:h, 0:w]
        return ((x * n // max(w, 1) + y // 3) % n).astype(np.uint8)
    raise ValueError(kind)


def composite(cw, ch, gct, frames, bg=0) -> list:
    """Ground truth for files of opaque frames without disposal: the first frame starts from the background colour
    (ref giflib.cpp:595-636), indices at or above the colour count leave the pixel as it was, frames are clipped."""
    pal = np.frombuffer(gct, np.uint8).reshape(-1, 3)
    n = len(pal)
    canvas = np.empty((ch, cw, 4), np.uint8)
    canvas[...] = [pal[bg, 2], pal[bg, 1], pal[bg, 0], 255] if bg < n else 255
    out = []
    for f in frames:
        idx = np.asarray(f["idx"])
        l, t = f.get("left", 0), f.get("top", 0)
        reg = idx[:max(0, min(idx.shape[0], ch - t)), :max(0, min(idx.shape[1], cw - l))]
        view = canvas[t:t + reg.shape[0], l:l + reg.shape[1]]
        ok = reg < n
        view[ok] = np.concatenate([pal[reg[ok].astype(int)][:, ::-1], np.full((int(ok.sum()), 1), 255, np.uint8)], 1)
        out.append(canvas.copy())
    return out


# ---------------------------------------------------------------- the catalogue


@dataclass
class Case:
    name: str
    gif: bytes
    frames: list              # composited BGRA canvases the decoder delivers: all, or those in front of a damaged one
    stats: LzwStats           # of the streams under test
    damage: str | None = None  # the kind of damage of a stream under test
    min_codes: set = field(default_factory=set)
    interlaced_heights: set = field(default_factory=set)
    overrun: int = 0          # pixels the last string of a frame has beyond the frame


def coded_frame(idx, min_code, extra=None, interlace=False, block=255, **kw):
    """A frame dict for write_gif whose stream encodes `idx` (plus `extra` indices behind the frame's last pixel) with
    lzw_encode(**kw); returns (frame, stats, codes)."""
    rows = interlace_rows(idx) if interlace else idx
    flat = rows.reshape(-1) if extra is None else np.concatenate([rows.reshape(-1), np.asarray(extra, np.uint8)])
    data, stats, codes = lzw_encode(flat, min_code, **kw)
    return dict(idx=idx, stream=(min_code, data), interlace=interlace, block=block), stats, codes


def _companion(cw, ch, n, seed):
    """A small literal-coded frame at the origin (every case is an animation of at least two frames)."""
    return dict(idx=content("gradient", min(ch, 8), min(cw, 16), n, seed))


def _file(name, cw, ch, gct, tested, stats, first=True, damage=None, **kw) -> Case:
    """An animation of the frames under test (`tested`) and a companion frame: behind them, or in front of them when
    `first` is False.  A damaged case decodes only the frames in front of its damaged one."""
    n = len(gct) // 3
    comp = _companion(cw, ch, n, len(name))
    frames = tested + [comp] if first else [comp] + tested
    gif = write_gif(cw, ch, frames, gct=gct)
    gt = composite(cw, ch, gct, frames)
    return Case(name, gif, gt[:0 if first else 1] if damage else gt, stats, damage, **kw)


def _single(name, idx, min_code, pal_colors, seed=0, block=255, extra=None, **kw) -> Case:
    h, w = idx.shape
    gct = palette(seed + 1000, pal_colors)
    f, stats, codes = coded_frame(idx, min_code, extra=extra, block=block, **kw)
    return _file(name, w, h, gct, [f], stats, min_codes={min_code}, overrun=_string_overrun(codes, h * w))


def _string_overrun(codes: list[Code], npix) -> int:
    """Pixels the string that fills the frame has beyond the frame's end (0 when a string ends exactly there)."""
    for a, b in zip(codes, codes[1:]):
        if a.pixels < npix < b.pixels:
            return b.pixels - npix
    return 0


@functools.lru_cache(maxsize=None)
def cases() -> tuple:
    out = []
    # table policies on noise (no runs: the table fills fastest), sizes that are no multiple of 32
    for mc, (w, h) in ((2, (333, 201)), (4, (301, 97)), (8, (257, 255))):
        idx = content("noise", h, w, 1 << mc, mc)
        out.append(_single(f"noise_full_mc{mc}", idx, mc, 1 << mc, seed=mc))
        out.append(_single(f"noise_deferred_mc{mc}", idx, mc, 1 << mc, seed=mc, clear="deferred", block="random"))
    out.append(_single("noise_deferred_2000x1500", content("noise", 1501, 1999, 256, 7), 8, 256, seed=7,
                       clear="deferred"))
    out.append(_single("frozen_4100_wide", content("noise", 23, 4100, 256, 8), 8, 256, seed=8, clear="deferred",
                       initial_clear=False))
    # clear codes at every width 3..12, two in a row, none at the start
    out.append(_single("clear_every_width", content("noise", 111, 256, 4, 9), 2, 4, seed=9,
                       clear=[3, 11, 27, 59, 123, 251, 507, 1019, 2043, 3000], double_clear=True))
    out.append(_single("clear_every_7", content("period", 45, 77, 16, 10), 4, 16, seed=10, clear=7, double_clear=True,
                       block=1))
    out.append(_single("no_initial_clear_mc3", content("period", 64, 96, 8, 11), 3, 8, seed=11, clear="deferred",
                       initial_clear=False))
    out.append(_single("no_initial_clear_mc1", content("noise", 90, 91, 2, 12), 1, 2, seed=12, initial_clear=False))
    # every minimum code size, palettes of other sizes than the code size says
    out.append(_single("flat_mc0_2900x2900", np.zeros((2900, 2900), np.uint8), 0, 2, seed=13, clear="deferred"))
    out.append(_single("flat_mc0_full", np.zeros((111, 130), np.uint8), 0, 4, seed=14))
    out.append(_single("flat_mc1", content("flat", 200, 333, 2, 15), 1, 2, seed=15, clear="deferred"))
    out.append(_single("period_mc1", content("period", 33, 65, 2, 16), 1, 2, seed=16, block="random"))
    for mc in (3, 5, 6, 7):
        out.append(_single(f"period_mc{mc}", content("period", 40 + mc, 50 + mc, 1 << mc, 20 + mc), mc, 1 << mc,
                           seed=20 + mc))
        out.append(_single(f"gradient_mc{mc}", content("gradient", 30 + mc, 70 - mc, 1 << mc, 30 + mc), mc, 1 << mc,
                           seed=30 + mc, block="random"))
    out.append(_single("mc8_pal4_out_of_palette", content("noise", 61, 67, 256, 40), 8, 4, seed=40))
    out.append(_single("mc2_pal256", content("gradient", 48, 50, 4, 41), 2, 256, seed=41))
    out.append(_single("one_pixel_mc2", np.array([[3]], np.uint8), 2, 4, seed=42))
    out.append(_single("one_pixel_mc0", np.zeros((1, 1), np.uint8), 0, 2, seed=43, initial_clear=False, eof=False))
    # the frame fills inside a round: more codes, garbage or nothing behind; the last string longer than the room
    idx = content("flat", 7, 45, 4, 44)
    out.append(_single("fill_then_more_codes", idx, 2, 4, seed=44, extra=np.ones(900, np.uint8)))
    out.append(_single("fill_then_garbage", content("period", 9, 37, 4, 45), 2, 4, seed=45, eof=False,
                       tail=bytes(range(7, 250, 3)), extra=np.zeros(300, np.uint8), block=1))
    out.append(_single("fill_no_eof", content("noise", 13, 29, 16, 46), 4, 16, seed=46, eof=False))
    out.append(_single("eof_then_garbage_blocks", content("gradient", 17, 19, 8, 47), 3, 8, seed=47,
                       tail=np.random.default_rng(47).integers(0, 256, 700, dtype=np.uint8).tobytes(), block="random"))
    out += _compositor_cases()
    out += [_reel("reel_96x64", 96, 64, 100, 90), _reel("reel_61x47", 61, 47, 100, 91)]
    out += _damaged_cases()
    return tuple(out)


def _reel(name, cw, ch, nframes, seed) -> Case:
    """An animation of `nframes` frames whose every knob is drawn at random: code size, clear policy, EOF, garbage
    behind it, sub-block size, interlace, content, size and position (on, across or off the canvas)."""
    rng = np.random.default_rng(seed)
    gct = palette(seed, 64)
    frames, stats, mcs = [], LzwStats(), set()
    for k in range(nframes):
        mc = int(rng.integers(2, 9))
        fw, fh = int(rng.integers(1, cw + 12)), int(rng.integers(1, ch + 12))
        idx = content(("flat", "noise", "period", "gradient")[k % 4], fh, fw, min(1 << mc, 80), seed * 1000 + k)
        f, s, _ = coded_frame(idx, mc, interlace=bool(rng.integers(0, 2)), block=(255, 1, "random")[k % 3],
                              clear=("full", "deferred", int(rng.integers(1, 40)))[int(rng.integers(0, 3))],
                              double_clear=bool(rng.integers(0, 2)), initial_clear=bool(rng.integers(0, 4)),
                              eof=bool(rng.integers(0, 4)), tail=bytes(int(rng.integers(0, 3)) * [0xA5]))
        f["left"], f["top"] = int(rng.integers(0, cw + 4)), int(rng.integers(0, ch + 4))
        frames.append(f)
        stats = stats.merge(s)
        mcs.add(mc)
    return _file(name, cw, ch, gct, frames, stats, min_codes=mcs)


def _compositor_cases():
    """Interlaced frames of every height 1..17 and frames hanging off the right / bottom edge or lying outside."""
    cw, ch = 40, 20
    gct = palette(50, 16)
    frames, stats = [], LzwStats()
    for k, fh in enumerate(range(1, 18)):
        fw = 3 + 2 * k
        mc = 4 if k % 3 else 8
        f, s, _ = coded_frame(content(("noise", "period", "gradient")[k % 3], fh, fw, 16 if mc == 4 else 40, 60 + k), mc,
                              interlace=True, block=(255, 1, "random")[k % 3], clear=("full", "deferred", 5)[k % 3])
        f["left"], f["top"] = (k * 5) % 37, (k * 3) % 19   # some hang off the right / bottom edge
        frames.append(f)
        stats = stats.merge(s)
    heights = set(range(1, 18))
    out = [_file("interlaced_heights_1_17", cw, ch, gct, frames, stats, min_codes={4, 8}, interlaced_heights=heights)]
    frames, stats = [], LzwStats()
    for k, (l, t, fw, fh) in enumerate(((30, 2, 17, 5), (3, 14, 9, 11), (33, 15, 12, 9), (40, 0, 5, 5), (0, 20, 6, 3),
                                        (45, 31, 4, 4), (0, 0, 40, 20))):
        f, s, _ = coded_frame(content("noise", fh, fw, 64, 70 + k), 6, clear="deferred")
        f["left"], f["top"] = l, t
        frames.append(f)
        stats = stats.merge(s)
    out.append(_file("off_canvas_out_of_palette", cw, ch, palette(51, 32), frames, stats, min_codes={6}))
    return out


def _damaged_cases():
    out = []
    h, w, mc = 60, 80, 4
    idx = content("noise", h, w, 16, 80)
    gct = palette(81, 16)
    _, stats, codes = coded_frame(idx, mc)
    eof = (1 << mc) + 1

    def add(kind, name, data, min_code=mc, st=stats, block=255):
        f = dict(idx=np.zeros((h, w), np.uint8), stream=(min_code, data), block=block)
        out.append(_file(f"damaged_{name}", w, h, gct, [f], st, first=False, damage=kind, min_codes={min_code}))

    for at in (0, 1, 31, 32, 45, 700):   # code indices: the initial clear code is code 0
        add("truncated", f"truncated_at{at}", truncate_in_code(codes, at))
        add("eof_early", f"eof_early_at{at}", eof_early(codes, at, eof))
        add("above_top", f"above_top_at{at}", above_top(codes, at), block=1)
        add("kwkwk_after_clear", f"kwkwk_after_clear_at{at}", kwkwk_after_clear(codes, at, mc), block="random")
    add("empty_stream", "empty_stream", b"")
    # the same kinds in a stream whose table is frozen, and at minimum code size 0
    _, fst, fcodes = coded_frame(content("noise", h, w, 256, 82), 8, clear="deferred")
    add("eof_early", "eof_early_frozen", eof_early(fcodes, 4500, 257), min_code=8, st=fst)
    add("truncated", "truncated_frozen", truncate_in_code(fcodes, 4600), min_code=8, st=fst)
    _, zst, zcodes = coded_frame(np.zeros((h, w), np.uint8), 0)
    add("truncated", "truncated_mc0", truncate_in_code(zcodes, 1), min_code=0, st=zst)
    add("eof_early", "eof_early_mc0", eof_early(zcodes, 2, 2), min_code=0, st=zst)
    add("above_top", "above_top_mc0", above_top(zcodes, 1), min_code=0, st=zst)
    return out
