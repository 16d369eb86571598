"""Test infrastructure: a catalogue of GIF encoder cases, a reader of the GIF files the encoder writes, and a plain
Python model of the reference's palette mapping that counts the corners each case reaches.

A case is a source GIF plus the BGRA frames the encoder is given:
  file cases      `frames` is None: the encoder gets the source's own composited frames, so the case also runs through
                  the heterogeneous batch (ImageOpsResize to the source size is a plain copy);
  designed cases  `frames` holds arbitrary BGRA frames (colours off the palette, alpha 127 / 128, frames smaller than
                  the canvas); only the per-image encoder takes those.

The palette mapping (ref giflib.cpp:934-1098) keeps a memo of the best entry per 15-bit crushed colour; the first pixel
to consult a bucket decides its entry, from its own colour when it is near black / white (every channel < 15 or > 240)
and from the bucket midpoint otherwise, and the memo lives on across consecutive frames whose colour maps are
byte-equal.  `map_frames` restates that walk serially and counts what it meets (ties, thresholds, owners whose stored
distance and own distance disagree, ...), so a test can assert both that the oracle's indices are the model's and that
every corner is reached.  `read_gif` counts the LZW side: clear codes, code widths, sub-block lengths, interlace."""
import functools
from collections import Counter
from dataclasses import dataclass, field

import numpy as np

from tests.gif_streams import content, gcb, palette, write_gif

# ---------------------------------------------------------------- reading the encoder's output


def _sub_blocks(d, p):
    lens, data = [], bytearray()
    while True:
        n = d[p]
        p += 1
        if n == 0:
            return bytes(data), lens, p
        lens.append(n)
        data += d[p:p + n]
        p += n


def lzw_read(data: bytes, min_code: int, npix: int) -> dict:
    """Decodes one code stream; returns the indices and what the stream did.  A clear code is `full` when the table
    held 4095 entries as it came (the encoder's clear-on-full); `last_fill` is set when the stream's last full clear
    has exactly one data code behind it, i.e. the frame's last new string was the one that filled the table."""
    clear, eoi = 1 << min_code, (1 << min_code) + 1
    acc = nb = p = 0
    width = min_code + 1
    table = [bytes([i]) for i in range(clear)] + [b"", b""]
    prev = None
    out = bytearray()
    st = dict(clears=0, full_clears=0, clear_widths=set(), widths=set(), codes=0, max_string=0, after_full=-1, eoi=False)
    while True:
        while nb < width and p < len(data):
            acc |= data[p] << nb
            nb += 8
            p += 1
        if nb < width:
            break
        code = acc & ((1 << width) - 1)
        acc >>= width
        nb -= width
        st["widths"].add(width)
        if code == clear:
            st["clears"] += 1
            st["clear_widths"].add(width)
            if len(table) == 4095:
                st["full_clears"] += 1
                st["after_full"] = 0
            table = table[:clear + 2]
            width, prev = min_code + 1, None
            continue
        if code == eoi:
            st["eoi"] = True
            break
        st["codes"] += 1
        if st["after_full"] >= 0:
            st["after_full"] += 1
        if prev is None:
            s = table[code]
        else:
            s = table[code] if code < len(table) else table[prev] + table[prev][:1]
            if len(table) < 4096:
                table.append(table[prev] + s[:1])
        st["max_string"] = max(st["max_string"], len(s))
        out += s
        prev = code
        if len(table) == 1 << width and width < 12:
            width += 1
    assert len(out) >= npix, "the code stream ends before the frame is full"
    st["last_fill"] = st.pop("after_full") == 1
    st["idx"] = np.frombuffer(bytes(out[:npix]), np.uint8)
    return st


def deinterlace(rows: np.ndarray) -> np.ndarray:
    h = rows.shape[0]
    order = [y for y0, dy in ((0, 8), (4, 8), (2, 4), (1, 2)) for y in range(y0, h, dy)]
    out = np.empty_like(rows)
    out[order] = rows
    return out


def read_gif(d: bytes) -> dict:
    """The container and every frame of a GIF the encoder wrote: palette, graphic control block, descriptor, sub-block
    lengths, and lzw_read's counts and indices (in raster order)."""
    assert d[:6] == b"GIF89a" and d[-1] == 0x3B
    sw, sh, packed = int.from_bytes(d[6:8], "little"), int.from_bytes(d[8:10], "little"), d[10]
    p = 13
    gct = None
    if packed & 0x80:
        n = 1 << ((packed & 7) + 1)
        gct, p = d[p:p + 3 * n], p + 3 * n
    frames, g = [], None
    while d[p] != 0x3B:
        if d[p] == 0x21:
            label = d[p + 1]
            body, lens, p = _sub_blocks(d, p + 2)
            if label == 0xF9 and lens[0] == 4:
                g = dict(disposal=(body[0] >> 2) & 7, transparent=body[3] if body[0] & 1 else -1)
            continue
        assert d[p] == 0x2C
        fw, fh, flags = int.from_bytes(d[p + 5:p + 7], "little"), int.from_bytes(d[p + 7:p + 9], "little"), d[p + 9]
        p += 10
        local = None
        if flags & 0x80:
            n = 1 << ((flags & 7) + 1)
            local, p = d[p:p + 3 * n], p + 3 * n
        min_code = d[p]
        data, lens, p = _sub_blocks(d, p + 1)
        st = lzw_read(data, min_code, fw * fh)
        rows = st.pop("idx").reshape(fh, fw)
        interlace = bool(flags & 0x40)
        frames.append(dict(width=fw, height=fh, interlace=interlace, local=local, colors=local or gct,
                           transparent=(g or {}).get("transparent", -1), disposal=(g or {}).get("disposal", 0),
                           min_code=min_code, blocks=lens, data_len=len(data),
                           idx=deinterlace(rows) if interlace else rows, **st))
        g = None
    return dict(width=sw, height=sh, gct=gct, frames=frames)


# ---------------------------------------------------------------- the palette mapping, serially, with its corners

def _l1(pal: np.ndarray, c) -> np.ndarray:
    return np.abs(pal - np.asarray(c, np.int64)).sum(1)


def _straddles(c: tuple) -> bool:
    """A bucket whose pixels fall on both sides of a threshold: channels all in 0..15 with one in 8..15, or all in
    240..255 with one in 240..247."""
    lo = all(v >> 3 <= 1 for v in c) and any(v >> 3 == 1 for v in c)
    hi = all(v >> 3 >= 30 for v in c) and any(v >> 3 == 30 for v in c)
    return lo or hi


def map_frames(frames, out: dict) -> Counter:
    """Runs the reference's palette mapping over the BGRA `frames` the encoder was given, with the palettes,
    transparent indices and disposals `out` (read_gif of the encoder's output) carries, asserts each frame's indices
    equal the output's, and counts the corners met."""
    f_ = Counter()
    sw, sh = out["width"], out["height"]
    prev = np.zeros((sh, sw, 4), np.uint8)
    memo, seen, last = {}, [], None
    pos = 0
    for k, (src, of) in enumerate(zip(frames, out["frames"])):
        colors, T = bytes(of["colors"]), of["transparent"]
        pal = np.frombuffer(colors, np.uint8).reshape(-1, 3).astype(np.int64)
        n = len(pal)
        if last is not None and last[0] == colors:
            pos += 1
            f_["memo_carried"] += 1
            if (last[1] is None) != (of["local"] is None):
                f_["local_equal_to_global"] += 1
        else:
            if last is not None and colors in seen:
                f_["palette_changes_back"] += 1
            if last is not None and (colors.startswith(last[0]) or last[0].startswith(colors)):
                f_["equal_bytes_other_count"] += 1
            memo, pos = {}, 0
        seen.append(colors)
        prev_valid = k > 0 and out["frames"][k - 1]["disposal"] in (0, 1)
        if k > 0 and T != -1:
            f_["prev_disposal_01" if prev_valid else "prev_disposal_23"] += 1
        if k == 0 and T != -1:
            f_["first_frame_with_transparent"] += 1
        if k > 0 and prev_valid and T == -1:
            f_["no_transparent_index"] += 1
        if T >= n:
            f_["transparent_ge_ncolors"] += 1
        h, w = src.shape[:2]
        got = of["idx"]
        assert got.shape == (h, w)
        for y in range(h):
            for x in range(w):
                B, G, R, A = (int(v) for v in src[y, x])
                if A in (127, 128):
                    f_[f"alpha{A}_{'transparent' if T != -1 else 'opaque'}"] += 1
                if A < 128 and T != -1:
                    best = T
                    f_["transparent_ge_ncolors_pixel"] += T >= n
                else:
                    c = (R >> 3, G >> 3, B >> 3)
                    owner = c not in memo
                    if owner:
                        lo, hi = [R < 15, G < 15, B < 15], [R > 240, G > 240, B > 240]
                        extreme = all(lo) or all(hi)
                        cmp_ = (R, G, B) if extreme else tuple((v & 0xF8) | 4 for v in (R, G, B))
                        d = _l1(pal, cmp_)
                        if T < n and T >= 0:
                            d[T] = 1 << 30
                        best = int(np.argmin(d))
                        least = int(d[best])
                        memo[c] = (best, (R, G, B), pos)
                        f_["extreme_owner"] += extreme
                        f_["two_channels_extreme"] += sum(lo) == 2 or sum(hi) == 2
                        f_["threshold_owner"] += any(v in (14, 15, 16, 239, 240, 241) for v in (R, G, B))
                        ties = np.flatnonzero(d == least)
                        if len(ties) > 1:
                            dup = any((pal[t] == pal[ties[0]]).all() for t in ties[1:])
                            f_["tie_duplicate_entry" if dup else "tie_equidistant"] += 1
                        if T >= 0 and T < n and _l1(pal[T:T + 1], cmp_)[0] < least:
                            f_["transparent_entry_nearest"] += 1
                        if _straddles((R, G, B)) and extreme:
                            f_["straddle_exact"] += 1
                        if _straddles((R, G, B)) and not extreme:
                            f_["straddle_midpoint"] += 1
                        if _straddles((R, G, B)):
                            other = (R, G, B) if not extreme else tuple((v & 0xF8) | 4 for v in (R, G, B))
                            d2 = _l1(pal, other)
                            if T < n and T >= 0:
                                d2[T] = 1 << 30
                            f_["straddle_choice_differs"] += int(np.argmin(d2)) != best
                        if pos > 0 and y * w + x >= (h * w) // 2:
                            f_["late_bucket_later_frame"] += 1
                    else:
                        best, who, opos = memo[c]
                        least = int(_l1(pal[best:best + 1], (R, G, B))[0])
                        if who != (R, G, B) and opos < pos:
                            f_["bucket_other_colour_earlier_frame"] += 1
                    if prev_valid and T != -1:
                        l_ = prev[y, x]
                        pd = abs(R - int(l_[2])) + abs(G - int(l_[1])) + abs(B - int(l_[0]))
                        f_["prev_equal_least"] += pd == least
                        f_["prev_least_minus_1"] += pd == least - 1
                        if owner:
                            own = int(_l1(pal[best:best + 1], (R, G, B))[0])
                            f_["owner_distances_disagree"] += (pd < least) != (pd < own)
                        if pd < least:
                            best = T
                            f_["prev_substituted"] += 1
                # the LZW encoder keeps the code size's low bits of an index (a transparent index >= 1 << code size)
                best &= (1 << of["min_code"]) - 1
                assert got[y, x] == best, f"frame {k} pixel ({x}, {y}): oracle index {got[y, x]}, model {best}"
        prev[:h, :w] = src
        last = (colors, of["local"])
    return f_


# ---------------------------------------------------------------- the catalogue

@dataclass
class EncCase:
    name: str
    gif: bytes
    frames: list | None = None    # designed BGRA frames; None = the source's composites
    features: set = field(default_factory=set)   # what the case is meant to reach
    palette_model: bool = True    # small enough for map_frames


def pal_of(colors, n=None) -> bytes:
    """RGB entries, padded to a power of two (at least `n`) with a far-off filler."""
    colors = list(colors)
    size = 2
    while size < max(len(colors), n or 0):
        size *= 2
    colors += [(128, 0, 255)] * (size - len(colors))
    return bytes(v for c in colors for v in c)


def _bgra(pal: bytes, idx: np.ndarray, alpha=None) -> np.ndarray:
    p = np.frombuffer(pal, np.uint8).reshape(-1, 3)
    out = np.empty(idx.shape + (4,), np.uint8)
    out[..., :3] = p[idx][..., ::-1]
    out[..., 3] = 255 if alpha is None else alpha
    return out


W, H = 64, 48   # the palette cases' canvas
LOW = [14, 15, 16]
HIGH = [239, 240, 241]
# every combination of threshold values, two-of-three mixes, the straddle buckets' neighbours and their midpoints
THRESH_COLORS = ([(a, b, c) for a in LOW for b in LOW for c in LOW] + [(a, b, c) for a in HIGH for b in HIGH for c in HIGH]
                 + [(14, 14, 200), (14, 200, 14), (200, 14, 14), (241, 241, 100), (100, 241, 241), (241, 60, 241),
                    (14, 14, 15), (241, 241, 240), (15, 240, 14)])
DECOYS = [(12, 12, 12), (11, 11, 11), (244, 244, 244), (246, 246, 246), (10, 12, 9), (20, 20, 20), (236, 236, 236),
          (0, 0, 0), (255, 255, 255), (12, 12, 200), (244, 244, 100)]


def _thresholds_file() -> EncCase:
    """Palette = threshold colours + decoys near the bucket midpoints; frames are those colours in several orders so
    buckets are first consulted by an extreme colour in one frame and a non-extreme one in another run."""
    cols = THRESH_COLORS + DECOYS
    pal = pal_of(cols, 128)
    n = len(cols)
    rng = np.random.default_rng(1)
    frames = []
    for k in range(4):
        order = rng.permutation(n)
        idx = np.resize(order, H * W).reshape(H, W).astype(np.uint8)
        if k == 2:
            idx = idx[::-1, ::-1].copy()
        frames.append(dict(idx=idx))
    return EncCase("thresholds", write_gif(W, H, frames, gct=pal), features={"thresholds"})


def _straddle_file(exact_first: bool) -> EncCase:
    """Buckets 8..15 and 240..247 per channel: the first pixel decides between its exact colour (14 / 241) and the
    midpoint (15 / 240 are not extreme); the palette makes the two choices differ.  The first frame consults each
    bucket at its last pixel, the second at its first: a wrong owner order picks the other side."""
    pairs = [((14, 14, 14), (15, 15, 15)), ((14, 9, 3), (15, 9, 3)), ((2, 14, 14), (2, 15, 14)),
             ((241, 241, 241), (240, 240, 240)), ((241, 250, 249), (240, 250, 249)), ((252, 241, 241), (252, 240, 241))]
    mids = [(11, 11, 11), (11, 12, 4), (4, 11, 11), (245, 245, 245), (245, 251, 251), (253, 245, 245)]
    cols = [c for p in pairs for c in p] + mids + [(90, 90, 90)]
    pal = pal_of(cols)
    first, second = (0, 1) if exact_first else (1, 0)
    filler = len(cols) - 1
    f0 = np.full((H, W), filler, np.uint8)
    f1 = np.full((H, W), filler, np.uint8)
    for i in range(len(pairs)):
        f0.flat[H * W - 1 - i] = 2 * i + first      # consulted last in frame 0
        f1.flat[i] = 2 * i + second                 # and first in frame 1
        f1.flat[H * W - 1 - i] = 2 * i + first
    name = "straddle_exact_first" if exact_first else "straddle_midpoint_first"
    return EncCase(name, write_gif(W, H, [dict(idx=f0), dict(idx=f1), dict(idx=f0[::-1].copy())], gct=pal),
                   features={"straddle"})


def _ties_file() -> EncCase:
    """Duplicate entries (lowest index wins), equidistant entries, the transparent entry the nearest (skipped), and
    a transparent index at or above the colour count."""
    cols = [(100, 100, 100), (50, 50, 50), (50, 50, 50), (60, 52, 52), (52, 60, 52), (52, 52, 60), (200, 10, 10),
            (204, 12, 12), (0, 0, 0), (44, 44, 44), (255, 255, 255), (150, 150, 150)]
    pal = pal_of(cols, 16)
    rng = np.random.default_rng(3)
    frames = []
    for k in range(5):
        idx = rng.integers(0, len(cols), (H, W)).astype(np.uint8)
        idx[rng.random((H, W)) < 0.15] = 7      # (204,12,12): its own entry is the transparent one in frames 1..
        frames.append(dict(idx=idx, gcb=gcb(1, 3, 7 if k in (1, 2) else (200 if k == 3 else None))))
    frames[4]["gcb"] = gcb(1, 3, 2)             # the duplicate's second copy transparent
    return EncCase("ties", write_gif(W, H, frames, gct=pal), features={"ties"})


def _memo_order_file() -> EncCase:
    """A run of 10 frames: frame 0 uses four colours, later frames bring buckets first consulted late in the frame and
    hit buckets with other colours than their owners'."""
    pal = palette(20, 64)
    frames = [dict(idx=np.zeros((H, W), np.uint8) + (np.arange(W) // 16).astype(np.uint8)[None, :])]
    for k in range(1, 10):
        idx = np.zeros((H, W), np.uint8) + (np.arange(W) // 16).astype(np.uint8)[None, :]
        y0 = H - 3 * k
        idx[y0:] = content("noise", H - y0, W, 64, 30 + k)[:, :]
        frames.append(dict(idx=idx))
    return EncCase("memo_late_buckets", write_gif(W, H, frames, gct=pal), features={"memo"})


def _near_palette():
    """64 colours that share crushed buckets pairwise, so a bucket's entry depends on which colour came first."""
    base = palette(21, 32)
    cols = []
    for i in range(32):
        r, g, b = base[3 * i:3 * i + 3]
        cols += [(r, g, b), ((r & 0xF8) | ((r + 5) & 7), g, (b & 0xF8) | ((b + 3) & 7))]
    return pal_of(cols)


def _palette_runs_file() -> EncCase:
    """Palettes that change and change back (the memo is cleared, not restored), a local table byte-equal to the
    global one (the memo carries over), and equal colour bytes with another count."""
    g = _near_palette()
    other = palette(22, 64)
    half = g[:96]                       # the first 32 entries of the global table: equal bytes, another count
    f = lambda s, n: dict(idx=content("noise", H, W, n, s))   # noqa: E731
    frames = [f(40, 64), f(41, 64), dict(f(42, 64), local=other), f(43, 64), dict(f(44, 64), local=g), f(45, 64),
              dict(f(46, 32), local=half), f(47, 64), dict(f(48, 32), local=half), dict(f(49, 32), local=half)]
    return EncCase("palette_runs", write_gif(W, H, frames, gct=g), features={"memo"})


def _prev_file(disposals, seed, name) -> EncCase:
    """Previous-frame substitution: every frame moves a few colours by a small step, so previous distances land on
    `least` and one below; disposals and transparent indices as given (None = no transparent index)."""
    cols = [(v, v, v) for v in range(40, 200, 12)] + [(97, 97, 97), (95, 97, 97), (100, 100, 100), (30, 90, 150),
                                                      (31, 90, 150), (33, 91, 150), (36, 90, 150)]
    pal = pal_of(cols, 32)
    n = len(cols)
    rng = np.random.default_rng(seed)
    base = rng.integers(0, n, (H, W)).astype(np.uint8)
    frames = []
    for k, (disp, t) in enumerate(disposals):
        idx = base.copy()
        m = rng.random((H, W)) < 0.3
        idx[m] = rng.integers(0, n, int(m.sum()))
        frames.append(dict(idx=idx, gcb=gcb(disp, 2, t)))
        base = idx
    return EncCase(name, write_gif(W, H, frames, gct=pal), features={"prev"})


def _owner_file() -> EncCase:
    """An owner pixel whose stored distance (from the bucket midpoint) says keep and whose own distance says take the
    transparent index: (97,97,97) resolves from (100,100,100) at distance 0 while it is 9 from that entry and 2 from
    the previous frame's (95,97,97)."""
    cols = [(97, 97, 97), (95, 97, 97), (100, 100, 100), (20, 200, 20), (60, 60, 60)]
    pal = pal_of(cols, 8)
    f0 = np.full((H, W), 1, np.uint8)
    f0[:, W // 2:] = 4
    f1 = f0.copy()
    f1[H // 2:, :W // 2] = 0
    return EncCase("owner_distances", write_gif(W, H, [dict(idx=f0, gcb=gcb(1, 3, 3)), dict(idx=f1, gcb=gcb(0, 3, 3)),
                                                         dict(idx=f0, gcb=gcb(1, 3, 3))], gct=pal), features={"prev"})


def _alpha_file() -> EncCase:
    """Transparent background (the first frame has a transparent index) with opaque shapes: Fit averages the edges
    to alpha 127 and 128, and colours to bucket edges."""
    cols = [(14, 14, 14), (16, 16, 16), (240, 240, 240), (242, 242, 242), (8, 200, 8), (200, 8, 200), (0, 0, 0),
            (255, 255, 255)]
    pal = pal_of(cols)
    y, x = np.mgrid[0:H, 0:W]
    frames = []
    for k in range(3):
        idx = ((x // 3 + y // 5 + k) % 6).astype(np.uint8)
        idx[(x + 2 * k) % 7 < 3] = 7            # the transparent index: leaves the background (alpha 0)
        frames.append(dict(idx=idx, gcb=gcb(2 if k == 0 else 1, 4, 7)))
    return EncCase("alpha_edges", write_gif(W, H, frames, gct=pal, bg=7), features={"alpha_fit"})


def _long_run_file(nframes, seed) -> EncCase:
    pal = _near_palette()
    frames = [dict(idx=content(("noise", "gradient", "period")[k % 3], H, W, 64, seed + k), gcb=gcb(k % 2, 2, 5 + k % 3))
              for k in range(nframes)]
    return EncCase(f"run_of_{nframes}", write_gif(W, H, frames, gct=pal), features={"memo", "prev"})


def _one_frame_runs_file(nframes, seed) -> EncCase:
    """Every frame its own local table: runs of one frame."""
    frames = [dict(idx=content("noise", H, W, 16, seed + k), local=palette(seed + k, 16), gcb=gcb(1, 2, k % 16))
              for k in range(nframes)]
    return EncCase(f"one_frame_runs_{nframes}", write_gif(W, H, frames, gct=palette(seed, 16)), features={"memo"})


# ---- designed frames: the per-image encoder only

def _designed_colours(seed, n, h, w, alpha=False):
    """Frames drawn from threshold values, bucket edges and palette neighbours."""
    rng = np.random.default_rng(seed)
    vals = np.array(LOW + HIGH + [0, 7, 8, 9, 127, 128, 247, 248, 255], np.uint8)
    out = []
    for _ in range(n):
        f = np.empty((h, w, 4), np.uint8)
        f[..., :3] = rng.choice(vals, (h, w, 3))
        m = rng.random((h, w)) < 0.4
        f[..., :3][m] = rng.integers(0, 256, (int(m.sum()), 3))
        f[..., 3] = rng.choice(np.array([0, 126, 127, 128, 129, 255], np.uint8), (h, w)) if alpha else 255
        f[0, :6, :3] = np.array(LOW + HIGH, np.uint8)[:, None]    # every threshold on all three channels
        out.append(f)
    return out


def _designed_cases():
    out = []
    pal = pal_of(THRESH_COLORS + DECOYS, 128)
    src = write_gif(W, H, [dict(idx=np.zeros((H, W), np.uint8), gcb=gcb(1, 2, 5)) for _ in range(3)], gct=pal)
    out.append(EncCase("designed_thresholds", src, _designed_colours(60, 3, H, W), features={"thresholds"}))
    src = write_gif(W, H, [dict(idx=np.zeros((H, W), np.uint8), gcb=gcb(d, 2, t))
                           for d, t in ((0, 9), (1, 9), (2, None), (3, 9), (1, 9))], gct=pal)
    out.append(EncCase("designed_alpha_transparent", src, _designed_colours(61, 5, H, W, alpha=True),
                       features={"alpha", "prev"}))
    src = write_gif(W, H, [dict(idx=np.zeros((H, W), np.uint8), gcb=gcb(1, 2)) for _ in range(2)], gct=pal)
    out.append(EncCase("designed_alpha_opaque", src, _designed_colours(62, 2, H, W, alpha=True), features={"alpha"}))
    src = write_gif(W, H, [dict(idx=np.zeros((H, W), np.uint8), gcb=gcb(1, 2, 40)) for _ in range(2)],
                    gct=pal_of(DECOYS, 16))
    out.append(EncCase("designed_transparent_ge_ncolors", src, _designed_colours(67, 2, H, W, alpha=True),
                       features={"ties"}))
    # small steps from frame to frame: previous distances equal to `least` and one below
    rng = np.random.default_rng(63)
    base = _designed_colours(64, 1, H, W)[0]
    frames = [base]
    for k in range(5):
        f = frames[-1].copy()
        step = rng.integers(-2, 3, (H, W, 3))
        f[..., :3] = np.clip(f[..., :3].astype(int) + step, 0, 255).astype(np.uint8)
        frames.append(f)
    src = write_gif(W, H, [dict(idx=np.zeros((H, W), np.uint8), gcb=gcb((0, 1, 3, 1, 2, 0)[k], 2, 9))
                           for k in range(6)], gct=pal)
    out.append(EncCase("designed_small_steps", src, frames, features={"prev"}))
    # frames smaller than the canvas (the first frame sets the canvas), interlaced at every height 17..1
    cw, ch = 23, 17
    gp = palette(65, 32)
    src = write_gif(cw, ch, [dict(idx=np.zeros((ch, cw), np.uint8), interlace=True, gcb=gcb(1, 2, 3)) for _ in range(17)],
                    gct=gp)
    frames = [_bgra(gp, content(("noise", "period", "flat")[k % 3], ch - k, cw - (k % 5), 32, 66 + k)) for k in range(17)]
    out.append(EncCase("designed_smaller_interlaced", src, frames, features={"smaller", "interlace"}))
    return out


# ---- LZW: code sizes, table fills, stream lengths, shapes

# widths of one-row noise frames of 256 colours, found by a search over widths with the oracle and frozen: code streams
# of 255 k - 1, 255 k and 255 k + 1 bytes, and one whose last new string is the one that fills the table
SUB_BLOCK_WIDTHS = {-1: 1026, 0: 1027, 1: 1028}
LAST_FILL_WIDTH = 3962


def _lzw_file(name, w, h, ncolors, kind, seed, interlace=False, nframes=2, features=()) -> EncCase:
    pal = palette(seed, ncolors)
    frames = [dict(idx=content(kind, h, w, ncolors, seed + k), interlace=interlace) for k in range(nframes)]
    return EncCase(name, write_gif(w, h, frames, gct=pal), features=set(features), palette_model=w * h <= 4096)


def lzw_cases():
    out = []
    for n in (2, 4, 8, 16, 32, 64, 128, 256):     # code sizes 2 (two- and four-colour tables) .. 8
        side = {2: 480, 4: 320, 8: 260, 16: 200, 32: 180, 64: 160, 128: 140, 256: 130}[n]
        out.append(_lzw_file(f"noise_fill_{n}_colors", side, side * 3 // 4, n, "noise", 100 + n, features={"fill"}))
    for k, width in SUB_BLOCK_WIDTHS.items():
        out.append(_lzw_file(f"length_255k{k:+d}", width, 1, 256, "noise", 200, nframes=1, features={"blocks"}))
    out.append(_lzw_file("last_code_fills", LAST_FILL_WIDTH, 1, 256, "noise", 300, nframes=1, features={"last_fill"}))
    out.append(_lzw_file("flat", 300, 200, 16, "flat", 400, features={"chains"}))
    out.append(_lzw_file("period", 301, 77, 8, "period", 401, features={"period"}))
    out.append(_lzw_file("one_by_one", 1, 1, 4, "noise", 402, features={"1x1"}))
    out.append(_lzw_file("one_row", 777, 1, 32, "gradient", 403, features={"1xN"}))
    out.append(_lzw_file("one_column", 1, 555, 32, "noise", 404, features={"Nx1"}))
    for fh in range(1, 18):
        out.append(_lzw_file(f"interlaced_h{fh}", 13, fh, 16, ("noise", "period", "gradient")[fh % 3], 500 + fh,
                             interlace=True, features={"interlace"}))
    return out


def big_cases():
    """Frames that fill the string table many times over."""
    return [_lzw_file("noise_640x480_256", 640, 480, 256, "noise", 600, nframes=2, features={"fill"}),
            _lzw_file("noise_1024x768_4", 1024, 768, 4, "noise", 601, nframes=2, features={"fill"})]


@functools.lru_cache(maxsize=None)
def palette_cases() -> tuple:
    """The W x H file cases: every palette-mapping corner the source's own frames can reach."""
    out = [_thresholds_file(), _straddle_file(True), _straddle_file(False), _ties_file(), _memo_order_file(),
           _palette_runs_file(), _owner_file(), _alpha_file(),
           _prev_file([(1, 5), (0, 5), (1, 6), (2, 5), (1, 5), (3, 5), (0, 5), (1, None), (0, 4)], 70, "prev_disposals"),
           _prev_file([(0, 3)] * 8, 71, "prev_run_of_8")]
    out += [_long_run_file(8, 80), _long_run_file(12, 90), _one_frame_runs_file(9, 100), _one_frame_runs_file(24, 110)]
    return tuple(out)


@functools.lru_cache(maxsize=None)
def cases() -> tuple:
    return palette_cases() + tuple(lzw_cases()) + tuple(_designed_cases())
