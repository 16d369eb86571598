"""Test infrastructure: a multi-scan JPEG writer whose every choice the caller steers -- the scan script (components,
spectral band Ss..Se, successive-approximation bits Ah / Al, in any order), the restart interval, which Huffman tables
each scan names -- and damaged variants of its files, with counts of the decoder corners each file reaches.

The entropy coding is libjpeg-turbo's (jcphuff.c for progressive scans, jchuff.c for sequential ones), including its
EOB runs of up to 32767 blocks and the correction bits of AC refinement scans buffered up to the next symbol.  Every
scan carries its own optimal Huffman tables (a DHT in front of its SOS unless the tables in force are the same,
jchuff.c's jpeg_gen_optimal_table).

The coefficients come from a seeded image (level shift, forward DCT, quantisation in numpy).  `expected()` is what a
decoder holds after every scan: the file's coefficients with the bits below each band's last Al cleared.

`cases()` is the catalogue the CPU check (tests/test_jpeg_scan_streams.py) and the device tests
(tests/test_gpu_batch_progressive.py) share."""
import functools
from dataclasses import dataclass, field

import numpy as np

from tests.jpeg_decode_cases import COLOR_SAMPLINGS, SAMPLINGS

# zigzag position k -> natural index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                   31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63])

# Annex K quantisation tables (luma, chroma), natural order
_QL = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29,
       51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121,
       120, 101, 72, 92, 95, 98, 112, 100, 103, 99]
_QC = [17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99,
       99, 99, 99, 99] + [99] * 32


def qtable(base, quality):
    s = 5000 // quality if quality < 50 else 200 - 2 * quality
    return np.clip((np.array(base) * s + 50) // 100, 1, 255).astype(np.int32)


# ---------------------------------------------------------------- coefficients


@dataclass
class Frame:
    w: int
    h: int
    factors: tuple          # ((h, v) per component)
    coef: list              # per component: (bh, bw, 64) int32, natural order, blocks of the padded MCU grid
    qt: list                # per component: (64,) natural order
    mcus: tuple             # (mcus_x, mcus_y)

    def true_blocks(self, c):
        """(bw, bh) of component c's true block grid (what a non-interleaved scan covers)."""
        mh = max(f[0] for f in self.factors)
        mv = max(f[1] for f in self.factors)
        hc, vc = self.factors[c]
        dw, dh = -(-self.w * hc // mh), -(-self.h * vc // mv)
        return -(-dw // 8), -(-dh // 8)


def _dct_matrix():
    m = np.zeros((8, 8))
    for k in range(8):
        for n in range(8):
            m[k, n] = (np.sqrt(1 / 8) if k == 0 else np.sqrt(2 / 8)) * np.cos(np.pi * (2 * n + 1) * k / 16)
    return m


def frame(sampling: str, w: int, h: int, seed: int, quality: int = 90, content: str = "noise") -> Frame:
    """Quantised coefficients of a seeded image.  Blocks of the padded MCU grid that no non-interleaved scan reaches
    keep their DC only, so sequential and progressive scripts describe the same decoded frame."""
    factors = SAMPLINGS[sampling][1]
    mh = max(f[0] for f in factors)
    mv = max(f[1] for f in factors)
    mx, my = -(-w // (8 * mh)), -(-h // (8 * mv))
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:my * 8 * mv, 0:mx * 8 * mh]
    D = _dct_matrix()
    coef, qts = [], []
    for c, (hc, vc) in enumerate(factors):
        bw, bh = mx * hc, my * vc
        if content == "flat":
            img = np.full((bh * 8, bw * 8), 128.0)
        else:
            sy, sx = mv // vc, mh // hc
            base = 128 + 60 * np.sin(xx[::sy, ::sx] / (7.0 + 3 * c)) * np.cos(yy[::sy, ::sx] / 11.0)
            img = base[:bh * 8, :bw * 8] + rng.normal(0, 25 if content == "noise" else 4, (bh * 8, bw * 8))
        blocks = (np.clip(img, 0, 255) - 128).reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3)
        dct = np.einsum("ij,abjk,lk->abil", D, blocks, D).reshape(bh, bw, 64)
        q = qtable(_QL if c == 0 else _QC, quality)
        cq = np.round(dct / q).astype(np.int32)
        tw, th = Frame(w, h, factors, [], [], (mx, my)).true_blocks(c)
        cq[th:, :, 1:] = 0
        cq[:, tw:, 1:] = 0
        coef.append(cq)
        qts.append(q)
    return Frame(w, h, factors, coef, qts, (mx, my))


# ---------------------------------------------------------------- scripts


@dataclass(frozen=True)
class Scan:
    comps: tuple        # frame component indices
    Ss: int = 0
    Se: int = 63
    Ah: int = 0
    Al: int = 0


def simple_progression(nc=3):
    """libjpeg-turbo's jpeg_simple_progression for three components."""
    return [Scan((0, 1, 2), 0, 0, 0, 1), Scan((0,), 1, 5, 0, 2), Scan((2,), 1, 63, 0, 1), Scan((1,), 1, 63, 0, 1),
            Scan((0,), 6, 63, 0, 2), Scan((0,), 1, 63, 2, 1), Scan((0, 1, 2), 0, 0, 1, 0), Scan((2,), 1, 63, 1, 0),
            Scan((1,), 1, 63, 1, 0), Scan((0,), 1, 63, 1, 0)]


def sequential_per_component():
    return [Scan((0,), 0, 63), Scan((1,), 0, 63), Scan((2,), 0, 63)]


# ---------------------------------------------------------------- bits and tables


class Bits:
    def __init__(self):
        self.parts = []

    def put(self, v, n):
        if n:
            self.parts.append(format(v & ((1 << n) - 1), "0%db" % n))

    def flush(self) -> bytes:
        s = "".join(self.parts)
        self.parts = []
        s += "1" * (-len(s) % 8)
        raw = int(s, 2).to_bytes(len(s) // 8, "big") if s else b""
        return raw.replace(b"\xff", b"\xff\x00")


def optimal_table(freq):
    """jchuff.c jpeg_gen_optimal_table: (bits[1..16], values)."""
    freq = list(freq) + [1]  # the reserved all-ones code point
    n = len(freq)
    codesize = [0] * n
    others = [-1] * n
    while True:
        c1 = c2 = -1
        v1 = v2 = None
        for i in range(n):
            if freq[i] and (v1 is None or freq[i] <= v1):
                v1, c1 = freq[i], i
        for i in range(n):
            if freq[i] and i != c1 and (v2 is None or freq[i] <= v2):
                v2, c2 = freq[i], i
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = [0] * 33
    for i in range(n):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    vals = [s for length in range(1, 33) for s in range(n - 1) if codesize[s] == length]
    return bits[1:17], vals


def codes_of(bits, vals):
    code, k, out = 0, 0, {}
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return out


def _nbits(v):
    return int(abs(int(v))).bit_length()


# ---------------------------------------------------------------- scan coding (two passes: symbols, then bits)


class _Coder:
    """Codes one scan; `emit(table, symbol)` and `bits(v, n)` are the two passes' sinks."""

    def __init__(self, fr: Frame, sc: Scan, progressive: bool, restart: int):
        self.fr, self.sc, self.prog, self.restart = fr, sc, progressive, restart

    def units(self):
        """(component slot i, block array view, by, bx) in scan order, with restart points as None."""
        fr, sc = self.fr, self.sc
        if len(sc.comps) == 1:
            c = sc.comps[0]
            tw, th = fr.true_blocks(c)
            mcus = [[(0, c, by, bx)] for by in range(th) for bx in range(tw)]
        else:
            mcus = []
            for my in range(fr.mcus[1]):
                for mx in range(fr.mcus[0]):
                    mcu = []
                    for i, c in enumerate(sc.comps):
                        hc, vc = fr.factors[c]
                        mcu += [(i, c, my * vc + y, mx * hc + x) for y in range(vc) for x in range(hc)]
                    mcus.append(mcu)
        return mcus

    def run(self, emit, bits, restart_cb):
        sc = self.sc
        self.eobrun, self.be = 0, []
        pred = [0, 0, 0]
        zz = ZIGZAG
        if self.prog and sc.Ss > 0 and sc.Ah == 0 and not self.restart:
            # AC first without restarts: an empty band only lengthens the EOB run, so walk the nonempty blocks
            c = sc.comps[0]
            tw, th = self.fr.true_blocks(c)
            band = self.fr.coef[c][:th, :tw][:, :, zz[sc.Ss:sc.Se + 1]]
            full = np.flatnonzero((np.abs(band) >> sc.Al).max(axis=2).reshape(-1))
            last = -1
            for b in full.tolist() + [th * tw]:
                gap = b - last - 1
                while gap:
                    take = min(gap, 0x7FFF - self.eobrun)
                    self.eobrun += take
                    gap -= take
                    if self.eobrun == 0x7FFF:
                        self.emit_eobrun(emit, bits)
                if b < th * tw:
                    self.ac_first(self.fr.coef[c][b // tw, b % tw][zz], 0, emit, bits)
                last = b
            self.emit_eobrun(emit, bits)
            return
        for m, mcu in enumerate(self.units()):
            if self.restart and m and m % self.restart == 0:
                self.emit_eobrun(emit, bits)
                restart_cb((m // self.restart - 1) & 7)
                pred = [0, 0, 0]
            for i, c, by, bx in mcu:
                blk = self.fr.coef[c][by, bx]
                if not self.prog:
                    self.seq_block(blk, i, pred, emit, bits)
                elif sc.Ss == 0 and sc.Ah == 0:
                    t = int(blk[0]) >> sc.Al
                    d = t - pred[i]
                    pred[i] = t
                    n = _nbits(d)
                    emit(0, i, n)
                    bits(d if d >= 0 else d - 1, n)
                elif sc.Ss == 0:
                    bits((int(blk[0]) >> sc.Al) & 1, 1)
                elif sc.Ah == 0:
                    self.ac_first(blk[zz], i, emit, bits)
                else:
                    self.ac_refine(blk[zz], i, emit, bits)
        self.emit_eobrun(emit, bits)

    def seq_block(self, blk, i, pred, emit, bits):
        d = int(blk[0]) - pred[i]
        pred[i] = int(blk[0])
        n = _nbits(d)
        emit(0, i, n)
        bits(d if d >= 0 else d - 1, n)
        z = blk[ZIGZAG]
        r = 0
        for k in range(1, 64):
            v = int(z[k])
            if v == 0:
                r += 1
                continue
            while r > 15:
                emit(1, i, 0xF0)
                r -= 16
            n = _nbits(v)
            emit(1, i, (r << 4) | n)
            bits(v if v >= 0 else v - 1, n)
            r = 0
        if r:
            emit(1, i, 0)

    def emit_eobrun(self, emit, bits):
        if self.eobrun:
            n = self.eobrun.bit_length() - 1
            emit(1, 0, n << 4)
            bits(self.eobrun, n)
            self.eobrun = 0
            for b in self.be:
                bits(b, 1)
            self.be = []

    def ac_first(self, z, i, emit, bits):
        sc = self.sc
        r = 0
        for k in range(sc.Ss, sc.Se + 1):
            v = int(z[k])
            t = abs(v) >> sc.Al
            if t == 0:
                r += 1
                continue
            self.emit_eobrun(emit, bits)
            while r > 15:
                emit(1, i, 0xF0)
                r -= 16
            n = t.bit_length()
            emit(1, i, (r << 4) | n)
            bits(t if v >= 0 else ~t, n)
            r = 0
        if r:
            self.eobrun += 1
            if self.eobrun == 0x7FFF:
                self.emit_eobrun(emit, bits)

    def ac_refine(self, z, i, emit, bits):
        sc = self.sc
        absv = [abs(int(z[k])) >> sc.Al for k in range(64)]
        eob = max([k for k in range(sc.Ss, sc.Se + 1) if absv[k] == 1], default=0)
        r, br = 0, []
        for k in range(sc.Ss, sc.Se + 1):
            t = absv[k]
            if t == 0:
                r += 1
                continue
            while r > 15 and k <= eob:
                self.emit_eobrun(emit, bits)
                emit(1, i, 0xF0)
                r -= 16
                for b in br:
                    bits(b, 1)
                br = []
            if t > 1:
                br.append(t & 1)
                continue
            self.emit_eobrun(emit, bits)
            emit(1, i, (r << 4) | 1)
            bits(0 if z[k] < 0 else 1, 1)
            for b in br:
                bits(b, 1)
            br = []
            r = 0
        if r or br:
            self.eobrun += 1
            self.be += br
            if self.eobrun == 0x7FFF or len(self.be) > 1000 - 63:
                self.emit_eobrun(emit, bits)


# ---------------------------------------------------------------- files


def _seg(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


@dataclass
class Stream:
    name: str
    data: bytes
    features: set = field(default_factory=set)
    fr: Frame = None
    script: list = None
    damaged: bool = False


def write(fr: Frame, script, progressive=True, restart=0, drop_code=None, bad_table_scan=None, truncate=None):
    """The file of `fr` coded by `script`.  Damage: drop_code = scan index whose DHT loses its longest AC code;
    bad_table_scan = scan index whose SOS names table 3 (never defined); truncate = (scan index, fraction of its
    entropy-coded bytes kept), after which the file ends."""
    out = bytearray(b"\xff\xd8")
    nc = len(fr.factors)
    out += _seg(0xDB, b"".join(bytes([c]) + bytes(fr.qt[c][ZIGZAG].astype(np.uint8)) for c in range(min(nc, 2))))
    sof = bytes([8]) + fr.h.to_bytes(2, "big") + fr.w.to_bytes(2, "big") + bytes([nc])
    for c, (hc, vc) in enumerate(fr.factors):
        sof += bytes([c + 1, (hc << 4) | vc, min(c, 1)])
    out += _seg(0xC2 if progressive else 0xC1, sof)
    if restart:
        out += _seg(0xDD, restart.to_bytes(2, "big"))
    last_dht = None
    for s, sc in enumerate(script):
        coder = _Coder(fr, sc, progressive, restart)
        freq = [[[0] * 256 for _ in range(3)] for _ in range(2)]  # [dc/ac][slot][symbol]
        coder.run(lambda t, i, sym: freq[t][i].__setitem__(sym, freq[t][i][sym] + 1), lambda v, n: None, lambda k: None)
        # one table per component slot and class, ids 0..2
        dht = b""
        tables = {}
        for t in range(2):
            for i in range(len(sc.comps)):
                if sum(freq[t][i]) == 0:
                    continue
                bits, vals = optimal_table(freq[t][i])
                tables[(t, i)] = codes_of(bits, vals)
                if drop_code == s and t == 1 and i == 0:
                    L = max(l for l in range(16) if bits[l])
                    bits = list(bits)
                    bits[L] -= 1
                    gone = vals[sum(bits[:L + 1])]
                    vals = [v for v in vals if v != gone]
                dht += bytes([(t << 4) | i]) + bytes(bits) + bytes(vals)
        if dht and dht != last_dht:  # (tables already in force need no second DHT)
            out += _seg(0xC4, dht)
            last_dht = dht
        sos = bytes([len(sc.comps)])
        for i, c in enumerate(sc.comps):
            t = 3 if bad_table_scan == s else i
            sos += bytes([c + 1, (t << 4) | t])
        sos += bytes([sc.Ss, sc.Se, (sc.Ah << 4) | sc.Al]) if progressive else bytes([0, 63, 0])
        out += _seg(0xDA, sos)
        data = bytearray()
        bw = Bits()

        def emit(t, i, sym):
            code, n = tables[(t, i)][sym]
            bw.put(code, n)

        def rst(k):
            data.extend(bw.flush())
            data.extend(bytes([0xFF, 0xD0 + k]))

        coder.run(emit, bw.put, rst)
        data += bw.flush()
        if truncate and truncate[0] == s:
            out += data[:int(len(data) * truncate[1])]
            return bytes(out)
        out += data
    return bytes(out + b"\xff\xd9")


def expected(fr: Frame, script, progressive=True):
    """Per component (bh, bw, 64) natural order: what a decoder holds after the script."""
    out = [np.zeros_like(c) for c in fr.coef]
    for sc in script:
        for c in sc.comps:
            src, dst = fr.coef[c], out[c]
            if len(sc.comps) == 1:
                tw, th = fr.true_blocks(c)
            else:
                th, tw = src.shape[0], src.shape[1]
            if not progressive:
                dst[:th, :tw] = src[:th, :tw]
                continue
            nat = ZIGZAG[sc.Ss:sc.Se + 1]
            v = src[:th, :tw][:, :, nat]
            if sc.Ss == 0:
                dst[:th, :tw, 0] = (v[:, :, 0] >> sc.Al) << sc.Al
            else:
                dst[:th, :tw][:, :, nat] = np.sign(v) * ((np.abs(v) >> sc.Al) << sc.Al)
    return out


# ---------------------------------------------------------------- catalogue


def _features(fr, script, progressive, restart):
    f = set()
    for sc in script:
        if not progressive:
            f.add("sequential_per_component")
            continue
        if sc.Ss == 0:
            f.add("dc_first_al%d" % sc.Al if sc.Ah == 0 else "dc_refine")
            f.add("dc_interleaved" if len(sc.comps) > 1 else "dc_per_component")
        elif sc.Ah == 0:
            f.add("ac_first")
            if (sc.Ss, sc.Se) not in ((1, 63), (1, 5), (6, 63)):
                f.add("ac_split_band")
        else:
            f.add("ac_refine")
            if sc.Al == 0:
                f.add("ac_chain_to_0")
    if restart:
        f.add("restart")
    # longest EOB run: blocks of a component whose band is empty in a row
    return f


def _eob_classes(fr, script):
    """Length classes (bit lengths) of the EOB runs the AC first scans code, and whether a run crosses a block row."""
    classes, crosses = set(), False
    for sc in script:
        if sc.Ss == 0 or sc.Ah != 0 or len(sc.comps) != 1:
            continue
        c = sc.comps[0]
        tw, th = fr.true_blocks(c)
        z = np.abs(fr.coef[c][:th, :tw][:, :, ZIGZAG[sc.Ss:sc.Se + 1]]) >> sc.Al
        empty = (z.max(axis=2) == 0).reshape(-1)
        run = 0
        for k, e in enumerate(empty.tolist() + [False]):
            if e:
                run += 1
                continue
            while run:
                take = min(run, 0x7FFF)
                classes.add(take.bit_length() - 1)
                if take > tw:
                    crosses = True
                run -= take
    return classes, crosses


SPLIT = [Scan((0, 1, 2), 0, 0, 0, 3), Scan((0, 1, 2), 0, 0, 3, 2), Scan((0, 1, 2), 0, 0, 2, 1),
         Scan((0, 1, 2), 0, 0, 1, 0), Scan((0,), 1, 2, 0, 3), Scan((0,), 3, 17, 0, 2), Scan((0,), 18, 63, 0, 1),
         Scan((1,), 1, 63, 0, 0), Scan((2,), 1, 9, 0, 1), Scan((2,), 10, 63, 0, 0), Scan((0,), 1, 2, 3, 2),
         Scan((0,), 1, 2, 2, 1), Scan((0,), 1, 2, 1, 0), Scan((0,), 3, 17, 2, 1), Scan((0,), 3, 17, 1, 0),
         Scan((0,), 18, 63, 1, 0), Scan((2,), 1, 9, 1, 0)]

PER_COMPONENT_DC = [Scan((0,), 0, 0, 0, 0), Scan((1,), 0, 0, 0, 2), Scan((2,), 0, 0, 0, 1), Scan((2,), 0, 0, 1, 0),
                    Scan((1,), 0, 0, 2, 1), Scan((1,), 0, 0, 1, 0), Scan((0,), 1, 63, 0, 1), Scan((1,), 1, 63, 0, 0),
                    Scan((2,), 1, 63, 0, 0), Scan((0,), 1, 63, 1, 0)]


@functools.lru_cache(maxsize=None)
def cases():
    out = []
    k = 0
    for s, sampling in enumerate(COLOR_SAMPLINGS):
        for w, h in ((203, 131), (77, 40), (16, 9)):
            k += 1
            fr = frame(sampling, w, h, seed=k)
            for name, script, prog, rst in (("simple", simple_progression(), True, 0),
                                            ("split", SPLIT, True, 0),
                                            ("dcpercomp", PER_COMPONENT_DC, True, 0),
                                            ("restart", simple_progression(), True, 3 + s),
                                            ("sequential", sequential_per_component(), False, 0),
                                            ("sequential_rst", sequential_per_component(), False, 2)):
                data = write(fr, script, prog, rst)
                f = _features(fr, script, prog, rst) | {"sampling_" + sampling}
                if w % (8 * max(a for a, _ in fr.factors)):
                    f.add("width_off_grid")
                cls, crosses = _eob_classes(fr, script)
                f |= {"eob_class_%d" % c for c in cls}
                if crosses:
                    f.add("eob_run_crosses_row")
                out.append(Stream("%s_%s_%dx%d" % (sampling, name, w, h), data, f, fr, script))
    # long EOB runs: a flat frame whose bands are empty over up to 35000 blocks (runs stop at the 32767 cap); in the
    # first luma band, nonzero blocks 2^c + 1 apart give a run of every length class
    fr = frame("444", 1600, 1400, seed=99, quality=50, content="flat")
    pos = 0
    for c in range(15):
        pos += (1 << c) + 1
        fr.coef[0][pos // 200, pos % 200, 1] = 40
    data = write(fr, simple_progression(), True, 0)
    cls, crosses = _eob_classes(fr, simple_progression())
    f = {"eob_class_%d" % c for c in cls} | ({"eob_run_crosses_row"} if crosses else set())
    out.append(Stream("444_long_eob_1600x1400", data, f | ({"eob_max_run"} if 14 in cls else set()), fr,
                      simple_progression()))
    return out


def damaged():
    """(name, file): truncation inside each scan, a code missing from a table, a scan naming an undefined table."""
    fr = frame("420", 203, 131, seed=5)
    script = simple_progression()
    out = []
    for s in range(len(script)):
        out.append(("truncated_scan%d" % s, write(fr, script, truncate=(s, 0.5))))
    out.append(("missing_code", write(fr, script, drop_code=1)))
    out.append(("undefined_table", write(fr, script, bad_table_scan=4)))
    out.append(("missing_code_sequential", write(fr, sequential_per_component(), False, drop_code=0)))
    return out


def over_budget():
    """A 4096 x 4096 4:4:4 file with 256 scans, all but the first empty AC bands: 2^26 + 2^19 block visits, a few
    hundred KB."""
    fr = frame("444", 4096, 4096, seed=3, content="flat")
    script = [Scan((0, 1, 2), 0, 0, 0, 0)] + [Scan((c % 3,), 1 + c // 3 % 63, 1 + c // 3 % 63, 0, 0) for c in range(255)]
    return write(fr, script)


FEATURES = ({"dc_first_al%d" % a for a in range(4)} | {"dc_refine", "dc_interleaved", "dc_per_component", "ac_first",
            "ac_split_band", "ac_refine", "ac_chain_to_0", "restart", "sequential_per_component", "width_off_grid",
            "eob_run_crosses_row", "eob_max_run"} | {"eob_class_%d" % c for c in range(15)} |
            {"sampling_" + s for s in COLOR_SAMPLINGS})


def check_coverage(streams):
    seen = set().union(*(s.features for s in streams))
    missing = FEATURES - seen
    assert not missing, sorted(missing)
