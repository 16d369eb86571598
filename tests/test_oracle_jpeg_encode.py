"""CPU: the baseline JPEG encoder's contract, held live against libjpeg-turbo through the cv2 here.

- oracle.jpeg_encode (oracle/oracle_jpeg_enc.c, the C restatement the batch tests take their expected bytes from)
  writes cv2's bytes over the whole case matrix of tests/jpeg_encode_cases.py;
- cv2 still writes the reference's golden files (tests/golden), so a cv2 that changed its output fails here instead
  of silently moving the bar;
- the matrix reaches what it is meant to: every cv2 file's scan is decoded with the Annex K tables and tokenised as
  jchuff.c codes it, and every DC category, AC size, ZRL run, EOB-less block, dummy-block kind, padding length and the
  stuffed padded byte is found somewhere in it.  The device encoder is held to the same files in
  tests/test_gpu_jpeg_encode.py."""
import pytest

from tests import jpeg_encode_cases as jc
from tests.cases import JPEG_CASES
from tests.jpeg_baseline_streams import ANNEX_K, EOB, ZRL, ac_tokens
from lilliput_b200.synth import synth_image

cv2 = pytest.importorskip("cv2")


def _first_diff(a, b):
    return next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))


# ---------------------------------------------------------------- scan reader


def _code_map(table):
    bits, vals = table
    out, code, k = {}, 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            out[format(code, f"0{n}b")] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return out


CODES = {k: _code_map(v) for k, v in ANNEX_K.items()}


def _sos_end(data: bytes) -> int:
    pos = 2
    while True:
        assert data[pos] == 0xFF
        m, seg = data[pos + 1], int.from_bytes(data[pos + 2:pos + 4], "big")
        pos += 2 + seg
        if m == 0xDA:
            return pos


class ScanFacts:
    """What one baseline file's scan holds, read with the Annex K tables (table index 0 luma, 1 chroma)."""

    def __init__(self, data: bytes, w: int, h: int, gray: bool):
        assert data[-2:] == b"\xff\xd9"
        stuffed = data[_sos_end(data):-2]
        raw = stuffed.replace(b"\xff\x00", b"\xff")
        assert stuffed.count(b"\xff") == stuffed.count(b"\xff\x00")  # every 0xFF stuffed, no markers
        s = "".join(format(b, "08b") for b in raw)
        self.dc = [set(), set()]
        self.ac = [set(), set()]
        self.max_zrl_run = 0
        self.ends_at_63 = False
        self.dummy = {}            # kind -> nonzero DC seen
        pos = 0

        def sym(codes):
            nonlocal pos
            for n in range(1, 17):
                v = codes.get(s[pos:pos + n])
                if v is not None:
                    pos += n
                    return v
            raise AssertionError(f"no Huffman code at bit {pos}")

        def extend(n):
            nonlocal pos
            if not n:
                return 0
            v = int(s[pos:pos + n], 2)
            pos += n
            return v if v >= 1 << (n - 1) else v - (1 << n) + 1

        hs = 1 if gray else 2
        mx_n, my_n = -(-w // (8 * hs)), -(-h // (8 * hs))
        ybw, ybh = -(-w // 8), -(-h // 8)
        pred = [0, 0, 0]
        for my in range(my_n):
            for mx in range(mx_n):
                blocks = [(0, k) for k in range(hs * hs)] + ([] if gray else [(1, 4), (2, 5)])
                dcs = []
                for comp, k in blocks:
                    t = 0 if comp == 0 else 1
                    cat = sym(CODES["dc_luma" if t == 0 else "dc_chroma"])
                    self.dc[t].add(cat)
                    pred[comp] += extend(cat)
                    z = [pred[comp]] + [0] * 63
                    i, zrl_run, toks = 1, 0, []
                    while i < 64:
                        rs = sym(CODES["ac_luma" if t == 0 else "ac_chroma"])
                        r, size = rs >> 4, rs & 15
                        if rs == 0:
                            toks.append(EOB)
                            break
                        if rs == 0xF0:
                            toks.append(ZRL)
                            zrl_run += 1
                            self.max_zrl_run = max(self.max_zrl_run, zrl_run)
                            i += 16
                            continue
                        zrl_run = 0
                        i += r
                        z[i] = extend(size)
                        toks.append((r, size, z[i]))
                        self.ac[t].add(size)
                        i += 1
                    assert i <= 64
                    self.ends_at_63 |= z[63] != 0
                    # the symbols read are the ones jchuff.c's encode_one_block makes of the block
                    assert toks == ac_tokens(z), (mx, my, k)
                    dcs.append(z[0])
                    if comp == 0 and not gray:
                        X, Y = 2 * mx + (k & 1), 2 * my + (k >> 1)
                        kind = ("corner" if X >= ybw and Y >= ybh else "right" if X >= ybw
                                else "bottom" if Y >= ybh else None)
                        if kind:
                            # jccoefct.c: a dummy block is all zero but for the DC of the block before it in the MCU
                            assert any(z[1:]) is False and z[0] == dcs[k - 1], (mx, my, k)
                            self.dummy[kind] = self.dummy.get(kind, False) or z[0] != 0
        self.pad_bits = len(s) - pos
        assert 0 <= self.pad_bits < 8 and s[pos:] == "1" * self.pad_bits  # 1-padding of the last byte only
        self.stuffed_pad = self.pad_bits > 0 and raw[-1] == 0xFF


# ---------------------------------------------------------------- tests


def test_reference_options_behave_as_documented():
    """The quality option as cv2 takes it: clamped to 0..100, 0 codes as 1, no option is 95."""
    img = jc.image("photo", 45, 37, 3, 1)
    ref = jc.reference
    assert ref(img, -5) == ref(img, 0) == ref(img, 1)
    assert ref(img, 101) == ref(img, 100)
    assert ref(img, None) == ref(img, 95)
    assert len({ref(img, q) for q in (1, 2, 50, 95, 100)}) == 5


@pytest.mark.parametrize("case", JPEG_CASES, ids=lambda c: f"seed{c[0]}")
def test_cv2_writes_the_golden_files(golden, case):
    seed, w, h, ch, q = case
    img = synth_image(seed, w, h, ch, noise=8.0)  # as tests/golden/make_golden.py made them
    assert jc.reference(img, q) == golden[f"jpeg_{seed}"].tobytes()


@pytest.mark.parametrize("group", ["edge", "quality", "launch"])
def test_oracle_matches_libjpeg_turbo(oracle, group):
    cases = {"edge": jc.edge_matrix, "quality": jc.quality_sweep, "launch": jc.launch_shapes}[group]()
    for case in cases:
        img = jc.case_image(case)
        q = case[4]
        got, want = oracle.jpeg_encode(img, 95 if q is None else q), jc.reference(img, q)
        assert got == want, (case, len(got), len(want), _first_diff(got, want))


def test_recorded_seeds_have_their_padding():
    """PAD_FF_SEED's scan ends in a 1-padded byte equal to 0xFF (stuffed); NO_PAD_SEED's bits fill its last byte."""
    for seed, want_pad in ((jc.PAD_FF_SEED, True), (jc.NO_PAD_SEED, False)):
        img = jc.image("noise", 40, 24, 3, seed)
        f = ScanFacts(jc.reference(img, 75), 40, 24, False)
        assert (f.stuffed_pad, f.pad_bits > 0) == (want_pad, want_pad), (seed, f.pad_bits)


def test_matrix_reaches_every_symbol_and_edge_class():
    """Decoded from cv2's files, not from the oracle's: what the matrix exercises does not depend on the code under
    test.  The launch shapes are left out (the 1080p frame alone is 4.7 MB); the two padding seeds are read."""
    dc, ac = [set(), set()], [set(), set()]
    zrl, at63, pads, stuffed_pad, dummy = 0, False, set(), False, {}
    small = [c for c in jc.launch_shapes() if c[1] * c[2] <= 40 * 24]
    for case in jc.edge_matrix() + jc.quality_sweep() + small:
        _, w, h, ch, q, _ = case
        f = ScanFacts(jc.reference(jc.case_image(case), q), w, h, ch == 1)
        for t in (0, 1):
            dc[t] |= f.dc[t]
            ac[t] |= f.ac[t]
        zrl = max(zrl, f.max_zrl_run)
        at63 |= f.ends_at_63
        pads.add(f.pad_bits)
        stuffed_pad |= f.stuffed_pad
        for k, v in f.dummy.items():
            dummy[k] = dummy.get(k, False) or v
    reached = {
        "luma DC categories 0-11": dc[0] >= set(range(12)),
        "chroma DC categories 0-11": dc[1] >= set(range(12)),
        "luma AC sizes 1-10": ac[0] >= set(range(1, 11)),
        "chroma AC sizes 1-10": ac[1] >= set(range(1, 11)),
        "two or more ZRLs in a row": zrl >= 2,
        "a block ending at coefficient 63": at63,
        "right dummy blocks with nonzero DC": dummy.get("right", False),
        "bottom dummy blocks with nonzero DC": dummy.get("bottom", False),
        "corner dummy blocks with nonzero DC": dummy.get("corner", False),
        "0-7 pad bits": pads == set(range(8)),
        "a stuffed padded byte": stuffed_pad,
    }
    print("\n".join(f"{'reached' if v else 'MISSING'}: {k}" for k, v in reached.items()))
    assert all(reached.values()), ({k for k, v in reached.items() if not v}, sorted(dc[0]), sorted(dc[1]),
                                   sorted(ac[0]), sorted(ac[1]), zrl, sorted(pads))
