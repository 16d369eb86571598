"""CPU: the checksum arithmetic of the PNG encoder (lilliput_b200/csrc/crc32_core.h), compiled for the host by
tests/native/crc32_sim.cpp.

The encoder never walks a file front to back: every warp checksums the piece it wrote and the pieces are joined --
CRC-32 by crc(A || B) = crc(A) * x^(8 |B|) xor crc(B) modulo the CRC polynomial, Adler-32 from per-piece partial sums.
Here those rules are checked against zlib.crc32 / zlib.adler32 over random buffers cut at random places."""
import ctypes as C
import os
import subprocess
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("crc32") / "libcrc32sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so,
                           os.path.join(ROOT, "tests", "native", "crc32_sim.cpp")])
    l = C.CDLL(so)
    l.crc32sim_update.restype = C.c_uint32
    l.crc32sim_update.argtypes = [C.c_uint32, C.c_char_p, C.c_long]
    l.crc32sim_combine.restype = C.c_uint32
    l.crc32sim_combine.argtypes = [C.c_uint32, C.c_uint32, C.c_ulonglong]
    for f in (l.crc32sim_chain, l.crc32sim_fold, l.crc32sim_adler):
        f.restype = C.c_uint32
        f.argtypes = [C.c_char_p, C.POINTER(C.c_long), C.c_int]
    return l


def _cuts(rng, n, npieces):
    inner = sorted(int(v) for v in rng.integers(0, n + 1, npieces - 1))
    return [0] + inner + [n]


def test_update_is_zlib_crc32(sim):
    rng = np.random.default_rng(1)
    assert sim.crc32sim_update(0, b"", 0) == 0
    assert sim.crc32sim_update(0, b"123456789", 9) == 0xCBF43926
    for n in (1, 2, 7, 255, 4096, 70001):
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert sim.crc32sim_update(0, d, n) == zlib.crc32(d)
        k = n // 3
        assert sim.crc32sim_update(zlib.crc32(d[:k]), d[k:], n - k) == zlib.crc32(d)


def test_combine_over_random_splits(sim):
    rng = np.random.default_rng(2)
    for t in range(200):
        n = int(rng.integers(0, 5000)) if t % 4 else int(rng.integers(0, 300000))
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        k = int(rng.integers(0, n + 1))
        got = sim.crc32sim_combine(zlib.crc32(d[:k]), zlib.crc32(d[k:]), n - k)
        assert got == zlib.crc32(d), (n, k)


def test_combine_lengths_past_32_bits(sim):
    """x^(8 n) by squaring, for lengths too long to materialise: crc(A || B || C) grouped as (A || B) || C and as
    A || (B || C) must agree, and a long length must equal the same length reached in two steps."""
    rng = np.random.default_rng(3)
    for _ in range(50):
        a, b, c = (int(v) for v in rng.integers(0, 1 << 32, 3))
        lb, lc = int(rng.integers(1, 1 << 40)), int(rng.integers(1, 1 << 40))
        left = sim.crc32sim_combine(sim.crc32sim_combine(a, b, lb), c, lc)
        right = sim.crc32sim_combine(a, sim.crc32sim_combine(b, c, lc), lb + lc)
        assert left == right
        # appending lb + lc bytes whose own CRC contribution is nil = appending lb of them, then lc
        assert sim.crc32sim_combine(a, 0, lb + lc) == sim.crc32sim_combine(sim.crc32sim_combine(a, 0, lb), 0, lc)
    run = bytes(1 << 20)
    assert sim.crc32sim_combine(zlib.crc32(b"lilliput"), zlib.crc32(run), len(run)) == zlib.crc32(b"lilliput" + run)


@pytest.mark.parametrize("npieces", [1, 2, 3, 32, 33, 257])
def test_pieces_chain_and_fold(sim, npieces):
    """The pairwise rule applied left to right, and the per-piece form (every piece weighted by the bytes behind it,
    xor-ed in any order) the pack kernel uses, on buffers cut into `npieces` pieces, empty ones included."""
    rng = np.random.default_rng(100 + npieces)
    for n in (0, 1, 31, 32, 33, 1000, 32767, 32768, 32769, 200000):
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        cuts = _cuts(rng, n, npieces)
        arr = (C.c_long * len(cuts))(*cuts)
        assert sim.crc32sim_chain(d, arr, npieces) == zlib.crc32(d), (n, cuts[:8])
        assert sim.crc32sim_fold(d, arr, npieces) == zlib.crc32(d), (n, cuts[:8])
        assert sim.crc32sim_adler(d, arr, npieces) == zlib.adler32(d), (n, cuts[:8])


def test_adler_of_saturated_bytes(sim):
    """0xFF everywhere: the partial sums are as large as they get for their length."""
    for n in (5552, 5553, 32768, 3 * 32768 + 17):
        d = b"\xff" * n
        cuts = list(range(0, n, 32768)) + [n]
        arr = (C.c_long * len(cuts))(*cuts)
        assert sim.crc32sim_adler(d, arr, len(cuts) - 1) == zlib.adler32(d), n
