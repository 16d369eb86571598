"""The heterogeneous batch's gate table without a GPU: which (item, rendition) pairs of lp_xbatch_transform_renditions,
lp_xbatch_decode_frames, lp_xbatch_decode_clips and lp_xbatch_encode_frames take the grid, and with which frame, output
size, crop, span, plan, clip and ICC profile, over every source format x sink x option class
(tests/native/xbatch_gates_sim.cu runs xbatch.cu's parse section on the CPU).  Each line must equal the one in
tests/golden/xbatch_gates_golden.npz, as must the number of times each header parser ran in a call; the golden's files
and calls are made by tests/golden/make_golden_xbatch_gates.py."""
import glob
import lzma
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
GOLDEN = os.path.join(ROOT, "tests", "golden", "xbatch_gates_golden.npz")


def build_sim(d):
    """The harness over the library's objects but xbatch.o (which it includes) and the pretend runtime; its path."""
    build = os.path.join(ROOT, "lilliput_b200", "csrc", "build")
    objs = [o for o in sorted(glob.glob(os.path.join(build, "*.o"))) if os.path.basename(o) != "xbatch.o"]
    nvcc = os.path.join(CUDA, "bin", "nvcc")
    if not shutil.which("g++") or not os.path.exists(nvcc) or len(objs) < 10:
        pytest.skip("needs g++, nvcc and the library's objects (run __graft_entry__.build() first)")
    nat = os.path.join(ROOT, "tests", "native")
    inc = ["-I" + os.path.join(ROOT, p) for p in ("include", "lilliput_b200/host", "lilliput_b200/csrc")]

    def run(cmd):
        r = subprocess.run(cmd, cwd=d, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, " ".join(cmd) + "\n" + r.stderr[-3000:]

    run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-Xcompiler", "-fPIC", *inc, "-c",
         os.path.join(nat, "xbatch_gates_sim.cu"), "-o", "xbatch_gates_sim.o"])
    run(["g++", "-O1", "-std=c++17", "-fPIC", "-I" + os.path.join(CUDA, "include"), "-c", os.path.join(nat, "fake_cudart.cpp"),
         "-o", "fake_cudart.o"])
    run(["g++", "-o", "xbatch_gates_sim", "xbatch_gates_sim.o", "fake_cudart.o", *objs, "-lpthread"])
    return os.path.join(d, "xbatch_gates_sim")


def gate_table(sim, d, names, blobs, spec):
    """The harness's lines for `spec` over the files (names[i]: blobs[i]), written into d"""
    for name, b in zip(names, blobs):
        with open(os.path.join(d, name), "wb") as f:
            f.write(b)
    with open(os.path.join(d, "spec.txt"), "w") as f:
        f.write(spec)
    r = subprocess.run([sim, "spec.txt"], cwd=d, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.endswith("calls\n"), r.stderr[-3000:]
    return r.stdout.splitlines()


def unpack(g):
    """(names, file bytes, spec, table lines) of a golden (files, spec and table lzma-compressed)"""
    names = [str(s) for s in g["names"]]
    ends = np.cumsum(g["lengths"])
    data, spec, table = (lzma.decompress(g[k].tobytes()) for k in ("files", "spec", "table"))
    blobs = [data[e - n:e] for e, n in zip(ends, g["lengths"])]
    return names, blobs, spec.decode(), table.decode().splitlines()


def test_gate_table_matches_the_golden(tmp_path):
    sim = build_sim(str(tmp_path))
    names, blobs, spec, want = unpack(np.load(GOLDEN))
    got = gate_table(sim, str(tmp_path), names, blobs, spec)
    call = ""
    diffs = []
    for a, b in zip(got, want):
        if b.startswith("call "):
            call = b
        if a != b:
            diffs.append(f"{call}\n  got  {a}\n  want {b}")
    assert not diffs and len(got) == len(want), f"{len(diffs)} lines differ, {len(got)} vs {len(want)} lines:\n" + \
        "\n".join(diffs[:40])
