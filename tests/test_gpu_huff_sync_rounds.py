"""GPU: the synchronisation rounds of the parallel JPEG entropy decoder under stress.

LP_HUFF_SPT=8 cuts every scan into subsequences of the minimum 1024 bits, so images need many synchronisation rounds
and a subsequence is often re-decoded from a neighbour's exit state that changed in the same round.  The launcher
reads the variable once per process, so each setting runs in a child process (this module run as a script).  Every
file -- the baseline stream catalogue (including the layouts whose components do not share the usual two table
pairs), 1080p files with the default and with optimised tables, gray, 4:4:4 and 4:2:2 -- goes through per-image decode
and lp_batch; the results must equal the oracle's pixels and the default setting's output byte for byte."""
import ctypes as C
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _corpus():
    """(name, file) pairs: the catalogue's scans without restart markers, then 1080p files written by cv2."""
    import cv2

    from lilliput_b200 import corpus
    from tests import jpeg_baseline_streams as jb

    files = [(s.name, s.data) for s in jb.cases() if not s.restart]
    for i in range(2):
        img = corpus.pcg64_frame(i)
        q90 = [cv2.IMWRITE_JPEG_QUALITY, 90]
        files.append((f"1080p_420_{i}", cv2.imencode(".jpg", img, q90)[1].tobytes()))
        files.append((f"1080p_420_opt_{i}", cv2.imencode(".jpg", img, q90 + [cv2.IMWRITE_JPEG_OPTIMIZE, 1])[1].tobytes()))
        files.append((f"1080p_gray_{i}", cv2.imencode(".jpg", cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), q90)[1].tobytes()))
        for tag, sf in (("444", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444), ("422", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422)):
            enc = cv2.imencode(".jpg", img, q90 + [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf])[1].tobytes()
            files.append((f"1080p_{tag}_{i}", enc))
    return files


def _child(inp: str, out: str) -> None:
    """Decode every file per image and through lp_batch; write results and the decoder's diagnostics."""
    from lilliput_b200 import abi

    lib = abi.load_cuda()
    clocks = lib.l.lp_huff_phase_clocks
    clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    lib.l.lp_batch_sync_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)]
    with open(inp, "rb") as f:
        files = pickle.load(f)
    ctr = (C.c_ulonglong * 8)()
    clocks(ctr, 1)
    res = {"decode": {}, "batch": {}, "rounds": {}}
    for name, data in files:
        try:
            res["decode"][name] = lib.decode(data)
        except abi.LilliputError as e:
            res["decode"][name] = e.code
    by = {}
    for name, data in files:
        by.setdefault(lib.header(data)[:2], []).append((name, data))
    for (W, H), group in sorted(by.items()):
        n = len(group)
        b = abi.Batch(lib, 0, n, W, H, max(1, W // 2), max(1, H // 2), 85,
                      max_in_bytes=sum(len(d) for _, d in group) + (1 << 20), out_cap=1 << 22, chunk=n)
        try:
            outs, status = b.transform([d for _, d in group])
            mean, mx = C.c_double(), C.c_int()
            lib.l.lp_batch_sync_rounds(b.h, C.byref(mean), C.byref(mx))
        finally:
            b.close()
        for (name, _), o, s in zip(group, outs, status):
            res["batch"][name] = (s, o)
        res["rounds"][(W, H)] = (mean.value, mx.value)
    clocks(ctr, 1)
    res["bits_sync"], res["bits_guess"] = int(ctr[6]), int(ctr[7])
    with open(out, "wb") as f:
        pickle.dump(res, f)


def _run(tmp_path, inp, spt):
    out = str(tmp_path / f"spt_{spt}.pkl")
    env = dict(os.environ)
    env.pop("LP_HUFF_SPT", None)
    if spt is not None:
        env["LP_HUFF_SPT"] = str(spt)
    subprocess.run([sys.executable, "-m", "tests.test_gpu_huff_sync_rounds", inp, out], cwd=ROOT, env=env,
                   check=True, timeout=1800)
    with open(out, "rb") as f:
        return pickle.load(f)


def test_many_rounds_match_oracle_and_default(tmp_path, oracle):
    files = _corpus()
    inp = str(tmp_path / "files.pkl")
    with open(inp, "wb") as f:
        pickle.dump(files, f)
    stress, default = _run(tmp_path, inp, 8), _run(tmp_path, inp, None)
    bad = []
    for name, data in files:
        want = oracle.jpeg_decode(data)[0]
        got = stress["decode"][name]
        if not isinstance(got, np.ndarray) or got.shape != want.shape or not np.array_equal(got, want):
            bad.append(f"{name}: per-image decode differs from the oracle")
        if not np.array_equal(got, default["decode"][name]):
            bad.append(f"{name}: per-image decode differs from the default setting")
        if stress["batch"][name][0] != 0 or stress["batch"][name] != default["batch"][name]:
            bad.append(f"{name}: lp_batch output differs from the default setting")
    assert bad == []
    # the stress setting really ran many rounds on the 1080p files, and re-decoded more than the default setting did
    mean, mx = stress["rounds"][(1920, 1080)]
    assert mx >= 4 and mean > default["rounds"][(1920, 1080)][0], (stress["rounds"], default["rounds"])
    # both settings decode the same streams once in their guess pass (the stress setting's subsequences overrun their
    # ends on more boundaries)
    assert 0 < default["bits_guess"] <= stress["bits_guess"] < 1.01 * default["bits_guess"]
    assert 0 < default["bits_sync"] < stress["bits_sync"], (default["bits_sync"], stress["bits_sync"])


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])
