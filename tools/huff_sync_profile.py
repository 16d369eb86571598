"""How much of the JPEG entropy decoder's work the synchronisation rounds redo.

Runs N 1080p q90 4:2:0 files (config 2's content, lilliput_b200.corpus.pcg64_frame, written by cv2) through lp_batch
and prints one JSON line: bits decoded in the guess pass and in the synchronisation rounds per image
(lp_huff_phase_clocks counters 7 and 6), the rounds' share of the stream (the guess pass decodes every bit of it once),
and the rounds per image.  Run it under two builds (LP_CUDA_LIB) to compare them.

    python tools/huff_sync_profile.py --n 64 [--optimized] [--spt K]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=64)
    ap.add_argument("--optimized", action="store_true", help="image-optimised Huffman tables")
    ap.add_argument("--spt", type=int, default=0, help="set LP_HUFF_SPT (subsequences per thread) for this run")
    a = ap.parse_args()
    if a.spt:
        os.environ["LP_HUFF_SPT"] = str(a.spt)
    import cv2

    from lilliput_b200 import abi, corpus

    prm = [cv2.IMWRITE_JPEG_QUALITY, 90] + ([cv2.IMWRITE_JPEG_OPTIMIZE, 1] if a.optimized else [])
    files = [cv2.imencode(".jpg", corpus.pcg64_frame(i), prm)[1].tobytes() for i in range(a.n)]
    lib = abi.load_cuda()
    clocks = lib.l.lp_huff_phase_clocks
    clocks.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    lib.l.lp_batch_sync_rounds.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)]
    ctr = (C.c_ulonglong * 8)()
    b = abi.Batch(lib, 0, a.n, 1920, 1080, 256, 256, 85, max_in_bytes=sum(map(len, files)) + (1 << 20), chunk=a.n)
    try:
        clocks(ctr, 1)
        _, status = b.transform(files)
        clocks(ctr, 1)
        mean, mx = C.c_double(), C.c_int()
        lib.l.lp_batch_sync_rounds(b.h, C.byref(mean), C.byref(mx))
    finally:
        b.close()
    assert status == [0] * a.n, status
    sync, guess = int(ctr[6]), int(ctr[7])
    print(json.dumps({"images": a.n, "optimized": a.optimized, "spt": a.spt or None,
                      "guess_bits_per_image": round(guess / a.n), "sync_bits_per_image": round(sync / a.n),
                      "sync_share_of_stream": round(sync / guess, 4) if guess else None,
                      "rounds": {"mean": round(mean.value, 2), "max": mx.value}}))


if __name__ == "__main__":
    main()
