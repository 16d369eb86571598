#!/usr/bin/env python
"""HDR PNG sources (a cICP chunk with a PQ or HLG transfer, 16-bit samples) through lp_xbatch_transform, against
per-image lp_transform on host threads over the same files: one JSON line per run, with the card's name, power limit
and maximum SM clock read in the same process.

Corpus, generated from --seed: --distinct 1920x1080 16-bit PNGs, half PQ / BT.2020 and half HLG / P3, every fourth one
RGBA (the others RGB); --items files per call, cycled over the distinct ones.  Runs: Fit 256x256 to JPEG q85 and to
WebP q85.  Every line carries the median images/s over --steps timed calls (after --warmup) of both paths, the grid
call's ms_decode (inflate, defilter, tone map, resize: device time summed over both lanes), launches and routing, and
whether the two paths wrote the same status and bytes for every item.

    python tools/bench_hdr_png.py [--items 256] [--distinct 16] [--steps 3] [--warmup 1] [--threads 8] [--seed 1]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import struct
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lilliput_b200 import abi  # noqa: E402
from lilliput_b200.synth import synth_image  # noqa: E402

W, H = 1920, 1080
RUNS = {"jpeg_q85": (".jpeg", {abi.JpegQuality: 85}), "webp_q85": (".webp", {abi.WebpQuality: 85})}


def gpu_info():
    import torch
    info = dict(gpu=torch.cuda.get_device_name(0))
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(out[0])
        info["max_sm_clock_mhz"] = float(out[1])
    except Exception as e:  # (reported, never guessed)
        info["power_limit_w"] = info["max_sm_clock_mhz"] = f"unavailable: {e}"
    return info


def _chunk(tag, data):
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def hdr_png(seed, rgba, primaries, transfer):
    """a 16-bit RGB(A) PNG: the synthetic 8-bit picture in the high bytes, noise in the low bytes; every row Sub-filtered"""
    rng = np.random.default_rng(seed)
    img = synth_image(seed, W, H, 4 if rgba else 3, noise=6.0)
    s = (img[..., [2, 1, 0, 3]] if rgba else img[..., ::-1]).astype(np.uint16) * 256
    s += rng.integers(0, 256, s.shape, dtype=np.uint16)
    a = np.ascontiguousarray(s.astype(">u2")).view(np.uint8).reshape(H, -1)
    bpp = (8 if rgba else 6)
    f = a.copy()
    f[:, bpp:] = a[:, bpp:] - a[:, :-bpp]
    raw = np.concatenate([np.ones((H, 1), np.uint8), f], axis=1).tobytes()
    return (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 16, 6 if rgba else 2, 0, 0, 0)) +
            _chunk(b"cICP", bytes([primaries, transfer, 0, 1])) + _chunk(b"IDAT", zlib.compress(raw, 6)) + _chunk(b"IEND", b""))


def corpus(distinct, seed):
    return [hdr_png(seed * 1000 + k, k % 4 == 3, *((9, 16) if k % 2 == 0 else (12, 18))) for k in range(distinct)]


def digest(status, outs):
    h = hashlib.sha256()
    for st, out in zip(status, outs):
        h.update(struct.pack("<iQ", int(st), len(out)))
        h.update(out)
    return h.hexdigest()


def grid_call(xb, files, n, opt, out_cap):
    """one timed lp_xbatch_transform call; the arrays are built outside the timed region"""
    bufs = [np.frombuffer(files[i % len(files)], np.uint8) for i in range(n)]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    out = np.empty((n, out_cap), np.uint8)
    out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
    out_lens, status = (C.c_size_t * n)(), (C.c_int * n)()
    copt = opt._c()
    t0 = time.perf_counter()
    rc = xb.transform_into(ptrs, lens, n, copt, out_ptrs, out_cap, out_lens, status)
    dt = time.perf_counter() - t0
    assert rc == 0, rc
    return dt, digest(list(status), [out[i, :out_lens[i]].tobytes() for i in range(n)]), xb.stats()


def per_image_call(lib, pool, files, n, opt, out_cap):
    """lp_transform of every item on the pool's host threads (each with its own stream)"""
    def one(i):
        try:
            return 0, lib.transform(files[i % len(files)], opt, dst_cap=out_cap)
        except abi.LilliputError as e:
            return e.code, b""
    t0 = time.perf_counter()
    res = list(pool.map(one, range(n)))
    dt = time.perf_counter() - t0
    return dt, digest([r[0] for r in res], [r[1] for r in res])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--items", type=int, default=256)
    ap.add_argument("--distinct", type=int, default=16)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    info = gpu_info()
    t0 = time.perf_counter()
    files = corpus(args.distinct, args.seed)
    gen_s = time.perf_counter() - t0
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0)
    out_cap = 1 << 20
    with ThreadPoolExecutor(args.threads) as pool:
        for name, (ft, enc) in RUNS.items():
            opt = abi.ImageOptions(FileType=ft, Width=256, Height=256, ResizeMethod=abi.ImageOpsFit, EncodeOptions=enc,
                                   EncodeTimeout_ns=600 * 10**9)
            for _ in range(args.warmup):
                grid_call(xb, files, args.items, opt, out_cap)
                per_image_call(lib, pool, files, args.items, opt, out_cap)
            grid_t, per_t = [], []
            for _ in range(args.steps):  # the two paths alternated
                dt, gdig, st = grid_call(xb, files, args.items, opt, out_cap)
                grid_t.append(dt)
                dt, pdig = per_image_call(lib, pool, files, args.items, opt, out_cap)
                per_t.append(dt)
            g, p = float(np.median(grid_t)), float(np.median(per_t))
            print(json.dumps(dict(
                run=name, items=args.items, distinct_files=args.distinct, source="1920x1080 16-bit PNG, PQ/BT.2020 + HLG/P3, 1 in 4 RGBA",
                fit=[256, 256], unit="images/s", grid_rate=round(args.items / g, 2), per_image_rate=round(args.items / p, 2),
                speedup=round(p / g, 3), per_image_threads=args.threads, grid_step_s=[round(t, 4) for t in grid_t],
                per_image_step_s=[round(t, 4) for t in per_t], grid_items=st["grid_items"], fallback_items=st["fallback_items"],
                launches=st["launches"], ms_decode=round(st["ms_decode"], 2), ms_resize=round(st["ms_resize"], 2),
                ms_encode=round(st["ms_encode"], 2), bytes_identical=gdig == pdig, sha256=gdig, corpus_gen_s=round(gen_s, 2),
                **info)), flush=True)
    xb.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
