#!/usr/bin/env python
"""lp_batch on grayscale JPEGs at the headline shape (4096 x 1920x1080 q90 -> Fit 256x256 q85), three corpora:

    colour  bench.py's config-2 corpus (4:2:0, made on the GPU)
    gray    the same pictures decoded to gray and written as one-component q90 files by cv2
    mixed   one gray file in four (items 3, 7, 11 ... of `gray`, the others of `colour`)

Per corpus: device stages (lp_batch_stage once, then lp_batch_run, wall clock around steps that end in a synchronise, and
the stage split from its events) and end to end from pinned host buffers (lp_batch_transform).  The corpora alternate
within one process, --rounds times; every item must come back LP_OK and the first few gray and mixed items must equal
lp_transform's bytes.  Prints one JSON line per measurement, with the card's name, power limit and SM clock.

    python tools/bench_batch_gray.py --rounds 2 --steps 5 --warmup 2
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lilliput_b200 import abi  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "not read", "max_sm_clock": "not read"}


def colour_files(lib, n):
    base, _arena, offs, lens = bench.make_corpus(lib, 0, n, 1000)
    return [C.string_at(base + o, ln) for o, ln in zip(offs, lens)]


def as_gray(files, threads):
    """Each picture decoded to one channel and written as a one-component JPEG of the corpus quality (host, cv2)."""
    import cv2

    def one(f):
        ok, b = cv2.imencode(".jpg", cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_GRAYSCALE),
                             [cv2.IMWRITE_JPEG_QUALITY, bench.Q_IN])
        assert ok
        return bytes(b)

    with ThreadPoolExecutor(threads) as pool:
        return list(pool.map(one, files))


class Pinned:
    """A corpus in pinned host memory with prebuilt pointer arrays, and pinned output slots."""

    def __init__(self, lib, files, out_cap):
        l = lib.l
        l.lp_host_alloc_pinned.restype = C.c_void_p
        l.lp_host_alloc_pinned.argtypes = [C.c_size_t]
        l.lp_host_free_pinned.argtypes = [C.c_void_p]
        self.l, n = l, len(files)
        self.n = n
        self.inp = l.lp_host_alloc_pinned(sum(map(len, files)))
        self.out = l.lp_host_alloc_pinned(n * out_cap)
        self.ptrs, self.lens = (C.c_void_p * n)(), (C.c_size_t * n)()
        o = 0
        for i, f in enumerate(files):
            C.memmove(self.inp + o, f, len(f))
            self.ptrs[i], self.lens[i] = self.inp + o, len(f)
            o += len(f)
        self.out_ptrs = (C.c_void_p * n)(*[self.out + i * out_cap for i in range(n)])
        self.out_lens, self.status = (C.c_size_t * n)(), (C.c_int * n)()
        self.staged = [(self.ptrs[i], self.lens[i]) for i in range(n)]

    def close(self):
        self.l.lp_host_free_pinned(self.inp)
        self.l.lp_host_free_pinned(self.out)


def device_rate(b, p, steps, warmup):
    st = b.stage(p.staged)
    assert st == [0] * p.n, "a file was refused"
    for _ in range(warmup):
        b.run()
    t0 = time.perf_counter()
    stages = {}
    for _ in range(steps):
        for k, v in b.run().items():  # lp_batch_run ends in a stream synchronise
            stages[k] = stages.get(k, 0.0) + v / steps
    wall = time.perf_counter() - t0
    return p.n * steps / wall, {k: round(v, 2) for k, v in stages.items()}, b.last_launches()


def e2e_rate(b, p, steps, warmup):
    for _ in range(warmup + 1):
        assert b.transform_into(p.ptrs, p.lens, p.n, p.out_ptrs, p.out_lens, p.status) == 0
    assert list(p.status) == [0] * p.n, "an item failed"
    t0 = time.perf_counter()
    for _ in range(steps):
        b.transform_into(p.ptrs, p.lens, p.n, p.out_ptrs, p.out_lens, p.status)
    return p.n * steps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-threads", type=int, default=max(1, min(16, os.cpu_count() or 1)),
                    help="threads writing the gray corpus")
    ap.add_argument("--check", type=int, default=8, help="gray and mixed items compared with lp_transform")
    a = ap.parse_args()
    lib = abi.load_cuda()
    info = card()
    opt = abi.ImageOptions(FileType=".jpeg", Width=bench.DST, Height=bench.DST, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: bench.Q_OUT})
    out_cap = 65536
    n = a.images
    colour = colour_files(lib, n)
    gray = as_gray(colour, a.host_threads)
    corpora = {"colour": colour, "gray": gray, "mixed": [gray[i] if i % 4 == 3 else colour[i] for i in range(n)]}
    pinned = {k: Pinned(lib, v, out_cap) for k, v in corpora.items()}
    b = abi.Batch(lib, 0, n, bench.SRC_W, bench.SRC_H, bench.DST, bench.DST, bench.Q_OUT,
                  max_in_bytes=max(sum(map(len, v)) for v in corpora.values()) + (1 << 20), out_cap=out_cap)
    try:
        for name in ("gray", "mixed"):
            b.stage(pinned[name].staged)
            b.run()
            outs, status = b.fetch(n)
            assert status == [0] * n
            for i in range(min(a.check, n)):
                assert outs[i] == lib.transform(corpora[name][i], opt), f"{name} item {i} differs from lp_transform"
        for r in range(a.rounds):
            for name, p in pinned.items():
                dev_wall, stages, launches = device_rate(b, p, a.steps, a.warmup)
                e2e = e2e_rate(b, p, a.steps, a.warmup)
                print(json.dumps({"src": f"{bench.SRC_W}x{bench.SRC_H}", "images": n, "corpus": name, "round": r,
                                  "input_mb": round(sum(map(len, corpora[name])) / 1e6, 1),
                                  "device_images_per_s": round(dev_wall, 1), "stage_ms_per_step": stages,
                                  "e2e_images_per_s": round(e2e, 1), "launches_per_step": launches, **info}), flush=True)
    finally:
        b.close()
        for p in pinned.values():
            p.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
