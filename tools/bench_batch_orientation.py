#!/usr/bin/env python
"""lp_batch on EXIF-rotated JPEGs: the same files with every EXIF tag 1, and with tags 1 / 6 / 8 / 3 in turn (the way
phone cameras tag portrait and upside-down shots).  The two corpora differ only in that tag byte, so their difference is
the cost of the orientation pass and the per-class resize launches.

Two shapes, Fit 256x256 q85:
    headline  bench.py's config-2 corpus (1080p 4:2:0 q90, made on the GPU), 4096 images
    camera    4032x3024 4:2:0 q90 from cv2 (--camera-distinct files repeated), 128 images

Per shape and corpus: device stages (lp_batch_stage once, then lp_batch_run, wall clock around steps that end in a
synchronise) and end to end from pinned host buffers (lp_batch_transform).  The corpora alternate within one process,
--rounds times; every item must come back LP_OK and the first few mixed items must equal lp_transform's bytes.  Prints
one JSON line per measurement, with the card's name and power limit.

    python tools/bench_batch_orientation.py --rounds 3 --steps 5 --warmup 2
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lilliput_b200 import abi  # noqa: E402
from lilliput_b200.synth import synth_image  # noqa: E402

MIX = (1, 6, 8, 3)


def with_exif_orientation(jpeg: bytes, orientation: int) -> bytes:
    """APP1 / EXIF with one IFD entry (0x0112 orientation) right behind SOI."""
    tiff = b"II*\x00\x08\x00\x00\x00" + b"\x01\x00" + b"\x12\x01\x03\x00\x01\x00\x00\x00" + bytes([orientation, 0, 0, 0]) + b"\x00\x00\x00\x00"
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + jpeg[2:]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "not read", "max_sm_clock": "not read"}


def headline_files(lib, n):
    base, _arena, offs, lens = bench.make_corpus(lib, 0, n, 1000)
    return [C.string_at(base + o, ln) for o, ln in zip(offs, lens)], (bench.SRC_W, bench.SRC_H)


def camera_files(n, distinct):
    import cv2
    w, h = 4032, 3024
    uniq = []
    for k in range(distinct):
        ok, b = cv2.imencode(".jpg", synth_image(3000 + k, w, h, 3), [cv2.IMWRITE_JPEG_QUALITY, 90])
        assert ok
        uniq.append(bytes(b))
    return [uniq[i % distinct] for i in range(n)], (w, h)


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
    dev_ms = 0.0
    for _ in range(steps):
        dev_ms += b.run()["total"]  # lp_batch_run ends in a stream synchronise
    wall = time.perf_counter() - t0
    return p.n * steps / wall, p.n * steps / (dev_ms / 1e3), b.last_launches()


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
    ap.add_argument("--shapes", default="headline,camera")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--headline-images", type=int, default=4096)
    ap.add_argument("--camera-images", type=int, default=128)
    ap.add_argument("--camera-distinct", type=int, default=16)
    ap.add_argument("--check", type=int, default=8, help="mixed-corpus items compared with lp_transform")
    a = ap.parse_args()
    lib = abi.load_cuda()
    info = card()
    opt = abi.ImageOptions(FileType=".jpeg", Width=bench.DST, Height=bench.DST, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: bench.Q_OUT})
    out_cap = 65536
    for shape in a.shapes.split(","):
        files, (w, h) = (headline_files(lib, a.headline_images) if shape == "headline"
                         else camera_files(a.camera_images, a.camera_distinct))
        corpora = {"tags_1": [with_exif_orientation(f, 1) for f in files],
                   "tags_1683": [with_exif_orientation(f, MIX[i % 4]) for i, f in enumerate(files)]}
        n = len(files)
        pinned = {k: Pinned(lib, v, out_cap) for k, v in corpora.items()}
        b = abi.Batch(lib, 0, n, w, h, bench.DST, bench.DST, bench.Q_OUT,
                      max_in_bytes=max(sum(map(len, v)) for v in corpora.values()) + (1 << 20), out_cap=out_cap)
        try:
            mixed = corpora["tags_1683"]
            b.stage(pinned["tags_1683"].staged)
            b.run()
            outs, status = b.fetch(n)
            assert status == [0] * n
            for i in range(min(a.check, n)):
                assert outs[i] == lib.transform(mixed[i], opt), f"{shape} item {i} differs from lp_transform"
            for r in range(a.rounds):
                for name, p in pinned.items():
                    dev_wall, dev_events, launches = device_rate(b, p, a.steps, a.warmup)
                    e2e = e2e_rate(b, p, a.steps, a.warmup)
                    print(json.dumps({"shape": shape, "src": f"{w}x{h}", "images": n, "corpus": name, "round": r,
                                      "device_images_per_s": round(dev_wall, 1),
                                      "device_images_per_s_events": round(dev_events, 1),
                                      "e2e_images_per_s": round(e2e, 1), "launches": launches, **info}), flush=True)
        finally:
            b.close()
            for p in pinned.values():
                p.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
