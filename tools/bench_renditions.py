#!/usr/bin/env python
"""Three renditions of every file: one lp_xbatch_transform_renditions call against one lp_xbatch_transform call per
rendition over the same files.  One JSON line per workload, with the card's name, power limit and maximum SM clock read
in the same process.

Renditions: Fit 256x256 JPEG q85, Fit 512x512 WebP q85 and Fit 96x96 PNG (the avatar / preview set a caller asks of
each upload).  Workloads, generated from --seed with lilliput_b200/corpus.py:
  headline  --headline-items 1920x1080 JPEG q90 files (bench.py's config-2 geometry), --distinct of them cycled
  config5   --mixed-items files of bench.py's config-5 mix (JPEG, RGB / RGBA PNG and lossy WebP at five sizes from 854x480
            to 3840x2160), item i mapped to its cell as bench.py maps it
After --warmup calls of each arm, the two arms alternate for --steps timed steps each in this process.  Every line
carries the median images/s of each arm (files per second, end to end: a host clock around calls that return with the
outputs in host memory), the device stage times of the last step (ms_decode / ms_resize / ms_encode: CUDA-event time
summed over both lanes; the per-rendition arm summed over its calls), h2d_bytes, the pair routing, and a SHA-256 over
every pair's status and bytes in item-major order, which must be equal for both arms.

    python tools/bench_renditions.py [--headline-items 2048] [--mixed-items 1000] [--distinct 8] [--steps 5] [--warmup 2]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lilliput_b200 import abi, corpus  # noqa: E402

T = 600 * 10**9
STAGES = ("ms_decode", "ms_resize", "ms_encode", "h2d_bytes", "grid_items", "fallback_items", "launches")


def renditions():
    def o(ext, w, h, enc):
        return abi.ImageOptions(FileType=ext, Width=w, Height=h, ResizeMethod=abi.ImageOpsFit, NormalizeOrientation=True,
                                EncodeOptions=enc, EncodeTimeout_ns=T)
    return [o(".jpeg", 256, 256, {abi.JpegQuality: 85}), o(".webp", 512, 512, {abi.WebpQuality: 85}), o(".png", 96, 96, {})]


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


def headline_files(n, distinct, seed):
    frames = corpus.synth_frames_gpu("cuda", distinct, 1920, 1080, 3, seed)
    files = corpus._pool_map(lambda im: corpus.encode_jpeg(im, 90), [frames[i] for i in range(distinct)])
    return [files[i % distinct] for i in range(n)]


def config5_files(n, distinct, seed):
    cells = corpus.corpus_config5("cuda", variants=distinct, seed0=seed)
    return [cells[corpus.c5_kind(i)][(i // 100) % distinct] for i in range(n)]


class Arena:
    """The files packed into one buffer and n * k output slots, item-major, shared by both arms"""

    def __init__(self, files, k, out_cap):
        self.n, self.k, self.out_cap = len(files), k, out_cap
        lens = [len(f) for f in files]
        self.blob = np.concatenate([np.frombuffer(bytes(f), np.uint8) for f in files])
        offs = np.concatenate([[0], np.cumsum(lens)[:-1]])
        self.ptrs = (C.c_void_p * self.n)(*[self.blob.ctypes.data + int(o) for o in offs])
        self.lens = (C.c_size_t * self.n)(*lens)
        self.out = np.empty((self.n * k, out_cap), np.uint8)
        self.out_ptrs = (C.c_void_p * (self.n * k))(*[self.out[p].ctypes.data for p in range(self.n * k)])
        self.out_lens = (C.c_size_t * (self.n * k))()
        self.status = (C.c_int * (self.n * k))()
        # one rendition's slots, for the per-rendition arm: pair (i, r) at i * k + r as in the renditions call
        self.rend_ptrs = [(C.c_void_p * self.n)(*[self.out[i * k + r].ctypes.data for i in range(self.n)]) for r in range(k)]
        self.rend_lens = [(C.c_size_t * self.n)() for _ in range(k)]
        self.rend_status = [(C.c_int * self.n)() for _ in range(k)]

    def digest(self, per_rendition):
        h = hashlib.sha256()
        for i in range(self.n):
            for r in range(self.k):
                p = i * self.k + r
                st, ln = ((self.rend_status[r][i], self.rend_lens[r][i]) if per_rendition else (self.status[p], self.out_lens[p]))
                h.update(int(st).to_bytes(4, "little", signed=True))
                h.update(self.out[p, :ln].tobytes())
        return h.hexdigest()

    def failures(self, per_rendition):
        return sum(1 for i in range(self.n) for r in range(self.k)
                   if (self.rend_status[r][i] if per_rendition else self.status[i * self.k + r]) != 0)


def run_workload(lib, xb, name, files, opts, args):
    l = lib.l
    k = len(opts)
    cs = [o._c() for o in opts]
    copts = (abi._ImageOptions * k)(*cs)
    a = Arena(files, k, args.out_cap)

    def renditions_call():
        rc = l.lp_xbatch_transform_renditions(xb.h, a.ptrs, a.lens, a.n, copts, k, a.out_ptrs, a.out_cap, a.out_lens, a.status)
        assert rc == 0, rc
        return xb.stats()

    def per_rendition_calls():
        total = {s: 0 for s in STAGES}
        for r in range(k):
            rc = l.lp_xbatch_transform(xb.h, a.ptrs, a.lens, a.n, C.byref(cs[r]), a.rend_ptrs[r], a.out_cap, a.rend_lens[r],
                                       a.rend_status[r])
            assert rc == 0, rc
            st = xb.stats()
            for s in STAGES:
                total[s] += st[s]
        return total

    arms = {"renditions_call": renditions_call, "one_call_per_rendition": per_rendition_calls}
    for _ in range(args.warmup):
        for fn in arms.values():
            fn()
    times = {arm: [] for arm in arms}
    last = {}
    for _ in range(args.steps):
        for arm, fn in arms.items():  # alternated, so drift in clocks or neighbours reaches both arms alike
            t0 = time.perf_counter()
            last[arm] = fn()
            times[arm].append(time.perf_counter() - t0)
    digests = {"renditions_call": a.digest(False), "one_call_per_rendition": a.digest(True)}
    out = dict(workload=name, items=a.n, renditions=[f"{o.FileType} Fit {o.Width}x{o.Height}" for o in opts],
               steps=args.steps, warmup=args.warmup, same_outputs=digests["renditions_call"] == digests["one_call_per_rendition"],
               sha256=digests["renditions_call"], failed_pairs=a.failures(False))
    for arm in arms:
        med = statistics.median(times[arm])
        out[arm] = dict(images_per_s=round(a.n / med, 1), step_s_median=round(med, 4),
                        step_s_spread=[round(min(times[arm]), 4), round(max(times[arm]), 4)],
                        **{s: (round(last[arm][s], 2) if isinstance(last[arm][s], float) else last[arm][s]) for s in STAGES})
    out["speedup"] = round(out["renditions_call"]["images_per_s"] / out["one_call_per_rendition"]["images_per_s"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--headline-items", type=int, default=2048)
    ap.add_argument("--mixed-items", type=int, default=1000)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out-cap", type=int, default=1 << 18)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--workloads", default="headline,config5")
    args = ap.parse_args()
    info = gpu_info()
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0)
    try:
        for name in args.workloads.split(","):
            if name == "headline":
                files = headline_files(args.headline_items, args.distinct, 1000 + args.seed)
            elif name == "config5":
                files = config5_files(args.mixed_items, args.distinct, 5000 + args.seed)
            else:
                raise SystemExit(f"unknown workload {name}")
            print(json.dumps(dict(info, **run_workload(lib, xb, name, files, renditions(), args))), flush=True)
    finally:
        xb.close()


if __name__ == "__main__":
    main()
