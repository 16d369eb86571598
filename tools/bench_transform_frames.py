#!/usr/bin/env python
"""Files and a model's input tensor from the same uploads: one lp_xbatch_transform_frames call against
lp_xbatch_transform_renditions followed by lp_xbatch_decode_frames over the same files, alternated in one process.  One
JSON line per workload, with the card's name, power limit and maximum SM clock read in the same process.

Outputs: Fit 256x256 JPEG q85 and Fit 512x512 WebP q85 (files), and a Fit 224x224 NCHW float16 RGB tensor normalised
with the ImageNet mean and deviation (a moderation or embedding model's input).  Workloads, generated from --seed with
lilliput_b200/corpus.py as tools/bench_renditions.py generates them:
  headline  --headline-items 1920x1080 JPEG q90 files, --distinct of them cycled
  config5   --mixed-items files of bench.py's config-5 mix
  rotated   the headline files with every third one tagged EXIF orientation 6 (the file sinks send those per image; the
            tensor takes them on the grid, decoded apart from the upright files)
After --warmup calls of each leg, the legs alternate for --steps timed steps each.  Every line carries each leg's median
files/s (a host clock around calls that return with the files in host memory and the tensor written), the device stage
times of the last step (ms_decode / ms_resize / ms_encode: CUDA-event time summed over both lanes, and over both calls of
the two-call leg), h2d_bytes, the pair routing, and a SHA-256 over every file pair's status and bytes (item-major) and
every tensor byte and frame status, which must be equal for both legs.

    python tools/bench_transform_frames.py [--headline-items 2048] [--mixed-items 1000] [--steps 5] [--warmup 2]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch_orientation import with_exif_orientation  # noqa: E402
from bench_renditions import Arena, config5_files, gpu_info, headline_files  # noqa: E402
from lilliput_b200 import abi  # noqa: E402

T = 600 * 10**9
STAGES = ("ms_decode", "ms_resize", "ms_encode", "h2d_bytes", "d2h_bytes", "grid_items", "fallback_items", "launches")
BOX = 224
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
SCALE = [1 / (255 * s) for s in STD] + [1.0]
BIAS = [-m / s for m, s in zip(MEAN, STD)] + [0.0]


def file_renditions():
    def o(ext, w, h, enc):
        return abi.ImageOptions(FileType=ext, Width=w, Height=h, ResizeMethod=abi.ImageOpsFit, NormalizeOrientation=True,
                                EncodeOptions=enc, EncodeTimeout_ns=T)
    return [o(".jpeg", 256, 256, {abi.JpegQuality: 85}), o(".webp", 512, 512, {abi.WebpQuality: 85})]


def frame_options():
    return abi.ImageOptions(FileType=".png", Width=BOX, Height=BOX, ResizeMethod=abi.ImageOpsFit, NormalizeOrientation=True)


def run_workload(lib, xb, name, files, args):
    import torch
    l = lib.l
    opts = file_renditions()
    k, n = len(opts), len(files)
    cs = [o._c() for o in opts]
    copts = (abi._ImageOptions * k)(*cs)
    fopt = frame_options()._c()
    a = Arena(files, k, args.out_cap)
    tensors = {leg: torch.empty((n, 3, BOX, BOX), dtype=torch.float16, device="cuda") for leg in ("one", "two")}
    sizes = {leg: [(C.c_int * n)() for _ in range(3)] for leg in tensors}
    frs = {leg: abi._FrameRendition(fopt, abi._frame_tensor(t.data_ptr(), t.numel() * t.element_size(), BOX, BOX, 3, True, True,
                                                            "f16", SCALE, BIAS), *[C.cast(s, C.c_void_p) for s in sizes[leg]])
           for leg, t in tensors.items()}

    def one_call():
        rc = l.lp_xbatch_transform_frames(xb.h, a.ptrs, a.lens, n, copts, k, a.out_ptrs, a.out_cap, a.out_lens, a.status,
                                          C.byref(frs["one"]), 1)
        assert rc == 0, rc
        return xb.stats()

    def two_calls():
        rc = l.lp_xbatch_transform_renditions(xb.h, a.ptrs, a.lens, n, copts, k, a.out_ptrs, a.out_cap, a.out_lens, a.status)
        assert rc == 0, rc
        total = dict(xb.stats())
        f = frs["two"]
        rc = l.lp_xbatch_decode_frames(xb.h, a.ptrs, a.lens, n, C.byref(fopt), C.byref(f.dst), *sizes["two"])
        assert rc == 0, rc
        st = xb.stats()
        for s in STAGES:
            total[s] += st[s]
        return total

    def digest(leg):
        h = hashlib.sha256()
        for p in range(n * k):
            h.update(int(a.status[p]).to_bytes(4, "little", signed=True))
            h.update(a.out[p, : a.out_lens[p]].tobytes())
        for arr in sizes[leg]:
            h.update(bytes(arr))
        h.update(tensors[leg].view(torch.uint8).cpu().numpy().tobytes())
        return h.hexdigest()

    legs = {"transform_frames": one_call, "renditions_then_decode_frames": two_calls}
    for _ in range(args.warmup):
        for fn in legs.values():
            fn()
    times = {leg: [] for leg in legs}
    last, digests = {}, {}
    for step in range(args.steps):
        for leg, fn in legs.items():  # alternated, so drift in clocks or neighbours reaches both legs alike
            t0 = time.perf_counter()
            last[leg] = fn()
            times[leg].append(time.perf_counter() - t0)
            if step == args.steps - 1:  # (the legs share the file slots: each is hashed right after it ran)
                digests[leg] = digest("one" if leg == "transform_frames" else "two")
    out = dict(workload=name, items=n, files=[f"{o.FileType} Fit {o.Width}x{o.Height}" for o in opts],
               tensor=f"Fit {BOX}x{BOX} NCHW f16 RGB normalised", steps=args.steps, warmup=args.warmup,
               same_outputs=digests["transform_frames"] == digests["renditions_then_decode_frames"],
               sha256=digests["transform_frames"], failed_frames=sum(1 for s in sizes["one"][2] if s != 0))
    for leg in legs:
        med = statistics.median(times[leg])
        out[leg] = dict(files_per_s=round(n / med, 1), step_s_median=round(med, 4),
                        step_s_spread=[round(min(times[leg]), 4), round(max(times[leg]), 4)],
                        **{s: (round(last[leg][s], 2) if isinstance(last[leg][s], float) else last[leg][s]) for s in STAGES})
    out["speedup"] = round(out["transform_frames"]["files_per_s"] / out["renditions_then_decode_frames"]["files_per_s"], 3)
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
    ap.add_argument("--workloads", default="headline,config5,rotated")
    args = ap.parse_args()
    info = gpu_info()
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0)
    try:
        for name in args.workloads.split(","):
            if name in ("headline", "rotated"):
                files = headline_files(args.headline_items, args.distinct, 1000 + args.seed)
                if name == "rotated":
                    files = [with_exif_orientation(bytes(f), 6) if i % 3 == 2 else f for i, f in enumerate(files)]
            elif name == "config5":
                files = config5_files(args.mixed_items, args.distinct, 5000 + args.seed)
            else:
                raise SystemExit(f"unknown workload {name}")
            print(json.dumps(dict(info, **run_workload(lib, xb, name, files, args))), flush=True)
    finally:
        xb.close()


if __name__ == "__main__":
    main()
