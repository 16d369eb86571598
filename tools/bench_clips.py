#!/usr/bin/env python
"""lp_xbatch_decode_clips against the alternatives, alternated in one process, on two corpora of animations:

    config4   bench.py's config-4 GIFs (128-frame 1280x720, field scrolling 4 px / frame), --items of them
    webp      bench_webp_sources.py's animations (lossy, lossless and alpha animated WebPs)

Every leg goes from host files to a device tensor: Fit 224x224, NCHW float16 RGB normalised with the ImageNet mean and
deviation (a video or frame-pooling classifier's input).

    clips     one lp_xbatch_decode_clips call, T = --frames per item
    frame0    one lp_xbatch_decode_frames call: frame 0 only, the floor
    webp      today's frame-exact route: lp_xbatch_transform to lossless animated WebP at 224, the selected frames decoded
              on the host (per-image WebP decoder) on --threads threads, normalised and uploaded

Every round checks that the clips and webp tensors agree within one ulp of float16.  Prints one JSON line per
measurement: clips/s, the call's stats, device bytes of canvases per animation, with the card's name, power limit and SM
clock.

    python tools/bench_clips.py --items 64 --rounds 3
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_batch_gray import card  # noqa: E402
from bench_frames import BIAS, BOX, SCALE  # noqa: E402
from lilliput_b200 import abi, corpus  # noqa: E402


def corpora(n):
    import torch
    import bench_webp_sources
    gifs = corpus.corpus_config4(torch.device("cuda"), min(n, 4), seed0=3000)
    return {"config4": [gifs[i % len(gifs)] for i in range(n)], "webp": bench_webp_sources.corpus(7, n, 48, 8)[0]}


def selected(F, T):
    return list(range(F)) if F <= T else [t * F // T for t in range(T)]


def ulp_apart(a, b):
    """the largest distance in float16 units in the last place between two tensors: bit patterns mapped to a monotonic
    integer line (sign-magnitude, so +0 and -0 meet and values of opposite sign are counted across zero)"""
    import torch

    def line(x):
        v = x.view(torch.int16).to(torch.int32)
        return torch.where(v < 0, -(v & 0x7FFF), v)
    return int((line(a) - line(b)).abs().max())


def clips_leg(xb, files, opt, T, out):
    t0 = time.perf_counter()
    r = xb.decode_clips(files, opt, T, out.data_ptr(), out.numel() * out.element_size(), BOX, BOX, 3, True, True, "f16",
                        SCALE, BIAS)
    return time.perf_counter() - t0, r[-1]


def frame0_leg(xb, files, opt, out):
    t0 = time.perf_counter()
    _, _, st = xb.decode_frames(files, opt, out.data_ptr(), out.numel() * out.element_size(), BOX, BOX, 3, True, True, "f16",
                                SCALE, BIAS)
    return time.perf_counter() - t0, st


def webp_leg(lib, xb, files, opt, T, out, pool):
    import torch
    t0 = time.perf_counter()
    o = abi.ImageOptions(**{**opt.__dict__, "FileType": ".webp", "EncodeOptions": {abi.WebpQuality: 101}})
    outs, st = xb.transform(files, o, out_cap=1 << 26)
    host = torch.zeros(out.shape, dtype=torch.float16).pin_memory()

    def one(i):
        if st[i]:
            return
        _, frames, _, _ = lib.webp_frames(outs[i])
        for t, k in enumerate(selected(len(frames), T)):
            f = frames[k]
            h, w = f.shape[:2]
            v = f[:, :, 2::-1].astype(np.float32) * np.float32(SCALE[:3]) + np.float32(BIAS[:3])
            host[i, t, :, :h, :w] = torch.from_numpy(np.ascontiguousarray(v.transpose(2, 0, 1))).to(torch.float16)

    list(pool.map(one, range(len(files))))
    out.copy_(host, non_blocking=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--threads", type=int, default=min(16, os.cpu_count() or 4))
    a = ap.parse_args()
    import torch
    lib = abi.load_cuda()
    info = card()
    xb = abi.XBatch(lib, 0)
    T = a.frames
    opt = abi.ImageOptions(FileType=".png", Width=BOX, Height=BOX, ResizeMethod=abi.ImageOpsFit, EncodeTimeout_ns=10**15)
    pool = ThreadPoolExecutor(a.threads)
    try:
        for name, files in corpora(a.items).items():
            n = len(files)
            inf = lib.webp_frames(files[0], decode=False)[0] if name == "webp" else lib.gif_info(files[0])
            F = inf["num_frames"] if name == "webp" else inf["frame_count"]
            canvas = inf["width"] * inf["height"] * 4
            clip = torch.empty((n, T, 3, BOX, BOX), dtype=torch.float16, device="cuda")
            ref = torch.zeros_like(clip)
            first = torch.empty((n, 3, BOX, BOX), dtype=torch.float16, device="cuda")
            clips_leg(xb, files[:4], opt, T, clip[:4])  # warm-up of every shape
            frame0_leg(xb, files[:4], opt, first[:4])
            webp_leg(lib, xb, files[:4], opt, T, ref[:4], pool)
            for r in range(a.rounds):
                for leg in ("clips", "frame0", "webp"):
                    if leg == "clips":
                        s, st = clips_leg(xb, files, opt, T, clip)
                    elif leg == "frame0":
                        s, st = frame0_leg(xb, files, opt, first)
                    else:
                        s, st = webp_leg(lib, xb, files, opt, T, ref, pool)
                    stats = xb.stats()
                    # device bytes of composited canvases per animation: a clip stores min(F, T), the others every frame
                    canvases = {"clips": min(F, T), "frame0": 1, "webp": F}[leg] * canvas
                    rec = {"tool": "bench_clips", "corpus": name, "leg": leg, "round": r, "items": n, "T": T, "s": round(s, 4),
                           "canvas_bytes_per_anim": canvases,
                           "clips_per_s": round(n / s, 1), "ok": st.count(0),
                           **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}, **info}
                    print(json.dumps(rec), flush=True)
                assert ulp_apart(clip, ref) <= 1, f"{name}: clips and the WebP route differ by {ulp_apart(clip, ref)} ulp"
    finally:
        pool.shutdown()
        xb.close()


if __name__ == "__main__":
    main()
