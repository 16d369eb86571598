#!/usr/bin/env python
"""lp_xbatch_decode_frames against the obvious alternative, alternated in one process, on two corpora:

    config5   bench.py's config-5 mix (60% JPEG, 25% PNG, 15% WebP; 854x480 .. 3840x2160)
    jpeg1080  bench.py's config-2 corpus (1920x1080 baseline JPEG q90)

Both legs go from host files to the same device tensor: Fit 224x224, NCHW float16 RGB normalised with the ImageNet mean
and deviation (a moderation or embedding model's input).

    frames    one lp_xbatch_decode_frames call into a torch tensor on the device
    png       lp_xbatch_transform to PNG (level 1), cv2 decode and normalisation on --threads host threads, upload

Every round checks that the two tensors agree (float16, one ulp).  Prints one JSON line per measurement: files/s, the
call's stats (ms_encode is the pack for the frames leg, the PNG encode for the other; launches; h2d / d2h bytes), with
the card's name, power limit and SM clock.

    python tools/bench_frames.py --items 1024 --rounds 3
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
import bench  # noqa: E402
from bench_batch_gray import card, colour_files  # noqa: E402
from lilliput_b200 import abi  # noqa: E402

MEAN = np.array([0.485, 0.456, 0.406])
STD = np.array([0.229, 0.224, 0.225])
SCALE = [float(1 / (255 * s)) for s in STD] + [1.0]
BIAS = [float(-m / s) for m, s in zip(MEAN, STD)] + [0.0]
BOX = 224


def corpora(lib, n):
    files, idx = bench.x_corpus(5, 0, n, 2, 0)
    return {"config5": [files[i] for i in idx], "jpeg1080": colour_files(lib, n)}


def frames_leg(xb, files, opt, out):
    t0 = time.perf_counter()
    _, _, st = xb.decode_frames(files, opt, out.data_ptr(), out.numel() * out.element_size(), BOX, BOX, 3, True, True, "f16",
                                SCALE, BIAS)
    return time.perf_counter() - t0, st


def png_leg(xb, files, opt, out, pool):
    import cv2
    import torch
    t0 = time.perf_counter()
    png = abi.ImageOptions(**{**opt.__dict__, "FileType": ".png", "EncodeOptions": {abi.PngCompression: 1}})
    outs, st = xb.transform(files, png, out_cap=BOX * BOX * 4 + (1 << 16))
    host = torch.zeros(out.shape, dtype=torch.float16).pin_memory()

    def one(i):
        if st[i]:
            return
        f = cv2.imdecode(np.frombuffer(outs[i], np.uint8), cv2.IMREAD_COLOR)  # (gray replicated, alpha dropped)
        h, w = f.shape[:2]
        v = f[:, :, ::-1].astype(np.float32) * np.float32(SCALE[:3]) + np.float32(BIAS[:3])
        host[i, :, :h, :w] = torch.from_numpy(np.ascontiguousarray(v.transpose(2, 0, 1))).to(torch.float16)

    list(pool.map(one, range(len(files))))
    out.copy_(host, non_blocking=True)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--threads", type=int, default=min(16, os.cpu_count() or 4))
    a = ap.parse_args()
    import torch
    lib = abi.load_cuda()
    info = card()
    xb = abi.XBatch(lib, 0)
    opt = abi.ImageOptions(FileType=".png", Width=BOX, Height=BOX, ResizeMethod=abi.ImageOpsFit, EncodeTimeout_ns=10**12)
    pool = ThreadPoolExecutor(a.threads)
    try:
        for name, files in corpora(lib, a.items).items():
            n = len(files)
            mb = sum(len(f) for f in files) / 1e6
            a_out = torch.empty((n, 3, BOX, BOX), dtype=torch.float16, device="cuda")
            b_out = torch.empty_like(a_out)
            frames_leg(xb, files[:64], opt, a_out[:64])  # warm-up of every shape
            png_leg(xb, files[:64], opt, b_out[:64], pool)
            for r in range(a.rounds):
                for leg in ("frames", "png"):
                    if leg == "frames":
                        s, st = frames_leg(xb, files, opt, a_out)
                    else:
                        s, st = png_leg(xb, files, opt, b_out, pool)
                    stats = xb.stats()
                    print(json.dumps({"tool": "bench_frames", "corpus": name, "leg": leg, "round": r, "items": n,
                                      "input_mb": round(mb, 2), "s": round(s, 4), "files_per_s": round(n / s, 1),
                                      "ok": st.count(0), **{k: (round(v, 3) if isinstance(v, float) else v)
                                                             for k, v in stats.items()}, **info}), flush=True)
                diff = (a_out.view(torch.int16).to(torch.int32) - b_out.view(torch.int16).to(torch.int32)).abs()
                assert int(diff.max()) <= 1, f"{name}: the two legs differ by {int(diff.max())} ulp"
    finally:
        pool.shutdown()
        xb.close()


if __name__ == "__main__":
    main()
