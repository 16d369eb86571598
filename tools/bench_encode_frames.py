#!/usr/bin/env python
"""lp_xbatch_encode_frames against what a caller does without it, alternated in one process, on four workloads:

    f16_webp    4096 x 3x256x256 float16 NCHW RGB (v / 255) to .webp q85, NoResize
    f16_jpeg    the same tensor to .jpeg q85, NoResize
    u8_png      512 x 1024x1024 uint8 NHWC RGBA to .png, Fit 512x512
    mixed       1024 uint8 NHWC RGB items of 64..1024 per side in a 1024 box to .jpeg q85, Fit 320x320

The content is smooth (a few cosines per channel plus light noise), made on the device from a seed.

    frames    one lp_xbatch_encode_frames call on the device tensor
    host      conversion to u8 BGR(A) on the device (torch), D2H, cv2.imencode(".png", level 0) on --threads host
              threads, then lp_xbatch_transform of those PNGs

The call's contract makes the two legs' files equal; every round checks the SHA-256 over all files and statuses.
Prints one JSON line per measurement: files/s, the call's stats, the unpack's algorithmic bytes (w*h*C*sizeof(dtype)
read, w*h*C written) over ms_decode and over 3.35 TB/s, with the card's name, power limit and SM clocks.

    python tools/bench_encode_frames.py --rounds 3
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from lilliput_b200 import abi  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
T = 10**12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                            "-i", "0"], capture_output=True, text=True, timeout=60).stdout.strip()
        name, power, clock, now = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "sm_clock": now}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "not read", "max_sm_clock": "not read"}


def content(n, H, W, ch, seed, convert):
    """n x H x W x ch on the device: smooth values in 0..255 (integers) passed through `convert`, made 32 items at a time"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.arange(H, device="cuda", dtype=torch.float32).view(1, H, 1)
    x = torch.arange(W, device="cuda", dtype=torch.float32).view(1, 1, W)
    span = torch.tensor([0.05, 0.05, 6.28], device="cuda").view(3, 1, 1, 1)
    out = None
    for i0 in range(0, n, 32):
        m = min(32, n - i0)
        planes = []
        for c in range(ch):
            f = torch.full((m, H, W), 128.0, device="cuda")
            for _ in range(3):
                fx, fy, ph = torch.rand((3, m, 1, 1), device="cuda", generator=g) * span
                f += 30 * torch.cos(fx * x + fy * y + ph)
            if c == 3:
                f = 255 - f / 2
            planes.append(f + 6 * torch.randn((m, H, W), device="cuda", generator=g))
        part = convert(torch.stack(planes, -1).round().clamp(0, 255))
        if out is None:
            out = torch.empty((n,) + tuple(part.shape[1:]), dtype=part.dtype, device="cuda")
        out[i0:i0 + m] = part
    return out


def workloads(quick):
    import torch
    k = 16 if quick else 1
    fit = lambda ext, eo, w: abi.ImageOptions(FileType=ext, Width=w, Height=w, ResizeMethod=abi.ImageOpsFit, EncodeOptions=eo,
                                              EncodeTimeout_ns=T)
    nr = lambda ext, eo: abi.ImageOptions(FileType=ext, ResizeMethod=abi.ImageOpsNoResize, EncodeOptions=eo, EncodeTimeout_ns=T)
    n = 4096 // k
    f16 = content(n, 256, 256, 3, 1, lambda v: (v / 255).permute(0, 3, 1, 2).to(torch.float16))  # RGB planes
    sizes = [256] * n, [256] * n
    yield "f16_webp", f16, sizes, dict(nchw=True, rgb=True, dtype="f16", scale=[255.0] * 4), nr(".webp", {abi.WebpQuality: 85})
    yield "f16_jpeg", f16, sizes, dict(nchw=True, rgb=True, dtype="f16", scale=[255.0] * 4), nr(".jpeg", {abi.JpegQuality: 85})
    del f16
    n = 512 // k
    u8 = content(n, 1024, 1024, 4, 2, lambda v: v.to(torch.uint8))
    yield "u8_png", u8, ([1024] * n, [1024] * n), dict(nchw=False, rgb=True, dtype="u8"), fit(".png", {}, 512)
    del u8
    n = 1024 // k
    u8 = content(n, 1024, 1024, 3, 3, lambda v: v.to(torch.uint8))
    rng = np.random.default_rng(4)
    w, h = [int(v) for v in rng.integers(64, 1025, n)], [int(v) for v in rng.integers(64, 1025, n)]
    yield "mixed", u8, (w, h), dict(nchw=False, rgb=True, dtype="u8"), fit(".jpeg", {abi.JpegQuality: 85}, 320)


def digest(outs, st):
    d = hashlib.sha256()
    for o, s in zip(outs, st):
        d.update(int(s).to_bytes(4, "little", signed=True) + len(o).to_bytes(8, "little") + o)
    return d.hexdigest()


def frames_leg(xb, t, sizes, lay, opt, out_cap):
    import torch
    torch.cuda.synchronize()
    ch = t.shape[1] if lay["nchw"] else t.shape[3]
    H, W = (t.shape[2], t.shape[3]) if lay["nchw"] else (t.shape[1], t.shape[2])
    t0 = time.perf_counter()
    outs, st = xb.encode_frames(t.data_ptr(), t.numel() * t.element_size(), sizes[0], sizes[1], opt, H, W, ch, out_cap=out_cap,
                                **lay)
    return time.perf_counter() - t0, outs, st


def host_leg(xb, t, sizes, lay, opt, out_cap, pool):
    import cv2
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    x = t.permute(0, 2, 3, 1) if lay["nchw"] else t
    if lay["dtype"] != "u8":  # (bias 0: x * scale rounds once, as the library's fmaf does)
        x = torch.nan_to_num(x.float() * torch.tensor(lay["scale"][: x.shape[3]], device="cuda"), nan=0.0).round().clamp(0, 255)
    x = x.to(torch.uint8)
    if lay["rgb"]:
        x = x[..., [2, 1, 0, 3][: x.shape[3]]]
    host = x.contiguous().cpu()

    def one(i):
        f = np.ascontiguousarray(host[i, : sizes[1][i], : sizes[0][i]].numpy())
        ok, b = cv2.imencode(".png", f, [cv2.IMWRITE_PNG_COMPRESSION, 0])
        assert ok
        return bytes(b)

    pngs = list(pool.map(one, range(len(sizes[0]))))
    outs, st = xb.transform(pngs, opt, out_cap=out_cap)
    return time.perf_counter() - t0, outs, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--threads", type=int, default=min(16, os.cpu_count() or 4))
    ap.add_argument("--quick", action="store_true", help="a sixteenth of every workload")
    a = ap.parse_args()
    import torch
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0, arena_bytes=24 << 30)  # (the tensors and the host leg's copies need the rest)
    pool = ThreadPoolExecutor(a.threads)
    try:
        for name, t, sizes, lay, opt in workloads(a.quick):
            n = len(sizes[0])
            ch = t.shape[1] if lay["nchw"] else t.shape[3]
            es = t.element_size()
            alg = sum(w * h for w, h in zip(*sizes)) * ch * (es + 1)
            out_cap = (1 << 20) + (2 << 20) * (opt.FileType == ".png")
            frames_leg(xb, t[:32], (sizes[0][:32], sizes[1][:32]), lay, opt, out_cap)  # warm-up of every shape
            host_leg(xb, t[:32], (sizes[0][:32], sizes[1][:32]), lay, opt, out_cap, pool)
            info = card()
            for r in range(a.rounds):
                digests = {}
                for leg in ("frames", "host"):
                    if leg == "frames":
                        s, outs, st = frames_leg(xb, t, sizes, lay, opt, out_cap)
                    else:
                        s, outs, st = host_leg(xb, t, sizes, lay, opt, out_cap, pool)
                    stats = xb.stats()
                    digests[leg] = digest(outs, st)
                    rec = {"tool": "bench_encode_frames", "workload": name, "leg": leg, "round": r, "items": n, "s": round(s, 4),
                           "files_per_s": round(n / s, 1), "ok": st.count(0), "out_mb": round(sum(map(len, outs)) / 1e6, 2),
                           **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}, **info}
                    if leg == "frames" and stats["ms_decode"] > 0:
                        rec["unpack_alg_bytes"] = alg
                        rec["unpack_gb_per_s"] = round(alg / (stats["ms_decode"] / 1e3) / 1e9, 1)
                        rec["unpack_share_of_3_35_tb_s"] = round(alg / HBM_BYTES_PER_S * 1e3 / stats["ms_decode"], 3)
                    print(json.dumps(rec), flush=True)
                    del outs
                assert digests["frames"] == digests["host"], f"{name}: the two legs' files differ"
            del t
            torch.cuda.empty_cache()
    finally:
        pool.shutdown()
        xb.close()


if __name__ == "__main__":
    main()
