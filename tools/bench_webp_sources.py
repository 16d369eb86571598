#!/usr/bin/env python
"""WebP sources through the heterogeneous batch: animations written by Pillow's WebP writer (libwebp's WebPAnimEncoder,
so frames after the first are sub-rectangles with their own blend / dispose flags) -> Fit 256x256 -> animated WebP q85.

Corpus (from --seed): --anims animations of --frames frames at 640x360; half lossy + alpha, a quarter lossless, a
quarter opaque lossy.  --distinct different files are encoded (Pillow's writer is slow) and repeated to --anims.
One JSON line: animations/s through lp_xbatch_transform end to end (median of --steps calls after --warmup), the lane
stage times, grid_items / fallback_items, and the same items through per-item lp_transform on --threads host threads;
the card name and power limit are read in the same run.

    python tools/bench_webp_sources.py --steps 5 --warmup 2
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """(name, power limit in W) of device 0, read-only queries."""
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, watts = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(watts)
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), None


def animation(rng, w, h, n, kind):
    """A static textured background with a moving, changing sprite: WebPAnimEncoder writes the changed rectangle."""
    from PIL import Image
    y, x = np.mgrid[0:h, 0:w]
    bg = np.stack([(x * 255 // (w - 1)), (y * 255 // (h - 1)), (x + y) % 256, np.full_like(x, 255)], -1).astype(np.uint8)
    bg[:, :, :3] = np.clip(bg[:, :, :3].astype(int) + rng.integers(-12, 13, (h, w, 3)), 0, 255).astype(np.uint8)
    if kind == "alpha":
        bg[:, :, 3] = np.where((x // 40 + y // 40) % 2 == 0, 255, 96).astype(np.uint8)
    frames = []
    for k in range(n):
        f = bg.copy()
        cx, cy = int(40 + (w - 80) * k / max(n - 1, 1)), int(h / 2 + (h / 3) * np.sin(k / 5))
        m = (np.abs(x - cx) < 48) & (np.abs(y - cy) < 36)
        f[m, :3] = ((rng.integers(0, 256, 3) + (x[m, None] * 3)) % 256).astype(np.uint8)
        f[m, 3] = 255
        frames.append(Image.fromarray(f if kind != "opaque" else f[:, :, :3]))
    buf = io.BytesIO()
    extra = dict(lossless=True, method=0) if kind == "lossless" else dict(quality=80, method=2)
    frames[0].save(buf, "WEBP", save_all=True, append_images=frames[1:], duration=40, loop=0, **extra)
    return buf.getvalue()


def corpus(seed, anims, frames, distinct):
    rng = np.random.default_rng(seed)
    kinds = ["alpha", "alpha", "lossless", "opaque"]  # half lossy + alpha, a quarter lossless, a quarter opaque
    made = [animation(rng, 640, 360, frames, kinds[k % 4]) for k in range(distinct)]
    return [made[k % distinct] for k in range(anims)], [kinds[k % distinct % 4] for k in range(anims)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--anims", type=int, default=128)
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--arena-gb", type=float, default=40)
    a = ap.parse_args()
    from lilliput_b200 import abi
    t0 = time.perf_counter()
    files, kinds = corpus(a.seed, a.anims, a.frames, a.distinct)
    t_corpus = time.perf_counter() - t0
    lib = abi.load_cuda()
    opt = abi.ImageOptions(FileType=".webp", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.WebpQuality: 85}, EncodeTimeout_ns=10**12)
    cap = 8 << 20
    xb = abi.XBatch(lib, 0, arena_bytes=int(a.arena_gb * (1 << 30)))
    try:
        for _ in range(a.warmup):
            xb.transform(files, opt, out_cap=cap)
        times, stats = [], []
        for _ in range(a.steps):
            t = time.perf_counter()
            outs, status = xb.transform(files, opt, out_cap=cap)
            times.append(time.perf_counter() - t)
            stats.append(xb.stats())
    finally:
        xb.close()
    med = float(np.median(times))
    st = stats[int(np.argsort(times)[len(times) // 2])]
    # the same items, one lp_transform per item on host threads (each thread its own stream)
    with ThreadPoolExecutor(a.threads) as ex:
        list(ex.map(lambda f: lib.transform(f, opt, dst_cap=cap), files[:a.threads]))  # warm-up
        t = time.perf_counter()
        per = list(ex.map(lambda f: lib.transform(f, opt, dst_cap=cap), files))
        t_per = time.perf_counter() - t
    same = sum(p == o for p, o in zip(per, outs))
    name, watts = card()
    print(json.dumps({
        "metric": "webp_sources_animations_per_s", "value": round(a.anims / med, 2), "unit": "animations/s",
        "card": name, "power_limit_w": watts,
        "workload": f"{a.anims} Pillow animations x {a.frames} frames 640x360 ({a.distinct} distinct, seed {a.seed}): "
                    f"1/2 lossy+alpha, 1/4 lossless, 1/4 opaque lossy -> Fit 256x256 -> animated WebP q85",
        "batch_s_median": round(med, 4), "batch_s_all": [round(x, 4) for x in times],
        "grid_items": st["grid_items"], "fallback_items": st["fallback_items"], "status_ok": sum(s == 0 for s in status),
        "lane_ms": {k: round(st[k], 2) for k in ("ms_parse", "ms_grid", "ms_fallback", "ms_total", "ms_decode", "ms_resize",
                                                  "ms_encode", "ms_busy_max_lane")},
        "per_item_lp_transform": {"threads": a.threads, "s": round(t_per, 4), "animations_per_s": round(a.anims / t_per, 2)},
        "speedup_vs_per_item": round(t_per / med, 2), "outputs_equal_to_per_item": same,
        "input_mb": round(sum(map(len, files)) / 1e6, 2), "corpus_s": round(t_corpus, 1),
    }))
    return 0 if same == len(files) else 1


if __name__ == "__main__":
    sys.exit(main())
