#!/usr/bin/env python
"""Lossless WebP output (WebpQuality 101) through lp_xbatch_transform: one JSON line per workload, with the card's name,
power limit and maximum SM clock read in the same process.

    png_sticker   4096 synthetic 512x512 RGBA PNGs (flat art, antialiased alpha) -> Fit 160x160
    gif_emoji     1024 synthetic 128x128 GIFs of 32 frames -> Fit 96x96, animated
    gif_config4   bench.py's config 4 corpus (256 x 128-frame 1280x720 GIFs) -> Fit 256x256, animated

Each line carries the median rate over --steps timed calls (after --warmup), the stage times of the last call and a
SHA-256 over the status, length and bytes of every item.

    --compare-lib PATH   also load another build of the library (the parent commit's, which writes every lossless item
                         per image) and alternate it with this one on a subset of every workload, two runs each; the
                         hashes of both builds must be equal
    --per-image          time the per-image lossless encoder (lp_encode_host -> webp_encoder_write) on one 3840x2160
                         RGBA frame and one 256x256 frame, alternated with --compare-lib's build when one is given
    --split              one more call per workload with LP_DEBUG set: the encoder's host time (stream heads and prefix
                         codes) against its device time (kernels and copies), summed over the call

    python tools/bench_lossless_webp.py [--workloads png_sticker,gif_emoji,gif_config4] [--steps 3] [--warmup 1]
                                        [--compare-lib PATH] [--per-image] [--split]
"""
import argparse
import ctypes as C
import hashlib
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from lilliput_b200 import abi  # noqa: E402

WORKLOADS = {
    "png_sticker": dict(n=4096, distinct=16, fit=(160, 160), out_cap=1 << 20, unit="images/s", subset=256),
    "gif_emoji": dict(n=1024, distinct=16, fit=(96, 96), out_cap=4 << 20, unit="animations/s", subset=64),
    "gif_config4": dict(n=256, distinct=4, fit=(256, 256), out_cap=64 << 20, unit="animations/s", subset=4),
}


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


# ---------------------------------------------------------------- corpora

def flat_art(rng, w, h, shapes=6):
    """BGRA flat-colour art: a few discs and bars on transparency, alpha antialiased over one pixel at the edges."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.zeros((h, w, 4), np.uint8)
    for _ in range(shapes):
        colour = rng.integers(0, 256, 3)
        if rng.random() < 0.6:
            cx, cy, r = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(w / 10, w / 3)
            cover = np.clip(r - np.hypot(x - cx, y - cy) + 0.5, 0, 1)
        else:
            x0, y0 = rng.uniform(0, w * 0.7), rng.uniform(0, h * 0.7)
            cover = np.clip(np.minimum(x - x0, x0 + w * 0.3 - x) + 0.5, 0, 1) * np.clip(np.minimum(y - y0, y0 + h * 0.2 - y) + 0.5, 0, 1)
        a = (cover * 255).astype(np.uint8)
        on = a > 0
        img[on, :3] = colour
        img[..., 3] = np.maximum(img[..., 3], a)
    return img


def png_sticker_files(distinct):
    import cv2
    files = []
    for k in range(distinct):
        ok, b = cv2.imencode(".png", flat_art(np.random.default_rng(100 + k), 512, 512))
        assert ok
        files.append(bytes(b))
    return files


def gif_emoji_files(distinct, frames=32, size=128):
    from PIL import Image
    files = []
    for k in range(distinct):
        rng = np.random.default_rng(200 + k)
        base = flat_art(rng, size, size, shapes=4)
        ims = []
        for t in range(frames):
            f = np.roll(base, (t * 3) % size, axis=1)
            rgb = np.where(f[..., 3:] > 127, f[..., :3], 255).astype(np.uint8)[:, :, ::-1]
            ims.append(Image.fromarray(np.ascontiguousarray(rgb)).quantize(32))
        buf = io.BytesIO()
        ims[0].save(buf, "GIF", save_all=True, append_images=ims[1:], duration=40, loop=0)
        files.append(buf.getvalue())
    return files


def gif_config4_files(distinct):
    import torch
    from lilliput_b200 import corpus
    return [f if isinstance(f, bytes) else np.asarray(f).tobytes() for f in corpus.corpus_config4(torch.device("cuda:0"), distinct, seed0=3000)]


def corpus_of(name, distinct):
    return {"png_sticker": png_sticker_files, "gif_emoji": gif_emoji_files, "gif_config4": gif_config4_files}[name](distinct)


# ---------------------------------------------------------------- runs

class Runner:
    """One library build with an lp_xbatch context and the call's arrays prepared outside the timed region."""

    def __init__(self, path, arena_bytes=0):
        self.lib = abi.Lib(path)
        self.xb = abi.XBatch(self.lib, 0, arena_bytes=arena_bytes)

    def close(self):
        self.xb.close()

    def run(self, files, n, opt, out_cap):
        bufs = [np.frombuffer(files[i % len(files)], np.uint8) for i in range(n)]
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        lens = (C.c_size_t * n)(*[b.size for b in bufs])
        out = np.empty((n, out_cap), np.uint8)
        out_ptrs = (C.c_void_p * n)(*[out[i].ctypes.data for i in range(n)])
        out_lens, status = (C.c_size_t * n)(), (C.c_int * n)()
        copt = opt._c()
        t0 = time.perf_counter()
        rc = self.xb.transform_into(ptrs, lens, n, copt, out_ptrs, out_cap, out_lens, status)
        dt = time.perf_counter() - t0
        assert rc == 0, rc
        h = hashlib.sha256()
        for i in range(n):
            h.update(int(status[i]).to_bytes(4, "little", signed=True) + int(out_lens[i]).to_bytes(8, "little"))
            h.update(out[i, :out_lens[i]].tobytes())
        return dt, h.hexdigest(), self.xb.stats()


def options(fit):
    return abi.ImageOptions(FileType=".webp", Width=fit[0], Height=fit[1], ResizeMethod=abi.ImageOpsFit,
                            EncodeOptions={abi.WebpQuality: 101}, EncodeTimeout_ns=600 * 10**9)


def capture_stderr(fn):
    """fn() with the process's fd 2 sent to a file; (result, the text written there)."""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+b") as tmp:
        os.dup2(tmp.fileno(), 2)
        try:
            res = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        return res, tmp.read().decode(errors="replace")


def per_image_times(builds, reps=5):
    """median seconds of lp_encode_host(".webp", lossless) per frame size and build, the builds alternated"""
    from lilliput_b200.synth import synth_image
    frames = {"3840x2160_rgba": synth_image(1, 3840, 2160, 4, noise=6.0), "256x256_rgba": synth_image(2, 256, 256, 4, noise=6.0)}
    out = {}
    for name, img in frames.items():
        times = {label: [] for label in builds}
        digests = {}
        for label, r in builds.items():  # warm-up
            digests[label] = hashlib.sha256(r.lib.encode(".webp", img, {abi.WebpQuality: 101})).hexdigest()
        for _ in range(reps):
            for label, r in builds.items():
                t0 = time.perf_counter()
                r.lib.encode(".webp", img, {abi.WebpQuality: 101})
                times[label].append(time.perf_counter() - t0)
        out[name] = {label: dict(median_ms=round(1e3 * float(np.median(t)), 3), min_ms=round(1e3 * min(t), 3), sha256=digests[label])
                     for label, t in times.items()}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--compare-lib", default=None)
    ap.add_argument("--per-image", action="store_true")
    ap.add_argument("--split", action="store_true")
    args = ap.parse_args()
    info = gpu_info()
    # (two builds in one process share the card: each gets a fixed arena instead of 72 % of what is free)
    arena = (24 << 30) if args.compare_lib else 0
    this = Runner(abi.CUDA_LIB, arena)
    parent = Runner(args.compare_lib, arena) if args.compare_lib else None
    for name in [w for w in args.workloads.split(",") if w]:
        w = WORKLOADS[name]
        files = corpus_of(name, w["distinct"])
        opt = options(w["fit"])
        for _ in range(args.warmup):
            this.run(files, w["n"], opt, w["out_cap"])
        times, digest, st = [], None, None
        for _ in range(args.steps):
            dt, digest, st = this.run(files, w["n"], opt, w["out_cap"])
            times.append(dt)
        line = dict(workload=name, items=w["n"], distinct_files=w["distinct"], fit=list(w["fit"]), unit=w["unit"],
                    rate=round(w["n"] / float(np.median(times)), 2), step_s=[round(t, 4) for t in times], sha256=digest,
                    grid_items=st["grid_items"], fallback_items=st["fallback_items"], launches=st["launches"],
                    ms_decode=round(st["ms_decode"], 2), ms_resize=round(st["ms_resize"], 2), ms_encode=round(st["ms_encode"], 2),
                    **info)
        if args.split:
            os.environ["LP_DEBUG"] = "1"
            _, text = capture_stderr(lambda: this.run(files, w["n"], opt, w["out_cap"]))
            del os.environ["LP_DEBUG"]
            host = dev = 0.0
            for m in re.finditer(r"vp8l batch: .*heads \(host\) ([0-9.]+) ms, device \+ copies ([0-9.]+) ms", text):
                host += float(m.group(1))
                dev += float(m.group(2))
            line.update(encoder_host_ms=round(host, 2), encoder_device_ms=round(dev, 2),
                        encoder_host_share=round(host / (host + dev), 4) if host + dev else None)
        if parent:
            k = w["subset"]
            runs = []
            for rep in range(2):
                for label, r in (("this", this), ("parent", parent)):
                    dt, h, s = r.run(files, k, opt, w["out_cap"])
                    runs.append(dict(build=label, rate=round(k / dt, 2), sha256=h, grid_items=s["grid_items"]))
            line["compare"] = dict(items=k, runs=runs, hashes_equal=len({r["sha256"] for r in runs}) == 1)
        print(json.dumps(line), flush=True)
    if args.per_image:
        builds = {"this": this}
        if parent:
            builds["parent"] = parent
        print(json.dumps(dict(workload="per_image_lossless_encode", **per_image_times(builds), **info)), flush=True)
    this.close()
    if parent:
        parent.close()
    return 0


if __name__ == "__main__":
    sys.exit(main())
