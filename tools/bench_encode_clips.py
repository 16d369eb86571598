#!/usr/bin/env python
"""lp_xbatch_encode_clips against what a caller does without it, alternated in one process, on three workloads:

    f16_webp     256 clips x 16 frames x 3x256x256 float16 NCHW RGB (v / 255) to animated .webp q85, Fit 256
    u8_lossless  64 clips x 48 frames x 512x512 uint8 NHWC RGBA to lossless animated .webp, Fit 160
    config4      16 of bench.py's config-4 GIFs (128 frames of 1280x720) through lp_xbatch_decode_clips (T = 128, u8 BGRA,
                 NoResize), then back to animated .webp q85 under NoResize with the start_ms differences as durations

The tensor content is smooth (a few cosines per channel plus light noise) and moves from frame to frame, made on the
device from a seed.

    clips     one lp_xbatch_encode_clips call on the device tensor
    host      conversion to u8 BGR(A) on the device (torch), D2H of the used frames, every clip's A_i built on --threads
              host threads (each frame a lossless exact VP8L by Pillow, method 0; timed as `build_s`), then
              lp_xbatch_transform of those files

The call's contract makes the two legs' files equal; every round checks the SHA-256 over all files and statuses.
Prints one JSON line per measurement: files/s, the call's stats, the unpack's share of the clips leg (ms_decode over
the leg's wall time), with the card's name, power limit and SM clock.

    python tools/bench_encode_clips.py --rounds 3
"""
import argparse
import hashlib
import io
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_encode_frames import card  # noqa: E402
from lilliput_b200 import abi, corpus  # noqa: E402

TIMEOUT = 10**12


def content(n, T, H, W, ch, seed, convert):
    """n * T frames of H x W x ch on the device (clip-major): smooth values in 0..255 that drift over a clip, through
    `convert`, made one clip at a time"""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.arange(H, device="cuda", dtype=torch.float32).view(1, H, 1)
    x = torch.arange(W, device="cuda", dtype=torch.float32).view(1, 1, W)
    k = torch.arange(T, device="cuda", dtype=torch.float32).view(T, 1, 1)
    out = None
    for i in range(n):
        planes = []
        for c in range(ch):
            f = torch.full((T, H, W), 128.0, device="cuda")
            for _ in range(3):
                fx, fy, ph, v = (torch.rand(4, device="cuda", generator=g) * torch.tensor([0.05, 0.05, 6.28, 0.3], device="cuda"))
                f += 30 * torch.cos(fx * x + fy * y + ph + v * k)
            if c == 3:
                f = 255 - f / 2
            planes.append(f + 6 * torch.randn((T, H, W), device="cuda", generator=g))
        part = convert(torch.stack(planes, -1).round().clamp(0, 255))
        if out is None:
            out = torch.empty((n * T,) + tuple(part.shape[1:]), dtype=part.dtype, device="cuda")
        out[i * T:(i + 1) * T] = part
    return out


def config4_clips(xb, items):
    """bench.py's config-4 GIFs through decode_clips: (u8 BGRA tensor, T, nframes, widths, heights, durations)"""
    import torch
    from lilliput_b200.abi import ImageOptions
    gifs = corpus.corpus_config4(torch.device("cuda"), min(items, 4), seed0=3000)
    files = [gifs[i % len(gifs)] for i in range(items)]
    lib = xb.lib
    T, H, W = 128, 720, 1280
    t = torch.zeros((items * T, H, W, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    opt = ImageOptions(FileType=".png", ResizeMethod=abi.ImageOpsNoResize, EncodeTimeout_ns=TIMEOUT)
    w, h, nf, index, start, st = xb.decode_clips(files, opt, T, t.data_ptr(), t.numel(), H, W, 4, False, False, "u8")
    assert st == [0] * items and max(nf) <= T
    ms = []
    for i, data in enumerate(files):
        _, delays, _, rc = lib.gif_frames(data)
        s = start[i * T:i * T + nf[i]]
        ms += [b - a for a, b in zip(s, s[1:])] + [delays[nf[i] - 1]] + [0] * (T - nf[i])
    return t, T, nf, w, h, ms


def workloads(xb, quick, names):
    import torch
    k = 8 if quick else 1
    fit = lambda eo, s: abi.ImageOptions(FileType=".webp", Width=s, Height=s, ResizeMethod=abi.ImageOpsFit, EncodeOptions=eo,
                                         EncodeTimeout_ns=TIMEOUT)
    n, T = 256 // k, 16
    if "f16_webp" in names:
        t = content(n, T, 256, 256, 3, 1, lambda v: (v / 255).permute(0, 3, 1, 2).to(torch.float16))
        yield ("f16_webp", t, T, [T] * n, [256] * n, [256] * n, [40] * (n * T),
               dict(nchw=True, rgb=True, dtype="f16", scale=[255.0] * 4), fit({abi.WebpQuality: 85}, 256))
        del t
    n, T = 64 // k, 48
    if "u8_lossless" in names:
        t = content(n, T, 512, 512, 4, 2, lambda v: v.to(torch.uint8))
        yield ("u8_lossless", t, T, [T] * n, [512] * n, [512] * n, [33] * (n * T), dict(nchw=False, rgb=True, dtype="u8"),
               fit({abi.WebpQuality: 101}, 160))
        del t
    if "config4" in names:
        t, T, nf, w, h, ms = config4_clips(xb, 16 // k)  # (16 clips of 128 720p frames: 7.5 GB of u8 BGRA)
        yield ("config4", t, T, nf, w, h, ms, dict(nchw=False, rgb=False, dtype="u8"),
               abi.ImageOptions(FileType=".webp", ResizeMethod=abi.ImageOpsNoResize, EncodeOptions={abi.WebpQuality: 85},
                                EncodeTimeout_ns=TIMEOUT))


def digest(outs, st):
    d = hashlib.sha256()
    for o, s in zip(outs, st):
        d.update(int(s).to_bytes(4, "little", signed=True) + len(o).to_bytes(8, "little") + o)
    return d.hexdigest()


def chunk(tag, payload):
    return tag + len(payload).to_bytes(4, "little") + payload + (b"\0" if len(payload) & 1 else b"")


def vp8l(frame):
    """a u8 BGR / BGRA frame as a lossless exact VP8L chunk (Pillow, method 0)"""
    from PIL import Image
    ch = frame.shape[2]
    bio = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(frame[:, :, [2, 1, 0, 3][:ch]]), "RGBA" if ch == 4 else "RGB").save(
        bio, "WEBP", lossless=True, exact=True, quality=0, method=0)
    b = bio.getvalue()
    assert b[12:16] == b"VP8L"
    return chunk(b"VP8L", b[20:20 + int.from_bytes(b[16:20], "little")])


def clip_webp(frames, durations, loops=0):
    """A_i: an animated WebP of full-canvas, no-blend, no-dispose lossless frames"""
    h, w, ch = frames[0].shape
    body = b"".join(chunk(b"ANMF", b"".join(v.to_bytes(3, "little") for v in (0, 0, w - 1, h - 1, ms)) + bytes([2]) + vp8l(f))
                    for f, ms in zip(frames, durations))
    vp8x = chunk(b"VP8X", bytes([0x02 | (0x10 if ch == 4 else 0), 0, 0, 0]) + (w - 1).to_bytes(3, "little") +
                 (h - 1).to_bytes(3, "little"))
    data = b"WEBP" + vp8x + chunk(b"ANIM", (0xFFFFFFFF).to_bytes(4, "little") + loops.to_bytes(2, "little")) + body
    return b"RIFF" + len(data).to_bytes(4, "little") + data


def dims(t, lay):
    return (t.shape[1], t.shape[2], t.shape[3]) if lay["nchw"] else (t.shape[3], t.shape[1], t.shape[2])


def clips_leg(xb, t, T, nf, w, h, ms, lay, opt, out_cap):
    import torch
    torch.cuda.synchronize()
    ch, H, W = dims(t, lay)
    t0 = time.perf_counter()
    outs, st = xb.encode_clips(t.data_ptr(), t.numel() * t.element_size(), T, nf, w, h, ms, opt, H, W, 0, ch, out_cap=out_cap, **lay)
    return time.perf_counter() - t0, 0.0, outs, st


def host_leg(xb, t, T, nf, w, h, ms, lay, opt, out_cap, pool):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = len(nf)
    used = torch.tensor([i * T + f for i in range(n) for f in range(nf[i])], device="cuda")
    x = t[used]
    x = x.permute(0, 2, 3, 1) if lay["nchw"] else x
    if lay["dtype"] != "u8":  # (bias 0: x * scale rounds once, as the library's fmaf does)
        x = torch.nan_to_num(x.float() * torch.tensor(lay["scale"][: x.shape[3]], device="cuda"), nan=0.0).round().clamp(0, 255)
    x = x.to(torch.uint8)
    if lay["rgb"]:
        x = x[..., [2, 1, 0, 3][: x.shape[3]]]
    host = x.contiguous().cpu().numpy()
    first = np.cumsum([0] + list(nf))
    tb = time.perf_counter()

    def one(i):
        frames = [host[first[i] + f, : h[i], : w[i]] for f in range(nf[i])]
        return clip_webp(frames, ms[i * T:i * T + nf[i]])

    files = list(pool.map(one, range(n)))
    build = time.perf_counter() - tb
    outs, st = xb.transform(files, opt, out_cap=out_cap)
    return time.perf_counter() - t0, build, outs, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--threads", type=int, default=min(16, os.cpu_count() or 4))
    ap.add_argument("--quick", action="store_true", help="an eighth of every workload")
    ap.add_argument("--workloads", default="f16_webp,u8_lossless,config4", help="comma-separated subset")
    a = ap.parse_args()
    import torch
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0, arena_bytes=24 << 30)  # (the tensors and the host leg's copies need the rest)
    pool = ThreadPoolExecutor(a.threads)
    try:
        for name, t, T, nf, w, h, ms, lay, opt in workloads(xb, a.quick, a.workloads.split(",")):
            n = len(nf)
            out_cap = 16 << 20
            warm = min(n, 4)  # (first calls of every shape: the encoders' pools, the per-image workers)
            clips_leg(xb, t[:warm * T], T, nf[:warm], w[:warm], h[:warm], ms[:warm * T], lay, opt, out_cap)
            host_leg(xb, t[:warm * T], T, nf[:warm], w[:warm], h[:warm], ms[:warm * T], lay, opt, out_cap, pool)
            info = card()
            for r in range(a.rounds):
                digests = {}
                for leg in ("clips", "host"):
                    if leg == "clips":
                        s, build, outs, st = clips_leg(xb, t, T, nf, w, h, ms, lay, opt, out_cap)
                    else:
                        s, build, outs, st = host_leg(xb, t, T, nf, w, h, ms, lay, opt, out_cap, pool)
                    stats = xb.stats()
                    digests[leg] = digest(outs, st)
                    rec = {"tool": "bench_encode_clips", "workload": name, "leg": leg, "round": r, "items": n, "frames": sum(nf),
                           "s": round(s, 4), "files_per_s": round(n / s, 2), "ok": st.count(0),
                           "out_mb": round(sum(map(len, outs)) / 1e6, 2),
                           **{k: (round(v, 3) if isinstance(v, float) else v) for k, v in stats.items()}, **info}
                    if leg == "clips":
                        rec["unpack_share"] = round(stats["ms_decode"] / 1e3 / s, 4)
                    else:
                        rec["build_s"] = round(build, 3)
                    print(json.dumps(rec), flush=True)
                    del outs
                assert digests["clips"] == digests["host"], f"{name}: the two legs' files differ"
            del t
            torch.cuda.empty_cache()
    finally:
        pool.shutdown()
        xb.close()


if __name__ == "__main__":
    main()
