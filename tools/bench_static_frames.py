#!/usr/bin/env python
"""DisableAnimatedOutput through the heterogeneous batch: frame 0 of every animation written as a still.

Three workloads, one JSON line each:
  gif_webp   bench.py's config 4 (256 synthetic 128-frame 1280x720 GIFs, its corpus, timing and JSON line) with
             DisableAnimatedOutput -> Fit 256x256 WebP q85;
  gif_gif    the same to ".gif";
  webp_webp  the animated WebP corpus of tools/bench_webp_sources.py (Pillow / WebPAnimEncoder animations, 640x360)
             with DisableAnimatedOutput -> Fit 256x256 WebP q85, timed around lp_xbatch_transform.

--compare-lib PATH: the same items end to end with this build and with the library at PATH (for instance the parent
commit's build, which sends all of them per image), on a subset: the builds alternate in one session, two runs each,
each run in its own process (LP_CUDA_LIB), and each run prints one SHA-256 over status, length and bytes of every item.

    python tools/bench_static_frames.py --which gif_webp,gif_gif,webp_webp --steps 3 --warmup 1
    python tools/bench_static_frames.py --compare-lib /path/to/liblilliput_b200.so --subset 32
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402


def with_flag(which):
    """bench.py's config 4 with DisableAnimatedOutput and the sink of `which`; the metric and workload say so."""
    cfg = bench.XCFG[4]
    ext = ".gif" if which == "gif_gif" else ".webp"
    sink = "GIF (one frame)" if ext == ".gif" else "still WebP q85"
    bench.XCFG[4] = dict(cfg, metric=f"animations_per_sec_128f_720p_gif_first_frame_to_256x256_{ext[1:]}",
                         workload=cfg["workload"].replace("animated WebP q85", sink) + ", DisableAnimatedOutput",
                         opt=dict(cfg["opt"], FileType=ext))
    x_options = bench.x_options

    def flagged(c):
        o = x_options(c)
        o.DisableAnimatedOutput = True
        return o
    bench.x_options = flagged


def webp_corpus(a):
    import bench_webp_sources as bws
    return bws.corpus(a.seed, a.anims, a.frames, a.distinct)[0]


def webp_options():
    from lilliput_b200 import abi
    return abi.ImageOptions(FileType=".webp", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                            EncodeOptions={abi.WebpQuality: 85}, EncodeTimeout_ns=10**12, DisableAnimatedOutput=True)


def run_webp(a):
    import bench_webp_sources as bws
    from lilliput_b200 import abi
    files = webp_corpus(a)
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0, arena_bytes=int(a.arena_gb * (1 << 30)))
    opt, cap = webp_options(), 1 << 20
    try:
        for _ in range(a.warmup):
            xb.transform(files, opt, out_cap=cap)
        times, stats = [], []
        for _ in range(a.steps):
            t = time.perf_counter()
            _, status = xb.transform(files, opt, out_cap=cap)
            times.append(time.perf_counter() - t)
            stats.append(xb.stats())
    finally:
        xb.close()
    med = float(np.median(times))
    st = stats[int(np.argsort(times)[len(times) // 2])]
    name, watts = bws.card()
    print(json.dumps({
        "metric": "webp_animations_first_frame_per_s", "value": round(len(files) / med, 2), "unit": "animations/s",
        "card": name, "power_limit_w": watts,
        "workload": f"{len(files)} Pillow animations x {a.frames} frames 640x360 ({a.distinct} distinct, seed {a.seed}) "
                    f"-> DisableAnimatedOutput, Fit 256x256 -> still WebP q85",
        "batch_s_median": round(med, 4), "batch_s_all": [round(x, 4) for x in times],
        "device_stages_per_s": round(len(files) / (st["ms_busy_max_lane"] / 1000.0), 2) if st["ms_busy_max_lane"] else None,
        "grid_items": st["grid_items"], "fallback_items": st["fallback_items"], "status_ok": sum(s == 0 for s in status),
        "h2d_bytes": st["h2d_bytes"], "input_bytes": sum(map(len, files)),
        "lane_ms": {k: round(st[k], 2) for k in ("ms_parse", "ms_grid", "ms_fallback", "ms_total", "ms_decode", "ms_resize",
                                                  "ms_encode", "ms_busy_max_lane")},
    }))
    return 0 if st["fallback_items"] == 0 and all(s == 0 for s in status) else 1


def e2e_once(path, steps):
    """One end-to-end run over the saved subset with whichever library LP_CUDA_LIB names: timing + SHA-256."""
    from lilliput_b200 import abi
    z = np.load(path, allow_pickle=False)
    lib = abi.load_cuda()
    xb = abi.XBatch(lib, 0)
    line = {"lib": os.path.abspath(abi.CUDA_LIB)}
    try:
        for part in ("gif_webp", "gif_gif", "webp_webp"):
            files = [z[k].tobytes() for k in sorted(z.files) if k.startswith("gif_" if part != "webp_webp" else "webp_")]
            opt = webp_options()
            if part == "gif_gif":
                opt.FileType = ".gif"
            xb.transform(files, opt, out_cap=8 << 20)  # warm-up
            times, h = [], None
            for _ in range(steps):
                t = time.perf_counter()
                outs, status = xb.transform(files, opt, out_cap=8 << 20)
                times.append(time.perf_counter() - t)
                d = hashlib.sha256()
                for s, o in zip(status, outs):
                    d.update(int(s).to_bytes(4, "little", signed=True) + len(o).to_bytes(8, "little") + o)
                h = h or d.hexdigest()
                assert h == d.hexdigest()
            st = xb.stats()
            line[part] = {"items": len(files), "s_median": round(float(np.median(times)), 4),
                          "items_per_s": round(len(files) / float(np.median(times)), 2), "sha256": h,
                          "grid_items": st["grid_items"], "fallback_items": st["fallback_items"]}
    finally:
        xb.close()
    print(json.dumps(line), flush=True)


def compare(a):
    import torch
    from lilliput_b200 import corpus
    import bench_webp_sources as bws
    dev = torch.device("cuda", 0)
    gifs = corpus.corpus_config4(dev, bench.XCFG[4]["distinct"], seed0=3000)
    gifs = [gifs[k % len(gifs)] for k in range(a.subset)]
    webps = webp_corpus(a)[:a.subset]
    torch.cuda.empty_cache()
    tmp = tempfile.mkdtemp(prefix="lp_static_frames_")
    path = os.path.join(tmp, "subset.npz")
    np.savez(path, **{f"gif_{k:04d}": np.asarray(f, np.uint8) for k, f in enumerate(gifs)},
             **{f"webp_{k:04d}": np.frombuffer(f, np.uint8) for k, f in enumerate(webps)})
    name, watts = bws.card()
    libs = [("this", None), ("other", os.path.abspath(a.compare_lib))]
    results = []
    for rnd in range(2):
        for tag, lib in libs:
            env = dict(os.environ)
            env.pop("LP_CUDA_LIB", None)
            if lib:
                env["LP_CUDA_LIB"] = lib
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--e2e-once", path, "--steps", str(a.steps)],
                               env=env, capture_output=True, text=True)
            if r.returncode:
                sys.stderr.write(r.stderr[-4000:])
                return 1
            res = json.loads(r.stdout.strip().splitlines()[-1])
            res.update(build=tag, round=rnd)
            results.append(res)
            print(json.dumps(res), flush=True)
    same = all(r[p]["sha256"] == results[0][p]["sha256"] for r in results for p in ("gif_webp", "gif_gif", "webp_webp"))
    print(json.dumps({"metric": "static_frames_e2e_compare", "card": name, "power_limit_w": watts, "subset": a.subset,
                      "outputs_identical_across_builds": same,
                      "items_per_s": {p: {tag: [r[p]["items_per_s"] for r in results if r["build"] == tag] for tag, _ in libs}
                                      for p in ("gif_webp", "gif_gif", "webp_webp")}}))
    return 0 if same else 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", default="gif_webp,gif_gif,webp_webp")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--anims", type=int, default=128)
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--arena-gb", type=float, default=40)
    ap.add_argument("--compare-lib", default=None)
    ap.add_argument("--subset", type=int, default=32)
    ap.add_argument("--e2e-once", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.e2e_once:
        return e2e_once(a.e2e_once, a.steps)
    if a.compare_lib:
        return compare(a)
    rc = 0
    for which in a.which.split(","):
        if which == "webp_webp":
            rc |= run_webp(a)
            continue
        # bench.py's config 4 in a process of its own (bench.main reads sys.argv and its tables once)
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--bench-one", which, "--steps", str(a.steps),
                            "--warmup", str(a.warmup)])
        rc |= r.returncode
    return rc


def bench_one(which, steps, warmup):
    with_flag(which)
    sys.argv = [sys.argv[0], "--config", "4", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--no-cpu-baseline"]
    return bench.main()


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--bench-one":
        rest = sys.argv[3:]
        steps = int(rest[rest.index("--steps") + 1])
        warmup = int(rest[rest.index("--warmup") + 1])
        sys.exit(bench_one(sys.argv[2], steps, warmup))
    sys.exit(main())
