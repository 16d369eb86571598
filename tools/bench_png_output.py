#!/usr/bin/env python
"""bench.py's config 5 (mixed JPEG / PNG / WebP, 854x480 .. 3840x2160 -> Fit 256x256 through lp_xbatch_transform) with
PNG output: FileType ".png", PngCompression 3, instead of JPEG q85.  Corpus, timing and the JSON line are bench.py's
own; the metric name ends in `_png` and the workload says PNG output, so the figure is never read as the JPEG one.
The per-item output buffer is 256 KiB: the largest file a 256x256 RGB frame can become (every DEFLATE chunk stored) is
229 889 B, so no item is refused for size.  `fallback_items` is in the line (config.fallback_items): 0 when every item
took the grid path.  Without a GPU the run fails, as bench.py does.

Takes bench.py's arguments (--config is always 5; --batch N for a subset a per-image build can finish), and one of its
own:

    --sha256   after the timed steps, print one SHA-256 over status, length and bytes of every item of the last step
               (stderr, `sha256 <hex>`): two builds of the library that write the same files print the same digest

    python tools/bench_png_output.py --gpus 1 --steps 1 --warmup 1 [--batch 1000] [--sha256]
"""
import hashlib
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def print_digest(path, prefix, outs, status, out_cap, world):
    h = hashlib.sha256()
    for st, out in zip(status, outs):
        h.update(struct.pack("<iQ", int(st), len(out)))
        h.update(out)
    print(f"sha256 {h.hexdigest()} ({prefix}, {len(outs)} items)", file=sys.stderr)


def main():
    digest = "--sha256" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--sha256"]
    cfg = bench.XCFG[5]
    bench.XCFG[5] = dict(cfg, metric="images_per_sec_mixed_jpeg_png_webp_480p_4k_to_256x256_png",
                         workload=cfg["workload"].replace("JPEG q85", "PNG, PngCompression 3 (PNG output)"),
                         opt=dict(cfg["opt"], FileType=".png", q_key="PngCompression", q=3), out_cap=1 << 18)
    if digest:
        bench.dump_outputs = print_digest  # (bench.py hands it every item of the last timed step)
        args += ["--dump-outputs", "sha256"]
    sys.argv = [sys.argv[0], "--config", "5"] + args
    return bench.main()


if __name__ == "__main__":
    sys.exit(main())
