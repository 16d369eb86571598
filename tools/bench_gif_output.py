#!/usr/bin/env python
"""bench.py's config 4 (256 synthetic 128-frame 1280x720 GIF animations -> Fit 256x256 through lp_xbatch_transform)
with GIF output: FileType ".gif" instead of ".webp".  Corpus, timing and the JSON line are bench.py's own; the metric
name ends in `_gif` and the workload says GIF output, so the figure is never read as the animated-WebP one.  Takes
bench.py's arguments (--config is always 4):

    python tools/bench_gif_output.py --gpus 1 --steps 1 --warmup 1
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    cfg = bench.XCFG[4]
    bench.XCFG[4] = dict(cfg, metric="animations_per_sec_128f_720p_gif_to_256x256_gif",
                         workload=cfg["workload"].replace("animated WebP q85", "GIF (GIF output)"),
                         opt=dict(cfg["opt"], FileType=".gif"))
    sys.argv = [sys.argv[0], "--config", "4"] + [a for a in sys.argv[1:]]
    return bench.main()


if __name__ == "__main__":
    sys.exit(main())
