#!/usr/bin/env python
"""bench.py's config 5 (mixed JPEG / PNG / WebP, 480p..4K -> Fit 256x256 JPEG q85 through lp_xbatch_transform) with
progressive JPEG output: JpegProgressive: 1 added to the encode options.  Corpus, timing and the JSON line are
bench.py's own; the metric name ends in `_progressive` and the workload says so, so the figure is never read as the
baseline-output one.  Takes bench.py's arguments (--config is always 5):

    python tools/bench_jpeg_progressive.py --gpus 1 --steps 1 --warmup 1
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from lilliput_b200 import abi  # noqa: E402


def main():
    cfg = bench.XCFG[5]
    bench.XCFG[5] = dict(cfg, metric=cfg["metric"] + "_progressive",
                         workload=cfg["workload"] + ", progressive JPEG output (JpegProgressive: 1)")
    baseline_options = bench.x_options

    def progressive_options(c):
        o = baseline_options(c)
        o.EncodeOptions[abi.JpegProgressive] = 1
        return o

    bench.x_options = progressive_options
    sys.argv = [sys.argv[0], "--config", "5"] + [a for a in sys.argv[1:]]
    return bench.main()


if __name__ == "__main__":
    sys.exit(main())
