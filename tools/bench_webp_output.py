#!/usr/bin/env python
"""bench.py's config 5 (mixed JPEG / PNG / WebP, 854x480 .. 3840x2160 -> Fit 256x256 through lp_xbatch_transform) with
WebP output: FileType ".webp", WebpQuality 85, instead of JPEG q85.  Corpus, timing and the JSON line are bench.py's
own; the metric name ends in `_webp` and the workload says WebP output, so the figure is never read as the JPEG one.
Takes bench.py's arguments (--config is always 5), and one of its own:

    --icc   put a 3 KiB ICC profile (one APP2 segment) into every JPEG of the corpus, so the time to read each
            profile and carry it into the output is in the figure

    python tools/bench_webp_output.py --gpus 1 --steps 1 --warmup 1 [--icc]
"""
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

ICC_BYTES = 3072


def icc_profile(n=ICC_BYTES):
    """Seeded bytes whose big-endian size field equals their length: a profile the WebP writer carries."""
    p = bytearray(np.random.default_rng(12345).integers(0, 256, n, dtype=np.uint8).tobytes())
    p[0:4] = struct.pack(">I", n)
    return bytes(p)


def with_icc(jpeg: np.ndarray, profile: bytes) -> np.ndarray:
    """The profile as one APP2 "ICC_PROFILE" segment behind SOI and the JFIF APP0 segment."""
    b = jpeg.tobytes()
    at = 4 + struct.unpack(">H", b[4:6])[0] if b[2:4] == b"\xff\xe0" else 2
    payload = b"ICC_PROFILE\0" + bytes([1, 1]) + profile
    seg = b"\xff\xe2" + struct.pack(">H", len(payload) + 2) + payload
    return np.frombuffer(b[:at] + seg + b[at:], np.uint8)


def main():
    icc = "--icc" in sys.argv
    args = [a for a in sys.argv[1:] if a != "--icc"]
    cfg = bench.XCFG[5]
    metric = "images_per_sec_mixed_jpeg_png_webp_480p_4k_to_256x256_q85_webp"
    workload = cfg["workload"].replace("JPEG q85", "WebP q85 (WebP output)")
    if icc:
        metric = metric.replace("mixed_jpeg_", "mixed_jpeg_icc_")
        workload += f", a {ICC_BYTES} B ICC profile in every JPEG (APP2), carried into its WebP"
    bench.XCFG[5] = dict(cfg, metric=metric, workload=workload, opt=dict(cfg["opt"], FileType=".webp", q_key="WebpQuality", q=85))
    if icc:
        corpus = bench.x_corpus
        profile = icc_profile()

        def x_corpus_with_icc(config, dev, n, distinct, rank):
            files, idx = corpus(config, dev, n, distinct, rank)
            return [with_icc(f, profile) if f[0] == 0xFF and f[1] == 0xD8 else f for f in files], idx
        bench.x_corpus = x_corpus_with_icc
    sys.argv = [sys.argv[0], "--config", "5"] + args
    return bench.main()


if __name__ == "__main__":
    sys.exit(main())
