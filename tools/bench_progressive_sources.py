#!/usr/bin/env python
"""bench.py with progressive JPEG sources (written by cv2 / libjpeg-turbo at q90 4:2:0 with IMWRITE_JPEG_PROGRESSIVE).
Corpus content, timing and the JSON line are bench.py's own; the metric name ends in `_progressive_src` and the
workload says so.  Modes:

    c2       config 2 (1080p -> 256x256 JPEG through lp_batch), every source progressive; bench.py's arguments
             (e.g. --device-resident for the device-resident split with per-stage ms)
    c2mix    the same with one source in a hundred progressive (the cost to a config-2 chunk)
    c5       config 5 (mixed formats through lp_xbatch) with its JPEG share re-encoded progressive
    perimage lp_transform on the progressive config-2 sources from several host threads (--images, --threads)

    python tools/bench_progressive_sources.py c2 --gpus 1 --steps 5 --warmup 2
"""
import json
import os
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def _progressive_imencode(every):
    """cv2.imencode that writes every `every`-th JPEG progressive (1: all of them)."""
    import cv2
    plain = cv2.imencode
    count = [0]
    lock = threading.Lock()

    def imencode(ext, img, flags=()):
        with lock:
            k = count[0]
            count[0] += 1
        if ext in (".jpg", ".jpeg") and k % every == 0:
            flags = list(flags) + [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
        return plain(ext, img, flags)
    cv2.imencode = imencode


def _label(metric_suffix, workload_suffix):
    """Rename the JSON line bench.py prints so the figure is never read as the baseline-source one."""
    real = print

    def relabel(*a, **k):
        if a and isinstance(a[0], str) and a[0].startswith("{"):
            try:
                d = json.loads(a[0])
                d["metric"] = d.get("metric", "") + metric_suffix
                if isinstance(d.get("config"), dict):
                    d["config"]["workload"] = d["config"].get("workload", "") + workload_suffix
                a = (json.dumps(d),) + a[1:]
            except ValueError:
                pass
        real(*a, **k)
    bench.print = relabel


def _c5():
    import cv2
    import numpy as np
    from lilliput_b200 import corpus
    made = corpus.corpus_config5

    def progressive_cells(*a, **k):
        cells = made(*a, **k)
        for key, lst in cells.items():
            for i, f in enumerate(lst):
                if bytes(f[:2]) == b"\xff\xd8":
                    img = cv2.imdecode(np.frombuffer(bytes(f), np.uint8), cv2.IMREAD_UNCHANGED)
                    ok, b = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
                    assert ok
                    lst[i] = type(f)(b.tobytes()) if isinstance(f, (bytes, bytearray)) else np.asarray(b).reshape(-1)
        return cells
    corpus.corpus_config5 = progressive_cells


def _per_image(args):
    import cv2
    from concurrent.futures import ThreadPoolExecutor

    from lilliput_b200 import abi
    from lilliput_b200.synth import synth_image
    n = int(args[args.index("--images") + 1]) if "--images" in args else 256
    threads = int(args[args.index("--threads") + 1]) if "--threads" in args else 16
    files = []
    for i in range(min(n, 64)):
        ok, b = cv2.imencode(".jpg", synth_image(1000 + i, bench.SRC_W, bench.SRC_H, 3),
                             [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
        files.append(bytes(b))
    lib = abi.load_cuda()
    opt = abi.ImageOptions(FileType=".jpeg", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85})
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda f: lib.transform(f, opt), files[:threads]))  # warm-up
        t0 = time.perf_counter()
        list(ex.map(lambda i: lib.transform(files[i % len(files)], opt), range(n)))
        dt = time.perf_counter() - t0
    print(json.dumps({"metric": "per_image_lp_transform_progressive_src", "value": n / dt, "unit": "images/s",
                      "images": n, "threads": threads}))
    return 0


def main():
    mode, rest = sys.argv[1], sys.argv[2:]
    if mode == "perimage":
        return _per_image(rest)
    if mode in ("c2", "c2mix"):
        _progressive_imencode(1 if mode == "c2" else 100)
        _label("_progressive_src" if mode == "c2" else "_progressive_src_1pct",
               ", cv2 q90 4:2:0 progressive sources" + ("" if mode == "c2" else " (one in a hundred)"))
        rest = ["--variant", "cv2"] + rest
    elif mode == "c5":
        _c5()
        _label("_progressive_src", ", JPEG share written progressive by cv2 q90")
        rest = ["--config", "5"] + rest
    else:
        raise SystemExit(__doc__)
    sys.argv = [sys.argv[0]] + rest
    return bench.main()


if __name__ == "__main__":
    sys.exit(main())
