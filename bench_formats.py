#!/usr/bin/env python3
"""Secondary measurement (NOT the bench.py contract line): the per-image C-ABI path for the rows of
SURVEY.md s.8 that were widened after the JPEG hot path -- PNG, GIF, WebP in and out -- timed on
the device next to the reference's own CPU code (oracle/_ref) on this box's host cores, same inputs,
same call (lp_transform / decode helpers), wall clock around the synchronous call (host<->device
copies included).  One image per call is the reference's API shape and the worst case for a GPU:
every one of these decoders / encoders is a serial entropy coder per stream, so the device only
wins on these formats once many streams are in flight (the batch ABI is JPEG-only today).

    python bench_formats.py            # prints one JSON line per workload
"""
import io
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from lilliput_b200 import abi  # noqa: E402
from lilliput_b200.synth import synth_image  # noqa: E402
from tests.png_writer import write_png  # noqa: E402

T = 600 * 10**9


def timed(fn, reps):
    fn()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t) / reps * 1e3


def main():
    cuda = abi.load_cuda()
    ref = abi.load_reference() if os.path.exists(abi.REF_LIB) else None
    import zlib  # noqa: F401  (png_writer)
    rows = []

    def add(name, workload, fn_for, reps=3):
        g = timed(lambda: fn_for(cuda), reps)
        c = timed(lambda: fn_for(ref), reps) if ref else None
        rows.append({"workload": name, "what": workload, "gpu_ms_per_call": round(g, 2),
                     "cpu_reference_ms_per_call": None if c is None else round(c, 2),
                     "speedup_vs_cpu": None if c is None else round(c / g, 3)})
        print(json.dumps(rows[-1]), flush=True)

    # ---- inputs
    rgba4k = synth_image(3, 3840, 2160, 4)
    png4k = cuda.encode(".png", rgba4k, {abi.PngCompression: 3})
    bgr1080 = synth_image(4, 1920, 1080, 3)
    webp_lossy = cuda.encode(".webp", bgr1080, {abi.WebpQuality: 80})
    webp_lossless = cuda.encode(".webp", synth_image(5, 1280, 720, 3), {abi.WebpQuality: 101})
    from PIL import Image
    frames = [Image.fromarray(synth_image(60 + i, 1280, 720, 3, noise=3.0)[:, :, ::-1].copy()).quantize(128) for i in range(8)]
    bio = io.BytesIO()
    frames[0].save(bio, "GIF", save_all=True, append_images=frames[1:], duration=50, loop=0)
    gif = bio.getvalue()

    add("png_decode_4k_rgba", "opencv_decoder_read_data on a 3840x2160 RGBA PNG (%d B)" % len(png4k),
        lambda lib: lib.decode(png4k))
    add("png_to_webp_config3", "lp_transform: 3840x2160 RGBA PNG -> Fit 512x512 -> WebP q80 + alpha (BASELINE config 3, one image)",
        lambda lib: lib.transform(png4k, abi.ImageOptions(FileType=".webp", Width=512, Height=512, ResizeMethod=abi.ImageOpsFit,
                                                          EncodeOptions={abi.WebpQuality: 80}, EncodeTimeout_ns=T)))
    add("webp_lossy_decode_1080p", "webp_decoder_decode on a 1920x1080 VP8 frame (%d B)" % len(webp_lossy),
        lambda lib: lib.webp_frames(webp_lossy))
    add("webp_lossless_decode_720p", "webp_decoder_decode on a 1280x720 VP8L frame (%d B)" % len(webp_lossless),
        lambda lib: lib.webp_frames(webp_lossless))
    add("webp_lossy_encode_512", "webp_encoder_write + flush, 512x512 BGR q80",
        lambda lib: lib.encode(".webp", bgr1080[:512, :512].copy(), {abi.WebpQuality: 80}))
    # a large frame whose alpha plane codes to many bits: the ALPH packer's worst case
    bgra4k_noisy = rgba4k.copy()
    bgra4k_noisy[:, :, 3] = np.random.Generator(np.random.PCG64(6)).integers(0, 256, (2160, 3840), dtype=np.uint8)
    add("webp_lossy_encode_4k_bgra", "webp_encoder_write + flush, 3840x2160 BGRA with a uniformly random alpha plane, q80",
        lambda lib: lib.encode(".webp", bgra4k_noisy, {abi.WebpQuality: 80}))
    add("gif_to_webp_config4", "lp_transform: 8-frame 1280x720 GIF -> Fit 256x256 -> animated WebP q80 (BASELINE config 4, 8 of 128 frames)",
        lambda lib: lib.transform(gif, abi.ImageOptions(FileType=".webp", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                                                        EncodeOptions={abi.WebpQuality: 80}, EncodeTimeout_ns=T)), reps=2)
    add("gif_to_gif_256", "lp_transform: the same GIF -> Fit 256x256 -> GIF",
        lambda lib: lib.transform(gif, abi.ImageOptions(FileType=".gif", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                                                        EncodeTimeout_ns=T)), reps=2)
    add("jpeg_transform_1080p", "lp_transform: 1920x1080 JPEG q90 -> Fit 256x256 -> JPEG q85 (the batch workload, one image per call)",
        lambda lib, j=cuda.encode(".jpeg", bgr1080, {abi.JpegQuality: 90}): lib.transform(
            j, abi.ImageOptions(FileType=".jpeg", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                                EncodeOptions={abi.JpegQuality: 85})), reps=10)


if __name__ == "__main__":
    main()
