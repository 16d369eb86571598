#!/usr/bin/env python
"""Per-image WebP decode (webp_decoder_*) across two builds of the library: byte identity and speed, in one session.

Each build runs in its own process (LP_CUDA_LIB), the builds alternating for --rounds rounds.  The first run of each build hashes,
for every file of a seeded corpus, every frame of abi.webp_frames with the container info, frame metadata and status, and
lp_transform of the file to JPEG, PNG and WebP (or the error it returns).  The corpus: lossy stills on 3- and 4-channel
canvases, lossy + ALPH, lossless with and without the alpha bit, Pillow animations (WebPAnimEncoder: frames after the
first are sub-rectangles with their own blend / dispose), damaged and truncated frames, sizes 1x1 to 3840x2160.  Then it
times the per-image decode: bench_formats.py's webp_lossy_decode_1080p and webp_lossless_decode_720p inputs, a 3840x2160
lossless frame and many-frame small-canvas animations (median ms per webp_frames call), every round.  One JSON line: whether every
hash agrees across the builds, and each build's timings per round, with the card name and power limit.

    python tools/webp_decode_identity.py --libs OLD.so NEW.so --rounds 3
"""
import argparse
import hashlib
import io
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def pillow_webp(img, **kw):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "WEBP", **kw)
    return buf.getvalue()


def pillow_animation(rng, w, h, n, kind):
    """A textured background with a moving sprite: WebPAnimEncoder writes the changed rectangle of each frame."""
    from PIL import Image
    y, x = np.mgrid[0:h, 0:w]
    bg = np.stack([x * 255 // max(w - 1, 1), y * 255 // max(h - 1, 1), (x + y) % 256, np.full_like(x, 255)], -1).astype(np.uint8)
    if kind == "alpha":
        bg[:, :, 3] = np.where((x // 16 + y // 16) % 2 == 0, 255, 96).astype(np.uint8)
    frames = []
    for k in range(n):
        f = bg.copy()
        cx, cy = int(w * (k + 1) / (n + 1)), int(h / 2 + (h / 4) * np.sin(k / 3))
        m = (np.abs(x - cx) < max(w // 10, 2)) & (np.abs(y - cy) < max(h // 8, 2))
        f[m, :3] = rng.integers(0, 256, 3).astype(np.uint8)
        f[m, 3] = 255
        frames.append(Image.fromarray(f if kind != "opaque" else f[:, :, :3]))
    buf = io.BytesIO()
    extra = dict(lossless=True, method=0) if kind == "lossless" else dict(quality=75, method=2)
    frames[0].save(buf, "WEBP", save_all=True, append_images=frames[1:], duration=40, loop=0, **extra)
    return buf.getvalue()


def damaged(name, data, rng):
    """The file with its image chunk cut short (container sizes rewritten) or with bytes of it overwritten."""
    from tests.webp_util import chunks_of, riff
    ch = chunks_of(data)
    k = max(i for i, (t, _) in enumerate(ch) if t in (b"VP8 ", b"VP8L", b"ALPH", b"ANMF"))
    out = {}
    p = ch[k][1]
    for frac in (0.3, 0.6, 0.95):
        cut = list(ch)
        cut[k] = (ch[k][0], p[:max(1, int(len(p) * frac))])
        out[f"{name}/cut{frac}"] = riff(cut)
    hit = bytearray(p)
    lo = min(len(hit) - 1, 24 if ch[k][0] == b"ANMF" else 10)
    for pos in rng.integers(lo, len(hit), 6):
        hit[pos] ^= 0x5A
    bad = list(ch)
    bad[k] = (ch[k][0], bytes(hit))
    out[f"{name}/flip"] = riff(bad)
    return out


def corpus(seed):
    from lilliput_b200.synth import synth_image
    rng = np.random.default_rng(seed)
    files = {}
    for w, h in [(1, 1), (7, 5), (17, 33), (640, 360), (1920, 1080)]:
        rgba = synth_image(seed + h, w, h, 4)
        files[f"lossy_alph_{w}x{h}"] = pillow_webp(rgba, quality=80)
        # opaque RGBA: a 4-channel image with no ALPH chunk (VP8X without the alpha flag, or a bare VP8)
        rgba[:, :, 3] = 255
        files[f"lossy_opaque_rgba_{w}x{h}"] = pillow_webp(rgba, quality=60)
    for w, h in [(1, 1), (7, 5), (17, 33), (640, 360), (1920, 1080), (3840, 2160)]:
        files[f"lossy_rgb_{w}x{h}"] = pillow_webp(synth_image(seed + w, w, h, 3), quality=80)
    for w, h in [(1, 1), (31, 9), (1280, 720)]:
        files[f"lossless_rgb_{w}x{h}"] = pillow_webp(synth_image(seed + 3 * w, w, h, 3), lossless=True, method=0)
    for w, h in [(1, 1), (31, 9), (1280, 720), (3840, 2160)]:
        files[f"lossless_alpha_{w}x{h}"] = pillow_webp(synth_image(seed + 5 * h, w, h, 4), lossless=True, method=0)
    for kind in ("alpha", "lossless", "opaque"):
        files[f"anim_{kind}_320x180"] = pillow_animation(rng, 320, 180, 12, kind)
        files[f"anim_{kind}_64x48"] = pillow_animation(rng, 64, 48, 40, kind)
    for name in ["lossy_rgb_640x360", "lossy_alph_640x360", "lossless_rgb_1280x720", "lossless_alpha_31x9",
                 "anim_alpha_320x180", "anim_lossless_64x48"]:
        files.update(damaged(name, files[name], rng))
    return files


def digest(*parts):
    h = hashlib.sha256()
    for p in parts:
        h.update(p if isinstance(p, bytes) else repr(p).encode())
    return h.hexdigest()


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def worker(corpus_path, out_path, hash_files):
    from lilliput_b200 import abi
    lib = abi.load_cuda()
    files = pickle.load(open(corpus_path, "rb"))
    log(f"worker {abi.CUDA_LIB}: {'hashing and timing' if hash_files else 'timing'}")
    hashes = {}
    outs = {".jpeg": {abi.JpegQuality: 85}, ".png": {abi.PngCompression: 3}, ".webp": {abi.WebpQuality: 85}}
    for name, data in files.items() if hash_files else ():
        t0 = time.perf_counter()
        info, frames, metas, rc = lib.webp_frames(data)
        hashes[f"{name}/frames"] = digest(info, metas, rc, *[(f.shape, f.tobytes()) for f in frames])
        for ext, enc in outs.items():
            opt = abi.ImageOptions(FileType=ext, Width=256, Height=256, ResizeMethod=abi.ImageOpsFit, EncodeOptions=enc,
                                   EncodeTimeout_ns=600 * 10**9)
            try:
                hashes[f"{name}/transform{ext}"] = digest(lib.transform(data, opt, dst_cap=64 << 20))
            except abi.LilliputError as e:
                hashes[f"{name}/transform{ext}"] = f"error {e}"
        log(f"  {name}: {len(frames)} frames, rc {rc}, {time.perf_counter() - t0:.2f} s")
    from lilliput_b200.synth import synth_image
    timed = {  # the first two are bench_formats.py's inputs
        "webp_lossy_decode_1080p": (lib.encode(".webp", synth_image(4, 1920, 1080, 3), {abi.WebpQuality: 80}), 15),
        "webp_lossless_decode_720p": (lib.encode(".webp", synth_image(5, 1280, 720, 3), {abi.WebpQuality: 101}), 10),
        "webp_lossless_decode_4k": (lib.encode(".webp", synth_image(3, 3840, 2160, 4), {abi.WebpQuality: 101}), 3),
        "webp_anim_64x48x40_decode": (files["anim_alpha_64x48"], 30),
        "webp_anim_lossless_64x48x40_decode": (files["anim_lossless_64x48"], 30),
    }
    ms = {}
    for name, (data, reps) in timed.items():
        hashes[f"{name}/input"] = digest(data)
        lib.webp_frames(data)
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            _, frames, _, rc = lib.webp_frames(data)
            t.append((time.perf_counter() - t0) * 1e3)
            assert rc == 0 and frames
        ms[name] = round(float(np.median(t)), 3)
        log(f"  {name}: {ms[name]} ms")
    json.dump({"hashes": hashes, "ms": ms}, open(out_path, "w"))


def card():
    r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=60)
    name, watts = [c.strip() for c in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(watts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--libs", nargs=2, metavar=("OLD", "NEW"))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--out-dir", default=None, help="keep each run's hashes and timings here (default: a temporary directory)")
    ap.add_argument("--worker", nargs=3, metavar=("CORPUS", "OUT", "HASH"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker[0], a.worker[1], a.worker[2] == "1")
    with tempfile.TemporaryDirectory() as tmp:
        out_dir = a.out_dir or tmp
        os.makedirs(out_dir, exist_ok=True)
        corpus_path = os.path.join(tmp, "corpus.pkl")
        files = corpus(a.seed)
        pickle.dump(files, open(corpus_path, "wb"))
        runs = {lib: [] for lib in a.libs}
        for r in range(a.rounds):
            for lib in a.libs:
                out = os.path.join(out_dir, f"run{r}_{('old', 'new')[a.libs.index(lib)]}.json")
                env = dict(os.environ, LP_CUDA_LIB=os.path.abspath(lib))
                subprocess.check_call([sys.executable, os.path.abspath(__file__), "--worker", corpus_path, out, str(int(r == 0))],
                                      env=env)
                runs[lib].append(json.load(open(out)))
    ref, new = runs[a.libs[0]][0]["hashes"], runs[a.libs[1]][0]["hashes"]
    differ = sorted(k for k in ref.keys() | new.keys() if ref.get(k) != new.get(k))
    name, watts = card()
    print(json.dumps({
        "card": name, "power_limit_w": watts, "files": len(files), "hashes_per_run": len(ref),
        "all_hashes_equal": not differ, "differ": differ[:20], "old": a.libs[0], "new": a.libs[1],
        "ms_per_call": {side: {row: [run["ms"][row] for run in runs[lib]] for row in runs[lib][0]["ms"]}
                        for side, lib in zip(("old", "new"), a.libs)},
    }))
    return 0 if not differ else 1


if __name__ == "__main__":
    sys.exit(main())
