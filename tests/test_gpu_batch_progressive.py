"""GPU: multi-scan (progressive, or one scan per component) JPEG sources in both batch entry points.

lp_batch decodes them in the chunk next to plain, optimised and restart files (one launch of the multi-scan kernel per
chunk, coefficients in the parallel decoders' scan order); its decoded windows and resized frames must equal the
oracle's full decode cut to the window, and its status and bytes lp_transform's.  lp_xbatch puts them on the grid in
groups of their own.  Per image, every catalogue stream of tests/jpeg_scan_streams.py goes through the same kernel with
the whole frame as its window."""
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests import jpeg_decode_cases as jc
from tests import jpeg_scan_streams as js

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
T = 10**12
STREAMS = js.cases()


def _cv2(img, q=90, **kw):
    flags = [cv2.IMWRITE_JPEG_QUALITY, q]
    if kw.get("progressive"):
        flags += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    if kw.get("optimize"):
        flags += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if kw.get("rst"):
        flags += [cv2.IMWRITE_JPEG_RST_INTERVAL, kw["rst"]]
    if kw.get("sampling"):
        flags += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, kw["sampling"]]
    ok, b = cv2.imencode(".jpg", img, flags)
    assert ok
    return bytes(b)


def _per_image(lib, data, opt, cap=1 << 22):
    try:
        return lib.transform(data, opt, dst_cap=cap), 0
    except abi.LilliputError as e:
        return b"", e.code


def _mixed(W, H, seed):
    """Plain, optimised, restart and progressive files in a seeded order with a run of four progressive files."""
    rng = np.random.default_rng(seed)
    kinds = ["plain", "optimize", "rst", "prog", "prog_rst", "prog", "plain", "seq"]
    rng.shuffle(kinds)
    kinds = kinds[:3] + ["prog"] * 4 + kinds[3:]
    files = []
    for k, kind in enumerate(kinds):
        img = synth_image(seed + k, W, H, 3)
        if kind == "seq":  # one scan per component, from the stream writer
            fr = js.frame("420", W, H, seed + k)
            files.append(js.write(fr, js.sequential_per_component(), progressive=False))
            continue
        files.append(_cv2(img, 80 + k, optimize=kind == "optimize", rst=3 if kind in ("rst", "prog_rst") else 0,
                          progressive=kind.startswith("prog")))
    return kinds, files


@pytest.mark.parametrize("geom", jc.BATCH_GEOMETRIES, ids=[f"{g[0]}x{g[1]}-{g[4]}-{g[2]}x{g[3]}" for g in jc.BATCH_GEOMETRIES])
def test_batch_windows_and_frames_with_multiscan_files(cuda_lib, oracle, geom):
    W, H, dw, dh, method = geom
    kinds, files = _mixed(W, H, W * 7 + H)
    n = len(files)
    if method == "fit":
        ew, eh = oracle.expected_size(W, H, dw, dh)
        crop = oracle.fit_rect(W, H, ew, eh)
    else:
        ew, eh, crop = dw, dh, (0, 0, W, H)
    win = jc.batch_window("444", W, H, crop)
    rm = abi.ImageOpsFit if method == "fit" else abi.ImageOpsResize
    b = abi.Batch(cuda_lib, 0, n, W, H, dw, dh, 85, max_in_bytes=sum(map(len, files)) + (1 << 20), resize_method=rm)
    try:
        assert b.stage(files) == [0] * n
        b.run()
        frames = b.decoded_windows(n, win.h)
        resized = b.resized_frames(n, ew, eh)
    finally:
        b.close()
    # a chunk boundary inside the run of progressive files: the resized frames of every chunk are kept
    b = abi.Batch(cuda_lib, 0, n, W, H, dw, dh, 85, max_in_bytes=sum(map(len, files)) + (1 << 20), resize_method=rm,
                  chunk=5)
    try:
        assert b.stage(files) == [0] * n
        b.run()
        resized_chunked = b.resized_frames(n, ew, eh)
    finally:
        b.close()
    bad = []
    for i, (kind, data) in enumerate(zip(kinds, files)):
        dec, _ = oracle.jpeg_decode(data)
        got = frames[i, :, :win.w * 3].reshape(win.h, win.w, 3)
        if not np.array_equal(got, dec[win.y0:win.y0 + win.h, win.x0:win.x0 + win.w]):
            bad.append(f"{i} {kind} window")
        want_r = oracle.fit(dec, ew, eh) if method == "fit" else oracle.resize(dec, ew, eh)
        if not np.array_equal(resized[i], want_r):
            bad.append(f"{i} {kind} resized")
        if not np.array_equal(resized_chunked[i], want_r):
            bad.append(f"{i} {kind} resized (chunk of 5)")
    assert bad == []


def _progressive_sources():
    """Progressive files as the web has them: cv2 (with and without a restart interval), Pillow, this library's own
    JpegProgressive output, and the stream catalogue at one size."""
    out = []
    W, H = 203, 131
    for k in range(3):
        img = synth_image(300 + k, W, H, 3)
        out.append(_cv2(img, 75 + 10 * k, progressive=True))
        out.append(_cv2(img, 85, progressive=True, rst=2 + k))
    try:
        import io

        from PIL import Image
        for k in range(2):
            bio = io.BytesIO()
            Image.fromarray(synth_image(310 + k, W, H, 3)[:, :, ::-1]).save(bio, "JPEG", quality=88, progressive=True)
            out.append(bio.getvalue())
    except ImportError:
        pass
    out += [s.data for s in STREAMS if (s.fr.w, s.fr.h) == (W, H)]
    return out


def test_batch_progressive_sources_equal_lp_transform(cuda_lib):
    W, H = 203, 131
    files = _progressive_sources()
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    own = cuda_lib.transform(_cv2(synth_image(320, W, H, 3)), abi.ImageOptions(
        FileType=".jpeg", Width=W, Height=H, ResizeMethod=abi.ImageOpsResize,
        EncodeOptions={abi.JpegQuality: 90, abi.JpegProgressive: 1}, EncodeTimeout_ns=T))
    files.append(own)
    # a run of progressive files across chunk boundaries, next to baseline neighbours
    files = [_cv2(synth_image(330, W, H, 3))] + files + [_cv2(synth_image(331, W, H, 3))]
    n = len(files)
    b = abi.Batch(cuda_lib, 0, n, W, H, 64, 64, 85, max_in_bytes=sum(map(len, files)) + (1 << 20), chunk=7)
    try:
        outs, status = b.transform(files)
    finally:
        b.close()
    for i, f in enumerate(files):
        want, code = _per_image(cuda_lib, f, opt)
        assert status[i] == code == 0 and outs[i] == want, i


def test_per_image_catalogue_matches_oracle(cuda_lib, oracle):
    bad = []
    for s in STREAMS:
        want, _ = oracle.jpeg_decode(s.data)
        got = cuda_lib.decode(s.data)
        if got.shape != want.shape or not np.array_equal(got, want):
            bad.append(s.name)
    assert bad == []


def test_damaged_and_over_budget_files_in_both_batch_apis(cuda_lib):
    W, H = 203, 131
    good = [_cv2(synth_image(340 + k, W, H, 3), progressive=k % 2 == 1) for k in range(4)]
    damaged = [d for _, d in js.damaged()]
    files = [good[0], *damaged[:6], good[1], *damaged[6:], good[2], good[3]]
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    want = [_per_image(cuda_lib, f, opt) for f in files]
    b = abi.Batch(cuda_lib, 0, len(files), W, H, 64, 64, 85, max_in_bytes=sum(map(len, files)) + (1 << 20), chunk=6)
    try:
        outs, status = b.transform(files)
    finally:
        b.close()
    for i in range(len(files)):
        assert (status[i], outs[i]) == (want[i][1], want[i][0]), i
    # over the work budget: lp_transform refuses it, lp_batch as well, lp_xbatch hands it to lp_transform
    big = js.over_budget()
    code = _per_image(cuda_lib, big, opt)[1]
    assert code != 0
    b = abi.Batch(cuda_lib, 0, 2, 4096, 4096, 64, 64, 85, max_in_bytes=len(big) + (1 << 20))
    try:
        _, status = b.transform([big])
    finally:
        b.close()
    assert status == [code]
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    try:
        outs, status = xb.transform(files + [big], opt, out_cap=1 << 22)
        st = xb.stats()
    finally:
        xb.close()
    for i in range(len(files)):
        assert (status[i], outs[i]) == (want[i][1], want[i][0]), i
    assert status[-1] == code
    assert st["fallback_items"] >= 1  # the file over the budget (damaged files that the grid refuses follow it)


@pytest.mark.parametrize("progressive_out", [False, True])
def test_xbatch_jpeg_share_with_progressive_sources(cuda_lib, progressive_out):
    """Config 5's JPEG share with progressive files from 480p to 4K: the well-formed colour ones run on the grid, the
    out-of-scope ones (gray, EXIF-rotated) go per image; every item equals lp_transform."""
    sizes = [(854, 480), (1280, 720), (1920, 1080), (3840, 2160), (500, 333)]
    files, out_of_scope = [], 0
    for k in range(20):
        w, h = sizes[k % 5]
        gray = k == 7
        img = synth_image(400 + k, w, h, 1 if gray else 3)
        files.append(_cv2(img, 70 + k, progressive=k % 4 != 0, optimize=True, rst=5 if k % 6 == 1 else 0))
        out_of_scope += gray
    rot = bytearray(files[2])
    tiff = (b"MM\x00\x2a\x00\x00\x00\x08\x00\x01\x01\x12\x00\x03\x00\x00\x00\x01\x00\x06\x00\x00\x00\x00\x00\x00")
    body = b"Exif\x00\x00" + tiff
    files.append(bytes(rot[:2]) + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + bytes(rot[2:]))
    out_of_scope += 1
    enc = {abi.JpegQuality: 85}
    if progressive_out:
        enc[abi.JpegProgressive] = 1
    opt = abi.ImageOptions(FileType=".jpeg", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit, NormalizeOrientation=True,
                           EncodeOptions=enc, EncodeTimeout_ns=T)
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=12 << 30)
    try:
        outs, status = xb.transform(files, opt, out_cap=1 << 22)
        st = xb.stats()
    finally:
        xb.close()
    for i, f in enumerate(files):
        want, code = _per_image(cuda_lib, f, opt)
        assert (status[i], outs[i]) == (code, want), i
    assert st["fallback_items"] == out_of_scope
    assert st["grid_items"] == len(files) - out_of_scope
    m = abi.MultiBatch(cuda_lib, [0], arena_bytes=6 << 30)
    try:
        outs2, status2 = m.transform(files[:8], opt, out_cap=1 << 22)
    finally:
        m.close()
    assert outs2 == outs[:8] and status2 == status[:8]
