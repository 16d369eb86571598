"""GPU: progressive JPEG output (JpegProgressive) from the device encoder, byte-identical to what the reference writes:
OpenCV's JPEG writer with IMWRITE_JPEG_PROGRESSIVE (libjpeg-turbo, jpeg_simple_progression, optimal tables per scan),
compared live through the cv2 here.  Through the encoder, lp_transform, the batch entry points, and small buffers."""
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image
from tests.jpeg_progressive_cases import image, matrix
from tests.png_writer import write_png

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
T = 10**12


def cv2_progressive(img, q):
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    assert ok
    return enc.tobytes()


def prog(q):
    return {abi.JpegQuality: q, abi.JpegProgressive: 1}


def _first_diff(a, b):
    return next((i for i in range(min(len(a), len(b))) if a[i] != b[i]), min(len(a), len(b)))


@pytest.mark.parametrize("w,h", sorted({(c[1], c[2]) for c in matrix()}))
def test_encoder_matches_libjpeg_turbo(cuda_lib, w, h):
    for content, cw, chh, ch, q in matrix():
        if (cw, chh) != (w, h):
            continue
        img = image(content, w, h, ch)
        got, want = cuda_lib.encode(".jpg", img, prog(q)), cv2_progressive(img, q)
        assert got == want, (content, w, h, ch, q, len(got), len(want), _first_diff(got, want))


def test_round_trip_equals_baseline_pixels(cuda_lib):
    """Progressive and baseline files of a frame carry the same coefficients: both decoders see the same pixels."""
    for ch, (w, h) in [(3, (255, 257)), (1, (33, 47)), (4, (640, 360))]:
        img = synth_image(40 + ch, w, h, ch, noise=5.0)
        img = img.reshape(h, w) if ch == 1 else img
        p = cuda_lib.encode(".jpg", img, prog(85))
        b = cuda_lib.encode(".jpg", img, {abi.JpegQuality: 85})
        assert np.array_equal(cuda_lib.decode(p), cuda_lib.decode(b))
        flag = cv2.IMREAD_UNCHANGED
        assert np.array_equal(cv2.imdecode(np.frombuffer(p, np.uint8), flag), cv2.imdecode(np.frombuffer(b, np.uint8), flag))


def _rgb_png(img):
    return write_png(img[:, :, ::-1], 2, 8)


def test_transform_from_every_source_kind(cuda_lib, oracle, golden):
    """lp_transform with JpegProgressive: cv2's progressive encode of the frame the baseline output is made from."""
    jpg = oracle.jpeg_encode(synth_image(11, 640, 360, 3), 90)
    png = _rgb_png(synth_image(12, 300, 200, 3))
    webp = cuda_lib.encode(".webp", synth_image(13, 256, 144, 3), {abi.WebpQuality: 85})
    gif = golden["gif_party-discord"].tobytes()
    base = abi.ImageOptions(FileType=".jpeg", Width=128, Height=128, ResizeMethod=abi.ImageOpsFit,
                            EncodeOptions={abi.JpegQuality: 85})
    opt = abi.ImageOptions(FileType=".jpeg", Width=128, Height=128, ResizeMethod=abi.ImageOpsFit, EncodeOptions=prog(85))
    for kind, data in [("jpeg", jpg), ("png", png), ("webp", webp)]:
        if kind == "jpeg":
            src, _ = oracle.jpeg_decode(data)
        elif kind == "png":
            src = oracle.png_decode(data)
            src = src[0] if isinstance(src, tuple) else src
        else:
            src = cuda_lib.decode(data)
        frame = oracle.fit(src, 128, 128)
        assert cuda_lib.transform(data, base) == oracle.jpeg_encode(frame, 85), kind  # the frame is the right one
        assert cuda_lib.transform(data, opt) == cv2_progressive(frame, 85), kind
    # GIF: the progressive file carries the coefficients of the baseline one (pinned elsewhere to the oracle)
    p, b = cuda_lib.transform(gif, opt), cuda_lib.transform(gif, base)
    assert b"\xff\xc2" in p
    assert np.array_equal(cv2.imdecode(np.frombuffer(p, np.uint8), cv2.IMREAD_UNCHANGED),
                          cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_UNCHANGED))


def _mixed_files(oracle, cuda_lib, golden):
    files = [oracle.jpeg_encode(synth_image(100 + k, w, h, 3), 90)
             for k, (w, h) in enumerate([(320, 180), (427, 240), (320, 180), (640, 360)])]
    files.append(_rgb_png(synth_image(200, 300, 200, 3)))
    files.append(cuda_lib.encode(".webp", synth_image(300, 256, 144, 3), {abi.WebpQuality: 85}))
    files.append(golden["gif_party-discord"].tobytes())          # per image
    files.append(b"\xff\xd8\xff\xe0 not a jpeg at all")          # error item
    return files


def _check_batch(cuda_lib, batch, files, opt, cap=1 << 22):
    outs, status = batch.transform(files, opt, out_cap=cap)
    for i, f in enumerate(files):
        try:
            want, code = cuda_lib.transform(f, opt, dst_cap=cap), 0
        except abi.LilliputError as e:
            want, code = b"", e.code
        assert status[i] == code, (i, status[i], code)
        assert outs[i] == want, (i, len(outs[i]), len(want))
    return outs, status


def test_xbatch_mixed_batch_takes_the_grid_path(cuda_lib, oracle, golden):
    files = _mixed_files(oracle, cuda_lib, golden)
    opt = abi.ImageOptions(FileType=".jpeg", Width=96, Height=96, ResizeMethod=abi.ImageOpsFit,
                           NormalizeOrientation=True, EncodeOptions=prog(85), EncodeTimeout_ns=T)
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    try:
        outs, status = _check_batch(cuda_lib, xb, files, opt)
        assert status[:7] == [0] * 7 and status[7] != 0
        st = xb.stats()
        assert st["grid_items"] >= 6  # the JPEG, PNG and WebP sources: encoded by the grid path, not handed over
        for o in outs[:7]:
            assert o[:2] == b"\xff\xd8" and b"\xff\xc2" in o
    finally:
        xb.close()


def test_multi_batch_follows(cuda_lib, oracle, golden):
    files = _mixed_files(oracle, cuda_lib, golden)
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions=prog(80), EncodeTimeout_ns=T)
    m = abi.MultiBatch(cuda_lib, [0, 0], arena_bytes=3 << 30)
    try:
        _check_batch(cuda_lib, m, files, opt)
        assert sum(m.stats(g)["grid_items"] for g in range(2)) >= 6
    finally:
        m.close()


def test_small_buffers_behave_as_baseline(cuda_lib, oracle):
    """A destination too small for the file: the same outcome as for baseline output (the data moves to a buffer the
    library owns and the caller sees ErrBufTooSmall), through the encoder and through the batch."""
    img = synth_image(7, 200, 150, 3)
    outcomes = []
    for opts in ({abi.JpegQuality: 85}, prog(85)):
        full = cuda_lib.encode(".jpg", img, opts)
        row = []
        for cap in (16, len(full) // 2, len(full) - 1):
            try:
                cuda_lib.encode(".jpg", img, opts, dst_cap=cap)
                row.append("ok")
            except abi.LilliputError as e:
                row.append(e.code)
        outcomes.append(row)
    assert outcomes[0] == outcomes[1]
    files = [oracle.jpeg_encode(synth_image(800 + k, 256, 256, 3), 90) for k in range(3)]
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions=prog(85), EncodeTimeout_ns=T)
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=1 << 30)
    try:
        _check_batch(cuda_lib, xb, files, opt, cap=700)  # too small for the output: the same error per item
    finally:
        xb.close()
