"""GPU: the batch entry points against per-image Transform semantics and the oracle."""
import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image

pytestmark = pytest.mark.gpu


def _corpus(oracle, n, w, h, q=90):
    return [oracle.jpeg_encode(synth_image(1000 + i, w, h, 3), q) for i in range(n)]


def test_batch_matches_oracle_small(cuda_lib, oracle):
    n, w, h = 13, 320, 180
    files = _corpus(oracle, n, w, h)
    b = abi.Batch(cuda_lib, 0, 16, w, h, 64, 64, 85, max_in_bytes=sum(map(len, files)) + 4096,
                  out_cap=32768, chunk=5)  # 3 chunks, last one ragged
    try:
        outs, status = b.transform(files)
        assert status == [0] * n
        for f, o in zip(files, outs):
            dec, _ = oracle.jpeg_decode(f)
            assert o == oracle.jpeg_encode(oracle.fit(dec, 64, 64), 85)
        assert b.last_launches() > 0
    finally:
        b.close()


def test_batch_equals_per_image_transform_1080p(cuda_lib, oracle):
    """BASELINE config 2 geometry on a few images: batch output == lp_transform output == oracle."""
    n, w, h = 6, 1920, 1080
    files = _corpus(oracle, n, w, h)
    opt = abi.ImageOptions(FileType=".jpeg", Width=256, Height=256, ResizeMethod=abi.ImageOpsFit,
                           NormalizeOrientation=True, EncodeOptions={abi.JpegQuality: 85})
    b = abi.Batch(cuda_lib, 0, 8, w, h, 256, 256, 85, max_in_bytes=sum(map(len, files)) + 4096)
    try:
        outs, status = b.transform(files)
        assert status == [0] * n
        for i, (f, o) in enumerate(zip(files, outs)):
            assert o == cuda_lib.transform(f, opt)
            if i < 2:
                dec, _ = oracle.jpeg_decode(f)
                assert o == oracle.jpeg_encode(oracle.fit(dec, 256, 256), 85)
    finally:
        b.close()


def test_batch_per_item_errors(cuda_lib, oracle):
    w, h = 160, 120
    good = _corpus(oracle, 3, w, h)
    wrong_size = oracle.jpeg_encode(synth_image(5, 96, 64, 3), 90)
    truncated = good[1][: len(good[1]) // 3]
    files = [good[0], wrong_size, b"\xff\xd8\xff garbage", truncated, good[2]]
    b = abi.Batch(cuda_lib, 0, 8, w, h, 32, 32, 85, max_in_bytes=1 << 20)
    try:
        outs, status = b.transform(files)
        assert status[0] == 0 and status[4] == 0
        assert status[1] == -10 and status[2] != 0
        assert outs[1] == b"" and outs[2] == b""
        # a truncated entropy segment decodes like libjpeg-turbo does (zeros after the end of
        # data), so it is reported as success with a full-size output
        assert status[3] in (0, -2)
        dec, _ = oracle.jpeg_decode(files[0])
        assert outs[0] == oracle.jpeg_encode(oracle.fit(dec, 32, 32), 85)
    finally:
        b.close()


def test_batch_where_no_image_is_usable(cuda_lib, oracle):
    """Every header is refused: there is no geometry to launch with (this used to divide by zero on the host --
    found by tests/native/host_batch_fake_gpu.cpp).  The context must stay usable."""
    w, h = 160, 120
    wrong_size = oracle.jpeg_encode(synth_image(5, 96, 64, 3), 90)
    files = [b"\xff\xd8\xff garbage", wrong_size, b"\x00", b"GIF89a not a jpeg"]
    b = abi.Batch(cuda_lib, 0, 8, w, h, 32, 32, 85, max_in_bytes=1 << 20)
    try:
        outs, status = b.transform(files)
        assert all(s != 0 for s in status) and all(o == b"" for o in outs)
        good = _corpus(oracle, 2, w, h)
        outs, status = b.transform(good)
        assert status == [0, 0]
        dec, _ = oracle.jpeg_decode(good[1])
        assert outs[1] == oracle.jpeg_encode(oracle.fit(dec, 32, 32), 85)
    finally:
        b.close()


def test_empty_batch(cuda_lib):
    b = abi.Batch(cuda_lib, 0, 4, 64, 64, 8, 8, 85, max_in_bytes=4096)
    try:
        outs, status = b.transform([])
        assert outs == [] and status == []
    finally:
        b.close()


@pytest.mark.parametrize("geom", [(333, 217, 64, 64), (640, 480, 100, 300), (96, 64, 96, 64),
                                  (1280, 720, 256, 256), (48, 1000, 31, 17), (1000, 48, 500, 20)])
def test_batch_roi_geometries(cuda_lib, oracle, geom):
    """The batch path decodes only the Fit crop window (+ chroma margin): odd sizes, windows that
    touch the image edges, tall / wide crops, and the same-size copy case must still equal the
    full-frame oracle result."""
    w, h, dw, dh = geom
    n = 3
    files = _corpus(oracle, n, w, h)
    b = abi.Batch(cuda_lib, 0, 4, w, h, dw, dh, 85, max_in_bytes=sum(map(len, files)) + 4096,
                  out_cap=max(65536, w * h))
    try:
        outs, status = b.transform(files)
        assert status == [0] * n
        ew, eh = oracle.expected_size(w, h, dw, dh)
        for f, o in zip(files, outs):
            dec, _ = oracle.jpeg_decode(f)
            assert o == oracle.jpeg_encode(oracle.fit(dec, ew, eh), 85)
    finally:
        b.close()


def test_batch_mixed_sampling_layouts_in_any_order(cuda_lib, oracle):
    """4:2:0, 4:2:2 and 4:4:4 files of one size in one batch, densest layout last and first: the per-chunk scratch
    layout follows the chunk's densest file, not the first file the context ever saw."""
    cv2 = pytest.importorskip("cv2")
    w, h = 320, 240
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85})
    files = []
    for k, sf in enumerate([cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
                            cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]):
        ok, b = cv2.imencode(".jpg", synth_image(900 + k, w, h, 3), [cv2.IMWRITE_JPEG_QUALITY, 90,
                                                                       cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf])
        assert ok
        files.append(bytes(b))
    b = abi.Batch(cuda_lib, 0, 8, w, h, 64, 64, 85, max_in_bytes=1 << 22, chunk=3)
    try:
        for order in (files, files[::-1], [files[2], files[0], files[2], files[1]]):
            outs, status = b.transform(order)
            assert status == [0] * len(order)
            for f, o in zip(order, outs):
                assert o == cuda_lib.transform(f, opt)
    finally:
        b.close()


def test_batch_restart_interval_streams_decode_in_parallel(cuda_lib, oracle):
    """DRI streams (one thread per restart interval) next to plain ones (self-synchronising decoder) in ONE batch:
    the kernel is chosen per image, outputs == lp_transform (which walks DRI streams with the multi-scan kernel)."""
    cv2 = pytest.importorskip("cv2")
    w, h = 480, 272
    opt = abi.ImageOptions(FileType=".jpeg", Width=96, Height=96, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85})
    files = []
    for k, rst in enumerate([0, 30, 1, 0, 7, 30, 1000]):   # 30 = one MCU row at 4:2:0; 1 = every MCU; 1000 > all MCUs
        ok, b = cv2.imencode(".jpg", synth_image(920 + k, w, h, 3), [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_RST_INTERVAL, rst])
        assert ok
        files.append(bytes(b))
    ok, b444 = cv2.imencode(".jpg", synth_image(929, w, h, 3), [cv2.IMWRITE_JPEG_QUALITY, 88, cv2.IMWRITE_JPEG_RST_INTERVAL, 5,
                                                                cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444])
    files.append(bytes(b444))
    damaged = bytearray(files[1])
    pos = damaged.find(b"\xff\xd3")
    if pos > 0:
        damaged[pos + 1] = 0xD5                                # a restart marker out of sequence
        files.append(bytes(damaged))
    b = abi.Batch(cuda_lib, 0, 16, w, h, 96, 96, 85, max_in_bytes=1 << 22, chunk=4)
    try:
        outs, status = b.transform(files)
        for i, (f, o) in enumerate(zip(files, outs)):
            try:
                want, code = cuda_lib.transform(f, opt), 0
            except abi.LilliputError as e:
                want, code = b"", e.code
            if i < 8:
                assert status[i] == 0 and code == 0 and o == want, i
            else:
                assert (status[i] != 0) or o == want              # damaged: refused by the batch, or decoded like per image
    finally:
        b.close()
