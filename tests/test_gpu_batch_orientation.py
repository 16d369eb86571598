"""GPU: EXIF-rotated and mirrored JPEGs in lp_batch.

Every item's status and bytes must equal lp_transform's for the same file and options (FileType .jpeg, quality,
ResizeMethod, Width / Height, NormalizeOrientation): the orientation is applied to every frame whether or not
NormalizeOrientation is set, the expected size comes from the header's size (turned only under NormalizeOrientation),
and Fit crops the oriented frame.  Items whose orientation swaps the axes can get another output size than the others
of the same batch; they must still come back at their own index."""
import struct

import numpy as np
import pytest

from lilliput_b200 import abi
from lilliput_b200.synth import synth_image

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")
SAMPLING = {"420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444}
Q = 85


def with_exif_orientation(jpeg: bytes, orientation: int, big_endian: bool = False) -> bytes:
    """APP1 / EXIF with one IFD entry (0x0112 orientation, SHORT) right behind SOI, in either TIFF byte order."""
    E = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(E + "HI", 42, 8) + struct.pack(E + "H", 1)
    tiff += struct.pack(E + "HHIH", 0x0112, 3, 1, orientation) + b"\x00\x00" + struct.pack(E + "I", 0)
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + jpeg[2:]


def jpeg(seed, w, h, sampling="420", q=90, **kw):
    flags = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    if kw.get("progressive"):
        flags += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    if kw.get("optimize"):
        flags += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if kw.get("rst"):
        flags += [cv2.IMWRITE_JPEG_RST_INTERVAL, kw["rst"]]
    ok, b = cv2.imencode(".jpg", synth_image(seed, w, h, 3), flags)
    assert ok
    return bytes(b)


def tagged(seed, w, h, orientation, **kw):
    return with_exif_orientation(jpeg(seed, w, h, **kw), orientation, big_endian=seed % 2 == 1)


def options(dw, dh, method, normalize):
    return abi.ImageOptions(FileType=".jpeg", Width=dw, Height=dh, ResizeMethod=method, NormalizeOrientation=normalize,
                            EncodeOptions={abi.JpegQuality: Q})


def per_image(lib, data, opt):
    try:
        return lib.transform(data, opt, dst_cap=1 << 22), 0
    except abi.LilliputError as e:
        return b"", e.code


def batch(lib, files, w, h, dw, dh, method=abi.ImageOpsFit, normalize=False, chunk=0, n=None):
    return abi.Batch(lib, 0, n or len(files), w, h, dw, dh, Q, max_in_bytes=sum(map(len, files)) + (1 << 20),
                     out_cap=1 << 18, resize_method=method, chunk=chunk, normalize_orientation=normalize)


def run(b, files, via):
    if via == "transform":
        return b.transform(files)
    b.stage(files)
    b.run()
    return b.fetch(len(files))


def assert_like_transform(lib, files, outs, status, opt):
    for i, f in enumerate(files):
        want, code = per_image(lib, f, opt)
        assert (status[i], outs[i]) == (code, want), f"item {i}: status {status[i]}, lp_transform {code}"


GEOMS = {"fit_square": (64, 64, abi.ImageOpsFit), "fit_wide": (96, 40, abi.ImageOpsFit),
         "fit_tall": (40, 90, abi.ImageOpsFit), "resize": (80, 50, abi.ImageOpsResize)}


@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalize"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_every_orientation_and_sampling_shuffled(cuda_lib, geom, normalize):
    """Orientations 0..9 (0 and 9 are no-ops) x 4:2:0 / 4:2:2 / 4:4:4, shuffled into one batch."""
    w, h = 320, 240
    dw, dh, method = GEOMS[geom]
    cases = [(o, s) for o in range(10) for s in SAMPLING]
    np.random.default_rng(7).shuffle(cases)
    files = [tagged(100 + k, w, h, o, sampling=s) for k, (o, s) in enumerate(cases)]
    b = batch(cuda_lib, files, w, h, dw, dh, method, normalize)
    try:
        outs, status = b.transform(files)
        assert status == [0] * len(files)
        assert_like_transform(cuda_lib, files, outs, status, options(dw, dh, method, normalize))
    finally:
        b.close()


@pytest.mark.parametrize("via", ["transform", "stage"])
@pytest.mark.parametrize("size", [(1001, 667), (490, 331), (667, 1001)])
def test_odd_sizes_across_chunks(cuda_lib, size, via):
    """Odd sizes and widths that are not multiples of 16: the crop's truncation is not symmetric under mirroring and the
    window's 16-pixel alignment falls differently on each side.  chunk=4 puts rotated and unrotated items on both sides
    of every chunk boundary, through the pipelined call and through stage / run / fetch."""
    w, h = size
    orients = [1, 6, 3, 8, 2, 1, 1, 5, 7, 4, 6, 1, 8]
    files = [tagged(300 + k, w, h, o, sampling=("420", "422", "444")[k % 3]) for k, o in enumerate(orients)]
    for normalize in (False, True):
        for dw, dh in ((100, 70), (64, 64)):
            b = batch(cuda_lib, files, w, h, dw, dh, normalize=normalize, chunk=4)
            try:
                outs, status = run(b, files, via)
                assert status == [0] * len(files)
                assert_like_transform(cuda_lib, files, outs, status, options(dw, dh, abi.ImageOpsFit, normalize))
            finally:
                b.close()


@pytest.mark.parametrize("via", ["transform", "stage"])
def test_two_output_sizes_in_one_batch(cuda_lib, via):
    """A Fit above the source size with Width != Height: under NormalizeOrientation the items that swap the axes get
    another output size (calculateExpectedSize takes another branch), so a chunk encodes two geometries."""
    w, h, dw, dh = 200, 120, 300, 150
    orients = [1, 6, 1, 8, 3, 5, 1, 2, 7]
    files = [tagged(500 + k, w, h, o) for k, o in enumerate(orients)]
    for normalize in (True, False):
        b = batch(cuda_lib, files, w, h, dw, dh, normalize=normalize, chunk=4)
        try:
            outs, status = run(b, files, via)
            assert status == [0] * len(files)
            opt = options(dw, dh, abi.ImageOpsFit, normalize)
            assert_like_transform(cuda_lib, files, outs, status, opt)
            sizes = {cv2.imdecode(np.frombuffer(o, np.uint8), cv2.IMREAD_COLOR).shape[:2] for o in outs}
            assert len(sizes) == (2 if normalize else 1), sizes
        finally:
            b.close()


def test_multiscan_restart_and_optimised_sources(cuda_lib):
    """Orientation comes after the IDCT: progressive, restart-interval and optimised-table files take the same path."""
    w, h = 480, 272
    files = []
    for k, o in enumerate([3, 6, 8]):
        files += [tagged(700 + 3 * k, w, h, o, progressive=True), tagged(701 + 3 * k, w, h, o, rst=5),
                  tagged(702 + 3 * k, w, h, o, optimize=True, sampling="444")]
    files += [jpeg(720, w, h, progressive=True), jpeg(721, w, h, rst=3)]
    for normalize in (False, True):
        b = batch(cuda_lib, files, w, h, 96, 72, normalize=normalize, chunk=5)
        try:
            outs, status = b.transform(files)
            assert status == [0] * len(files)
            assert_like_transform(cuda_lib, files, outs, status, options(96, 72, abi.ImageOpsFit, normalize))
        finally:
            b.close()


def test_camera_size_batch(cuda_lib):
    """4032 x 3024 4:2:0, tagged 1 / 6 / 8 / 3 as phone cameras tag them."""
    w, h = 4032, 3024
    files = [tagged(800 + k, w, h, o, q=92) for k, o in enumerate([1, 6, 8, 3, 6, 1, 8])]
    b = batch(cuda_lib, files, w, h, 256, 256, normalize=True)
    try:
        outs, status = b.transform(files)
        assert status == [0] * len(files)
        assert_like_transform(cuda_lib, files, outs, status, options(256, 256, abi.ImageOpsFit, True))
    finally:
        b.close()


@pytest.mark.parametrize("dims", [(80, 60), (50, 90), (64, 64)])
def test_resized_frames_against_the_oracle(cuda_lib, oracle, dims):
    """The device pixels, independently of the per-image path: oracle decode, oracle orientation, oracle Fit."""
    w, h = 333, 250
    dw, dh = dims
    orients = list(range(1, 9)) + [6, 1]
    files = [tagged(900 + k, w, h, o) for k, o in enumerate(orients)]
    b = batch(cuda_lib, files, w, h, dw, dh)
    try:
        assert b.stage(files) == [0] * len(files)
        b.run()
        got = b.resized_frames(len(files), *oracle.expected_size(w, h, dw, dh))
        for i, (f, o) in enumerate(zip(files, orients)):
            dec, _ = oracle.jpeg_decode(f)
            ew, eh = oracle.expected_size(w, h, dw, dh)
            assert np.array_equal(got[i], oracle.fit(oracle.orient(dec, o), ew, eh)), f"item {i} orientation {o}"
    finally:
        b.close()


def test_damaged_rotated_files(cuda_lib):
    """A damaged rotated file gets the status lp_batch gives an unrotated file with the same damage; its neighbours are
    unaffected."""
    w, h = 320, 240
    plain = jpeg(950, w, h)
    sos = plain.find(b"\xff\xda")
    scan = sos + 2 + int.from_bytes(plain[sos + 2:sos + 4], "big")
    flipped = bytearray(plain)
    for p in range(scan + 40, len(plain) - 2, 97):
        flipped[p] ^= 0x5A
    flipped = bytes(flipped).replace(b"\xff\xd9", b"\xff\x00")[:-2] + b"\xff\xd9"
    damages = {"truncated": plain[: len(plain) // 3], "flipped": flipped, "header": plain[:sos + 6]}
    files, pairs = [], []
    for k, (name, bad) in enumerate(damages.items()):
        files.append(tagged(960 + k, w, h, 6))
        pairs.append((len(files), len(files) + 1))
        files += [with_exif_orientation(bad, (6, 3, 8)[k]), bad, tagged(970 + k, w, h, 8)]
    b = batch(cuda_lib, files, w, h, 64, 64, chunk=3)
    try:
        outs, status = b.transform(files)
        opt = options(64, 64, abi.ImageOpsFit, False)
        for rotated, unrotated in pairs:
            assert status[rotated] == status[unrotated]
        for i in range(len(files)):
            if any(i in p for p in pairs):
                continue
            assert status[i] == 0
            assert outs[i] == per_image(cuda_lib, files[i], opt)[0]
    finally:
        b.close()


def test_all_top_left_batch_launches_as_before(cuda_lib, oracle):
    """A batch with no rotated item: the launches, decoded-window stride and resized stride of a context that takes
    rotated files are those the geometry alone gives, with normalize_orientation 0 and 1; one rotated item adds exactly
    the orientation launch and its class's resize."""
    w, h = 320, 240
    files = [jpeg(1000 + k, w, h) for k in range(5)] + [tagged(1010, w, h, 1), tagged(1011, w, h, 0)]
    rotated = files[:3] + [tagged(1012, w, h, 6)] + files[3:]
    launches = []
    for normalize in (False, True):
        b = batch(cuda_lib, rotated, w, h, 64, 64, normalize=normalize)
        try:
            outs, status = b.transform(files)
            assert status == [0] * len(files)
            n = b.last_launches()
            launches.append(n)
            b.stage(files)
            b.run()
            assert b.last_launches() == n
            # Fit 64x64 of 320x240: crop x 40..280, window x aligned out to 32..288 -> 256 px x 3 B rows
            win = b.decoded_windows(len(files), 240)
            assert win.shape == (len(files), 240, 256 * 3)
            assert b.resized_frames(len(files), 64, 64).shape == (len(files), 64, 64, 3)
            dec, _ = oracle.jpeg_decode(files[0])
            assert np.array_equal(win[0].reshape(240, 256, 3), dec[:, 32:288])
            outs2, status2 = b.transform(rotated)
            assert status2 == [0] * len(rotated)
            assert b.last_launches() == n + 2
        finally:
            b.close()
    assert launches[0] == launches[1]
