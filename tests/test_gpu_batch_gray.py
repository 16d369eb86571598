"""GPU: grayscale (one-component) JPEGs in lp_batch.

Every item's status and bytes must equal lp_transform's for the same file and options (FileType .jpeg, quality,
ResizeMethod, Width / Height, NormalizeOrientation): a gray file is decoded into a 1-channel frame, oriented, resized on
one channel and written as a one-component JPEG, at its own index, next to the colour items of the same batch."""
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
GEOMS = {"fit_square": (64, 64, abi.ImageOpsFit), "fit_wide": (96, 40, abi.ImageOpsFit),
         "fit_tall": (40, 90, abi.ImageOpsFit), "resize": (80, 50, abi.ImageOpsResize)}


def with_exif_orientation(jpeg: bytes, orientation: int, big_endian: bool = False) -> bytes:
    """APP1 / EXIF with one IFD entry (0x0112 orientation, SHORT) right behind SOI, in either TIFF byte order."""
    E = ">" if big_endian else "<"
    tiff = (b"MM" if big_endian else b"II") + struct.pack(E + "HI", 42, 8) + struct.pack(E + "H", 1)
    tiff += struct.pack(E + "HHIH", 0x0112, 3, 1, orientation) + b"\x00\x00" + struct.pack(E + "I", 0)
    body = b"Exif\x00\x00" + tiff
    return jpeg[:2] + b"\xff\xe1" + (len(body) + 2).to_bytes(2, "big") + body + jpeg[2:]


def jpeg(seed, w, h, sampling="gray", q=90, orientation=None, **kw):
    """A cv2-written JPEG: one component for sampling "gray", else YCbCr at that chroma sampling."""
    flags = [cv2.IMWRITE_JPEG_QUALITY, q]
    if sampling != "gray":
        flags += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    if kw.get("progressive"):
        flags += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    if kw.get("optimize"):
        flags += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if kw.get("rst"):
        flags += [cv2.IMWRITE_JPEG_RST_INTERVAL, kw["rst"]]
    ok, b = cv2.imencode(".jpg", synth_image(seed, w, h, 1 if sampling == "gray" else 3), flags)
    assert ok
    b = bytes(b)
    return b if orientation is None else with_exif_orientation(b, orientation, big_endian=seed % 2 == 1)


def sof_components(data: bytes) -> int:
    """Nf of the frame header."""
    pos = 2
    while pos + 4 <= len(data):
        assert data[pos] == 0xFF
        m, seg = data[pos + 1], int.from_bytes(data[pos + 2:pos + 4], "big")
        if m in (0xC0, 0xC1, 0xC2):
            return data[pos + 9]
        pos += 2 + seg
    raise AssertionError("no frame header")


def with_sampling_byte(data: bytes, hv: int) -> bytes:
    """The same file with the sampling factors of its first component overwritten."""
    pos = data.find(b"\xff\xc0")
    assert pos > 0 and data[pos + 9] == 1 and data[pos + 11] == 0x11
    return data[:pos + 11] + bytes([hv]) + data[pos + 12:]


def options(dw, dh, method=abi.ImageOpsFit, normalize=False):
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


def check(lib, files, w, h, dw, dh, method=abi.ImageOpsFit, normalize=False, chunk=0, via="transform", all_ok=True):
    b = batch(lib, files, w, h, dw, dh, method, normalize, chunk)
    try:
        outs, status = run(b, files, via)
        if all_ok:
            assert status == [0] * len(files)
        assert_like_transform(lib, files, outs, status, options(dw, dh, method, normalize))
        return outs, status
    finally:
        b.close()


@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalize"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_all_gray_batch(cuda_lib, geom, normalize):
    """A batch of gray files only: every output is a one-component file of the size lp_transform gives."""
    w, h = 320, 240
    dw, dh, method = GEOMS[geom]
    files = [jpeg(100 + k, w, h) for k in range(9)]
    outs, _ = check(cuda_lib, files, w, h, dw, dh, method, normalize)
    for o in outs:
        assert sof_components(o) == 1
        assert cv2.imdecode(np.frombuffer(o, np.uint8), cv2.IMREAD_UNCHANGED).ndim == 2


@pytest.mark.parametrize("normalize", [False, True], ids=["plain", "normalize"])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_gray_and_colour_every_orientation_shuffled(cuda_lib, geom, normalize):
    """Orientations 0..9 (0 and 9 are no-ops) x 4:2:0 / 4:2:2 / 4:4:4 / gray in both EXIF byte orders, shuffled into
    one batch: results at the caller's index."""
    w, h = 320, 240
    dw, dh, method = GEOMS[geom]
    cases = [(o, s) for o in range(10) for s in ("420", "422", "444", "gray", "gray")]
    np.random.default_rng(11).shuffle(cases)
    files = [jpeg(200 + k, w, h, s, orientation=o) for k, (o, s) in enumerate(cases)]
    outs, _ = check(cuda_lib, files, w, h, dw, dh, method, normalize)
    for o, (_, s) in zip(outs, cases):
        assert sof_components(o) == (1 if s == "gray" else 3)


@pytest.mark.parametrize("via", ["transform", "stage"])
@pytest.mark.parametrize("size", [(1001, 667), (490, 331), (667, 1001), (17, 9), (8, 8), (1, 1)])
def test_odd_sizes_across_chunks(cuda_lib, size, via):
    """Sizes that are not multiples of 8 or 16, down to one pixel; chunk=4 puts gray, colour, rotated and unrotated
    items on both sides of every chunk boundary (one chunk is all gray and unrotated, one all gray and rotated)."""
    w, h = size
    kinds = ["gray", "420", "gray", "444", "gray", "gray", "gray", "gray", "422", "gray", "gray", "gray", "gray", "420",
             "gray"]
    orients = [1, 6, 3, 8, 1, 1, 1, 1, 2, 5, 6, 7, 4, 1, 8]
    files = [jpeg(300 + k, w, h, s, orientation=o) for k, (s, o) in enumerate(zip(kinds, orients))]
    for normalize in (False, True):
        for dw, dh in ((100, 70), (64, 64)):
            check(cuda_lib, files, w, h, dw, dh, normalize=normalize, chunk=4, via=via)


@pytest.mark.parametrize("via", ["transform", "stage"])
def test_two_output_sizes_in_one_batch(cuda_lib, via):
    """A Fit above the source size with Width != Height under NormalizeOrientation: the items that swap the axes get
    another output size, so a chunk with both kinds encodes up to four geometries (channels x size)."""
    w, h, dw, dh = 200, 120, 300, 150
    kinds = ["gray", "420", "gray", "gray", "444", "gray", "420", "gray", "gray"]
    orients = [1, 6, 6, 8, 1, 5, 7, 2, 1]
    files = [jpeg(500 + k, w, h, s, orientation=o) for k, (s, o) in enumerate(zip(kinds, orients))]
    for normalize in (True, False):
        outs, _ = check(cuda_lib, files, w, h, dw, dh, normalize=normalize, chunk=5, via=via)
        sizes = {cv2.imdecode(np.frombuffer(o, np.uint8), cv2.IMREAD_UNCHANGED).shape[:2] for o in outs}
        assert len(sizes) == (2 if normalize else 1), sizes


ENTROPY = {"annex_k": {}, "optimised": {"optimize": True}, "rst_1": {"rst": 1}, "rst_row": {"rst": 60}, "rst_7": {"rst": 7},
           "progressive": {"progressive": True}, "progressive_rst": {"progressive": True, "rst": 7},
           "q1": {"q": 1}, "q50": {"q": 50}, "q100": {"q": 100}, "q100_optimised": {"q": 100, "optimize": True}}


@pytest.mark.parametrize("kind", list(ENTROPY))
def test_every_entropy_path_on_one_block_mcus(cuda_lib, kind):
    """The self-synchronising decoder, the restart-interval decoder and the multi-scan decoder on 8 x 8 MCUs, in a batch
    large enough to take the parallel paths, with rotated gray and colour neighbours.  480 / 8 = 60 MCUs per row."""
    w, h = 480, 272
    files = []
    for k in range(6):
        files.append(jpeg(600 + k, w, h, orientation=(None, 6, 3, None, 8, 2)[k], **ENTROPY[kind]))
    files.insert(2, jpeg(650, w, h, "420", **ENTROPY[kind]))
    files.append(jpeg(651, w, h, "444", orientation=6))
    for normalize in (False, True):
        check(cuda_lib, files, w, h, 96, 72, normalize=normalize, chunk=5)


@pytest.mark.parametrize("size,n", [((1920, 1080), 6), ((4032, 3024), 4)])
def test_large_gray_batches(cuda_lib, size, n):
    """Full-size frames: 135 x 135 blocks inside the 1080p crop (several spans and bands of the IDCT kernel per image)."""
    w, h = size
    files = [jpeg(800 + k, w, h, orientation=(None, 6, None, 3)[k % 4], q=92) for k in range(n)]
    files.append(jpeg(850, w, h, "420", q=92))
    check(cuda_lib, files, w, h, 256, 256, normalize=True)


@pytest.mark.parametrize("hv", [0x22, 0x12, 0x21], ids=["2x2", "1x2", "2x1"])
def test_single_component_with_declared_subsampling(cuda_lib, hv):
    """A one-component scan is never interleaved: whatever factors the frame header declares for the component, an MCU is
    one 8 x 8 block.  lp_batch answers what lp_transform answers."""
    w, h = 330, 250
    plain = jpeg(900, w, h)
    files = [with_sampling_byte(plain, hv), plain, with_sampling_byte(jpeg(901, w, h, rst=3), hv),
             with_exif_orientation(with_sampling_byte(jpeg(902, w, h, optimize=True), hv), 6), jpeg(903, w, h, "420")]
    outs, status = check(cuda_lib, files, w, h, 64, 64, all_ok=False)
    assert status[1] == 0 and status[4] == 0
    if status[0] == 0:
        assert outs[0] == outs[1]  # the declared factors change nothing in the pixels


def test_damaged_gray_files(cuda_lib):
    """A damaged gray file gets the status lp_batch gives a colour file with the same damage, and lp_transform's where
    the damage is in the header; its neighbours are unaffected."""
    w, h = 320, 240

    def damages(plain, other_size):
        sos = plain.find(b"\xff\xda")
        scan = sos + 2 + int.from_bytes(plain[sos + 2:sos + 4], "big")
        flipped = bytearray(plain)
        for p in range(scan + 40, len(plain) - 2, 97):
            flipped[p] ^= 0x5A
        flipped = bytes(flipped).replace(b"\xff\xd9", b"\xff\x00")[:-2] + b"\xff\xd9"
        dht = plain.find(b"\xff\xc4")
        bad_dht = plain[:dht + 5] + b"\xff" * 16 + plain[dht + 21:]  # code-length counts that over-subscribe the code space
        return {"truncated": plain[: len(plain) // 3], "flipped": flipped, "header": plain[:sos + 6], "dht": bad_dht,
                "size": other_size}

    gray = damages(jpeg(950, w, h), jpeg(951, w + 8, h))
    colour = damages(jpeg(950, w, h, "420"), jpeg(951, w + 8, h, "420"))
    files, pairs = [], {}
    for k, name in enumerate(gray):
        files.append(jpeg(960 + k, w, h, orientation=6))
        pairs[name] = (len(files), len(files) + 1)
        files += [gray[name], colour[name], jpeg(970 + k, w, h, "444")]
    opt = options(64, 64)
    b = batch(cuda_lib, files, w, h, 64, 64, chunk=3)
    try:
        outs, status = b.transform(files)
    finally:
        b.close()
    in_pair = {i for p in pairs.values() for i in p}
    for name, (g, c) in pairs.items():
        assert status[g] == status[c], name
        if status[g] == 0:
            assert outs[g] == per_image(cuda_lib, files[g], opt)[0], name
    for name in ("header", "dht"):
        assert status[pairs[name][0]] == per_image(cuda_lib, files[pairs[name][0]], opt)[1] != 0, name
    assert status[pairs["size"][0]] == -10  # LP_ERR_BAD_ARGUMENT: not the context's size
    for i in range(len(files)):
        if i not in in_pair:
            assert status[i] == 0
            assert outs[i] == per_image(cuda_lib, files[i], opt)[0]


@pytest.mark.parametrize("dims", [(80, 60), (50, 90), (64, 64)])
def test_frames_against_the_oracle(cuda_lib, oracle, dims):
    """The device pixels, independently of the per-image path: the decoded windows of the unrotated gray items against
    the oracle's gray decode, and every resized frame against oracle decode, orientation and Fit."""
    w, h = 333, 250
    dw, dh = dims
    orients = list(range(1, 9)) + [6, 1, 1]
    kinds = ["gray"] * 9 + ["420", "gray"]
    files = [jpeg(1100 + k, w, h, s, orientation=o) for k, (s, o) in enumerate(zip(kinds, orients))]
    b = batch(cuda_lib, files, w, h, dw, dh)
    try:
        assert b.stage(files) == [0] * len(files)
        b.run()
        assert [b.item_channels(i) for i in range(len(files))] == [1 if s == "gray" else 3 for s in kinds]
        ew, eh = oracle.expected_size(w, h, dw, dh)
        resized = b.frame_slots(len(files), resized=True)
        windows = b.frame_slots(len(files), resized=False)
        assert resized.shape[1] == ew * eh * 3  # slots stay spaced for three channels
        left, top, cw, ch = oracle.fit_rect(w, h, ew, eh)
        x0, x1 = left & ~15, min((left + cw + 15) & ~15, w)
        stride = x1 - x0 if (x0, x1) == (0, w) else (x1 - x0 + 15) // 16 * 16
        for i, (f, o, s) in enumerate(zip(files, orients, kinds)):
            dec, _ = oracle.jpeg_decode(f)
            want = oracle.fit(oracle.orient(dec, o), ew, eh)
            if s == "gray":
                assert dec.ndim == 2
                got = resized[i, : ew * eh].reshape(eh, ew)
                if o == 1:
                    win = windows[i, : stride * ch].reshape(ch, stride)[:, : x1 - x0]
                    assert np.array_equal(win, dec[top:top + ch, x0:x1]), f"item {i}: decoded window"
            else:
                got = resized[i].reshape(eh, ew, 3)
            assert np.array_equal(got, want), f"item {i} orientation {o} {s}"
    finally:
        b.close()


def test_launches_per_sub_class(cuda_lib):
    """A chunk launches one resize per sub-class (channels x orientation class) present, one orientation pass per channel
    count with rotated items and one encode (two kernels) per channel count and output size.  So an all-gray chunk costs
    what an all-colour one does, and no gray item means no extra launch."""
    w, h = 320, 240
    colour = [jpeg(1200 + k, w, h, "420") for k in range(6)]
    gray = [jpeg(1210 + k, w, h) for k in range(6)]
    b = batch(cuda_lib, colour, w, h, 64, 64, n=8)
    opt = options(64, 64)
    try:
        def launches(files):
            outs, status = b.transform(files)
            assert status == [0] * len(files)
            assert_like_transform(cuda_lib, files, outs, status, opt)
            n = b.last_launches()
            b.stage(files)
            b.run()
            assert b.last_launches() == n
            return n

        base = launches(colour)
        assert launches(gray) == base                                  # the same pipeline on one channel, no image map
        assert launches(colour[:3] + gray[:1] + colour[3:]) == base + 3     # + gray resize, gray FDCT, gray entropy
        assert launches(gray[:3] + colour[:1] + gray[3:]) == base + 3
        rotated_gray = with_exif_orientation(gray[0], 6)
        assert launches(gray[:5] + [rotated_gray]) == base + 2         # + gray orientation pass, its class's resize
        assert launches(colour[:4] + gray[:1] + [rotated_gray]) == base + 3 + 2
        assert launches(colour[:3] + [with_exif_orientation(colour[0], 3)] + gray[:1] + [rotated_gray]) == base + 3 + 2 + 2
        assert launches(colour) == base
    finally:
        b.close()


def test_xbatch_still_hands_gray_to_the_per_image_path(cuda_lib):
    """lp_xbatch's routing is unchanged: a gray JPEG is a fallback item there, with lp_transform's bytes."""
    files = [jpeg(1300, 320, 240), jpeg(1301, 320, 240, "420")]
    opt = options(64, 64)
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=2 << 30)
    try:
        outs, status = xb.transform(files, opt, out_cap=1 << 18)
        st = xb.stats()
    finally:
        xb.close()
    assert status == [0, 0]
    assert outs == [per_image(cuda_lib, f, opt)[0] for f in files]
    assert st["fallback_items"] == 1 and st["grid_items"] == 1
