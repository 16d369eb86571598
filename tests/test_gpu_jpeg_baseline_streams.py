"""GPU: the baseline JPEG streams of tests/jpeg_baseline_streams.py through the three device entropy decoders.

Per image (lp_decode_host), a scan without restart markers runs on the self-synchronising parallel decoder and a DRI
scan on the multi-scan decoder, as one sequential scan; in lp_batch, DRI scans go to the restart-interval decoder
instead.  Every catalogue file must
decode to the oracle's pixels on each path, and the damaged files must be accepted or refused as written down below."""
import ctypes as C

import numpy as np
import pytest

from lilliput_b200 import abi
from tests import jpeg_baseline_streams as jb
from tests import jpeg_decode_cases as jc

pytestmark = pytest.mark.gpu
T = 10**12
STREAMS = jb.cases()
DAMAGED = jb.damaged()

# (per-image decode accepts, lp_batch accepts) for each damaged file.  Where the oracle differs, the device follows
# libjpeg-turbo: it refuses an all-ones code and a truncated scan.  The restart-interval decoder of the batch refuses
# a scan whose RSTn markers do not count 0, 1, ... 7, 0 ... in step with its intervals, where the per-image walk
# (like the oracle) takes the next marker whatever its number.
DEVICE_DAMAGED = {
    "all_ones_code": (False, False),
    "ac_run_past_63": (False, False),
    "rst_wrong_number": (True, False),
    "rst_missing": (False, False),
    "truncated": (False, False),
    "truncated_rst": (False, False),
    "no_eoi": (True, True),
    "no_eoi_rst": (True, True),
    "missing_code": (False, False),
    "missing_code_rst": (False, False),
}


def _parallel_ctas(lib) -> int:
    """CTAs of the parallel decoder that completed a decode since the last call (lp_huff_phase_clocks counter 5)."""
    f = lib.l.lp_huff_phase_clocks
    f.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    out = (C.c_ulonglong * 8)()
    assert f(out, 1) == 0
    return int(out[5])


def _dri(data: bytes) -> int:
    """The restart interval the file's DRI segment sets before its scan, 0 without one."""
    pos, ri = 2, 0
    while pos + 4 <= len(data) and data[pos] == 0xFF and data[pos + 1] != 0xDA:
        n = int.from_bytes(data[pos + 2:pos + 4], "big")
        if data[pos + 1] == 0xDD:
            ri = int.from_bytes(data[pos + 4:pos + 6], "big")
        pos += 2 + n
    return ri


def _decode(lib, data):
    try:
        return lib.decode(data)
    except abi.LilliputError:
        return None


def _oracle(oracle, data):
    try:
        return oracle.jpeg_decode(data)[0]
    except RuntimeError:
        return None


def test_per_image_catalogue_matches_oracle(cuda_lib, oracle):
    _parallel_ctas(cuda_lib)
    bad = []
    for s in STREAMS:
        assert (_dri(s.data) != 0) == (s.restart != 0), s.name
        got = _decode(cuda_lib, s.data)
        ran = _parallel_ctas(cuda_lib)
        if ran != (0 if s.restart else 1):
            bad.append(f"{s.name}: {ran} parallel decodes")
        want = oracle.jpeg_decode(s.data)[0]
        if got is None or got.shape != want.shape or not np.array_equal(got, want):
            bad.append(s.name)
    assert bad == []


def _groups():
    by = {}
    for s in STREAMS:
        w, h = map(int, s.name.rsplit("_", 1)[1].split("x"))
        by.setdefault((w, h), []).append(s)
    return sorted(by.items())


@pytest.mark.parametrize("crop", [False, True], ids=["same_size", "cropping_fit"])
def test_batch_windows_match_oracle(cuda_lib, oracle, crop):
    bad = []
    for (W, H), group in _groups():
        files = [s.data for s in group]
        n = len(files)
        dw, dh = (max(1, W // 2), H) if crop else (W, H)
        ew, eh = oracle.expected_size(W, H, dw, dh)
        box = oracle.fit_rect(W, H, ew, eh)
        b = abi.Batch(cuda_lib, 0, n, W, H, dw, dh, 85, max_in_bytes=sum(map(len, files)) + (1 << 20), chunk=n)
        try:
            status = b.stage(files)
            _parallel_ctas(cuda_lib)
            b.run()
            ran = _parallel_ctas(cuda_lib)
            slots = b.frame_slots(n, resized=False)
        finally:
            b.close()
        assert status == [0] * n, [(s.name, st) for s, st in zip(group, status) if st]
        if ran != sum(1 for s in group if not s.restart):
            bad.append(f"{W}x{H}: {ran} parallel decodes")
        for i, s in enumerate(group):
            ch = 1 if s.sampling == "gray" else 3
            win = jc.batch_window(s.sampling, W, H, box)
            got = slots[i, :win.h * win.row_stride].reshape(win.h, win.row_stride)[:, :win.w * ch]
            want = oracle.jpeg_decode(s.data)[0][win.y0:win.y0 + win.h, win.x0:win.x0 + win.w]
            if not np.array_equal(got, want.reshape(win.h, win.w * ch)):
                bad.append(s.name)
    assert bad == []


def test_xbatch_jpeg_groups_equal_lp_transform(cuda_lib):
    opt = abi.ImageOptions(FileType=".jpeg", Width=64, Height=64, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    files = [s.data for s in STREAMS]
    xb = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    try:
        outs, status = xb.transform(files, opt, out_cap=1 << 22)
        st = xb.stats()
    finally:
        xb.close()
    bad = []
    for s, out, code in zip(STREAMS, outs, status):
        try:
            want, wcode = cuda_lib.transform(s.data, opt, dst_cap=1 << 22), 0
        except abi.LilliputError as e:
            want, wcode = b"", e.code
        if (code, out) != (wcode, want) or code:
            bad.append(s.name)
    assert bad == []
    # colour files run on the grid; one-component files go to lp_transform
    assert st["grid_items"] == sum(1 for s in STREAMS if s.sampling != "gray")


@pytest.mark.parametrize("name,data,restart", DAMAGED, ids=[d[0] for d in DAMAGED])
def test_damaged_streams_on_every_path(cuda_lib, oracle, name, data, restart):
    assert _dri(data) == restart
    per_image, batch = DEVICE_DAMAGED[name]
    got = _decode(cuda_lib, data)
    assert (got is not None) == per_image
    want = _oracle(oracle, data)
    if got is not None and want is not None:
        assert np.array_equal(got, want)
    opt = abi.ImageOptions(FileType=".jpeg", Width=32, Height=32, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85}, EncodeTimeout_ns=T)
    W, H = cuda_lib.header(data)[:2]
    b = abi.Batch(cuda_lib, 0, 1, W, H, 32, 32, 85, max_in_bytes=len(data) + (1 << 20))
    try:
        outs, status = b.transform([data])
    finally:
        b.close()
    assert (status[0] == 0) == batch
    if batch and per_image:
        assert outs[0] == cuda_lib.transform(data, opt, dst_cap=1 << 22)
