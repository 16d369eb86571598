"""GPU: the hand-built VP8L / ALPH catalogue (tests/vp8l_streams.py) and its damaged and truncated streams through the
device decoder, per image (webp_decoder_*) and in the heterogeneous batch (lp_xbatch_transform): status as libwebp,
pixels as libwebp and as the host build of the same cores."""
import numpy as np
import pytest

from lilliput_b200 import abi
from tests import vp8l_streams as vs
from tests.test_gpu_xbatch import check_against_per_image
from tests.test_webp_lossless_streams import core_decode, libwebp
from tests.webp_util import vp8_cpu_lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    return vp8_cpu_lib()


def _device(cuda_lib, data):
    info, frames, _, rc = cuda_lib.webp_frames(data)
    return rc, (frames[0] if rc == 0 and frames else None)


def test_catalogue_on_the_device(cuda_lib, lib):
    bad = []
    for case in vs.cases():
        want = libwebp(case.data)
        rc, got = _device(cuda_lib, case.data)
        crc, host = core_decode(lib, case.data)
        if rc != 0 or got is None:
            bad.append(f"{case.name}: device rc {rc}")
            continue
        got = got[:, :, :want.shape[2]] if got.shape[2] > want.shape[2] else got
        if got.shape != want.shape or not np.array_equal(got, want):
            bad.append(f"{case.name}: pixels differ from libwebp")
        elif crc != 0 or not np.array_equal(got, host[:, :, :got.shape[2]]):
            bad.append(f"{case.name}: pixels differ from the host cores")
    assert not bad, bad[:20]


def test_damaged_streams_on_the_device(cuda_lib, lib):
    bad = []
    for d in vs.damaged_cases():
        lw = libwebp(d.data)
        rc, got = _device(cuda_lib, d.data)
        if (lw is not None) != (rc == 0):
            bad.append(f"{d.name}: libwebp {'accepts' if lw is not None else 'refuses'}, device rc {rc}")
        elif lw is not None:
            crc, host = core_decode(lib, d.data)
            if crc != 0 or not np.array_equal(got[:, :, :host.shape[2]], host):
                bad.append(f"{d.name}: device pixels differ from the host cores")
    assert not bad, bad[:20]


@pytest.fixture(scope="module")
def xb(cuda_lib):
    x = abi.XBatch(cuda_lib, 0, arena_bytes=4 << 30)
    yield x
    x.close()


def test_truncated_lossy_refused_in_the_batch_as_per_image(cuda_lib, xb):
    """The batch decodes simple lossy stills in one grid launch (webp_vp8_decode_batch): a truncated one must come
    back refused exactly as per image, next to well-formed lossy + ALPH files that take the per-image path."""
    files = [c.data for c in vs.cases() if c.kind == "alph_still"]
    trunc = [d for d in vs.damaged_cases() if d.group in ("trunc_vp8", "trunc_vp8_partitions")]
    files += [d.data for d in trunc[::7]]
    refused = sum(libwebp(f) is None for f in files)
    assert refused > 10
    opt = abi.ImageOptions(FileType=".jpeg", Width=32, Height=32, ResizeMethod=abi.ImageOpsFit,
                           EncodeOptions={abi.JpegQuality: 85})
    _, status = check_against_per_image(cuda_lib, xb, files, opt)
    for f, s in zip(files, status):
        assert (s == 0) == (libwebp(f) is not None)
