// Host build of lilliput_b200/csrc/jpeg_scan_core.h (multi-scan JPEG entropy decoding) for the CPU suite.  It runs
// exactly the per-image walk jpeg_multiscan_kernel runs on the device, for a region of interest given in MCUs: the
// ROI's coefficient blocks in scan order ([roi MCU][block in MCU]) and, outside the ROI, the nonzero masks.
// tests/test_jpeg_scan_streams.py compares a windowed decode with the whole-frame decode cut to the window.
#include <cstring>
#include <vector>

#define LP_JSC_HOST
#include "../../lilliput_b200/csrc/jpeg_scan_core.h"
#include "../../lilliput_b200/csrc/kernels.cuh"

static const uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// info[0..3] = mcus_x, mcus_y, blocks per MCU, block visits.  roi = (mx0, my0, mcx, mcy) in MCUs; mcx = 0: the whole
// frame.  out: roi blocks * 64 int16.  Returns the decoder's status (0, -3), or a negative lp_status from parsing,
// or 1 when `cap` is too small.
extern "C" int jscan_decode(const uint8_t* file, long len, const int* roi, int16_t* out, long cap, int* info) {
    lp::JpegHeader h;
    int rc = lp::jpeg_parse_header(file, (size_t)len, &h);
    if (rc) return rc;
    if (!h.multiscan) return -8;
    std::vector<lp::JpegScanDesc> scans(lp::kMultiscanMaxScans);
    std::vector<lp::JpegHuffSet> sets(lp::kMultiscanMaxSets);
    int nscans = 0, nsets = 0;
    rc = lp::jpeg_parse_scans(file, (size_t)len, h, scans.data(), (int)scans.size(), &nscans, sets.data(), (int)sets.size(),
                              &nsets);
    if (rc) return rc;
    lp::JpegDecodeItem it;
    memset(&it, 0, sizeof(it));
    it.width = h.width;
    it.height = h.height;
    it.ncomp = h.ncomp;
    it.mcus_x = h.mcus_x;
    it.mcus_y = h.mcus_y;
    for (int c = 0; c < h.ncomp; c++) {
        it.h[c] = h.comp[c].h;
        it.v[c] = h.comp[c].v;
        it.dw[c] = (h.width * h.comp[c].h + h.maxh - 1) / h.maxh;
        it.dh[c] = (h.height * h.comp[c].v + h.maxv - 1) / h.maxv;
    }
    it.roi_mx0 = roi[2] ? roi[0] : 0;
    it.roi_my0 = roi[2] ? roi[1] : 0;
    it.roi_mcx = roi[2] ? roi[2] : h.mcus_x;
    it.roi_mcy = roi[2] ? roi[3] : h.mcus_y;
    it.nscans = (uint32_t)nscans;
    const lp::ScanOrder so = lp::scan_order(it);
    info[0] = h.mcus_x;
    info[1] = h.mcus_y;
    info[2] = so.nb;
    info[3] = (int)lp::jpeg_multiscan_visits(h, scans.data(), nscans);
    const size_t blocks = lp::roi_blocks(it, so);
    if ((long)(blocks * 64) > cap) return 1;
    memset(out, 0, blocks * 64 * sizeof(int16_t));
    std::vector<uint64_t> masks(so.total, 0);
    return lp::multiscan_decode(it, scans.data(), sets.data(), file, out, lp::roi_is_frame(it) ? nullptr : masks.data(),
                                kZigzag);
}
