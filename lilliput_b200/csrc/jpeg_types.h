// jpeg_types.h -- the JPEG decoder's device-format descriptors (one image, one scan, one Huffman table set).
// Plain structs with no CUDA dependency, so the shared host / device decode core (jpeg_scan_core.h) and the CPU
// suite's host build of it read the same layout the kernels do.
#pragma once
#include <stdint.h>

namespace lp {

// One scan of a multi-scan file (progressive: T.81 Annex G; or non-interleaved sequential).
struct JpegScanDesc {
    uint32_t data_off, data_len;  // entropy-coded segment, from the start of the item's file (JpegDecodeItem::scan_off)
    int32_t ns;                   // components in the scan
    int32_t ci[3], td[3], ta[3];  // frame component index, DC / AC table ids
    int32_t Ss, Se, Ah, Al;       // spectral band and successive-approximation bit positions
    int32_t restart_interval;
    int32_t table_set;            // Huffman tables in force at this scan: index into the batch's table-set array
    int32_t progressive;
};

// Device-side description of one image to decode (array of these lives in HBM).
struct JpegDecodeItem {
    uint64_t scan_off;    // offset of the entropy-coded segment in the batch scan buffer (multi-scan: of the file)
    uint32_t scan_len;    // bytes
    uint32_t table_set;   // index into the Huffman table-set array (multi-scan: first JpegScanDesc of the item,
                          // whose scans carry their own table sets)
    uint64_t coef_off;    // int16 offset of this image's coefficient blocks
    uint64_t frame_off;   // byte offset of this image's packed output frame
    int32_t width, height, ncomp;
    int32_t mcus_x, mcus_y, restart_interval;
    int32_t h[3], v[3];   // sampling factors
    int32_t dw[3], dh[3]; // true downsampled component size in samples
    // tiles of jpeg_idct_color_kernel (one CTA each): tiles_x spans of tile_mcx ROI MCU columns, bands of tile_mcy
    // ROI MCU rows
    int32_t tile_mcx, tile_mcy, tiles_x;
    uint16_t qt[3][64];     // per-component quantisation table, natural order
    int32_t td[3], ta[3];
    int32_t status;         // written by the decode kernel: 0 ok, <0 corrupt
    int32_t frame_channels; // 1 or 3
    // parallel Huffman path (jpeg_huff_parallel.cu)
    uint64_t clean_off;     // byte offset of this image's unstuffed bit string
    uint64_t state_off;     // SubState offset (2 * nsub entries reserved)
    uint64_t dcdiff_off;    // int16 offset of this image's DC-difference array (MCU order); multi-scan items:
                            // uint64 offset of their nonzero masks (jpeg_scan_core.h), the same slot layout
    uint32_t clean_len;     // written by jpeg_unstuff_kernel
    uint32_t pad_;
    // Region of interest.  Only MCUs [roi_mx0, roi_mx0+roi_mcx) x [roi_my0, roi_my0+roi_mcy) get
    // coefficients, in scan order ([roi MCU][block in MCU]); the packed frame holds
    // the pixel window [win_x0, win_x0+win_w) x [win_y0, win_y0+win_h) with rows win_stride apart.
    // A full decode has roi = every MCU and win = the whole image.
    int32_t roi_mx0, roi_my0, roi_mcx, roi_mcy;
    int32_t win_x0, win_y0, win_w, win_h;
    uint32_t win_stride;
    uint32_t nscans;        // 0: one interleaved scan.  > 0: decoded by jpeg_multiscan_kernel from its scans
                            // [table_set, table_set + nscans), which the parallel passes skip: a multi-scan file, or
                            // per image a baseline file with restart markers (one scan)
};

// Huffman decode tables for one image (or many images sharing them), device format.
constexpr int kHuffAcLookBits = 12;    // AC lookahead of the parallel decoder (jpeg_huff_parallel.cu)
constexpr int kHuffLongPrefixes = 16;  // second-level tables per AC table for codes longer than that
struct JpegHuffSet {
    // [class*4+id]: 9-bit lookahead: (len<<8)|symbol, 0 when the code is longer than 9 bits
    uint16_t look[8][512];
    int32_t maxcode[8][18];  // canonical decode for long codes; maxcode[17] = sentinel
    int32_t valoffset[8][17];
    uint8_t vals[8][256];
    // AC codes longer than kHuffAcLookBits, two-level: long_prefix[id][j] = their first kHuffAcLookBits
    // bits (0xFFFF = unused slot), long_sub[id][j][next 4 bits] = (len<<8)|symbol, 0 = not a codeword.
    // Canonical codes put every long code behind a handful of all-ones prefixes (8 for the Annex K
    // tables); prefixes that do not fit here are left to the bit-by-bit walk.
    uint16_t long_prefix[4][kHuffLongPrefixes];
    uint16_t long_sub[4][kHuffLongPrefixes][16];
};

}  // namespace lp
