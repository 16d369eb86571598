// oracle_webp.cpp -- TEST INFRASTRUCTURE (oracle/): the WebP codec logic as a CPU library.
//
// Unlike the C restatements next to it, this oracle is NOT an independent second implementation: it
// compiles the very headers the device kernels are built from (lilliput_b200/csrc/vp8_core.h,
// vp8l_core.h, vp8_enc_core.h, vp8l_enc_core.h) for the host, with serial drivers around them.  What
// that buys: the exact decoding / encoding logic of the product can be checked bit-for-bit against
// the reference's libwebp (oracle/_ref) on a machine without a GPU, and the GPU tests then only have
// to show that the parallel schedule (warp-cooperative reconstruction, parallel bit packing ...)
// reproduces this serial run.  Pinned: tests/test_webp_core.py + tests/golden/webp_golden.npz (made
// by the reference), and in the build container a 1 496-configuration libwebp encoder sweep.
// libwebp 1.5.0 is the algorithm's home (deps/build-deps-linux.sh:235; call sites ref webp.cpp:65-112,
// 309-350); the bitstream formats are RFC 6386 (VP8) and the WebP lossless specification (VP8L).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../lilliput_b200/csrc/vp8_core.h"

extern "C" int vp8_cpu_info(const uint8_t* d, size_t n, int* w, int* h) {
    if (n < 10 || d[3] != 0x9d || d[4] != 0x01 || d[5] != 0x2a) return 1;
    *w = ((d[7] << 8) | d[6]) & 0x3fff;
    *h = ((d[9] << 8) | d[8]) & 0x3fff;
    return 0;
}

// Decodes a VP8 key-frame payload to interleaved BGR.  `stage` 0 = final, 1 = skip loop filter.
extern "C" int vp8_cpu_decode_bgr(const uint8_t* d, size_t n, uint8_t* out, int stride, int stage,
                                  uint8_t* yuv_out) {
    vp8::FrameHdr h;
    vp8::BoolDec br;
    uint8_t proba[1056];
    if (vp8::parse_frame_header(d, n, h, br, proba)) return 1;
    std::vector<uint8_t> mem(vp8::work_bytes(h.mb_w, h.mb_h));
    vp8::Work w;
    vp8::work_carve(mem.data(), h.mb_w, h.mb_h, w);
    memcpy(w.proba, proba, 1056);
    if (vp8::decode_macroblocks(d, h, br, w)) return 2;
    if (stage == 0 && h.filter_type > 0)
        for (int y = 0; y < h.mb_h; y++)
            for (int x = 0; x < h.mb_w; x++) vp8::filter_macroblock(h, w, x, y);
    const int ys = h.mb_w * 16, cs = h.mb_w * 8;
    if (yuv_out) memcpy(yuv_out, w.y, (size_t)ys * h.mb_h * 16 * 3 / 2);
    for (int y = 0; y < h.height; y++)
        for (int x = 0; x < h.width; x++) {
            const int u = vp8::upsample_at(w.u, cs, h.width, h.height, x, y);
            const int v = vp8::upsample_at(w.v, cs, h.width, h.height, x, y);
            vp8::yuv_to_bgr(w.y[(size_t)y * ys + x], u, v, out + (size_t)y * stride + 3 * x);
        }
    return 0;
}

// ---- VP8L (lossless) and ALPH, same idea ---------------------------------------------------
#include "../lilliput_b200/csrc/vp8l_core.h"

// Decodes a "VP8L" chunk payload to BGRA (channels = 4) or BGR (3).
extern "C" int vp8l_cpu_decode(const uint8_t* d, size_t n, int w, int h, uint8_t* out, int channels) {
    std::vector<uint8_t> mem((size_t)w * h * 16 + (32u << 20));
    vp8l::Arena a{mem.data(), mem.size(), 0};
    uint32_t* px = nullptr;
    const int rc = vp8l::decode_vp8l(d, n, w, h, a, &px);
    if (rc) return rc;
    for (size_t i = 0; i < (size_t)w * h; i++) {
        out[i * channels + 0] = (uint8_t)px[i];
        out[i * channels + 1] = (uint8_t)(px[i] >> 8);
        out[i * channels + 2] = (uint8_t)(px[i] >> 16);
        if (channels == 4) out[i * 4 + 3] = (uint8_t)(px[i] >> 24);
    }
    return 0;
}

// Decodes an "ALPH" chunk payload to a w*h alpha plane.
extern "C" int alph_cpu_decode(const uint8_t* d, size_t n, int w, int h, uint8_t* alpha) {
    std::vector<uint8_t> mem((size_t)w * h * 16 + (32u << 20));
    vp8l::Arena a{mem.data(), mem.size(), 0};
    return vp8l::decode_alph(d, n, w, h, a, alpha);
}

// ---- VP8L encoder core, host build: whole stream written serially (the device packs pixels in parallel)
#include "../lilliput_b200/csrc/vp8l_enc_core.h"

// channels 3/4: a "VP8L" chunk payload from a BGR(A) frame; channels 1: an ALPH chunk payload
// (header byte + headerless VP8L stream) from a plane.  Returns the size, or -1 if it does not fit.
extern "C" long vp8l_cpu_encode(const uint8_t* frame, size_t step, int w, int h, int channels, uint8_t* out, size_t cap) {
    std::vector<uint32_t> hist(4 * 256, 0);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint32_t r = vp8lenc::residual_at(frame, step, channels, x, y);
            hist[(r >> 8) & 255]++;
            hist[256 + ((r >> 16) & 255)]++;
            hist[512 + (r & 255)]++;
            hist[768 + (r >> 24)]++;
        }
    vp8lenc::BitWriter bw;
    vp8lenc::CodeTable t;
    if (channels == 1) bw.put(1, 8);  // ALPH header: lossless compression, no filter, no pre-processing
    vp8lenc::write_stream_head(bw, w, h, channels == 4, channels != 1, channels != 1, hist.data(), &t);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            uint64_t bits;
            int n;
            vp8lenc::pixel_bits(vp8lenc::residual_at(frame, step, channels, x, y), t, &bits, &n);
            bw.put((uint32_t)bits, n > 32 ? 32 : n);
            if (n > 32) bw.put((uint32_t)(bits >> 32), n - 32);
        }
    bw.flush();
    if (bw.bytes.size() > cap) return -1;
    memcpy(out, bw.bytes.data(), bw.bytes.size());
    return (long)bw.bytes.size();
}

// ---- VP8 lossy encoder core, host build
#include "../lilliput_b200/csrc/vp8_enc_core.h"

// BGR(A) frame -> "VP8 " chunk payload.  Returns the size (0 = failed).  `recon_bgr` (optional) gets
// what a decoder WITHOUT loop filter would show, for debugging.
static long vp8_cpu_encode_impl(const uint8_t* frame, size_t step, int w, int h, int channels, int quality,
                                int filter_level, int try_i4, uint8_t* out, size_t cap) {
    vp8enc::Params P;
    P.try_i4 = try_i4;
    P.width = w;
    P.height = h;
    P.mb_w = (w + 15) >> 4;
    P.mb_h = (h + 15) >> 4;
    P.q = vp8enc::quality_to_q(quality);
    P.filter_level = filter_level < 0 ? vp8enc::filter_level_for_q(P.q) : filter_level;
    const int ys = P.mb_w * 16, cs = P.mb_w * 8, yh = P.mb_h * 16, ch = P.mb_h * 8;
    std::vector<uint8_t> sy((size_t)ys * yh), su((size_t)cs * ch), sv((size_t)cs * ch);
    std::vector<uint8_t> ry(sy.size()), ru(su.size()), rv(sv.size());
    auto px = [&](int x, int y) { return frame + (size_t)(y < h ? y : h - 1) * step + (size_t)(x < w ? x : w - 1) * channels; };
    for (int y = 0; y < yh; y++)
        for (int x = 0; x < ys; x++) {
            const uint8_t* p = px(x, y);
            sy[(size_t)y * ys + x] = (uint8_t)vp8enc::rgb_to_y(p[2], p[1], p[0]);
        }
    for (int y = 0; y < ch; y++)
        for (int x = 0; x < cs; x++) {
            int r = 0, g = 0, b = 0;
            for (int dy = 0; dy < 2; dy++)
                for (int dx = 0; dx < 2; dx++) {
                    const uint8_t* p = px(2 * x + dx, 2 * y + dy);
                    b += p[0];
                    g += p[1];
                    r += p[2];
                }
            su[(size_t)y * cs + x] = (uint8_t)vp8enc::rgb_to_u(r, g, b);
            sv[(size_t)y * cs + x] = (uint8_t)vp8enc::rgb_to_v(r, g, b);
        }
    std::vector<int16_t> levels((size_t)P.mb_w * P.mb_h * 25 * 16);
    std::vector<uint8_t> modes((size_t)P.mb_w * P.mb_h * vp8enc::kModeStride);
    vp8enc::Buffers B{sy.data(), su.data(), sv.data(), ry.data(), ru.data(), rv.data(), levels.data(), modes.data()};
    vp8enc::analyse_and_reconstruct(P, B);
    // the device's scratch sizes (webp_encode_lossy_batch)
    std::vector<uint8_t> part0(vp8enc::part0_scratch_bytes(P)), tokens(vp8enc::token_scratch_bytes(P)), aux(vp8enc::kAuxBytes);
    const size_t n = vp8enc::write_bitstream(P, B, part0.data(), part0.size(), tokens.data(), tokens.size(), aux.data(), out, cap);
    return n == vp8enc::kPart0TooLarge ? -1 : (long)n;
}
// the encoder as the device runs it (vp8enc::kTryI4: whether macroblocks weigh 4x4 against 16x16 prediction; a frame
// whose first partition outgrows the format's limit coded again with 16x16 prediction only).  Returns 0 = failed.
extern "C" long vp8_cpu_encode(const uint8_t* frame, size_t step, int w, int h, int channels, int quality,
                               int filter_level, uint8_t* out, size_t cap) {
    long n = vp8_cpu_encode_impl(frame, step, w, h, channels, quality, filter_level, vp8enc::kTryI4, out, cap);
    if (n < 0 && vp8enc::kTryI4) n = vp8_cpu_encode_impl(frame, step, w, h, channels, quality, filter_level, 0, out, cap);
    return n < 0 ? 0 : n;
}
// ... and with the choice forced on or off, no retry (measurements, tests of both paths).  Returns 0 = failed, -1 = the
// first partition outgrew the format's limit.
extern "C" long vp8_cpu_encode_i4(const uint8_t* frame, size_t step, int w, int h, int channels, int quality,
                                  int filter_level, int try_i4, uint8_t* out, size_t cap) {
    return vp8_cpu_encode_impl(frame, step, w, h, channels, quality, filter_level, try_i4, out, cap);
}
// the scratch the encoder gets for a w x h frame: [0] first partition, [1] token partitions
extern "C" void vp8_cpu_scratch_bytes(int w, int h, size_t* sizes) {
    vp8enc::Params P{};
    P.width = w;
    P.height = h;
    P.mb_w = (w + 15) >> 4;
    P.mb_h = (h + 15) >> 4;
    sizes[0] = vp8enc::part0_scratch_bytes(P);
    sizes[1] = vp8enc::token_scratch_bytes(P);
}

// The exact worst case of the first partition, from the format's fixed probabilities: what the sizing constants of
// vp8_enc_core.h (kPart0HeaderBits, kPart0MbBits) must cover.  A boolean coded with probability `p` shifts the coder
// log2(range / new range) bits out, and over a partition these sum (telescoping) to at least the bits written, so a
// boolean's worst is that ratio's maximum over the ranges the coder can hold (128..255).  `header` gets the worst frame
// header, `per_mb` the worst macroblock: skip flag at any probability, the costliest luma coding (sixteen sub-block modes,
// every context chosen adversarially through the neighbours, by a walk over the four modes above the next block) and
// the costliest chroma mode.
static double bool_bits(int bit, int p) {
    double worst = 0;
    for (uint32_t r = 128; r < 256; r++) {
        const uint32_t split = 1 + (((r - 1) * (uint32_t)p) >> 8);
        const double b = std::log2((double)r / (double)(bit ? r - split : split));
        worst = b > worst ? b : worst;
    }
    return worst;
}
static double bool_bits_any(int p) { return std::fmax(bool_bits(0, p), bool_bits(1, p)); }
static double i4_mode_bits(int mode, const uint8_t* prob) {
    const uint32_t nodes = vp8enc::kVp8BModePathNodes[mode], bits = vp8enc::kVp8BModePathBits[mode];
    double b = 0;
    for (int k = 0; k < (int)(bits >> 8); k++) b += bool_bits((int)((bits >> k) & 1u), prob[(nodes >> (4 * k)) & 15u]);
    return b;
}
extern "C" void vp8_cpu_part0_worst_bits(double* header, double* per_mb) {
    const double b128 = bool_bits_any(128);
    double h = 29 * b128 + std::fmax(bool_bits(0, 128), bool_bits(1, 128) + 8 * b128);  // fixed fields, skip probability
    const uint8_t* upd = &kVp8CoeffUpdateProba[0][0][0][0];
    for (int i = 0; i < vp8enc::kNumProbas; i++) h += std::fmax(bool_bits(0, upd[i]), bool_bits(1, upd[i]) + 8 * b128);
    *header = h;
    double skip = 0;
    for (int p = 1; p < 256; p++) skip = std::fmax(skip, bool_bits_any(p));
    static double cost[10][10][10];  // [above][left][mode]
    for (int t = 0; t < 10; t++)
        for (int l = 0; l < 10; l++)
            for (int m = 0; m < 10; m++) cost[t][l][m] = i4_mode_bits(m, kVp8BModesProba[t][l]);
    // sub-blocks in raster order; the state is the mode last placed in each column (10^4 states).  Modes above the top
    // row and left of the left column belong to the neighbours: any of the ten.
    std::vector<double> best(10000, -1.0), next(10000);
    best[0] = 0;
    for (int n = 0; n < 16; n++) {
        const int bx = n & 3, by = n >> 2;
        std::fill(next.begin(), next.end(), -1.0);
        for (int s = 0; s < 10000; s++) {
            if (best[s] < 0) continue;
            int col[4] = {s % 10, s / 10 % 10, s / 100 % 10, s / 1000};
            for (int m = 0; m < 10; m++) {
                double c = 0;
                for (int t = 0; t < 10; t++)
                    for (int l = 0; l < 10; l++)
                        if ((by == 0 || t == col[bx]) && (bx == 0 || l == col[bx - 1])) c = std::fmax(c, cost[t][l][m]);
                int nc[4] = {col[0], col[1], col[2], col[3]};
                nc[bx] = m;
                const int ns = nc[0] + 10 * nc[1] + 100 * nc[2] + 1000 * nc[3];
                next[ns] = std::fmax(next[ns], best[s] + c);
            }
        }
        best.swap(next);
    }
    double i4 = 0;
    for (double b : best) i4 = std::fmax(i4, b);
    i4 += bool_bits(0, 145);
    const double i16 = bool_bits(1, 145) + std::fmax(bool_bits(1, 156) + b128, bool_bits(0, 156) + bool_bits_any(163));
    const double uv = std::fmax(bool_bits(0, 142), bool_bits(1, 142) + std::fmax(bool_bits(0, 114), bool_bits(1, 114) + bool_bits_any(183)));
    *per_mb = skip + std::fmax(i4, i16) + uv;
}

// Self-check of the data forms of the 4x4 predictors and of the sub-block mode costs (vp8_enc_core.h) against the code
// forms (vp8::pred_4x4, vp8enc::i4_mode<false>) on `iters` random borders / probability rows.  Returns mismatches.
extern "C" long vp8_cpu_check_pred4_tables(long iters, unsigned seed) {
    long bad = 0;
    uint32_t x = seed ? seed : 1u;
    auto rnd = [&]() { x ^= x << 13; x ^= x >> 17; x ^= x << 5; return x; };
    for (long it = 0; it < iters; it++) {
        uint8_t buf[6 * 32];
        for (auto& b : buf) b = (it % 3 == 0) ? (uint8_t)((rnd() & 1) * 255) : (uint8_t)rnd();
        uint8_t* d = buf + 32 + 8;  // a 4x4 block with its borders at stride 32
        uint8_t e[13];
        for (int k = 0; k < 4; k++) e[k] = d[(3 - k) * 32 - 1];
        e[4] = d[-32 - 1];
        for (int k = 0; k < 8; k++) e[5 + k] = d[-32 + k];
        const int dc = (e[5] + e[6] + e[7] + e[8] + e[0] + e[1] + e[2] + e[3] + 4) >> 3;
        uint8_t prob[9];
        for (auto& p : prob) p = (uint8_t)(1 + rnd() % 255);
        for (int m = 0; m < 10; m++) {
            vp8::pred_4x4(d, 32, m);
            for (int p = 0; p < 16; p++)
                if (vp8enc::pred4_px(m, p, e, dc) != d[(p >> 2) * 32 + (p & 3)]) bad++;
            if (vp8enc::i4_mode_cost(m, prob) != vp8enc::i4_mode<false>(nullptr, m, prob)) bad++;
        }
        if (it < 100)  // the tabulated context costs against the walk over the format's probabilities
            for (int m = 0; m < 10; m++)
                if (vp8enc::i4_mode_cost_ctx((int)(it / 10), (int)(it % 10), m) != vp8enc::i4_mode<false>(nullptr, m, kVp8BModesProba[it / 10][it % 10])) bad++;
    }
    return bad;
}
