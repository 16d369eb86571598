// The heterogeneous batch's gate table on the host: xbatch.cu's parse section (parse_item and everything it calls)
// over a list of calls, one line per (item, rendition) pair -- which pairs take the grid, and with which decoded frame,
// output size, crop, span, plan, clip and ICC profile -- and per call how many times each header parser ran.  No
// kernel runs: link with the library's other objects (not xbatch.o) and tests/native/fake_cudart.cpp
// (tests/test_xbatch_gates.py builds and runs it).
//
// Spec (argv[1], run from the directory of the files it names):
//   file <name>                                    one input file, in order
//   call files|frames|tensor <T> <max_size>        a call: lp_xbatch_transform_renditions, lp_xbatch_decode_frames
//                                                  (T = 0) / lp_xbatch_decode_clips (T slots), lp_xbatch_encode_frames
//   box <W> <H> <C>                                tensor calls: the tensor's box
//   items <i> ...                                  files / frames calls: the files, by index
//   sizes <w> <h> ...                              tensor calls: each item's frame size
//   rend <ext> <method> <w> <h> <norm> <timeout> <frames> <duration> <dao> <key> <value> ...
//                                                  one per rendition (frames and tensor calls: one)
//   run                                            parse every pair and print the table
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lilliput_host.hpp"
#include "lp_opencv.h"

// every header parser the parse section calls, counted
enum { C_JPEG, C_SCANS, C_PNG, C_CICP, C_PNG_ICC, C_JPEG_ICC, C_WEBP, C_GIF, C_GIF_HDR, C_N };
static long g_count[C_N];
static const char* const g_count_name[C_N] = {"jpeg", "scans", "png", "cicp", "png_icc", "jpeg_icc", "webp", "gif", "gif_hdr"};
template <class... A>
static int counted_jpeg_parse_header(A... a) { g_count[C_JPEG]++; return lp::jpeg_parse_header(a...); }
template <class... A>
static int counted_jpeg_parse_scans(A... a) { g_count[C_SCANS]++; return lp::jpeg_parse_scans(a...); }
template <class... A>
static int counted_png_parse(A... a) { g_count[C_PNG]++; return lp::png_parse(a...); }
template <class... A>
static int counted_png_extract_cicp(A... a) { g_count[C_CICP]++; return lp::png_extract_cicp(a...); }
template <class... A>
static int counted_png_extract_icc(A... a) { g_count[C_PNG_ICC]++; return lp::png_extract_icc(a...); }
template <class... A>
static int counted_opencv_decoder_get_jpeg_icc(A... a) { g_count[C_JPEG_ICC]++; return opencv_decoder_get_jpeg_icc(a...); }
template <class... A>
static bool counted_webp_plan_parse(A... a) { g_count[C_WEBP]++; return lp::webp_plan_parse(a...); }
template <class... A>
static lp::GifAnimPlan* counted_gif_plan_parse(A... a) { g_count[C_GIF]++; return lp::gif_plan_parse(a...); }
template <class... A>
static int counted_gif_header_frames(A... a) { g_count[C_GIF_HDR]++; return lp::gif_header_frames(a...); }
#define jpeg_parse_header counted_jpeg_parse_header
#define jpeg_parse_scans counted_jpeg_parse_scans
#define png_parse counted_png_parse
#define png_extract_cicp counted_png_extract_cicp
#define png_extract_icc counted_png_extract_icc
#define opencv_decoder_get_jpeg_icc counted_opencv_decoder_get_jpeg_icc
#define webp_plan_parse counted_webp_plan_parse
#define gif_plan_parse counted_gif_plan_parse
#define gif_header_frames counted_gif_header_frames
#include "xbatch.cu"
#undef jpeg_parse_header
#undef jpeg_parse_scans
#undef png_parse
#undef png_extract_cicp
#undef png_extract_icc
#undef opencv_decoder_get_jpeg_icc
#undef webp_plan_parse
#undef gif_plan_parse
#undef gif_header_frames

// (the library's static runtime defines it; the objects reference it)
extern "C" char __cudaInitModule(void**) { return 0; }

static std::vector<uint8_t> read_file(const std::string& p) {
    std::ifstream f(p, std::ios::binary);
    return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

static const char* kind_name(Kind k) {
    static const char* const n[] = {"fallback", "jpeg", "png", "webp", "gif", "frame"};
    return n[k];
}

static uint32_t fnv(const std::vector<uint8_t>& v) {
    uint32_t h = 2166136261u;
    for (uint8_t b : v) h = (h ^ b) * 16777619u;
    return h;
}

// one line per pair; a pair that goes per image is only its verdict
static void print_pair(const lp_xbatch& X, const std::vector<std::string>& names, int i, int r) {
    const XItem& it = X.items[(size_t)i * X.k + r];
    printf("%s r%d %s mask=%x", names[i].c_str(), r, kind_name(it.kind), X.mask[i]);
    if (it.kind == K_FALLBACK) {
        printf("\n");
        return;
    }
    printf(" src=%dx%dx%d out=%dx%d crop=%d,%d,%d,%d span=%zu", it.w, it.h, it.ch, it.ow, it.oh, it.cx, it.cy, it.cw, it.chh, it.span);
    if (it.kind == K_JPEG) printf(" sampling=%x multiscan=%d", it.jpeg_sampling, (int)it.jpeg_multiscan);
    if (it.kind == K_PNG)
        printf(" png=%dx%d hdr=%d transfer=%d primaries=%d", it.png ? it.png->width : -1, it.png ? it.png->height : -1, (int)it.hdr,
               it.transfer, it.primaries);
    if (it.kind == K_WEBP && it.webp)
        printf(" plan=%zu blend0=%d dispose0=%d animation=%d", it.webp->frames.size(), it.webp->frames[0].blend,
               it.webp->frames[0].dispose, (int)it.webp_animation);
    if (it.kind == K_GIF && it.gif) {
        int w = 0, h = 0, nf = 0;
        gif_plan_info(it.gif.get(), &w, &h, &nf, nullptr, nullptr);
        printf(" plan=%d gif_frames=%d", nf, it.gif_frames);
    }
    printf(" nframes=%d clip=", it.nframes);
    for (size_t t = 0; t < it.clip.size(); t++) printf("%s%d@%lld", t ? "," : "", it.clip[t], (long long)it.clip_ms[t]);
    printf(" icc=%zu:%08x\n", it.icc.size(), fnv(it.icc));
}

int main(int argc, char** argv) {
    if (argc != 2) {
        fprintf(stderr, "usage: %s spec\n", argv[0]);
        return 2;
    }
    std::ifstream spec(argv[1]);
    std::vector<std::string> file_names;
    std::vector<std::vector<uint8_t>> files;
    std::string mode;
    int T = 0, max_size = 0, calls = 0;
    lp_frame_tensor box{};
    std::vector<int> items, sizes;
    std::vector<std::string> exts;                 // (the options point into these)
    std::vector<std::vector<int>> enc_opts;
    std::vector<lp_image_options> opts;
    std::string line;
    while (std::getline(spec, line)) {
        std::istringstream s(line);
        std::string op;
        s >> op;
        if (op == "file") {
            std::string name;
            s >> name;
            file_names.push_back(name);
            files.push_back(read_file(name));
        } else if (op == "call") {
            s >> mode >> T >> max_size;
            items.clear();
            sizes.clear();
            exts.clear();
            enc_opts.clear();
            opts.clear();
            exts.reserve(kMaxRenditions);
            enc_opts.reserve(kMaxRenditions);
        } else if (op == "box") {
            s >> box.width >> box.height >> box.channels;
        } else if (op == "items") {
            for (int v; s >> v;) items.push_back(v);
        } else if (op == "sizes") {
            for (int v; s >> v;) sizes.push_back(v);
        } else if (op == "rend") {
            lp_image_options o{};
            long long timeout = 0, duration = 0;
            exts.emplace_back();
            s >> exts.back() >> o.resize_method >> o.width >> o.height >> o.normalize_orientation >> timeout >> o.max_encode_frames >>
                duration >> o.disable_animated_output;
            enc_opts.emplace_back();
            for (int v; s >> v;) enc_opts.back().push_back(v);
            o.file_type = exts.back().c_str();
            o.encode_timeout_ns = timeout;
            o.max_encode_duration_ns = duration;
            o.encode_options = enc_opts.back().data();
            o.encode_options_len = enc_opts.back().size();
            opts.push_back(o);
        } else if (op == "run") {
            lp_xbatch X;
            memset(&X.cfg, 0, sizeof X.cfg);
            X.cfg.max_size = max_size;
            X.k = (int)opts.size();
            for (const lp_image_options& o : opts) X.rend.push_back(mode == "frames" ? frames_rendition(o) : make_rendition(o));
            std::vector<const uint8_t*> in;
            std::vector<size_t> in_len;
            std::vector<std::string> names;
            std::vector<int> src_w, src_h;
            if (mode == "tensor") {
                for (size_t q = 0; q + 1 < sizes.size(); q += 2) {
                    src_w.push_back(sizes[q]);
                    src_h.push_back(sizes[q + 1]);
                    names.push_back("frame" + std::to_string(sizes[q]) + "x" + std::to_string(sizes[q + 1]));
                }
                X.frames = box;
                X.src_w = src_w.data();
                X.src_h = src_h.data();
            } else {
                for (int f : items) {
                    in.push_back(files[f].data());
                    in_len.push_back(files[f].size());
                    names.push_back(file_names[f]);
                }
                X.in = in.data();
                X.in_len = in_len.data();
                X.clip_t = mode == "frames" ? T : 0;
            }
            const int n = (int)names.size();
            X.items.resize((size_t)n * X.k);
            X.mask.assign((size_t)n, 0);
            memset(g_count, 0, sizeof g_count);
            for (int i = 0; i < n; i++) parse_item(&X, i);
            printf("call %d %s k=%d T=%d max_size=%d\n", calls++, mode.c_str(), X.k, T, max_size);
            for (int i = 0; i < n; i++)
                for (int r = 0; r < X.k; r++) print_pair(X, names, i, r);
            printf("parsed");
            for (int c = 0; c < C_N; c++) printf(" %s=%ld", g_count_name[c], g_count[c]);
            printf("\n");
        }
    }
    printf("done: %d calls\n", calls);
    return 0;
}
