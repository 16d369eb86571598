// lilliput_host.cpp -- C++ mirror of lilliput's Go policy layer (see header).
// Every function cites the Go it follows.  No pixel arithmetic happens here:
// all of it is behind the per-image C ABI (lp_opencv.h).
#include "lilliput_host.hpp"

#include <new>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>

namespace lilliput {

// ---------------------------------------------------------------- Framebuffer

Framebuffer::Framebuffer(int w, int h) : buf((size_t)w * (size_t)h * 4) {}

Framebuffer::~Framebuffer() { Close(); }

void Framebuffer::Close() {
    if (mat) {
        opencv_mat_release(mat);
        mat = nullptr;
    }
}

// ref opencv.go:223-228: memset the Go slice, then reset the mat.
void Framebuffer::Clear() {
    if (!buf.empty()) memset(buf.data(), 0, buf.size());
    if (mat) opencv_mat_reset(mat);
}

Error Framebuffer::Create3Channel(int w, int h) {
    Error e = resizeMat(w, h, PixelType{CV_8UC3});
    if (e) return e;
    Clear();
    return LP_OK;
}

Error Framebuffer::Create4Channel(int w, int h) {
    Error e = resizeMat(w, h, PixelType{CV_8UC4});
    if (e) return e;
    Clear();
    return LP_OK;
}

// ref opencv.go:250-267: release the old mat, coerce depth > 8 to 8U keeping
// the channel count, wrap buf; NULL from the C side means ErrBufTooSmall.
Error Framebuffer::resizeMat(int w, int h, PixelType t) {
    if (mat) {
        opencv_mat_release(mat);
        mat = nullptr;
    }
    if (t.Depth() > 8) t.v = opencv_type_convert_depth(t.v, CV_8U);
    opencv_mat m = opencv_mat_create_from_data(w, h, t.v, buf.data(), buf.size());
    if (!m) return LP_ERR_BUF_TOO_SMALL;
    mat = m;
    width = w;
    height = h;
    pixelType = t;
    return LP_OK;
}

// ref opencv.go:271-279: dims are re-read from the mat afterwards (SURVEY
// Appendix C quirk 7 depends on this refresh).
void Framebuffer::TonemapToSDR(int transfer, int primaries) {  // ref opencv.go:791-810
    if (!mat || Width() <= 0 || Height() <= 0) return;
    lp_mat_tonemap_to_sdr(mat, transfer, primaries);
}

void Framebuffer::OrientationTransform(int orientation) {
    if (!mat) return;
    opencv_mat_orientation_transform((CVImageOrientation)orientation, mat);
    width = opencv_mat_get_width(mat);
    height = opencv_mat_get_height(mat);
}

// ref opencv.go:294-309
Error Framebuffer::ResizeTo(int w, int h, Framebuffer* dst) {
    if (w < 1) w = 1;
    if (h < 1) h = 1;
    Error e = dst->resizeMat(w, h, pixelType);
    if (e) return e;
    opencv_mat_resize(mat, dst->mat, w, h, CV_INTER_AREA);
    return LP_OK;
}

static Error handleOpenCVError(int rc) {  // ref opencv.go:399-426
    return rc == OPENCV_SUCCESS ? LP_OK : (LP_ERR_OPENCV - rc);
}

// ref opencv.go:312-319
Error Framebuffer::ClearToTransparent(int x, int y, int w, int h) {
    if (!mat) return LP_ERR_FRAMEBUF_NO_PIXELS;
    return handleOpenCVError(opencv_mat_clear_to_transparent(mat, x, y, w, h));
}

// ref opencv.go:331-363.  float64 arithmetic, int() truncation as in Go.
void fitCropRect(int srcW, int srcH, int dstW, int dstH, int* left, int* top, int* wc, int* hc) {
    double aspectIn = (double)srcW / (double)srcH;
    double aspectOut = (double)dstW / (double)dstH;
    int widthPostCrop, heightPostCrop;
    if (aspectIn > aspectOut) {
        widthPostCrop = (int)((aspectOut * (double)srcH) + 0.5);
        heightPostCrop = srcH;
    } else {
        heightPostCrop = (int)(((double)srcW / aspectOut) + 0.5);
        widthPostCrop = srcW;
    }
    if (widthPostCrop < 1) widthPostCrop = 1;
    if (heightPostCrop < 1) heightPostCrop = 1;
    int l = (int)((double)(srcW - widthPostCrop) * 0.5);
    if (l < 0) l = 0;
    int t = (int)((double)(srcH - heightPostCrop) * 0.5);
    if (t < 0) t = 0;
    *left = l;
    *top = t;
    *wc = widthPostCrop;
    *hc = heightPostCrop;
}

// ref opencv.go:326-374
Error Framebuffer::Fit(int w, int h, Framebuffer* dst) {
    if (!mat) return LP_ERR_FRAMEBUF_NO_PIXELS;
    int left, top, wc, hc;
    fitCropRect(width, height, w, h, &left, &top, &wc, &hc);
    opencv_mat view = opencv_mat_crop(mat, left, top, wc, hc);
    if (!view) return LP_ERR_BAD_ARGUMENT;  // (cannot happen for a rectangle fitCropRect made; the CUDA ABI refuses others)
    Error e = dst->resizeMat(w, h, pixelType);
    if (e) {
        opencv_mat_release(view);
        return e;
    }
    opencv_mat_resize(view, dst->mat, w, h, CV_INTER_AREA);
    opencv_mat_release(view);
    return LP_OK;
}

Error Framebuffer::CopyToOffsetWithAlphaBlending(Framebuffer* src, int x, int y, int w, int h) {
    return handleOpenCVError(opencv_copy_to_region_with_alpha(src->mat, mat, x, y, w, h));
}

Error Framebuffer::CopyToOffsetNoBlend(Framebuffer* src, int x, int y, int w, int h) {
    return handleOpenCVError(opencv_copy_to_region(src->mat, mat, x, y, w, h));
}

// ------------------------------------------------ container sniffers (host)

static inline uint32_t be32(const uint8_t* p) {
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
static const uint8_t kPngMagic[8] = {0x89, 0x50, 0x4e, 0x47, 0x0d, 0x0a, 0x1a, 0x0a};

// Walks PNG chunks the way pngChunkIter does (ref opencv.go:467-511): a chunk
// is visited when its 12 framing bytes fit, even if its body is truncated.
template <class F>
static void walkPngChunks(const uint8_t* png, size_t len, F&& visit) {
    if (len < 8 || memcmp(png, kPngMagic, 8) != 0) return;
    size_t off = 8;
    while (off + 12 <= len) {
        size_t next = off + (size_t)be32(png + off) + 12;
        if (!visit(png + off + 4, next)) return;
        off = next;
    }
}

bool detectAPNG(const uint8_t* img, size_t len) {  // ref opencv.go:623-637
    bool found = false;
    walkPngChunks(img, len, [&](const uint8_t* type, size_t) {
        if (!memcmp(type, "acTL", 4) || !memcmp(type, "fcTL", 4) || !memcmp(type, "fdAT", 4)) {
            found = true;
            return false;
        }
        return true;
    });
    return found;
}

static int detectContentLengthPNG(const uint8_t* png, size_t len) {  // ref opencv.go:513-531
    int result = (int)len;
    walkPngChunks(png, len, [&](const uint8_t* type, size_t next) {
        if (!memcmp(type, "IEND", 4)) {
            result = (int)std::min(next, len);
            return false;
        }
        return true;
    });
    return result;
}

// ref opencv.go:533-609: walk marker segments; inside entropy-coded data skip
// to the first 0xFF that is followed by neither 0x00, 0xFF nor RSTn.
static int detectContentLengthJPEG(const uint8_t* j, size_t len) {
    if (len < 3 || j[0] != 0xFF || j[1] != 0xD8 || j[2] != 0xFF) return (int)len;
    size_t idx = 0;
    while (idx + 1 < len && j[idx] == 0xFF) {
        uint8_t seg = j[idx + 1];
        size_t next = idx + 2;
        if (seg == 0xD9) return (int)next;
        if (seg == 0xFF) {
            idx++;
            continue;
        }
        bool unsized = seg == 0x01 || seg == 0xD8 || (seg >= 0xD0 && seg <= 0xD7);
        if (unsized) {
            idx = next;
            continue;
        }
        if (idx + 3 >= len) break;
        next += ((size_t)j[idx + 2] << 8) | j[idx + 3];
        if (seg == 0xDA) {
            for (; next < len; next++) {
                if (j[next] != 0xFF) continue;
                if (next + 1 >= len) {
                    next = len;
                    break;
                }
                uint8_t peek = j[next + 1];
                if (peek == 0xFF) continue;
                if (peek != 0 && (peek < 0xD0 || peek > 0xD7)) break;
            }
        }
        idx = next;
    }
    return (int)len;
}

int detectContentLength(const uint8_t* img, size_t len) {  // ref opencv.go:611-620
    return std::min(detectContentLengthJPEG(img, len), detectContentLengthPNG(img, len));
}

bool pngChunkTypes(const uint8_t* img, size_t len, std::vector<std::array<uint8_t, 4>>* types) {
    types->clear();
    if (len < 8 || memcmp(img, kPngMagic, 8) != 0) return false;  // makePngChunkIter's error
    walkPngChunks(img, len, [&](const uint8_t* type, size_t) {
        types->push_back({type[0], type[1], type[2], type[3]});
        return true;
    });
    return true;
}

// ------------------------------------------------------------ OpenCV adapter

class OpenCVDecoder : public Decoder {  // ref opencv.go:131-137, 442-463
  public:
    static Error Create(const uint8_t* buf, size_t len, std::unique_ptr<Decoder>* out) {
        opencv_mat m = opencv_mat_create_from_data((int)len, 1, CV_8U, (void*)buf, len);
        if (!m) return LP_ERR_BUF_TOO_SMALL;
        opencv_decoder d = opencv_decoder_create(m);
        if (!d) {
            opencv_mat_release(m);
            return LP_ERR_INVALID_IMAGE;
        }
        auto* self = new OpenCVDecoder;
        self->mat = m;
        self->decoder = d;
        self->buf = buf;
        self->len = len;
        out->reset(self);
        return LP_OK;
    }
    ~OpenCVDecoder() override {
        opencv_decoder_release(decoder);
        opencv_mat_release(mat);
    }
    Error Header(ImageHeader* h) override {  // ref opencv.go:639-661
        if (!hasReadHeader && !opencv_decoder_read_header(decoder)) return LP_ERR_INVALID_IMAGE;
        hasReadHeader = true;
        h->width = opencv_decoder_get_width(decoder);
        h->height = opencv_decoder_get_height(decoder);
        h->pixelType.v = opencv_decoder_get_pixel_type(decoder);
        h->orientation = opencv_decoder_get_orientation(decoder);
        h->numFrames = detectAPNG(buf, len) ? 2 : 1;
        h->contentLength = detectContentLength(buf, len);
        return LP_OK;
    }
    std::string Description() override {
        const char* s = opencv_decoder_get_description(decoder);
        return s ? s : "";
    }
    Error DecodeTo(Framebuffer* f) override {  // ref opencv.go:816-839
        if (hasDecoded) return LP_ERR_EOF;
        ImageHeader h;
        Error e = Header(&h);
        if (e) return e;
        e = f->resizeMat(h.width, h.height, h.pixelType);
        if (e) return e;
        if (!opencv_decoder_read_data(decoder, f->mat)) return LP_ERR_DECODING_FAILED;
        hasDecoded = true;
        f->blend = NoBlend;
        f->dispose = DisposeToBackgroundColor;
        f->xOffset = 0;
        f->yOffset = 0;
        f->duration_ns = 0;
        return LP_OK;
    }
    Error SkipFrame() override { return LP_ERR_SKIP_NOT_SUPPORTED; }  // ref opencv.go:841-843
    std::vector<uint8_t> ICC() override {  // ref opencv.go:691-728
        std::vector<uint8_t> icc(32768);  // ICCProfileBufferSize, ref lilliput.go:15
        std::string d = Description();
        int n = 0;
        if (d == "JPEG")
            n = opencv_decoder_get_jpeg_icc((void*)buf, len, icc.data(), icc.size());
        else if (d == "PNG")
            n = opencv_decoder_get_png_icc((void*)buf, len, icc.data(), icc.size());
        icc.resize(n > 0 ? n : 0);
        return icc;
    }
    bool CICP(::lilliput::CICP* out) override {  // ref opencv.go:745-768
        if (Description() != "PNG" || len == 0) return false;
        uint8_t primaries = 0, transfer = 0, matrix = 0, fullRange = 0;
        if (!opencv_decoder_get_png_cicp((void*)buf, len, &primaries, &transfer, &matrix, &fullRange)) return false;
        out->Primaries = primaries;
        out->Transfer = transfer;
        out->Matrix = matrix;
        out->FullRange = fullRange != 0;
        return true;
    }

  private:
    opencv_mat mat = nullptr;
    opencv_decoder decoder = nullptr;
    const uint8_t* buf = nullptr;
    size_t len = 0;
    bool hasReadHeader = false, hasDecoded = false;
};

class OpenCVEncoder : public Encoder {  // ref opencv.go:139-144, 847-905
  public:
    static Error Create(const std::string& ext, uint8_t* dst, size_t cap,
                        std::unique_ptr<Encoder>* out) {
        if (cap < 1) return LP_ERR_BUF_TOO_SMALL;
        opencv_mat m = opencv_mat_create_empty_from_data((int)cap, dst);
        if (!m) return LP_ERR_BUF_TOO_SMALL;
        opencv_encoder e = opencv_encoder_create(ext.c_str(), m);
        if (!e) {
            opencv_mat_release(m);
            return LP_ERR_INVALID_IMAGE;
        }
        auto* self = new OpenCVEncoder;
        self->encoder = e;
        self->dst = m;
        self->dstBuf = dst;
        out->reset(self);
        return LP_OK;
    }
    ~OpenCVEncoder() override {
        opencv_encoder_release(encoder);
        opencv_mat_release(dst);
    }
    Error Encode(Framebuffer* f, const std::map<int, int>& opt, bool* content,
                 size_t* out_len) override {  // ref opencv.go:872-900
        *content = false;
        if (!f) return LP_ERR_EOF;
        std::vector<int> optList;
        for (auto& kv : opt) {
            optList.push_back(kv.first);
            optList.push_back(kv.second);
        }
        if (!opencv_encoder_write(encoder, f->mat, optList.empty() ? nullptr : optList.data(),
                                  optList.size()))
            return LP_ERR_INVALID_IMAGE;
        // overflow is signalled by the destination mat having moved off dstBuf
        if (opencv_mat_get_data(dst) != (void*)dstBuf) return LP_ERR_BUF_TOO_SMALL;
        *out_len = (size_t)opencv_mat_get_height(dst);  // rows == encoded length
        *content = true;
        return LP_OK;
    }

  private:
    opencv_encoder encoder = nullptr;
    opencv_mat dst = nullptr;
    uint8_t* dstBuf = nullptr;
};

// ------------------------------------------------------------------ GIF adapter

static std::atomic<uint64_t> gifMaxFrameDimension{10000};  // ref giflib.go:39,49-52,305-307
void SetGIFMaxFrameDimension(uint64_t dim) { gifMaxFrameDimension.store(dim); }

class GifDecoder : public Decoder {  // ref giflib.go:14-30, 56-234
  public:
    static Error Create(const uint8_t* buf, size_t len, std::unique_ptr<Decoder>* out) {
        opencv_mat m = opencv_mat_create_from_data((int)len, 1, CV_8U, (void*)buf, len);
        if (!m) return LP_ERR_BUF_TOO_SMALL;
        giflib_decoder d = giflib_decoder_create(m);
        if (!d) {
            opencv_mat_release(m);
            return LP_ERR_INVALID_IMAGE;
        }
        auto* self = new GifDecoder;
        self->mat = m;
        self->decoder = d;
        self->len = len;
        out->reset(self);
        return LP_OK;
    }
    ~GifDecoder() override {
        giflib_decoder_release(decoder);
        opencv_mat_release(mat);
    }
    Error Header(ImageHeader* h) override {  // ref giflib.go:76-85
        h->width = giflib_decoder_get_width(decoder);
        h->height = giflib_decoder_get_height(decoder);
        h->pixelType.v = CV_8UC4;
        h->orientation = 1;
        readAnimationInfo();
        h->numFrames = info.frame_count;
        h->contentLength = (int)len;
        return LP_OK;
    }
    std::string Description() override { return "GIF"; }
    Error DecodeTo(Framebuffer* f) override {  // ref giflib.go:180-219
        ImageHeader h;
        Header(&h);
        Error e = f->resizeMat(h.width, h.height, h.pixelType);
        if (e) return e;
        const int next = (int)giflib_decoder_decode_frame_header(decoder);
        if (next == giflib_decoder_eof) return LP_ERR_EOF;
        if (next == giflib_decoder_error) return LP_ERR_INVALID_IMAGE;
        const int maxDim = (int)gifMaxFrameDimension.load();
        if (giflib_decoder_get_frame_width(decoder) > maxDim || giflib_decoder_get_frame_height(decoder) > maxDim)
            return LP_ERR_INVALID_IMAGE;
        if (!giflib_decoder_decode_frame(decoder, f->mat)) return LP_ERR_DECODING_FAILED;
        f->duration_ns = (int64_t)giflib_decoder_get_prev_frame_delay(decoder) * 10 * 1000000;
        f->blend = NoBlend;
        // Go stores the C value straight into DisposeMethod: 1 (GIF_DISPOSE_BACKGROUND) happens to
        // equal DisposeToBackgroundColor; 2 (previous) matches no case in applyDisposeMethod
        f->dispose = (DisposeMethod)giflib_decoder_get_prev_frame_disposal(decoder);
        f->xOffset = 0;
        f->yOffset = 0;
        return LP_OK;
    }
    Error SkipFrame() override {  // ref giflib.go:223-234
        const int next = (int)giflib_decoder_skip_frame(decoder);
        if (next == giflib_decoder_eof) return LP_ERR_EOF;
        if (next == giflib_decoder_error) return LP_ERR_INVALID_IMAGE;
        return LP_OK;
    }
    uint32_t BackgroundColor() override {  // ref giflib.go:131-134
        readAnimationInfo();
        return ((uint32_t)info.bg_red << 16) | ((uint32_t)info.bg_green << 8) | (uint32_t)info.bg_blue |
               ((uint32_t)info.bg_alpha << 24);
    }
    int LoopCount() override {
        readAnimationInfo();
        return info.loop_count;
    }
    int64_t Duration_ns() override {
        readAnimationInfo();
        return (int64_t)info.duration_ms * 1000000;
    }
    giflib_decoder GifHandle() override { return decoder; }

  private:
    void readAnimationInfo() {  // ref giflib.go:138-151 (lazy, cached)
        if (!infoRead) {
            info = giflib_decoder_get_animation_info(decoder);
            infoRead = true;
        }
    }
    opencv_mat mat = nullptr;
    giflib_decoder decoder = nullptr;
    size_t len = 0;
    bool infoRead = false;
    GifAnimationInfo info{};
};

class GifEncoder : public Encoder {  // ref giflib.go:239-300
  public:
    static Error Create(Decoder* decodedBy, uint8_t* dst, size_t cap, std::unique_ptr<Encoder>* out) {
        if (!decodedBy || !decodedBy->GifHandle()) return LP_ERR_INVALID_IMAGE;  // ErrGifEncoderNeedsDecoder
        giflib_encoder e = giflib_encoder_create(dst, cap);
        if (!e) return LP_ERR_BUF_TOO_SMALL;
        auto* self = new GifEncoder;
        self->encoder = e;
        self->decoder = decodedBy->GifHandle();
        out->reset(self);
        return LP_OK;
    }
    ~GifEncoder() override { giflib_encoder_release(encoder); }
    Error Encode(Framebuffer* f, const std::map<int, int>&, bool* content, size_t* out_len) override {
        *content = false;
        if (hasFlushed) return LP_ERR_EOF;
        if (!f) {
            if (!giflib_encoder_flush(encoder, decoder)) return LP_ERR_INVALID_IMAGE;
            hasFlushed = true;
            *out_len = (size_t)giflib_encoder_get_output_length(encoder);
            *content = true;
            return LP_OK;
        }
        if (frameIndex == 0) giflib_encoder_init(encoder, decoder, f->Width(), f->Height());
        if (!giflib_encoder_encode_frame(encoder, decoder, f->mat)) return LP_ERR_INVALID_IMAGE;
        frameIndex++;
        return LP_OK;  // (nil, nil): send the next frame
    }

  private:
    giflib_encoder encoder = nullptr;
    giflib_decoder decoder = nullptr;
    int frameIndex = 0;
    bool hasFlushed = false;
};

static std::string lower(std::string s) {
    for (auto& c : s) c = (char)tolower((unsigned char)c);
    return s;
}

// ------------------------------------------------------------------ WebP adapter

class WebpDecoder : public Decoder {  // ref webp.go:13-18, 30-176
  public:
    static Error Create(const uint8_t* buf, size_t len, std::unique_ptr<Decoder>* out) {
        opencv_mat m = opencv_mat_create_from_data((int)len, 1, CV_8U, (void*)buf, len);
        if (!m) return LP_ERR_BUF_TOO_SMALL;
        webp_decoder d = webp_decoder_create(m);
        if (!d) {
            opencv_mat_release(m);
            return LP_ERR_INVALID_IMAGE;
        }
        auto* self = new WebpDecoder;
        self->mat = m;
        self->decoder = d;
        self->len = len;
        out->reset(self);
        return LP_OK;
    }
    ~WebpDecoder() override {
        webp_decoder_release(decoder);
        opencv_mat_release(mat);
    }
    Error Header(ImageHeader* h) override {  // ref webp.go:50-59
        h->width = webp_decoder_get_width(decoder);
        h->height = webp_decoder_get_height(decoder);
        h->pixelType.v = webp_decoder_get_pixel_type(decoder);
        h->orientation = 1;
        h->numFrames = webp_decoder_get_num_frames(decoder);
        h->contentLength = (int)len;
        return LP_OK;
    }
    std::string Description() override { return "WEBP"; }
    Error DecodeTo(Framebuffer* f) override {  // ref webp.go:139-171
        if (!f) return LP_ERR_EOF;
        ImageHeader h;
        Header(&h);
        Error e = f->resizeMat(h.width, h.height, h.pixelType);
        if (e) return e;
        if (!webp_decoder_decode(decoder, f->mat)) {
            if (webp_decoder_has_more_frames(decoder) == 0) return LP_ERR_EOF;
            return LP_ERR_DECODING_FAILED;
        }
        // NB: the C side re-creates the mat at the frame's own size (ref webp.cpp:319-320) while the
        // Go Framebuffer keeps the canvas width/height it was resized to; mirrored as is.
        f->duration_ns = (int64_t)webp_decoder_get_prev_frame_delay(decoder) * 1000000;
        f->xOffset = webp_decoder_get_prev_frame_x_offset(decoder);
        f->yOffset = webp_decoder_get_prev_frame_y_offset(decoder);
        f->dispose = (DisposeMethod)webp_decoder_get_prev_frame_dispose(decoder);
        f->blend = (BlendMethod)webp_decoder_get_prev_frame_blend(decoder);
        webp_decoder_advance_frame(decoder);
        return LP_OK;
    }
    Error SkipFrame() override { return LP_ERR_SKIP_NOT_SUPPORTED; }  // ref webp.go:174-176
    std::vector<uint8_t> ICC() override {                             // ref webp.go:103-107
        std::vector<uint8_t> icc(32768);  // ICCProfileBufferSize, ref lilliput.go:15
        icc.resize(webp_decoder_get_icc(decoder, icc.data(), icc.size()));
        return icc;
    }
    uint32_t BackgroundColor() override { return webp_decoder_get_bg_color(decoder); }
    int LoopCount() override { return (int)webp_decoder_get_loop_count(decoder); }
    int64_t Duration_ns() override { return (int64_t)webp_decoder_get_total_duration(decoder) * 1000000; }

  private:
    webp_decoder decoder = nullptr;
    opencv_mat mat = nullptr;
    size_t len = 0;
};

bool iccHeaderIsSane(const uint8_t* icc, size_t len) {
    if (!icc || len < 128) return false;
    const size_t declared = ((size_t)icc[0] << 24) | ((size_t)icc[1] << 16) | ((size_t)icc[2] << 8) | icc[3];
    return declared == len;
}

class WebpEncoder : public Encoder {  // ref webp.go:20-26, 178-261
  public:
    static Error Create(Decoder* decodedBy, uint8_t* dst, size_t cap, std::unique_ptr<Encoder>* out) {
        std::vector<uint8_t> icc = decodedBy ? decodedBy->ICC() : std::vector<uint8_t>();
        if (!iccHeaderIsSane(icc.data(), icc.size())) icc.clear();
        const uint32_t bg = decodedBy ? decodedBy->BackgroundColor() : 0xFFFFFFFFu;
        const int loops = decodedBy ? decodedBy->LoopCount() : 0;
        // the encoder borrows the profile until flush (ref webp.cpp:397-398 keeps the pointer, webp.go keeps the
        // slice alive in the encoder struct): it lives in this object, not on Create's stack
        std::unique_ptr<WebpEncoder> self(new WebpEncoder);
        self->icc = std::move(icc);
        self->encoder = webp_encoder_create(dst, cap, self->icc.empty() ? nullptr : self->icc.data(), self->icc.size(),
                                            bg, loops);
        if (!self->encoder) return LP_ERR_BUF_TOO_SMALL;
        out->reset(self.release());
        return LP_OK;
    }
    ~WebpEncoder() override {
        if (encoder) webp_encoder_release(encoder);
    }
    Error Encode(Framebuffer* f, const std::map<int, int>& opt, bool* content, size_t* out_len) override {
        *content = false;
        if (hasFlushed) return LP_ERR_EOF;
        if (!f) {
            const size_t n = webp_encoder_flush(encoder);
            if (n == 0) return LP_ERR_INVALID_IMAGE;
            hasFlushed = true;
            *out_len = n;
            *content = true;
            return LP_OK;
        }
        std::vector<int> flat;
        for (const auto& kv : opt) {
            flat.push_back(kv.first);
            flat.push_back(kv.second);
        }
        const int delay = (int)(f->duration_ns / 1000000);
        const size_t n = webp_encoder_write(encoder, f->mat, flat.empty() ? nullptr : flat.data(), flat.size(), delay,
                                            (int)f->blend, (int)f->dispose, 0, 0);
        if (n == 0) return LP_ERR_INVALID_IMAGE;
        frameIndex++;
        return LP_OK;  // (nil, nil): send the next frame
    }

  private:
    webp_encoder encoder = nullptr;
    std::vector<uint8_t> icc;  // borrowed by `encoder`
    int frameIndex = 0;
    bool hasFlushed = false;
};

// ref lilliput.go:129-164.  GIF goes to the giflib adapter, WebP to the WebP adapter; AVIF / video are
// routed away BEFORE the OpenCV adapter is tried and reported as LP_ERR_UNSUPPORTED (out of scope,
// DESIGN.md s.8) rather than silently mis-decoded.
Error NewDecoder(const uint8_t* buf, size_t len, std::unique_ptr<Decoder>* out) {
    if (len == 0) return LP_ERR_INVALID_IMAGE;
    if (len >= 6 && (!memcmp(buf, "GIF87a", 6) || !memcmp(buf, "GIF89a", 6)))
        return GifDecoder::Create(buf, len, out);
    if (len >= 12 && !memcmp(buf, "RIFF", 4) && !memcmp(buf + 8, "WEBP", 4))  // ref lilliput.go:104-109,147-150
        return WebpDecoder::Create(buf, len, out);
    if (len >= 12 && !memcmp(buf + 4, "ftyp", 4) &&
        (!memcmp(buf + 8, "avif", 4) || !memcmp(buf + 8, "avis", 4)))
        return LP_ERR_UNSUPPORTED;
    return OpenCVDecoder::Create(buf, len, out);
}

// ref lilliput.go:180-202
Error NewEncoder(const std::string& ext_, Decoder* decodedBy, uint8_t* dst, size_t cap,
                 std::unique_ptr<Encoder>* out) {
    std::string ext = lower(ext_);
    if (ext == ".gif") return GifEncoder::Create(decodedBy, dst, cap, out);
    if (ext == ".webp") return WebpEncoder::Create(decodedBy, dst, cap, out);  // ref lilliput.go:185-187
    if (ext == ".avif" || ext == ".thumbhash") return LP_ERR_UNSUPPORTED;
    if (ext == ".mp4" || ext == ".webm") return LP_ERR_INVALID_IMAGE;
    return OpenCVEncoder::Create(ext_, dst, cap, out);
}

// ------------------------------------------------------------------ ImageOps

void calculateExpectedSize(int ow, int oh, int rw, int rh, int* w, int* h) {  // ref ops.go:243-255
    int m = std::min(ow, oh);
    if (rw == rh && rw > m) {
        *w = m;
        *h = m;
    } else if (rw > ow && rh > oh && rw != rh) {
        *w = ow;
        *h = oh;
    } else {
        *w = rw;
        *h = rh;
    }
}

ImageOps::ImageOps(int maxSize_) : maxSize(maxSize_) {
    frames[0].reset(new Framebuffer(maxSize, maxSize));
    frames[1].reset(new Framebuffer(maxSize, maxSize));
}

void ImageOps::Clear() {
    frames[0]->Clear();
    frames[1]->Clear();
    if (animatedCompositeBuffer) animatedCompositeBuffer->Clear();
}

Error ImageOps::decode(Decoder* d) { return d->DecodeTo(active()); }  // ref ops.go:154-165

// ref ops.go:132-150
Error ImageOps::setupAnimatedFrameBuffers(Decoder*, int icw, int ich, bool alpha) {
    if (animatedCompositeBuffer) return LP_OK;
    animatedCompositeBuffer.reset(new Framebuffer(icw, ich));
    Error e = alpha ? animatedCompositeBuffer->Create4Channel(icw, ich)
                    : animatedCompositeBuffer->Create3Channel(icw, ich);
    if (e) return e;
    return animatedCompositeBuffer->ClearToTransparent(0, 0, icw, ich);
}

Error ImageOps::applyDisposeMethod() {  // ref ops.go:552-562
    Framebuffer* a = active();
    if (a->dispose == DisposeToBackgroundColor)
        return animatedCompositeBuffer->ClearToTransparent(a->xOffset, a->yOffset, a->Width(),
                                                           a->Height());
    return LP_OK;
}

Error ImageOps::applyBlendMethod() {  // ref ops.go:566-582
    Framebuffer* a = active();
    if (a->blend == UseAlphaBlending)
        return animatedCompositeBuffer->CopyToOffsetWithAlphaBlending(a, a->xOffset, a->yOffset,
                                                                      a->Width(), a->Height());
    return animatedCompositeBuffer->CopyToOffsetNoBlend(a, a->xOffset, a->yOffset, a->Width(),
                                                        a->Height());
}

void ImageOps::copyFramePropertiesAndSwap() {  // ref ops.go:586-591
    secondary()->duration_ns = active()->duration_ns;
    secondary()->dispose = active()->dispose;
    secondary()->blend = active()->blend;
    swap();
}

// ref ops.go:170-204
Error ImageOps::fit(Decoder* d, int icw, int ich, int ocw, int och, bool animated, bool alpha) {
    int nw, nh;
    calculateExpectedSize(icw, ich, ocw, och, &nw, &nh);
    Error e;
    if (animated) {
        if ((e = setupAnimatedFrameBuffers(d, icw, ich, alpha))) return e;
        if ((e = applyBlendMethod())) return e;
        if ((e = animatedCompositeBuffer->Fit(nw, nh, secondary()))) return e;
        if ((e = applyDisposeMethod())) return e;
        copyFramePropertiesAndSwap();
        return LP_OK;
    }
    if ((e = active()->Fit(nw, nh, secondary()))) return e;
    copyFramePropertiesAndSwap();
    return LP_OK;
}

// ref ops.go:208-238
Error ImageOps::resize(Decoder* d, int icw, int ich, int ocw, int och, bool animated, bool alpha) {
    Error e;
    if (animated) {
        if ((e = setupAnimatedFrameBuffers(d, icw, ich, alpha))) return e;
        if ((e = applyBlendMethod())) return e;
        if ((e = animatedCompositeBuffer->ResizeTo(ocw, och, secondary()))) return e;
        if ((e = applyDisposeMethod())) return e;
        copyFramePropertiesAndSwap();
        return LP_OK;
    }
    if ((e = active()->ResizeTo(ocw, och, secondary()))) return e;
    copyFramePropertiesAndSwap();
    return LP_OK;
}

// ref ops.go:449-470 (+ inputCanvasSize :474-479)
Error ImageOps::transformCurrentFrame(Decoder* d, const ImageOptions& opt, const ImageHeader& h,
                                      int, bool* swapped) {
    *swapped = false;
    if (opt.ResizeMethod == LP_OPS_NO_RESIZE && !h.IsAnimated()) return LP_OK;
    int iw = h.width, ih = h.height;
    if (opt.NormalizeOrientation && ImageHeader::SwapsAxes(h.orientation)) std::swap(iw, ih);
    int ow = opt.Width, oh = opt.Height;
    if (opt.ResizeMethod == LP_OPS_NO_RESIZE) {
        ow = iw;
        oh = ih;
    }
    Error e;
    switch (opt.ResizeMethod) {
        case LP_OPS_FIT:
        case LP_OPS_NO_RESIZE:
            e = fit(d, iw, ih, ow, oh, h.IsAnimated(), h.HasAlpha());
            break;
        case LP_OPS_RESIZE:
            e = resize(d, iw, ih, ow, oh, h.IsAnimated(), h.HasAlpha());
            break;
        default:
            return LP_ERR_BAD_ARGUMENT;
    }
    if (!e) *swapped = true;
    return e;
}

Error ImageOps::skipToEnd(Decoder* d) {  // ref ops.go:336-344
    for (;;) {
        Error e = d->SkipFrame();
        if (e) return e;
    }
}

// ref ops.go:352-444 (+ the colour set-up of initializeTransform, ops.go:483-545).  Differences from the Go are
// only the ones the scope table excludes: no ICC synthesised from cICP (SURVEY 2 #6: color_info.cpp's lcms profiles
// stay the reference's).  HDR (PQ / HLG) sources ARE tone-mapped after every decode, as ops.go:154-165 does.  What IS mirrored of the cICP policy: an SDR cICP chunk of a PNG source
// is re-attached to a PNG output (ops.go:306-332); an HDR (PQ / HLG) tag is never re-emitted (ops.go:513-517).
Error ImageOps::Transform(Decoder* d, const ImageOptions& opt, uint8_t* dst, size_t dst_cap,
                          size_t* out_len, Encoder* encoder) {
    struct CompositeGuard {  // the deferred close at ops.go:353-358
        std::unique_ptr<Framebuffer>& p;
        ~CompositeGuard() { p.reset(); }
    } guard{animatedCompositeBuffer};

    *out_len = 0;
    ImageHeader h;
    Error e = d->Header(&h);
    if (e) return e;
    std::unique_ptr<::lilliput::CICP> outputCICP, tonemapCICP;  // ref ops.go:511-517
    {
        // HDR sources are tone-mapped unconditionally, right after every decode (ops.go:154-165); an SDR cICP is
        // signalling only and travels to a PNG output untouched
        ::lilliput::CICP c;
        if (d->CICP(&c)) (c.IsHDR() ? tonemapCICP : outputCICP).reset(new ::lilliput::CICP(c));
    }
    auto applyOutputCICP = [&](size_t n) -> size_t {  // ref ops.go:310-332
        if (!outputCICP || n == 0) return n;
        if (n < sizeof kPngMagic || memcmp(dst, kPngMagic, sizeof kPngMagic) != 0) return n;
        return opencv_png_insert_cicp(dst, n, dst_cap, outputCICP->Primaries, outputCICP->Transfer,
                                      outputCICP->Matrix, outputCICP->FullRange ? 1 : 0);
    };
    std::unique_ptr<Encoder> own;
    if (!encoder && (e = NewEncoder(opt.FileType, d, dst, dst_cap, &own))) return e;
    Encoder* enc = encoder ? encoder : own.get();

    int frameCount = 0;
    int64_t duration = 0;
    auto deadline =
        std::chrono::steady_clock::now() + std::chrono::nanoseconds(opt.EncodeTimeout_ns);
    auto encodeEmpty = [&](size_t* n) -> Error {
        bool content = false;
        Error ee = enc->Encode(nullptr, opt.EncodeOptions, &content, n);
        if (ee == LP_OK && !content) *n = 0;
        if (ee == LP_OK) *n = applyOutputCICP(*n);  // ref ops.go:285-291
        return ee;
    };

    for (;;) {
        e = decode(d);
        bool emptyFrame = false;
        if (e) {
            if (e != LP_ERR_EOF) return e;
            emptyFrame = true;
        }
        if (!emptyFrame && tonemapCICP) active()->TonemapToSDR(tonemapCICP->Transfer, tonemapCICP->Primaries);
        duration += active()->duration_ns;
        if (opt.MaxEncodeDuration_ns != 0 && duration > opt.MaxEncodeDuration_ns) {
            e = skipToEnd(d);
            if (e != LP_ERR_EOF) return e;
            return encodeEmpty(out_len);
        }
        // applied on EVERY iteration, regardless of NormalizeOrientation (ops.go:392)
        active()->OrientationTransform(h.orientation);

        bool swapped = false;
        if (!emptyFrame) {
            if ((e = transformCurrentFrame(d, opt, h, frameCount, &swapped))) return e;
        }
        bool content = false;
        size_t n = 0;
        if (emptyFrame)
            e = enc->Encode(nullptr, opt.EncodeOptions, &content, &n);
        else
            e = enc->Encode(active(), opt.EncodeOptions, &content, &n);
        if (e) return e;
        if (content) {
            *out_len = applyOutputCICP(n);  // ref ops.go:274-281
            return LP_OK;
        }
        frameCount++;
        if (opt.DisableAnimatedOutput) return encodeEmpty(out_len);
        if (opt.MaxEncodeFrames != 0 && frameCount == opt.MaxEncodeFrames) {
            e = skipToEnd(d);
            if (e != LP_ERR_EOF) return e;
            return encodeEmpty(out_len);
        }
        if (std::chrono::steady_clock::now() > deadline) return LP_ERR_ENCODE_TIMEOUT;
        if (swapped) swap();
    }
}

}  // namespace lilliput

// ------------------------------------------------------------------- C entry

using namespace lilliput;

static ImageOptions fromC(const lp_image_options* o) {
    ImageOptions r;
    r.FileType = o->file_type ? o->file_type : "";
    r.Width = o->width;
    r.Height = o->height;
    r.ResizeMethod = o->resize_method;
    r.NormalizeOrientation = o->normalize_orientation != 0;
    for (size_t i = 0; i + 1 < o->encode_options_len; i += 2)
        r.EncodeOptions[o->encode_options[i]] = o->encode_options[i + 1];
    r.MaxEncodeFrames = o->max_encode_frames;
    r.MaxEncodeDuration_ns = o->max_encode_duration_ns;
    r.EncodeTimeout_ns = o->encode_timeout_ns;
    r.DisableAnimatedOutput = o->disable_animated_output != 0;
    r.ForceSdr = o->force_sdr != 0;
    return r;
}

// The stage helpers below size their own framebuffers from the file's header; a real caller's ImageOps has
// a fixed maxSize and refuses larger images with ErrBufTooSmall (ref opencv.go:250-267).  Same rule here, so a
// hostile header cannot make a helper allocate gigabytes.
static const int kHelperMaxSide = 8192;

// One ImageOps per calling thread, reused across calls like a long-lived
// Go ImageOps (ref ops.go:83-91); re-created if max_size changes.
static ImageOps* thread_ops(int max_size) {
    thread_local std::unique_ptr<ImageOps> ops;
    thread_local int ops_size = 0;
    if (!ops || ops_size != max_size) {
        ops.reset(new ImageOps(max_size));
        ops_size = max_size;
    }
    return ops.get();
}

static int lp_transform_impl(const uint8_t* in, size_t in_len, const lp_image_options* opt,
                            uint8_t* dst, size_t dst_cap, size_t* out_len, int max_size) {
    if (!in || !opt || !dst || !out_len) return LP_ERR_BAD_ARGUMENT;
    std::unique_ptr<Decoder> d;
    Error e = NewDecoder(in, in_len, &d);
    if (e) return e;
    return thread_ops(max_size)->Transform(d.get(), fromC(opt), dst, dst_cap, out_len);
}

namespace lilliput {

// Stands where the still ".png" encoder (OpenCVEncoder) stands in Transform, and answers as it does: the first frame
// completes the output, an end of stream before any frame is LP_ERR_EOF
class FrameEncoder : public Encoder {
  public:
    explicit FrameEncoder(const FrameSink& s) : sink(s) {}
    Error Encode(Framebuffer* f, const std::map<int, int>&, bool* content, size_t* out_len) override {
        *content = false;
        if (!f) return LP_ERR_EOF;
        Error e = sink(f);
        if (e) return e;
        *out_len = 0;
        *content = true;
        return LP_OK;
    }

  private:
    const FrameSink& sink;
};

Error TransformToFrame(const uint8_t* in, size_t in_len, const lp_image_options* c_opt, int max_size, const FrameSink& sink) {
    try {
        if (!in || !c_opt) return LP_ERR_BAD_ARGUMENT;
        std::unique_ptr<Decoder> d;
        Error e = NewDecoder(in, in_len, &d);
        if (e) return e;
        ImageOptions opt = fromC(c_opt);
        opt.FileType = ".png";
        FrameEncoder enc(sink);
        size_t n = 0;
        uint8_t none = 0;
        return thread_ops(max_size)->Transform(d.get(), opt, &none, 0, &n, &enc);
    } catch (const std::bad_alloc&) {  // (as lp_transform reports an allocation the input makes impossible)
        return LP_ERR_BUF_TOO_SMALL;
    } catch (...) {
        return LP_ERR_BAD_ARGUMENT;
    }
}

// Stands where the encoder stands in Transform for TransformToClip: every frame is counted and its duration summed; a
// selected one goes to the sink.  The frame after which no slot is left completes the output; an end of stream completes
// it too once a frame has arrived, and is LP_ERR_EOF before any (as FrameEncoder answers).
class ClipEncoder : public Encoder {
  public:
    ClipEncoder(int F, int T, const ClipSink& s, int* index, int64_t* ms) : frames(F), slots(T), sink(s), frame_index(index), start_ms(ms) {}
    Error Encode(Framebuffer* f, const std::map<int, int>&, bool* content, size_t* out_len) override {
        *content = false;
        *out_len = 0;
        if (!f) {
            if (k == 0) return LP_ERR_EOF;
            *content = true;
            return LP_OK;
        }
        const int used = std::min(frames, slots);
        if (next < used && k == (frames <= slots ? next : (int)((int64_t)next * frames / slots))) {
            Error e = sink(f, next);
            if (e) return e;
            frame_index[next] = k;
            start_ms[next] = ms;
            next++;
        }
        ms += f->duration_ns / 1000000;
        k++;
        *content = next >= used;
        return LP_OK;
    }

  private:
    int frames, slots;
    const ClipSink& sink;
    int* frame_index;
    int64_t* start_ms;
    int k = 0, next = 0;  // frames seen, slots filled
    int64_t ms = 0;       // durations of the frames seen
};

Error TransformToClip(const uint8_t* in, size_t in_len, const lp_image_options* c_opt, int max_size, int T, const ClipSink& sink,
                      int* nframes, int* frame_index, int64_t* start_ms) {
    *nframes = 0;
    for (int t = 0; t < T; t++) {
        frame_index[t] = -1;
        start_ms[t] = 0;
    }
    try {
        if (!in || !c_opt || T < 1) return LP_ERR_BAD_ARGUMENT;
        std::unique_ptr<Decoder> d;
        Error e = NewDecoder(in, in_len, &d);
        if (e) return e;
        ImageHeader h;
        if ((e = d->Header(&h))) return e;
        // (an APNG's header says 2, but Transform decodes its first frame only)
        const int F = dynamic_cast<OpenCVDecoder*>(d.get()) ? 1 : std::max(h.numFrames, 0);
        ImageOptions opt = fromC(c_opt);
        opt.MaxEncodeFrames = 0;
        opt.MaxEncodeDuration_ns = 0;
        opt.DisableAnimatedOutput = false;
        opt.EncodeTimeout_ns = 1000000000000000000LL;  // (INT64_MAX would overflow Transform's now() + timeout)
        ClipEncoder enc(F, T, sink, frame_index, start_ms);
        size_t n = 0;
        uint8_t none = 0;
        e = thread_ops(max_size)->Transform(d.get(), opt, &none, 0, &n, &enc);
        if (!e) *nframes = F;
        return e;
    } catch (const std::bad_alloc&) {
        return LP_ERR_BUF_TOO_SMALL;
    } catch (...) {
        return LP_ERR_BAD_ARGUMENT;
    }
}

// A decoder of `nframes` w x h frames of 3 (BGR) or 4 (BGRA) channels whose pixels `fill` writes.  One frame: it answers
// as OpenCVDecoder answers for an 8-bit PNG of colour type 2 or 6 without ancillary chunks (orientation 1, no ICC
// profile, no cICP, no GIF handle).  Several: as WebpDecoder answers for an animated WebP of full-canvas frames with no
// blending or disposal, frame k lasting duration_ms[k], background 0xFFFFFFFF and loop count `loops` (webp.go:50-59,
// 139-176; the alpha flag gives the channel count), with no ICC profile either.
class FrameDecoder : public Decoder {
  public:
    FrameDecoder(int w, int h, int channels, int nframes, const int* duration_ms, int loops, const ClipFill& f)
        : width(w), height(h), type(channels == 4 ? CV_8UC4 : CV_8UC3), frames(nframes), ms(duration_ms), loops(loops), fill(f) {}
    Error Header(ImageHeader* h) override {
        h->width = width;
        h->height = height;
        h->pixelType.v = type;
        h->orientation = 1;
        h->numFrames = frames;
        return LP_OK;
    }
    std::string Description() override { return frames > 1 ? "WEBP" : "PNG"; }
    Error DecodeTo(Framebuffer* f) override {  // as OpenCVDecoder::DecodeTo, or WebpDecoder::DecodeTo
        if (next >= frames) return LP_ERR_EOF;
        Error e = f->resizeMat(width, height, PixelType{type});
        if (e) return e;
        if ((e = fill(f, next))) return e;
        const bool anim = frames > 1;
        f->blend = NoBlend;
        f->dispose = anim ? NoDispose : DisposeToBackgroundColor;
        f->xOffset = 0;
        f->yOffset = 0;
        f->duration_ns = anim ? (int64_t)ms[next] * 1000000 : 0;
        next++;
        return LP_OK;
    }
    Error SkipFrame() override { return LP_ERR_SKIP_NOT_SUPPORTED; }
    int LoopCount() override { return frames > 1 ? loops : 0; }
    int64_t Duration_ns() override {
        int64_t total = 0;
        for (int k = 0; frames > 1 && k < frames; k++) total += ms[k];
        return total * 1000000;
    }

  private:
    int width, height, type, frames;
    const int* ms;
    int loops;
    const ClipFill& fill;
    int next = 0;  // the frame DecodeTo delivers next
};

Error TransformFromClip(int w, int h, int channels, int nframes, const int* duration_ms, int loop_count, const lp_image_options* opt,
                        int max_size, const ClipFill& fill, uint8_t* dst, size_t dst_cap, size_t* out_len) {
    try {
        if (!opt || !dst || !out_len || nframes < 1 || (nframes > 1 && !duration_ms)) return LP_ERR_BAD_ARGUMENT;
        FrameDecoder d(w, h, channels, nframes, duration_ms, loop_count, fill);
        return thread_ops(max_size)->Transform(&d, fromC(opt), dst, dst_cap, out_len);
    } catch (const std::bad_alloc&) {
        return LP_ERR_BUF_TOO_SMALL;
    } catch (...) {
        return LP_ERR_BAD_ARGUMENT;
    }
}

Error TransformFromFrame(int w, int h, int channels, const lp_image_options* opt, int max_size, const FrameSink& fill, uint8_t* dst,
                         size_t dst_cap, size_t* out_len) {
    return TransformFromClip(w, h, channels, 1, nullptr, 0, opt, max_size, [&](Framebuffer* f, int) { return fill(f); }, dst, dst_cap,
                             out_len);
}

}  // namespace lilliput

static int lp_decode_host_impl(const uint8_t* in, size_t in_len, uint8_t* pixels,
                              size_t pixels_cap, int* width, int* height, int* type,
                              int* orientation) {
    std::unique_ptr<Decoder> d;
    Error e = NewDecoder(in, in_len, &d);
    if (e) return e;
    ImageHeader h;
    if ((e = d->Header(&h))) return e;
    if (width) *width = h.width;
    if (height) *height = h.height;
    if (type) *type = h.pixelType.v;
    if (orientation) *orientation = h.orientation;
    if (!pixels) return LP_OK;
    PixelType t = h.pixelType;
    if (t.Depth() > 8) t.v = opencv_type_convert_depth(t.v, CV_8U);
    if (type) *type = t.v;
    size_t need = (size_t)h.width * h.height * t.Channels();
    if (need > pixels_cap) return LP_ERR_BUF_TOO_SMALL;
    int side = std::max(h.width, h.height);
    if (side > kHelperMaxSide) return LP_ERR_BUF_TOO_SMALL;  // like an ImageOps whose framebuffers are smaller than the image
    Framebuffer f(side, side);
    if ((e = d->DecodeTo(&f))) return e;
    if (lp_mat_sync_host(f.mat)) return LP_ERR_CUDA;
    memcpy(pixels, opencv_mat_get_data(f.mat), need);
    return LP_OK;
}

static Error wrapPixels(Framebuffer& f, const uint8_t* src, int w, int h, int type) {
    Error e = f.resizeMat(w, h, PixelType{type});
    if (e) return e;
    memcpy(f.buf.data(), src, (size_t)w * h * opencv_type_channels(type));
    lp_mat_mark_host_dirty(f.mat);
    return LP_OK;
}

static int lp_fit_host_impl(const uint8_t* src, int sw, int sh, int type, uint8_t* dst, int dw,
                           int dh) {
    int side = std::max(std::max(sw, sh), std::max(dw, dh));
    Framebuffer a(side, side), b(side, side);
    Error e = wrapPixels(a, src, sw, sh, type);
    if (e) return e;
    if ((e = a.Fit(dw, dh, &b))) return e;
    if (lp_mat_sync_host(b.mat)) return LP_ERR_CUDA;
    memcpy(dst, opencv_mat_get_data(b.mat), (size_t)dw * dh * opencv_type_channels(type));
    return LP_OK;
}

static int lp_resize_host_impl(const uint8_t* src, int sw, int sh, int type, int cx, int cy, int cw,
                              int ch, uint8_t* dst, int dw, int dh, int interpolation) {
    int side = std::max(std::max(sw, sh), std::max(dw, dh));
    Framebuffer a(side, side), b(side, side);
    Error e = wrapPixels(a, src, sw, sh, type);
    if (e) return e;
    if (cx < 0 || cy < 0 || cw < 1 || ch < 1 || cx + cw > sw || cy + ch > sh)
        return LP_ERR_BAD_ARGUMENT;
    opencv_mat view = opencv_mat_crop(a.mat, cx, cy, cw, ch);
    if (!view) return LP_ERR_BAD_ARGUMENT;
    e = b.resizeMat(dw, dh, PixelType{type});
    if (!e) opencv_mat_resize(view, b.mat, dw, dh, interpolation);
    opencv_mat_release(view);
    if (e) return e;
    if (lp_mat_sync_host(b.mat)) return LP_ERR_CUDA;
    memcpy(dst, opencv_mat_get_data(b.mat), (size_t)dw * dh * opencv_type_channels(type));
    return LP_OK;
}

static int lp_encode_host_impl(const char* ext, const uint8_t* pixels, int w, int h, int type,
                              const int* opt, size_t opt_len, uint8_t* dst, size_t dst_cap,
                              size_t* out_len) {
    int side = std::max(w, h);
    Framebuffer a(side, side);
    Error e = wrapPixels(a, pixels, w, h, type);
    if (e) return e;
    std::unique_ptr<Encoder> enc;
    e = NewEncoder(ext, nullptr, dst, dst_cap, &enc);
    if (e) return e;
    std::map<int, int> o;
    for (size_t i = 0; i + 1 < opt_len; i += 2) o[opt[i]] = opt[i + 1];
    bool content = false;
    e = enc->Encode(&a, o, &content, out_len);
    if (e || content) return e;
    return enc->Encode(nullptr, o, &content, out_len);  // multi-frame encoders answer at the flush (ops.go:285-292)
}

static int lp_orient_host_impl(const uint8_t* src, int w, int h, int type, int orientation,
                              uint8_t* dst, int* ow, int* oh) {
    int side = std::max(w, h);
    Framebuffer a(side, side);
    Error e = wrapPixels(a, src, w, h, type);
    if (e) return e;
    a.OrientationTransform(orientation);
    if (lp_mat_sync_host(a.mat)) return LP_ERR_CUDA;
    *ow = a.Width();
    *oh = a.Height();
    memcpy(dst, opencv_mat_get_data(a.mat), (size_t)w * h * opencv_type_channels(type));
    return LP_OK;
}

static int lp_tonemap_host_impl(uint8_t* pixels, int w, int h, int type, int transfer, int primaries) {
    if (!pixels || w <= 0 || h <= 0) return LP_ERR_BAD_ARGUMENT;
    int side = std::max(w, h);
    Framebuffer a(side, side);
    Error e = wrapPixels(a, pixels, w, h, type);
    if (e) return e;
    a.TonemapToSDR(transfer, primaries);
    if (lp_mat_sync_host(a.mat)) return LP_ERR_CUDA;
    memcpy(pixels, opencv_mat_get_data(a.mat), (size_t)w * h * opencv_type_channels(type));
    return LP_OK;
}

static int lp_gif_get_info_impl(const uint8_t* in, size_t in_len, lp_gif_info* info) {
    if (!in || !info) return LP_ERR_BAD_ARGUMENT;
    std::unique_ptr<Decoder> d;
    Error e = NewDecoder(in, in_len, &d);
    if (e) return e;
    if (!d->GifHandle()) return LP_ERR_BAD_ARGUMENT;
    ImageHeader h;
    if ((e = d->Header(&h))) return e;
    info->width = h.width;
    info->height = h.height;
    info->frame_count = h.numFrames;
    info->loop_count = d->LoopCount();
    info->duration_ms = (int)(d->Duration_ns() / 1000000);
    info->background_color = d->BackgroundColor();
    return LP_OK;
}

static int lp_gif_decode_frames_host_impl(const uint8_t* in, size_t in_len, uint8_t* frames, size_t frames_cap,
                                         int max_frames, int* n_frames, int* delays_ms, int* disposals) {
    if (!in || !frames || !n_frames) return LP_ERR_BAD_ARGUMENT;
    *n_frames = 0;
    std::unique_ptr<Decoder> d;
    Error e = NewDecoder(in, in_len, &d);
    if (e) return e;
    if (!d->GifHandle()) return LP_ERR_BAD_ARGUMENT;
    ImageHeader h;
    if ((e = d->Header(&h))) return e;
    const size_t frame_bytes = (size_t)h.width * h.height * 4;
    // like ImageOps, ONE framebuffer receives every frame (the compositor builds on its content)
    if (std::max(h.width, h.height) > kHelperMaxSide) return LP_ERR_BUF_TOO_SMALL;
    Framebuffer f(std::max(h.width, h.height), std::max(h.width, h.height));
    for (int i = 0; i < max_frames; i++) {
        e = d->DecodeTo(&f);
        if (e == LP_ERR_EOF) return LP_OK;
        if (e) return e;
        if ((size_t)(i + 1) * frame_bytes > frames_cap) return LP_ERR_BUF_TOO_SMALL;
        if (lp_mat_sync_host(f.mat)) return LP_ERR_CUDA;
        memcpy(frames + (size_t)i * frame_bytes, opencv_mat_get_data(f.mat), frame_bytes);
        if (delays_ms) delays_ms[i] = (int)(f.duration_ns / 1000000);
        if (disposals) disposals[i] = (int)f.dispose;
        *n_frames = i + 1;
    }
    return LP_OK;
}

// Raw webp_decoder_* walk (ref webp.hpp:35-51,74-75): every frame exactly as webp_decoder_decode
// leaves it in the mat (frame-sized, BGR or BGRA), packed back to back into `frames`.
// meta[8*i..] = width, height, channels, x_offset, y_offset, delay_ms, dispose, blend.
// info[0..7] = canvas width, canvas height, pixel type, frame count, total duration, loop count,
// background colour, ICC length.
static int lp_webp_decode_frames_host_impl(const uint8_t* in, size_t in_len, uint8_t* frames, size_t frames_cap,
                                          int max_frames, int* n_frames, int* meta, unsigned int* info) {
    if (!in || !n_frames) return LP_ERR_BAD_ARGUMENT;
    *n_frames = 0;
    opencv_mat src = opencv_mat_create_from_data((int)in_len, 1, CV_8U, (void*)in, in_len);
    if (!src) return LP_ERR_BUF_TOO_SMALL;
    webp_decoder d = webp_decoder_create(src);
    if (!d) {
        opencv_mat_release(src);
        return LP_ERR_INVALID_IMAGE;
    }
    const int cw = webp_decoder_get_width(d), ch = webp_decoder_get_height(d), type = webp_decoder_get_pixel_type(d);
    if (info) {
        std::vector<uint8_t> icc(32768);
        info[0] = (unsigned)cw;
        info[1] = (unsigned)ch;
        info[2] = (unsigned)type;
        info[3] = (unsigned)webp_decoder_get_num_frames(d);
        info[4] = (unsigned)webp_decoder_get_total_duration(d);
        info[5] = webp_decoder_get_loop_count(d);
        info[6] = webp_decoder_get_bg_color(d);
        info[7] = (unsigned)webp_decoder_get_icc(d, icc.data(), icc.size());
    }
    int rc = LP_OK;
    size_t used = 0;
    if (std::max(cw, ch) > kHelperMaxSide) {
        webp_decoder_release(d);
        opencv_mat_release(src);
        return frames ? LP_ERR_BUF_TOO_SMALL : LP_OK;  // header-only queries still answer
    }
    opencv_mat m = opencv_mat_create(cw, ch, type);
    for (int i = 0; frames && i < max_frames; i++) {
        if (!webp_decoder_decode(d, m)) {
            rc = (i >= webp_decoder_get_num_frames(d)) ? LP_OK : LP_ERR_DECODING_FAILED;
            break;
        }
        if (lp_mat_sync_host(m)) {
            rc = LP_ERR_CUDA;
            break;
        }
        const int w = opencv_mat_get_width(m), h = opencv_mat_get_height(m);
        const int chn = opencv_type_channels(type);
        const size_t row = (size_t)w * chn;  // cv::Mat::create leaves the mat continuous
        if (used + row * h > frames_cap) {
            rc = LP_ERR_BUF_TOO_SMALL;
            break;
        }
        const uint8_t* px = (const uint8_t*)opencv_mat_get_data(m);
        memcpy(frames + used, px, row * h);
        used += row * h;
        if (meta) {
            int* q = meta + 8 * i;
            q[0] = w;
            q[1] = h;
            q[2] = chn;
            q[3] = webp_decoder_get_prev_frame_x_offset(d);
            q[4] = webp_decoder_get_prev_frame_y_offset(d);
            q[5] = webp_decoder_get_prev_frame_delay(d);
            q[6] = webp_decoder_get_prev_frame_dispose(d);
            q[7] = webp_decoder_get_prev_frame_blend(d);
        }
        *n_frames = i + 1;
        webp_decoder_advance_frame(d);
    }
    opencv_mat_release(m);
    webp_decoder_release(d);
    opencv_mat_release(src);
    return rc;
}

// ---- C ABI entry points.  No C++ exception may cross the boundary: an allocation the input makes
//      impossible (a header that declares a 60000 x 60000 canvas ...) is reported like the Go side reports a
//      framebuffer that is too small.
#define LP_GUARDED(call)                      \
    try {                                     \
        return call;                          \
    } catch (const std::bad_alloc&) {         \
        return LP_ERR_BUF_TOO_SMALL;          \
    } catch (...) {                           \
        return LP_ERR_BAD_ARGUMENT;           \
    }
extern "C" int lp_transform(const uint8_t* in, size_t in_len, const lp_image_options* opt,
                            uint8_t* dst, size_t dst_cap, size_t* out_len, int max_size) { LP_GUARDED(lp_transform_impl(in, in_len, opt, dst, dst_cap, out_len, max_size)) }
extern "C" int lp_decode_host(const uint8_t* in, size_t in_len, uint8_t* pixels,
                              size_t pixels_cap, int* width, int* height, int* type,
                              int* orientation) { LP_GUARDED(lp_decode_host_impl(in, in_len, pixels, pixels_cap, width, height, type, orientation)) }
extern "C" int lp_fit_host(const uint8_t* src, int sw, int sh, int type, uint8_t* dst, int dw,
                           int dh) { LP_GUARDED(lp_fit_host_impl(src, sw, sh, type, dst, dw, dh)) }
extern "C" int lp_resize_host(const uint8_t* src, int sw, int sh, int type, int cx, int cy, int cw,
                              int ch, uint8_t* dst, int dw, int dh, int interpolation) { LP_GUARDED(lp_resize_host_impl(src, sw, sh, type, cx, cy, cw, ch, dst, dw, dh, interpolation)) }
extern "C" int lp_encode_host(const char* ext, const uint8_t* pixels, int w, int h, int type,
                              const int* opt, size_t opt_len, uint8_t* dst, size_t dst_cap,
                              size_t* out_len) { LP_GUARDED(lp_encode_host_impl(ext, pixels, w, h, type, opt, opt_len, dst, dst_cap, out_len)) }
extern "C" int lp_tonemap_host(uint8_t* pixels, int w, int h, int type, int transfer, int primaries) {
    LP_GUARDED(lp_tonemap_host_impl(pixels, w, h, type, transfer, primaries))
}
extern "C" int lp_orient_host(const uint8_t* src, int w, int h, int type, int orientation,
                              uint8_t* dst, int* ow, int* oh) { LP_GUARDED(lp_orient_host_impl(src, w, h, type, orientation, dst, ow, oh)) }
extern "C" int lp_detect_apng(const uint8_t* in, size_t in_len) { return in && detectAPNG(in, in_len) ? 1 : 0; }
extern "C" int lp_detect_content_length(const uint8_t* in, size_t in_len) { return in ? detectContentLength(in, in_len) : 0; }
static int lp_png_chunk_types_impl(const uint8_t* in, size_t in_len, uint8_t* types, int cap) {
    std::vector<std::array<uint8_t, 4>> t;
    if (!in || !pngChunkTypes(in, in_len, &t)) return -1;
    for (int i = 0; types && i < cap && i < (int)t.size(); i++) memcpy(types + 4 * i, t[i].data(), 4);
    return (int)t.size();
}
extern "C" int lp_png_chunk_types(const uint8_t* in, size_t in_len, uint8_t* types, int cap) { LP_GUARDED(lp_png_chunk_types_impl(in, in_len, types, cap)) }
extern "C" int lp_gif_get_info(const uint8_t* in, size_t in_len, lp_gif_info* info) { LP_GUARDED(lp_gif_get_info_impl(in, in_len, info)) }
extern "C" int lp_gif_decode_frames_host(const uint8_t* in, size_t in_len, uint8_t* frames, size_t frames_cap,
                                         int max_frames, int* n_frames, int* delays_ms, int* disposals) { LP_GUARDED(lp_gif_decode_frames_host_impl(in, in_len, frames, frames_cap, max_frames, n_frames, delays_ms, disposals)) }
extern "C" int lp_webp_decode_frames_host(const uint8_t* in, size_t in_len, uint8_t* frames, size_t frames_cap,
                                          int max_frames, int* n_frames, int* meta, unsigned int* info) { LP_GUARDED(lp_webp_decode_frames_host_impl(in, in_len, frames, frames_cap, max_frames, n_frames, meta, info)) }
