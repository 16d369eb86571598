// lilliput_host.hpp -- C++ mirror of lilliput's Go policy layer for the
// ImageOps.Transform hot path.  Go is not available in the build image, so the
// host side above the C ABI is written in C++ with the reference's own names,
// argument meaning and error behaviour:
//
//   Framebuffer          ref opencv.go:118-129, 207-440
//   Decoder / Encoder    ref lilliput.go:42-98
//   OpenCVDecoder        ref opencv.go:442-463, 639-661, 816-843
//   OpenCVEncoder        ref opencv.go:847-905
//   GifDecoder / GifEncoder  ref giflib.go:56-300
//   WebpDecoder          ref webp.go:13-176
//   NewDecoder           ref lilliput.go:129-164
//   NewEncoder           ref lilliput.go:180-202
//   ImageOps::Transform  ref ops.go:352-444 (+ helpers 154-350, 449-591)
//
// It talks ONLY to the per-image C ABI (include/lp_opencv.h), so the same
// translation unit links against liblilliput_b200 (CUDA) or against the
// reference's shims (oracle/_ref) -- that is how the parity tests and the CPU
// baseline run the identical policy code on both.
#pragma once
#include <cstddef>
#include <cstdint>
#include <array>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "lilliput_b200.h"
#include "lp_giflib.h"
#include "lp_webp.h"
#include "lp_opencv.h"

namespace lilliput {

// Go `error` values of the package (ref lilliput.go:25-30) map onto lp_status.
using Error = int;

// ref opencv.go:20-60 (DisposeMethod / BlendMethod)
// fixed underlying type: the Go types are plain ints and decoders store other codes in them (GIF's
// "restore previous" is 2, ref giflib.go:218), which an unfixed two-value enum may not hold
enum DisposeMethod : int { NoDispose = 0, DisposeToBackgroundColor = 1 };
enum BlendMethod : int { UseAlphaBlending = 0, NoBlend = 1 };

struct PixelType {
    int v = 0;
    int Depth() const { return opencv_type_depth(v); }
    int Channels() const { return opencv_type_channels(v); }
};

// ref opencv.go:131-204
struct ImageHeader {
    int width = 0, height = 0;
    PixelType pixelType;
    int orientation = 1;
    int numFrames = 1;
    int contentLength = 0;
    bool IsAnimated() const { return numFrames > 1; }
    bool HasAlpha() const { return pixelType.Channels() == 4; }
    static bool SwapsAxes(int o) { return o >= 5 && o <= 8; }  // ref opencv.go:98-107
};

// ref opencv.go:118-129.  `buf` stands in for the Go []byte: the Framebuffer
// owns width*height*4 bytes of host memory and the mat wraps them.
class Framebuffer {
  public:
    Framebuffer(int width, int height);  // NewFramebuffer, ref opencv.go:207-212
    ~Framebuffer();
    void Close();
    void Clear();                                              // ref opencv.go:223-228
    Error Create3Channel(int w, int h);                        // ref opencv.go:231-237
    Error Create4Channel(int w, int h);                        // ref opencv.go:240-246
    Error resizeMat(int w, int h, PixelType t);                // ref opencv.go:250-267
    void OrientationTransform(int orientation);                // ref opencv.go:271-279
    void TonemapToSDR(int transfer, int primaries);            // ref opencv.go:791-810
    Error ResizeTo(int w, int h, Framebuffer* dst);            // ref opencv.go:294-309
    Error ClearToTransparent(int x, int y, int w, int h);      // ref opencv.go:312-319
    Error Fit(int w, int h, Framebuffer* dst);                 // ref opencv.go:326-374
    Error CopyToOffsetWithAlphaBlending(Framebuffer* src, int x, int y, int w, int h);  // :430
    Error CopyToOffsetNoBlend(Framebuffer* src, int x, int y, int w, int h);            // :437
    int Width() const { return width; }
    int Height() const { return height; }
    PixelType Type() const { return pixelType; }

    std::vector<uint8_t> buf;
    opencv_mat mat = nullptr;
    int width = 0, height = 0;
    PixelType pixelType;
    int64_t duration_ns = 0;
    int xOffset = 0, yOffset = 0;
    DisposeMethod dispose = NoDispose;
    BlendMethod blend = UseAlphaBlending;
};

struct CICP {  // ref opencv.go:719-741 (ITU-T H.273 code points carried by a PNG cICP chunk)
    uint8_t Primaries = 0, Transfer = 0, Matrix = 0;
    bool FullRange = false;
    bool IsHDR() const { return Transfer == 16 || Transfer == 18; }  // PQ / HLG, ref color_info.cpp:39-42
};

class Decoder {  // ref lilliput.go:42-88
  public:
    virtual ~Decoder() {}
    virtual Error Header(ImageHeader* out) = 0;
    virtual std::string Description() = 0;
    virtual Error DecodeTo(Framebuffer* f) = 0;
    virtual Error SkipFrame() = 0;
    virtual std::vector<uint8_t> ICC() { return {}; }
    virtual uint32_t BackgroundColor() { return 0xFFFFFFFFu; }
    virtual int LoopCount() { return 0; }
    virtual int64_t Duration_ns() { return 0; }
    virtual giflib_decoder GifHandle() { return nullptr; }  // Go: type assertion to *gifDecoder
    // Go: type assertion to interface{ CICP() (CICP, bool) } (ops.go:511); only the PNG decoder has one
    virtual bool CICP(::lilliput::CICP*) { return false; }
};

// SetGIFMaxFrameDimension (ref giflib.go:44-52; default 10000, giflib.go:39,305-307)
void SetGIFMaxFrameDimension(uint64_t dim);

class Encoder {  // ref lilliput.go:90-98
  public:
    virtual ~Encoder() {}
    // Returns LP_OK with *out_len > 0 when content is complete, LP_OK with
    // *content == false when the encoder wants another frame (Go: nil, nil).
    virtual Error Encode(Framebuffer* f, const std::map<int, int>& opt, bool* content,
                         size_t* out_len) = 0;
};

struct ImageOptions {  // ref ops.go:26-65
    std::string FileType;
    int Width = 0, Height = 0;
    int ResizeMethod = LP_OPS_NO_RESIZE;
    bool NormalizeOrientation = false;
    std::map<int, int> EncodeOptions;
    int MaxEncodeFrames = 0;
    int64_t MaxEncodeDuration_ns = 0;
    int64_t EncodeTimeout_ns = 0;
    bool DisableAnimatedOutput = false;
    bool ForceSdr = false;
};

Error NewDecoder(const uint8_t* buf, size_t len, std::unique_ptr<Decoder>* out);
Error NewEncoder(const std::string& ext, Decoder* decodedBy, uint8_t* dst, size_t dst_cap,
                 std::unique_ptr<Encoder>* out);

// ICCHeaderIsSane (ref color_info.cpp:70-79): the WebP writer carries a profile only when it is at least a header
// (128 B) long and its big-endian size field equals its length; any other profile is dropped and the output written
// untagged (ref webp.go:190-197)
bool iccHeaderIsSane(const uint8_t* icc, size_t len);

// ref ops.go:243-255
void calculateExpectedSize(int origW, int origH, int reqW, int reqH, int* w, int* h);
// ref opencv.go:331-363 (the crop rectangle Fit hands to opencv_mat_crop)
void fitCropRect(int srcW, int srcH, int dstW, int dstH, int* left, int* top, int* wc, int* hc);
// ref opencv.go:533-637
int detectContentLength(const uint8_t* img, size_t len);
bool detectAPNG(const uint8_t* img, size_t len);
// ref opencv.go:468-511: chunk types in the order pngChunkIter visits them; false if not a PNG
bool pngChunkTypes(const uint8_t* img, size_t len, std::vector<std::array<uint8_t, 4>>* types);

class ImageOps {  // ref ops.go:67-150
  public:
    explicit ImageOps(int maxSize);  // NewImageOps, ref ops.go:83-91
    // ref ops.go:352-444.  encoder: used in place of NewEncoder(opt.FileType, ...) when given (dst and dst_cap then
    // only matter to what it writes)
    Error Transform(Decoder* d, const ImageOptions& opt, uint8_t* dst, size_t dst_cap,
                    size_t* out_len, Encoder* encoder = nullptr);
    void Clear();

  private:
    Framebuffer* active() { return frames[frameIndex].get(); }
    Framebuffer* secondary() { return frames[1 - frameIndex].get(); }
    void swap() { frameIndex = 1 - frameIndex; }
    Error decode(Decoder* d);
    Error fit(Decoder* d, int icw, int ich, int ocw, int och, bool animated, bool alpha);
    Error resize(Decoder* d, int icw, int ich, int ocw, int och, bool animated, bool alpha);
    Error setupAnimatedFrameBuffers(Decoder* d, int icw, int ich, bool alpha);
    Error applyDisposeMethod();
    Error applyBlendMethod();
    void copyFramePropertiesAndSwap();
    Error transformCurrentFrame(Decoder* d, const ImageOptions& opt, const ImageHeader& h,
                                int frameCount, bool* swapped);
    Error skipToEnd(Decoder* d);

    std::unique_ptr<Framebuffer> frames[2];
    int frameIndex = 0;
    std::unique_ptr<Framebuffer> animatedCompositeBuffer;
    int maxSize;
};

// The frame Transform would encode to PNG, handed to `sink` instead of an encoder: lp_transform(in, opt with FileType
// ".png") up to its first Encode call, whose Framebuffer (8-bit gray, BGR or BGRA) goes to sink.  Returns Transform's
// status, which is sink's when Transform gets that far.
using FrameSink = std::function<Error(Framebuffer*)>;
Error TransformToFrame(const uint8_t* in, size_t in_len, const lp_image_options* opt, int max_size, const FrameSink& sink);

// Every frame Transform hands its encoder, offered in order, with clip slots given to a chosen few: lp_transform(in, opt)
// with MaxEncodeFrames, MaxEncodeDuration and DisableAnimatedOutput off, no deadline, and a ClipEncoder in place of the
// encoder.  F is the frame count the decoder's Header() reports (1 for every source the OpenCV decoder takes); slot s
// of T holds frame s while F <= T, otherwise frame floor(s * F / T), and sink(frame, s) receives it (8-bit gray, BGR or
// BGRA).  Transform stops after the last selected frame (the encoder answers with content), or at the end of the
// stream.  *nframes = F; frame_index[s] and start_ms[s] (T entries each): the frame of slot s and the sum of the
// durations (ms) of the frames before it, or -1 and 0 for a slot never filled.  Returns Transform's status.
using ClipSink = std::function<Error(Framebuffer*, int slot)>;
Error TransformToClip(const uint8_t* in, size_t in_len, const lp_image_options* opt, int max_size, int T, const ClipSink& sink,
                      int* nframes, int* frame_index, int64_t* start_ms);

// The mirror of TransformToFrame: lp_transform of an 8-bit PNG of a w x h frame of `channels` (3: BGR, 4: BGRA) into dst.
// Transform runs with a FrameDecoder, which answers every Decoder call as OpenCVDecoder answers for such a PNG; its
// DecodeTo sizes the framebuffer (resizeMat) and then calls fill, which writes the frame's pixels into it.
Error TransformFromFrame(int w, int h, int channels, const lp_image_options* opt, int max_size, const FrameSink& fill, uint8_t* dst,
                         size_t dst_cap, size_t* out_len);

// The animated form: lp_transform of A, an animated WebP of `nframes` (>= 2) full-canvas w x h frames of `channels`,
// with no blending or disposal, frame k lasting duration_ms[k], background 0xFFFFFFFF and loop_count, whose frames are
// lossless.  The FrameDecoder then answers as WebpDecoder answers for A, and its DecodeTo calls fill(framebuffer, k)
// for frame k.  nframes == 1 is TransformFromFrame (durations and loop count unused).
using ClipFill = std::function<Error(Framebuffer*, int frame)>;
Error TransformFromClip(int w, int h, int channels, int nframes, const int* duration_ms, int loop_count, const lp_image_options* opt,
                        int max_size, const ClipFill& fill, uint8_t* dst, size_t dst_cap, size_t* out_len);

}  // namespace lilliput
