// abi_opencv.cu -- lilliput's per-image cgo surface (include/lp_opencv.h, same symbols as the
// reference's opencv.hpp:61-132) implemented over the sm_90a kernels.
//
// A mat that wraps caller memory keeps that pointer for the Go side and owns a packed mirror in
// HBM; pixels live on the device between calls and cross PCIe only as compressed bytes in
// (opencv_decoder_read_data) and encoded bytes out (opencv_encoder_write), or on an explicit
// lp_mat_sync_host.  Calls are synchronous on a per-host-thread stream, like the reference's.
// There is no CPU implementation behind these symbols: without a CUDA device every
// pixel-touching call fails loudly.
#include <algorithm>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"
#include "lp_opencv.h"

namespace lp {

thread_local long g_launches = 0;

static std::once_flag g_dev_once;
static int g_dev_status = LP_ERR_CUDA;

int ensure_device() {
    std::call_once(g_dev_once, [] {
        int n = 0;
        cudaError_t e = cudaGetDeviceCount(&n);
        if (e != cudaSuccess || n == 0) {
            fprintf(stderr,
                    "[lilliput_b200] no CUDA device available (%s); this library has no CPU path\n",
                    e == cudaSuccess ? "0 devices" : cudaGetErrorString(e));
            g_dev_status = LP_ERR_CUDA;
            return;
        }
        // keep freed stream-ordered allocations cached: per-image calls reuse them
        int dev = 0;
        cudaGetDevice(&dev);
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t thr = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
        g_dev_status = LP_OK;
    });
    return g_dev_status;
}

cudaStream_t thread_stream() {
    thread_local cudaStream_t st = nullptr;
    if (!st) cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    return st;
}

int fill_launch(uint8_t* dst, size_t step, int C, int w, int h, int b, int g, int r, int a,
                cudaStream_t st);

// Device allocation shared between a mat and its crop views.
struct DevBuf {
    uint8_t* p = nullptr;
    size_t bytes = 0;
    ~DevBuf() {
        if (p) cudaFreeAsync(p, thread_stream());
    }
};

static std::shared_ptr<DevBuf> dev_alloc(size_t bytes) {
    auto b = std::make_shared<DevBuf>();
    // +256: bulk row copies read up to 15 bytes past a row segment
    if (cudaMallocAsync(&b->p, bytes + 256, thread_stream()) != cudaSuccess) {
        fprintf(stderr, "[lilliput_b200] cudaMallocAsync(%zu) failed: %s\n", bytes,
                cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    b->bytes = bytes;
    return b;
}

struct Mat {
    uint8_t* host = nullptr;   // caller memory (never freed here) or owned_host
    size_t host_cap = 0;       // datalimit - data
    std::vector<uint8_t> owned_host;
    std::shared_ptr<DevBuf> dev;
    size_t dev_off = 0;        // byte offset of this mat's (0,0) in dev (crop views)
    size_t dev_step = 0;       // row stride in the device buffer
    int rows = 0, cols = 0, type = 0;
    size_t step = 0;           // host row stride
    bool host_valid = false, dev_valid = false;
    bool is_view = false;

    int channels() const { return ((type >> 3) & 63) + 1; }
    size_t elem() const {
        static const int bytes[8] = {1, 1, 2, 2, 4, 4, 8, 2};
        return (size_t)channels() * bytes[type & 7];
    }
    uint8_t* dptr() const { return dev ? dev->p + dev_off : nullptr; }
};

// Make the device mirror current (allocating + uploading when the host copy is newer).
static int ensure_dev(Mat* m) {
    int rc = ensure_device();
    if (rc) return rc;
    const size_t row = (size_t)m->cols * m->elem();
    if (!m->dev) {
        m->dev = dev_alloc(row * m->rows);
        if (!m->dev) return LP_ERR_CUDA;
        m->dev_off = 0;
        m->dev_step = row;
        m->dev_valid = false;
    }
    if (!m->dev_valid) {
        if (m->host && m->rows > 0 && row > 0)
            LP_CUDA_OK(cudaMemcpy2DAsync(m->dptr(), m->dev_step, m->host, m->step, row, m->rows,
                                         cudaMemcpyHostToDevice, thread_stream()));
        m->dev_valid = true;
    }
    return LP_OK;
}

// (Re)allocate the device mirror for new dimensions without uploading (about to be overwritten).
static int fresh_dev(Mat* m, int cols, int rows, int type) {
    int rc = ensure_device();
    if (rc) return rc;
    if (cols < 0 || rows < 0) return LP_ERR_BAD_ARGUMENT;
    Mat shape;
    shape.type = type;
    const size_t row = (size_t)cols * shape.elem();
    if (!m->dev || m->is_view || m->dev->bytes < row * rows) {
        auto fresh = dev_alloc(row * rows);
        if (!fresh) return LP_ERR_CUDA;  // `m` keeps its old geometry and contents
        m->dev = fresh;
    }
    m->cols = cols;
    m->rows = rows;
    m->type = type;
    m->step = row;
    m->dev_off = 0;
    m->dev_step = row;
    m->is_view = false;
    // From here on the device buffer is the one that matches the geometry (the caller is about to fill it; if that
    // fails its contents are undefined, as a failed cv:: call leaves them).  The host memory may be smaller than
    // the new geometry, so it must never be uploaded from again until lp_mat_sync_host has rewritten it.
    m->dev_valid = true;
    m->host_valid = false;
    return LP_OK;
}

struct Decoder {
    const uint8_t* data = nullptr;
    size_t len = 0;
    JpegHeader jpeg;
    PngHeader png;
    bool is_png = false;
    bool header_ok = false;
    std::string description;
};

struct Encoder {
    std::string ext;
    Mat* dst = nullptr;
};

static int sync_stream() {
    LP_CUDA_OK(cudaStreamSynchronize(thread_stream()));
    return LP_OK;
}

// Decode one baseline JPEG into m (device mirror).  Used by opencv_decoder_read_data.
static int decode_jpeg_into(const Decoder* d, Mat* m) {
    const JpegHeader& h = d->jpeg;
    if (!h.supported && !h.multiscan) {
        fprintf(stderr, "[lilliput_b200] JPEG variant not supported on the device path (sampling layout)\n");
        return LP_ERR_UNSUPPORTED;
    }
    // The Huffman tables in force and, for the files one thread walks scan by scan (jpeg_multiscan_kernel), the scans:
    // multi-scan files (progressive, or one scan per component) and baseline files with restart markers.  Other
    // baseline files go to the self-synchronising parallel decoder.
    std::vector<JpegScanDesc> scans;
    std::vector<JpegHuffSet> sets(1);
    int nscans = 0, nsets = 1;
    if (h.multiscan) {
        scans.resize(kMultiscanMaxScans);
        sets.resize(kMultiscanMaxSets);
        int rc = jpeg_parse_scans(d->data, d->len, h, scans.data(), (int)scans.size(), &nscans, sets.data(),
                                  (int)sets.size(), &nsets);
        if (rc) return rc;
        const size_t visits = jpeg_multiscan_visits(h, scans.data(), nscans);
        if (visits > kMultiscanMaxVisits) {
            fprintf(stderr, "[lilliput_b200] multi-scan JPEG: %zu block visits over %d scans exceed the serial decoder's budget\n",
                    visits, nscans);
            return LP_ERR_UNSUPPORTED;
        }
    } else {
        jpeg_build_huff_set(h, &sets[0]);
        if (h.restart_interval) {  // one scan visits every block once, so no visit budget: any size decodes
            scans.resize(1);
            jpeg_baseline_scan(h, &scans[0]);
            nscans = 1;
        }
    }
    const bool parallel = nscans == 0;
    cudaStream_t st = thread_stream();
    JpegDecodeItem it;
    memset(&it, 0, sizeof(it));
    it.scan_off = 0;
    it.scan_len = (uint32_t)h.scan_length;
    it.table_set = 0;
    it.restart_interval = h.restart_interval;
    const uint32_t total_blocks = jpeg_decode_item(h, &it);
    uint32_t tiles = 0;
    const uint32_t blocks = jpeg_item_set_window(&it, 0, 0, h.width, h.height, false, &tiles);  // whole image
    if (!parallel) {  // its scans are [0, nscans) of d_scans; the whole frame is the window, so no masks
        it.restart_interval = 0;
        it.table_set = 0;
        it.nscans = (uint32_t)nscans;
    }

    uint8_t* scratch = nullptr;
    const size_t upload_len = parallel ? h.scan_length : d->len;  // walked scan by scan: the whole file
    const size_t scan_bytes = round_up(upload_len + 16, (size_t)256);
    const size_t sets_b = round_up(sizeof(JpegHuffSet) * (size_t)nsets, (size_t)256);
    const size_t scans_b = round_up(sizeof(JpegScanDesc) * (size_t)nscans + 16, (size_t)256);
    const size_t coef_bytes = round_up((size_t)blocks * 64 * sizeof(int16_t), (size_t)256);
    const size_t clean_b = parallel ? round_up(huff_clean_bytes(h.scan_length), (size_t)256) : 0;
    const size_t states_b = parallel ? round_up(2 * huff_nsub(h.scan_length) * 8, (size_t)256) : 0;
    const size_t nslots_b = parallel ? round_up(2 * huff_nsub(h.scan_length) * 4, (size_t)256) : 0;
    const size_t dcdiff_b = parallel ? round_up((size_t)total_blocks * 2, (size_t)256) : 0;
    const size_t total = 1024 + sets_b + scan_bytes + coef_bytes + clean_b + states_b + nslots_b +
                         dcdiff_b + scans_b;
    LP_CUDA_OK(cudaMallocAsync(&scratch, total, st));
    JpegDecodeItem* d_item = reinterpret_cast<JpegDecodeItem*>(scratch);
    JpegHuffSet* d_hs = reinterpret_cast<JpegHuffSet*>(scratch + 1024);
    uint8_t* d_scan = scratch + 1024 + sets_b;
    int16_t* d_coef = reinterpret_cast<int16_t*>(d_scan + scan_bytes);
    uint8_t* d_clean = reinterpret_cast<uint8_t*>(d_coef) + coef_bytes;
    uint8_t* d_states = d_clean + clean_b;
    uint8_t* d_nslots = d_states + states_b;
    uint8_t* d_dcdiff = d_nslots + nslots_b;
    JpegScanDesc* d_scans = reinterpret_cast<JpegScanDesc*>(d_dcdiff + dcdiff_b);
    LP_CUDA_OK(cudaMemcpyAsync(d_item, &it, sizeof(it), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d_hs, sets.data(), sizeof(JpegHuffSet) * nsets, cudaMemcpyHostToDevice, st));
    if (parallel) {
        LP_CUDA_OK(cudaMemcpyAsync(d_scan, d->data + h.scan_offset, h.scan_length, cudaMemcpyHostToDevice, st));
    } else {
        LP_CUDA_OK(cudaMemcpyAsync(d_scans, scans.data(), sizeof(JpegScanDesc) * nscans, cudaMemcpyHostToDevice, st));
        LP_CUDA_OK(cudaMemcpyAsync(d_scan, d->data, d->len, cudaMemcpyHostToDevice, st));
    }
    JpegDecodeBatch b;
    b.items = d_item;
    b.tables = d_hs;
    b.scan = d_scan;
    b.coef = d_coef;
    b.frames = m->dptr();
    b.n = 1;
    b.max_tiles_per_image = (int)tiles;
    b.clean = d_clean;
    b.states = d_states;
    b.nslots = reinterpret_cast<uint32_t*>(d_nslots);
    b.dcdiff = reinterpret_cast<int16_t*>(d_dcdiff);
    if (!parallel) {
        b.n_multiscan = 1;
        b.scans = d_scans;
    }
    int rc = jpeg_decode_launch(b, st, nullptr);
    JpegDecodeItem back;
    if (!rc) {
        LP_CUDA_OK(cudaMemcpyAsync(&back, d_item, sizeof(back), cudaMemcpyDeviceToHost, st));
        rc = sync_stream();
    }
    cudaFreeAsync(scratch, st);
    if (rc) return rc;
    return back.status == 0 ? LP_OK : LP_ERR_DECODING_FAILED;
}

// Decode one PNG into m (device mirror).  Used by opencv_decoder_read_data.
static int decode_png_into(const Decoder* d, Mat* m) {
    const PngHeader& h = d->png;
    if (h.idat_total < 2) return LP_ERR_DECODING_FAILED;
    cudaStream_t st = thread_stream();
    PngDecodeItem it;
    png_decode_item(h, (uint32_t)m->dev_step, &it);
    // the IDAT payloads form ONE zlib stream: gather them on the host, one H2D copy
    std::vector<uint8_t> z(h.idat_total + 16, 0);
    size_t o = 0;
    for (const PngSegment& sgm : h.idat) {
        memcpy(z.data() + o, d->data + sgm.offset, sgm.length);
        o += sgm.length;
    }
    const size_t zb = round_up(z.size(), (size_t)256);
    const size_t rawb = round_up((size_t)it.raw_total + 16, (size_t)256);
    uint8_t* scratch = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&scratch, 4096 + zb + rawb, st));
    PngDecodeItem* d_item = reinterpret_cast<PngDecodeItem*>(scratch);
    uint8_t* d_z = scratch + 4096;
    uint8_t* d_raw = d_z + zb;
    static_assert(sizeof(PngDecodeItem) <= 4096, "item fits its slot");
    LP_CUDA_OK(cudaMemcpyAsync(d_item, &it, sizeof(it), cudaMemcpyHostToDevice, st));
    LP_CUDA_OK(cudaMemcpyAsync(d_z, z.data(), z.size(), cudaMemcpyHostToDevice, st));
    PngDecodeBatch b;
    b.items = d_item;
    b.z = d_z;
    b.raw = d_raw;
    b.frames = m->dptr();
    b.n = 1;
    b.max_width = h.width;
    b.max_height = h.height;
    int rc = png_decode_launch(b, st);
    PngDecodeItem back;
    if (!rc) {
        LP_CUDA_OK(cudaMemcpyAsync(&back, d_item, sizeof(back), cudaMemcpyDeviceToHost, st));
        rc = sync_stream();  // also keeps `z` alive until the copy has been consumed
    }
    cudaFreeAsync(scratch, st);
    if (rc) return rc;
    return back.status == 0 ? LP_OK : LP_ERR_DECODING_FAILED;
}

// Accessors for the other adapters (gif_decode.cu), which do not see the Mat layout.
const uint8_t* mat_host_bytes(const void* mat, size_t* len) {
    const Mat* m = static_cast<const Mat*>(mat);
    if (!m || !m->host) return nullptr;
    *len = (size_t)m->cols * m->rows * m->elem();
    return m->host;
}
// Read-only device view of a mat (uploading the host copy first when it is newer).
int mat_device_view(void* mat, int* cols, int* rows, int* type, const uint8_t** dev, size_t* step) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m || m->rows <= 0 || m->cols <= 0) return LP_ERR_BAD_ARGUMENT;
    int rc = ensure_dev(m);
    if (rc) return rc;
    *cols = m->cols;
    *rows = m->rows;
    *type = m->type;
    *dev = m->dptr();
    *step = m->dev_step;
    return LP_OK;
}
int mat_bind_device_frame(void* mat, int cols, int rows, int type, uint8_t** dev, size_t* step) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m) return LP_ERR_BAD_ARGUMENT;
    int rc = fresh_dev(m, cols, rows, type);
    if (rc) return rc;
    *dev = m->dptr();
    *step = m->dev_step;
    return LP_OK;
}
void mat_mark_device_written(void* mat) {
    Mat* m = static_cast<Mat*>(mat);
    m->dev_valid = true;
    m->host_valid = false;
}

}  // namespace lp

using namespace lp;

extern "C" {

const int CV_INTER_AREA = 3;
const int CV_INTER_LINEAR = 1;
const int CV_INTER_CUBIC = 2;

const char* lp_backend_name(void) { return "cuda-sm90a"; }

// ---- type helpers (ref opencv.cpp:83-96) ----------------------------------------------------
int opencv_type_depth(int type) {
    static const int bytes[8] = {1, 1, 2, 2, 4, 4, 8, 2};
    return bytes[type & 7] * 8;
}
int opencv_type_channels(int type) { return ((type >> 3) & 511) + 1; }
int opencv_type_convert_depth(int t, int depth) { return (depth & 7) | (t & ~7); }

// ---- mats (ref opencv.cpp:22-81, 196-241) ---------------------------------------------------
opencv_mat opencv_mat_create(int width, int height, int type) {
    if (width < 0 || height < 0) return nullptr;  // (the reference's cv::Mat would throw; nothing throws across this ABI)
    Mat* m = new Mat;
    m->cols = width;
    m->rows = height;
    m->type = type;
    m->step = (size_t)width * m->elem();
    try {
        m->owned_host.resize(m->step * height);
    } catch (const std::exception&) {  // no exception crosses the C ABI: an impossible size is a NULL mat
        delete m;
        return nullptr;
    }
    m->host = m->owned_host.data();
    m->host_cap = m->owned_host.size();
    m->host_valid = true;
    return m;
}

opencv_mat opencv_mat_create_from_data(int width, int height, int type, void* data,
                                       size_t data_len) {
    if (width < 0 || height < 0) return nullptr;
    Mat tmp;
    tmp.type = type;
    size_t total = (size_t)width * height * tmp.elem();
    if (total > data_len) return nullptr;  // -> ErrBufTooSmall (ref opencv.cpp:29-32)
    Mat* m = new Mat;
    m->cols = width;
    m->rows = height;
    m->type = type;
    m->step = (size_t)width * m->elem();
    m->host = static_cast<uint8_t*>(data);
    m->host_cap = data_len;
    m->host_valid = true;
    return m;
}

opencv_mat opencv_mat_create_empty_from_data(int length, void* data) {
    // 0 rows x 1 col CV_8U over `length` bytes of capacity (ref opencv.cpp:38-49)
    Mat* m = new Mat;
    m->cols = 1;
    m->rows = 0;
    m->type = CV_8U;
    m->step = 1;
    m->host = static_cast<uint8_t*>(data);
    m->host_cap = (size_t)length;
    m->host_valid = true;
    return m;
}

bool opencv_mat_set_row_stride(opencv_mat mat, size_t stride) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m) return false;
    if (m->step == stride) return true;
    size_t width_stride = (size_t)m->cols * m->elem();
    if (stride < width_stride || m->step != width_stride) return false;
    if (stride * m->rows > m->host_cap) return false;
    m->step = stride;
    m->dev_valid = false;  // the host layout changed under the mirror
    return true;
}

void opencv_mat_release(opencv_mat mat) { delete static_cast<Mat*>(mat); }

int opencv_mat_get_width(const opencv_mat mat) { return mat ? static_cast<const Mat*>(mat)->cols : 0; }
int opencv_mat_get_height(const opencv_mat mat) { return mat ? static_cast<const Mat*>(mat)->rows : 0; }
void* opencv_mat_get_data(const opencv_mat mat) { return mat ? static_cast<const Mat*>(mat)->host : nullptr; }

int lp_mat_sync_host(opencv_mat mat) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m) return LP_ERR_BAD_ARGUMENT;
    if (m->host_valid || !m->dev_valid) return LP_OK;
    const size_t row = (size_t)m->cols * m->elem();
    if (row * m->rows > m->host_cap) {  // e.g. after an axis-swapping orientation into a small buffer
        try {
            m->owned_host.resize(row * m->rows);
        } catch (const std::exception&) {
            return LP_ERR_BUF_TOO_SMALL;
        }
        m->host = m->owned_host.data();
        m->host_cap = m->owned_host.size();
    }
    m->step = row;
    LP_CUDA_OK(cudaMemcpy2DAsync(m->host, m->step, m->dptr(), m->dev_step, row, m->rows,
                                 cudaMemcpyDeviceToHost, thread_stream()));
    int rc = sync_stream();
    if (!rc) m->host_valid = true;
    return rc;
}

// Additive: Framebuffer.TonemapToSDR (ref opencv.go:791-810 -> color_info.cpp:239-270 tonemap_rgb_8u_inplace) on the
// device mirror of the mat.  In the reference this is a call on the Go buffer; here the pixels live in HBM.
int lp_mat_tonemap_to_sdr(opencv_mat mat, int transfer, int primaries) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m || m->rows <= 0 || m->cols <= 0) return LP_OK;
    if ((m->type & 7) != 0 || (m->channels() != 3 && m->channels() != 4)) return LP_OK;  // the reference returns silently
    int rc = ensure_dev(m);
    if (rc) return rc;
    rc = tonemap_to_sdr_launch(m->dptr(), m->dev_step, m->channels(), m->cols, m->rows, transfer, primaries, thread_stream());
    if (rc) return rc;
    m->dev_valid = true;
    m->host_valid = false;
    return sync_stream();
}

void lp_mat_mark_host_dirty(opencv_mat mat) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m) return;
    m->host_valid = true;
    m->dev_valid = false;
}

void opencv_mat_resize(const opencv_mat src, opencv_mat dst, int width, int height,
                       int interpolation) {
    Mat* s = static_cast<Mat*>(src);
    Mat* d = static_cast<Mat*>(dst);
    if (!s || !d || width < 1 || height < 1 || s->cols < 1 || s->rows < 1) return;  // (cv::resize asserts on these)
    if (interpolation != CV_INTER_LINEAR && interpolation != CV_INTER_AREA && interpolation != CV_INTER_CUBIC) {
        fprintf(stderr, "[lilliput_b200] opencv_mat_resize: interpolation %d is not supported\n", interpolation);
        return;  // nothing touched: `dst` keeps its geometry and contents
    }
    if (ensure_dev(s)) return;
    if (fresh_dev(d, width, height, s->type)) return;
    ResizeArgs a;
    a.src = s->dptr();
    a.src_img_stride = 0;
    a.src_row_stride = s->dev_step;
    a.channels = s->channels();
    a.crop_x = 0;
    a.crop_y = 0;
    a.crop_w = s->cols;
    a.crop_h = s->rows;
    a.dst = d->dptr();
    a.dst_img_stride = 0;
    a.dst_row_stride = d->dev_step;
    a.dst_w = width;
    a.dst_h = height;
    a.n = 1;
    a.interpolation = interpolation;
    int rc = resize_launch(a, thread_stream());
    // also on failure: `d` already has the new geometry and a device buffer of that size, while its host
    // memory may be smaller -- the (undefined) device contents are the ones that count from here on
    d->dev_valid = true;
    d->host_valid = false;
    if (rc) {
        fprintf(stderr, "[lilliput_b200] opencv_mat_resize failed (%d)\n", rc);
        return;
    }
    sync_stream();
}

opencv_mat opencv_mat_crop(const opencv_mat src, int x, int y, int width, int height) {
    Mat* s = static_cast<Mat*>(src);
    if (!s) return nullptr;
    // cv::Mat(m, Rect) throws on a rectangle that leaves the matrix (ref opencv.cpp:211-215 does not catch it); here
    // such a view would make every later kernel read outside the allocation, so it is refused
    if (x < 0 || y < 0 || width < 0 || height < 0 || (long long)x + width > s->cols || (long long)y + height > s->rows) {
        fprintf(stderr, "[lilliput_b200] opencv_mat_crop: (%d,%d %dx%d) is not inside %dx%d\n", x, y, width, height,
                s->cols, s->rows);
        return nullptr;
    }
    if (ensure_dev(s)) return nullptr;
    Mat* v = new Mat;
    v->cols = width;
    v->rows = height;
    v->type = s->type;
    v->step = s->step;
    v->host = s->host ? s->host + (size_t)y * s->step + (size_t)x * s->elem() : nullptr;
    v->host_cap = 0;
    v->host_valid = false;
    v->dev = s->dev;
    v->dev_off = s->dev_off + (size_t)y * s->dev_step + (size_t)x * s->elem();
    v->dev_step = s->dev_step;
    v->dev_valid = true;
    v->is_view = true;
    return v;
}

void opencv_mat_orientation_transform(CVImageOrientation orientation, opencv_mat mat) {
    Mat* m = static_cast<Mat*>(mat);
    const int o = (int)orientation;
    if (!m || o <= 1 || o > 8) return;  // TL: nothing to do
    if (ensure_dev(m)) return;
    const bool swap = o >= 5;
    const int W = swap ? m->rows : m->cols, H = swap ? m->cols : m->rows;
    const size_t row = (size_t)W * m->elem();
    auto out = dev_alloc(row * H);
    if (!out) return;
    // the kernel expects a packed source; mirrors are packed unless this is a view
    if (m->dev_step != (size_t)m->cols * m->elem()) {
        fprintf(stderr, "[lilliput_b200] orientation on a strided view is not supported\n");
        return;
    }
    if (orient_launch(m->dptr(), m->cols, m->rows, m->channels(), o, out->p, thread_stream())) return;
    sync_stream();
    m->dev = out;
    m->dev_off = 0;
    m->dev_step = row;
    m->cols = W;
    m->rows = H;
    m->step = row;
    m->is_view = false;
    m->dev_valid = true;
    m->host_valid = false;
}

void opencv_mat_reset(opencv_mat mat) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m) return;
    if (m->host && m->host_valid && !m->dev) {  // never touched the device: plain host zeroing
        for (int y = 0; y < m->rows; y++) memset(m->host + (size_t)y * m->step, 0, (size_t)m->cols * m->elem());
        return;
    }
    if (ensure_dev(m)) return;
    cudaMemset2DAsync(m->dptr(), m->dev_step, 0, (size_t)m->cols * m->elem(), m->rows, thread_stream());
    sync_stream();
    m->dev_valid = true;
    m->host_valid = false;
}

void opencv_mat_set_color(opencv_mat mat, int red, int green, int blue, int alpha) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m || ensure_dev(m)) return;
    // cv::Scalar(b,g,r[,a]) applied channel-wise; a 3-value scalar leaves a 4th channel 0
    fill_launch(m->dptr(), m->dev_step, m->channels(), m->cols, m->rows, blue, green, red,
                alpha >= 0 ? alpha : 0, thread_stream());
    sync_stream();
    m->host_valid = false;
}

int opencv_mat_clear_to_transparent(opencv_mat mat, int xOffset, int yOffset, int width, int height) {
    Mat* m = static_cast<Mat*>(mat);
    if (!m) return OPENCV_ERROR_NULL_MATRIX;
    if (xOffset < 0 || yOffset < 0 || (long long)xOffset + width > m->cols || (long long)yOffset + height > m->rows)
        return OPENCV_ERROR_OUT_OF_BOUNDS;
    if (width <= 0 || height <= 0) return OPENCV_ERROR_INVALID_DIMENSIONS;
    if (m->channels() != 3 && m->channels() != 4) return OPENCV_ERROR_INVALID_CHANNEL_COUNT;
    if (ensure_dev(m)) return OPENCV_ERROR_UNKNOWN;
    if (cudaMemset2DAsync(m->dptr() + (size_t)yOffset * m->dev_step + (size_t)xOffset * m->elem(),
                          m->dev_step, 0, (size_t)width * m->elem(), height, thread_stream()) != cudaSuccess)
        return OPENCV_ERROR_UNKNOWN;
    if (sync_stream()) return OPENCV_ERROR_UNKNOWN;
    m->host_valid = false;
    return OPENCV_SUCCESS;
}

static int copy_region_common(opencv_mat src, opencv_mat dst, int xOffset, int yOffset, int width,
                              int height, bool blend) {
    Mat* s = static_cast<Mat*>(src);
    Mat* d = static_cast<Mat*>(dst);
    if (!s || !d || s->rows == 0 || s->cols == 0 || d->rows == 0 || d->cols == 0)
        return OPENCV_ERROR_NULL_MATRIX;
    if (xOffset < 0 || yOffset < 0 || (long long)xOffset + width > d->cols || (long long)yOffset + height > d->rows)
        return OPENCV_ERROR_OUT_OF_BOUNDS;
    if (width <= 0 || height <= 0) return OPENCV_ERROR_INVALID_DIMENSIONS;
    const int sc = s->channels(), dc = d->channels();
    if (blend) {
        if ((sc != 1 && sc != 3 && sc != 4) || (dc != 3 && dc != 4)) return OPENCV_ERROR_INVALID_CHANNEL_COUNT;
    } else if (sc != dc) {
        if (!((sc == 3 && dc == 4) || (sc == 4 && dc == 3) || (sc == 1 && (dc == 3 || dc == 4))))
            return OPENCV_ERROR_INVALID_CHANNEL_COUNT;
    }
    if (ensure_dev(s) || ensure_dev(d)) return OPENCV_ERROR_UNKNOWN;
    cudaStream_t st = thread_stream();
    const uint8_t* sp = s->dptr();
    size_t sstep = s->dev_step;
    std::shared_ptr<DevBuf> tmp;
    if (s->cols != width || s->rows != height) {  // cv::resize(INTER_LINEAR) to the ROI size
        tmp = dev_alloc((size_t)width * height * sc);
        if (!tmp) return blend ? OPENCV_ERROR_ALPHA_BLENDING_FAILED : OPENCV_ERROR_COPY_FAILED;
        ResizeArgs a{sp, 0, sstep, sc, 0, 0, s->cols, s->rows, tmp->p, 0, (size_t)width * sc, width, height, 1, 1};
        if (resize_launch(a, st)) return OPENCV_ERROR_RESIZE_FAILED;
        sp = tmp->p;
        sstep = (size_t)width * sc;
    }
    uint8_t* dp = d->dptr() + (size_t)yOffset * d->dev_step + (size_t)xOffset * dc;
    int rc = blend ? blend_region_launch(sp, sstep, sc, dp, d->dev_step, dc, width, height, st)
                   : copy_region_launch(sp, sstep, sc, dp, d->dev_step, dc, width, height, st);
    if (rc || sync_stream()) return blend ? OPENCV_ERROR_ALPHA_BLENDING_FAILED : OPENCV_ERROR_COPY_FAILED;
    d->host_valid = false;
    return OPENCV_SUCCESS;
}

int opencv_copy_to_region_with_alpha(opencv_mat src, opencv_mat dst, int xOffset, int yOffset,
                                     int width, int height) {
    return copy_region_common(src, dst, xOffset, yOffset, width, height, true);
}
int opencv_copy_to_region(opencv_mat src, opencv_mat dst, int xOffset, int yOffset, int width,
                          int height) {
    return copy_region_common(src, dst, xOffset, yOffset, width, height, false);
}

// ---- decoder (ref opencv.cpp:99-171) --------------------------------------------------------
opencv_decoder opencv_decoder_create(const opencv_mat buf) {
    const Mat* m = static_cast<const Mat*>(buf);
    if (!m || !m->host) return nullptr;
    const size_t len = (size_t)m->cols * m->rows;
    if (len < 4) return nullptr;
    Decoder* d = new Decoder;
    d->data = m->host;
    d->len = len;
    if (d->data[0] == 0xFF && d->data[1] == 0xD8 && d->data[2] == 0xFF) {
        d->description = "JPEG";
        return d;
    }
    static const uint8_t png[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    if (len >= 8 && !memcmp(d->data, png, 8)) {
        d->description = "PNG";
        return d;
    }
    delete d;  // cv::ImageDecoder::empty(): no decoder recognises the signature
    return nullptr;
}

const char* opencv_decoder_get_description(const opencv_decoder d) {
    if (!d) return nullptr;
    static thread_local std::string desc;
    desc = static_cast<Decoder*>(d)->description;
    return desc.c_str();
}

void opencv_decoder_release(opencv_decoder d) { delete static_cast<Decoder*>(d); }

bool opencv_decoder_set_source(opencv_decoder d, const opencv_mat buf) {
    Decoder* dd = static_cast<Decoder*>(d);
    const Mat* m = static_cast<const Mat*>(buf);
    if (!dd || !m || !m->host) return false;
    dd->data = m->host;
    dd->len = (size_t)m->cols * m->rows;
    dd->header_ok = false;
    return true;
}

bool opencv_decoder_read_header(opencv_decoder d) {
    Decoder* dd = static_cast<Decoder*>(d);
    if (!dd) return false;
    if (dd->description == "JPEG") {
        int rc = jpeg_parse_header(dd->data, dd->len, &dd->jpeg);
        dd->header_ok = (rc == LP_OK);
        return dd->header_ok;
    }
    dd->is_png = true;
    dd->header_ok = png_parse(dd->data, dd->len, &dd->png) == LP_OK;
    return dd->header_ok;
}

int opencv_decoder_get_width(const opencv_decoder d) {
    const Decoder* dd = static_cast<Decoder*>(d);
    return dd->is_png ? dd->png.width : dd->jpeg.width;
}
int opencv_decoder_get_height(const opencv_decoder d) {
    const Decoder* dd = static_cast<Decoder*>(d);
    return dd->is_png ? dd->png.height : dd->jpeg.height;
}
int opencv_decoder_get_pixel_type(const opencv_decoder d) {
    const Decoder* dd = static_cast<Decoder*>(d);
    if (dd->is_png)  // 16-bit files report CV_16UCn; the 8-bit Framebuffer strips them (opencv.go:255)
        return (dd->png.bit_depth == 16 ? CV_16U : CV_8U) + ((dd->png.out_channels - 1) << 3);
    return dd->jpeg.ncomp == 1 ? CV_8UC1 : CV_8UC3;
}
int opencv_decoder_get_orientation(const opencv_decoder d) {
    const Decoder* dd = static_cast<Decoder*>(d);
    return dd->is_png ? dd->png.orientation : dd->jpeg.orientation;
}

bool opencv_decoder_read_data(opencv_decoder d, opencv_mat dst) {
    Decoder* dd = static_cast<Decoder*>(d);
    Mat* m = static_cast<Mat*>(dst);
    if (!dd || !m || !dd->header_ok) return false;
    int rc;
    if (dd->is_png) {
        if (fresh_dev(m, dd->png.width, dd->png.height, (dd->png.out_channels - 1) << 3)) return false;
        rc = decode_png_into(dd, m);
    } else {
        const int type = dd->jpeg.ncomp == 1 ? CV_8UC1 : CV_8UC3;
        if (fresh_dev(m, dd->jpeg.width, dd->jpeg.height, type)) return false;
        rc = decode_jpeg_into(dd, m);
    }
    if (rc) return false;
    m->dev_valid = true;
    m->host_valid = false;
    return true;
}

// ---- encoder (ref opencv.cpp:173-194) -------------------------------------------------------
opencv_encoder opencv_encoder_create(const char* ext, opencv_mat dst) {
    if (!ext || !dst) return nullptr;
    Encoder* e = new Encoder;
    e->ext = ext;
    for (auto& c : e->ext) c = (char)tolower((unsigned char)c);
    e->dst = static_cast<Mat*>(dst);
    return e;
}

void opencv_encoder_release(opencv_encoder e) { delete static_cast<Encoder*>(e); }

bool opencv_encoder_write(opencv_encoder e, const opencv_mat src, const int* opt, size_t opt_len) {
    Encoder* enc = static_cast<Encoder*>(e);
    Mat* s = static_cast<Mat*>(src);
    if (!enc || !s) return false;
    if (enc->ext == ".png") {
        int level;
        bool adaptive;
        png_encode_policy(opt, opt_len, &level, &adaptive);
        if (ensure_dev(s)) return false;
        std::vector<uint8_t> file;
        if (png_encode_frame(s->dptr(), s->dev_step, s->cols, s->rows, s->channels(), level, adaptive, &file,
                             thread_stream()) != LP_OK)
            return false;
        Mat* d = enc->dst;
        if (file.size() > d->host_cap) {  // overflow: data moves off the caller's buffer (opencv.go:890-895)
            d->owned_host.resize(file.size());
            d->host = d->owned_host.data();
            d->host_cap = file.size();
        }
        memcpy(d->host, file.data(), file.size());
        d->rows = (int)file.size();
        d->cols = 1;
        d->host_valid = true;
        return true;
    }
    if (enc->ext != ".jpeg" && enc->ext != ".jpg" && enc->ext != ".jpe") {
        fprintf(stderr, "[lilliput_b200] encoder for '%s' is not implemented on the device path yet\n",
                enc->ext.c_str());
        return false;
    }
    int quality = 95;  // OpenCV's default
    bool progressive = false;
    for (size_t i = 0; i + 1 < opt_len; i += 2) {
        if (opt[i] == CV_IMWRITE_JPEG_QUALITY) quality = std::min(std::max(opt[i + 1], 0), 100);
        if (opt[i] == CV_IMWRITE_JPEG_PROGRESSIVE) progressive = opt[i + 1] != 0;
    }
    if (ensure_dev(s)) return false;
    cudaStream_t st = thread_stream();
    const int W = s->cols, H = s->rows, C = s->channels();
    // worst case is bounded by the raw size for sane inputs; give generous room
    const size_t cap = round_up((size_t)W * H * 3 + 4096, (size_t)256);
    const size_t scratch_bytes = jpeg_encode_scratch_bytes(W, H, C, 1, cap, progressive);
    uint8_t* buf = nullptr;
    if (cudaMallocAsync(&buf, scratch_bytes + cap + 256, st) != cudaSuccess) return false;
    JpegEncodeBatch b;
    b.frames = s->dptr();
    b.frame_img_stride = 0;
    b.frame_row_stride = s->dev_step;
    b.width = W;
    b.height = H;
    b.channels = C;
    b.quality = quality;
    b.n = 1;
    b.out = buf + scratch_bytes + 256;
    b.out_cap = cap;
    b.out_len = reinterpret_cast<uint32_t*>(buf + scratch_bytes);
    b.scratch = buf;
    b.progressive = progressive;
    bool ok = jpeg_encode_launch(b, st, nullptr) == LP_OK;
    uint32_t n = 0;
    if (ok) ok = cudaMemcpyAsync(&n, b.out_len, 4, cudaMemcpyDeviceToHost, st) == cudaSuccess && !sync_stream();
    if (ok && (n == 0 || (size_t)n > cap)) ok = false;  // (n > cap cannot come from the kernel; never read past the buffer)
    if (ok) {
        Mat* d = enc->dst;
        if ((size_t)n > d->host_cap) {
            // The reference lets OpenCV reallocate: data moves off the caller's buffer and Go
            // reports ErrBufTooSmall from the pointer inequality (ref opencv.go:890-895).
            d->owned_host.resize(n);
            d->host = d->owned_host.data();
            d->host_cap = n;
        }
        ok = cudaMemcpyAsync(d->host, b.out, n, cudaMemcpyDeviceToHost, st) == cudaSuccess && !sync_stream();
        d->rows = (int)n;
        d->cols = 1;
        d->host_valid = true;
    }
    cudaFreeAsync(buf, st);
    return ok;
}

// ---- container metadata (ref opencv.cpp:253-464): host byte parsing ------------------------
static uint32_t be32(const uint8_t* p) {
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}

// jpeg_read_icc_profile semantics: APP2 "ICC_PROFILE\0" seq/count chunks concatenated in order.
int opencv_decoder_get_jpeg_icc(void* src, size_t src_len, void* dest, size_t dest_len) {
    const uint8_t* in = static_cast<const uint8_t*>(src);
    if (!in || src_len < 4 || in[0] != 0xFF || in[1] != 0xD8) return 0;
    struct Chunk { const uint8_t* p; size_t n; };
    std::vector<Chunk> chunks(256, Chunk{nullptr, 0});
    int count = 0;
    size_t pos = 2;
    while (pos + 4 <= src_len) {
        if (in[pos] != 0xFF) { pos++; continue; }
        uint8_t m = in[pos + 1];
        if (m == 0xFF) { pos++; continue; }
        if (m == 0xD9 || m == 0xDA) break;
        if (m == 0x01 || (m >= 0xD0 && m <= 0xD7)) { pos += 2; continue; }
        size_t seg = ((size_t)in[pos + 2] << 8) | in[pos + 3];
        if (seg < 2 || pos + 2 + seg > src_len) return 0;
        const uint8_t* p = in + pos + 4;
        size_t n = seg - 2;
        if (m == 0xE2 && n >= 14 && !memcmp(p, "ICC_PROFILE\0", 12)) {
            int seq = p[12], cnt = p[13];
            if (seq == 0 || cnt == 0 || seq > cnt) return 0;
            if (count == 0) count = cnt;
            else if (count != cnt) return 0;
            if (chunks[seq].p) return 0;
            chunks[seq] = Chunk{p + 14, n - 14};
        }
        pos += 2 + seg;
    }
    if (count == 0) return 0;
    size_t total = 0;
    for (int i = 1; i <= count; i++) {
        if (!chunks[i].p) return 0;
        total += chunks[i].n;
    }
    if (total == 0 || total > dest_len) return 0;
    uint8_t* o = static_cast<uint8_t*>(dest);
    for (int i = 1; i <= count; i++) {
        memcpy(o, chunks[i].p, chunks[i].n);
        o += chunks[i].n;
    }
    return (int)total;
}

int opencv_decoder_get_png_icc(void* src, size_t src_len, void* dest, size_t dest_len) {
    return png_extract_icc(static_cast<const uint8_t*>(src), src_len, static_cast<uint8_t*>(dest), dest_len);
}

int opencv_decoder_get_png_cicp(void* src, size_t src_len, uint8_t* primaries, uint8_t* transfer,
                                uint8_t* matrix, uint8_t* full_range) {
    uint8_t v[4];
    if (!src || !png_extract_cicp(static_cast<const uint8_t*>(src), src_len, v)) return 0;
    *primaries = v[0];
    *transfer = v[1];
    *matrix = v[2];
    *full_range = v[3];
    return 1;
}

static uint32_t crc32_bytes(const uint8_t* p, size_t n) {
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) {
        c ^= p[i];
        for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0xEDB88320u & (0u - (c & 1)));
    }
    return ~c;
}

// ref opencv.cpp:413-464: insert a 16-byte cICP chunk right after IHDR, in place.
size_t opencv_png_insert_cicp(void* png, size_t png_len, size_t png_cap, uint8_t primaries,
                              uint8_t transfer, uint8_t matrix, uint8_t full_range) {
    static const uint8_t sig[8] = {0x89, 0x50, 0x4E, 0x47, 0x0D, 0x0A, 0x1A, 0x0A};
    uint8_t* buf = static_cast<uint8_t*>(png);
    if (!buf || png_len < 8 + 12 || png_len + 16 > png_cap) return png_len;
    if (memcmp(buf, sig, 8) != 0 || memcmp(buf + 12, "IHDR", 4) != 0) return png_len;
    size_t insert_at = 8 + 12 + (size_t)be32(buf + 8);
    if (insert_at > png_len) return png_len;
    uint8_t chunk[16] = {0, 0, 0, 4, 'c', 'I', 'C', 'P', primaries, transfer, matrix, full_range};
    uint32_t crc = crc32_bytes(chunk + 4, 8);
    chunk[12] = (uint8_t)(crc >> 24);
    chunk[13] = (uint8_t)(crc >> 16);
    chunk[14] = (uint8_t)(crc >> 8);
    chunk[15] = (uint8_t)crc;
    memmove(buf + insert_at + 16, buf + insert_at, png_len - insert_at);
    memcpy(buf + insert_at, chunk, 16);
    return png_len + 16;
}

}  // extern "C"
