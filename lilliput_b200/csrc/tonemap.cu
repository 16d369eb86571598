// tonemap.cu -- HDR (PQ / HLG) pixels of 8-bit frames -> SDR BT.709, in place, on sm_90a.
//
// Replaces: tonemap_rgb_8u_inplace -> tonemap_rgb_to_sdr (ref color_info.cpp:112-236), which
// Framebuffer.TonemapToSDR (ref opencv.go:791-810) runs right after the decode of a source whose PNG cICP chunk
// (or AVIF colour box) signals a PQ or HLG transfer (ref ops.go:154-165, 511-517):
//   u8 / 255 -> EOTF (ST.2084 PQ or HLG) -> cv::TonemapReinhard(gamma 1.0, intensity 0.6, light_adapt 0.2,
//   color_adapt 0.3) -> 3x3 primaries matrix to BT.709 -> x 255, round to nearest, saturate.
// cv::TonemapReinhard is not a per-pixel map: it normalises the frame to [min, max] twice and uses the log-mean,
// log-min, log-max and the channel / grey means of the normalised frame -- global reductions inside ONE image
// (SURVEY 8(f)3).  Here: n frames of any sizes in one call, four passes, each ONE launch over the flat list of every
// frame's blocks (a frame is cut into blocks of 4096 pixels from its own width and height only); the first three each
// write one record per block and a fold launch (one block per frame) combines a frame's records in a fixed order.  No
// atomics: a frame's sums are bit-identical whether the call holds it alone or next to a thousand others, which lets the
// per-image path (n = 1) and the heterogeneous batch give the same bytes.  The EOTF is recomputed in every pass instead
// of keeping a 12-byte-per-pixel fp32 copy, so a pass reads 3-4 bytes per pixel and only the last one writes.  The
// scalar glue between the passes runs on the host in the reference's precisions (host and device powf / expf may differ
// in the last ulp): one D2H of the n records and one H2D of the n scalar sets per pass, three round trips per call.
// The arithmetic is fp32 like OpenCV's; the reference's own SIMD evaluation order differs in the last ulp, which shows
// as +-1 LSB on ~0.01 % of the samples (tests/test_gpu_tonemap.py states the tolerance; oracle.tonemap_to_sdr is the
// restatement pinned on oracle/_ref).
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "kernels.cuh"

namespace lp {

struct TmScalars {
    int transfer;                 // 16 = PQ, 18 = HLG, anything else = none
    float a1, b1;                 // first normalisation: im = lin * a1 + b1
    float map_key, intensity;     // Reinhard
    float glob[3];                // color_adapt * channel mean + (1 - color_adapt) * grey mean
    float a2, b2;                 // second normalisation
    int use_matrix;
    float m[9];
};
struct TmReduce {
    float mn, mx;                 // pass 1 / pass 3: min, max over all channels
    float lmn, lmx;               // pass 2: min / max of log(max(grey, 1e-4))
    double slog, sgray, sch[3];   // pass 2: sums
};

__device__ __forceinline__ float tm_pq(float x) {
    const float m1 = 0.1593017578125f, m2 = 78.84375f, c1 = 0.8359375f, c2 = 18.8515625f, c3 = 18.6875f;
    const float xp = powf(x, 1.0f / m2);
    const float num = fmaxf(xp - c1, 0.0f), den = c2 - c3 * xp;
    return powf(num / den, 1.0f / m1);
}
__device__ __forceinline__ float tm_hlg(float x) {
    const float a = 0.17883277f, b = 0.28466892f, c = 0.55991073f;
    return x <= 0.5f ? x * x / 3.0f : (expf((x - c) / a) + b) / 12.0f;
}
__device__ __forceinline__ float tm_eotf(int transfer, uint8_t v) {
    const float x = (float)v * (1.0f / 255.0f);
    return transfer == 16 ? tm_pq(x) : transfer == 18 ? tm_hlg(x) : x;
}

// the pre-normalisation Reinhard output of one pixel (ref: cv::TonemapReinhardImpl::process)
__device__ __forceinline__ void tm_reinhard(const TmScalars& s, const float im[3], float out[3]) {
    const float gray = im[0] * 0.299f + im[1] * 0.587f + im[2] * 0.114f;
    const float ca = 0.3f, la = 0.2f;
#pragma unroll
    for (int i = 0; i < 3; i++) {
        float adapt = ca * im[i] + (1.0f - ca) * gray;
        adapt = la * adapt + (1.0f - la) * s.glob[i];
        adapt = powf(s.intensity * adapt, s.map_key);
        out[i] = im[i] * (1.0f / (adapt + im[i]));
    }
}

// One block of a pass: kTmPerThread pixels per thread, kTmThreads apart, from the frame's pixel
// (blockIdx.x - block0) * kTmBlockPixels in row-major order.  Which pixels a block covers and the order in which its
// record is combined depend on the frame's own width and height only.
constexpr int kTmThreads = 256, kTmPerThread = 16;
constexpr uint32_t kTmBlockPixels = kTmThreads * kTmPerThread;

struct TmJob {
    uint8_t* px;
    unsigned long long step;
    int w, h, channels;
    uint32_t block0, nblocks;  // the frame's blocks in the flat block list of the call
};

__device__ __forceinline__ void tm_identity(TmReduce& r) {
    r.mn = r.lmn = FLT_MAX;
    r.mx = r.lmx = -FLT_MAX;
    r.slog = r.sgray = r.sch[0] = r.sch[1] = r.sch[2] = 0.0;
}
__device__ __forceinline__ void tm_combine(TmReduce& r, const TmReduce& o) {
    r.mn = fminf(r.mn, o.mn);
    r.mx = fmaxf(r.mx, o.mx);
    r.lmn = fminf(r.lmn, o.lmn);
    r.lmx = fmaxf(r.lmx, o.lmx);
    r.slog += o.slog;
    r.sgray += o.sgray;
#pragma unroll
    for (int i = 0; i < 3; i++) r.sch[i] += o.sch[i];
}

// the block's records -> out, in a fixed order: a butterfly inside every warp, then warps 0..7 in turn by thread 0.
// SUMS = false: only mn / mx are live (the other fields of `out` are the identity's).
template <bool SUMS>
__device__ __forceinline__ void tm_block_reduce(TmReduce r, TmReduce* out) {
    __shared__ TmReduce warps[kTmThreads / 32];
    for (int o = 16; o; o >>= 1) {
        r.mn = fminf(r.mn, __shfl_xor_sync(0xffffffffu, r.mn, o));
        r.mx = fmaxf(r.mx, __shfl_xor_sync(0xffffffffu, r.mx, o));
        if constexpr (SUMS) {
            r.lmn = fminf(r.lmn, __shfl_xor_sync(0xffffffffu, r.lmn, o));
            r.lmx = fmaxf(r.lmx, __shfl_xor_sync(0xffffffffu, r.lmx, o));
            r.slog += __shfl_xor_sync(0xffffffffu, r.slog, o);
            r.sgray += __shfl_xor_sync(0xffffffffu, r.sgray, o);
#pragma unroll
            for (int i = 0; i < 3; i++) r.sch[i] += __shfl_xor_sync(0xffffffffu, r.sch[i], o);
        }
    }
    if ((threadIdx.x & 31) == 0) warps[threadIdx.x >> 5] = r;
    __syncthreads();
    if (threadIdx.x == 0) {
        TmReduce t = warps[0];
        for (int k = 1; k < kTmThreads / 32; k++) tm_combine(t, warps[k]);
        *out = t;
    }
}

// the frame whose blocks hold flat block b: the last job with block0 <= b (every job has at least one block)
__device__ __forceinline__ int tm_job_of(const TmJob* jobs, int n, uint32_t b) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (jobs[mid].block0 <= b) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// PASS 1: min / max of the EOTF; 2: log-mean, grey and channel sums; 3: min / max of the Reinhard output (one record
// per block into part); 4: the final map, in place
template <int PASS>
__global__ void __launch_bounds__(kTmThreads) tonemap_pass_kernel(const TmJob* jobs, int n, const TmScalars* scal, TmReduce* part) {
    const TmJob& J = jobs[tm_job_of(jobs, n, blockIdx.x)];
    const TmScalars& s = scal[&J - jobs];
    const int w = J.w, ch = J.channels;
    const size_t npx = (size_t)w * J.h;
    size_t p = (size_t)(blockIdx.x - J.block0) * kTmBlockPixels + threadIdx.x;
    uint32_t y = (uint32_t)(p / (uint32_t)w), x = (uint32_t)(p - (size_t)y * w);
    const uint32_t dy = kTmThreads / w, dx = kTmThreads % w;  // the step of kTmThreads pixels in rows and columns
    TmReduce r;
    tm_identity(r);
    for (int j = 0; j < kTmPerThread && p < npx; j++) {
        uint8_t* q = J.px + (size_t)y * J.step + (size_t)x * ch;
        float lin[3];
#pragma unroll
        for (int i = 0; i < 3; i++) lin[i] = tm_eotf(s.transfer, q[i]);
        p += kTmThreads;
        y += dy;
        x += dx;
        if (x >= (uint32_t)w) {
            x -= w;
            y++;
        }
        if constexpr (PASS == 1) {
            r.mn = fminf(r.mn, fminf(fminf(lin[0], lin[1]), lin[2]));
            r.mx = fmaxf(r.mx, fmaxf(fmaxf(lin[0], lin[1]), lin[2]));
        } else {
        float im[3];
#pragma unroll
        for (int i = 0; i < 3; i++) im[i] = lin[i] * s.a1 + s.b1;
        if constexpr (PASS == 2) {
            const float gray = im[0] * 0.299f + im[1] * 0.587f + im[2] * 0.114f;
            const float lg = logf(fmaxf(gray, 1e-4f));
            r.lmn = fminf(r.lmn, lg);
            r.lmx = fmaxf(r.lmx, lg);
            r.slog += (double)lg;
            r.sgray += (double)gray;
#pragma unroll
            for (int i = 0; i < 3; i++) r.sch[i] += (double)im[i];
        } else {
        float out[3];
        tm_reinhard(s, im, out);
        if constexpr (PASS == 3) {
            r.mn = fminf(r.mn, fminf(fminf(out[0], out[1]), out[2]));
            r.mx = fmaxf(r.mx, fmaxf(fmaxf(out[0], out[1]), out[2]));
        } else {
        float t[3];
#pragma unroll
        for (int i = 0; i < 3; i++) t[i] = out[i] * s.a2 + s.b2;
        float c[3] = {t[0], t[1], t[2]};
        if (s.use_matrix) {
#pragma unroll
            for (int k = 0; k < 3; k++) c[k] = s.m[k * 3] * t[0] + s.m[k * 3 + 1] * t[1] + s.m[k * 3 + 2] * t[2];
        }
        if (s.transfer == 8) {  // linear light: display gamma (ref color_info.cpp:226-228); PQ / HLG already carry theirs
#pragma unroll
            for (int i = 0; i < 3; i++) c[i] = powf(c[i], 1.0f / 2.2f);
        }
#pragma unroll
        for (int i = 0; i < 3; i++) {
            const int v = __float2int_rn(c[i] * 255.0f);
            q[i] = (uint8_t)min(max(v, 0), 255);
        }
        // alpha, when present, is untouched (ref color_info.cpp:262-267)
        }
        }
        }
    }
    if constexpr (PASS != 4) tm_block_reduce<PASS == 2>(r, part + blockIdx.x);
}

// one block per frame: the frame's block records, in block order per thread and then tm_block_reduce's order -> red[f]
__global__ void __launch_bounds__(kTmThreads) tonemap_fold_kernel(const TmJob* jobs, const TmReduce* part, TmReduce* red) {
    const TmJob& J = jobs[blockIdx.x];
    TmReduce r;
    tm_identity(r);
    for (uint32_t b = threadIdx.x; b < J.nblocks; b += kTmThreads) tm_combine(r, part[J.block0 + b]);
    tm_block_reduce<true>(r, red + blockIdx.x);
}

static void normalise_coeffs(float mn, float mx, float* a, float* b) {  // cv::TonemapImpl::process: (src - min) / (max - min)
    if ((double)mx - (double)mn > DBL_EPSILON) {
        const double alpha = 1.0 / ((double)mx - (double)mn);
        *a = (float)alpha;
        *b = (float)(-(double)mn * alpha);
    } else {
        *a = 1.0f;
        *b = 0.0f;
    }
}

static bool tm_takes(const TmFrame& f) {  // the reference returns silently on anything else
    return f.w > 0 && f.h > 0 && (f.channels == 3 || f.channels == 4);
}
static uint32_t tm_blocks(const TmFrame& f) { return (uint32_t)ceil_div((size_t)f.w * f.h, (size_t)kTmBlockPixels); }

size_t tonemap_batch_scratch_bytes(const TmFrame* frames, int n) {
    size_t jobs = 0, blocks = 0;
    for (int k = 0; k < n; k++)
        if (tm_takes(frames[k])) {
            jobs++;
            blocks += tm_blocks(frames[k]);
        }
    if (!jobs) return 0;
    return round_up(jobs * sizeof(TmJob), (size_t)256) + round_up(jobs * sizeof(TmScalars), (size_t)256) +
           round_up(jobs * sizeof(TmReduce), (size_t)256) + round_up(blocks * sizeof(TmReduce), (size_t)256);
}

int tonemap_batch_launch(const TmFrame* frames, int n, void* d_scratch, size_t scratch_bytes, cudaStream_t st) {
    std::vector<TmJob> jobs;
    std::vector<const TmFrame*> src;
    uint32_t blocks = 0;
    for (int k = 0; k < n; k++) {
        const TmFrame& f = frames[k];
        if (!tm_takes(f)) continue;
        jobs.push_back(TmJob{f.px, (unsigned long long)f.step, f.w, f.h, f.channels, blocks, tm_blocks(f)});
        src.push_back(&f);
        blocks += jobs.back().nblocks;
    }
    const int m = (int)jobs.size();
    if (!m) return LP_OK;
    if (!d_scratch || scratch_bytes < tonemap_batch_scratch_bytes(frames, n)) return LP_ERR_BUF_TOO_SMALL;
    uint8_t* sp = static_cast<uint8_t*>(d_scratch);
    auto take = [&](size_t bytes) {
        uint8_t* p = sp;
        sp += round_up(bytes, (size_t)256);
        return p;
    };
    TmJob* d_jobs = reinterpret_cast<TmJob*>(take(m * sizeof(TmJob)));
    TmScalars* d_scal = reinterpret_cast<TmScalars*>(take(m * sizeof(TmScalars)));
    TmReduce* d_red = reinterpret_cast<TmReduce*>(take(m * sizeof(TmReduce)));
    TmReduce* d_part = reinterpret_cast<TmReduce*>(take((size_t)blocks * sizeof(TmReduce)));
    std::vector<TmScalars> s((size_t)m);
    std::vector<TmReduce> r((size_t)m);
    memset(s.data(), 0, s.size() * sizeof(TmScalars));
    for (int k = 0; k < m; k++) s[k].transfer = src[k]->transfer;
    LP_CUDA_OK(cudaMemcpyAsync(d_jobs, jobs.data(), m * sizeof(TmJob), cudaMemcpyHostToDevice, st));
    // one pass, its fold, and the per-frame records home
    auto reduce = [&](auto pass) {
        if (cudaMemcpyAsync(d_scal, s.data(), m * sizeof(TmScalars), cudaMemcpyHostToDevice, st) != cudaSuccess) return false;
        pass<<<blocks, kTmThreads, 0, st>>>(d_jobs, m, d_scal, d_part);
        tonemap_fold_kernel<<<m, kTmThreads, 0, st>>>(d_jobs, d_part, d_red);
        g_launches += 2;
        return cudaGetLastError() == cudaSuccess &&
               cudaMemcpyAsync(r.data(), d_red, m * sizeof(TmReduce), cudaMemcpyDeviceToHost, st) == cudaSuccess &&
               cudaStreamSynchronize(st) == cudaSuccess;
    };
    if (!reduce(tonemap_pass_kernel<1>)) return LP_ERR_CUDA;
    for (int k = 0; k < m; k++) normalise_coeffs(r[k].mn, r[k].mx, &s[k].a1, &s[k].b1);
    if (!reduce(tonemap_pass_kernel<2>)) return LP_ERR_CUDA;
    for (int k = 0; k < m; k++) {
        const double total = (double)jobs[k].w * jobs[k].h;
        const float log_mean = (float)(r[k].slog / total);
        const double log_min = r[k].lmn, log_max = r[k].lmx;
        const float key = (float)((log_max - (double)log_mean) / (log_max - log_min));
        s[k].map_key = 0.3f + 0.7f * powf(key, 1.4f);
        s[k].intensity = expf(-0.6f);
        const float gray_mean = (float)(r[k].sgray / total);
        for (int i = 0; i < 3; i++) s[k].glob[i] = 0.3f * (float)(r[k].sch[i] / total) + (1.0f - 0.3f) * gray_mean;
    }
    if (!reduce(tonemap_pass_kernel<3>)) return LP_ERR_CUDA;
    // ref color_info.cpp:160-197: primaries -> BT.709 (channel order as stored; unknown primaries pass through)
    static const float bt2020[9] = {1.6605f, -0.5876f, -0.0728f, -0.1246f, 1.1329f, -0.0083f, -0.0182f, -0.1006f, 1.1187f};
    static const float p3[9] = {1.2249f, -0.2247f, -0.0002f, -0.0420f, 1.0419f, 0.0001f, -0.0197f, 0.0754f, 0.9443f};
    static const float bt601[9] = {1.0440f, -0.0440f, 0.0000f, -0.0000f, 1.0000f, 0.0000f, 0.0000f, 0.0000f, 1.0000f};
    static const float xyz[9] = {1.0569715f, -0.2039770f, 0.0556301f, 0.0415551f, 1.8759675f, -0.9692436f, -0.4986108f, -1.5373832f, 3.2409699f};
    for (int k = 0; k < m; k++) {
        normalise_coeffs(r[k].mn, r[k].mx, &s[k].a2, &s[k].b2);
        const int pr = src[k]->primaries;
        const float* mat = pr == 9 ? bt2020 : (pr == 12 || pr == 11) ? p3 : pr == 6 ? bt601 : pr == 10 ? xyz : nullptr;
        s[k].use_matrix = mat != nullptr;
        if (mat) memcpy(s[k].m, mat, sizeof(s[k].m));
    }
    LP_CUDA_OK(cudaMemcpyAsync(d_scal, s.data(), m * sizeof(TmScalars), cudaMemcpyHostToDevice, st));
    tonemap_pass_kernel<4><<<blocks, kTmThreads, 0, st>>>(d_jobs, m, d_scal, d_part);
    g_launches++;
    return cudaGetLastError() == cudaSuccess ? LP_OK : LP_ERR_CUDA;
}

int tonemap_to_sdr_launch(uint8_t* d_px, size_t step, int channels, int w, int h, int transfer, int primaries, cudaStream_t st) {
    const TmFrame f{d_px, step, w, h, channels, transfer, primaries};
    const size_t bytes = tonemap_batch_scratch_bytes(&f, 1);
    if (!d_px || !bytes) return LP_OK;
    void* scratch = nullptr;
    LP_CUDA_OK(cudaMallocAsync(&scratch, bytes, st));
    const int rc = tonemap_batch_launch(&f, 1, scratch, bytes, st);
    cudaFreeAsync(scratch, st);
    return rc;
}

}  // namespace lp
