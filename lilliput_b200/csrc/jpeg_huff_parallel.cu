// jpeg_huff_parallel.cu -- intra-image parallel Huffman decoding of a baseline JPEG scan that has
// NO restart markers (BASELINE config 2's primary corpus), one CTA per image.
//
// Replaces the bit-serial part of libjpeg-turbo's jdhuff.c that cv::ImageDecoder::readData runs for
// the reference (ref opencv.cpp:166-171).  Results (quantised coefficients) are identical to a
// sequential decode; only the schedule differs.
//
// JPEG's Huffman code self-synchronises: a decoder started at an arbitrary bit falls back onto
// true codeword boundaries (and the true position inside the MCU) after a few dozen symbols.  So
//   1. jpeg_unstuff_kernel   removes FF00 byte stuffing and finds the end of the entropy-coded
//                            segment, giving a plain bit string (block scan + compaction);
//   2. jpeg_huff_sync_kernel cuts it into 1024-bit subsequences; every thread decodes its own from a
//                            guessed state, then re-decodes from its left neighbour's exit state
//                            until no exit state changes (a fixed point that is exact by induction
//                            from subsequence 0).  A prefix sum of the per-subsequence coefficient
//                            counts gives every subsequence its absolute output position, and one
//                            last decode writes whole coefficient blocks (zero-filled by the thread
//                            that opens them) and DC differences;
//   3. the same kernel then turns DC differences into DC values with a per-component prefix sum.
// (Scheme after Weissenberger & Schmidt, "Accelerating JPEG Decompression on GPUs", restated from
// the published description.)
#include <cstdlib>

#include "common.cuh"
#include "kernels.cuh"

namespace lp {

// Diagnostics: SM cycles (clock64, thread 0 of every CTA) spent in the phases of the sync kernels, summed over the
// CTAs since the last reset: [0] table set-up, [1] guess pass, [2] synchronisation rounds, [3] prefix sum + write
// pass, [4] DC pass, [5] CTAs.  Four clock reads and five atomics per CTA.  Not cycles: [6] bits decoded in the
// synchronisation rounds, [7] bits decoded in the guess pass (a shared-memory atomic per decode, two atomics per CTA).
__device__ unsigned long long g_huff_phase[8];
#define LP_PHASE_MARK(k)                                             \
    do {                                                             \
        if (threadIdx.x == 0) {                                      \
            const long long now_ = clock64();                        \
            atomicAdd(&g_huff_phase[k], (unsigned long long)(now_ - s_tphase)); \
            s_tphase = now_;                                         \
        }                                                            \
    } while (0)

constexpr uint32_t kMinSubBits = 1024;  // shortest subsequence (bits); scratch is sized for this
// Subsequences per thread and pass.  Synchronising the position inside the MCU (not just the
// codeword boundary) takes several hundred symbols, so short subsequences need ~10 re-decode rounds;
// sizing them so that one pass is exactly kSubPerThread full rounds of the CTA cuts that to ~2
// (measured: 10.9 rounds at 1024 bits, 1.9 at one subsequence per thread of 512).
constexpr uint32_t kSubPerThread = 1;
// Threads (= subsequences per pass) of the sync kernel.  384 threads at 4 CTAs/SM keep as many threads per SM as 512
// at 3 within the same 40 registers, and the longer subsequences (~9.3 kbit at 1080p) need fewer rounds (1.2 instead
// of 1.9 at BASELINE config 2): measured 5 % less entropy-stage time on the H100 (DESIGN.md §5).
#ifndef LP_HUFF_THREADS
#define LP_HUFF_THREADS 384
#endif
constexpr int kHuffThreads = LP_HUFF_THREADS;
constexpr int kUnstuffThreads = 512;  // the unstuff kernel: 8 KB tiles of 16-byte vectors

__constant__ uint8_t c_zigzag_p[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                       12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                       35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                       58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// ------------------------------------------------------------------ block scan helper

template <int THREADS>
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* total, uint32_t* warp_sums) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        uint32_t s = lane < THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        if (lane < THREADS / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    const uint32_t base = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[THREADS / 32 - 1];
    __syncthreads();
    return base + inc - v;
}

// ------------------------------------------------------------------ 1. unstuff

// clean[] gets the entropy-coded bytes with every "FF 00" reduced to "FF"; the segment ends at the
// first FF that is followed by anything else (a marker).  clean_len[img] = bytes written.
// One CTA per image, 8 KB tiles: every thread takes one aligned 16-byte vector, learns its
// neighbours' edge bytes by shuffle, a block scan places the kept bytes in a shared staging
// tile, and the tile leaves as 4-byte words (stuffed bytes are ~0.4 % of the stream, so this is a
// copy that occasionally closes a gap).  The marker search rides along: only the tile that holds
// the marker pays for the second look.
__global__ void __launch_bounds__(kUnstuffThreads)
    jpeg_unstuff_kernel(JpegDecodeItem* items, const uint8_t* scan, uint8_t* clean) {
    __shared__ uint32_t warp_sums[kUnstuffThreads / 32];
    __shared__ uint32_t s_end;
    __shared__ __align__(16) uint8_t stage[kUnstuffThreads * 16 + 16];
    JpegDecodeItem& it = items[blockIdx.x];
    const uint8_t* src = scan + it.scan_off;
    const uint32_t len = it.scan_len;
    uint8_t* dst = clean + it.clean_off;
    const int tid = threadIdx.x, lane = tid & 31;
    // restart-interval-parallel path (jpeg_decode.cu): clean_len holds its interval count; multi-scan items: the
    // serial multi-scan kernel
    if (it.restart_interval != 0 || it.nscans != 0) return;
    if (it.status != 0) {
        if (tid == 0) it.clean_len = 0;
        return;
    }
    if (tid == 0) s_end = len;
    __syncthreads();
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 15);
    const uint8_t* abase = src - mis;  // 16-byte aligned; the bytes before src belong to the same upload
    uint32_t carry = 0;
    uint32_t end = len;
    constexpr uint32_t kTile = kUnstuffThreads * 16;
    for (uint32_t t0 = 0; t0 < mis + end; t0 += kTile) {
        const uint32_t aoff = t0 + (uint32_t)tid * 16;      // offset from abase
        const int64_t i0 = (int64_t)aoff - (int64_t)mis;    // stream index of this thread's first byte
        uint4 w = make_uint4(0, 0, 0, 0);
        if (aoff < mis + len + 16) w = *reinterpret_cast<const uint4*>(abase + aoff);
        // neighbours' edge bytes
        uint32_t prev = __shfl_up_sync(0xffffffffu, w.w >> 24, 1);
        uint32_t next = __shfl_down_sync(0xffffffffu, w.x & 0xffu, 1);
        if (lane == 0) prev = i0 > 0 ? src[i0 - 1] : 0;
        if (lane == 31) next = (i0 + 16 < (int64_t)len) ? src[i0 + 16] : 0xD9u;
        // Per-byte classification, four bytes per instruction (SIMD-in-register compares):
        //   stuffed zero = 00 preceded by FF (dropped); marker = FF followed by anything but 00.
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
        uint32_t m00[4], mff[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            m00[q] = __vcmpeq4(ws[q], 0u);
            mff[q] = __vcmpeq4(ws[q], 0xFFFFFFFFu);
        }
        const uint32_t prev_ff = prev == 0xFFu ? 0xFFu : 0u, next_00 = next == 0x00u ? 0xFF000000u : 0u;
        uint32_t drop16 = 0, mark16 = 0;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint32_t pff = (mff[q] << 8) | (q ? mff[q - 1] >> 24 : prev_ff);            // byte before is FF
            const uint32_t n00 = (m00[q] >> 8) | (q < 3 ? m00[q + 1] << 24 : next_00);        // byte after is 00
            const uint32_t d = m00[q] & pff, mk = mff[q] & ~n00;
            drop16 |= (((d & 0x01010101u) * 0x01020408u) >> 24 & 0xFu) << (4 * q);           // byte masks -> 4 bits
            mark16 |= (((mk & 0x01010101u) * 0x01020408u) >> 24 & 0xFu) << (4 * q);
        }
        // bytes of this vector that lie inside the stream [0, len)
        const int64_t lo = -i0, hi = (int64_t)len - i0;  // valid k: lo <= k < hi
        uint32_t valid16 = 0xFFFFu;
        if (lo > 0) valid16 &= lo >= 16 ? 0u : (0xFFFFu << lo);
        if (hi < 16) valid16 &= hi <= 0 ? 0u : (0xFFFFu >> (16 - hi));
        // the first byte of the stream has no predecessor (whatever sits in memory before it)
        if (lo >= 0 && lo < 16) drop16 &= ~(1u << (int)lo);
        // the last byte of the stream counts as followed by a marker byte
        if (hi >= 1 && hi <= 16) {
            const int kl = (int)hi - 1;
            if (((ws[kl >> 2] >> (8 * (kl & 3))) & 0xFFu) == 0xFFu) mark16 |= 1u << kl;
        }
        mark16 &= valid16;
        const uint32_t my_marker = mark16 ? (uint32_t)(i0 + (__ffs(mark16) - 1)) : 0xFFFFFFFFu;
        if (__syncthreads_or(my_marker != 0xFFFFFFFFu)) {
            if (my_marker != 0xFFFFFFFFu) atomicMin(&s_end, my_marker);
            __syncthreads();
            end = s_end;
        }
        uint32_t keep = valid16 & ~drop16;
        {
            const int64_t he = (int64_t)end - i0;  // bytes at or after the marker are dropped
            if (he < 16) keep &= he <= 0 ? 0u : (0xFFFFu >> (16 - he));
        }
        uint8_t bsrc[16];
#pragma unroll
        for (int k = 0; k < 16; k++) bsrc[k] = (uint8_t)(ws[k >> 2] >> (8 * (k & 3)));
        const uint32_t cnt = __popc(keep);
        uint32_t total;
        const uint32_t ex = block_excl_scan<kUnstuffThreads>(cnt, &total, warp_sums);
        {
            uint32_t o = ex;
#pragma unroll
            for (int k = 0; k < 16; k++)
                if (keep & (1u << k)) stage[o++] = bsrc[k];
        }
        __syncthreads();
        // staged tile -> dst[carry, carry + total): bytes up to 4-byte alignment, words, tail bytes
        uint8_t* d = dst + carry;
        const uint32_t head = min(total, (uint32_t)((4 - (reinterpret_cast<uintptr_t>(d) & 3)) & 3));
        const uint32_t nwords = (total - head) >> 2;
        const uint32_t tail0 = head + (nwords << 2);
        if ((uint32_t)tid < head) d[tid] = stage[tid];
        for (uint32_t j = tid; j < nwords; j += kUnstuffThreads) {
            const uint8_t* q = stage + head + 4 * j;
            *reinterpret_cast<uint32_t*>(d + head + 4 * j) = (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
        }
        if (tail0 + tid < total) d[tail0 + tid] = stage[tail0 + tid];
        carry += total;
        __syncthreads();
    }
    if (tid == 0) it.clean_len = carry;
    // zero padding so the 8-byte window loads past the end read defined data
    for (uint32_t k = tid; k < 32; k += kUnstuffThreads) dst[carry + k] = 0;
}

// ------------------------------------------------------------------ 2. sync + write

struct alignas(8) SubState {
    uint32_t p;      // absolute bit position of the first symbol that starts after this subsequence
    uint32_t phase;  // (block-in-MCU << 6) | zig-zag index expected at p
};

constexpr int kDcBits = 9, kAcBits = kHuffAcLookBits;  // a longer code in ANY lane sends the whole warp through the slow walk

// Per-CTA decode tables.  DC tables are indexed by the next 9 bits, AC tables by the next 11
// (longer codes -- well under 0.1 % of symbols with the Annex-K tables -- take the canonical walk).
struct HuffShared {
    uint16_t dc_look[4][1 << kDcBits];  // (len << 8) | symbol, 0 = longer code
    uint16_t ac_look[4][1 << kAcBits];  // bit 15 set: AC code longer than kAcBits -> ac_sub[entry & 0x7FFF]
    uint16_t ac_sub[4 * kHuffLongPrefixes][16];  // next 4 bits -> (len << 8) | symbol, 0 = not a codeword
    int32_t maxcode[8][18];
    int32_t valoffset[8][17];
    uint8_t vals[8][256];
    uint8_t zz[64];
    uint8_t blk_dc[16], blk_ac[16];  // table id per block-in-MCU
    uint8_t blk_comp[16], blk_bx[16], blk_by[16];
    // The usual layout -- the first n_first blocks of an MCU (component 0) share one DC/AC table pair
    // and all the others share another -- lets the symbol loop pick its lookahead table with a
    // compare + select instead of a table walk on every block boundary.
    uint32_t two_tables, n_first;
    uint32_t dcb_first, dcb_rest, acb_first, acb_rest;  // shared-memory byte addresses
};

// MSB-first bit reader over the unstuffed string: the two 32-bit words the next symbol can touch
// (a code is at most 16 bits, its value bits at most 15) plus a bit offset, so a peek is one funnel
// shift and a skip one add; a third word is always in flight (its load is issued ~32 bits early).
struct BitWin {
    const uint32_t* w;  // word after `nextw`
    uint32_t w0, w1;    // big-endian words; the next bit is bit (31 - bo) of w0
    uint32_t nextw;     // prefetched, still little-endian
    uint32_t bo;        // 0..31 after refill()
    __device__ __forceinline__ void init(const uint8_t* s, uint32_t p) {
        const uint32_t* base = reinterpret_cast<const uint32_t*>(s) + (p >> 5);
        w0 = __byte_perm(base[0], 0, 0x0123);
        w1 = __byte_perm(base[1], 0, 0x0123);
        nextw = base[2];
        w = base + 3;
        bo = p & 31;
    }
    __device__ __forceinline__ void refill() {
        if (bo >= 32) {
            w0 = w1;
            w1 = __byte_perm(nextw, 0, 0x0123);
            nextw = *w++;
            bo -= 32;
        }
    }
    __device__ __forceinline__ uint32_t peek() const { return __funnelshift_l(w1, w0, bo); }  // next 32 bits
    __device__ __forceinline__ void skip(int n) { bo += n; }  // n <= 31 between refills
};

// Decode symbols that START in [p, limit).  Returns the exit state and the number of coefficient
// slots consumed.  WRITE: store coefficients (DC slot receives the DC *difference*) starting at
// absolute slot `pos`.
//
// WRITE stores whole blocks: the coefficient array is not cleared beforehand.  The span that decodes
// a block's DC symbol owns that block: it zero-fills the block's 128 bytes before its first
// coefficient store and, if the block is still open at `limit`, decodes on past `limit` (at most to
// `end_bits`, the end of the stream) until the block closes.  A span that starts inside a block
// (z > 0) stores nothing until that block closes; its owner writes it.  So every block is written by
// one thread and no ordering between threads is needed.
template <bool WRITE, bool TWO>
__device__ __forceinline__ void decode_span_t(const HuffShared& hs, const uint8_t* s, uint32_t& p, uint32_t limit,
                                            uint32_t end_bits, uint32_t& phase, uint32_t& nslots, int nb,
                                            uint64_t pos, uint64_t total_slots, const JpegDecodeItem* it,
                                            int16_t* coef, int16_t* dcdiff, int* status) {
    uint32_t blk = phase >> 6, z = phase & 63;
    const uint32_t z_start = z;
    uint32_t closed = 0;                       // blocks completed in this span
    int32_t bits_left = (int32_t)(limit - p);  // symbols that START before `limit` belong to this span
    // WRITE: an owned block that is still open at `limit` is decoded to its end, but not past the stream
    const int32_t own_floor = (int32_t)limit - (int32_t)end_bits;
    bool own = z_start == 0;  // WRITE: the current block was opened by this span
    BitWin bw;
    bw.init(s, p);
    // WRITE: running block position.  Coefficients of the region of interest are stored in MCU (scan)
    // order -- block b of ROI MCU (rx, ry) at ((ry * roi_mcx + rx) * nb + b) * 64 -- so closing a block
    // is "advance by 64"; only an MCU change (one close in nb) looks at the ROI again.
    int16_t* dstblk = nullptr;  // current block's coefficients; meaningful only while `inside`
    bool inside = false;        // the current MCU lies in the region of interest
    int16_t* dcp = nullptr;     // DC difference slot of the current block (all blocks, MCU order)
    int mx = 0, my = 0;
    uint32_t blocks_left = 0;
    bool bad = false;
    int16_t* coef_base = nullptr;
    const uint32_t zzb = (uint32_t)__cvta_generic_to_shared(&hs.zz[0]);
    auto set_mcu = [&]() {  // first block of MCU (mx, my)
        const int rmx = mx - it->roi_mx0, rmy = my - it->roi_my0, rcx = it->roi_mcx;
        inside = (unsigned)rmx < (unsigned)rcx && (unsigned)rmy < (unsigned)it->roi_mcy;
        dstblk = coef_base + ((size_t)rmy * rcx + rmx) * ((size_t)nb * 64);
    };
    if (WRITE) {
        if (pos >= total_slots) {
            nslots = 0;
            return;
        }
        blocks_left = (uint32_t)((total_slots - pos + z_start) >> 6);  // counted from the start of the current block
        coef_base = coef + it->coef_off;
        const uint32_t mcu = (uint32_t)((pos >> 6) / (uint32_t)nb);
        const uint32_t mcus_x = (uint32_t)it->mcus_x;
        mx = (int)(mcu % mcus_x);
        my = (int)(mcu / mcus_x);
        set_mcu();
        dstblk += blk * 64;
        dcp = dcdiff + (pos >> 6);
    }
    // shared-memory byte addresses of the current block's lookahead tables
    const uint32_t n_first = hs.n_first, dcbF = hs.dcb_first, dcbR = hs.dcb_rest, acbF = hs.acb_first, acbR = hs.acb_rest;
    uint32_t dcb, acb;
    auto set_tables = [&]() {
        if (TWO) {
            dcb = blk < n_first ? dcbF : dcbR;
            acb = blk < n_first ? acbF : acbR;
        } else {
            dcb = (uint32_t)__cvta_generic_to_shared(&hs.dc_look[hs.blk_dc[blk]][0]);
            acb = (uint32_t)__cvta_generic_to_shared(&hs.ac_look[hs.blk_ac[blk]][0]);
        }
    };
    set_tables();
    // The symbol step uses selects instead of branches: lanes of a warp sit at unrelated places of
    // unrelated subsequences, so every branch here would be a divergent one.  Coefficient slots are
    // not counted per symbol: slots = 64 * blocks closed + z_end - z_start.
    while (bits_left > 0 || (WRITE && own && z != 0 && bits_left > own_floor)) {
        bw.refill();
        const uint32_t top = bw.peek();
        const bool isdc = z == 0;
        const uint32_t idx = isdc ? (top >> (32 - kDcBits)) : (top >> (32 - kAcBits));
        int e;
        asm volatile("ld.shared.s16 %0, [%1];" : "=r"(e) : "r"((isdc ? dcb : acb) + idx * 2u));
        if (__builtin_expect(e <= 0, 0)) {  // longer than the lookahead (rare)
            if (e < 0) {
                // AC code of 13..16 bits: its prefix has a second-level table indexed by the next 4 bits
                e = hs.ac_sub[e & 0x7FFF][(top >> (32 - kAcBits - 4)) & 15u];
            } else {
                // canonical walk: DC codes past the lookahead, AC prefixes without a second-level table
                const int t = isdc ? hs.blk_dc[blk] : 4 + hs.blk_ac[blk];
                int len = (isdc ? kDcBits : kAcBits) + 1;
                int code = (int)(top >> (32 - len));
                while (len <= 16 && code > hs.maxcode[t][len]) {
                    len++;
                    code = (int)(top >> (32 - len));
                }
                if (len <= 16) e = (len << 8) | hs.vals[t][(code + hs.valoffset[t][len]) & 0xFF];
            }
            if (e == 0) {  // not a codeword: a wrong guess, or a corrupt stream
                if (WRITE) {
                    *status = -3;
                    break;
                }
                bw.skip(1);
                bits_left -= 1;
                continue;
            }
        }
        const int len = e >> 8, sym = e & 0xFF;
        const uint32_t r = (uint32_t)sym >> 4, sz = (uint32_t)sym & 15;
        const bool ez = (sz == 0) && !isdc;  // EOB or ZRL (DC symbols have r == 0 and are values)
        // slots this symbol advances: value r+1, ZRL 16, EOB "to the end"; reaching or passing 64
        // closes the block (a ZRL or run that would leave the block ends it, as libjpeg does)
        const uint32_t adv = ez ? (r == 15 ? 16u : 64u) : r + 1;
        const uint32_t zt = z + adv;
        const int used = len + (ez ? 0 : (int)sz);
        if (WRITE) {
            // value, destination and store without a branch: lanes sit in unrelated symbols
            const uint32_t t2 = top << len;
            const uint32_t raw = __funnelshift_l(t2, 0u, sz);  // next sz bits (0 when sz == 0)
            const int val = (int)raw + ((int)t2 >= 0 ? (int)((0xFFFFFFFFu << sz) + 1u) : 0);  // T.81 F.2.2.1 EXTEND
            uint32_t zi;
            asm volatile("ld.shared.u8 %0, [%1];" : "=r"(zi) : "r"(zzb + ((zt - 1u) & 63u)));
            int16_t* const where = isdc ? dcp : dstblk + zi;  // DC difference: every block; AC: inside the ROI
            const bool inblk = zt <= 64;
            bad |= !ez && !inblk;  // coefficient index past 63: corrupt data
            if (isdc && inside) {  // opening a block (z == 0 implies own): clear it before its AC stores
                uint4* const q = reinterpret_cast<uint4*>(dstblk);
#pragma unroll
                for (int k = 0; k < 8; k++) q[k] = make_uint4(0, 0, 0, 0);
            }
            if (!ez && inblk && own && (isdc || inside)) *where = (int16_t)val;
        }
        bw.skip(used);
        bits_left -= used;
        const bool fin = zt >= 64;  // block finished
        z = fin ? 0u : zt;
        if (WRITE) own |= fin;
        if (!WRITE) {
            // lanes sit at unrelated places, so SOME lane closes a block in nearly every iteration: keep the
            // bookkeeping to selects instead of a branch the whole warp would walk through
            closed += fin ? 1u : 0u;
            const uint32_t nxt = blk + 1 == (uint32_t)nb ? 0u : blk + 1;
            blk = fin ? nxt : blk;
            set_tables();
        } else if (fin) {
            closed++;
            blk++;
            dstblk += 64;
            if (blk == (uint32_t)nb) {
                blk = 0;
                if (++mx == it->mcus_x) {
                    mx = 0;
                    my++;
                }
                set_mcu();
            }
            set_tables();
            if (--blocks_left == 0) break;  // every MCU produced: the rest is padding
            dcp++;
        }
    }
    if (WRITE && bad) *status = -3;
    p = limit - (uint32_t)bits_left;  // bits_left <= 0 here unless the stream ended early
    phase = (blk << 6) | z;
    nslots = closed * 64 + z - z_start;
}

// Two copies of the symbol loop: the usual two-table-pair layout selects its lookahead tables with a
// compare, anything else looks them up per block.  hs.two_tables is uniform across the CTA.
template <bool WRITE>
__device__ __forceinline__ void decode_span(const HuffShared& hs, const uint8_t* s, uint32_t& p, uint32_t limit,
                                            uint32_t end_bits, uint32_t& phase, uint32_t& nslots, int nb,
                                            uint64_t pos, uint64_t total_slots, const JpegDecodeItem* it,
                                            int16_t* coef, int16_t* dcdiff, int* status) {
    if (hs.two_tables)
        decode_span_t<WRITE, true>(hs, s, p, limit, end_bits, phase, nslots, nb, pos, total_slots, it, coef, dcdiff, status);
    else
        decode_span_t<WRITE, false>(hs, s, p, limit, end_bits, phase, nslots, nb, pos, total_slots, it, coef, dcdiff, status);
}

// ---- 3. DC differences -> DC values
__device__ __forceinline__ void dc_prefix_pass(const JpegDecodeItem& it, int16_t* coef, const int16_t* dcdiff, int nb,
                                               uint32_t* warp_sums) {
    const int tid = threadIdx.x;
    // per component, prefix sum over ALL blocks in MCU (scan)
    //         order; only blocks inside the region of interest are stored.  kDcRun consecutive blocks
    //         per thread and tile: their loads are in flight together and one block scan serves them all.
    constexpr int kDcRun = 8;
    const uint32_t mcus_x = (uint32_t)it.mcus_x;
    const int roi_mx0 = it.roi_mx0, roi_my0 = it.roi_my0, roi_mcx = it.roi_mcx, roi_mcy = it.roi_mcy;
    int koff = 0;
    for (int c = 0; c < it.ncomp; c++) {
        const uint32_t bpc = (uint32_t)(it.h[c] * it.v[c]);
        const uint32_t nblk = mcus_x * (uint32_t)it.mcus_y * bpc;
        const int16_t* dsrc = dcdiff + koff;
        int16_t* cdst = coef + it.coef_off + (size_t)koff * 64;
        uint32_t dc_before = 0;  // signed prefix sum through unsigned wrap-around arithmetic
        for (uint32_t base = 0; base < nblk; base += kHuffThreads * kDcRun) {
            const uint32_t j0 = base + (uint32_t)tid * kDcRun;
            const uint32_t mcu0 = j0 / bpc, kk0 = j0 % bpc;
            int d[kDcRun];
            uint32_t sum = 0;
            {
                uint32_t mcu = mcu0, kk = kk0;
#pragma unroll
                for (int r = 0; r < kDcRun; r++) {
                    d[r] = j0 + r < nblk ? dsrc[(size_t)mcu * nb + kk] : 0;
                    sum += (uint32_t)d[r];
                    if (++kk == bpc) {
                        kk = 0;
                        mcu++;
                    }
                }
            }
            uint32_t total;
            const uint32_t ex = block_excl_scan<kHuffThreads>(sum, &total, warp_sums);
            uint32_t run = dc_before + ex;
            dc_before += total;
            uint32_t mcu = mcu0, kk = kk0;
            int mx = (int)(mcu0 % mcus_x) - roi_mx0, my = (int)(mcu0 / mcus_x) - roi_my0;
#pragma unroll
            for (int r = 0; r < kDcRun; r++) {
                run += (uint32_t)d[r];
                if (j0 + r < nblk && (unsigned)mx < (unsigned)roi_mcx && (unsigned)my < (unsigned)roi_mcy)
                    cdst[(((size_t)my * roi_mcx + mx) * nb + kk) * 64] = (int16_t)(int)run;
                if (++kk == bpc) {
                    kk = 0;
                    mcu++;
                    if (++mx == (int)mcus_x - roi_mx0) {
                        mx = -roi_mx0;
                        my++;
                    }
                }
            }
        }
        koff += (int)bpc;
    }
}

// At 512 threads, 3 CTAs/SM (40 registers) measured faster than 4 at 32 registers (spills in the write pass) or 2 at
// 62; at 384 threads, 4 CTAs/SM (40 registers) measured faster than 256 threads at 4 (62) or 5 (48) (DESIGN.md §5)
#ifndef LP_HUFF_MIN_CTAS
#define LP_HUFF_MIN_CTAS 4
#endif
__global__ void __launch_bounds__(kHuffThreads, LP_HUFF_MIN_CTAS)
    jpeg_huff_sync_kernel(JpegDecodeItem* items, const JpegHuffSet* tables, const uint8_t* clean,
                          SubState* states_all, uint32_t* nslots_all, int16_t* coef, int16_t* dcdiff_all,
                          uint32_t sub_per_thread) {
    __shared__ HuffShared hs;
    __shared__ uint32_t warp_sums[kHuffThreads / 32];
    __shared__ uint32_t s_carry;
    __shared__ int s_status;
    JpegDecodeItem& it = items[blockIdx.x];
    const int tid = threadIdx.x;
    if (it.status != 0 || it.restart_interval != 0 || it.nscans != 0) return;  // (DRI images: one thread per restart interval instead)
    __shared__ long long s_tphase;  // (shared, not a register pair every thread would carry through the loops)
    __shared__ unsigned long long s_bits[2];  // diagnostics: bits decoded in the synchronisation rounds, in the guess pass
    if (tid == 0) s_tphase = clock64();
    // ---- build the per-CTA tables
    {
        const JpegHuffSet* g = tables + it.table_set;
        for (int i = tid; i < 8 * 18; i += kHuffThreads) (&hs.maxcode[0][0])[i] = (&g->maxcode[0][0])[i];
        for (int i = tid; i < 8 * 17; i += kHuffThreads) (&hs.valoffset[0][0])[i] = (&g->valoffset[0][0])[i];
        for (int i = tid; i < 8 * 256; i += kHuffThreads) (&hs.vals[0][0])[i] = (&g->vals[0][0])[i];
        for (int i = tid; i < 4 * (1 << kDcBits); i += kHuffThreads) (&hs.dc_look[0][0])[i] = (&g->look[0][0])[i];
        for (int i = tid; i < 4 * (1 << kAcBits); i += kHuffThreads) (&hs.ac_look[0][0])[i] = 0;
        if (tid < 64) hs.zz[tid] = c_zigzag_p[tid];
        if (tid == 0) {
            int k = 0;
            for (int c = 0; c < it.ncomp; c++)
                for (int j = 0; j < it.h[c] * it.v[c]; j++, k++) {
                    hs.blk_dc[k] = (uint8_t)it.td[c];
                    hs.blk_ac[k] = (uint8_t)it.ta[c];
                    hs.blk_comp[k] = (uint8_t)c;
                    hs.blk_bx[k] = (uint8_t)(j % it.h[c]);
                    hs.blk_by[k] = (uint8_t)(j / it.h[c]);
                }
            const int nfirst = it.h[0] * it.v[0];
            bool two = true;
            for (int b = 0; b < k; b++) {
                const int ref = b < nfirst ? 0 : nfirst;
                if (hs.blk_dc[b] != hs.blk_dc[ref] || hs.blk_ac[b] != hs.blk_ac[ref]) two = false;
            }
            const int rest = nfirst < k ? nfirst : 0;
            hs.two_tables = two;
            hs.n_first = (uint32_t)nfirst;
            hs.dcb_first = (uint32_t)__cvta_generic_to_shared(&hs.dc_look[hs.blk_dc[0]][0]);
            hs.acb_first = (uint32_t)__cvta_generic_to_shared(&hs.ac_look[hs.blk_ac[0]][0]);
            hs.dcb_rest = (uint32_t)__cvta_generic_to_shared(&hs.dc_look[hs.blk_dc[rest]][0]);
            hs.acb_rest = (uint32_t)__cvta_generic_to_shared(&hs.ac_look[hs.blk_ac[rest]][0]);
            s_status = 0;
            s_carry = 0;
            s_bits[0] = s_bits[1] = 0;
        }
    }
    __syncthreads();
    {
        // widen the 9-bit AC lookahead tables to 11 bits, then add the 10- and 11-bit codes
        const JpegHuffSet* g = tables + it.table_set;
        for (int i = tid; i < 4 * (1 << kAcBits); i += kHuffThreads) {
            const int t = i >> kAcBits, idx = i & ((1 << kAcBits) - 1);
            uint16_t e = g->look[4 + t][idx >> (kAcBits - 9)];
            if (!e) {
                // no code of <= 9 bits is a prefix of idx, so the canonical walk continues at 10
                for (int len = 10; len <= kAcBits; len++) {
                    const int code = idx >> (kAcBits - len);
                    if (code <= hs.maxcode[4 + t][len]) {
                        e = (uint16_t)((len << 8) | hs.vals[4 + t][(code + hs.valoffset[4 + t][len]) & 0xFF]);
                        break;
                    }
                }
            }
            hs.ac_look[t][idx] = e;
        }
        for (int i = tid; i < 4 * kHuffLongPrefixes * 16; i += kHuffThreads)
            (&hs.ac_sub[0][0])[i] = (&g->long_sub[0][0][0])[i];
    }
    __syncthreads();
    if (tid < 4 * kHuffLongPrefixes) {
        const uint32_t pfx = (tables + it.table_set)->long_prefix[tid / kHuffLongPrefixes][tid % kHuffLongPrefixes];
        // (0xFFFF = unused slot; the builder never emits a prefix of more than kAcBits bits)
        if (pfx < (1u << kAcBits)) hs.ac_look[tid / kHuffLongPrefixes][pfx] = (uint16_t)(0x8000u | (uint32_t)tid);
    }
    __syncthreads();
    int nb = 0;
    for (int c = 0; c < it.ncomp; c++) nb += it.h[c] * it.v[c];
    const uint8_t* s = clean + it.clean_off;
    const uint32_t total_bits = it.clean_len * 8u;
    uint32_t kSubBits = (total_bits + kHuffThreads * sub_per_thread - 1) / (kHuffThreads * sub_per_thread);
    kSubBits = max(kMinSubBits, (kSubBits + 31u) & ~31u);
    const uint32_t nsub = (total_bits + kSubBits - 1) / kSubBits;
    SubState* st = states_all + it.state_off;      // nsub entries (second half: work lists)
    uint32_t* ns = nslots_all + it.state_off;      // [0,nsub): slots consumed per subsequence
    uint32_t* list_a = reinterpret_cast<uint32_t*>(st + nsub);  // 2*nsub uint32 = two work lists
    uint32_t* list_b = list_a + nsub;
    const uint64_t total_slots = (uint64_t)it.mcus_x * it.mcus_y * nb * 64;
    int16_t* dcdiff = dcdiff_all + it.dcdiff_off;

    LP_PHASE_MARK(0);
    // ---- pass 0: every subsequence from a guessed state (exact only for subsequence 0)
    for (uint32_t i = tid; i < nsub; i += kHuffThreads) {
        uint32_t p = i * kSubBits, phase = 0, n = 0;
        const uint32_t limit = min((i + 1) * kSubBits, total_bits);
        decode_span<false>(hs, s, p, limit, total_bits, phase, n, nb, 0, 0, nullptr, nullptr, nullptr, nullptr);
        atomicAdd(&s_bits[1], (unsigned long long)(p - i * kSubBits));
        st[i] = SubState{p, phase};
        ns[i] = n;
    }
    __syncthreads();
    LP_PHASE_MARK(1);
    // ---- synchronisation.  A subsequence is re-decoded from its left neighbour's exit state whenever
    //      that state changed; changes are collected in a work list so later (sparse) rounds keep all
    //      lanes busy.  States are updated in place: a reader that races with a writer sees either
    //      the old or the new 8-byte state, and in the first case the writer has queued it again.
    //      Round 1 visits every subsequence >= 1.  The fixed point is exact by induction from 0.
    uint32_t* cur_list = list_a;
    uint32_t* nxt_list = list_b;
    uint32_t cur_count = nsub > 0 ? nsub - 1 : 0;
    bool first_round = true;
    uint32_t rounds = 0;
    while (cur_count > 0) {
        rounds++;
        if (tid == 0) s_carry = 0;  // next list length
        __syncthreads();
        for (uint32_t k = tid; k < cur_count; k += kHuffThreads) {
            const uint32_t i = first_round ? k + 1 : cur_list[k];
            const uint64_t in64 = *reinterpret_cast<volatile uint64_t*>(&st[i - 1]);
            const SubState in{(uint32_t)in64, (uint32_t)(in64 >> 32)};
            const SubState old = st[i];
            uint32_t p = in.p, phase = in.phase, n = 0;
            const uint32_t limit = min((i + 1) * kSubBits, total_bits);
            if (p < limit) {
                decode_span<false>(hs, s, p, limit, total_bits, phase, n, nb, 0, 0, nullptr, nullptr, nullptr, nullptr);
                atomicAdd(&s_bits[0], (unsigned long long)(p - in.p));
            }
            ns[i] = n;  // slots consumed depend on the entry state even when the exit state does not
            if (p != old.p || phase != old.phase) {
                // only an exit-state change can affect the right neighbour
                *reinterpret_cast<volatile uint64_t*>(&st[i]) = ((uint64_t)phase << 32) | p;
                if (i + 1 < nsub) nxt_list[atomicAdd(&s_carry, 1u)] = i + 1;
            }
        }
        __syncthreads();
        cur_count = s_carry;
        __syncthreads();
        uint32_t* t = cur_list;
        cur_list = nxt_list;
        nxt_list = t;
        first_round = false;
    }
    if (tid == 0) {
        it.pad_ = rounds;  // diagnostics: synchronisation rounds this image needed
        atomicAdd(&g_huff_phase[6], s_bits[0]);
        atomicAdd(&g_huff_phase[7], s_bits[1]);
    }
    LP_PHASE_MARK(2);
    SubState* cur = st;
    // ---- prefix sum of slot counts, then the writing decode.  Every thread learns each tile's total
    //      from the scan, so the running offset lives in a register (no shared carry, no extra barriers).
    uint64_t slots_before = 0;
    for (uint32_t base = 0; base < nsub; base += kHuffThreads) {
        const uint32_t i = base + tid;
        const uint32_t v = i < nsub ? ns[i] : 0;
        uint32_t total;
        const uint32_t ex = block_excl_scan<kHuffThreads>(v, &total, warp_sums);
        const uint64_t pos = slots_before + ex;
        slots_before += total;
        if (i < nsub) {
            uint32_t p = i == 0 ? 0u : cur[i - 1].p;
            uint32_t phase = i == 0 ? 0u : cur[i - 1].phase;
            uint32_t n = 0;
            const uint32_t limit = min((i + 1) * kSubBits, total_bits);
            int status = 0;
            // the slot position implied by the prefix sum must agree with the carried phase
            if (pos < total_slots &&
                (uint32_t)(pos % ((uint64_t)nb * 64)) != ((phase >> 6) * 64 + (phase & 63)))
                status = -3;
            if (!status && p < limit)
                decode_span<true>(hs, s, p, limit, total_bits, phase, n, nb, pos, total_slots, &it, coef, dcdiff, &status);
            if (status) s_status = status;
        }
    }
    if (tid == 0 && slots_before < total_slots) s_status = -3;  // the stream ended before the last MCU
    __syncthreads();
    if (s_status) {
        if (tid == 0) it.status = s_status;
        return;
    }
    LP_PHASE_MARK(3);
    dc_prefix_pass(it, coef, dcdiff, nb, warp_sums);
    LP_PHASE_MARK(4);
    if (tid == 0) atomicAdd(&g_huff_phase[5], 1ull);
}


// ------------------------------------------------------------------ launcher

// host: read (and optionally clear) the phase counters of the current device
int jpeg_huff_phase_clocks(unsigned long long out[8], int reset) {
    LP_CUDA_OK(cudaDeviceSynchronize());
    LP_CUDA_OK(cudaMemcpyFromSymbol(out, g_huff_phase, sizeof(unsigned long long) * 8));
    if (reset) {
        unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        LP_CUDA_OK(cudaMemcpyToSymbol(g_huff_phase, z, sizeof(z)));
    }
    return LP_OK;
}

int jpeg_huff_parallel_slots() {
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, jpeg_huff_sync_kernel, kHuffThreads, 0);
    return sms * per_sm;
}

int jpeg_huff_parallel_launch(const JpegHuffParallelArgs& a, cudaStream_t st) {
    if (a.n <= 0) return LP_OK;
    static const uint32_t spt = getenv("LP_HUFF_SPT") ? (uint32_t)atoi(getenv("LP_HUFF_SPT")) : kSubPerThread;
    jpeg_unstuff_kernel<<<a.n, kUnstuffThreads, 0, st>>>(a.items, a.scan, a.clean);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    jpeg_huff_sync_kernel<<<a.n, kHuffThreads, 0, st>>>(a.items, a.tables, a.clean,
                                                       reinterpret_cast<SubState*>(a.states), a.nslots, a.coef,
                                                       a.dcdiff, spt);
    g_launches++;
    LP_CUDA_OK(cudaGetLastError());
    return LP_OK;
}

}  // namespace lp
