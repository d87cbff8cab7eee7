// jsgpu_huff.cu — entropy decode (stage A): FF00 unstuffing pre-pass + two Huffman kernels.
//
//   k_unstuff      a warp walks restart intervals of one image: 128 raw bytes per step, stuffed zeros
//                  found with one shuffle, kept-byte ranks from three __ballot_sync (the per-lane
//                  count is 0..4, so three ballots give its exclusive prefix); each lane's kept
//                  bytes are packed by a PRMT (selector from a 16-entry table) and OR-ed into a
//                  zeroed shared-memory ring, which leaves as 16-byte stores of big-endian words into
//                  an aligned, 0xFF-padded copy of the interval.  (BuffAddByte, ImgDecode.cpp:1386-1573.)
//   k_huff_warp    ONE WARP PER RESTART INTERVAL, warp-uniform symbol loop; lane i owns coefficients
//                  2i,2i+1 so a block leaves as one coalesced 128-byte row.  Right when there are few,
//                  long intervals (BASELINE config 5: no DRI) — a serial chain per interval.
//   k_huff_lane    one LANE per restart interval, 32 intervals per warp; blocks are assembled in
//                  per-lane shared-memory rows and written out cooperatively (coalesced).  Right when
//                  there are many short intervals (configs 1-4): 32x fewer issue slots per symbol.
// Both kernels share the look-up tables staged in shared memory and produce identical output:
// dequantised int16 coefficient rows in natural order (DecodeIdctSet, :2270-2303) whose slot 0
// holds the running DC predictor sum (m_nDcLum += m_anDctBlock[0], :3280).
#include "jsgpu_internal.h"
#include "jsgpu_phuff_core.cuh"
#include "jsgpu_scan.cuh"
#include <algorithm>
#include <cstdlib>

#define FULL 0xffffffffu

// ------------------------------------------------------------------------------------------------
// unstuff
// ------------------------------------------------------------------------------------------------
// The stuffed-zero test of one raw word.  `word` holds the interval's bytes rel0 .. rel0+3 in memory order and `prev` the word
// before it (its last byte precedes word's first).  One bit per byte of the word: dn = a stuffed zero (a 00 behind an FF, not
// the interval's first byte), rm = does not reach the output (a stuffed zero or outside the interval).
__device__ __forceinline__ void us_classify(uint32_t prev, uint32_t word, int rel0, uint32_t len, uint32_t& dn, uint32_t& rm)
{
    const int vlo = max(0, -rel0), vhi = min(4, (int)len - rel0);
    const uint32_t vn = (vhi > vlo) ? (((1u << vhi) - 1u) & ~((1u << vlo) - 1u)) : 0u;         // bytes inside the interval
    const uint32_t an = (rel0 <= 0 && rel0 > -4) ? (vn & ~(1u << (-rel0))) : vn;               // ... that may be a stuffed zero (not the first)
    const uint32_t pw = __byte_perm(prev, word, 0x6543);                // byte j = the byte before word's byte j
    const uint32_t npw = ~pw;
    const uint32_t z = ~(((word & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | word | 0x7F7F7F7Fu);          // byte == 0x00 (flag in bit 7)
    const uint32_t f = ~(((npw & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | npw | 0x7F7F7F7Fu);            // previous byte == 0xFF
    dn = ((((z & f) >> 7) * 0x00204081u) >> 21) & an;                                          // stuffed zeros, as a nibble
    rm = dn | (vn ^ 15u);
}

// PRMT selector that packs the bytes a removal nibble keeps to the low end of a word (4 = a byte of the zero operand): in memory
// order for a little-endian ring, or with the first kept byte most significant for a big-endian shift register
__device__ __forceinline__ uint32_t us_selector(uint32_t rm, bool big_endian)
{
    uint32_t sel = 0, n = 0;
    for (uint32_t i = 0; i < 4; i++) {
        const uint32_t j = big_endian ? 3 - i : i;
        if (!(rm >> j & 1)) sel |= j << (4 * n++);
    }
    for (; n < 4; n++) sel |= 4u << (4 * n);
    return sel;
}

#define US_RING 1024                        // bytes of staging ring per warp (two 512-byte halves)
// place the (<= 4) low bytes of `kk` at byte offset o of a zeroed ring: two result-less shared ORs
__device__ __forceinline__ void ring_place(uint32_t* ring, uint32_t kk, uint32_t o)
{
    const uint32_t sh = (o & 3) * 8, A = (o >> 2) & (US_RING / 4 - 1);
    atomicOr(&ring[A], kk << sh);
    atomicOr(&ring[(A + 1) & (US_RING / 4 - 1)], __funnelshift_l(kk, 0, sh));
}
// the 16-byte group at byte offset `off` of the ring as big-endian words; the group is re-zeroed
__device__ __forceinline__ uint4 ring_take(uint32_t* ring, uint32_t off)
{
    uint4* rp = reinterpret_cast<uint4*>(ring + ((off & (US_RING - 1)) >> 2));
    const uint4 v = *rp;
    *rp = make_uint4(0, 0, 0, 0);
    return make_uint4(__byte_perm(v.x, 0, 0x0123), __byte_perm(v.y, 0, 0x0123), __byte_perm(v.z, 0, 0x0123), __byte_perm(v.w, 0, 0x0123));
}

// the side tables of an unstuffed interval: length, where its copy starts, stuffed bytes
__device__ __forceinline__ void us_close(const DevBatch& b, uint32_t gw, uint32_t wr, uint64_t dst0, uint32_t nstuff)
{
    b.seg_ulen[gw] = wr; b.seg_uoff[gw] = dst0; b.seg_nstuff[gw] = nstuff;
    if (nstuff > JS_STUFF_LIST) b.ovf_list[atomicAdd(b.ovf_count, 1u)] = gw;     // rare: the MCU map of this interval needs the raw re-walk
}

__global__ void __launch_bounds__(128) k_unstuff(DevBatch b)
{
    __shared__ __align__(16) uint32_t s_ring[4][US_RING / 4];
    __shared__ uint32_t s_sel[16];          // us_selector, little-endian, by removal nibble
    __shared__ uint32_t s_cnt[4];           // stuffed bytes seen in the current interval, per warp
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t* const ring = s_ring[wid];
    if (threadIdx.x < 16) s_sel[threadIdx.x] = us_selector(threadIdx.x, false);
    for (uint32_t i = lane; i < US_RING / 4; i += 32) ring[i] = 0;
    __syncthreads();
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {            // grid.y = image (strided beyond 65535 images)
    const DevImage& im = b.img[ii];
    if (!im.valid || im.psync) continue;        // long intervals: k_unstuff_long (a warp per 4 KB, not per interval)
    const uint32_t nseg = im.nseg, seg_first = im.seg_first, kstep = (gridDim.x * blockDim.x) >> 5;
    const uint8_t* const scan = b.bits + im.scan_off;
    const uint64_t ubase = im.ubits_off;
    uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    // a warp walks intervals k, k + kstep, ...; the bounds of the next one are requested while this one is processed
    uint32_t ns0 = 0, ne0 = 0;
    if (k < nseg) { ns0 = b.seg_start[seg_first + k]; ne0 = b.seg_end[seg_first + k]; }
    for (; k < nseg; k += kstep) {
    const uint32_t gw = seg_first + k;
    const uint32_t s0 = ns0, len = ne0 - ns0;
    if (k + kstep < nseg) { ns0 = b.seg_start[gw + kstep]; ne0 = b.seg_end[gw + kstep]; }
    const uint8_t* seg = scan + s0;
    // destination: 16-byte aligned, never overlapping the neighbours (see DESIGN.md §3)
    const uint64_t dst0 = ubase + (uint64_t)(s0 & ~15u) + (unsigned long long)JS_USLACK * k;
    uint8_t* dst = b.ubits + dst0;
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(seg) & 3);
    const uint32_t* abase = reinterpret_cast<const uint32_t*>(seg - mis);
    uint32_t wr = 0, fl = 0, carry = 0;
    const uint32_t lt = (1u << lane) - 1;
    if (lane == 0) s_cnt[wid] = 0;
    __syncwarp();
    // rows are requested one ahead of their use
    auto load_row = [&](uint32_t rp) -> uint32_t {
        const int r0 = (int)(rp + 4 * lane) - (int)mis;
        return (r0 + 3 >= 0 && r0 < (int)len) ? __ldg(abase + (rp >> 2) + lane) : 0u;
    };
    uint32_t nword = load_row(0);
    for (uint32_t rpos = 0; rpos < len + mis; rpos += 128) {
        const int rel0 = (int)(rpos + 4 * lane) - (int)mis;                       // interval offset of this lane's byte 0
        const uint32_t word = nword;
        if (rpos + 128 < len + mis) nword = load_row(rpos + 128);
        uint32_t up = __shfl_up_sync(FULL, word, 1);
        if (lane == 0) up = carry;
        carry = __shfl_sync(FULL, word, 31);
        uint32_t dn, rm;
        us_classify(up, word, rel0, len, dn, rm);
        const uint32_t kk = __byte_perm(word, 0, s_sel[rm]);
        const uint32_t cnt = 4 - __popc(rm);                                                // 0..4 kept bytes
        const uint32_t b0 = __ballot_sync(FULL, cnt & 1), b1 = __ballot_sync(FULL, cnt & 2), b2 = __ballot_sync(FULL, cnt & 4);
        const uint32_t o = wr + __popc(b0 & lt) + 2 * __popc(b1 & lt) + 4 * __popc(b2 & lt);
        if (__any_sync(FULL, dn != 0)) {              // remember where bytes were dropped (MCU file map): unstuffed index of the preceding FF
            uint32_t d = dn;
            while (d) {
                const uint32_t j = __ffs(d) - 1; d &= d - 1;
                const uint32_t idx = atomicAdd(&s_cnt[wid], 1u);
                if (idx < JS_STUFF_LIST) b.seg_stuff[(size_t)gw * JS_STUFF_LIST + idx] = o + __popc(~rm & ((1u << j) - 1u)) - 1;
            }
        }
        ring_place(ring, kk, o);
        wr += __popc(b0) + 2 * __popc(b1) + 4 * __popc(b2);
        __syncwarp();
        if (wr - fl >= 512) {                          // a 512-byte half is complete: big-endian words out, half re-zeroed
            *reinterpret_cast<uint4*>(dst + fl + 16 * lane) = ring_take(ring, fl + 16 * lane);
            fl += 512;
            __syncwarp();
        }
    }
    // pad with 16 bytes of 1-bits (the JPEG pad value; no valid code is all ones) so readers can over-fetch
    if (lane < 4) ring_place(ring, 0xFFFFFFFFu, wr + 4 * lane);
    __syncwarp();
    #pragma unroll 1
    for (uint32_t off = 16 * lane; off < wr + 16 - fl; off += 512) *reinterpret_cast<uint4*>(dst + fl + off) = ring_take(ring, fl + off);
    __syncwarp();
    if (lane == 0) us_close(b, gw, wr, dst0, s_cnt[wid]);
    __syncwarp();
    }
    }
}

// ------------------------------------------------------------------------------------------------
// unstuff, one LANE per restart interval (the default for short intervals): with a restart marker every few MCUs an interval is
// ~300 bytes, i.e. 2-3 of k_unstuff's 128-byte rows plus as much fixed work per interval again (~490 warp instructions per
// interval, the kernel ALU-bound).  Here 32 intervals advance together, one 32-bit word per lane and step: the
// stuffed-zero test, the PRMT that packs the kept bytes and a 64-bit shift register are per lane and branch-free, raw bytes come in
// as 16-byte loads (one per four steps), output words go to a per-lane ring in shared memory and leave as 64-byte runs of 16-byte
// stores.  Output format and side tables (seg_ulen / seg_uoff / seg_nstuff / seg_stuff / ovf_list) are exactly k_unstuff's.
// ------------------------------------------------------------------------------------------------
#define UN_WARPS 8
#define UN_PITCH 36                         // words per lane row: a 32-word ring + 4 (keeps rows 16-byte aligned)
__global__ void __launch_bounds__(UN_WARPS * 32) k_unstuff_lane(DevBatch b)
{
    __shared__ __align__(16) uint32_t s_rows[UN_WARPS][32][UN_PITCH];
    __shared__ uint32_t s_selbe[16];        // us_selector, big-endian, by removal nibble
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x < 16) s_selbe[threadIdx.x] = us_selector(threadIdx.x, true);
    __syncthreads();
    uint32_t* const myrow = s_rows[wid][lane];
    uint32_t (*const rows)[UN_PITCH] = s_rows[wid];
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {
        const DevImage& im = b.img[ii];
        if (!im.valid || im.psync) continue;
        const uint32_t nseg = im.nseg, seg_first = im.seg_first;
        const uint8_t* const scan = b.bits + im.scan_off;
        for (uint32_t k0 = (blockIdx.x * UN_WARPS + wid) * 32; k0 < nseg; k0 += gridDim.x * UN_WARPS * 32) {
            const uint32_t k = k0 + lane; const bool live = k < nseg;
            const uint32_t gw = seg_first + (live ? k : k0);
            const uint32_t s0 = b.seg_start[gw], len = live ? b.seg_end[gw] - s0 : 0u;
            const uint64_t dst0 = im.ubits_off + (uint64_t)(s0 & ~15u) + (unsigned long long)JS_USLACK * (live ? k : k0);
            const uint8_t* const seg = scan + s0;
            const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(seg) & 15);
            const uint4* const abase = reinterpret_cast<const uint4*>(seg - mis);
            const uint32_t nwords = live ? (mis + len + 3) >> 2 : 0u;             // aligned words this lane walks
            const uint32_t nmax = __reduce_max_sync(FULL, nwords);
            unsigned long long acc = 0; uint32_t nacc = 0;                          // bytes waiting for a full output word (low end of acc)
            uint32_t wr = 0, nstuff = 0, wpos = 0, fpos = 0, prevw = 0;
            // flush: every lane whose ring holds `n` ready 16-byte pieces (0..4) gets them written behind what it has flushed so far
            auto flush = [&](uint32_t n) {
                const unsigned long long a = (unsigned long long)(uintptr_t)(b.ubits + dst0) + (unsigned long long)fpos * 4;
                const uint32_t off = fpos & 31;
                __syncwarp();
                #pragma unroll
                for (int r = 0; r < 4; r++) {
                    const int src = r * 8 + (lane >> 2); const uint32_t piece = lane & 3;
                    const unsigned long long sa = __shfl_sync(FULL, a, src);
                    const uint32_t sn = __shfl_sync(FULL, n, src), so = __shfl_sync(FULL, off, src);
                    if (piece < sn) *reinterpret_cast<uint4*>(sa + piece * 16) = *reinterpret_cast<const uint4*>(&rows[src][(so + piece * 4) & 31]);
                }
                __syncwarp();
                fpos += n * 4;
            };
            auto emit = [&](uint32_t w) { myrow[wpos & 31] = w; wpos++; };
            uint4 nxt = make_uint4(0, 0, 0, 0);
            if (nwords) nxt = __ldg(abase);
            auto step = [&](uint32_t j, uint32_t word) {
                if (j >= nwords) return;
                uint32_t dn, rm;
                us_classify(prevw, word, (int)(4 * j) - (int)mis, len, dn, rm);
                const uint32_t cnt = 4 - __popc(rm);
                if (dn) {                                   // where bytes were dropped (MCU file map): unstuffed index of the FF before each
                    uint32_t d = dn;
                    while (d) {
                        const uint32_t jj = __ffs(d) - 1; d &= d - 1;
                        if (nstuff < JS_STUFF_LIST) b.seg_stuff[(size_t)gw * JS_STUFF_LIST + nstuff] = wr + __popc(~rm & ((1u << jj) - 1u)) - 1;
                        nstuff++;
                    }
                }
                acc = (acc << (8 * cnt)) | __byte_perm(word, 0, s_selbe[rm]);
                nacc += cnt; wr += cnt;
                if (nacc >= 4) { emit((uint32_t)(acc >> (8 * (nacc - 4)))); nacc -= 4; }
                prevw = word;
            };
            for (uint32_t j = 0; j < nmax; j += 4) {
                const uint4 cur = nxt;
                if (j + 4 < nwords) nxt = __ldg(abase + (j >> 2) + 1);              // the next 16 bytes, one group ahead
                if (j && (j & 15) == 0) flush((wpos - fpos >= 16) ? 4u : 0u);
                step(j, cur.x); step(j + 1, cur.y); step(j + 2, cur.z); step(j + 3, cur.w);
            }
            flush((wpos - fpos >= 16) ? 4u : 0u);               // room for the padding: fewer than 16 words stay behind
            // 16 bytes of 1-bits behind the data (the JPEG pad value; no valid code is all ones) so readers can over-fetch, zeros up
            // to the next 16-byte boundary
            if (live) {
                const uint32_t total_words = ((wr + 16 + 15) & ~15u) >> 2;
                uint32_t pad_left = 16;
                while (wpos < total_words) {
                    const uint32_t n = min(4u, pad_left);
                    const uint32_t v = (n == 4) ? 0xFFFFFFFFu : (n == 0) ? 0u : (0xFFFFFFFFu << (8 * (4 - n)));
                    pad_left -= n;
                    acc = (acc << 32) | v; nacc += 4;
                    emit((uint32_t)(acc >> (8 * (nacc - 4)))); nacc -= 4;
                }
            }
            // what is left in the rings: at most 7 pieces per lane
            { const uint32_t pend = (wpos - fpos) >> 2; flush(min(pend, 4u)); }
            { const uint32_t pend = (wpos - fpos) >> 2; flush(min(pend, 4u)); }
            if (live) us_close(b, gw, wr, dst0, nstuff);
        }
    }
}

int js_launch_unstuff(const DevBatch& b, cudaStream_t s)
{
    if (b.nseg_total == 0 || b.max_nseg == 0) return 0;
    static const int mode = [] { const char* e = getenv("JSGPU_UNSTUFF"); return e ? atoi(e) : 1; }();   // 0 = warp per interval (k_unstuff)
    if (mode == 0 || b.max_nseg < 256) {           // few intervals per image: a warp per interval keeps more lanes busy
        dim3 grid((b.max_nseg + 3) / 4, b.nimg < 65535u ? b.nimg : 65535u);
        // persistent over an image's intervals: enough CTAs to fill the GPU ~8x, at most one warp per interval
        const uint32_t want = (JS_H100_SMS * 16u * 8u + grid.y - 1) / grid.y;
        if (grid.x > want) grid.x = want < 1 ? 1 : want;
        k_unstuff<<<grid, 128, 0, s>>>(b);
        return 1;
    }
    dim3 grid((b.max_nseg + UN_WARPS * 32 - 1) / (UN_WARPS * 32), b.nimg < 65535u ? b.nimg : 65535u);
    const uint32_t want = (JS_H100_SMS * 8u * 4u + grid.y - 1) / grid.y;
    if (grid.x > want) grid.x = want < 1 ? 1 : want;
    k_unstuff_lane<<<grid, UN_WARPS * 32, 0, s>>>(b);
    return 1;
}

// ------------------------------------------------------------------------------------------------
// unstuff, long intervals (images on the self-synchronising path): one warp per 4096 raw bytes instead of one warp
// per interval, so that a scan without restart markers (one 2.5 MB interval per 4K image) is not one serial walk:
//   k_unstuff_count   warp per chunk: how many bytes of the chunk reach the output
//   k_unstuff_scan    warp per interval: exclusive prefix sums -> output offset of every chunk; interval totals
//   k_unstuff_long    warp per chunk: the same row logic as k_unstuff, written at the chunk's output offset.  Chunk
//                     boundaries fall inside 16-byte groups and 32-bit words of the output, so the first group and the
//                     tail of every chunk are OR-ed into the (pre-zeroed) pool with atomics; everything in between
//                     leaves as whole 16-byte stores.
// The row tables for the MCU file map (rowtab / rowmask) are written as in k_unstuff.
// ------------------------------------------------------------------------------------------------
#define UL_WARPS 8
__device__ __forceinline__ uint32_t ul_base(uint32_t s0, uint32_t k) { return (s0 >> 12) + 2u * k; }
// interval (index inside the image) owning chunk slot cs and the chunk's index inside it; false = unused slot
__device__ __forceinline__ bool ul_find(const DevBatch& b, const DevImage& im, uint32_t cs, uint32_t& k, uint32_t& j, uint32_t& s0, uint32_t& len, uint32_t& mis)
{
    uint32_t lo = 0, hi = im.nseg - 1;
    while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (ul_base(b.seg_start[im.seg_first + mid], mid) <= cs) lo = mid; else hi = mid - 1; }
    k = lo; s0 = b.seg_start[im.seg_first + k]; len = b.seg_end[im.seg_first + k] - s0;
    mis = (uint32_t)(reinterpret_cast<uintptr_t>(b.bits + im.scan_off + s0) & 3);
    const uint32_t base = ul_base(s0, k), nch = len ? ((len + mis + 4095) >> 12) : 0u;
    if (cs < base || cs - base >= nch) return false;
    j = cs - base;
    return true;
}
// One 128-byte raw row of an interval: this lane's word, the nibble `rm` of its bytes that do not reach the output
// (stuffed zeros, bytes outside the interval) and the stuffed-zero nibble `dn`.  carry = the previous row's last word.
__device__ __forceinline__ void ul_row(const uint32_t* abase, uint32_t rpos, uint32_t lane, uint32_t mis, uint32_t len, uint32_t& carry, uint32_t& word, uint32_t& rm)
{
    const int rel0 = (int)(rpos + 4 * lane) - (int)mis;
    word = (rel0 + 3 >= 0 && rel0 < (int)len) ? __ldg(abase + (rpos >> 2) + lane) : 0u;
    uint32_t up = __shfl_up_sync(FULL, word, 1);
    if (lane == 0) up = carry;
    carry = __shfl_sync(FULL, word, 31);
    uint32_t dn;
    us_classify(up, word, rel0, len, dn, rm);
}

__global__ void __launch_bounds__(UL_WARPS * 32) k_unstuff_count(DevBatch b)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {
        const DevImage& im = b.img[ii];
        if (!im.valid || !im.psync) continue;
        for (uint32_t cs = blockIdx.x * UL_WARPS + wid; cs < im.cs_nslots; cs += gridDim.x * UL_WARPS) {
            uint32_t k, j, s0, len, mis;
            if (!ul_find(b, im, cs, k, j, s0, len, mis)) { if (lane == 0) { b.cs_cnt[im.cs_first + cs] = 0; b.cs_seg[im.cs_first + cs] = 0xffffffffu; } continue; }
            const uint32_t* abase = reinterpret_cast<const uint32_t*>(b.bits + im.scan_off + s0 - mis);
            uint32_t carry = j ? __ldg(abase + (j << 10) - 1) : 0u, tot = 0;
            uint32_t rp0 = j << 12;
            for (uint32_t r = 0; r < 32 && rp0 + 128 * r < len + mis; r++) {
                uint32_t word, rm;
                ul_row(abase, rp0 + 128 * r, lane, mis, len, carry, word, rm);
                tot += 4 - __popc(rm);
            }
            tot = __reduce_add_sync(FULL, tot);
            if (lane == 0) { b.cs_cnt[im.cs_first + cs] = tot; b.cs_seg[im.cs_first + cs] = k; }
        }
    }
}

__global__ void __launch_bounds__(128) k_unstuff_scan(DevBatch b)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint32_t ii = blockIdx.x; ii < b.nimg; ii += gridDim.x) {
        const DevImage& im = b.img[ii];
        if (!im.valid || !im.psync) continue;
        for (uint32_t k = wid; k < im.nseg; k += 4) {
            const uint32_t gw = im.seg_first + k, s0 = b.seg_start[gw], len = b.seg_end[gw] - s0;
            const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(b.bits + im.scan_off + s0) & 3);
            const uint32_t nch = len ? ((len + mis + 4095) >> 12) : 0u;
            const size_t c0 = im.cs_first + ul_base(s0, k);
            uint32_t run = 0;
            for (uint32_t c = 0; c < nch; c += 32) {
                uint32_t inc;
                const uint32_t ex = js_warp_scan((c + lane < nch) ? b.cs_cnt[c0 + c + lane] : 0u, 0u, js_add, inc);
                if (c + lane < nch) b.cs_off[c0 + c + lane] = run + ex;
                run += __shfl_sync(FULL, inc, 31);
            }
            if (lane == 0) {
                b.seg_ulen[gw] = run; b.seg_nstuff[gw] = len - run;
                b.seg_uoff[gw] = im.ubits_off + (uint64_t)(s0 & ~15u) + (unsigned long long)JS_USLACK * k;
            }
        }
    }
}

__global__ void __launch_bounds__(UL_WARPS * 32) k_unstuff_long(DevBatch b)
{
    __shared__ __align__(16) uint32_t s_ring[UL_WARPS][US_RING / 4];
    __shared__ uint32_t s_sel[16];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t* const ring = s_ring[wid];
    if (threadIdx.x < 16) s_sel[threadIdx.x] = us_selector(threadIdx.x, false);
    for (uint32_t i = lane; i < US_RING / 4; i += 32) ring[i] = 0;
    __syncthreads();
    // one 16-byte group of the ring -> dst; shared = other chunks own part of the group: OR it in
    auto flush_group = [&](uint8_t* dst, uint32_t ring_off, bool shared) {
        const uint4 o = ring_take(ring, ring_off);
        if (!shared) *reinterpret_cast<uint4*>(dst) = o;
        else {
            uint32_t* d = reinterpret_cast<uint32_t*>(dst);
            if (o.x) atomicOr(d, o.x); if (o.y) atomicOr(d + 1, o.y); if (o.z) atomicOr(d + 2, o.z); if (o.w) atomicOr(d + 3, o.w);
        }
    };
    const uint32_t lt = (1u << lane) - 1;
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {
        const DevImage& im = b.img[ii];
        if (!im.valid || !im.psync) continue;
        for (uint32_t cs = blockIdx.x * UL_WARPS + wid; cs < im.cs_nslots; cs += gridDim.x * UL_WARPS) {
            const uint32_t k = b.cs_seg[im.cs_first + cs];
            if (k == 0xffffffffu) continue;
            const uint32_t gw = im.seg_first + k, s0 = b.seg_start[gw], len = b.seg_end[gw] - s0;
            const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(b.bits + im.scan_off + s0) & 3);
            const uint32_t j = cs - ul_base(s0, k), nch = (len + mis + 4095) >> 12;
            const uint32_t O = b.cs_off[im.cs_first + cs];                      // unstuffed bytes of the interval before this chunk
            uint8_t* const dst = b.ubits + b.seg_uoff[gw] + (O & ~15u);          // 16-byte group holding the chunk's first output byte
            const uint32_t* abase = reinterpret_cast<const uint32_t*>(b.bits + im.scan_off + s0 - mis);
            const size_t rt0 = (size_t)(im.rt_off + (s0 >> 7) + 2u * k);
            uint32_t carry = j ? __ldg(abase + (j << 10) - 1) : 0u;
            uint32_t wr = O & 15u, fl = 0;
            const uint32_t wr0 = wr, rp0 = j << 12;
            for (uint32_t r = 0; r < 32 && rp0 + 128 * r < len + mis; r++) {
                const uint32_t rpos = rp0 + 128 * r;
                uint32_t word, rm;
                ul_row(abase, rpos, lane, mis, len, carry, word, rm);
                const uint32_t kk = __byte_perm(word, 0, s_sel[rm]);
                const uint32_t cnt = 4 - __popc(rm);
                {
                    uint32_t mw = rm << ((lane & 7) * 4);
                    mw |= __shfl_xor_sync(FULL, mw, 1); mw |= __shfl_xor_sync(FULL, mw, 2); mw |= __shfl_xor_sync(FULL, mw, 4);
                    if ((lane & 7) == 0) reinterpret_cast<uint32_t*>(b.rowmask + rt0 + (rpos >> 7))[lane >> 3] = mw;
                    if (lane == 0) b.rowtab[rt0 + (rpos >> 7)] = O + (wr - wr0);
                }
                const uint32_t b0 = __ballot_sync(FULL, cnt & 1), b1 = __ballot_sync(FULL, cnt & 2), b2 = __ballot_sync(FULL, cnt & 4);
                ring_place(ring, kk, wr + __popc(b0 & lt) + 2 * __popc(b1 & lt) + 4 * __popc(b2 & lt));
                wr += __popc(b0) + 2 * __popc(b1) + 4 * __popc(b2);
                __syncwarp();
                if (wr - fl >= 512) {
                    flush_group(dst + fl + 16 * lane, fl + 16 * lane, fl == 0 && lane == 0);
                    fl += 512;
                    __syncwarp();
                }
            }
            uint32_t end = wr;
            if (j + 1 == nch) {            // last chunk of the interval: 16 bytes of 1-bits behind the data (readers over-fetch)
                if (lane < 4) ring_place(ring, 0xFFFFFFFFu, wr + 4 * lane);
                end = wr + 16;
                __syncwarp();
            }
            #pragma unroll 1
            for (uint32_t off = 16 * lane; fl + off < end; off += 512) flush_group(dst + fl + off, fl + off, true);
            __syncwarp();
        }
    }
}

int js_launch_unstuff_long(const DevBatch& b, uint32_t max_cs, cudaStream_t s)
{
    if (max_cs == 0) return 0;
    dim3 grid((max_cs + UL_WARPS - 1) / UL_WARPS, b.nimg < 65535u ? b.nimg : 65535u);
    const uint32_t want = (JS_H100_SMS * 8u * 4u + grid.y - 1) / grid.y;
    if (grid.x > want) grid.x = want < 1 ? 1 : want;
    k_unstuff_count<<<grid, UL_WARPS * 32, 0, s>>>(b);
    k_unstuff_scan<<<b.nimg < 65535u ? b.nimg : 65535u, 128, 0, s>>>(b);
    k_unstuff_long<<<grid, UL_WARPS * 32, 0, s>>>(b);
    return 3;
}

// ------------------------------------------------------------------------------------------------
// shared pieces
// ------------------------------------------------------------------------------------------------
struct HuffTabs {                       // shared-memory staged tables of ONE image
    uint16_t lut[6][JS_LUT_SIZE];       // [comp*2 + class]  (len<<8)|symbol, 0 = not decidable from the prefix
    uint32_t qz[3][80];                 // quantiser | natural index<<16 ; entries 64..79 = no-op (nat 127)
};

__device__ __forceinline__ void stage_tables(HuffTabs& t, const DevImage& im, const DevTableSet* ts)
{
    for (uint32_t c = 0; c < im.ns; c++) {
        const uint4* s0 = reinterpret_cast<const uint4*>(ts->lut[im.slot_dc[c]]);
        const uint4* s1 = reinterpret_cast<const uint4*>(ts->lut[im.slot_ac[c]]);
        uint4* d0 = reinterpret_cast<uint4*>(t.lut[c * 2]);
        uint4* d1 = reinterpret_cast<uint4*>(t.lut[c * 2 + 1]);
        for (uint32_t i = threadIdx.x; i < JS_LUT_SIZE * 2 / 16; i += blockDim.x) { d0[i] = __ldg(s0 + i); d1[i] = __ldg(s1 + i); }
        stage_qz(t.qz[c], ts->qz[im.dqt[c]]);
    }
}

// What an interval's end tells (both Huffman kernels): read past its data -> OVERRUN; else 8 or more bits left over after a
// decode without a bad code or a coefficient overflow -> LEFTOVER
__device__ __forceinline__ uint32_t seg_end_status(uint32_t status, uint32_t consumed, uint32_t avail)
{
    if (consumed > avail) return status | 2;
    if (!(status & 5) && avail - consumed >= 8) return status | 16;
    return status;
}

// Block-DC map (ImgDecode.cpp:3524-3608 in gather form): cell (mx*eh+h, my*ev+v) keeps the DC of block (h, v) of MCU (mx, my)
// iff no later MCU overwrites it: (h < eh or last MCU column) and (v < ev or last MCU row)
__device__ __forceinline__ bool blk_dc_kept(uint32_t h, uint32_t v, uint32_t eh, uint32_t ev, uint32_t mx, uint32_t my, uint32_t mcu_xmax, uint32_t mcu_ymax)
{
    return (h < eh || mx == mcu_xmax - 1) && (v < ev || my == mcu_ymax - 1);
}

// In-order entry search of ReadScanVal (ImgDecode.cpp:1145-1164) for prefixes the LUT cannot decide.
__device__ __noinline__ uint32_t huff_slow(const DevTableSet* ts, uint32_t slot, uint32_t top)
{
    uint32_t n = ts->ent_n[slot];
    for (uint32_t i = 0; i < n; i++) {
        uint32_t l = ts->ent_len[slot][i];
        if (l == 0 || l > 16) continue;
        if ((top & (0xffffffffu << (32 - l))) == ts->ent_bits[slot][i]) return (l << 8) | ts->ent_sym[slot][i];
    }
    return 0;
}

// Second-level / exceptional look-up: e is the first-level entry (0 or 0x8000|offset).
__device__ __forceinline__ uint32_t huff_level2(const DevTableSet* ts, uint32_t slot, uint32_t e, uint32_t top)
{
    if (e & 0x8000) {
        if (ts->lut2_overflow[slot]) return huff_slow(ts, slot, top);
        return __ldg(&ts->lut2[slot][(e & 0x7FFF) + ((top >> (32 - 16)) & ((1u << JS_LUT2_BITS) - 1))]);
    }
    return 0;     // no code has this prefix (the reference's search would fail too)
}

// Per-thread bit reader over an unstuffed, 4-byte aligned, 0xFF-padded interval (k_unstuff stores it as
// big-endian 32-bit words, so a loaded word is already in bit order).
struct Bits {
    unsigned long long w; int nb; const uint32_t* p; uint32_t words; uint32_t nx;
    __device__ __forceinline__ void init(const uint8_t* base) {
        p = reinterpret_cast<const uint32_t*>(base);
        uint32_t a = __ldg(p), c = __ldg(p + 1);
        nx = __ldg(p + 2);                                 // always one word ahead: the load latency hides behind ~6 symbols
        w = ((unsigned long long)a << 32) | c; nb = 64; p += 3; words = 2;
    }
    __device__ __forceinline__ void refill() {          // call when nb <= 32
        uint32_t x = nx;
        nx = __ldg(p);
        w |= (unsigned long long)x << (32 - nb);
        nb += 32; p++; words++;
    }
    __device__ __forceinline__ uint32_t consumed() const { return 32u * words - (uint32_t)nb; }
    __device__ __forceinline__ uint32_t top32() const { return (uint32_t)(w >> 32); }
};

// value bits + T.81 F.12 EXTEND (HuffmanDc2Signed, ImgDecode.cpp:859-866) + precision divide (:1234-1238)
__device__ __forceinline__ int take_value(Bits& s, uint32_t size, uint32_t precision)
{
    uint32_t t = s.top32();
    uint32_t v = (size == 0) ? 0u : (t >> (32 - size));
    int neg = ((int)~t) >> 31;                                   // all ones when the leading value bit is 0
    int val = (int)v - (neg & (int)((1u << size) - 1));
    s.w <<= size; s.nb -= (int)size;
    if (precision > 8) val /= (1 << (precision - 8));
    return val;
}

// ------------------------------------------------------------------------------------------------
// MCU file map, intervals consumed to their very last bit.  The entry of the first MCU after an RSTn is the
// reader state at the END of the previous interval (lazy restart, ImgDecode.cpp:1644-1680).  When that
// interval was used up exactly, the reference's byte-position array is drained and reports what is left in
// its LAST slot (ScanBuffConsume shifts pos[1..3] down and never clears pos[3], :934-953): the file position
// of the last byte that entered the 4-byte accumulator while it held three others.  The accumulator is
// topped up before every code and every value read (BuffTopup, :1292-1323), so that byte is unstuffed byte
// c*+3, where c* is the largest whole-byte count consumed at any of those moments that still left >= 4
// bytes (c* <= D-4).  Usually c* = D-4 and the answer is the interval's last byte; when a single read
// stepped over two byte boundaries near the end it is an earlier one.  One thread per interval re-reads the
// code lengths of the last MCU(s) to find c*.  (Verified against the CPU oracle on every boundary of the
// test corpus; tests/jpeg_cases.py compares the map exactly.)
// ------------------------------------------------------------------------------------------------
#define EM_SPAN 1024                        // intervals examined per CTA pass (about one in eight is drained exactly)
__global__ void __launch_bounds__(128) k_finalize_mcumap_emptied(DevBatch b)
{
    __shared__ uint32_t s_list[EM_SPAN];
    __shared__ uint32_t s_n;
    __shared__ __align__(16) uint16_t s_lut[6][JS_LUT_SIZE];      // first-level tables of the current image, [comp*2 + class]
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {            // grid.y = image (strided beyond 65535 images)
    const DevImage& im = b.img[ii];
    if (!im.valid || !im.restart_en || im.nseg < 2 || b.ex_flag[ii]) continue;
    if (blockIdx.x * EM_SPAN + 1 >= im.nseg) continue;
    const DevTableSet* ts = b.tables + im.table_set;
    const uint32_t ns = im.ns, ri = im.ri, nmcu = im.nmcu;
    const uint32_t nb0 = im.H[0] * im.V[0], nb1 = (ns == 3) ? im.H[1] * im.V[1] : 0, nb2 = (ns == 3) ? im.H[2] * im.V[2] : 0;
    __syncthreads();
    for (uint32_t c = 0; c < ns; c++) {
        const uint4* s0 = reinterpret_cast<const uint4*>(ts->lut[im.slot_dc[c]]);
        const uint4* s1 = reinterpret_cast<const uint4*>(ts->lut[im.slot_ac[c]]);
        for (uint32_t i = threadIdx.x; i < JS_LUT_SIZE * 2 / 16; i += blockDim.x) {
            reinterpret_cast<uint4*>(s_lut[c * 2])[i] = __ldg(s0 + i); reinterpret_cast<uint4*>(s_lut[c * 2 + 1])[i] = __ldg(s1 + i);
        }
    }
    const uint32_t sdc0 = im.slot_dc[0], sac0 = im.slot_ac[0], sdc1 = im.slot_dc[1], sac1 = im.slot_ac[1], sdc2 = im.slot_dc[2], sac2 = im.slot_ac[2];
    for (uint32_t base = blockIdx.x * EM_SPAN; base + 1 < im.nseg; base += gridDim.x * EM_SPAN) {
        // pass 1: which intervals of this span were drained exactly?  (compacted, so that pass 2 runs with full warps)
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < EM_SPAN; i += blockDim.x) {
            const uint32_t k = base + i;
            if (k + 1 >= im.nseg) break;
            const uint32_t gw = im.seg_first + k;
            const uint32_t D = b.seg_ulen[gw];
            if (D >= 4 && b.seg_endbits[gw] == 8 * D && !b.seg_status[gw] && min(k * ri + ri, nmcu) < nmcu)
                s_list[atomicAdd(&s_n, 1u)] = k;                         // (D < 4 reports 0: k_finalize_mcumap_fast did that)
        }
        __syncthreads();
        const uint32_t n = s_n;
        for (uint32_t li = threadIdx.x; li < n; li += blockDim.x) {
        const uint32_t k = s_list[li];
        const uint32_t gw = im.seg_first + k;
        const uint32_t D = b.seg_ulen[gw];
        const uint32_t m0 = k * ri, m1 = min(m0 + ri, nmcu);
        const uint32_t lim = 8 * (D - 3);                                // top-ups at bit positions below this still see >= 4 bytes
        uint32_t mm = m1 - 1;
        while (mm > m0 && b.mcu_bitpos[im.mcu_off + mm] >= lim) mm--;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(b.ubits + b.seg_uoff[gw]);
        uint32_t bp = (mm == m0) ? 0u : b.mcu_bitpos[im.mcu_off + mm], last = bp;
        uint32_t cw = bp >> 5, w0 = __ldg(w + cw), w1 = __ldg(w + cw + 1);   // bit window: two words, reloaded when bp leaves the first
        bool ok = true;
        for (uint32_t m = mm; m < m1 && ok && bp < lim; m++)
            #pragma unroll 1
            for (uint32_t c = 0; c < ns && ok && bp < lim; c++) {
                const uint32_t nb = (c == 0) ? nb0 : (c == 1) ? nb1 : nb2;
                const uint32_t sdc = (c == 0) ? sdc0 : (c == 1) ? sdc1 : sdc2, sac = (c == 0) ? sac0 : (c == 1) ? sac1 : sac2;
                const uint16_t* ldc = s_lut[c * 2]; const uint16_t* lac = s_lut[c * 2 + 1];
                for (uint32_t bi = 0; bi < nb && ok && bp < lim; bi++) {
                    uint32_t pos = 0;
                    while (pos < 64 && bp < lim) {
                        last = bp;                                        // top-up before the code
                        if ((bp >> 5) != cw) { cw = bp >> 5; w0 = __ldg(w + cw); w1 = __ldg(w + cw + 1); }
                        const uint32_t top = __funnelshift_l(w1, w0, bp & 31);
                        uint32_t e = (pos ? lac : ldc)[top >> (32 - JS_LUT_BITS)];
                        if (e & 0x8000) e = huff_level2(ts, pos ? sac : sdc, e, top);
                        if (e == 0) { ok = false; break; }
                        bp += e >> 8;
                        if (bp < lim) last = bp;                          // top-up before the value bits
                        if (pos && (e & 0xFF) == 0) break;                // EOB
                        bp += e & 15;
                        pos += pos ? ((e >> 4) & 15) + 1 : 1;
                    }
                }
            }
        if (!ok) continue;
        const uint32_t j = (last >> 3) + 3;                              // unstuffed index of the reported byte (<= D-1)
        // its raw offset: walk back from the end of the raw interval, skipping stuffed zeros
        const uint32_t s0 = b.seg_start[gw], len = b.seg_end[gw] - s0;
        const uint8_t* seg = b.bits + im.scan_off + s0;
        uint32_t r = len - 1, t = D - 1 - j;
        for (;;) {
            if (r > 0 && seg[r] == 0 && seg[r - 1] == 0xFF) r--;         // a stuffed zero: its FF is the data byte
            if (t == 0 || r == 0) break;
            t--; r--;
        }
        b.mcu_map[im.mcu_off + m1] = (im.file_pos + s0 + r) << 4;
        }
        __syncthreads();
    }
    }
}

int js_launch_finalize_emptied(const DevBatch& b, cudaStream_t s)
{
    if (!b.mcu_map || b.nimg == 0 || b.max_nseg < 2) return 0;
    const dim3 grid(std::min<uint32_t>((b.max_nseg + EM_SPAN - 1) / EM_SPAN, 64u), b.nimg < 65535u ? b.nimg : 65535u);
    k_finalize_mcumap_emptied<<<grid, 128, 0, s>>>(b);
    return 1;
}

// ------------------------------------------------------------------------------------------------
// warp per restart interval
// ------------------------------------------------------------------------------------------------
struct WarpShared { HuffTabs t; uint32_t histo[6][17]; };

__device__ __forceinline__ void flush_histo(const DevBatch& b, uint32_t img, uint32_t (*histo)[17])
{
    const DevImage& pim = b.img[img];
    for (uint32_t i = threadIdx.x; i < 6 * 17; i += blockDim.x) {
        uint32_t c = i / 34, cls = (i / 17) & 1, l = i % 17;
        uint32_t v = histo[c * 2 + cls][l];
        if (v && c < pim.ns) { uint32_t slot = cls ? pim.slot_ac[c] : pim.slot_dc[c]; atomicAdd(&b.histo[((size_t)img * 8 + slot) * 17 + l], v); }
    }
}

__global__ void __launch_bounds__(JS_HUFF_WARPS * 32) k_huff_warp(DevBatch b)
{
    __shared__ WarpShared sh;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t cur_img = 0xffffffffu;
    for (uint32_t it = blockIdx.x; it < b.nitems; it += gridDim.x) {
        const uint2 item = b.items[it];
        const DevImage& gim = b.img[item.x];
        const DevTableSet* ts = b.tables + gim.table_set;
        if (item.x != cur_img) {
            __syncthreads();
            if (cur_img != 0xffffffffu && b.want_histo) { flush_histo(b, cur_img, sh.histo); __syncthreads(); }
            for (uint32_t i = threadIdx.x; i < 6 * 17; i += blockDim.x) (&sh.histo[0][0])[i] = 0;
            stage_tables(sh.t, gim, ts);
            cur_img = item.x;
            __syncthreads();
        }
        const uint32_t k = item.y + wid;
        if (k >= gim.nseg) continue;
        // hoist everything the hot loop needs into registers
        const uint32_t ns = gim.ns, precision = gim.precision, ri = gim.ri, nmcu = gim.nmcu, mcu_xmax = gim.mcu_xmax;
        const uint32_t sidx = gim.seg_first + k;
        const uint32_t ulen = b.seg_ulen[sidx];
        Bits s; s.init(b.ubits + b.seg_uoff[sidx]);
        const uint32_t m0 = k * ri, m1 = min(m0 + ri, nmcu);
        uint32_t mx = m0 % mcu_xmax, my = m0 / mcu_xmax;
        int dcs[3] = {0, 0, 0};
        uint32_t status = 0;
        uint32_t* const coef32 = reinterpret_cast<uint32_t*>(b.coef);
        const bool want_ac = b.decode_ac != 0;
        for (uint32_t m = m0; m < m1 && !(status & 7); m++) {
            if (s.consumed() > ulen * 8) { status |= 2; break; }       // ran off the end of the interval (corrupt or truncated data): stop reading
            if (lane == 0) b.mcu_bitpos[gim.mcu_off + m] = s.consumed();
            #pragma unroll 1
            for (uint32_t c = 0; c < ns; c++) {
                const uint16_t* lut_dc = sh.t.lut[c * 2];
                const uint16_t* lut_ac = sh.t.lut[c * 2 + 1];
                const uint32_t* qz = sh.t.qz[c];
                const uint32_t nh = gim.H[c], nv = gim.V[c], cw = gim.cw[c];
                const uint32_t slot_dc = gim.slot_dc[c], slot_ac = gim.slot_ac[c];
                const size_t row0 = gim.coef_row[c] + (size_t)(my * nv) * cw + mx * nh;
                uint32_t hdc = 0, hac = 0;
                int dc = dcs[c];
                #pragma unroll 1
                for (uint32_t bi = 0; bi < nh * nv; bi++) {
                    uint32_t acc = 0;
                    // ---- DC symbol ----
                    if (s.nb <= 32) s.refill();
                    uint32_t e = lut_dc[s.top32() >> (32 - JS_LUT_BITS)];
                    if (e == 0 || (e & 0x8000)) e = huff_level2(ts, slot_dc, e, s.top32());
                    if (e == 0) { status |= 1; break; }
                    uint32_t len = e >> 8;
                    s.w <<= len; s.nb -= (int)len;
                    hdc += (lane == len);
                    uint32_t pos;
                    {
                        uint32_t run = (e >> 4) & 15, size = e & 15;
                        int val = take_value(s, size, precision);
                        uint32_t q = qz[run];                      // run is 0 for every legal DC symbol
                        int cf = (int)(short)(val * (int)(q & 0xFFFF));
                        uint32_t nat = q >> 16;
                        int dcdiff = 0;
                        if (nat == 0) dcdiff = cf;
                        else if (want_ac && lane == (nat >> 1)) acc = (nat & 1) ? __byte_perm(acc, (uint32_t)cf, 0x5410) : __byte_perm(acc, (uint32_t)cf, 0x3254);   // a DC symbol with a run nibble stores an AC value: none in DC-only mode (the reference runs no IDCT there)
                        dc = (int)(short)(dc + dcdiff);
                        pos = 1 + run;
                    }
                    // ---- AC symbols ----
                    while (pos < 64) {
                        if (s.nb <= 32) s.refill();
                        e = lut_ac[s.top32() >> (32 - JS_LUT_BITS)];
                        if (e == 0 || (e & 0x8000)) e = huff_level2(ts, slot_ac, e, s.top32());
                        if (e == 0) { status |= 1; break; }
                        len = e >> 8;
                        s.w <<= len; s.nb -= (int)len;
                        hac += (lane == len);
                        if ((e & 0xFF) == 0) break;               // EOB
                        uint32_t run = (e >> 4) & 15, size = e & 15;
                        int val = take_value(s, size, precision);
                        uint32_t kk = pos + run;
                        uint32_t q = qz[kk];                       // kk <= 78; entries >= 64 are no-ops
                        uint32_t cf = (uint32_t)(val * (int)(q & 0xFFFF));
                        uint32_t nat = q >> 16;
                        if (want_ac && lane == (nat >> 1)) acc = (nat & 1) ? __byte_perm(acc, cf, 0x5410) : __byte_perm(acc, cf, 0x3254);
                        pos = kk + 1;
                    }
                    if (pos > 64) status |= 4;
                    if (lane == 0) acc = __byte_perm(acc, (uint32_t)dc, 0x3254);
                    const uint32_t v = bi / nh, h = bi - v * nh;
                    if (lane == 0 && blk_dc_kept(h, v, gim.eh[c], gim.ev[c], mx, my, mcu_xmax, gim.mcu_ymax))
                        (((c == 0) ? b.blk_y : (c == 1) ? b.blk_cb : b.blk_cr) + gim.blk_off)[(my * gim.ev[c] + v) * gim.blk_xmax + (mx * gim.eh[c] + h)] = (int16_t)dc;
                    coef32[(row0 + (size_t)v * cw + h) * 32 + lane] = acc;
                    if (status & 7) break;
                }
                dcs[c] = dc;
                if (b.want_histo && lane >= 1 && lane <= 16) { atomicAdd(&sh.histo[c * 2][lane], hdc); atomicAdd(&sh.histo[c * 2 + 1][lane], hac); }
                if (status & 7) break;
            }
            if (++mx == mcu_xmax) { mx = 0; my++; }
        }
        const uint32_t consumed = s.consumed();
        status = seg_end_status(status, consumed, ulen * 8);
        if (lane == 0) {
            b.seg_endbits[sidx] = consumed;
            b.seg_status[sidx] = status;
            if (status) atomicOr(&b.img_status[item.x], status);
        }
    }
    __syncthreads();
    if (cur_img != 0xffffffffu && b.want_histo) flush_histo(b, cur_img, sh.histo);
}

int js_launch_huffman_warp(const DevBatch& b, int sm_count, cudaStream_t s)
{
    if (b.nitems == 0) return 0;
    uint32_t grid = (uint32_t)sm_count * 8;
    if (grid > b.nitems) grid = b.nitems;
    k_huff_warp<<<grid, JS_HUFF_WARPS * 32, 0, s>>>(b);
    return 1;
}

// ------------------------------------------------------------------------------------------------
// lane per restart interval
// ------------------------------------------------------------------------------------------------
#define LN_WARPS   (JS_LANE_SEGS / 32)
#define ROW_PITCH  208                      // bytes per lane row: 64 coefficients, 8 dummy slots, 16 code-length counters; 16-byte aligned
#define ROW_HIST   144                      // byte offset of the counter for length 1 (length 0 = "no code" lands in the dummy slots)
#define LN_TAB     JS_LANE_TAB                   // entries per staged table: first level, then its second level
// Dynamic shared memory of the lane kernel:
//   LaneHdr | lane rows [LN_WARPS][32][ROW_PITCH] | tables [nl][LN_TAB]
// nl = DevBatch::lane_nlut: the distinct (class,Th) tables an image selects are staged once each (Cb and Cr
// normally share theirs), second level right behind its first level (one base register per table).
// A lane row = its block's 64 coefficients + dummy slots + its AC code-length counters (one 32-bit word per
// length): a lane only touches its own row, so the result-less shared atomic is conflict-free and nothing
// waits on it; the counters are summed into LaneHdr::histo once per (MCU, component).
struct LaneHdr {
    uint32_t histo[6][17];
    LaneTabs t;
};
static_assert(sizeof(LaneHdr) % 16 == 0, "the lane rows behind LaneHdr are read as uint4");
static inline size_t lane_smem_bytes(uint32_t nl)
{
    return sizeof(LaneHdr) + (size_t)LN_WARPS * 32 * ROW_PITCH + (size_t)nl * LN_TAB * 2;
}

// Bit window as two 32-bit registers (hi = next 32 bits, lo = the 32 after), funnel-shift consume; one word in flight behind it.
struct Win {
    uint32_t hi, lo; int nb; uint32_t nx; uint32_t idx; const uint32_t* base;
    __device__ __forceinline__ void init(const uint8_t* b) { init_at(b, 0); }
    // start at absolute bit `bitpos` of the interval (virtual restart intervals): idx stays an absolute word index,
    // so consumed() is the absolute bit position
    __device__ __forceinline__ void init_at(const uint8_t* b, uint32_t bitpos) {
        base = reinterpret_cast<const uint32_t*>(b);
        const uint32_t w = bitpos >> 5;
        hi = __ldg(base + w); lo = __ldg(base + w + 1);
        nx = __ldg(base + w + 2); idx = w + 3; nb = 64;
        consume(bitpos & 31);
    }
    // Top up when 32 bits or fewer are left (6 <= nb then).  The look-ahead word is reloaded IN PLACE by a
    // predicated load: written as a C++ conditional, the compiler loads into a temporary and copies it into
    // `nx` at the end of the same step, i.e. waits for the global load it was supposed to hide (22 % of the
    // kernel's stall samples in the round-1 profile).
    __device__ __forceinline__ void refill_if_low() {
        const uint32_t need = (nb <= 32) ? 1u : 0u;
        if (need) {
            hi |= __funnelshift_rc(nx, 0, nb);             // nx >> nb, 0 when nb == 32
            lo = __funnelshift_rc(0, nx, nb);              // nx << (32 - nb), nx when nb == 32
            nb += 32;
        }
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p ld.global.nc.u32 %0, [%1];\n\t}" : "+r"(nx) : "l"(base + idx), "r"(need));
        idx += need;
    }
    __device__ __forceinline__ void consume(uint32_t n) { hi = __funnelshift_l(lo, hi, n); lo <<= n; nb -= (int)n; }
    __device__ __forceinline__ uint32_t consumed() const { return 32u * (idx - 1) - (uint32_t)nb; }
};

// GENERIC = false: the common case compiled without run-time feature checks (AC decode on, 8-bit
// precision).  GENERIC = true: DC-only mode and 12-bit precision honoured at run time.
// HISTO: also count code lengths per (class, table) (CimgDecode::m_anDhtHisto, ImgDecode.cpp:1217).
// VSEG: the lanes decode VIRTUAL restart intervals — the 4096-bit slots of long real intervals, whose first MCU start,
// MCU index and DC predictors the self-synchronising passes found (jsgpu_phuff_core.cuh) — instead of real ones.
template <bool GENERIC, bool HISTO, bool VSEG>
__global__ void __launch_bounds__(LN_WARPS * 32, 3) k_huff_lane(DevBatch b)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    LaneHdr& sh = *reinterpret_cast<LaneHdr*>(smem_raw);
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint8_t* const rows0 = smem_raw + sizeof(LaneHdr);
    uint16_t* const lutb = reinterpret_cast<uint16_t*>(rows0 + LN_WARPS * 32 * ROW_PITCH);
    uint8_t* const myrows = rows0 + wid * 32 * ROW_PITCH;
    uint8_t* const myrow = myrows + lane * ROW_PITCH;
    for (uint32_t i = lane; i < 32 * ROW_PITCH / 4; i += 32) reinterpret_cast<uint32_t*>(myrows)[i] = 0;
    const bool want_ac = GENERIC ? (b.decode_ac != 0) : true;
    uint32_t cur_img = 0xffffffffu, cur_sig = 0xffffffffu, cur_set = 0xffffffffu;
    const uint32_t nit = VSEG ? b.nvitems : b.nlitems;
    for (uint32_t it = blockIdx.x; it < nit; it += gridDim.x) {      // strided: images of different entropy spread over all CTAs
        const uint2 item = VSEG ? b.vitems[it] : b.litems[it];       // (image, first interval or slot); JS_LANE_SEGS of them per item
        const DevImage& gim = b.img[item.x];
        const DevTableSet* ts = b.tables + gim.table_set;
        if (item.x != cur_img) {
            __syncthreads();
            if (HISTO && cur_img != 0xffffffffu) { flush_histo(b, cur_img, sh.histo); __syncthreads(); }
            if (HISTO) for (uint32_t i = threadIdx.x; i < 6 * 17; i += blockDim.x) (&sh.histo[0][0])[i] = 0;
            if (gim.tab_sig != cur_sig || gim.table_set != cur_set) {   // a different table selection: restage
                lane_stage(sh.t, lutb, gim, ts);
                cur_sig = gim.tab_sig; cur_set = gim.table_set;
            }
            cur_img = item.x;
            __syncthreads();
        }
        const uint32_t kbase = item.y + wid * 32;
        if (kbase >= (VSEG ? gim.ph_nslots : gim.nseg)) continue;   // warp-uniform
        const uint32_t k = kbase + lane;
        const uint32_t ns = gim.ns, ri = gim.ri, nmcu = gim.nmcu, mcu_xmax = gim.mcu_xmax;
        const uint32_t pshift = (GENERIC && gim.precision > 8) ? gim.precision - 8 : 0;
        bool live, vfinal = true; uint32_t sidx, m0, nm, nm_max;
        int dc0 = 0, dc1 = 0, dc2 = 0;
        Win s;
        if (!VSEG) {
            live = k < gim.nseg;
            sidx = gim.seg_first + (live ? k : kbase);
            s.init(b.ubits + b.seg_uoff[sidx]);
            m0 = k * ri;
            nm = live ? (min(m0 + ri, nmcu) - m0) : 0;               // MCUs this lane decodes
            nm_max = min(ri, nmcu - kbase * ri);                     // longest interval in this warp (the first lane's)
        } else {
            PhSegs sg; sg.start = b.seg_start + gim.seg_first; sg.ulen = b.seg_ulen + gim.seg_first; sg.uoff = b.seg_uoff + gim.seg_first; sg.nseg = gim.nseg;
            PhSlots a; a.x = b.ph_x + gim.ph_first; a.ver = b.ph_ver + gim.ph_first; a.k = b.ph_k + gim.ph_first;
            a.cnt = b.ph_cnt + gim.ph_first; a.aux = b.ph_aux + gim.ph_first; a.pre = b.ph_pre + gim.ph_first;
            PhVseg v; v.k = 0; v.bit = 0; v.m0 = 0; v.nm = 0; v.dc0 = v.dc1 = v.dc2 = 0; v.final = false;
            live = (k < gim.ph_nslots) && ph_vseg(sg, ri, nmcu, a, k, v);
            sidx = gim.seg_first + (live ? v.k : 0u);
            s.init_at(b.ubits + b.seg_uoff[sidx], live ? v.bit : 0u);
            m0 = live ? v.m0 : 0u; nm = live ? v.nm : 0u; vfinal = v.final;
            if (live) { dc0 = v.dc0; dc1 = v.dc1; dc2 = v.dc2; }
            nm_max = __reduce_max_sync(FULL, nm);
            if (nm_max == 0) continue;                               // warp-uniform
        }
        uint32_t mx = m0 % mcu_xmax, my = m0 / mcu_xmax;
        uint32_t status = 0;
        const uint32_t avail = b.seg_ulen[sidx] * 8;
        #pragma unroll 1
        for (uint32_t mi = 0; mi < nm_max; mi++) {
            bool mlive = (mi < nm) && !(status & 7);
            if (mlive && s.consumed() > avail) { status |= 2; mlive = false; }     // ran off the end of the interval (corrupt or truncated data): stop reading
            if (mlive) b.mcu_bitpos[gim.mcu_off + m0 + mi] = s.consumed();
            #pragma unroll 1
            for (uint32_t c = 0; c < ns; c++) {
                const uint16_t* lut_dc = lutb + sh.t.li[c * 2] * LN_TAB;
                const uint16_t* lut_ac = lutb + sh.t.li[c * 2 + 1] * LN_TAB;
                const uint32_t* qz = sh.t.qz[c];
                const uint32_t nh = gim.H[c], nv = gim.V[c], cw = gim.cw[c];
                const uint32_t ehc = gim.eh[c], evc = gim.ev[c], blk_xmax = gim.blk_xmax, mcu_ymax = gim.mcu_ymax;
                int16_t* const blkmap = ((c == 0) ? b.blk_y : (c == 1) ? b.blk_cb : b.blk_cr) + gim.blk_off;
                int dc = (c == 0) ? dc0 : (c == 1) ? dc1 : dc2;
                uint32_t bh = 0, bv = 0;
                #pragma unroll 1
                for (uint32_t bi = 0; bi < nh * nv; bi++) {
                    bool active = mlive && !(status & 7);
                    uint32_t pos = 64;
                    if (active) {
                        // ---- DC symbol ----
                        s.refill_if_low();
                        uint32_t e = lut_dc[s.hi >> (32 - JS_LUT_BITS)];
                        if (e & 0x8000) e = lut_dc[JS_LUT_SIZE + (e & 0x7FFF) + ((s.hi >> 16) & ((1u << JS_LUT2_BITS) - 1))];
                        if (e == 0) { status |= 1; active = false; }
                        else {
                            const uint32_t len = e >> 8, run = (e >> 4) & 15, size = e & 15;
                            if (HISTO) atomicAdd(&sh.histo[c * 2][len], 1u);
                            s.consume(len);
                            s.refill_if_low();          // a 16-bit code + 16 value bits can exceed what is left
                            const uint32_t t = s.hi;
                            const uint32_t v = (size == 0) ? 0u : (t >> (32 - size));
                            int val = (int)v - (((int)~t >> 31) & (int)((1u << size) - 1));
                            s.consume(size);
                            if (GENERIC && pshift) val /= (1 << pshift);
                            const uint32_t q = qz[run];
                            const int cf = (int)(short)(val * (int)(q & 0xFFFF));
                            const uint32_t nat = q >> 16;
                            int dcdiff = 0;
                            if (nat == 0) dcdiff = cf;
                            else if (want_ac) *reinterpret_cast<uint16_t*>(myrow + nat * 2) = (uint16_t)cf;    // run-nibble DC symbol: an AC value (none in DC-only mode)
                            dc = (int)(short)(dc + dcdiff);
                            pos = 1 + run;
                        }
                    }
                    // ---- AC symbols: every lane advances its own interval by one symbol per step ----
                    uint32_t emin = 0xffffffffu;                 // an entry of 0 (no code has this prefix) also ends the block like an EOB
                    auto ac_step = [&]() {

                            s.refill_if_low();
                            uint32_t e = lut_ac[s.hi >> (32 - JS_LUT_BITS)];
                            if (e & 0x8000) e = lut_ac[JS_LUT_SIZE + (e & 0x7FFF) + ((s.hi >> 16) & ((1u << JS_LUT2_BITS) - 1))];
                            const uint32_t len = e >> 8, size = e & 15, run = (e >> 4) & 15;
                            if (HISTO) atomicAdd(reinterpret_cast<uint32_t*>(myrow + (ROW_HIST - 4)) + len, 1u);
                            emin = min(emin, e);
                            // value bits follow the code: take them from the window before consuming both at once
                            const uint32_t t = __funnelshift_l(s.lo, s.hi, len);
                            uint32_t v; asm("shr.u32 %0, %1, %2;" : "=r"(v) : "r"(t), "r"(32u - size));   // 0 when size == 0 (shift clamps at 32)
                            uint32_t msk; asm("shr.u32 %0, %1, %2;" : "=r"(msk) : "r"(0xffffffffu), "r"(32u - size));
                            int val = (int)v - (((int)~t >> 31) & (int)msk);
                            if (GENERIC && pshift) val /= (1 << pshift);
                            s.consume(len + size);
                            const uint32_t kk = pos + run;
                            const uint32_t q = qz[kk];                                   // kk <= 78; entries >= 64 point at dummy slots
                            if (want_ac) *reinterpret_cast<uint16_t*>(myrow + (q >> 16) * 2) = (uint16_t)(val * (int)(q & 0xFFFF));
                            pos = ((e & 0xFF) == 0) ? 128u : kk + 1;                     // EOB ends the block (its dummy store hit slot >= 64 or rewrote 0*q)
                    };
                    while (__any_sync(FULL, pos < 64)) {       // two symbols per vote: the second step is simply predicated off where the block ended
                        if (pos < 64) ac_step();
                        if (pos < 64) ac_step();
                    }
                    if (emin == 0) status |= 1;
                    if (pos > 64 && pos < 128) status |= 4;
                    const uint32_t v = bv, h = bh;                        // block (h, v) inside the MCU, kept incrementally (no division)
                    if (++bh == nh) { bh = 0; bv++; }
                    if (active) {
                        *reinterpret_cast<uint16_t*>(myrow) = (uint16_t)dc;
                        if (blk_dc_kept(h, v, ehc, evc, mx, my, mcu_xmax, mcu_ymax))
                            blkmap[(my * evc + v) * blk_xmax + (mx * ehc + h)] = (int16_t)dc;
                    }
                    // ---- cooperative write-out: 4 rows per step, 16 bytes per lane, then re-zero ----
                    const unsigned long long myaddr = active ? (unsigned long long)((gim.coef_row[c] + (size_t)(my * nv + v) * cw + (mx * nh + h)) * 128) : ~0ull;
                    __syncwarp();
                    #pragma unroll
                    for (int r = 0; r < 8; r++) {
                        const int src = r * 4 + (lane >> 3);
                        unsigned long long a = __shfl_sync(FULL, myaddr, src);
                        uint4* sp = reinterpret_cast<uint4*>(myrows + src * ROW_PITCH + (lane & 7) * 16);
                        uint4 val = *sp;
                        *sp = make_uint4(0, 0, 0, 0);
                        if (a != ~0ull) *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(b.coef) + a + (lane & 7) * 16) = val;
                    }
                    __syncwarp();
                }
                if (c == 0) dc0 = dc; else if (c == 1) dc1 = dc; else dc2 = dc;
                if (HISTO) {
                    // lane l sums AC length (l & 15) + 1 over lanes [16 * (l >> 4), +16); rotated so that the 32 lanes hit 32 banks
                    __syncwarp();
                    uint8_t* hp = myrows + (lane >> 4) * 16 * ROW_PITCH + ROW_HIST + (lane & 15) * 4;
                    uint32_t tot = 0;
                    #pragma unroll
                    for (int k2 = 0; k2 < 16; k2++) { uint32_t* q = reinterpret_cast<uint32_t*>(hp + ((k2 + lane) & 15) * ROW_PITCH); tot += *q; *q = 0; }
                    tot += __shfl_xor_sync(FULL, tot, 16);
                    if (lane < 16 && tot) atomicAdd(&sh.histo[c * 2 + 1][lane + 1], tot);
                    __syncwarp();
                }
            }
            if (++mx == mcu_xmax) { mx = 0; my++; }
        }
        if (live) {
            const uint32_t consumed = s.consumed();
            if (!VSEG) {
                status = seg_end_status(status, consumed, avail);
                b.seg_endbits[sidx] = consumed;
                b.seg_status[sidx] = status;
                if (status) atomicOr(&b.img_status[item.x], status);
            } else {
                if (vfinal) {                                   // the virtual interval that ends the real one reports its end state
                    status = seg_end_status(status, consumed, avail);
                    b.seg_endbits[sidx] = consumed;
                }
                if (status) { atomicOr(&b.seg_status[sidx], status); atomicOr(&b.img_status[item.x], status); }   // cleared by k_ph_scan
            }
        }
    }
    __syncthreads();
    if (HISTO && cur_img != 0xffffffffu) flush_histo(b, cur_img, sh.histo);
}

template <bool VSEG>
static int launch_lane(const DevBatch& b, int sm_count, cudaStream_t s)
{
    static bool attr_set[JS_MAX_DEVICES] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (dev >= 0 && dev < JS_MAX_DEVICES && !attr_set[dev]) {       // the attribute is per device
        const int mx = (int)lane_smem_bytes(6);
        cudaFuncSetAttribute(k_huff_lane<false, false, VSEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        cudaFuncSetAttribute(k_huff_lane<true, false, VSEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        cudaFuncSetAttribute(k_huff_lane<false, true, VSEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        cudaFuncSetAttribute(k_huff_lane<true, true, VSEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        attr_set[dev] = true;
    }
    const size_t smem = lane_smem_bytes(b.lane_nlut);
    const uint32_t nit = VSEG ? b.nvitems : b.nlitems;
    uint32_t grid = (uint32_t)sm_count * 3;
    if (grid > nit) grid = nit;
    const bool generic = !b.decode_ac || b.any_p12;
    const dim3 blk(LN_WARPS * 32);
    if (b.want_histo) {
        if (generic) k_huff_lane<true, true, VSEG><<<grid, blk, smem, s>>>(b); else k_huff_lane<false, true, VSEG><<<grid, blk, smem, s>>>(b);
    } else {
        if (generic) k_huff_lane<true, false, VSEG><<<grid, blk, smem, s>>>(b); else k_huff_lane<false, false, VSEG><<<grid, blk, smem, s>>>(b);
    }
    return 1;
}

int js_launch_huffman_lane(const DevBatch& b, int sm_count, cudaStream_t s)
{
    if (b.nlitems == 0) return 0;
    if (!b.lane_l2_smem) return js_launch_huffman_warp(b, sm_count, s);   // a second level too large to stage (pathological DHT): the warp kernel reads it from global memory
    return launch_lane<false>(b, sm_count, s);
}

int js_launch_huffman_lane_vseg(const DevBatch& b, int sm_count, cudaStream_t s)
{
    if (b.nvitems == 0) return 0;
    return launch_lane<true>(b, sm_count, s);
}
