// jsgpu_kernels.cu — hand-written sm_90a kernels of the scan-decode path.
//
// Pipeline (one batch, all images at once; DESIGN.md §4):
//   K0 k_marker_scan      find RSTn markers / end of scan per image      (replaces the lazy RST
//                         detection of BuffAddByte, ImgDecode.cpp:1402-1434)
//   K1 k_huff_warp        entropy decode, ONE WARP PER RESTART INTERVAL  (ReadScanVal /
//      k_huff_lane        DecodeScanComp / DecodeIdctSet, ImgDecode.cpp:1072-1286,1604-1800,
//                         2270-2303) -> dequantised int16 coefficient rows, slot 0 = running DC
//   K2 k_idct_*           IDCT + level shift + chroma replication + YCC->RGB (DecodeIdctCalc*,
//                         SetFullRes, CalcChannelPreviewFull: :2372-2423,2468-2561,4619-4821)
//   K3 k_finalize_*       block-DC maps, MCU file map, brightest pixel / average luma
//
// Bit-exactness rules used throughout: integer sums wrap mod 2^32 (C int overflow of the
// reference is two's complement on every target it ran on); int16 stores truncate; float
// colour math uses __fmul_rn/__fadd_rn/__fsub_rn/__fdiv_rn so no FMA contraction can happen.
#include "jsgpu_internal.h"
#include "jsgpu_ycc.cuh"
#include "jsgpu_detail.cuh"     // js_raw_of_unstuffed
#include <cstdio>
#include <cstdlib>
#include <algorithm>

#define FULL 0xffffffffu

// ------------------------------------------------------------------------------------------------
// K0: marker scan.  What both forms share: the load of 16 scan bytes, the recording of RST markers and the close-out of an image.
// ------------------------------------------------------------------------------------------------
// the 16 scan bytes at `off` as four little-endian words, zero beyond the scan's n bytes (scan_off is 16-byte aligned)
template <typename U>
__device__ __forceinline__ uint4 ms_load16(const uint8_t* p, U off, U n)
{
    if (off + 16 <= n) return __ldg(reinterpret_cast<const uint4*>(p + off));
    uint32_t w[4] = {0, 0, 0, 0};
    if (off < n) for (int i = 0; i < 16; i++) if (off + i < n) w[i >> 2] |= (uint32_t)p[off + i] << (8 * (i & 3));
    return make_uint4(w[0], w[1], w[2], w[3]);
}

// RST markers of image ii (bit i of `mask`: a marker at scan offset pos0 + i), numbered from `rank` on: interval `rank` ends at
// the marker and the next one starts behind it.  seg_start / seg_end: the image's nseg intervals.
template <typename M>
__device__ __forceinline__ void ms_record_rst(const DevBatch& b, uint32_t ii, uint32_t* seg_start, uint32_t* seg_end, uint32_t nseg,
                                              const uint8_t* p, M mask, uint32_t pos0, uint32_t rank)
{
    while (mask) {
        const uint32_t i = (uint32_t)((sizeof(M) == 8) ? __ffsll((long long)mask) : __ffs((int)mask)) - 1; mask &= mask - 1;
        const uint32_t pos = pos0 + i;
        if (rank < nseg) seg_end[rank] = pos;
        if (rank + 1 < nseg) seg_start[rank + 1] = pos + 2;
        if (((uint32_t)p[pos + 1] & 7u) != (rank & 7u)) atomicOr(&b.img_status[ii], 32u);    // out of sequence: the reference logs it (ImgDecode.cpp:1414-1424)
        rank++;
    }
}

// the scan of image ii ends at endpos after `found` RST markers: the last found interval runs to the end, the ones no marker
// delimits are empty there
__device__ __forceinline__ void ms_close(const DevBatch& b, uint32_t ii, const DevImage& im, uint32_t found, uint32_t endpos)
{
    uint32_t* const seg_start = b.seg_start + im.seg_first;
    uint32_t* const seg_end = b.seg_end + im.seg_first;
    const uint32_t nf = found + 1;                // intervals delimited by the markers found
    if (nf <= im.nseg) seg_end[nf - 1] = endpos;
    for (uint32_t k = nf; k < im.nseg; k++) { seg_start[k] = endpos; seg_end[k] = endpos; }
    b.scan_end[ii] = endpos;
    b.nseg_found[ii] = nf;
    b.stats[(size_t)ii * 16 + 11] = (int32_t)found;    // m_nRestartRead (ImgDecode.cpp:1414)
    if (nf < im.nseg) atomicOr(&b.img_status[ii], 8u);
    if (nf > im.nseg) atomicOr(&b.img_status[ii], 32u);        // more restart markers than intervals: the reference restarts at each one it meets
}

// one CTA per image walks the scan bytes in order
#define MS_THREADS 512
__global__ void __launch_bounds__(MS_THREADS) k_marker_scan(DevBatch b)
{
    const DevImage& im = b.img[blockIdx.x];
    if (!im.valid) return;
    __shared__ uint32_t s_warp[MS_THREADS / 32];
    __shared__ uint32_t s_term;
    const uint8_t* p = b.bits + im.scan_off;
    const uint64_t n = im.scan_len;
    const uint32_t t = threadIdx.x, lane = t & 31, wid = t >> 5;
    uint32_t* seg_start = b.seg_start + im.seg_first;
    uint32_t* seg_end   = b.seg_end + im.seg_first;
    if (t == 0) seg_start[0] = 0;
    uint32_t found = 0;            // RST markers accepted so far (uniform after each iteration)
    uint32_t term = 0xffffffffu;
    // 64 bytes per thread and iteration (32 KB per CTA pass): three barriers per pass, so few of them per image
    for (uint64_t base = 0; base < n; base += MS_THREADS * 64) {
        if (t == 0) s_term = 0xffffffffu;
        __syncthreads();
        const uint64_t off0 = base + (uint64_t)t * 64;
        uint4 v[4];
        #pragma unroll
        for (int c = 0; c < 4; c++) v[c] = ms_load16(p, off0 + 16 * c, n);
        uint32_t nextb = __shfl_down_sync(FULL, v[0].x, 1) & 0xFF;        // first byte of the next thread's chunk
        if (lane == 31) nextb = (off0 + 64 < n) ? p[off0 + 64] : 0;
        unsigned long long mask = 0;        // bit i: RST marker starts at off0+i
        uint32_t myterm = 0xffffffffu;
        #pragma unroll
        for (int c = 0; c < 4; c++) {
            // FF bytes are rare (~1/200): test a whole word for "any byte == FF" first and only then look at its bytes
            const uint32_t ws[5] = {v[c].x, v[c].y, v[c].z, v[c].w, (c < 3) ? v[c < 3 ? c + 1 : 3].x : nextb};
            #pragma unroll
            for (int wi = 0; wi < 4; wi++) {
                const uint32_t w = ws[wi];
                if (((~w - 0x01010101u) & w & 0x80808080u) == 0) continue;     // no byte of w is 0xFF
                #pragma unroll
                for (int j = 0; j < 4; j++) {
                    if (((w >> (8 * j)) & 0xFF) != 0xFF) continue;
                    const int i = c * 16 + wi * 4 + j;
                    if (off0 + i + 1 >= n) continue;
                    const uint32_t m = (j < 3) ? ((w >> (8 * j + 8)) & 0xFF) : (ws[wi + 1] & 0xFF);
                    if (m >= 0xD0 && m <= 0xD7) mask |= 1ull << i;
                    else if (m != 0x00 && m != 0xFF && myterm == 0xffffffffu) myterm = (uint32_t)(off0 + i);
                }
            }
        }
        if (myterm != 0xffffffffu) atomicMin(&s_term, myterm);
        __syncthreads();
        term = s_term;
        if (term != 0xffffffffu) {          // drop markers at/after the terminating marker
            if (off0 >= term) mask = 0;
            else if (term - off0 < 64) mask &= (1ull << (uint32_t)(term - off0)) - 1ull;
        }
        uint32_t cnt = __popcll(mask);
        // block exclusive scan of cnt
        uint32_t inc = cnt;
        #pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(FULL, inc, d); if (lane >= d) inc += y; }
        if (lane == 31) s_warp[wid] = inc;
        __syncthreads();
        uint32_t wbase = 0, total = 0;
        #pragma unroll
        for (int w = 0; w < MS_THREADS / 32; w++) { uint32_t y = s_warp[w]; if (w < wid) wbase += y; total += y; }
        ms_record_rst(b, blockIdx.x, seg_start, seg_end, im.nseg, p, mask, (uint32_t)off0, found + wbase + inc - cnt);
        found += total;
        if (term != 0xffffffffu) break;
        __syncthreads();                    // s_warp / s_term are rewritten by the next pass
    }
    __syncthreads();
    if (t == 0) ms_close(b, blockIdx.x, im, found, (term != 0xffffffffu) ? term : (uint32_t)n);
}

// ------------------------------------------------------------------------------------------------
// K0 (chunked form, the default): the same result from ONE parallel pass.  A warp takes the next 4096-byte chunk of the batch (a
// ticket, so chunks are taken in order), finds its RSTn markers and its first other marker with byte-parallel compares, and gets
// the number of RST markers in the image's earlier chunks by decoupled look-back: every chunk publishes "my own count" at once and
// "count of everything up to me" as soon as it knows it, and a chunk that needs its predecessors reads back through those words, 32
// at a time, until it meets one that already holds a running total.  The combining rule carries the end of scan: markers behind
// the first terminating marker do not count.  Replaces the CTA-per-image walk with its three barriers per 32 KB.
// ------------------------------------------------------------------------------------------------
#define MC_CHUNK 4096u
#define MC_AGG   (1ull << 62)               // status: own aggregate published
#define MC_PFX   (2ull << 62)               // status: inclusive prefix published
#define MC_TERM  (1ull << 61)               // a terminating marker lies in the covered range
__device__ __forceinline__ unsigned long long mc_combine(unsigned long long left, unsigned long long right)
{
    // (count, term) pairs, left range before right range: behind a terminator nothing counts
    if (left & MC_TERM) return left & (MC_TERM | 0xffffffffull);
    return ((left + right) & 0xffffffffull) | (right & MC_TERM);
}
__device__ __forceinline__ uint32_t mc_nib(uint32_t m) { return (((m & 0x01010101u) * 0x01020408u) >> 24) & 15u; }   // one flag per byte -> 4 bits

__global__ void __launch_bounds__(256) k_marker_scan2(DevBatch b)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long* const ticket = b.mc_state + b.mc_total;
    __shared__ uint32_t s_base;
    for (;;) {
        // one ticket per CTA and round (eight consecutive chunks, one per warp): a ticket per warp is 156 K atomics on one address
        __syncthreads();
        if (threadIdx.x == 0) s_base = (uint32_t)atomicAdd(ticket, 8ull);
        __syncthreads();
        if (s_base >= b.mc_total) return;
        const uint32_t c = s_base + wid;
        if (c >= b.mc_total) continue;
        const uint32_t ii = b.mc_img[c];
        const DevImage& im = b.img[ii];
        const uint32_t ci = c - (uint32_t)im.mc_first;                  // chunk index inside the image
        const uint8_t* p = b.bits + im.scan_off;
        const uint32_t n = (uint32_t)im.scan_len, base = ci * MC_CHUNK;
        // 16-byte pieces r*32 + lane of the chunk (coalesced), zero beyond the scan
        uint4 v[8];
        #pragma unroll
        for (int r = 0; r < 8; r++) v[r] = ms_load16(p, base + (uint32_t)(r * 32 + lane) * 16, n);
        const uint32_t after = (base + MC_CHUNK < n) ? (uint32_t)p[base + MC_CHUNK] : 0u;      // the byte behind the chunk
        // per piece: bit i of rst / trm = byte i is an FF followed by D0..D7 / by anything but 00, FF, D0..D7 (and not the last byte of the scan)
        uint32_t rst[8], trm[8];
        #pragma unroll
        for (int r = 0; r < 8; r++) {
            uint32_t nextw = __shfl_down_sync(FULL, v[r].x, 1);                                  // first word of the next piece
            const uint32_t wrap = (r < 7) ? __shfl_sync(FULL, v[r < 7 ? r + 1 : 7].x, 0) : after;
            if (lane == 31) nextw = wrap;
            const uint32_t ws[5] = { v[r].x, v[r].y, v[r].z, v[r].w, nextw };
            uint32_t mr = 0, mt = 0;
            #pragma unroll
            for (int wi = 0; wi < 4; wi++) {
                const uint32_t w = ws[wi], nw = __byte_perm(w, ws[wi + 1], 0x4321);             // byte j = the byte after w's byte j
                const uint32_t isff = __vcmpeq4(w, 0xFFFFFFFFu);
                const uint32_t isd = __vcmpeq4(nw & 0xF8F8F8F8u, 0xD0D0D0D0u);
                const uint32_t skip = isd | __vcmpeq4(nw, 0u) | __vcmpeq4(nw, 0xFFFFFFFFu);
                mr |= mc_nib(isff & isd) << (4 * wi);
                mt |= mc_nib(isff & ~skip) << (4 * wi);
            }
            // an FF that is the last byte of the scan has no marker byte
            const uint32_t off = base + (uint32_t)(r * 32 + lane) * 16;
            const uint32_t valid = (off + 16 < n) ? 0xFFFFu : (off + 1 < n) ? ((1u << (n - 1 - off)) - 1u) : 0u;
            rst[r] = mr & valid; trm[r] = mt & valid;
        }
        // first terminating marker of the chunk (position inside the chunk), RST markers before it
        uint32_t myterm = 0xffffffffu;
        #pragma unroll
        for (int r = 7; r >= 0; r--) if (trm[r]) myterm = (uint32_t)(r * 32 + lane) * 16 + (uint32_t)__ffs(trm[r]) - 1;
        const uint32_t cterm = __reduce_min_sync(FULL, myterm);
        uint32_t cntp[8], total = 0;                  // exclusive rank of each of my pieces among the chunk's RST markers
        #pragma unroll
        for (int r = 0; r < 8; r++) {
            if (cterm != 0xffffffffu) {                // drop markers at / behind the terminator
                const uint32_t pos0 = (uint32_t)(r * 32 + lane) * 16;
                if (pos0 >= cterm) rst[r] = 0; else if (cterm - pos0 < 16) rst[r] &= (1u << (cterm - pos0)) - 1u;
            }
            const uint32_t cnt = __popc(rst[r]);
            uint32_t inc = cnt;
            #pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(FULL, inc, d); if (lane >= d) inc += y; }
            cntp[r] = total + inc - cnt;
            total += __shfl_sync(FULL, inc, 31);
        }
        // ---- look-back ----
        const unsigned long long mine = (unsigned long long)total | ((cterm != 0xffffffffu) ? MC_TERM : 0ull);
        unsigned long long excl = 0;                   // aggregate of the image's chunks before this one
        volatile unsigned long long* const st = b.mc_state + im.mc_first;
        if (ci == 0) { if (lane == 0) { __threadfence(); st[0] = mine | MC_PFX; } }
        else {
            if (lane == 0) { __threadfence(); st[ci] = mine | MC_AGG; }
            int hi = (int)ci - 1;                      // window [hi-31, hi], lane l looks at hi - l
            bool done = false;
            while (!done) {
                const int idx = hi - (int)lane;
                unsigned long long w = 0;
                do { w = (idx >= 0) ? st[idx] : MC_PFX; } while (__any_sync(FULL, (w >> 62) == 0));       // all 32 published (or before the image)
                // nearest predecessor that holds a running total ends the walk; combine everything from there up to hi
                const uint32_t pf = __ballot_sync(FULL, (w >> 62) == 2);
                const int stop = pf ? (__ffs(pf) - 1) : 31;             // lane index (distance from hi) of the first prefix word
                unsigned long long acc = (idx >= 0 && (int)lane <= stop) ? (w & (MC_TERM | 0xffffffffull)) : 0ull;
                // ordered reduction: lane `stop` is leftmost ... lane 0 rightmost; fold right-to-left so that left ranges come first
                #pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const unsigned long long o = __shfl_down_sync(FULL, acc, d);       // lanes further right? no: lane+d is further LEFT in the file
                    if ((int)lane + d <= stop) acc = mc_combine(o, acc);
                }
                const unsigned long long win = __shfl_sync(FULL, acc, 0);               // chunks [hi-stop, hi]
                excl = mc_combine(win, excl);
                if (pf || hi - 31 <= 0) done = true; else hi -= 32;
            }
            if (lane == 0) { __threadfence(); st[ci] = mc_combine(excl, mine) | MC_PFX; }
        }
        excl = __shfl_sync(FULL, excl, 0);
        const bool dead = (excl & MC_TERM) != 0;       // the scan ended in an earlier chunk: nothing here counts
        const uint32_t found0 = (uint32_t)(excl & 0xffffffffull);
        uint32_t* const seg_start = b.seg_start + im.seg_first;
        uint32_t* const seg_end = b.seg_end + im.seg_first;
        if (!dead) {
            if (ci == 0 && lane == 0) seg_start[0] = 0;
            #pragma unroll
            for (int r = 0; r < 8; r++) ms_record_rst(b, ii, seg_start, seg_end, im.nseg, p, rst[r], base + (uint32_t)(r * 32 + lane) * 16, found0 + cntp[r]);
            // the chunk that holds the end of the scan — the first terminating marker, or the last chunk when there is none — closes the image
            const bool last = (ci + 1 == im.mc_n);
            if ((cterm != 0xffffffffu || last) && lane == 0) ms_close(b, ii, im, found0 + total, (cterm != 0xffffffffu) ? base + cterm : n);
        }
    }
}

int js_launch_marker_scan(const DevBatch& b, uint64_t max_scan_len, cudaStream_t s)
{
    if (b.nimg == 0) return 0;
    // Which form: the CTA-per-image walk is the faster one when there are many images of similar size (cfg2);
    // the chunked pass wins when a few CTAs would do all the work — a single image (the drop-in class), fewer images than the
    // device holds CTAs, or sizes so uneven that the largest images set the time (cfg4).
    static const int mode = [] { const char* e = getenv("JSGPU_MARKER"); return e ? atoi(e) : 2; }();       // 0 = per image, 1 = chunked, 2 = choose
    const bool uneven = (unsigned long long)max_scan_len * b.nimg > 2ull * b.bits_len;
    const bool chunked = b.mc_total != 0 && (mode == 1 || (mode == 2 && (b.nimg < 2 * JS_H100_SMS || uneven)));
    if (!chunked) { k_marker_scan<<<b.nimg, MS_THREADS, 0, s>>>(b); return 1; }
    cudaMemsetAsync(b.mc_state, 0, ((size_t)b.mc_total + 1) * 8, s);
    uint32_t grid = (b.mc_total + 7) / 8;
    if (grid > JS_H100_SMS * 8u) grid = JS_H100_SMS * 8u;
    k_marker_scan2<<<grid, 256, 0, s>>>(b);
    return 1;
}

// ------------------------------------------------------------------------------------------------
// K2 (simple form): straightforward IDCT and colour kernels.  These are the readable,
// obviously-correct statement of Appendix A.8-A.10 of SURVEY.md on the device; the fused tiled
// kernel (js_launch_idct_fused) is checked against them and against the CPU oracle.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_idct_simple(DevBatch b, const int32_t* __restrict__ li, const float* __restrict__ lf)
{
    // one thread per (block, sample); blockIdx.y = image, strided beyond 65535 images
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {
    const DevImage& im = b.img[ii];
    if (!im.valid || (b.simple_only_nonstd && im.std_layout)) continue;
    uint32_t nblk = im.nmcu * im.bpm;
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < nblk * 64; g += gridDim.x * blockDim.x) {
        uint32_t blk = g >> 6, yx = g & 63;
        // block -> (comp, bx, by)
        uint32_t c = 0, r = blk;
        for (; c < im.ns; c++) { uint32_t n = im.cw[c] * im.ch[c]; if (r < n) break; r -= n; }
        uint32_t bx = r % im.cw[c], by = r / im.cw[c];
        const int16_t* row = b.coef + (im.coef_row[c] + r) * 64;
        int dc = row[0];
        int out;
        if (b.idct_mode == 0) {
            uint32_t s = 0;
            for (int vu = 1; vu < 64; vu++) s += (uint32_t)(li[yx * 64 + vu] * (int)row[vu]);     // DecodeIdctCalcFixedpt, :2402-2423
            int n = (int)s; n /= 4; n >>= 10;
            short nv = (short)n; nv = (short)(nv * 8 + dc);                                          // SetFullRes, :2513-2515
            out = nv;
        } else {
            float f = 0.f;
            for (int vu = 1; vu < 64; vu++) f = __fadd_rn(f, __fmul_rn(lf[yx * 64 + vu], (float)row[vu]));   // :2381-2383
            f = __fmul_rn(f, 0.25f);
            short nv = (short)((short)(int)__fmul_rn(f, 8.0f) + dc);                          // float -> int (cvttss2si) -> short, as the x86 build does                                   // :2517-2519
            out = nv;
        }
        // destination (SetFullRes addressing, :2498-2557)
        uint32_t mx = bx / im.H[c], h = bx % im.H[c], my = by / im.V[c], v = by % im.V[c];
        uint32_t x = yx & 7, y = yx >> 3;
        uint32_t px0 = mx * im.mcu_w + h * 8 + x * im.eh[c];
        uint32_t py0 = my * im.mcu_h + v * 8 + y * im.ev[c];
        int16_t* map = ((c == 0) ? b.pix_y : (c == 1) ? b.pix_cb : b.pix_cr) + im.pix_off;
        // A component with 1 < H < Hmax (or V) replicates each of its blocks over 8*eh x 8*ev pixels but places them only 8 apart, so
        // inside an MCU its blocks OVERLAP; the reference writes them one after the other (v outer, h inner, :3340-3400), the later
        // block wins.  Here every pixel is written by exactly that block: the last one in (v,h) order that covers it.
        for (uint32_t iv = 0; iv < im.ev[c]; iv++) for (uint32_t ih = 0; ih < im.eh[c]; ih++) {
            uint32_t px = px0 + ih, py = py0 + iv;
            const uint32_t dx = px - mx * im.mcu_w, dy = py - my * im.mcu_h;
            if (h != min(im.H[c] - 1, dx >> 3) || v != min(im.V[c] - 1, dy >> 3)) continue;
            if (px < im.wp && py < im.hp) map[(size_t)py * im.wp + px] = (int16_t)out;
        }
    }
    }
}

__global__ void __launch_bounds__(256) k_color_simple(DevBatch b)
{
    // CalcChannelPreviewFull (ImgDecode.cpp:4693-4792), PREVIEW_RGB, no preview shift; strided beyond 65535 images
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {
    const DevImage& im = b.img[ii];
    if (!im.valid || (b.simple_only_nonstd && im.std_layout)) continue;     // uniform over the CTA: the shuffles below stay full-warp
    const uint32_t npx = im.wp * im.hp;
    unsigned long long best = 0, sum = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += gridDim.x * blockDim.x) {
        uint32_t px = i % im.wp, py = i / im.wp;
        int ty = b.pix_y[im.pix_off + i], tcb = 0, tcr = 0;
        if (im.ns == 3) { tcb = b.pix_cb[im.pix_off + i]; tcr = b.pix_cr[im.pix_off + i]; }
        const YccFast o = ycc_fast(ty, tcb, tcr);
        uint32_t inv = im.hp - 1 - py;
        reinterpret_cast<uint32_t*>(b.dib + im.dib_off)[(size_t)inv * im.wp + px] = o.b | (o.g << 8) | (o.r << 16);   // [B,G,R,0], :4786-4789
        sum += (uint32_t)(o.y + 128);
        unsigned long long key = ((unsigned long long)(uint32_t)(ty + 32768) << 32) | (0xffffffffu - i);        // first strict max in raster order
        best = max(best, key);
    }
    for (int d = 16; d; d >>= 1) { best = max(best, __shfl_xor_sync(FULL, best, d)); sum += __shfl_xor_sync(FULL, sum, d); }
    if ((threadIdx.x & 31) == 0) { atomicMax(&b.bright_key[ii], best); atomicAdd(&b.sum_y[ii], sum); }
    }
}

int js_launch_idct_simple(const DevBatch& b, const int32_t* li, const float* lf, cudaStream_t s)
{
    if (b.nimg == 0) return 0;
    dim3 grid(2048, std::min<uint32_t>(b.nimg, 65535u));
    k_idct_simple<<<grid, 256, 0, s>>>(b, li, lf);
    k_color_simple<<<grid, 256, 0, s>>>(b);
    return 2;
}

// ------------------------------------------------------------------------------------------------
// K3: finalisation — scalar statistics (ImgDecode.cpp:4802-4819) and the MCU file map.  (The block-DC maps,
// :3524-3608, are written by the Huffman kernels.)
// ------------------------------------------------------------------------------------------------
__global__ void k_finalize_stats(DevBatch b)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b.nimg) return;
    const DevImage& im = b.img[i];
    int32_t* st = b.stats + (size_t)i * 16;
    if (!im.valid) return;
    unsigned long long key = b.bright_key[i], sum = b.sum_y[i];
    uint32_t idx = 0xffffffffu - (uint32_t)(key & 0xffffffffu);
    int by = (int)(uint32_t)(key >> 32) - 32768;
    int bcb = 0, bcr = 0;
    if (im.ns == 3) { bcb = b.pix_cb[im.pix_off + idx]; bcr = b.pix_cr[im.pix_off + idx]; }
    if (by == -32768) { bcb = bcr = -32768; idx = 0; }      // no pixel beat the initial m_nBrightY (:4664-4667, strict '>')
    const YccFast o = ycc_fast(by, bcb, bcr);
    st[0] = (int32_t)(uint32_t)sum; st[1] = (int32_t)(uint32_t)(sum >> 32);
    unsigned long long npix = (unsigned long long)(im.hp + 1) * (im.wp + 1);      // :4690 (sic)
    st[2] = (int32_t)((uint32_t)sum / npix);                                       // nSumY is a 32-bit unsigned, :4635
    st[3] = by; st[4] = bcb; st[5] = bcr; st[6] = (int32_t)o.r; st[7] = (int32_t)o.g; st[8] = (int32_t)o.b;
    st[9] = (int32_t)((idx % im.wp) / im.mcu_w); st[10] = (int32_t)((idx / im.wp) / im.mcu_h);
    // Where the accumulator stands after the last MCU (m_anScanBuffPtr_pos[0], m_nScanBuffPtr_align: the reference's
    // "Next position in scan buffer" and compression-ratio lines, ImgDecode.cpp:3659-3667, 3726): inside the last interval's
    // data while bits of it remain, else on the FF of the marker that ends the scan (BuffAddByte keeps it as data, :1527-1561).
    if (!b.ex_flag[i] && im.nseg) {
        const uint32_t k = im.nseg - 1, sidx = im.seg_first + k, D = b.seg_ulen[sidx], eb = b.seg_endbits[sidx];
        uint32_t pos;
        if ((eb >> 3) < D) pos = im.file_pos + b.seg_start[sidx] + js_raw_of_unstuffed(b, im, k, eb >> 3);
        else pos = im.file_pos + b.scan_end[i] + ((eb >> 3) - D);
        st[12] = (int32_t)pos; st[13] = (int32_t)(eb & 7);
        st[14] = (int32_t)(im.file_pos + b.scan_end[i]);
    }
}

// MCU file map (ImgDecode.cpp:3229, 5104-5113): m_pMcuFileMap[m] = (file position of the byte
// holding the accumulator's head bit << 4) + bit offset, sampled when MCU m starts.  K1 records
// the UNSTUFFED bit offset of every MCU start inside its restart interval; here one warp per
// interval re-walks the raw bytes (32 per step, kept-byte ranks from one ballot) and turns
// unstuffed byte indices into file offsets.  Quirks reproduced (SURVEY.md A.11): the first MCU
// after an RSTn records the state reached at the END of the previous interval because the
// reference handles restarts lazily (:1644-1680); when an interval is consumed to its last bit
// the emptied accumulator keeps the position of the last byte it loaded, alignment 0 (:934-953).
__global__ void __launch_bounds__(128) k_finalize_mcumap(DevBatch b)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t novf = *b.ovf_count;                     // intervals k_finalize_mcumap_fast could not do (list from k_unstuff)
    for (uint32_t oi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; oi < novf; oi += (gridDim.x * blockDim.x) >> 5) {
    const uint32_t gw = b.ovf_list[oi];
    uint32_t lo = 0, hi = b.nimg - 1;                       // image owning segment gw
    while (lo < hi) { uint32_t mid = (lo + hi + 1) >> 1; if (b.img[mid].seg_first <= gw) lo = mid; else hi = mid - 1; }
    const DevImage& im = b.img[lo];
    if (!im.valid || b.ex_flag[lo]) continue;
    const uint32_t k = gw - im.seg_first;
    if (k >= im.nseg) continue;
    const uint32_t s0 = b.seg_start[gw], len = b.seg_end[gw] - s0;
    const uint8_t* seg = b.bits + im.scan_off + s0;
    const uint32_t m0 = k * im.ri, m1 = min(m0 + im.ri, im.nmcu);
    // targets t = 0..nt-1: MCU m0+t for t < m1-m0 (t = 0 only for the very first interval),
    // then the end state of this interval, which belongs to MCU m1.
    const uint32_t nown = m1 - m0;
    const uint32_t nt = nown + ((m1 < im.nmcu) ? 1u : 0u);
    uint32_t tcur = (k == 0) ? 0u : 1u;
    auto tbits = [&](uint32_t t) -> uint32_t { return (t < nown) ? b.mcu_bitpos[im.mcu_off + m0 + t] : b.seg_endbits[gw]; };
    auto tmcu  = [&](uint32_t t) -> uint32_t { return (t < nown) ? (m0 + t) : m1; };
    uint32_t tgt = (tcur < nt) ? tbits(tcur) : 0;
    uint32_t ubase = 0, prev_ff = 0, last_kept = 0;
    for (uint32_t base = 0; base < len && tcur < nt; base += 32) {
        bool in = base + lane < len;
        uint32_t bj = in ? seg[base + lane] : 0;
        uint32_t pj = __shfl_up_sync(FULL, bj, 1);
        if (lane == 0) pj = prev_ff ? 0xFFu : 0u;
        bool kept = in && !(bj == 0 && pj == 0xFF && (base + lane) > 0);
        uint32_t km = __ballot_sync(FULL, kept);
        uint32_t pre = __popc(km & ((1u << lane) - 1)), tot = __popc(km);
        prev_ff = (__shfl_sync(FULL, bj, 31) == 0xFF) ? 1u : 0u;
        while (tcur < nt && (tgt >> 3) < ubase + tot) {
            uint32_t u = (tgt >> 3) - ubase;
            uint32_t hit = __ballot_sync(FULL, kept && pre == u);
            uint32_t raw = base + (uint32_t)(__ffs(hit) - 1);
            if (lane == 0) b.mcu_map[im.mcu_off + tmcu(tcur)] = ((im.file_pos + s0 + raw) << 4) + (tgt & 7);
            tcur++;
            tgt = (tcur < nt) ? tbits(tcur) : 0;
        }
        if (km) last_kept = base + (31 - __clz(km));
        ubase += tot;
    }
    // targets at (or past) the end of the data: accumulator emptied
    while (tcur < nt) {
        if (lane == 0) b.mcu_map[im.mcu_off + tmcu(tcur)] = (len ? ((im.file_pos + s0 + last_kept) << 4) : 0u);
        tcur++;
    }
    }
}

// Fast MCU file map: one thread per MCU, using the stuffed-byte list k_unstuff recorded per interval
// (raw offset of unstuffed byte u = u + number of stuffed zeros before it).  Intervals with more
// stuffed bytes than the list holds are left to k_finalize_mcumap (the raw re-walk above).
__global__ void __launch_bounds__(256) k_finalize_mcumap_fast(DevBatch b)
{
    for (uint32_t ii = blockIdx.y; ii < b.nimg; ii += gridDim.y) {      // strided beyond 65535 images
    const DevImage& im = b.img[ii];
    if (!im.valid || b.ex_flag[ii]) continue;                 // damaged image: k_huff_exact wrote its map
    for (uint32_t m = blockIdx.x * blockDim.x + threadIdx.x; m < im.nmcu; m += gridDim.x * blockDim.x) {
        uint32_t k = m / im.ri, t = m - k * im.ri, bit;
        if (t > 0) bit = b.mcu_bitpos[im.mcu_off + m];
        else if (k == 0) bit = 0;
        else { k -= 1; bit = b.seg_endbits[im.seg_first + k]; }       // lazy restart: end state of the previous interval
        const uint32_t sidx = im.seg_first + k;
        const uint32_t ns = b.seg_nstuff[sidx];
        if (ns > JS_STUFF_LIST && !im.psync) continue;                  // handled by the raw re-walk kernel (long intervals: row table below)
        const uint32_t D = b.seg_ulen[sidx];
        uint32_t u = bit >> 3, al = bit & 7;
        uint32_t val;
        if (u >= D) {                                                   // accumulator emptied (ImgDecode.cpp:934-953)
            if (D < 4) { val = 0; b.mcu_map[im.mcu_off + m] = val; continue; }   // pos[] still holds the zeros of the last reset
            u = D - 1; al = 0;
        }
        const uint32_t raw = js_raw_of_unstuffed(b, im, k, u);
        val = ((im.file_pos + b.seg_start[sidx] + raw) << 4) + al;
        b.mcu_map[im.mcu_off + m] = val;
    }
    }
}

// The MCU file map needs nothing from the IDCT: its kernels go on a second stream next to K2 (jsgpu_api.cu), only the scalar
// statistics (brightest pixel, luma sum) wait for it.
int js_launch_finalize_maps(const DevBatch& b, cudaStream_t s)
{
    if (b.nimg == 0 || !b.mcu_map || !b.nseg_total) return 0;
    dim3 grid(32, std::min<uint32_t>(b.nimg, 65535u));
    k_finalize_mcumap_fast<<<grid, 256, 0, s>>>(b);
    k_finalize_mcumap<<<std::min<uint32_t>((b.nseg_total + 3) / 4, JS_H100_SMS * 8), 128, 0, s>>>(b);      // walks the overflow list only
    return 2;
}
int js_launch_finalize_stats(const DevBatch& b, cudaStream_t s)
{
    if (b.nimg == 0) return 0;
    k_finalize_stats<<<(b.nimg + 127) / 128, 128, 0, s>>>(b);
    return 1;
}

// ------------------------------------------------------------------------------------------------
// Output checksums (jsgpu_batch_checksums): one 64-bit sum per output buffer of every image, computed where the
// outputs live, so that a batch caller (bench.py verifies EVERY image of EVERY rank this way) can compare a whole
// batch with the reference's CPU decode without moving 21 MB per image over PCIe.  The sum is over 32-bit words w_i
// (16-bit buffers: two elements per word, an odd last element zero-extended) of mix(w_i, i): order-independent to
// accumulate, position-sensitive.  tests/oracle harness (oracle/ref_harness.cpp: ck_words) computes the same.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ck_mix(uint32_t w, unsigned long long i)
{
    unsigned long long x = (unsigned long long)w + (i + 1ull) * 0x9E3779B97F4A7C15ull;
    x ^= x >> 32; x *= 0xD6E8FEB86659FD93ull; x ^= x >> 29;
    return x;
}
// words [0, nfull) of p, plus (odd16) the low half of word nfull
__device__ __forceinline__ unsigned long long ck_span(const uint32_t* p, unsigned long long nfull, bool odd16, unsigned long long first, unsigned long long step)
{
    unsigned long long s = 0;
    for (unsigned long long i = first; i < nfull; i += step) s += ck_mix(__ldg(p + i), i);
    if (odd16 && first == 0) s += ck_mix((uint32_t)reinterpret_cast<const uint16_t*>(p)[2 * nfull], nfull);
    return s;
}
__global__ void __launch_bounds__(256) k_checksums(DevBatch b, unsigned long long* ck)
{
    __shared__ unsigned long long s_red[8];
    const uint32_t ii = blockIdx.y;
    const DevImage& im = b.img[ii];
    if (!im.valid) return;
    const unsigned long long first = blockIdx.x * blockDim.x + threadIdx.x, step = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long npx = (unsigned long long)im.wp * im.hp, nblk = (unsigned long long)im.blk_xmax * im.blk_ymax;
    for (int w = 0; w < 10; w++) {
        unsigned long long s = 0;
        const bool c3 = im.ns == 3;
        switch (w) {
        case 0: s = ck_span(reinterpret_cast<const uint32_t*>(b.pix_y + im.pix_off), npx >> 1, npx & 1, first, step); break;
        case 1: if (c3) s = ck_span(reinterpret_cast<const uint32_t*>(b.pix_cb + im.pix_off), npx >> 1, npx & 1, first, step); break;
        case 2: if (c3) s = ck_span(reinterpret_cast<const uint32_t*>(b.pix_cr + im.pix_off), npx >> 1, npx & 1, first, step); break;
        case 3: s = ck_span(reinterpret_cast<const uint32_t*>(b.dib + im.dib_off), npx, false, first, step); break;
        case 4: s = ck_span(reinterpret_cast<const uint32_t*>(b.blk_y + im.blk_off), nblk >> 1, nblk & 1, first, step); break;
        case 5: if (c3) s = ck_span(reinterpret_cast<const uint32_t*>(b.blk_cb + im.blk_off), nblk >> 1, nblk & 1, first, step); break;
        case 6: if (c3) s = ck_span(reinterpret_cast<const uint32_t*>(b.blk_cr + im.blk_off), nblk >> 1, nblk & 1, first, step); break;
        case 7: s = ck_span(b.mcu_map + im.mcu_off, im.nmcu, false, first, step); break;
        case 8: s = ck_span(b.histo + (size_t)ii * 2 * 4 * 17, 2 * 4 * 17, false, first, step); break;
        case 9: s = ck_span(reinterpret_cast<const uint32_t*>(b.stats + (size_t)ii * 16 + 2), 9, false, first, step); break;    // m_nAvgY, brightest pixel Y/Cb/Cr/R/G/B, its MCU
        }
        #pragma unroll
        for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(FULL, s, d);
        if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long t = 0;
            for (int q = 0; q < 8; q++) t += s_red[q];
            if (t) atomicAdd(&ck[(size_t)ii * JSGPU_CK_WORDS_INTERNAL + w], t);
        }
        __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        ck[(size_t)ii * JSGPU_CK_WORDS_INTERNAL + 10] = b.img_status[ii];
        ck[(size_t)ii * JSGPU_CK_WORDS_INTERNAL + 11] = ((unsigned long long)im.wp << 32) | im.hp;
    }
}

int js_launch_checksums(const DevBatch& b, unsigned long long* ck, cudaStream_t s)
{
    if (b.nimg == 0) return 0;
    cudaMemsetAsync(ck, 0, (size_t)b.nimg * JSGPU_CK_WORDS_INTERNAL * 8, s);
    for (uint32_t i0 = 0; i0 < b.nimg; i0 += 65535u) {           // grid.y limit
        DevBatch bb = b; bb.img = b.img + i0; bb.nimg = std::min<uint32_t>(b.nimg - i0, 65535u);
        bb.histo = b.histo + (size_t)i0 * 2 * 4 * 17; bb.stats = b.stats + (size_t)i0 * 16; bb.img_status = b.img_status + i0;
        k_checksums<<<dim3(32, bb.nimg), 256, 0, s>>>(bb, ck + (size_t)i0 * JSGPU_CK_WORDS_INTERNAL);
    }
    return 1;
}
