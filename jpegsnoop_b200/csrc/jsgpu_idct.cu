// jsgpu_idct.cu — stage B, fused: dequantised coefficients -> IDCT -> level shift -> chroma replication ->
// int16 Y/Cb/Cr maps + BGRA DIB + brightest-pixel / luma-sum statistics, one pass, nothing re-read from HBM.
// (DecodeIdctCalcFixedpt / DecodeIdctCalcFloat + SetFullRes + CalcChannelPreviewFull, ImgDecode.cpp:2372-2423, 2468-2561,
// 4619-4821.)
//
// Work unit = one TILE: one MCU row x (32/Hmax) MCUs, i.e. 32 luma blocks wide.  One tile kernel, k_idct_tile<P1, EHS>, walks
// the tiles for every IDCT arithmetic; P1 is the phase-1 policy (how one block's coefficients become samples), EHS the chroma
// replication of phase 2.  Phase 1 gives every LANE ONE 8x8 BLOCK (a warp = 32 horizontally adjacent blocks of one component
// row).  Phase 2 (whole CTA): the tile's samples, staged in shared memory as planes, are read back 8 pixels per thread and
// leave as 16-byte stores: three int16 map rows and two BGRA quads (phase2x, jsgpu_idct_common.cuh).  The policy only changes
// phase 1 and how many CTAs per SM the kernel is built for; shared-memory layout, thread count and grid size are the same.
#include "jsgpu_idct_common.cuh"
#include "build/idct_baked.h"
#include "build/idct_baked_f.h"
#include <cstring>

// Launch shape: 4 warps per CTA — three take one 32-block group each in phase 1 (a 4:2:0 tile has 64 Y + 16 Cb + 16 Cr
// blocks), all four share phase 2, whose 8 chroma-row groups then split evenly.  Coefficient rows are not prefetched into
// registers for the next tile: that would cost 32 registers, and at 96 registers x 128 threads x 5 CTAs, 20 warps per SM
// instead of 15 hide the same latency better.
#define IDCT_THREADS 128

// Phase-1 policies (JsTileIdct):
//
// Integer IDCT (the -DIDCT_FIXEDPT build), table in shared memory (JS_TILE_INT_SMEM) or as immediates (JS_TILE_INT_BAKED):
//   * the reference IDCT is s[yx] = sum_{vu>=1} Li[yx][vu]*c[vu], with Li = (int)(Lf*1024) — not separable, so no row/column
//     factorisation is bit-exact.  But Li is mirror-symmetric up to a few entries: Li[y][7-x][v][u] = (-1)^u Li[y][x][v][u]
//     (same in y/v) except where float rounding of the host cosf made the two halves truncate differently.  The host splits
//     Li = S + D (IdctSym); S needs only the 4x4 quadrant: each coefficient is accumulated into one of four parity accumulators
//     per quadrant sample (16 MACs instead of 64), four outputs per quadrant sample come from a butterfly, and D (non-zero for
//     <= 4 coefficient positions; 3 with glibc) is added per output.  All integer, wrapping mod 2^32 like the reference's int.
//   * the table entry is warp-uniform (every lane works on the same (sample, coefficient) pair of a different block), so it is
//     fetched by broadcast LDS.128 or, when the host table equals the build-time copy, baked into the instruction stream as
//     immediates; the MAC loop is fully unrolled with static accumulator indices: ~1 IMAD per MAC, no per-coefficient control
//     flow.  The shared-memory table is what runs when the host libm's table differs from the build-time copy.
//
// Float IDCT (JS_TILE_FLOAT; the reference's shipping default: DecodeIdctCalcFloat, ImgDecode.cpp:2372-2392; SetFullRes' float
// branch :2517-2519): the reference adds the 63 products of a sample one at a time, in natural index order, each product and
// each sum rounded to fp32 (x86-64 SSE scalar code, no FMA: oracle/Makefile).  Float addition is not associative, so there is no
// symmetric shortcut: every sample needs its own 63 multiply + 63 add, in that order.  What is exact: (a) skipping a coefficient
// that is zero in all 32 blocks of the warp (a sum that starts at +0 is never -0, so adding a +-0 product changes nothing);
// (b) the table as instruction immediates (build/idct_baked_f.h), used only when it equals, bit for bit, the table the host
// class computed with its libm (js_idctf_baked_matches) — otherwise the image takes the literal kernels (k_idct_simple).
// 64 fp32 accumulators per lane.
//
// CTAs per SM the kernel is built for: the float IDCT needs more registers.
static constexpr int idct_min_ctas(JsTileIdct p1) { return p1 == JS_TILE_FLOAT ? 4 : 5; }

template <JsTileIdct P1, int EHS>
__global__ void __launch_bounds__(IDCT_THREADS, idct_min_ctas(P1)) k_idct_tile(DevBatch b, const IdctSym* __restrict__ sym, const ColorTabs* __restrict__ ctab,
                                                                                uint32_t tile_first, uint32_t tile_count)
{
    extern __shared__ __align__(16) uint8_t smem[];
    Idct2Tables& T = *reinterpret_cast<Idct2Tables*>(smem);
    uint8_t* const planes0 = smem + sizeof(Idct2Tables) + sizeof(TileGeo);    // two plane buffers: one barrier per tile (see the loop)
    const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // stage the tables once per CTA
    if (P1 == JS_TILE_INT_SMEM) {
        for (uint32_t i = tid; i < 64 * 4; i += blockDim.x) T.s4[i] = reinterpret_cast<const int4*>(sym->s4)[i];
        for (uint32_t i = tid; i < 64; i += blockDim.x) T.corrT[i] = make_int4(sym->corr[0][i], sym->corr[1][i], sym->corr[2][i], sym->corr[3][i]);
    }
    if (tid == 0) {
        if (P1 == JS_TILE_FLOAT) T.ncorr = 0;
        else { T.ncorr = sym->ncorr; for (int j = 0; j < 4; j++) T.corr_pos[j] = sym->corr_pos[j]; }
        T.rb_ok = ctab->rb_ok;
    }
    for (uint32_t i = tid; i < 256; i += blockDim.x) { T.tr[i] = (int16_t)(ctab->tr[i] - 128); T.tb[i] = (int16_t)(ctab->tb[i] - 128); }
    __syncthreads();
    const int ncorr = T.ncorr;

    TileGeo& G = *reinterpret_cast<TileGeo*>(smem + sizeof(Idct2Tables));
    uint32_t cur_img = 0xffffffffu;
    // per-thread statistics of the current image, kept across its tiles: brightest pixel (key + value) and the luma sum
    unsigned long long best = 0; int bestm = -0x7fffffff - 1; uint32_t acc_y = 0;
    auto flush_stats = [&](uint32_t img) {
        unsigned long long s64 = acc_y;
        #pragma unroll
        for (int d = 16; d; d >>= 1) { best = max(best, __shfl_xor_sync(FULL, best, d)); s64 += __shfl_xor_sync(FULL, s64, d); }
        if (lane == 0 && best) { atomicMax(&b.bright_key[img], best); atomicAdd(&b.sum_y[img], s64); }
        best = 0; bestm = -0x7fffffff - 1; acc_y = 0;
    };
    // Each CTA walks a contiguous run of tiles (same image for hundreds of tiles: descriptor loads hit L1,
    // coefficient rows and output rows advance sequentially).
    const uint32_t t_begin = (uint32_t)(((unsigned long long)tile_count * blockIdx.x) / gridDim.x);
    const uint32_t t_end = (uint32_t)(((unsigned long long)tile_count * (blockIdx.x + 1)) / gridDim.x);

    for (uint32_t ti = t_begin; ti < t_end; ti++) {
        const uint4 tile = b.tiles[tile_first + ti];       // (image, mcu row, first mcu col, mcus in tile)
        if (tile.x != cur_img) {                           // block-uniform; once or twice per CTA
            if (cur_img != 0xffffffffu) flush_stats(cur_img);
            __syncthreads();
            if (tid == 0) {
                const DevImage& gi = b.img[tile.x];
                G.ns = gi.ns; G.tile_mcus = gi.tile_mcus; G.mcu_w = gi.mcu_w; G.mcu_h = gi.mcu_h; G.wp = gi.wp; G.hp = gi.hp;
                G.evc = (gi.ns == 3) ? gi.ev[1] : 1; G.pix_off = gi.pix_off; G.dib_off = gi.dib_off;
                for (int c = 0; c < 3; c++) { G.H[c] = gi.H[c]; G.V[c] = gi.V[c]; G.cw[c] = gi.cw[c]; G.coef_row[c] = gi.coef_row[c]; }
            }
            __syncthreads();
            cur_img = tile.x;
        }
        const TileGeo& im = G;
        // Sample planes are double-buffered: phase 1 of tile t+1 may start while slower warps still read tile t's
        // planes in phase 2; it cannot run further ahead than the barrier of tile t+1, which every warp reaches
        // only after finishing phase 2 of tile t, so the buffer written for tile t+2 is free by then.
        uint8_t* const planes = planes0 + ((ti - t_begin) & 1) * b.tile_plane_bytes;
        const uint32_t ns = im.ns, U = im.tile_mcus;
        const uint32_t trow = tile.y, mcol0 = tile.z, nmt = tile.w;
        // per-component tile geometry
        // (scalars, not arrays: runtime-indexed arrays would live in local memory)
        const uint32_t hu0 = im.H[0] * U, hu1 = (ns == 3) ? im.H[1] * U : 0, hu2 = (ns == 3) ? im.H[2] * U : 0;
        const uint32_t cnt0 = hu0 * im.V[0], cnt1 = hu1 * im.V[1], cnt2 = hu2 * im.V[2];
        const uint32_t pbase0 = 0, pbase1 = cnt0 * 128, pbase2 = (cnt0 + cnt1) * 128;
        const uint32_t ppitch0 = hu0 * 16, ppitch1 = hu1 * 16, ppitch2 = hu2 * 16;
        const uint32_t nblk = cnt0 + cnt1 + cnt2;
        // ---------------- phase 1: one block per lane ----------------
        for (uint32_t g = wid; g * 32 < nblk; g += (blockDim.x >> 5)) {
            uint32_t i = g * 32 + lane;
            uint32_t c = 0;
            if (i >= cnt0) { i -= cnt0; c = 1; if (i >= cnt1) { i -= cnt1; c = 2; } }
            if (c >= ns) c = 0;                                    // lanes past the last block (never valid)
            const uint32_t Hc = im.H[c];
            const uint32_t huc = (c == 0) ? hu0 : (c == 1) ? hu1 : hu2;
            const uint32_t pbc = (c == 0) ? pbase0 : (c == 1) ? pbase1 : pbase2;
            const uint32_t ppc = (c == 0) ? ppitch0 : (c == 1) ? ppitch1 : ppitch2;
            const uint32_t v = i / huc, col = i - v * huc;
            const bool valid = (g * 32 + lane < nblk) && (col < nmt * Hc);
            const size_t row = im.coef_row[c] + (size_t)(trow * im.V[c] + v) * im.cw[c] + (mcol0 * Hc + col);
            uint4 cw4[8];
            if (valid) {
                const uint4* rp = reinterpret_cast<const uint4*>(b.coef + row * 64);
                #pragma unroll
                for (int k = 0; k < 8; k++) cw4[k] = __ldg(rp + k);
            } else {
                #pragma unroll
                for (int k = 0; k < 8; k++) cw4[k] = make_uint4(0, 0, 0, 0);
            }
            const uint32_t* cw = reinterpret_cast<const uint32_t*>(cw4);
#define JS_COEF(n) (((n) & 1) ? ((int)cw[(n) >> 1] >> 16) : (int)(short)(cw[(n) >> 1] & 0xFFFF))
            if (P1 == JS_TILE_FLOAT) {
                const int dc = (int)(short)(cw[0] & 0xFFFF);
                float acc[64];
                #pragma unroll
                for (int q = 0; q < 64; q++) acc[q] = 0.0f;
#define JS_CF(n) ((float)JS_COEF(n))
#define JS_NZ(n) (__any_sync(FULL, ((n) & 1) ? (cw[(n) >> 1] >> 16) != 0u : (cw[(n) >> 1] & 0xFFFFu) != 0u))
                JS_BAKED_FMACS(acc, JS_CF, JS_NZ)
#undef JS_CF
#undef JS_NZ
                uint8_t* pl = planes + pbc + (v * 8) * ppc + col * 16;
                #pragma unroll
                for (int y = 0; y < 8; y++) {
                    uint32_t o[8];
                    #pragma unroll
                    for (int x = 0; x < 8; x++) {
                        const float f = __fmul_rn(acc[y * 8 + x], 0.25f);                                   // fSum *= 0.25 (:2388)
                        o[x] = (uint32_t)((int)(short)(int)__fmul_rn(f, 8.0f) + dc) & 0xFFFFu;               // (short)(f*8) + dc, stored to a short (:2517-2519)
                    }
                    if (valid) *reinterpret_cast<uint4*>(pl + y * ppc) = make_uint4(o[0] | (o[1] << 16), o[2] | (o[3] << 16), o[4] | (o[5] << 16), o[6] | (o[7] << 16));
                }
                continue;
            }
            const uint32_t dc2 = __byte_perm(cw[0], 0, 0x1010);    // the DC predictor sum in both halves
            int acc[4][16];
            #pragma unroll
            for (int p = 0; p < 4; p++)
                #pragma unroll
                for (int q = 0; q < 16; q++) acc[p][q] = 0;
            if (P1 == JS_TILE_INT_BAKED) {
                JS_BAKED_MACS(acc, JS_COEF)                       // 63 x 16 IMADs with immediate operands
            } else {
                #pragma unroll
                for (int n = 1; n < 64; n++) {
                    const int cn = JS_COEF(n);
                    const int p = ((n >> 3) & 1) * 2 + (n & 1);        // parity class of (v,u)
                    #pragma unroll
                    for (int gq = 0; gq < 4; gq++) {
                        const int4 t = T.s4[n * 4 + gq];               // warp-uniform
                        acc[p][gq * 4 + 0] += t.x * cn; acc[p][gq * 4 + 1] += t.y * cn;
                        acc[p][gq * 4 + 2] += t.z * cn; acc[p][gq * 4 + 3] += t.w * cn;
                    }
                }
            }
            // corrections: coefficients at the (<=4) positions whose table entries are not mirror-symmetric
            int cj[4] = {0, 0, 0, 0};
            if (P1 == JS_TILE_INT_SMEM && valid) {
                const int16_t* r16 = b.coef + row * 64;
                #pragma unroll
                for (int j = 0; j < 4; j++) if (j < ncorr) cj[j] = r16[T.corr_pos[j]];
            }
            // butterfly + finalise + store this block's 8 rows into the component plane
            uint8_t* pl = planes + pbc + (v * 8) * ppc + col * 16;
            #pragma unroll
            for (int y = 0; y < 4; y++) {
                uint32_t top[8], bot[8];
                #pragma unroll
                for (int x = 0; x < 4; x++) {
                    const int q = y * 4 + x;
                    const int a00 = acc[0][q], a01 = acc[1][q], a10 = acc[2][q], a11 = acc[3][q];
                    const int A = a00 + a01, B = a00 - a01, C2 = a10 + a11, D = a10 - a11;
                    int s0 = A + C2, s1 = B + D, s2 = A - C2, s3 = B - D;     // (y,x) (y,7-x) (7-y,x) (7-y,7-x)
                    if (P1 == JS_TILE_INT_BAKED) {         // the baked table's asymmetric entries, as immediates (a few +-coefficient adds)
                        int t0, t1, t2, t3;
                        JS_BAKED_CORR_TERM(y * 8 + x, JS_COEF, t0) JS_BAKED_CORR_TERM(y * 8 + 7 - x, JS_COEF, t1)
                        JS_BAKED_CORR_TERM((7 - y) * 8 + x, JS_COEF, t2) JS_BAKED_CORR_TERM((7 - y) * 8 + 7 - x, JS_COEF, t3)
                        s0 += t0; s1 += t1; s2 += t2; s3 += t3;
                    } else if (ncorr > 0) {
                        const int4 d0 = T.corrT[y * 8 + x], d1 = T.corrT[y * 8 + 7 - x], d2 = T.corrT[(7 - y) * 8 + x], d3 = T.corrT[(7 - y) * 8 + 7 - x];
                        s0 += d0.x * cj[0] + d0.y * cj[1] + d0.z * cj[2] + d0.w * cj[3];
                        s1 += d1.x * cj[0] + d1.y * cj[1] + d1.z * cj[2] + d1.w * cj[3];
                        s2 += d2.x * cj[0] + d2.y * cj[1] + d2.z * cj[2] + d2.w * cj[3];
                        s3 += d3.x * cj[0] + d3.y * cj[1] + d3.z * cj[2] + d3.w * cj[3];
                    }
                    top[x] = fin_pre(s0); top[7 - x] = fin_pre(s1); bot[x] = fin_pre(s2); bot[7 - x] = fin_pre(s3);
                }
                if (valid) {
                    *reinterpret_cast<uint4*>(pl + y * ppc) = make_uint4(fin_pair(top[0], top[1], dc2), fin_pair(top[2], top[3], dc2), fin_pair(top[4], top[5], dc2), fin_pair(top[6], top[7], dc2));
                    *reinterpret_cast<uint4*>(pl + (7 - y) * ppc) = make_uint4(fin_pair(bot[0], bot[1], dc2), fin_pair(bot[2], bot[3], dc2), fin_pair(bot[4], bot[5], dc2), fin_pair(bot[6], bot[7], dc2));
                }
            }
#undef JS_COEF
        }
        __syncthreads();
        // ---------------- phase 2: 8 pixels x (chroma row group) per thread, vector stores ----------------
        {
            P2x a;
            a.planes = planes; a.pbase1 = pbase1; a.pbase2 = pbase2; a.ppitch0 = ppitch0; a.ppitch1 = ppitch1; a.ppitch2 = ppitch2;
            a.opr = (nmt * im.mcu_w) >> 3; a.px0 = mcol0 * im.mcu_w; a.py0 = trow * im.mcu_h; a.wp = im.wp; a.hp = im.hp; a.mcu_h = im.mcu_h;
            a.mapy = b.pix_y + im.pix_off; a.mapcb = b.pix_cb + im.pix_off; a.mapcr = b.pix_cr + im.pix_off; a.dib = b.dib + im.dib_off;
            a.ns = ns; a.evc = im.evc; a.gflag = ctab->gflag;
            uint32_t sum = 0;                               // packed halves, < 2^16 each within one tile
            phase2x<EHS>(a, T, lane, wid, best, bestm, sum);
            acc_y += (sum & 0xFFFF) + (sum >> 16);
        }
    }
    if (cur_img != 0xffffffffu) flush_stats(cur_img);
}

// ------------------------------------------------------------------------------------------------
// Colour tables.  ConvertYCCtoRGBFastFloat is a function of three 8-bit integers (y,cb,cr after >>3
// and clamping).  Mathematically R = y + 1.402cr + 128, B = y + 1.772cb + 128, G = y - (0.114*1.772cb +
// 0.299*1.402cr)/0.587 + 128, i.e. "y plus a chroma term", and the float evaluation agrees with that
// integer form except where a rounding lands next to an integer.  This kernel evaluates the EXACT float
// routine for all 2^24 inputs on the device, derives the additive terms, and verifies them: tr/tb are
// used only if they reproduce R/B for every (y,c) pair (rb_ok), and each (cb,cr) pair whose G term is
// not valid for all 256 y values is marked 0x7FFF so those pixels take the exact float path.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_build_color_tables(ColorTabs* t)
{
    const int idx = blockIdx.x * 256 + threadIdx.x;          // 0..65535
    const int cb = (idx >> 8) - 128, cr = (idx & 255) - 128;
    // candidate terms from y = 0 (floor of the unclamped float, +128 included)
    float vr0, vg0, vb0; ycc_float_core(0.f, (float)cb, (float)cr, vr0, vg0, vb0);
    const int dR = (int)floorf(vr0), dB = (int)floorf(vb0), dG = (int)floorf(vg0);
    bool okR = true, okB = true, okG = true;
    for (int y = -128; y <= 127; y++) {
        const uint32_t px = ycc_fast_bgra(y << 3, cb << 3, cr << 3);
        const int r = (px >> 16) & 255, g = (px >> 8) & 255, bl = px & 255;
        okR = okR && (r == min(255, max(0, y + dR))); okB = okB && (bl == min(255, max(0, y + dB))); okG = okG && (g == min(255, max(0, y + dG)));
    }
    t->tg[idx] = okG ? (int16_t)dG : (int16_t)0x7FFF;
    if (!okG) atomicAdd(&t->n_unsafe, 1);
    const int cand = (-(JS_GA * cb + JS_GB * cr)) >> 23;               // arithmetic candidate for dG - 128
    if (!okG || cand != dG - 128) { atomicOr(&t->gflag[idx >> 5], 1u << (idx & 31)); atomicAdd(&t->n_gflag, 1); }
    if (cb == 0) { t->tr[cr + 128] = (int16_t)dR; if (!okR) atomicAnd(&t->rb_ok, 0); }
    if (cr == 0) { t->tb[cb + 128] = (int16_t)dB; if (!okB) atomicAnd(&t->rb_ok, 0); }
}

int js_launch_build_color_tables(ColorTabs* t, cudaStream_t s)
{
    cudaMemsetAsync(t, 0, sizeof(ColorTabs), s);
    const int32_t one = 1;
    cudaMemcpyAsync(&t->rb_ok, &one, sizeof one, cudaMemcpyHostToDevice, s);
    cudaStreamSynchronize(s);
    k_build_color_tables<<<256, 256, 0, s>>>(t);
    return 1;
}

int js_idct_baked_matches(const int32_t* li) { return memcmp(li, kBakedLi, sizeof kBakedLi) == 0; }
int js_idctf_baked_matches(const float* lf) { return memcmp(lf, kBakedLfBits, sizeof kBakedLfBits) == 0; }

// One launch per non-empty chroma replication class.
template <JsTileIdct P1>
static int launch_tiles(const DevBatch& b, const IdctSym* sym, const ColorTabs* ctab, int sm_count, cudaStream_t s)
{
    static bool attr_set_dev[JS_MAX_DEVICES] = {};       // the attribute is per device
    int dev = 0; cudaGetDevice(&dev); if (dev < 0 || dev >= JS_MAX_DEVICES) dev = 0;
    if (!attr_set_dev[dev]) {
        const int mx = (int)(sizeof(Idct2Tables) + sizeof(TileGeo) + 48 * 1024);
        cudaFuncSetAttribute(k_idct_tile<P1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        cudaFuncSetAttribute(k_idct_tile<P1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        cudaFuncSetAttribute(k_idct_tile<P1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
        attr_set_dev[dev] = true;
    }
    const size_t smem = sizeof(Idct2Tables) + sizeof(TileGeo) + 2 * (size_t)b.tile_plane_bytes;
    int n = 0;
    for (int cls = 0; cls < 3; cls++) {
        const uint32_t cnt = b.tcls_count[cls];
        if (!cnt) continue;
        uint32_t grid = (uint32_t)sm_count * idct_min_ctas(P1);
        if (grid > cnt) grid = cnt;
        if (cls == 0) k_idct_tile<P1, 0><<<grid, IDCT_THREADS, smem, s>>>(b, sym, ctab, b.tcls_first[cls], cnt);
        else if (cls == 1) k_idct_tile<P1, 1><<<grid, IDCT_THREADS, smem, s>>>(b, sym, ctab, b.tcls_first[cls], cnt);
        else k_idct_tile<P1, 2><<<grid, IDCT_THREADS, smem, s>>>(b, sym, ctab, b.tcls_first[cls], cnt);
        n++;
    }
    return n;
}

int js_launch_idct_fused(const DevBatch& b, const IdctSym* sym, const ColorTabs* ctab, int sm_count, JsTileIdct idct, cudaStream_t s)
{
    switch (idct) {
    case JS_TILE_INT_SMEM:  return launch_tiles<JS_TILE_INT_SMEM>(b, sym, ctab, sm_count, s);
    case JS_TILE_INT_BAKED: return launch_tiles<JS_TILE_INT_BAKED>(b, sym, ctab, sm_count, s);
    default:                return launch_tiles<JS_TILE_FLOAT>(b, sym, ctab, sm_count, s);
    }
}
