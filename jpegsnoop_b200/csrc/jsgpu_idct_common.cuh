// jsgpu_idct_common.cuh — pieces of the fused IDCT+colour tile kernel (k_idct_tile, jsgpu_idct.cu): shared-memory tables,
// sample finalisation, the exact colour routine and the packed-s16x2 phase 2.
#pragma once
#include "jsgpu_internal.h"
#include "jsgpu_ycc.cuh"
#define FULL 0xffffffffu

struct __align__(16) Idct2Tables {
    int4 s4[64 * 4];
    int4 corrT[64];
    int  ncorr; int corr_pos[4];
    int  rb_ok; int pad0, pad1;
    int16_t tr[256], tb[256];            // chroma terms of R and B WITHOUT the +128 level shift
};

// ConvertYCCtoRGBFastFloat for the few pixels the verified tables do not cover; out of line, so that phase 2's hot loop stays small.
static __device__ __noinline__ uint32_t ycc_exact(int py, int pcb, int pcr) { return ycc_fast_bgra(py, pcb, pcr); }

// Sample finalisation, two samples at a time: the reference's (short)(trunc(s/4) >> 10) * 8 + dc.  trunc(s/4) then >>10 is
// (s + bias) >> 12 with bias = 3 when s < 0, and ((s + bias) >> 12) * 8 == ((s + bias) >> 9) & ~7, so after the 32-bit
// bias-and-shift the two results are packed, masked and level-shifted by the DC sum with packed 16-bit operations;
// __viaddmin_s16x2(a, b, 0x7FFF7FFF) is a per-half wrapping add (min with the largest short never clamps), i.e. exactly
// the reference's `short n = n*8 + dc` truncation (ImgDecode.cpp:2513-2515).
__device__ __forceinline__ uint32_t fin_pre(int s) { return (uint32_t)((s - 3 * (s >> 31)) >> 9); }
__device__ __forceinline__ uint32_t fin_pair(uint32_t a, uint32_t b, uint32_t dc2)
{
    return __viaddmin_s16x2(__byte_perm(a, b, 0x5410) & 0xFFF8FFF8u, dc2, 0x7FFF7FFFu);
}

// Per-CTA copy of what the tile loop needs from the current image's descriptor (a CTA walks a contiguous run of
// tiles, i.e. stays on one image for hundreds of tiles: one global read per image instead of per tile).
struct TileGeo {
    uint32_t ns, tile_mcus, H[3], V[3], cw[3], mcu_w, mcu_h, wp, hp, evc, pad;
    unsigned long long coef_row[3], pix_off, dib_off;
};

struct P2x {
    const uint8_t* planes; uint32_t pbase1, pbase2, ppitch0, ppitch1, ppitch2;
    uint32_t opr, px0, py0, wp, hp, mcu_h, ns, evc;
    int16_t* mapy; int16_t* mapcb; int16_t* mapcr; uint8_t* dib; const uint32_t* gflag;
};

// s16x2 helpers
__device__ __forceinline__ uint32_t clamp255_add(uint32_t a, uint32_t b) { return __viaddmin_s16x2_relu(a, b, 0x00FF00FFu); }   // max(min(a+b,255),0) per half
__device__ __forceinline__ uint32_t dup16(int v) { return __byte_perm((uint32_t)v, 0, 0x1010); }
__device__ __forceinline__ uint32_t pack16(int lo, int hi) { return __byte_perm((uint32_t)lo, (uint32_t)hi, 0x5410); }

template <int EHS>
// best/bestm: this thread's brightest-pixel candidate so far, as (value, earliest raster position) key and as plain value;
// the caller may keep them across tiles of one image (ties are resolved on the full key, so processing order does not matter).
__device__ __forceinline__ void phase2x(const P2x& a, const Idct2Tables& T, uint32_t lane, uint32_t wid, unsigned long long& best, int& bestm, uint32_t& sum2)
{
    constexpr int NC = 8 >> EHS;
    const uint32_t nwarps = blockDim.x >> 5;
    const uint32_t px = lane * 8;
    for (uint32_t rg = wid; rg * a.evc < a.mcu_h; rg += nwarps) {
        if (lane >= a.opr) continue;
        uint32_t cbw[4], crw[4];                  // replicated chroma, packed for the map stores (= per-pair chroma)
        uint32_t dR[4], dG[4], dB[4];             // per pixel pair: chroma terms packed s16x2
        uint32_t unsafe = 0;                      // bit k: pixel k must take the exact float routine
        int cs[NC], rs[NC];
        if (a.ns == 3) {
            const uint8_t* pcb = a.planes + a.pbase1 + rg * a.ppitch1 + ((px >> EHS) << 1);
            const uint8_t* pcr = a.planes + a.pbase2 + rg * a.ppitch2 + ((px >> EHS) << 1);
            if (EHS == 0) {
                const uint4 u = *reinterpret_cast<const uint4*>(pcb), v = *reinterpret_cast<const uint4*>(pcr);
                cbw[0] = u.x; cbw[1] = u.y; cbw[2] = u.z; cbw[3] = u.w; crw[0] = v.x; crw[1] = v.y; crw[2] = v.z; crw[3] = v.w;
                #pragma unroll
                for (int j = 0; j < NC; j++) { cs[j] = (j & 1) ? ((int)cbw[j >> 1] >> 16) : (int)(short)(cbw[j >> 1] & 0xFFFF); rs[j] = (j & 1) ? ((int)crw[j >> 1] >> 16) : (int)(short)(crw[j >> 1] & 0xFFFF); }
            } else if (EHS == 1) {
                const uint2 u = *reinterpret_cast<const uint2*>(pcb), v = *reinterpret_cast<const uint2*>(pcr);
                cs[0] = (int)(short)(u.x & 0xFFFF); cs[1] = (int)u.x >> 16; cs[2] = (int)(short)(u.y & 0xFFFF); cs[3] = (int)u.y >> 16;
                rs[0] = (int)(short)(v.x & 0xFFFF); rs[1] = (int)v.x >> 16; rs[2] = (int)(short)(v.y & 0xFFFF); rs[3] = (int)v.y >> 16;
                cbw[0] = __byte_perm(u.x, 0, 0x1010); cbw[1] = __byte_perm(u.x, 0, 0x3232); cbw[2] = __byte_perm(u.y, 0, 0x1010); cbw[3] = __byte_perm(u.y, 0, 0x3232);
                crw[0] = __byte_perm(v.x, 0, 0x1010); crw[1] = __byte_perm(v.x, 0, 0x3232); crw[2] = __byte_perm(v.y, 0, 0x1010); crw[3] = __byte_perm(v.y, 0, 0x3232);
            } else {
                const uint32_t u = *reinterpret_cast<const uint32_t*>(pcb), v = *reinterpret_cast<const uint32_t*>(pcr);
                cs[0] = (int)(short)(u & 0xFFFF); cs[1] = (int)u >> 16; rs[0] = (int)(short)(v & 0xFFFF); rs[1] = (int)v >> 16;
                cbw[0] = cbw[1] = __byte_perm(u, 0, 0x1010); cbw[2] = cbw[3] = __byte_perm(u, 0, 0x3232);
                crw[0] = crw[1] = __byte_perm(v, 0, 0x1010); crw[2] = crw[3] = __byte_perm(v, 0, 0x3232);
            }
        } else {
            #pragma unroll
            for (int j = 0; j < NC; j++) { cs[j] = 0; rs[j] = 0; }
            cbw[0] = cbw[1] = cbw[2] = cbw[3] = 0; crw[0] = crw[1] = crw[2] = crw[3] = 0;
        }
        int tRs[NC], tGs[NC], tBs[NC];
        uint32_t gw[NC], gs[NC];                  // exact-path bitmap words: requested here, looked at after the first row's arithmetic
        #pragma unroll
        for (int j = 0; j < NC; j++) {
            const int cbc = max(-128, min(127, cs[j] >> 3)), crc = max(-128, min(127, rs[j] >> 3));
            const uint32_t gi = (uint32_t)(((cbc + 128) << 8) | (crc + 128));
            tRs[j] = T.tr[crc + 128]; tBs[j] = T.tb[cbc + 128];
            tGs[j] = (-(JS_GA * cbc + JS_GB * crc)) >> 23;                         // verified arithmetic form of the G chroma term
            gw[j] = __ldg(&a.gflag[gi >> 5]); gs[j] = gi & 31;
        }
        #pragma unroll
        for (int p = 0; p < 4; p++) {
            if (EHS == 0)      { dR[p] = pack16(tRs[2 * p], tRs[2 * p + 1]); dG[p] = pack16(tGs[2 * p], tGs[2 * p + 1]); dB[p] = pack16(tBs[2 * p], tBs[2 * p + 1]); }
            else if (EHS == 1) { dR[p] = dup16(tRs[p]); dG[p] = dup16(tGs[p]); dB[p] = dup16(tBs[p]); }
            else               { dR[p] = dup16(tRs[p >> 1]); dG[p] = dup16(tGs[p >> 1]); dB[p] = dup16(tBs[p >> 1]); }
        }
        for (uint32_t r2 = 0; r2 < a.evc; r2++) {
            const uint32_t oy = rg * a.evc + r2;
            const uint4 yv = *reinterpret_cast<const uint4*>(a.planes + oy * a.ppitch0 + px * 2);
            const uint32_t yw[4] = {yv.x, yv.y, yv.z, yv.w};
            const uint32_t ay = a.py0 + oy, ax = a.px0 + px;
            const size_t mi = (size_t)ay * a.wp + ax;
            *reinterpret_cast<uint4*>(a.mapy + mi) = yv;
            if (a.ns == 3) {
                *reinterpret_cast<uint4*>(a.mapcb + mi) = make_uint4(cbw[0], cbw[1], cbw[2], cbw[3]);
                *reinterpret_cast<uint4*>(a.mapcr + mi) = make_uint4(crw[0], crw[1], crw[2], crw[3]);
            }
            uint32_t bgra[8];
            #pragma unroll
            for (int p = 0; p < 4; p++) {
                // per half: (y >> 3) via a biased logical shift, then Y8 = clamp(y>>3, -128, 127) + 128 in one packed op
                const uint32_t u = ((yw[p] ^ 0x80008000u) >> 3) & 0x1FFF1FFFu;              // (y + 32768) >> 3 = (y >> 3) + 4096
                const uint32_t y8 = clamp255_add(u, 0xF080F080u);                            // + (128 - 4096), clamped to 0..255
                const uint32_t rp = clamp255_add(y8, dR[p]), gp = clamp255_add(y8, dG[p]), bp = clamp255_add(y8, dB[p]);
                sum2 += y8;                                                                   // halves stay < 2^16 within a tile
                bgra[2 * p]     = __byte_perm(__byte_perm(bp, gp, 0x0040), rp, 0x5410);
                bgra[2 * p + 1] = __byte_perm(__byte_perm(bp, gp, 0x0062), rp, 0x7610);
            }
            if (r2 == 0) {
                #pragma unroll
                for (int j = 0; j < NC; j++) if ((gw[j] >> gs[j]) & 1) unsafe |= ((1u << (1 << EHS)) - 1) << (j << EHS);
                if (!T.rb_ok) unsafe = 0xFF;
            }
            if (unsafe) {              // rare (a handful of (cb,cr) pairs): the exact float routine, out of line
                #pragma unroll
                for (int k = 0; k < 8; k++) if (unsafe >> k & 1) {
                    const int yraw = (k & 1) ? ((int)yw[k >> 1] >> 16) : (int)(short)(yw[k >> 1] & 0xFFFF);
                    const int cbr = (k & 1) ? ((int)cbw[k >> 1] >> 16) : (int)(short)(cbw[k >> 1] & 0xFFFF);
                    const int crr = (k & 1) ? ((int)crw[k >> 1] >> 16) : (int)(short)(crw[k >> 1] & 0xFFFF);
                    bgra[k] = ycc_exact(yraw, cbr, crr);
                }
            }
            // brightest pixel: first strict maximum of raw Y in raster order
            const uint32_t m2 = __vmaxs2(__vmaxs2(yw[0], yw[1]), __vmaxs2(yw[2], yw[3]));
            const int m = max((int)(short)(m2 & 0xFFFF), (int)m2 >> 16);
            if (m >= bestm) {           // rare once the running maximum is high
                int kf = 7;
                #pragma unroll
                for (int k = 7; k >= 0; k--) { const int yraw = (k & 1) ? ((int)yw[k >> 1] >> 16) : (int)(short)(yw[k >> 1] & 0xFFFF); if (yraw == m) kf = k; }
                const unsigned long long key = ((unsigned long long)(uint32_t)(m + 32768) << 32) | (0xffffffffu - (uint32_t)(mi + kf));
                if (key > best) { best = key; bestm = m; }      // equal value: the earlier raster position wins
            }
            uint4* dp = reinterpret_cast<uint4*>(a.dib + ((size_t)(a.hp - 1 - ay) * a.wp + ax) * 4);
            dp[0] = make_uint4(bgra[0], bgra[1], bgra[2], bgra[3]);
            dp[1] = make_uint4(bgra[4], bgra[5], bgra[6], bgra[7]);
        }
    }
}

