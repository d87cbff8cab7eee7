// jsgpu_phuff_core.cuh — per-thread logic of the self-synchronising Huffman passes for LONG restart intervals
// (scans without restart markers — BASELINE config 5 — or with a DRI of a whole MCU row and more), where "one
// lane per restart interval" has nothing to run in parallel.  The reference decodes such an interval as one serial
// walk (ImgDecode.cpp:3164-3630; a restart only at :1644-1680); the symbol boundaries inside it are found here by
// decoding from many places at once and letting the decoders fall into step:
//
//   slots      the unstuffed copy of an interval is cut into 4096-bit sub-sequences ("slots").
//   guess      slot i is decoded from its first bit as if an MCU (DC of block 0) started there, to the first symbol
//              start at/after its end: exit state X_i = (bit position, block in MCU, zig-zag index).  A Huffman
//              decoder started on a wrong grid locks onto the true one after a few hundred bits, so most X_i are
//              already the true states.
//   fix        round r: slot i is decoded again from X_{i-1} (slot 0 from the true start) iff X_{i-1} changed in
//              round r-1; it counts the MCU starts inside it, remembers where the first one is, sums the DC
//              differences per component before/after it, and replaces X_i if it came out different.  A round that
//              changes nothing ends the iteration (then every X_i is the true state, by induction from slot 0).
//   scan       exclusive prefix sums over the slots of an interval: MCU index and DC predictors at the first MCU
//              start of every slot -> each slot is a VIRTUAL restart interval for the lane kernel (k_huff_lane<VSEG>),
//              which then decodes every symbol exactly once, writes the coefficient rows and counts the code lengths.
//
// Everything in this header but the shared-memory staging (device only) is plain C++ shared by the device kernels
// (jsgpu_phuff.cu, jsgpu_huff.cu) and by the host model the CPU test-suite runs (tests/native/phuff_model.cpp): JS_HD is
// __host__ __device__ under nvcc.
#pragma once
#include "jsgpu_internal.h"

#if defined(__CUDACC__)
#define JS_HD __host__ __device__ __forceinline__
#else
#define JS_HD inline
#endif

#define PH_SUB_BITS    4096u
#define PH_SUB_SHIFT   12
#define PH_DEAD        0xffffffffffffffffull     // state of a slot that belongs to no interval
#define PH_NONE        0xffffffffu
#define PH_MAX_BPM     48                        // 3 components x 4 x 4 blocks
#ifndef PH_GUESS_BITS
#define PH_GUESS_BITS  2048u                     // the guess decodes only the last PH_GUESS_BITS of its slot: enough to lock on for ~9 slots in 10
#endif
#define PH_MAX_ROUNDS  10                        // fix rounds enqueued up front (each ends at once when the previous changed nothing)

// Shared-memory staged decode tables of one image, as the lane kernel lays them out: table j at lutb + j * JS_LANE_TAB
// (first level JS_LUT_SIZE entries, then its second level).
struct PhTabs {
    const uint16_t* lutb;
    const uint32_t* qz;            // [3][80]: quantiser | natural index << 16 of zig-zag position k, per component
    const uint16_t* blk_dc;        // [bpm] offset (uint16 units into lutb) of the DC table of block i of an MCU
    const uint16_t* blk_ac;        // [bpm] ... of its AC table
    const uint8_t*  blk_c;         // [bpm] its component
    uint32_t bpm, pshift;          // blocks per MCU; precision - 8 (ReadScanVal's divide, ImgDecode.cpp:1234-1238)
};

// What the lane kernel and the self-synchronising passes stage in shared memory besides the tables themselves (lane_stage).
struct LaneTabs {
    uint32_t qz[3][80];            // quantiser | natural index<<16 ; entries 64..79 -> dummy slots past the row
    uint32_t li[6];                // [comp*2 + class] -> staged table index
    uint32_t lslot[6];             // staged table index -> slot
    uint32_t nl, pad;
};

#if defined(__CUDACC__)
// One component's quantiser row for the decode loops: the table's entries at zig-zag positions 0..63, then no-ops (quantiser 0,
// a dummy slot past the row) where a run carries the position beyond 63.  All threads of the CTA.
__device__ __forceinline__ void stage_qz(uint32_t* row, const uint32_t* q)
{
    for (uint32_t i = threadIdx.x; i < 80; i += blockDim.x) row[i] = (i < 64) ? q[i] : ((64u + (i & 7)) << 16);
}

// Stage the decode tables of image im: its distinct (class, Th) tables, table j at lutb + j * JS_LANE_TAB, and its quantiser
// rows.  All threads of the CTA; one barrier inside (the table list thread 0 makes), the caller synchronises before and after.
__device__ __forceinline__ void lane_stage(LaneTabs& t, uint16_t* lutb, const DevImage& im, const DevTableSet* ts)
{
    if (threadIdx.x == 0) {
        uint32_t n = 0;
        for (uint32_t c = 0; c < im.ns; c++) for (uint32_t cls = 0; cls < 2; cls++) {
            const uint32_t slot = cls ? im.slot_ac[c] : im.slot_dc[c];
            uint32_t j = 0;
            while (j < n && t.lslot[j] != slot) j++;
            if (j == n) t.lslot[n++] = slot;
            t.li[c * 2 + cls] = j;
        }
        t.nl = n;
    }
    __syncthreads();
    const uint32_t nl = t.nl;
    for (uint32_t j = 0; j < nl; j++) {
        const uint32_t slot = t.lslot[j];
        const uint4* s0 = reinterpret_cast<const uint4*>(ts->lut[slot]);
        uint4* d0 = reinterpret_cast<uint4*>(lutb + j * JS_LANE_TAB);
        for (uint32_t i = threadIdx.x; i < JS_LUT_SIZE * 2 / 16; i += blockDim.x) d0[i] = __ldg(s0 + i);
        const uint4* s1 = reinterpret_cast<const uint4*>(ts->lut2[slot]);
        uint4* d1 = reinterpret_cast<uint4*>(lutb + j * JS_LANE_TAB + JS_LUT_SIZE);
        const uint32_t used = min(ts->lut2_used[slot], (uint32_t)JS_LANE_L2S);     // <= JS_LANE_L2S: the launchers refuse the batch otherwise
        for (uint32_t i = threadIdx.x; i < used * 2 / 16; i += blockDim.x) d1[i] = __ldg(s1 + i);
    }
    for (uint32_t c = 0; c < im.ns; c++) stage_qz(t.qz[c], ts->qz[im.dqt[c]]);
}
#endif

JS_HD unsigned long long ph_pack(uint32_t pos, uint32_t blk, uint32_t zz) { return (unsigned long long)pos | ((unsigned long long)blk << 32) | ((unsigned long long)zz << 40); }
JS_HD uint32_t ph_pos(unsigned long long x) { return (uint32_t)x; }
JS_HD uint32_t ph_blk(unsigned long long x) { return (uint32_t)(x >> 32) & 0xFFu; }
JS_HD uint32_t ph_zz(unsigned long long x)  { return (uint32_t)(x >> 40) & 0xFFu; }

// First slot of interval k (raw start s0 inside the image's scan): derived from where k_unstuff puts its unstuffed
// copy, (s0 & ~15) + JS_USLACK*k, so consecutive intervals never share a slot (copy k+1 starts >= 35 bytes after the
// end of copy k, see DESIGN.md §3) and no prefix sum over interval lengths is needed to find it.
JS_HD uint32_t ph_slot_base(uint32_t s0, uint32_t k)
{
    return (uint32_t)((((unsigned long long)(s0 & ~15u) + (unsigned long long)JS_USLACK * k) >> 9) + k);
}
JS_HD uint32_t ph_nsub(uint32_t ulen_bytes) { return (ulen_bytes + 511u) >> 9; }

// Interval of an image that owns `slot`, or PH_NONE (a gap between intervals).
JS_HD uint32_t ph_find_interval(const uint32_t* seg_start, const uint32_t* seg_ulen, uint32_t nseg, uint32_t slot)
{
    if (nseg == 0) return PH_NONE;
    uint32_t lo = 0, hi = nseg - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (ph_slot_base(seg_start[mid], mid) <= slot) lo = mid; else hi = mid - 1;
    }
    const uint32_t base = ph_slot_base(seg_start[lo], lo);
    if (slot < base) return PH_NONE;
    return (slot - base < ph_nsub(seg_ulen[lo])) ? lo : PH_NONE;
}

// ---- bit window over an unstuffed interval (big-endian 32-bit words, see k_unstuff) --------------------------------
JS_HD uint32_t ph_ldw(const uint32_t* p)
{
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
JS_HD uint32_t ph_fsl(uint32_t lo, uint32_t hi, uint32_t n)      // high word of (hi:lo) << (n & 31)
{
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(lo, hi, n);
#else
    n &= 31; return n ? ((hi << n) | (lo >> (32 - n))) : hi;
#endif
}
// Position-based window: the four words from the one holding bit `pos` onwards.  A peek is ONE funnel shift (its shift count
// is taken modulo 32, i.e. pos & 31 for free); moving on costs nothing until the position crosses a word boundary (at most once
// per symbol: code + value <= 31 bits), then the words shift down and the one three words ahead is requested — ~10 symbols
// before it is looked at, so the L2 latency of these scattered 4-byte loads stays off the dependency chain.
struct PhWin {
    uint32_t w0, w1, w2, w3; const uint32_t* nextp;          // nextp: address of the word after w3
    JS_HD void init(const uint32_t* words, uint32_t bitpos) {
        const uint32_t* p = words + (bitpos >> 5);
        w0 = ph_ldw(p); w1 = ph_ldw(p + 1); w2 = ph_ldw(p + 2); w3 = ph_ldw(p + 3); nextp = p + 4;
    }
    JS_HD uint32_t peek(uint32_t pos) const { return ph_fsl(w1, w0, pos); }                     // 32 bits from `pos` (inside w0)
    // 32 bits from p2, pos <= p2 <= pos + 31 (value bits behind a code)
    JS_HD uint32_t peek_at(uint32_t pos, uint32_t p2) const { return ((p2 ^ pos) & ~31u) ? ph_fsl(w2, w1, p2) : ph_fsl(w1, w0, p2); }
    JS_HD void advance(uint32_t pos, uint32_t npos) {       // npos - pos <= 32
#if defined(__CUDA_ARCH__)
        // predicated in-place reload: written as a C++ conditional the compiler loads into a temporary and copies it at the
        // end of the same step, i.e. waits for the very load that is to be hidden (cf. Win in jsgpu_huff.cu)
        const uint32_t cross = ((npos ^ pos) >> 5) ? 1u : 0u;
        if (cross) { w0 = w1; w1 = w2; w2 = w3; }
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %2, 0;\n\t@p ld.global.nc.u32 %0, [%1];\n\t}" : "+r"(w3) : "l"(nextp), "r"(cross));
        nextp += cross;
#else
        if ((npos ^ pos) >> 5) { w0 = w1; w1 = w2; w2 = w3; w3 = ph_ldw(nextp); nextp++; }
#endif
    }
};

// What a fix run learns about its slot.
struct PhCount {
    uint32_t nmcu;                 // MCU starts (symbol start with block 0, zig-zag 0) at bit positions in [entry, exit)
    uint32_t fpos;                 // bit position of the first one (PH_NONE: none)
    int tot0, tot1, tot2;          // sum of the dequantised DC differences read in the slot, per component
    int bef0, bef1, bef2;          // ... of those read before the first MCU start
};

// Decode from (pos, blk, zz) to the first symbol start at or after `lim`; returns the exit state.  The symbol semantics
// are the lane kernel's (DC: position 1 + high nibble; AC: EOB = symbol byte 0, otherwise position += run + 1; a block is
// closed when the position reaches 64).  Where no code matches — a decoder on a wrong grid, the pad bits behind the last
// MCU, or damaged data — one bit is skipped and decoding goes on in the same state (what ReadScanVal itself does,
// ImgDecode.cpp:1178-1187), so a wrong entry state cannot poison the slots behind it: the decoder falls back into step.
template <bool COUNT>
JS_HD unsigned long long ph_run(const PhTabs& t, const uint32_t* words, uint32_t pos, uint32_t blk, uint32_t zz, uint32_t lim, PhCount& o)
{
    o.nmcu = 0; o.fpos = PH_NONE; o.tot0 = o.tot1 = o.tot2 = 0; o.bef0 = o.bef1 = o.bef2 = 0;
    if (pos >= lim) return ph_pack(pos, blk, zz);
    PhWin s; s.init(words, pos);
    uint32_t dcoff = t.blk_dc[blk], acoff = t.blk_ac[blk], c = t.blk_c[blk];
    // ONE symbol per iteration, whatever it is: on the device the 32 lanes of a warp walk 32 different slots, and a loop
    // nest (block / DC / AC) would leave most of them waiting at every level (measured: 16 of 32 lanes active); with a flat
    // loop and selects instead of branches they stay together until their slots end.
    while (pos < lim) {
        const uint32_t top = s.peek(pos);
        const bool isdc = (zz == 0);
        const uint32_t off = isdc ? dcoff : acoff;
        uint32_t e = t.lutb[off + (top >> (32 - JS_LUT_BITS))];
        if (e & 0x8000) e = t.lutb[off + JS_LUT_SIZE + (e & 0x7FFF) + ((top >> 16) & ((1u << JS_LUT2_BITS) - 1))];
        if (e == 0) { s.advance(pos, pos + 1); pos += 1; continue; }           // rare (see above)
        const uint32_t len = e >> 8, size = e & 15, run = (e >> 4) & 15;
        if (COUNT && isdc) {                                         // one symbol in ~20: worth a branch, the lanes rejoin at once
            if (blk == 0) {                                          // an MCU starts here
                if (o.nmcu == 0) { o.fpos = pos; o.bef0 = o.tot0; o.bef1 = o.tot1; o.bef2 = o.tot2; }
                o.nmcu++;
            }
            const uint32_t q = t.qz[c * 80 + run];
            if ((q >> 16) == 0) {        // a DC symbol whose coefficient lands in natural position 0 is a DC difference
                const uint32_t tv = s.peek_at(pos, pos + len);     // value bits follow the code
                const uint32_t v = size ? (tv >> (32 - size)) : 0u;
                int val = (int)v - ((((int)~tv) >> 31) & (int)((1u << size) - 1u));      // T.81 F.12 EXTEND (HuffmanDc2Signed, :859-866)
                if (t.pshift) val /= (1 << t.pshift);
                const int d = (int)(short)(val * (int)(q & 0xFFFF));                      // dequantised, short like the reference's
                o.tot0 += (c == 0) ? d : 0; o.tot1 += (c == 1) ? d : 0; o.tot2 += (c == 2) ? d : 0;
            }
        }
        const uint32_t npos = pos + len + size;
        s.advance(pos, npos); pos = npos;
        zz = isdc ? 1 + run : (((e & 0xFF) == 0) ? 64u : zz + run + 1);
        if (zz >= 64) {                                              // block closed
            zz = 0; blk = (blk + 1 == t.bpm) ? 0u : blk + 1;
            dcoff = t.blk_dc[blk]; acoff = t.blk_ac[blk]; c = t.blk_c[blk];
        }
    }
    return ph_pack(pos, blk, zz);
}

// Slot-indexed work arrays of ONE image (pointers already offset by DevImage::ph_first); every array has
// ph_nslots + 1 entries (the prefix sums need the one-past-the-end element).
struct PhSlots {
    unsigned long long* x;         // exit state of the slot
    uint32_t* ver;                 // fix round in which x last changed (0 = the guess)
    uint32_t* k;                   // interval (index inside the image) the slot belongs to, PH_NONE = unused
    uint4*    cnt;                 // (nmcu, tot0, tot1, tot2) of the slot's latest fix run
    uint4*    aux;                 // (fpos, bef0, bef1, bef2)
    uint4*    pre;                 // exclusive prefix sums of cnt over the image's slots (k_ph_scan)
};
// The restart intervals of ONE image (pointers already offset by DevImage::seg_first).
struct PhSegs {
    const uint32_t* start; const uint32_t* ulen; const unsigned long long* uoff; uint32_t nseg;
};

JS_HD void ph_guess_slot(const PhTabs& t, const PhSegs& sg, const uint8_t* ubits, const PhSlots& a, uint32_t slot)
{
    const uint32_t k = ph_find_interval(sg.start, sg.ulen, sg.nseg, slot);
    a.k[slot] = k; a.ver[slot] = 0;
    a.cnt[slot] = make_uint4(0, 0, 0, 0); a.aux[slot] = make_uint4(PH_NONE, 0, 0, 0);
    if (k == PH_NONE) { a.x[slot] = PH_DEAD; return; }
    const uint32_t i = slot - ph_slot_base(sg.start[k], k), end = sg.ulen[k] * 8u;
    const uint32_t s0 = i << PH_SUB_SHIFT, lim = (s0 + PH_SUB_BITS < end) ? s0 + PH_SUB_BITS : end;
    // slot 0 starts at the true start of the interval; the others only need their exit state, which a decoder started
    // PH_GUESS_BITS before the slot's end reaches as well as one started at its beginning (the fix rounds repair the rest)
    const uint32_t pos0 = (i == 0 || lim - s0 <= PH_GUESS_BITS) ? s0 : lim - PH_GUESS_BITS;
    PhCount o;
    a.x[slot] = ph_run<false>(t, reinterpret_cast<const uint32_t*>(ubits + sg.uoff[k]), pos0, 0, 0, lim, o);
}

// One fix round for one slot; returns true when its exit state changed.
JS_HD bool ph_fix_slot(const PhTabs& t, const PhSegs& sg, const uint8_t* ubits, const PhSlots& a, uint32_t slot, uint32_t round)
{
    const uint32_t k = a.k[slot];
    if (k == PH_NONE) return false;
    const uint32_t i = slot - ph_slot_base(sg.start[k], k), end = sg.ulen[k] * 8u;
    unsigned long long entry;
    if (i == 0) { if (round != 1) return false; entry = ph_pack(0, 0, 0); }
    else { if (a.ver[slot - 1] != round - 1) return false; entry = a.x[slot - 1]; }
    unsigned long long nx = PH_DEAD;
    PhCount o; o.nmcu = 0; o.fpos = PH_NONE; o.tot0 = o.tot1 = o.tot2 = 0; o.bef0 = o.bef1 = o.bef2 = 0;
    if (entry != PH_DEAD) {
        const uint32_t lim = (((i + 1) << PH_SUB_SHIFT) < end) ? ((i + 1) << PH_SUB_SHIFT) : end;
        nx = ph_run<true>(t, reinterpret_cast<const uint32_t*>(ubits + sg.uoff[k]), ph_pos(entry), ph_blk(entry), ph_zz(entry), lim, o);
    }
    a.cnt[slot] = make_uint4(o.nmcu, (uint32_t)o.tot0, (uint32_t)o.tot1, (uint32_t)o.tot2);
    a.aux[slot] = make_uint4(o.fpos, (uint32_t)o.bef0, (uint32_t)o.bef1, (uint32_t)o.bef2);
    if (nx != a.x[slot]) { a.x[slot] = nx; a.ver[slot] = round; return true; }
    return false;
}

// The virtual restart interval a slot stands for, once the fix rounds have settled and k_ph_scan has run.
struct PhVseg {
    uint32_t k;                    // real interval (index inside the image)
    uint32_t bit;                  // absolute bit position (inside the real interval) of its first MCU
    uint32_t m0, nm;               // first MCU (index inside the image) and number of MCUs
    int dc0, dc1, dc2;             // DC predictors at its start (ImgDecode.cpp:3280,3355,3386: running short sums)
    bool final;                    // it ends the real interval: reports the end bit position / leftover / overrun
};
// ri = MCUs per restart interval, nmcu = MCUs of the image.  Returns false for unused slots and slots without work.
JS_HD bool ph_vseg(const PhSegs& sg, uint32_t ri, uint32_t nmcu, const PhSlots& a, uint32_t slot, PhVseg& v)
{
    const uint32_t k = a.k[slot];
    if (k == PH_NONE) return false;
    const uint32_t base = ph_slot_base(sg.start[k], k), nsub = ph_nsub(sg.ulen[k]);
    const uint4 P = a.pre[slot], PB = a.pre[base], PE = a.pre[base + nsub], C = a.cnt[slot], A = a.aux[slot];
    const uint32_t cntk = (nmcu - k * ri < ri) ? nmcu - k * ri : ri;          // MCUs the interval must hold
    const uint32_t M = P.x - PB.x, T = PE.x - PB.x, hiN = M + C.x;
    const uint32_t tgt = (T < cntk) ? T : cntk;
    v.final = (M < tgt) && (hiN >= tgt);
    uint32_t mlo = (M < cntk) ? M : cntk, mhi = (hiN < cntk) ? hiN : cntk;
    if (v.final && T < cntk) mhi = cntk;       // data for fewer MCUs than expected: the last decoder runs on and reports the error
    v.k = k; v.bit = A.x; v.m0 = k * ri + mlo; v.nm = mhi - mlo;
    v.dc0 = (int)(short)((P.y - PB.y) + A.y); v.dc1 = (int)(short)((P.z - PB.z) + A.z); v.dc2 = (int)(short)((P.w - PB.w) + A.w);
    return v.nm > 0 && C.x > 0;
}
