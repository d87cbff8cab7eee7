// jsgpu_detail.cuh — what the serial reference-semantics walk (jsgpu_exact.cu) and the parallel "Detailed Decode" kernels
// (jsgpu_detail.cu) share: the file position of an unstuffed byte (also the MCU file map's, jsgpu_kernels.cu), the code search
// and value decode of ReadScanVal, the dequantising store of DecodeIdctSet, the encoding of DecodeScanCompPrint's report
// lines as jsgpu_detail_events, and the scan-error report's events and cap rule.
#pragma once
#include "jsgpu_internal.h"

// Where the raw-byte walk of js_raw_of_unstuffed stopped: raw offset r of unstuffed byte `kept` of interval k.  A caller that asks
// for increasing positions of one interval passes it along, so that the walk resumes instead of starting over.
struct JsRawCursor { uint32_t k, r, kept; };

// Raw offset (inside interval k of image im) of unstuffed byte u: u plus the stuffed zeros before it — from the short list
// k_unstuff keeps per interval, from the row table of k_unstuff_long (long intervals), or, for a short interval with more
// stuffed bytes than the list holds, by walking its raw bytes (from `cur` on when it lies before u).  A stuffed FF 00 pair maps
// to its FF.
__device__ __forceinline__ uint32_t js_raw_of_unstuffed(const DevBatch& b, const DevImage& im, uint32_t k, uint32_t u, JsRawCursor* cur = nullptr)
{
    const uint32_t sidx = im.seg_first + k, ns = b.seg_nstuff[sidx];
    const uint32_t s0 = b.seg_start[sidx], len = b.seg_end[sidx] - s0;
    if (im.psync) {
        const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(b.bits + im.scan_off + s0) & 3);
        const size_t rt0 = (size_t)(im.rt_off + (s0 >> 7) + 2u * k);
        const uint32_t nrows = (len + mis + 127) >> 7;
        uint32_t lo = u >> 7, hi = min(nrows - 1, (u + ns + mis) >> 7);      // rowtab[r] <= 128 r: the row holding u is not before u / 128
        while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (b.rowtab[rt0 + mid] <= u) lo = mid; else hi = mid - 1; }
        uint32_t need = u - b.rowtab[rt0 + lo];                     // kept bytes of the row before the one we want
        const uint4 mk = b.rowmask[rt0 + lo];
        uint32_t w = ~mk.x, off = 0, c = __popc(w);                  // set bit = this raw byte of the row is kept
        if (need >= c) { need -= c; w = ~mk.y; off = 32; c = __popc(w);
            if (need >= c) { need -= c; w = ~mk.z; off = 64; c = __popc(w);
                if (need >= c) { need -= c; w = ~mk.w; off = 96; } } }
        return (lo << 7) - mis + off + __fns(w, 0, (int)need + 1);
    }
    if (ns <= JS_STUFF_LIST) {
        uint32_t raw = u;
        for (uint32_t j = 0; j < ns; j++) raw += (b.seg_stuff[(size_t)sidx * JS_STUFF_LIST + j] < u) ? 1u : 0u;
        return raw;
    }
    const uint8_t* seg = b.bits + im.scan_off + s0;
    uint32_t r = 0, kept = 0;
    if (cur && cur->k == k && cur->kept <= u) { r = cur->r; kept = cur->kept; }
    for (; r < len; r++) {
        if (seg[r] == 0 && r > 0 && seg[r - 1] == 0xFF) continue;
        if (kept == u) break;
        kept++;
    }
    if (cur) { cur->k = k; cur->r = r; cur->kept = kept; }
    return r;
}

// The code search of ReadScanVal (ImgDecode.cpp:1118-1164) on the accumulator `buff` holding `avail` bits: direct look-up
// when at least DHT_FAST_SIZE bits are there, else the in-order search, in both cases only codes no longer than the bits
// actually in the accumulator.  For a prefix-free table both give "the one code that matches", which the two-level table of
// the fast path delivers too.  Returns (length << 8) | symbol, 0 = no code.
__device__ __forceinline__ uint32_t js_find_code(const DevTableSet* ts, uint32_t slot, uint32_t buff, uint32_t avail)
{
    uint32_t e = ts->lut[slot][buff >> (32 - JS_LUT_BITS)];
    if (e & 0x8000) {
        if (ts->lut2_overflow[slot]) {
            e = 0;
            const uint32_t n = ts->ent_n[slot];
            for (uint32_t i = 0; i < n; i++) {
                const uint32_t l = ts->ent_len[slot][i];
                if (l == 0 || l > 16) continue;
                if ((buff & (0xffffffffu << (32 - l))) == ts->ent_bits[slot][i] && l <= avail) { e = (l << 8) | ts->ent_sym[slot][i]; break; }
            }
            return e;
        }
        e = ts->lut2[slot][(e & 0x7FFF) + ((buff >> 16) & ((1u << JS_LUT2_BITS) - 1))];
    }
    if (e && (e >> 8) > avail) e = 0;
    return e;
}

// The value of `bits2` value bits v: HuffmanDc2Signed (ImgDecode.cpp:859-866), then the precision divide of :1234-1238
__device__ __forceinline__ int js_huff_value(uint32_t v, uint32_t bits2, uint32_t precision)
{
    int val = (v >= (1u << (bits2 - 1))) ? (int)v : (int)(v - ((1u << bits2) - 1));
    if (precision >= 8) val /= (1 << (precision - 8));
    return val;
}

// DecodeIdctSet, ImgDecode.cpp:2270-2303: coefficient ncoef + zrl (zig-zag), dequantised, stored in natural order
__device__ __forceinline__ void js_idct_set(short* dct, const DevTableSet* ts, uint32_t dqt, uint32_t ncoef, uint32_t zrl, short val)
{
    const uint32_t ind = ncoef + zrl;
    if (ind >= 64) return;
    const uint32_t q = ts->qz[dqt][ind];                        // quantiser | natural index << 16
    dct[q >> 16] = (short)(val * (int)(q & 0xFFFF));
}

// One line of DecodeScanCompPrint / DecodeScanImg as a jsgpu_detail_event (include/jsgpu.h, JSGPU_DT_*).
__device__ __forceinline__ void js_detail_put(jsgpu_detail_event& ev, uint32_t kind, uint32_t seq, uint32_t a = 0, uint32_t b = 0,
                                              uint32_t c = 0, uint32_t d = 0, uint32_t e = 0, uint32_t f = 0)
{
    ev.kind = kind; ev.seq = seq; ev.a = a; ev.b = b; ev.c = c; ev.d = d; ev.e = e; ev.f = f;
}
// ReportVlc (ImgDecode.cpp:2152-2232) of one symbol: where its first bit is, what it decoded to, which coefficients it covers,
// how many bits code and value took, and the EOB / ERROR / EOB64 note (special: 0 "", 1 EOB, 2 ERROR, 3 EOB64)
__device__ __forceinline__ void js_detail_vlc(jsgpu_detail_event& ev, uint32_t seq, uint32_t pos, uint32_t align, uint32_t zrl, short val,
                                              uint32_t coef_start, uint32_t coef_end, uint32_t bits, uint32_t special)
{
    js_detail_put(ev, JSGPU_DT_VLC, seq, pos, align, zrl, (uint32_t)(int)val, coef_start | (coef_end << 8) | (bits << 16), special);
}

// The scan-error report (jsgpu_scan_errors): counts back to a scan's start (warn_num and the end position are set by the caller).
__device__ __forceinline__ void js_ex_reset(JsExResult* res)
{
    res->nerr_lines = 0; res->nevents = 0; res->scan_bad = 0; res->restart_read = 0; res->done = 0;
}
// One error event making `lines` error lines; ev[] (cap entries) keeps the first ones, the counts go on.
__device__ __forceinline__ void js_ex_event(JsExResult* res, JsExEvent* ev, uint32_t cap, uint32_t code, uint32_t lines,
                                            uint32_t a = 0, uint32_t b = 0, uint32_t c = 0, uint32_t d = 0, uint32_t e = 0)
{
    res->nerr_lines += lines;
    if (res->nevents < cap) ev[res->nevents] = JsExEvent{code, a, b, c, d, e, 0, 0};
    res->nevents++;
}
// The "first nErrMaxDecodeScan instances" rule (ImgDecode.cpp:1100-1110 and its copies): the event only while fewer than
// err_max have been counted in `warn` (m_nWarnBadScanNum), and the cap line after the one that reaches err_max.
__device__ __forceinline__ void js_ex_warn(JsExResult* res, JsExEvent* ev, uint32_t cap, uint32_t err_max, uint32_t& warn, uint32_t code,
                                           uint32_t lines, uint32_t a = 0, uint32_t b = 0, uint32_t c = 0, uint32_t d = 0, uint32_t e = 0)
{
    if (warn >= err_max) return;
    js_ex_event(res, ev, cap, code, lines, a, b, c, d, e);
    if (++warn >= err_max) js_ex_event(res, ev, cap, JS_EX_CAP, 1, err_max);
}
