// jsgpu_exact.cu — the reference's behaviour on DAMAGED scans (SURVEY.md §8f N2), bit for bit.
//
// The fast kernels decode restart intervals independently and stop an interval at the first thing that cannot be a
// well-formed stream (no matching code, data running out, data left over, a missing or unexpected marker); they flag the
// image.  What JPEGsnoop does then is the point of the tool: ReadScanVal consumes ONE bit and tries again
// (ImgDecode.cpp:1166-1187), a stray marker's FF is kept as data and the block flagged (BuffAddByte :1527-1561,
// DecodeScanComp :1683-1706), restart markers are honoured where they are FOUND, not where they are expected
// (:1644-1680, :3180-3200), a block that underflows contributes only its DC (:1737-1760 returns before the IDCT),
// after an overread every remaining MCU row still decodes one MCU (:3173-3174, 3621-3625), and every such event is
// a log line, capped by nErrMaxDecodeScan (:1100-1110 ...).  None of that is interval-local, so an image whose status
// word is non-zero is decoded AGAIN here, by ONE thread, as the same serial walk over the raw bytes with the same
// 32-bit accumulator and per-byte file positions (ImgDecode.h:618-636).  It writes the same intermediate the fast
// path writes (coefficient rows, slot 0 = running DC; block-DC maps; MCU file map; code-length histogram) so the
// IDCT / colour kernels run unchanged, plus a list of error events the host class turns into the reference's lines.
// Slow by construction (one serial chain per damaged image); exactness is what matters here.
#include "jsgpu_internal.h"
#include "jsgpu_detail.cuh"

#define EX_SCANBUF_OK      0u
#define EX_SCANBUF_BADMARK 1u
enum { EX_RSV_OK, EX_RSV_EOB, EX_RSV_UNDERFLOW, EX_RSV_RST_TERM };              // ImgDecode.h:166-171

struct Ex {
    const uint8_t* data; uint32_t n, file_pos;
    uint32_t buff, vacant, ptr;                  // ptr: offset inside the scan (file position = file_pos + ptr)
    uint32_t pos[4], err[4], latch_err, num, align;
    bool scan_end, scan_bad, cur_err, restart_flag;
    uint32_t restart_read, restart_last, restart_expect, mcus_left, rst_interval, warn_bad_num, err_max;
    uint32_t precision; bool decode_ac;
    short css[3][16];                            // m_anDcLumCss / m_anDcChrCbCss / m_anDcChrCrCss: DC sum of block (v,h) of the current MCU
    JsExResult* res;
    uint32_t* histo;                             // [2][4][17] of this image
    const DevTableSet* ts;
    short dct[64];
    uint32_t bits_used;                          // m_nScanBitsUsed1 + m_nScanBitsUsed2 of the last ReadScanVal
    JsDetailOut dt;                              // "Detailed Decode" of the chosen MCUs (DecodeScanCompPrint)
};

// one line of the detailed decode; seq = error events issued so far, so the host can interleave both lists as the reference's log does
__device__ __forceinline__ jsgpu_detail_event* ex_detail_slot(Ex& x)
{
    const uint32_t n = x.dt.hdr[0]++;
    return (n < x.dt.ev_cap) ? x.dt.ev + n : nullptr;
}
__device__ __forceinline__ void ex_detail(Ex& x, uint32_t kind, uint32_t a = 0, uint32_t b = 0, uint32_t c = 0)
{
    if (jsgpu_detail_event* ev = ex_detail_slot(x)) js_detail_put(*ev, kind, x.res->nevents, a, b, c);
}

__device__ __forceinline__ void ex_event(Ex& x, uint32_t code, uint32_t lines, uint32_t a = 0, uint32_t b = 0, uint32_t c = 0, uint32_t d = 0, uint32_t e = 0)
{
    JsExResult* r = x.res;
    r->nerr_lines += lines;
    if (r->nevents < JS_EX_MAX_EVENTS) { JsExEvent& ev = r->ev[r->nevents]; ev.code = code; ev.a = a; ev.b = b; ev.c = c; ev.d = d; ev.e = e; ev.pad0 = ev.pad1 = 0; }
    r->nevents++;
}
// the "first nErrMaxDecodeScan instances" pattern (ImgDecode.cpp:1100-1110 and its copies)
__device__ __forceinline__ void ex_warn(Ex& x, uint32_t code, uint32_t lines, uint32_t a = 0, uint32_t b = 0, uint32_t c = 0, uint32_t d = 0, uint32_t e = 0)
{
    if (x.warn_bad_num < x.err_max) {
        ex_event(x, code, lines, a, b, c, d, e);
        x.warn_bad_num++;
        if (x.warn_bad_num >= x.err_max) ex_event(x, JS_EX_CAP, 1, x.err_max);
    }
}
__device__ __forceinline__ uint32_t ex_fbuf(const Ex& x, uint32_t off) { return (off < x.n) ? (uint32_t)__ldg(x.data + off) : 0u; }   // WindowBuf.cpp:639-713: bytes past EOF read as 0

// ImgDecode.cpp:974-988 / 1000-1004
__device__ __forceinline__ void ex_scanbuf_add(Ex& x, uint32_t byte, uint32_t filepos, uint32_t err)
{
    x.buff += byte << (x.vacant - 8); x.vacant -= 8;
    if (x.num >= 4) return;
    x.err[x.num] = err; x.pos[x.num++] = filepos;
}
// ImgDecode.cpp:921-955
__device__ __forceinline__ void ex_scanbuf_consume(Ex& x, uint32_t nbits)
{
    x.buff = (nbits >= 32) ? 0u : (x.buff << nbits);
    x.vacant += nbits;
    const uint32_t nbytes = (x.align + nbits) / 8;
    for (uint32_t i = 0; i < nbytes; i++) {
        x.pos[0] = x.pos[1]; x.pos[1] = x.pos[2]; x.pos[2] = x.pos[3];
        x.err[0] = x.err[1]; x.err[1] = x.err[2]; x.err[2] = x.err[3]; x.err[3] = EX_SCANBUF_OK;
        if (x.err[0] != EX_SCANBUF_OK) x.latch_err = x.err[0];
        x.num--;
    }
    x.align = (x.align + nbits) % 8;
}
// ImgDecode.cpp:1386-1573
__device__ __noinline__ void ex_buff_add_byte(Ex& x)
{
    if (x.restart_flag) return;
    const uint32_t b0 = ex_fbuf(x, x.ptr), b1 = ex_fbuf(x, x.ptr + 1);
    uint32_t marker = 0;
    if (b0 == 0xFF) {
        marker = b1;
        if (marker >= 0xD0 && marker <= 0xD7) {
            x.restart_read++; x.restart_last = marker - 0xD0;
            if (x.restart_last != x.restart_expect) ex_event(x, JS_EX_RST_MISMATCH, 1, x.restart_expect, x.restart_last, x.file_pos + x.ptr);
            x.restart_expect = (x.restart_last + 1) % 8;
            x.restart_flag = true;
            return;
        }
    }
    if (b0 == 0xFF && b1 == 0x00)      { ex_scanbuf_add(x, b0, x.file_pos + x.ptr, EX_SCANBUF_OK); x.ptr += 2; }
    else if (b0 == 0xFF && b1 == 0xFF) { ex_scanbuf_add(x, b0, x.file_pos + x.ptr, EX_SCANBUF_OK); x.ptr += 1; }
    else if (b0 == 0xFF && marker != 0) {
        if (x.warn_bad_num < x.err_max) {
            ex_event(x, JS_EX_MARKER_NOTE, (marker != 0xD9) ? 1u : 0u, marker, x.file_pos + x.ptr);        // one normal line; an error line too unless it is EOI
            x.warn_bad_num++;
            if (x.warn_bad_num >= x.err_max) ex_event(x, JS_EX_CAP, 1, x.err_max);
        }
        ex_scanbuf_add(x, b0, x.file_pos + x.ptr, EX_SCANBUF_BADMARK); x.ptr += 1;
    } else { ex_scanbuf_add(x, b0, x.file_pos + x.ptr, EX_SCANBUF_OK); x.ptr += 1; }
}
// ImgDecode.cpp:1292-1323
__device__ __forceinline__ void ex_buff_topup(Ex& x)
{
    bool done = (x.vacant < 8);
    if (x.scan_end) done = true;
    while (!done) {
        ex_buff_add_byte(x);
        if (x.restart_flag) done = true;
        if (x.vacant < 8) done = true;
    }
}
// ImgDecode.cpp:2693-2703 + 4038-4075
__device__ __forceinline__ void ex_restart_scan_buf(Ex& x, uint32_t ptr)
{
    x.scan_end = false; x.scan_bad = false; x.buff = 0; x.ptr = ptr;
    x.align = 0; for (int i = 0; i < 4; i++) { x.pos[i] = 0; x.err[i] = EX_SCANBUF_OK; }
    x.latch_err = EX_SCANBUF_OK; x.num = 0; x.vacant = 32; x.cur_err = false;
    x.restart_flag = false; x.mcus_left = x.rst_interval;
}

// ImgDecode.cpp:1072-1286
__device__ __noinline__ int ex_read_scan_val(Ex& x, uint32_t cls, uint32_t tbl, uint32_t& zrl, int& val)
{
    zrl = 0; val = 0; x.bits_used = 0;
    if (x.vacant == 32 && x.restart_flag) return EX_RSV_RST_TERM;
    if (x.vacant >= 32) {
        ex_warn(x, JS_EX_OVERREAD_BEFORE, 1, x.pos[0], x.align);
        x.scan_end = true; x.scan_bad = true;
        return EX_RSV_UNDERFLOW;
    }
    ex_buff_topup(x);
    const uint32_t e = js_find_code(x.ts, cls * 4 + tbl, x.buff, 32 - x.vacant);
    uint32_t bits1, code;
    if (e) { bits1 = e >> 8; code = e & 0xFF; }
    else {
        if (x.restart_flag) return EX_RSV_RST_TERM;
        bits1 = 1; code = 0xFFFFFFFFu;                       // :1178-1187: move one bit and let the caller try again
    }
    if (bits1 < 17) x.histo[(cls * 4 + tbl) * 17 + bits1]++;
    x.bits_used = bits1;
    ex_scanbuf_consume(x, bits1);
    if (x.vacant > 32) {
        ex_event(x, JS_EX_OVERREAD_AFTER_CODE, 1, x.pos[0], x.align);
        x.scan_end = true; x.scan_bad = true;
        return EX_RSV_UNDERFLOW;
    }
    ex_buff_topup(x);
    if (code != 0xFFFFFFFFu) {
        zrl = (code & 0xF0) >> 4;
        const uint32_t bits2 = code & 0x0F;
        x.bits_used += bits2;
        if (zrl == 0 && bits2 == 0) return EX_RSV_EOB;
        if (bits2 == 0) { val = 0; return EX_RSV_OK; }
        const uint32_t v = x.buff >> (32 - bits2);                                            // ExtractBits, :898-903
        val = js_huff_value(v, bits2, x.precision);
        ex_scanbuf_consume(x, bits2);
        if (x.vacant > 32) {
            ex_event(x, JS_EX_OVERREAD_AFTER_BITS, 1, x.pos[0], x.align);
            x.scan_end = true; x.scan_bad = true;
            return EX_RSV_UNDERFLOW;
        }
        return EX_RSV_OK;
    }
    ex_warn(x, JS_EX_NOCODE, 1, x.pos[0], x.align, tbl, x.buff);
    x.scan_bad = true;
    return EX_RSV_UNDERFLOW;
}

// DecodeScanComp, ImgDecode.cpp:1604-1835, and — print = true — its verbose twin DecodeScanCompPrint (:1859-2090), which differs
// in three ways: every symbol becomes a ReportVlc line, AC coefficients are kept even in DC-only mode, and the IDCT always runs.
// Returns false when the block ended in an underflow (no IDCT is run for it: its samples are the DC alone).
__device__ __noinline__ bool ex_decode_scan_comp(Ex& x, uint32_t tdc, uint32_t tac, uint32_t tdqt, short& dc_lum, short& dc_cb, short& dc_cr,
                                                  bool print, uint32_t mx, uint32_t my)
{
    uint32_t zrl; int val; bool done = false, bdc = true; uint32_t ncoef = 0;
    uint32_t special = 0;                                        // strSpecial: 0 "", 1 EOB, 2 ERROR, 3 EOB64 (keeps its value across symbols)
    for (int i = 0; i < 64; i++) x.dct[i] = 0;
    if (print) ex_detail(x, JSGPU_DT_BLOCK, tdqt, mx, my);
    while (!done) {
        ex_buff_topup(x);
        const uint32_t saved_pos = x.pos[0], saved_err = x.latch_err, saved_align = x.align;
        int r = ex_read_scan_val(x, bdc ? 0 : 1, bdc ? tdc : tac, zrl, val);
        if (r == EX_RSV_RST_TERM) {                              // :1644-1680: the restart is handled where the marker is met
            dc_lum = dc_cb = dc_cr = 0;                              // DecodeRestartDcState (:2693-2703) clears the per-block copies too
            for (int i = 0; i < 16; i++) { x.css[0][i] = 0; x.css[1][i] = 0; x.css[2][i] = 0; }
            x.ptr += 2;
            ex_restart_scan_buf(x, x.ptr);
            x.restart_flag = false;
            ex_buff_topup(x);
            r = ex_read_scan_val(x, bdc ? 0 : 1, bdc ? tdc : tac, zrl, val);
        }
        if (saved_err == EX_SCANBUF_BADMARK) {                   // :1683-1706
            x.cur_err = true; x.scan_bad = true;
            ex_warn(x, JS_EX_BADMARK, 1, saved_pos, saved_align);
            x.latch_err = EX_SCANBUF_OK;
        }
        const uint32_t coef_start = ncoef, coef_end = ncoef + zrl;
        const short v2 = (short)(val & 0xFFFF);
        if (r == EX_RSV_OK) {
            if (print) special = 0;
            if (bdc) { js_idct_set(x.dct, x.ts, tdqt, ncoef, zrl, v2); bdc = false; }
            else if (x.decode_ac || print) js_idct_set(x.dct, x.ts, tdqt, ncoef, zrl, v2);
        } else if (r == EX_RSV_EOB) {
            if (bdc) { js_idct_set(x.dct, x.ts, tdqt, ncoef, zrl, v2); bdc = false; } else done = true;
            special = 1;
        } else if (r == EX_RSV_UNDERFLOW) {                      // :1737-1760
            if (x.warn_bad_num < x.err_max) special = 2;
            ex_warn(x, JS_EX_BADCODE, 1, saved_pos, saved_align);
            x.cur_err = true;
            if (print) if (jsgpu_detail_event* ev = ex_detail_slot(x)) js_detail_vlc(*ev, x.res->nevents, saved_pos, saved_align, zrl, v2, coef_start, coef_end, x.bits_used, special);
            return false;
        }
        ncoef += 1 + zrl;
        if (ncoef == 64) { special = 3; done = true; }
        else if (ncoef > 64) {                                   // :1776-1797
            ex_warn(x, JS_EX_NCOEF, 1, saved_pos, saved_align, ncoef);
            x.cur_err = true; x.scan_bad = true; done = true; ncoef = 64;
        }
        if (print) if (jsgpu_detail_event* ev = ex_detail_slot(x)) js_detail_vlc(*ev, x.res->nevents, saved_pos, saved_align, zrl, v2, coef_start, coef_end, x.bits_used, special);
    }
    if (print) {                                                 // ReportDctMatrix (:2104-2131): the dequantised block, natural order
        const uint32_t nb = x.dt.hdr[1]++;
        if (nb < x.dt.mat_cap) { for (int i = 0; i < 64; i++) x.dt.mat[(size_t)nb * 64 + i] = x.dct[i]; }
        ex_detail(x, JSGPU_DT_MATRIX, nb);
    }
    return true;
}

// One thread re-decodes one damaged image.  grid = images, 32 threads per CTA (lane 0 works).
// The same walk serves the "Detailed Decode" of chosen MCUs (m_bDetailVlc, SetDetailVlc :4898) of a damaged image, and of a healthy
// one when the parallel form (jsgpu_detail.cu) is not taken (JSGPU_DETAIL_WALK=1, no MCU file map) — then without touching any output (the fast path has produced them) except the
// coefficient rows of the printed MCUs in DC-only mode, which the reference decodes in full — and ends after the last MCU of the range.
__global__ void __launch_bounds__(32) k_huff_exact(DevBatch b, int err_max, jsgpu_detail dtl, JsDetailOut dump, uint32_t* scratch_histo)
{
    const uint32_t ii = blockIdx.x;
    if (threadIdx.x != 0) return;
    const bool wr = b.ex_flag[ii] != 0;                          // damaged: this walk produces the outputs
    const bool detail = dtl.enable && dtl.image == ii && b.img[ii].valid;
    if (!wr && !detail) return;
    const DevImage& im = b.img[ii];
    Ex x;
    x.data = b.bits + im.scan_off; x.n = (uint32_t)im.scan_len; x.file_pos = im.file_pos;
    x.ts = b.tables + im.table_set;
    x.res = b.ex_res + ii; x.histo = wr ? b.histo + (size_t)ii * 2 * 4 * 17 : scratch_histo;
    x.res->nerr_lines = 0; x.res->nevents = 0; x.res->scan_bad = 0; x.res->restart_read = 0; x.res->done = 0;
    x.err_max = (uint32_t)err_max; x.warn_bad_num = 0;
    x.precision = im.precision; x.decode_ac = b.decode_ac != 0;
    x.rst_interval = im.restart_en ? im.ri : 0;                 // m_nRestartInterval (0 when DRI is off: never looked at then)
    x.restart_read = 0; x.restart_last = 0; x.restart_expect = 0; x.bits_used = 0;
    x.dt = dump;
    const uint32_t dt_base = dtl.mcu_y * im.mcu_xmax + dtl.mcu_x;
    for (int i = 0; i < 16; i++) { x.css[0][i] = 0; x.css[1][i] = 0; x.css[2][i] = 0; }
    ex_restart_scan_buf(x, 0);
    ex_buff_topup(x);
    short dc_lum = 0, dc_cb = 0, dc_cr = 0;
    const uint32_t ns = im.ns;
    int16_t* const blk_y = b.blk_y + im.blk_off; int16_t* const blk_cb = b.blk_cb + im.blk_off; int16_t* const blk_cr = b.blk_cr + im.blk_off;
    const size_t nb = (size_t)im.blk_xmax * im.blk_ymax;
    bool all_done = false;
    for (uint32_t my = 0; my < im.mcu_ymax && !all_done; my++) {
        bool stop = false;
        for (uint32_t mx = 0; mx < im.mcu_xmax && !stop; mx++) {
            const uint32_t mcu = my * im.mcu_xmax + mx;
            if (!wr && (unsigned long long)mcu >= (unsigned long long)dt_base + dtl.len) { all_done = true; break; }     // nothing left to print
            if (im.restart_en && x.mcus_left == 0 && !x.restart_flag) ex_event(x, JS_EX_RST_MISSING, 1, x.pos[0], x.align);     // :3180-3200
            if (wr) b.mcu_map[im.mcu_off + mcu] = (x.pos[0] << 4) + x.align;                                                       // :3229
            const bool print = detail && mcu >= dt_base && (unsigned long long)mcu < (unsigned long long)dt_base + dtl.len;        // :3235-3241
            if (print) ex_detail(x, JSGPU_DT_MCU);
            for (uint32_t c = 0; c < ns; c++) {
                const uint32_t tdc = im.slot_dc[c], tac = im.slot_ac[c] - 4, tdqt = im.dqt[c];
                for (uint32_t v = 0; v < im.V[c]; v++) for (uint32_t h = 0; h < im.H[c]; h++) {
                    const bool full = ex_decode_scan_comp(x, tdc, tac, tdqt, dc_lum, dc_cb, dc_cr, print, mx, my);
                    if (x.cur_err) {                             // CheckScanErrors, :2605-2660 (two lines per instance)
                        ex_warn(x, JS_EX_MCU, 2, mx, my, c | (h << 8) | (v << 16), x.pos[0], x.align);
                        x.cur_err = false;
                    }
                    short& dc = (c == 0) ? dc_lum : (c == 1) ? dc_cb : dc_cr;
                    dc = (short)(dc + x.dct[0]);                 // :3280, 3355, 3386
                    // the coefficient row the IDCT kernels read: slot 0 = DC sum; AC only when the IDCT ran for this block
                    const bool ac = full && (x.decode_ac || print);
                    if (wr || (print && !x.decode_ac)) {
                        int16_t* row = b.coef + (im.coef_row[c] + (size_t)(my * im.V[c] + v) * im.cw[c] + (mx * im.H[c] + h)) * 64;
                        row[0] = dc;
                        for (int i = 1; i < 64; i++) row[i] = ac ? x.dct[i] : (short)0;
                    }
                    x.css[c][v * 4 + h] = dc;                    // :3282, 3357, 3388
                }
            }
            // block-DC maps, :3524-3608: written after the MCU from the per-block copies (which a restart inside the MCU has
            // cleared), with the reference's own addressing, overlaps included
            if (wr) for (uint32_t c = 0; c < ns; c++)
                for (uint32_t v = 0; v < im.V[c]; v++) for (uint32_t h = 0; h < im.H[c]; h++) {
                    const size_t bi = (size_t)(my * im.ev[c] + v) * im.blk_xmax + (mx * im.eh[c] + h);
                    if (bi < nb) ((c == 0) ? blk_y : (c == 1) ? blk_cb : blk_cr)[bi] = x.css[c][v * 4 + h];
                }
            if (im.restart_en) x.mcus_left--;
            if (x.scan_end && x.scan_bad) stop = true;           // :3621-3625
        }
    }
    if (!wr) return;
    x.res->scan_bad = x.scan_bad ? 1u : 0u; x.res->restart_read = x.restart_read; x.res->done = 1;
    x.res->end_pos = x.pos[0]; x.res->end_align = x.align;
    b.stats[(size_t)ii * 16 + 11] = (int32_t)x.restart_read;     // m_nRestartRead
    b.stats[(size_t)ii * 16 + 12] = (int32_t)x.pos[0]; b.stats[(size_t)ii * 16 + 13] = (int32_t)x.align;
}

// Before the re-decode: which images need it, and their intermediates back to the state the reference starts from
// (ClrFullRes and the memsets of :2900-2965: everything an abandoned decode leaves untouched reads as 0).
__global__ void __launch_bounds__(256) k_exact_prepare(DevBatch b)
{
    const uint32_t ii = blockIdx.x;
    const DevImage& im = b.img[ii];
    const bool need = im.valid && b.img_status[ii] != 0;
    if (threadIdx.x == 0) b.ex_flag[ii] = need ? 1u : 0u;
    if (!need) return;
    for (uint32_t c = 0; c < im.ns; c++) {
        uint4* p = reinterpret_cast<uint4*>(b.coef + im.coef_row[c] * 64);
        const size_t n = (size_t)im.cw[c] * im.ch[c] * 8;
        for (size_t i = threadIdx.x; i < n; i += blockDim.x) p[i] = make_uint4(0, 0, 0, 0);
    }
    const size_t nb = (size_t)im.blk_xmax * im.blk_ymax;
    for (size_t i = threadIdx.x; i < nb; i += blockDim.x) { b.blk_y[im.blk_off + i] = 0; if (im.ns == 3) { b.blk_cb[im.blk_off + i] = 0; b.blk_cr[im.blk_off + i] = 0; } }
    for (uint32_t i = threadIdx.x; i < im.nmcu; i += blockDim.x) b.mcu_map[im.mcu_off + i] = 0;
    for (uint32_t i = threadIdx.x; i < 2 * 4 * 17; i += blockDim.x) b.histo[(size_t)ii * 2 * 4 * 17 + i] = 0;
}

int js_launch_exact(const DevBatch& b, int err_max, const jsgpu_detail& dtl, const JsDetailOut& dump, uint32_t* scratch_histo, cudaStream_t s)
{
    if (b.nimg == 0) return 0;
    k_exact_prepare<<<b.nimg, 256, 0, s>>>(b);
    k_huff_exact<<<b.nimg, 32, 0, s>>>(b, err_max, dtl, dump, scratch_histo);
    return 2;
}
