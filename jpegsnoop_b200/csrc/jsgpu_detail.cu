// jsgpu_detail.cu — the "Detailed Decode" of an MCU range (SetDetailVlc, ImgDecode.cpp:4880-4904) of a HEALTHY image, in
// parallel: one thread per MCU.
//
// The Huffman stage has recorded where every MCU starts inside its restart interval (mcu_bitpos, unstuffed bits; inside the
// real interval on the self-synchronising path too), so an MCU's symbols can be decoded without the ones before it.  Each
// thread decodes its MCU the way DecodeScanCompPrint does (:1859-2094) and reports what the serial walk of jsgpu_exact.cu
// reports for it, in the same encoding (jsgpu_detail.cuh): the separator, one line per block, one ReportVlc line per symbol
// (:2152-2232), one ReportDctMatrix per block (:2104-2131).
//   k_detail_count  how many events each MCU makes (blocks per MCU are fixed: bpm); in DC-only mode it also writes the printed
//                   blocks' full coefficient rows before the IDCT, as DecodeScanCompPrint runs the IDCT on them;
//   k_detail_scan   exclusive scan of the counts (one CTA) -> event offsets and totals, which the host reads to size the arrays;
//                   and the one scan event a healthy walk can meet, the end-of-scan marker note, written where the walk would;
//   k_detail_emit   the events and matrices (runs after the MCU file map: the first symbol after an RSTn is reported where the
//                   previous interval left the reader, the map entry of that MCU, ImgDecode.cpp:1644-1680, 3229).
// Damaged images take the serial walk instead (jsgpu_exact.cu): resynchronisation and lazy restarts are not interval-local.
#include "jsgpu_detail.cuh"
#include "jsgpu_scan.cuh"
#include <climits>

#define DT_THREADS 128

// the 32 bits from bit `bit` on of one restart interval's unstuffed copy (stored as big-endian 32-bit words, padded past its end:
// a healthy scan decodes no symbol that reaches the padding)
struct DtBits {
    const uint32_t* w;
    __device__ __forceinline__ uint32_t peek(uint32_t bit) const {
        const uint32_t i = bit >> 5;
        return __funnelshift_l(__ldg(w + i + 1), __ldg(w + i), bit & 31);
    }
};

// The marker that ends the scan, as BuffAddByte meets it (ImgDecode.cpp:1486-1561: an FF followed by neither 00, FF nor RSTn).
// The accumulator is topped up to at least 25 bits before every code and after it (BuffTopup :1292-1323), so the walk reaches
// that marker at the first top-up, in the last interval, with at least 8 D - 24 bits consumed (D = the interval's unstuffed
// bytes).  Returns that threshold, LLONG_MAX when the scan has no such marker.
__device__ __forceinline__ long long dt_marker_threshold(const DevBatch& b, const DevImage& im, uint32_t ii, uint32_t& marker)
{
    const uint64_t se = b.scan_end[ii];
    const uint32_t b0 = (se < im.scan_len) ? b.bits[im.scan_off + se] : 0u, b1 = (se + 1 < im.scan_len) ? b.bits[im.scan_off + se + 1] : 0u;
    marker = b1;
    if (b0 != 0xFF || b1 == 0x00 || b1 == 0xFF || (b1 >= 0xD0 && b1 <= 0xD7)) return LLONG_MAX;
    return 8ll * b.seg_ulen[im.seg_first + im.nseg - 1] - 24;
}

// Decodes MCU m (a healthy one) as DecodeScanCompPrint does.  Returns its event count; lastp = the last top-up point (bits
// consumed when the last code of the MCU had been read).  EMIT: writes the events to ev[] and the matrices from mat[] on,
// with seq = note_n once the end-of-scan marker has been met (prev_met: before this MCU; T: dt_marker_threshold).
// ROWS: writes the coefficient rows of the MCU's blocks (AC included; slot 0, the running DC sum, stays).
template <bool EMIT, bool ROWS>
__device__ uint32_t dt_mcu(const DevBatch& b, const DevImage& im, uint32_t m, long long T, uint32_t note_n, bool prev_met,
                           jsgpu_detail_event* ev, int16_t* mat, uint32_t mat0, uint32_t& lastp)
{
    const uint32_t k = m / im.ri, t = m - k * im.ri, sidx = im.seg_first + k;
    const bool last = k + 1 == im.nseg;
    const DtBits in = { reinterpret_cast<const uint32_t*>(b.ubits + b.seg_uoff[sidx]) };
    const DevTableSet* ts = b.tables + im.table_set;
    const uint32_t pos0 = im.file_pos + b.seg_start[sidx];
    const uint32_t mx = m % im.mcu_xmax, my = m / im.mcu_xmax;
    uint32_t bit = (t > 0) ? b.mcu_bitpos[im.mcu_off + m] : 0u;
    bool lazy = t == 0 && k > 0;                                   // the first symbol after an RSTn
    bool met = prev_met;
    JsRawCursor cur = { ~0u, 0, 0 };                                // symbol positions only increase inside the MCU
    uint32_t nev = 0, blk = 0;
    lastp = bit;
    if (EMIT) js_detail_put(ev[nev], JSGPU_DT_MCU, met ? note_n : 0u);
    nev++;
    for (uint32_t c = 0; c < im.ns; c++) {
        const uint32_t tdc = im.slot_dc[c], tac = im.slot_ac[c] - 4, tdqt = im.dqt[c];
        for (uint32_t v = 0; v < im.V[c]; v++) for (uint32_t h = 0; h < im.H[c]; h++) {
            short dct[64];
            for (int i = 0; i < 64; i++) dct[i] = 0;
            if (EMIT) js_detail_put(ev[nev], JSGPU_DT_BLOCK, met ? note_n : 0u, tdqt, mx, my);
            nev++;
            uint32_t ncoef = 0, special = 0;
            bool bdc = true, done = false;
            while (!done) {
                const uint32_t s = bit;
                const uint32_t e = js_find_code(ts, bdc ? tdc : 4 + tac, in.peek(bit), 32);
                const uint32_t cl = e >> 8, code = e & 0xFF, zrl = code >> 4, bits2 = code & 15;
                bit += cl; lastp = bit;                              // top-up after the code
                if (last && (long long)bit >= T) met = true;
                int val = 0;
                if (bits2) { val = js_huff_value(in.peek(bit) >> (32 - bits2), bits2, im.precision); bit += bits2; }
                const short v2 = (short)(val & 0xFFFF);
                const uint32_t coef_start = ncoef, coef_end = ncoef + zrl;
                if (zrl == 0 && bits2 == 0) {                        // EOB (for the DC symbol: a difference of 0)
                    if (bdc) { js_idct_set(dct, ts, tdqt, ncoef, zrl, v2); bdc = false; } else done = true;
                    special = 1;
                } else {
                    special = 0;
                    js_idct_set(dct, ts, tdqt, ncoef, zrl, v2);      // printed: AC kept even in DC-only mode
                    bdc = false;
                }
                ncoef += 1 + zrl;
                if (ncoef == 64) { special = 3; done = true; }
                else if (ncoef > 64) done = true;                    // (flags the image: it takes the serial walk)
                if (EMIT) {
                    uint32_t pos, align;
                    if (lazy) { const uint32_t mm = b.mcu_map[im.mcu_off + m]; pos = mm >> 4; align = mm & 15; }
                    else { pos = pos0 + js_raw_of_unstuffed(b, im, k, s >> 3, &cur); align = s & 7; }
                    js_detail_vlc(ev[nev], met ? note_n : 0u, pos, align, zrl, v2, coef_start, coef_end, cl + bits2, special);
                }
                lazy = false;
                nev++;
            }
            if (EMIT) {
                int16_t* mt = mat + (size_t)(mat0 + blk) * 64;
                for (int i = 0; i < 64; i++) mt[i] = dct[i];
                js_detail_put(ev[nev], JSGPU_DT_MATRIX, met ? note_n : 0u, mat0 + blk);
            }
            nev++;
            if (ROWS) {
                int16_t* row = b.coef + (im.coef_row[c] + (size_t)(my * im.V[c] + v) * im.cw[c] + (mx * im.H[c] + h)) * 64;
                for (int i = 1; i < 64; i++) row[i] = dct[i];
            }
            blk++;
        }
    }
    return nev;
}

// MCUs first .. first + n - 1 of image `image`; those from `base` on are printed.  first = base - 1 (or the last MCU the walk
// decodes when nothing is printed): its last top-up tells whether the marker was met before the first printed line.
__global__ void __launch_bounds__(DT_THREADS) k_detail_count(DevBatch b, JsDetailRange r, uint32_t* cnt, uint32_t* lastp, int rows)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= r.n) return;
    const DevImage& im = b.img[r.image];
    const uint32_t m = r.first + j;
    const bool print = m >= r.base;
    uint32_t lp, nev;
    if (print && rows) nev = dt_mcu<false, true>(b, im, m, LLONG_MAX, 0, false, nullptr, nullptr, 0, lp);
    else nev = dt_mcu<false, false>(b, im, m, LLONG_MAX, 0, false, nullptr, nullptr, 0, lp);
    cnt[j] = print ? nev : 0u;
    lastp[j] = lp;
}

__global__ void __launch_bounds__(1024) k_detail_scan(DevBatch b, JsDetailRange r, uint32_t* cnt, const uint32_t* lastp, uint32_t* hdr, JsErrCfg cfg)
{
    __shared__ uint32_t s_warp[33];
    const uint32_t tid = threadIdx.x;
    uint32_t total = 0;
    for (uint32_t base = 0; base < r.n; base += 1024) {
        uint32_t* const c = cnt + base + tid;
        const bool in = base + tid < r.n;
        const uint32_t excl = js_block_scan<1024>(in ? *c : 0u, 0u, js_add, total, s_warp);
        if (in) *c = excl;
    }
    if (tid != 0) return;
    const DevImage& im = b.img[r.image];
    hdr[0] = total; hdr[1] = r.nprint * im.bpm;
    // the end-of-scan marker note (BuffAddByte, ImgDecode.cpp:1527-1543) when the walk's last top-up reaches it and the cap still
    // allows a line, plus the cap line when this one reaches it (:1100-1110); the fields the walk sets for a healthy image, the
    // others as they were
    uint32_t marker;
    const long long T = dt_marker_threshold(b, im, r.image, marker);
    bool met;
    if (r.n) met = (r.first + r.n - 1) / im.ri + 1 == im.nseg && (long long)lastp[r.n - 1] >= T;
    else met = im.nseg == 1 && 0 >= T;                           // nothing decoded: the first top-up only
    JsExResult* res = b.ex_res + r.image;
    js_ex_reset(res);
    uint32_t warn = cfg.warn_start;
    if (met) js_ex_warn(res, res->ev, JS_EX_MAX_EVENTS, cfg.err_max, warn, JS_EX_MARKER_NOTE, marker != 0xD9, marker, im.file_pos + b.scan_end[r.image]);
    res->warn_num = warn;
}

__global__ void __launch_bounds__(DT_THREADS) k_detail_emit(DevBatch b, JsDetailRange r, const uint32_t* off, const uint32_t* lastp, JsDetailOut out)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= r.nprint) return;
    const DevImage& im = b.img[r.image];
    const uint32_t m = r.base + j, jj = m - r.first;
    uint32_t marker;
    const long long T = dt_marker_threshold(b, im, r.image, marker);
    const uint32_t k = m / im.ri, t = m - k * im.ri;
    const bool last = k + 1 == im.nseg;
    const bool prev_met = last && (t ? (long long)lastp[jj - 1] >= T : (k == 0 && 0 >= T));
    uint32_t lp;
    dt_mcu<true, false>(b, im, m, T, b.ex_res[r.image].nevents, prev_met, out.ev + off[jj], out.mat, j * im.bpm, lp);
}

int js_launch_detail_count(const DevBatch& b, const JsDetailRange& r, uint32_t* scratch, uint32_t* hdr, const JsErrCfg& cfg, cudaStream_t s)
{
    uint32_t* cnt = scratch; uint32_t* lastp = scratch + r.n;
    int n = 0;
    if (r.n) { k_detail_count<<<(r.n + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, s>>>(b, r, cnt, lastp, b.decode_ac ? 0 : 1); n++; }
    k_detail_scan<<<1, 1024, 0, s>>>(b, r, cnt, lastp, hdr, cfg);
    return n + 1;
}

int js_launch_detail_emit(const DevBatch& b, const JsDetailRange& r, const uint32_t* scratch, const JsDetailOut& out, cudaStream_t s)
{
    if (!r.nprint) return 0;
    k_detail_emit<<<(r.nprint + DT_THREADS - 1) / DT_THREADS, DT_THREADS, 0, s>>>(b, r, scratch, scratch + r.n, out);
    return 1;
}
