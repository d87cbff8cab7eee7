// jsgpu_internal.h — device-side data layout shared by the kernels (jsgpu_kernels.cu) and the
// C-ABI / host orchestration (jsgpu_api.cu).  See DESIGN.md §3 "Data layout in HBM".
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include <string>
#include "../../include/jsgpu.h"

#define JS_LUT_BITS   10                 // direct Huffman look-up width (reference uses 9: ImgDecode.h:96)
#define JS_LUT_SIZE   (1 << JS_LUT_BITS)
#define JS_LUT2_BITS  (16 - JS_LUT_BITS)
#define JS_LUT2_SIZE  8192               // second-level entries per slot (256 sub-tables of 32)
#define JS_MAX_CODES  260
#define JS_USLACK     48                 // bytes of slack per restart interval in the unstuffed pool (16 pad + flush rounding + alignment)
#define JS_STUFF_LIST 6                  // stuffed-byte positions recorded per restart interval
#define JS_MAX_DEVICES 64                // per-device "function attribute set" flags of the launchers
#define JS_H100_SMS   132u               // grid-size heuristics of the small helper kernels (the main kernels take the device's SM count)
#define JS_NSLOT      8                  // (class,Th) pairs: slot = class*4 + Th

// An owning, growable buffer of device memory (DevBuf) or pinned host memory (PinBuf).  reserve(n) keeps it while it holds
// n bytes; otherwise it is replaced, contents lost, by one of n + n/8 + 256 bytes, so that slowly growing sizes rarely reallocate.
template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct OwnedBuf {
    void* p = nullptr; size_t cap = 0;
    OwnedBuf() = default;
    OwnedBuf(const OwnedBuf&) = delete;
    OwnedBuf& operator=(const OwnedBuf&) = delete;
    ~OwnedBuf() { if (p) Free(p); }
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) Free(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 256;
        cudaError_t e = Alloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    template <class T> T* as() const { return (T*)p; }
};
using DevBuf = OwnedBuf<cudaMalloc, cudaFree>;
using PinBuf = OwnedBuf<cudaMallocHost, cudaFreeHost>;

// serial reference-semantics path (jsgpu_exact.cu): per-image result = the public jsgpu_scan_errors
typedef jsgpu_scan_errors JsExResult; typedef jsgpu_scan_event JsExEvent;
#define JS_EX_MAX_EVENTS JSGPU_MAX_EVENTS
#define JS_EX_OVERREAD_BEFORE JSGPU_EV_OVERREAD_BEFORE
#define JS_EX_OVERREAD_AFTER_CODE JSGPU_EV_OVERREAD_AFTER_CODE
#define JS_EX_OVERREAD_AFTER_BITS JSGPU_EV_OVERREAD_AFTER_BITS
#define JS_EX_NOCODE JSGPU_EV_NOCODE
#define JS_EX_CAP JSGPU_EV_CAP
#define JS_EX_RST_MISMATCH JSGPU_EV_RST_MISMATCH
#define JS_EX_MARKER_NOTE JSGPU_EV_MARKER_NOTE
#define JS_EX_BADMARK JSGPU_EV_BADMARK
#define JS_EX_BADCODE JSGPU_EV_BADCODE
#define JS_EX_NCOEF JSGPU_EV_NCOEF
#define JS_EX_MCU JSGPU_EV_MCU
#define JS_EX_RST_MISSING JSGPU_EV_RST_MISSING

// Device form of one jsgpu_tables set.
struct DevTableSet {
    // two-level direct look-up (first match in SetDhtEntry order, exactly like ImgDecode.cpp:1145-1164):
    //   lut[slot][top JS_LUT_BITS bits]: (len<<8)|symbol for a code of len <= JS_LUT_BITS,
    //                                    0x8000|offset  -> second level, 0 -> no code has this prefix
    //   lut2[slot][offset + next (16-JS_LUT_BITS) bits]: (len<<8)|symbol, 0 -> no code
    uint16_t lut[JS_NSLOT][JS_LUT_SIZE];
    uint16_t lut2[JS_NSLOT][JS_LUT2_SIZE];
    uint32_t lut2_overflow[JS_NSLOT];        // 1: second level did not fit -> in-order entry search for 0x8000 prefixes
    uint32_t lut2_used[JS_NSLOT];            // second-level entries in use (a multiple of 1 << JS_LUT2_BITS)
    uint32_t ent_bits[JS_NSLOT][JS_MAX_CODES];   // left-justified code bits, in SetDhtEntry order
    uint8_t  ent_len [JS_NSLOT][JS_MAX_CODES];
    uint8_t  ent_sym [JS_NSLOT][JS_MAX_CODES];
    uint32_t ent_n[JS_NSLOT];
    uint32_t qz[4][64];                      // per DQT id, zig-zag position k: quantiser | natural_index<<16
};

// Device descriptor of one image of the batch.
struct DevImage {
    uint32_t valid;                 // 0 = skipped (the reference would return early)
    uint32_t ns, precision;
    uint32_t mcu_w, mcu_h, mcu_xmax, mcu_ymax, blk_xmax, blk_ymax, wp, hp;
    uint32_t nmcu;
    uint32_t ri;                    // MCUs per restart interval (= nmcu when DRI is off)
    uint32_t restart_en;
    uint32_t nseg, seg_first;       // expected segments; index of the first one in the segment arrays
    uint32_t bpm;                   // blocks per MCU
    uint32_t H[3], V[3], eh[3], ev[3];
    uint32_t slot_dc[3], slot_ac[3];// LUT slot per component
    uint32_t tab_sig;               // ns, slots and DQT selectors packed: equal (table_set, tab_sig) <=> same staged decode tables
                                    // (not the same MCU layout: sampling factors and precision are not in it, k_ph_sync restages those per image)
    uint32_t dqt[3];
    uint32_t table_set;
    uint32_t file_pos;              // file offset of scan_off
    uint32_t cw[3], ch[3];          // coefficient plane size in blocks
    uint64_t scan_off, scan_len;    // into the batch bitstream
    uint64_t coef_row[3];           // first 128-byte row of each component plane in the coef pool
    uint64_t pix_off, dib_off, blk_off, mcu_off;
    uint64_t ubits_off;             // this image's region in the unstuffed-bitstream pool
    uint32_t std_layout;            // 1 = every component has H in {1,Hmax} and V in {1,Vmax} (fused IDCT kernel applies)
    uint32_t tile_mcus;             // MCUs per IDCT tile (32 / Hmax)
    uint32_t tiles_per_row;
    uint32_t psync;                 // 1 = long restart intervals: decoded through the self-synchronising passes (jsgpu_phuff_core.cuh)
    uint32_t ph_nslots;             // ... number of 4096-bit slots reserved for this image (its slot arrays hold ph_nslots + 1 entries)
    uint64_t ph_first;              // ... first entry of this image in the slot arrays
    uint32_t cs_nslots;             // ... 4096-byte chunk slots of k_unstuff_long reserved for this image
    uint64_t cs_first;              // ... first entry of this image in the chunk arrays
    uint64_t mc_first;              // first 4096-byte chunk of this image in the marker-scan chunk arrays (k_marker_scan2)
    uint32_t mc_n, mc_pad;          // ... and how many it has
    uint64_t row_off;               // first entry of this image in the per-pixel-row array of the preview pass (jsgpu_preview.cu)
    uint64_t rt_off;                // first entry of this image in the row table (k_unstuff: unstuffed bytes before every 128-byte raw row of a long interval)
};

// Everything a kernel needs about the current batch (passed by value).
struct DevBatch {
    const DevImage*    img;
    const DevTableSet* tables;
    uint32_t           nimg;
    const uint8_t*     bits;        // batch bitstream
    uint64_t           bits_len;
    // segments (expected count per image; seg_end == seg_start for missing ones)
    uint32_t*          seg_start;   // relative to img.scan_off
    uint32_t*          seg_end;
    uint32_t*          seg_endbits; // unstuffed bit position where decoding of the segment stopped
    uint32_t*          seg_status;
    uint32_t*          seg_ulen;    // unstuffed length of each interval
    uint32_t*          seg_nstuff;  // number of stuffed zeros in each interval
    uint32_t*          seg_stuff;   // [nseg][JS_STUFF_LIST] unstuffed index of the FF before each stuffed zero
    unsigned long long* seg_uoff;   // where its unstuffed copy starts in ubits
    uint8_t*           ubits;       // unstuffed, 16-byte aligned, 0xFF-padded copies of all intervals
    uint32_t           nseg_total;
    uint32_t*          mc_img;      // marker scan: image of every 4096-byte chunk (all images back to back)
    unsigned long long* mc_state;   // ... its look-back word (status | end-of-scan seen | RST markers), zeroed per decode; [mc_total] = ticket counter
    uint32_t           mc_total;
    uint32_t*          scan_end;    // [nimg] relative offset of the terminating marker
    uint32_t*          nseg_found;  // [nimg]
    // work lists
    const uint2*       items;       // Huffman, warp kernel: (image, first segment), JS_HUFF_WARPS per item
    uint32_t           nitems;
    const uint2*       litems;      // Huffman, lane kernel: (image, first segment), JS_LANE_SEGS per item
    uint32_t           nlitems;
    const uint2*       items_np;    // the same two lists without the images that take the self-synchronising path
    uint32_t           nitems_np;
    const uint2*       litems_np;
    uint32_t           nlitems_np;
    const uint2*       vitems;      // self-synchronising passes and the lane kernel over virtual intervals: (image, first slot), JS_LANE_SEGS per item
    uint32_t           nvitems;
    // slot arrays of the self-synchronising passes (all images back to back, see PhSlots)
    unsigned long long* ph_x; uint32_t* ph_ver; uint32_t* ph_k; uint4* ph_cnt; uint4* ph_aux; uint4* ph_pre;
    uint32_t*          ph_nchg;     // [PH_MAX_ROUNDS + 2] slots whose exit state changed in fix round r
    uint32_t*          ph_list[2];  // fix round r >= 2 works through the slots whose predecessor changed in round r-1: per image a list (at its
    uint32_t*          ph_nl[2];    // ph_first) written in round r-1 into ph_list[(r-1)&1], its length in ph_nl[(r-1)&1][image]
    uint32_t*          cs_cnt; uint32_t* cs_off; uint32_t* cs_seg;    // k_unstuff_long: bytes kept per chunk, their exclusive prefix, owning interval
    uint32_t*          rowtab;      // self-synchronised images: unstuffed bytes before every 128-byte raw row of an interval ...
    uint4*             rowmask;     // ... and which of the row's 128 raw bytes do not reach the unstuffed copy (MCU file map without a re-walk)
    const uint4*       tiles;       // IDCT: (image, mcu_row, mcu_col0, nmcu) [ntiles], grouped by chroma replication class
    uint32_t           ntiles;
    uint32_t           tcls_first[3], tcls_count[3];   // tiles whose images have chroma eh = 1, 2, 4
    // pools
    int16_t*           coef;        // 64 int16 per block, natural order, slot 0 = cumulative DC
    uint32_t*          mcu_bitpos;  // unstuffed bit offset of each MCU start within its segment
    int16_t*           pix_y; int16_t* pix_cb; int16_t* pix_cr;
    uint8_t*           dib;
    int16_t*           blk_y; int16_t* blk_cb; int16_t* blk_cr;
    uint32_t*          mcu_map;
    uint32_t*          histo;       // [nimg][2][4][17]
    int32_t*           stats;       // [nimg][16]
    unsigned long long* bright_key; // [nimg] packed (Y+32768)<<32 | ~pixel_index
    unsigned long long* sum_y;      // [nimg]
    uint32_t*          img_status;  // [nimg]
    uint32_t*          ex_flag;     // [nimg] 1 = re-decoded by the serial reference-semantics path (k_huff_exact): the finalize kernels leave its MCU map alone
    JsExResult*        ex_res;      // [nimg] its error events
    // options
    int                decode_ac, want_histo, idct_mode;
    uint32_t           max_nseg;             // most restart intervals in one image of the batch
    uint32_t*          ovf_count;            // number of intervals with more stuffed bytes than JS_STUFF_LIST ...
    uint32_t*          ovf_list;             // ... and their segment indices (appended by k_unstuff, walked by k_finalize_mcumap)
    uint32_t           lane_nlut;            // lane Huffman kernel: most distinct (class,Th) tables any image uses (<= 6)
    int                lane_l2_smem;         // ... and every used table's second level fits JS_LANE_L2S entries
    int                any_p12;              // some image has sample precision > 8 (ReadScanVal's divide, ID:1234-1238)
    int                simple_only_nonstd;   // simple IDCT kernels skip images the fused kernel handled
    uint32_t           tile_plane_bytes;     // shared-memory plane bytes the largest tile needs
};

#define JS_HUFF_WARPS 4              // warps (= restart intervals in flight) per Huffman CTA, warp kernel
#define JS_LANE_SEGS  256            // restart intervals per CTA pass, lane kernel (8 warps x 32 lanes)
#define JS_LANE_L2S   512            // second-level entries per table the lane kernel stages in shared memory
#define JS_LANE_TAB   (JS_LUT_SIZE + JS_LANE_L2S)   // entries per staged table: first level, then its second level
#define JS_PSYNC_MIN_BLOCKS 192      // blocks per restart interval from which an image takes the self-synchronising path

// launchers (jsgpu_kernels.cu) — each returns the number of kernels it enqueued
int js_launch_marker_scan(const DevBatch& b, uint64_t max_scan_len, cudaStream_t s);
int js_launch_unstuff(const DevBatch& b, cudaStream_t s);
int js_launch_unstuff_long(const DevBatch& b, uint32_t max_cs, cudaStream_t s);      // images with long intervals (DevImage::psync)
int js_launch_huffman_warp(const DevBatch& b, int sm_count, cudaStream_t s);
int js_launch_huffman_lane(const DevBatch& b, int sm_count, cudaStream_t s);
int js_launch_huffman_lane_vseg(const DevBatch& b, int sm_count, cudaStream_t s);   // over the virtual intervals the self-synchronising passes found
int js_launch_selfsync(const DevBatch& b, int sm_count, cudaStream_t s);            // guess + fix rounds + scan (jsgpu_phuff.cu)
int js_launch_idct_simple(const DevBatch& b, const int32_t* li, const float* lf, cudaStream_t s);
struct IdctSym; struct ColorTabs;
// phase 1 of the fused tile kernel (jsgpu_idct.cu): integer IDCT with the table in shared memory or as immediates, float IDCT
enum JsTileIdct { JS_TILE_INT_SMEM, JS_TILE_INT_BAKED, JS_TILE_FLOAT };
int js_launch_idct_fused(const DevBatch& b, const IdctSym* sym, const ColorTabs* ctab, int sm_count, JsTileIdct idct, cudaStream_t s);
int js_idct_baked_matches(const int32_t* li);
int js_idctf_baked_matches(const float* lf);
int js_launch_build_color_tables(ColorTabs* t, cudaStream_t s);
// "Detailed Decode" (jsgpu_set_detail): where it writes — the event and matrix arrays the context sized for this decode and
// their counters (hdr[0] events, hdr[1] blocks, counted in full; an array keeps what fits its capacity; hdr[2] the path) ...
struct JsDetailOut {
    jsgpu_detail_event* ev; int16_t* mat; uint32_t* hdr;
    unsigned long long ev_cap, mat_cap;
};
// ... and, for the parallel path (jsgpu_detail.cu), which MCUs: first .. first+n-1 are decoded, base .. base+nprint-1 printed
struct JsDetailRange { uint32_t image, base, first, n, nprint; };
// the error report's state at the start of a scan: m_nScanErrMax, m_nWarnBadScanNum, m_bScanErrorsDisable
struct JsErrCfg { uint32_t err_max, warn_start, disable; };
int js_launch_exact(const DevBatch& b, const JsErrCfg& cfg, const jsgpu_detail& dtl, const JsDetailOut& dump, uint32_t* scratch_histo, cudaStream_t s);       // damaged images, again, with the reference's semantics (jsgpu_exact.cu)
// the same walk of one image for its events alone (no output is written): events 0 .. ev_cap-1 go to ev, the counts to *res
int js_launch_exact_events(const DevBatch& b, uint32_t image, const JsErrCfg& cfg, JsExResult* res, uint32_t* scratch_histo, JsExEvent* ev, uint32_t ev_cap, cudaStream_t s);
int js_launch_detail_count(const DevBatch& b, const JsDetailRange& r, uint32_t* scratch, uint32_t* hdr, const JsErrCfg& cfg, cudaStream_t s);   // count pass + scan (+ DC-only rows)
int js_launch_detail_emit(const DevBatch& b, const JsDetailRange& r, const uint32_t* scratch, const JsDetailOut& out, cudaStream_t s);  // events + matrices (after the MCU file map)
int js_launch_export(const DevBatch& b, uint32_t image, int mode, uint8_t* out, uint64_t npx, int sm_count, cudaStream_t s);   // Export-to-TIFF sample array
int js_launch_finalize_maps(const DevBatch& b, cudaStream_t s);     // MCU file map (independent of the IDCT)
int js_launch_finalize_stats(const DevBatch& b, cudaStream_t s);    // brightest pixel / average luma / end-of-scan position (after the IDCT)
// CalcChannelPreviewFull with non-default settings: clipping/histogram conversion, channel selection, YCC shift (jsgpu_preview.cu)
int js_launch_preview(const DevBatch& b, const jsgpu_preview& pv, jsgpu_colour_stats* st, uint32_t* rowclip, uint64_t rows_total,
                      uint32_t max_hp, int sm_count, cudaStream_t s);
// byte-pattern search (jsgpu_search.cu): its own streams and buffers, created on first use and kept by the context
struct JsSearch;
int  js_search_run(JsSearch** s, int device, int sm_count, const uint8_t* data, uint64_t n, const uint8_t* pats, const uint32_t* lens,
                   uint32_t npat, uint64_t* counts, uint32_t* pos, uint64_t cap, std::string& err);
int  js_find_run(JsSearch** s, int device, int sm_count, const uint8_t* data, uint64_t n, uint64_t start, uint32_t value,
                 uint32_t len, int forward, const jsgpu_overlay* ovl, uint32_t novl, int* found, uint64_t* found_pos, std::string& err);
int  js_find_all_run(JsSearch** s, int device, int sm_count, const uint8_t* data, uint64_t n, uint32_t value, uint32_t len,
                     uint64_t* count, uint32_t* pos, uint64_t cap, std::string& err);
int  js_find_markers_run(JsSearch** s, int device, int sm_count, const uint8_t* data, uint64_t n, const jsgpu_overlay* ovl,
                         uint32_t novl, uint32_t* soi_pos, uint64_t soi_cap, uint64_t* nsoi, uint32_t* term_pos, uint64_t term_cap,
                         uint64_t* nterm, std::string& err);
void js_search_free(JsSearch* s);
#define JSGPU_CK_WORDS_INTERNAL 12   // == JSGPU_CK_WORDS (include/jsgpu.h)
int js_launch_checksums(const DevBatch& b, unsigned long long* ck, cudaStream_t s);
int js_launch_finalize_emptied(const DevBatch& b, cudaStream_t s);   // after js_launch_finalize: drained-interval MCU map entries

// Quadrant-symmetric decomposition of the integer IDCT table (built on the host at table upload,
// jsgpu_api.cu): Li[y][x][vu] = sign * S[min(y,7-y)][min(x,7-x)][vu] + D, where the sign flips with the
// parity of u (x mirrored) and v (y mirrored), and D is non-zero only for `ncorr` coefficient positions.
struct IdctSym {
    int32_t s4[64][4][4];        // [vu][q/4][q%4]: S for quadrant sample q = y*4+x (y,x < 4), int4-friendly
    int32_t ncorr;               // number of coefficient positions with a non-zero correction (<= 4), -1 = not decomposable
    int32_t corr_pos[4];         // their natural indices
    int32_t corr[4][64];         // D[j][yx]
};

// Verified integer form of ConvertYCCtoRGBFastFloat (built and checked on the device by
// k_build_color_tables): R = clamp(y + tr[cr]), B = clamp(y + tb[cb]), G = clamp(y + tg[cb][cr]);
// tg == 0x7FFF marks the (cb,cr) pairs for which the additive form is not exact for every y.
struct ColorTabs {
    int16_t tr[256], tb[256];
    int32_t rb_ok, n_unsafe;
    int16_t tg[65536];
    // arithmetic form of the G term: tg - 128 == (-(JS_GA*cb + JS_GB*cr)) >> 23 wherever the matching bit of
    // gflag is clear (verified on the device for all 65536 pairs); set bits (and tg == 0x7FFF) take the exact path
    uint32_t gflag[2048];
    int32_t n_gflag;
};
#define JS_GA 2886824        // 0.114f*(2-2*0.114f)/0.587f * 2^23
#define JS_GB 5990609        // 0.299f*(2-2*0.299f)/0.587f * 2^23
