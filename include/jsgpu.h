/* jsgpu.h — C-ABI of the H100 scan decoder (libjsgpu.so).
 *
 * This is the drop-in boundary for JPEGsnoop's per-MCU scan-decode path.  Everything above
 * it (the CimgDecode class with the reference's public surface, see
 * jpegsnoop_b200/csrc/host/ImgDecode.h) is host C++; everything below it is hand-written
 * CUDA for sm_90a.  Signatures use plain pointers and sizes only.  Every entry point names
 * the reference interface it replaces (paths relative to /root/reference/source).
 *
 * Conventions: every function returns JSGPU_OK (0) or a negative JSGPU_E* code and never
 * throws; jsgpu_last_error() gives text for the last failure on that context.  A context is
 * bound to one CUDA device and must be driven from one host thread at a time (the reference
 * decoder is single-threaded and non-re-entrant too: ImgDecode.cpp:142-234).  The context
 * owns all device memory; pointers it hands out stay valid until the next
 * jsgpu_batch_begin() / jsgpu_free() on that context.  There is NO CPU fallback: without a
 * CUDA device jsgpu_init() fails with JSGPU_ENODEV.
 */
#ifndef JSGPU_H
#define JSGPU_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define JSGPU_OK          0
#define JSGPU_ENODEV     -1   /* no usable CUDA device / driver                      */
#define JSGPU_EINVAL     -2   /* bad argument or descriptor                          */
#define JSGPU_ENOMEM     -3   /* device or pinned-host allocation failed             */
#define JSGPU_ECUDA      -4   /* a CUDA call or kernel failed                        */
#define JSGPU_ESTATE     -5   /* call out of order (e.g. decode before batch_begin)  */
#define JSGPU_EUNSUP     -6   /* image not decodable by this path (as the reference: */
                              /* Ns not in {1,3}, sampling factor > 4, ...)          */

#define JSGPU_MAX_DHT_CODES 260     /* MAX_DHT_CODES, ImgDecode.h:68 */

typedef struct jsgpu_ctx jsgpu_ctx;

/* One set of decode tables = the state CimgDecode holds after CjfifDecode's DQT/DHT setter
 * calls: m_anDqtCoeffZz (ImgDecode.h:570, filled by SetDqtEntry ImgDecode.cpp:424-453) and
 * m_anDhtLookup_{bitlen,bits,code} + m_anDhtLookupSize (ImgDecode.h:609-613, filled by
 * SetDhtEntry/SetDhtSize ImgDecode.cpp:748-847).  Entry order is the order of SetDhtEntry
 * calls (canonical: length ascending, code ascending — JfifDecode.cpp:3535-3595); the
 * decoder honours "first matching entry wins" (ImgDecode.cpp:1145-1164).  POD on purpose:
 * this is the blob that is broadcast rank0 -> all ranks over NCCL before a multi-GPU batch. */
typedef struct {
    uint16_t dqt_zz[4][64];                          /* quantiser of zig-zag position k   */
    uint32_t dht_size[2][4];                         /* [class DC=0/AC=1][Th]             */
    uint32_t dht_bits[2][4][JSGPU_MAX_DHT_CODES];    /* code << (32-len), left-justified  */
    uint8_t  dht_len [2][4][JSGPU_MAX_DHT_CODES];    /* code length 1..16                 */
    uint8_t  dht_code[2][4][JSGPU_MAX_DHT_CODES];    /* symbol byte (run<<4 | size)       */
} jsgpu_tables;

/* One image of a batch = the arguments of SetImageDetails / SetSofSampFactors /
 * SetDqtTables / SetDhtTables / SetPrecision (ImgDecode.cpp:505-624) plus where its
 * entropy-coded segment lives inside the batch bitstream buffer (the nStart argument of
 * DecodeScanImg, ImgDecode.cpp:2723).  Component arrays are indexed by component INDEX-1
 * (index 1=Y,2=Cb,3=Cr as the reference addresses them: ImgDecode.cpp:3059-3061,3113-3118). */
typedef struct {
    uint32_t dim_x, dim_y;                /* SOF X,Y                                        */
    uint32_t num_sof_comps, num_sos_comps;
    uint32_t precision;                   /* SOF P (8 or 12)                                */
    uint32_t restart_en, restart_interval;/* DRI                                            */
    uint32_t samp_h[4], samp_v[4];
    uint32_t dqt_sel[4];
    uint32_t dht_dc_sel[4], dht_ac_sel[4];
    uint32_t table_set;                   /* index into the sets given to upload_tables     */
    uint32_t file_pos;                    /* file offset of scan_offset (for the MCU map)   */
    uint64_t scan_offset;                 /* first ECS byte, offset into the batch bitstream */
    uint64_t scan_length;                 /* bytes readable from scan_offset (to file end)   */
} jsgpu_image_desc;

/* Where image i's outputs live (element offsets into the pools below) and its geometry as
 * derived by ImgDecode.cpp:2773-2872. */
typedef struct {
    uint32_t mcu_w, mcu_h, mcu_xmax, mcu_ymax, blk_xmax, blk_ymax;
    uint32_t img_x, img_y;                /* padded size = GetImageSize()                   */
    uint32_t num_segments;                /* restart intervals expected                     */
    uint32_t status;                      /* after decode: 0 ok, else JSGPU_ST_* bits       */
    uint64_t pix_off;                     /* int16 elements into pix_y/pix_cb/pix_cr pools   */
    uint64_t dib_off;                     /* bytes into the DIB pool                         */
    uint64_t blk_off;                     /* int16 elements into the block-DC pools          */
    uint64_t mcu_off;                     /* uint32 elements into the MCU file-map pool      */
} jsgpu_image_layout;

#define JSGPU_ST_BADCODE   1u   /* no Huffman code matched (ImgDecode.cpp:1257-1282)        */
#define JSGPU_ST_OVERRUN   2u   /* read past the end of a restart interval (:1096-1115)     */
#define JSGPU_ST_COEFOVF   4u   /* nNumCoeffs > 64 (:1776-1797)                             */
#define JSGPU_ST_MISSING   8u   /* fewer RSTn markers than the DRI interval implies (:3180) */
#define JSGPU_ST_LEFTOVER 16u   /* data left in an interval after its last MCU              */
#define JSGPU_ST_RSTSEQ   32u   /* an RSTn marker out of sequence (ImgDecode.cpp:1414-1424)   */
#define JSGPU_ST_EXACT 0x40000000u  /* the image was decoded again by the serial reference-semantics path
                                       (jsgpu_batch_errors has its error events; outputs are the reference's) */

typedef struct {
    int32_t idct_mode;      /* 0 = integer IDCT (the -DIDCT_FIXEDPT build, ImgDecode.cpp:2402-2423,
                               2512-2515; default), 1 = float IDCT (:2372-2392, 2517-2519)       */
    int32_t decode_ac;      /* m_bDecodeScanAc (ImgDecode.cpp:1723-1725,1818); default 1          */
    int32_t huff_kernel;    /* 0 = auto (3 for images with long restart intervals, else 2 or 1 by the
                               number of intervals), 1 = one warp per restart interval, 2 = one lane
                               per restart interval, 3 = self-synchronising passes for long intervals */
    int32_t idct_kernel;    /* 1 = simple reference kernels; 0 (auto), 2 and 3 all = fused tile
                               kernel where it applies, simple kernels elsewhere                   */
    int32_t want_histo;     /* accumulate m_anDhtHisto (ImgDecode.cpp:1190-1191); default 1      */
    int32_t want_mcu_map;   /* build m_pMcuFileMap (ImgDecode.cpp:3229); default 1               */
    int32_t device_markers; /* ignored: RSTn and the end of scan are always found on the GPU      */
    uint32_t scan_err_max;  /* CSnoopConfig::nErrMaxDecodeScan (SnoopConfig.cpp:89), taken literally: the capped error lines of
                               a scan are reported while fewer than this many were (0: none at all); jsgpu_init sets 20   */
} jsgpu_options;

/* Device pointers of the output pools of the current batch (owned by the context). */
typedef struct {
    int16_t*  pix_y;  int16_t* pix_cb; int16_t* pix_cr;  /* m_pPixValY/Cb/Cr  (ImgDecode.h:454-456) */
    uint8_t*  dib;                                       /* m_pDibTemp bits, BGRA bottom-up (:4786)  */
    int16_t*  blk_y;  int16_t* blk_cb; int16_t* blk_cr;  /* m_pBlkDcValY/Cb/Cr (ImgDecode.h:459-461) */
    uint32_t* mcu_map;                                   /* m_pMcuFileMap      (ImgDecode.h:444)     */
    uint32_t* dht_histo;                                 /* [n][2][4][17]      (ImgDecode.h:615)     */
    int32_t*  stats;                                     /* [n][16], see JSGPU_STAT_*               */
    int16_t*  coef;                                      /* intermediate coefficient rows            */
    uint8_t*  bitstream;                                 /* device copy of the batch bitstream       */
} jsgpu_pools;

/* stats[n][16] = the scalar results of CalcChannelPreviewFull (ImgDecode.cpp:4722-4730,4805-4819) */
#define JSGPU_STAT_SUMY_LO   0   /* low/high 32 bits of the 64-bit sum of nFinalY              */
#define JSGPU_STAT_SUMY_HI   1
#define JSGPU_STAT_AVGY      2   /* m_nAvgY                                                     */
#define JSGPU_STAT_BRIGHT_Y  3   /* m_nBrightY, Cb, Cr                                          */
#define JSGPU_STAT_BRIGHT_CB 4
#define JSGPU_STAT_BRIGHT_CR 5
#define JSGPU_STAT_BRIGHT_R  6   /* m_nBrightR, G, B                                            */
#define JSGPU_STAT_BRIGHT_G  7
#define JSGPU_STAT_BRIGHT_B  8
#define JSGPU_STAT_BRIGHT_MX 9   /* m_ptBrightMcu                                               */
#define JSGPU_STAT_BRIGHT_MY 10
#define JSGPU_STAT_NRST      11  /* m_nRestartRead                                              */
#define JSGPU_STAT_END_POS   12  /* m_anScanBuffPtr_pos[0] / m_nScanBuffPtr_align after the last MCU: the reference's      */
#define JSGPU_STAT_END_ALIGN 13
#define JSGPU_STAT_END_MARK  14  /* file position of the marker that ends the scan (BuffAddByte logs it, ImgDecode.cpp:1527-1543) */  /* "Next position in scan buffer" and compression-ratio lines (ImgDecode.cpp:3659-3726)  */
#define JSGPU_STAT_WORDS     16
#define JSGPU_HISTO_WORDS    136 /* dht_histo words per image: [2][4][17]                      */

/* Output selectors for jsgpu_batch_download */
#define JSGPU_OUT_PIX_Y   0
#define JSGPU_OUT_PIX_CB  1
#define JSGPU_OUT_PIX_CR  2
#define JSGPU_OUT_DIB     3
#define JSGPU_OUT_BLK_Y   4
#define JSGPU_OUT_BLK_CB  5
#define JSGPU_OUT_BLK_CR  6
#define JSGPU_OUT_MCU_MAP 7
#define JSGPU_OUT_HISTO   8
#define JSGPU_OUT_STATS   9

/* --- lifetime -------------------------------------------------------------------------- */
/* Replaces the CimgDecode constructor's device-independent setup (ImgDecode.cpp:142-234). */
int  jsgpu_init(int device, jsgpu_ctx** out);
void jsgpu_free(jsgpu_ctx* ctx);
const char* jsgpu_last_error(const jsgpu_ctx* ctx);
const char* jsgpu_strerror(int code);
int  jsgpu_version(void);
/* CUDA stream all work of this context is enqueued on (a cudaStream_t). */
void* jsgpu_stream(jsgpu_ctx* ctx);
int  jsgpu_sync(jsgpu_ctx* ctx);

/* --- tables ---------------------------------------------------------------------------- */
/* The IDCT look-up tables of PrecalcIdct (ImgDecode.cpp:2313-2351): li[yx*64+vu] =
 * m_anIdctLookup, lf[yx*64+vu] = m_afIdctLookup.  They depend on the HOST libm's cosf, so the
 * host computes them with the reference's expression and hands them over; the device never
 * recomputes them. */
int jsgpu_set_idct_tables(jsgpu_ctx* ctx, const int32_t* li, const float* lf);
int jsgpu_set_options(jsgpu_ctx* ctx, const jsgpu_options* opt);
int jsgpu_get_options(jsgpu_ctx* ctx, jsgpu_options* opt);
/* The error report's state when the next decode's scans start (jsgpu_init: 0, 0): warn_start = m_nWarnBadScanNum, the capped
 * lines already counted (the cap after ScanErrorsDisable, ImgDecode.cpp:1014-1018, which Reset() keeps, :127); disable =
 * m_bScanErrorsDisable, which drops the uncapped "Expected RST marker index" line (:1417).  Each scan's final count comes back
 * in jsgpu_scan_errors.warn_num. */
int jsgpu_set_scan_error_state(jsgpu_ctx* ctx, uint32_t warn_start, int disable);
/* Replaces SetDqtEntry / SetDhtEntry / SetDhtSize state (ImgDecode.cpp:424-453,748-847):
 * builds the device look-up tables for `nsets` table sets. */
int jsgpu_upload_tables(jsgpu_ctx* ctx, const jsgpu_tables* sets, uint32_t nsets);

/* Multi-GPU: images of a batch are partitioned across GPUs (one process or thread per GPU, no data-path collective); the
 * one exchange is this broadcast of the shared table blob (jsgpu_tables is POD) from rank `root` to every rank of an NCCL
 * communicator, over NVLink.  `nccl_comm` is the caller's ncclComm_t for ctx's device; on `root`, sets[0..nsets) is the
 * source, on the others the destination.  libnccl is resolved at run time (dlopen), so single-GPU users need no NCCL:
 * JSGPU_EUNSUP if it cannot be found.  Blocks until the blob is in host memory on this rank; every rank then calls
 * jsgpu_upload_tables().  (SURVEY.md §8b/e; the Python driver's torch.distributed broadcast does the same thing.) */
int jsgpu_bcast_tables(jsgpu_ctx* ctx, jsgpu_tables* sets, uint32_t nsets, void* nccl_comm, int root);

/* --- batch decode (replaces the body of CimgDecode::DecodeScanImg, ImgDecode.cpp:2723-3745,
 *     i.e. HOT LOOPS 1-4 of SURVEY.md §3.3, for n images at once) ------------------------- */
/* Geometry (ImgDecode.cpp:2773-2872), validation (:2755-2770,2821-2825,3047-3123) and device
 * allocation (:2892-2987) for n images whose scan bytes occupy `bitstream_bytes` bytes.
 * Images the reference would refuse get layout.status != 0 / JSGPU_EUNSUP semantics: they are
 * skipped, exactly as DecodeScanImg returns early. */
int jsgpu_batch_begin(jsgpu_ctx* ctx, const jsgpu_image_desc* imgs, uint32_t n, uint64_t bitstream_bytes);
int jsgpu_batch_layout(jsgpu_ctx* ctx, jsgpu_image_layout* out, uint32_t n);
int jsgpu_batch_pools(jsgpu_ctx* ctx, jsgpu_pools* out);
/* Copy the batch bitstream (host memory, pinned or pageable) to the device, asynchronously
 * on the context stream.  Replaces the per-byte CwindowBuf::Buf() fetch
 * (ImgDecode.cpp:1398-1399, WindowBuf.cpp:639-713). */
int jsgpu_batch_upload(jsgpu_ctx* ctx, const uint8_t* host_bitstream, uint64_t bytes);
/* Enqueue marker scan + Huffman + dequant/IDCT/upsample + colour conversion + statistics
 * for the whole batch on the context stream (asynchronous). */
int jsgpu_batch_decode(jsgpu_ctx* ctx);
/* After jsgpu_sync(): per-image status words and scalar results are in the layout/stats. */
int jsgpu_batch_download(jsgpu_ctx* ctx, int which, uint32_t image, void* host_dst, uint64_t bytes);
/* Device-side times (ms) of the last jsgpu_batch_decode, measured with CUDA events on the
 * context stream: [0] marker scan, [1] Huffman, [2] IDCT+colour, [3] stats/map finalise,
 * [4] total.  Forces a sync.  JSGPU_ESTATE unless the context's current batch was decoded on
 * it (not after a jsgpu_decode_batch_host that was cut into image ranges). */
int jsgpu_batch_stage_ms(jsgpu_ctx* ctx, float* ms5);
/* Device stopwatch on the context stream (CUDA events): start records an event, stop records a
 * second one, synchronises on it and returns the elapsed milliseconds. */
int jsgpu_timer_start(jsgpu_ctx* ctx);
int jsgpu_timer_stop(jsgpu_ctx* ctx, float* ms);
/* Number of kernels launched by the last jsgpu_batch_decode. */
int jsgpu_batch_launches(jsgpu_ctx* ctx);
/* Diagnostics of the self-synchronising Huffman passes of the last jsgpu_batch_decode (images with long restart
 * intervals — no DRI, or a DRI of an MCU row and more — whose single serial walk, ImgDecode.cpp:3164-3630, is cut into
 * 4096-bit slots): info[0] = images on that path, info[1] = slots reserved, info[2] = fix rounds enqueued (R),
 * info[3..3+R] = slots whose state changed in fix round 1..R+... (0 from the round in which everything had settled).
 * n = capacity of info in words (16 is enough).  Forces a sync. */
int jsgpu_batch_selfsync_info(jsgpu_ctx* ctx, uint32_t* info, uint32_t n);

/* What the reference logs for a damaged scan.  An image whose status word came out non-zero is decoded a second time by a
 * serial path that follows ReadScanVal / BuffAddByte / DecodeScanComp / DecodeScanImg literally (one-bit resynchronisation
 * ImgDecode.cpp:1166-1187, stray markers :1486-1561 and :1683-1706, lazy restarts :1644-1680, error cap :1100-1110); its
 * outputs replace the fast path's and its log events are kept for the caller.  code: see JSGPU_EV_*; a..e: the numbers the
 * reference prints in that line (file position, bit alignment, table, accumulator ...). */
#define JSGPU_EV_OVERREAD_BEFORE     1  /* "*** ERROR: Overread scan segment (before nCode)! @ Offset: %s"   a=pos b=align        */
#define JSGPU_EV_OVERREAD_AFTER_CODE 2  /* "*** ERROR: Overread scan segment (after nCode)! @ Offset: %s"                         */
#define JSGPU_EV_OVERREAD_AFTER_BITS 3  /* "*** ERROR: Overread scan segment (after bitstring)! @ Offset: %s"                     */
#define JSGPU_EV_NOCODE              4  /* "*** ERROR: Can't find huffman bitstring @ %s, table %u, value [0x%08x]" c=tbl d=buff  */
#define JSGPU_EV_CAP                 5  /* "    Only reported first %u instances of this message..."          a=cap               */
#define JSGPU_EV_RST_MISMATCH        6  /* "  ERROR: Expected RST marker index RST%u got RST%u @ 0x%08X.0"    a,b,c               */
#define JSGPU_EV_MARKER_NOTE         7  /* "  Scan Data encountered marker   0xFF%02X @ 0x%08X.0" (plain line) a=marker b=pos;
                                           followed by "  NOTE: Marker wasn't EOI (0xFFD9)" (error line) unless a == 0xD9       */
#define JSGPU_EV_BADMARK             8  /* "*** ERROR: Bad marker @ %s"                                                           */
#define JSGPU_EV_BADCODE             9  /* "*** ERROR: Bad huffman code @ %s"                                                     */
#define JSGPU_EV_NCOEF              10  /* "*** ERROR: @ %s, nNumCoeffs>64 [%u]"                             c=n                  */
#define JSGPU_EV_MCU                11  /* "*** ERROR: Bad scan data in MCU(%u,%u): %s @ Offset %s" + "           MCU located at
                                           pixel=(%u,%u)"  a=mcu x b=mcu y c=comp|h<<8|v<<16 d=pos e=align                        */
#define JSGPU_EV_RST_MISSING        12  /* "  Expect Restart interval elapsed @ %s" (plain) + "    ERROR: Restart marker not detected" */
#define JSGPU_MAX_EVENTS 256
typedef struct { uint32_t code, a, b, c, d, e, pad0, pad1; } jsgpu_scan_event;
typedef struct {
    uint32_t nerr_lines;      /* error lines (AddLineErr) the reference writes for this scan                               */
    uint32_t nevents;         /* events seen; the first JSGPU_MAX_EVENTS are in ev[]                                       */
    uint32_t scan_bad;        /* m_bScanBad at the end of the scan                                                        */
    uint32_t restart_read;    /* m_nRestartRead                                                                           */
    uint32_t done;
    uint32_t end_pos, end_align;  /* m_anScanBuffPtr_pos[0], m_nScanBuffPtr_align after the last MCU */
    uint32_t warn_num;        /* m_nWarnBadScanNum after the scan: scan_warn_start plus the capped lines counted              */
    jsgpu_scan_event ev[JSGPU_MAX_EVENTS];
} jsgpu_scan_errors;
/* Error events of image `image` of the last decode (JSGPU_ESTATE when it did not take the serial path: status without
 * JSGPU_ST_EXACT).  The counts are complete; ev[] holds the first JSGPU_MAX_EVENTS events.  Forces a sync. */
int jsgpu_batch_errors(jsgpu_ctx* ctx, uint32_t image, jsgpu_scan_errors* out);
/* Events first .. first+n-1 of all nevents of that image (n * 32 bytes); JSGPU_EINVAL past nevents.  Events past the first
 * JSGPU_MAX_EVENTS come from a second, events-only walk of the image over the resident scan, with the decode's cap, start
 * count and disable flag: it writes no output and gives the same events.  Forces a sync. */
int jsgpu_batch_error_events(jsgpu_ctx* ctx, uint32_t image, uint32_t first, uint32_t n, jsgpu_scan_event* out);

/* Checksums of the outputs of every image of the last jsgpu_batch_decode, computed on the device (forces a sync):
 * ck[i][0..2] m_pPixValY/Cb/Cr, [3] the DIB, [4..6] m_pBlkDcValY/Cb/Cr, [7] m_pMcuFileMap, [8] m_anDhtHisto, [9] the nine
 * scalars m_nAvgY, m_nBrightY/Cb/Cr, m_nBrightR/G/B, m_ptBrightMcu.x/.y, [10] the status word, [11] (img_x << 32) | img_y.
 * Entries of absent buffers (Cb/Cr of a one-component scan, skipped images) are 0.  Each checksum is
 *   sum over 32-bit little-endian words w_i of the buffer (16-bit buffers: two elements per word, an odd last element
 *   zero-extended) of  mix(w_i, i),  mix(w, i): x = w + (i+1)*0x9E3779B97F4A7C15; x ^= x >> 32; x *= 0xD6E8FEB86659FD93;
 *   x ^= x >> 29   (64-bit wrap-around arithmetic),
 * so a caller holding the reference's buffers (ImgDecode.h:444-461) can verify a whole batch without copying it back. */
#define JSGPU_CK_WORDS 12
int jsgpu_batch_checksums(jsgpu_ctx* ctx, uint64_t* ck, uint32_t n);

/* --- channel preview, colour statistics and histograms (SURVEY.md §8f N3/N4) -------------------------------------------
 * CimgDecode::CalcChannelPreviewFull (ImgDecode.cpp:4619-4821) beyond its default: the clipping/histogram colour
 * conversion ConvertYCCtoRGB/CapYccRange/CapRgbRange (:4229-4601) taken when CSnoopConfig::bHistoEn or bStatClipEn is set,
 * the channel selection ChannelExtract (:4832-4876) and the YCC level shift from a given MCU on (SetPreviewYccOffset,
 * :650-659).  With the defaults (all zero, mode 1) jsgpu_batch_decode's fused kernel has produced exactly this already. */
typedef struct {
    int32_t hist_en;        /* m_bHistEn  (ImgDecode.cpp:2740)                                                        */
    int32_t statclip_en;    /* m_bStatClipEn (:2741); either one selects ConvertYCCtoRGB instead of ...FastFloat (:4745) */
    int32_t mode;           /* m_nPreviewMode: 1 RGB, 2 YCC, 3 R, 4 G, 5 B, 6 Y, 7 Cb, 8 Cr (snoop.h:100-108); 0 = 1 */
    int32_t shift_y, shift_cb, shift_cr;          /* m_nPreviewShiftY/Cb/Cr                                            */
    uint32_t shift_mcu_x, shift_mcu_y;            /* m_nPreviewShiftMcuX/Y: applied to MCUs at or after this one (:4735) */
    uint32_t ycc_warn_budget;                     /* YCC_CLIP_REPORT_MAX - m_nWarnYccClipNum (ImgDecode.h:50): how many
                                                     "YCC Clipped" notes may still be issued (and counted, :4372-4378)  */
    uint32_t detail_en;                           /* m_bDetailVlc: also keep the RGB of MCU (detail_mcu_x, detail_mcu_y) BEFORE the    */
    uint32_t detail_mcu_x, detail_mcu_y;          /* channel selection, for the "Detailed IDCT Dump (RGB)" (ImgDecode.cpp:4757-4764)   */
    uint32_t pad;
} jsgpu_preview;
#define JSGPU_CC_HISTO_BINS  128    /* HISTO_BINS (ImgDecode.h:157)      */
#define JSGPU_Y_HISTO_BINS   2048   /* FULL_HISTO_BINS (ImgDecode.h:162) */
#define JSGPU_MAX_YCC_WARN   10     /* YCC_CLIP_REPORT_MAX               */
/* channel order of the range arrays: 0-2 pre-ranged Y,Cb,Cr (nPreclipY.. of PixelCcHisto, ImgDecode.h:236-280), 3-5 ranged
 * Y,Cb,Cr before the clip (nClipY..), 6-8 R,G,B before the clip (nPreclipR..), 9-11 R,G,B after it (nClipR..).
 * min/max start at 0 like the reference's memset (ImgDecode.cpp:3147); sums are 64-bit here, the reference's are `int`
 * (the caller truncates).  clip[]: nClipYUnder, YOver, CbUnder, CbOver, CrUnder, CrOver (counted only while notes are issued:
 * at most ycc_warn_budget in total), RUnder, ROver, GUnder, GOver, BUnder, BOver. */
typedef struct { uint32_t mcu_x, mcu_y; int32_t y, cb, cr; uint32_t kind; uint32_t px, py; } jsgpu_ycc_warn;   /* kind: index into clip[0..5]; px, py: the pixel */
typedef struct {
    uint32_t cc_histo[3][JSGPU_CC_HISTO_BINS];    /* m_anCcHisto_r/g/b                                                 */
    uint32_t y_histo[JSGPU_Y_HISTO_BINS];         /* m_anHistoYFull                                                    */
    int32_t  vmin[12], vmax[12];
    int64_t  vsum[12];
    uint64_t count;                               /* m_sHisto.nCount                                                   */
    uint32_t clip[12];
    uint32_t nwarn, pad;
    jsgpu_ycc_warn warn[JSGPU_MAX_YCC_WARN];      /* the notes, in the reference's (raster, Y/Cb/Cr) order             */
    uint32_t detail_rgb[32][32];                  /* [row][column] inside the detail MCU: R << 16 | G << 8 | B         */
} jsgpu_colour_stats;
/* Recompute the DIB (and stats[] SUMY/AVGY) of every image of the current batch from its pixel maps with `p`; the statistics
 * of this pass are kept for jsgpu_batch_colour_stats.  jsgpu_set_preview makes jsgpu_batch_decode do so itself whenever the
 * settings differ from the defaults. */
int jsgpu_set_preview(jsgpu_ctx* ctx, const jsgpu_preview* p);
int jsgpu_batch_preview(jsgpu_ctx* ctx, const jsgpu_preview* p);
int jsgpu_batch_colour_stats(jsgpu_ctx* ctx, uint32_t image, jsgpu_colour_stats* out);

/* --- "Detailed Decode" of chosen MCUs (CimgDecode::SetDetailVlc, ImgDecode.cpp:4898; DecodeScanCompPrint :1859-2090) ------
 * For `len` MCUs from (mcu_x, mcu_y) of image `image` the reference prints every Huffman symbol (ReportVlc :2152-2232) and each
 * block's coefficient matrix (ReportDctMatrix :2104-2131), whatever `len` is.  For an image whose status word is 0 one GPU thread
 * per MCU of the range decodes it from the MCU's recorded start (count pass, scan, emit pass); a damaged image takes the serial
 * reference-semantics walk (the one that re-decodes it), and so does every image when the environment variable
 * JSGPU_DETAIL_WALK=1 is set (read once per process) or the MCU file map is off (want_mcu_map = 0).  Both give the same events.
 * The context keeps the events and matrices of the last jsgpu_batch_decode (sized for them at each decode) until the next one;
 * jsgpu_batch_detail_info / _events / _matrices read them in full, jsgpu_batch_detail returns the first JSGPU_MAX_DETAIL_*.
 * In DC-only mode the printed MCUs are decoded in full (AC + IDCT), as DecodeScanCompPrint does. */
typedef struct { int32_t enable; uint32_t image, mcu_x, mcu_y, len; } jsgpu_detail;
#define JSGPU_DT_MCU    1   /* an MCU of the range starts: the blank separator line (ImgDecode.cpp:3249-3251)                     */
#define JSGPU_DT_BLOCK  2   /* "    Lum (Tbl #0), MCU=[x,y]": a = DQT table, b = MCU x, c = MCU y (:1873-1889)                     */
#define JSGPU_DT_VLC    3   /* ReportVlc: a = file position, b = bit alignment, c = ZRL, d = value, e = first coefficient |
                               last << 8 | bits of code and value << 16, f = 0 "", 1 "EOB", 2 "ERROR", 3 "EOB64"                  */
#define JSGPU_DT_MATRIX 4   /* ReportDctMatrix: a = index into matrix[]                                                           */
typedef struct { uint32_t kind, seq, a, b, c, d, e, f; } jsgpu_detail_event;   /* seq: error events (jsgpu_scan_errors.ev) logged before it */
#define JSGPU_MAX_DETAIL_EVENTS 8192
#define JSGPU_MAX_DETAIL_BLOCKS 512
typedef struct {
    uint32_t nevents, nblocks, pad0, pad1;       /* counted in full; the arrays keep the first JSGPU_MAX_DETAIL_* (all of
                                                    them: jsgpu_batch_detail_events / _matrices) */
    jsgpu_detail_event ev[JSGPU_MAX_DETAIL_EVENTS];
    int16_t matrix[JSGPU_MAX_DETAIL_BLOCKS][64]; /* m_anDctBlock: dequantised, natural order, [0] = the DC difference */
} jsgpu_detail_dump;
int jsgpu_set_detail(jsgpu_ctx* ctx, const jsgpu_detail* d);
int jsgpu_batch_detail(jsgpu_ctx* ctx, jsgpu_detail_dump* out);
/* info[0] = events, info[1] = blocks (matrices) of the last decode's detailed decode, in full; info[2] = the path that made them
 * (JSGPU_DETAIL_SERIAL / JSGPU_DETAIL_PARALLEL); info[3] = 0.  Forces a sync. */
#define JSGPU_DETAIL_SERIAL   0
#define JSGPU_DETAIL_PARALLEL 1
int jsgpu_batch_detail_info(jsgpu_ctx* ctx, uint32_t info[4]);
/* Events first .. first+n-1 (n * 32 bytes), matrices first .. first+n-1 (n * 64 int16, natural order, [0] = the DC difference)
 * of the last decode's detailed decode; JSGPU_EINVAL past info[0] / info[1].  A JSGPU_DT_MATRIX event's `a` indexes the
 * matrices.  Force a sync. */
int jsgpu_batch_detail_events(jsgpu_ctx* ctx, uint32_t first, uint32_t n, jsgpu_detail_event* out);
int jsgpu_batch_detail_matrices(jsgpu_ctx* ctx, uint32_t first, uint32_t n, int16_t* out);

/* --- Export-to-TIFF consumer (SURVEY.md §8f N4) ---------------------------------------------------------------------------
 * The three-samples-per-pixel, top-down array CJPEGsnoopDoc::OnToolsExporttiff (JPEGsnoopDoc.cpp:2061-2180) hands to
 * FileTiff::WriteFile, packed on the device from image `image` of the current batch and copied to host_out
 * (img_x * img_y * 3 bytes, 6 for RGB16).  YCC8 needs a three-component scan (the reference reads all three pixel maps). */
#define JSGPU_EXPORT_RGB8  0   /* the DIB's R,G,B                                    (JPEGsnoopDoc.cpp:2108-2124) */
#define JSGPU_EXPORT_RGB16 1   /* ... as 16-bit samples value << 8, big-endian       (:2125-2130)                 */
#define JSGPU_EXPORT_YCC8  2   /* pixel maps clipped to -1024..1023, (0x400 + v) >> 3 (:2133-2170)                 */
int jsgpu_batch_export(jsgpu_ctx* ctx, uint32_t image, int mode, void* host_out, uint64_t bytes);

/* One-call end-to-end form: host bitstream in, host outputs out (any pointer may be NULL to
 * skip that output).  Output buffers hold the images back to back in batch order using the
 * element offsets of jsgpu_batch_layout.  Small batches run H2D, decode and D2H on the context
 * stream, and the context keeps the decoded batch as jsgpu_batch_decode leaves it.  Large ones
 * (>= 16 images and >= 64 MB of bitstream, images laid out in increasing, 16-byte aligned scan
 * offsets) are cut into 8 image ranges, each with its own stream and device pools, so the
 * device-to-host copy of one range overlaps upload and decode of the next.  From the moment such a
 * batch is planned, this context holds its layout only, and after the decode the statuses:
 * jsgpu_batch_layout works; every other batch query (download, pools, stage_ms, checksums, errors,
 * export, preview ...) returns JSGPU_ESTATE, also when a range failed, until the next
 * jsgpu_batch_begin.  The data already is in `out`. */
typedef struct {
    int16_t* pix_y; int16_t* pix_cb; int16_t* pix_cr; uint8_t* dib;
    int16_t* blk_y; int16_t* blk_cb; int16_t* blk_cr; uint32_t* mcu_map;
    uint32_t* dht_histo; int32_t* stats;
} jsgpu_host_outputs;
int jsgpu_decode_batch_host(jsgpu_ctx* ctx, const jsgpu_image_desc* imgs, uint32_t n,
                            const uint8_t* host_bitstream, uint64_t bitstream_bytes,
                            const jsgpu_host_outputs* out);

/* --- byte-pattern search (Tools -> Search Executable for DQT, JPEGsnoopDoc.cpp:1233-1529) ---------------------------------
 * Replaces the Doc's loop "start = 0; while CwindowBuf::BufSearchX(start, pat, L, forward) finds p: report p; start = p + 1"
 * (WindowBuf.cpp:243-331) for `npat` patterns at once, in one streaming pass over the n bytes at `data` (host memory).
 * Pattern k is lens[k] bytes (8..256) at patterns + lens[0] + .. + lens[k-1].  It reports exactly what that loop reports:
 * every p where the pattern matches byte for byte, 1 <= p <= n - 2 lens[k] + 2 (the reference never reports offset 0 and
 * stops short of the last 2 L - 2 bytes), and p - 1 was not reported itself (a run of overlapping matches reports every
 * other one).  counts[k] receives pattern k's full count; pos receives at most `cap` positions, ascending per pattern,
 * pattern k's after pattern k-1's.  Files of 2^32 bytes or more are refused (JSGPU_EINVAL): the reference's offsets are 32-bit.
 * The file is streamed in chunks (64 MiB; the environment variable JSGPU_SEARCH_CHUNK_BYTES, read at every call, changes
 * that) through pinned double buffers on the search's own streams; the batch of the context is left untouched.  Synchronous. */
#define JSGPU_SEARCH_MAX_PATTERNS 32
#define JSGPU_SEARCH_MIN_LEN      8
#define JSGPU_SEARCH_MAX_LEN      256
int jsgpu_search_bytes(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, const uint8_t* patterns, const uint32_t* lens, uint32_t npat,
                       uint64_t* counts, uint32_t* pos, uint64_t cap);

/* --- value search (Tools -> Img Search Fwd / Rev, JPEGsnoopDoc.cpp:829-932) -----------------------------------------------
 * Returns what CwindowBuf::BufSearch(start, value, len, forward, found_pos) (WindowBuf.cpp:149-212) returns over the n bytes at
 * `data` with `noverlays` overlays applied (overlay k replaces overlays[k].len bytes from file offset overlays[k].start, also past
 * the end of the file; the last one listed wins, as the reference's Buf() does, WindowBuf.cpp:655-681).  Each position p compares the big-endian value of the len (1..4) bytes at p, bytes past
 * the end of the file reading as 0, with `value`:
 *   forward  tests start + 1, start + 2, ... and stops after the first p with p + len - 1 >= n (tested too; when
 *            start + len >= n that is start + 1 alone);
 *   reverse  tests start - 1 down to 0; from start 0 it tests 0 once.
 * *found = 1 and *found_pos = the first match in that order, or *found = 0 and *found_pos = the last position tested.
 * The file is streamed in chunks (JSGPU_SEARCH_CHUNK_BYTES, as jsgpu_search_bytes) in search order through pinned staging
 * buffers, the overlays patched in on the host; the search stops at the first chunk that holds a match, and no chunk past it
 * reaches the device.  Files of 2^32 bytes or more and starts of 2^32 - 1 or more are refused (JSGPU_EINVAL): the
 * reference's positions are 32-bit.  The batch of the context is left untouched.  Synchronous. */
typedef struct { uint64_t start; uint64_t len; const uint8_t* data; } jsgpu_overlay;
int jsgpu_find_value(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, uint64_t start, uint32_t value, uint32_t len, int forward,
                     const jsgpu_overlay* overlays, uint32_t noverlays, int* found, uint64_t* found_pos);

/* --- every match of a value (finding every JPEG in a file) ----------------------------------------------------------------
 * Every p in [0, n - len] whose big-endian len (1..4) bytes equal `value`, in ascending order; overlapping matches are all
 * reported (FF D8 FF D8 FF holds FF D8 FF twice).  For FF D8 FF the positions p >= 1 are exactly the ones a chain of
 * CwindowBuf::BufSearch(prev, 0xFFD8FF, 3, forward) calls from 0 visits, the chain JPEGsnoop's extract-all runs.
 * *count receives the complete count; pos receives at most `cap` positions.  The file is streamed in chunks
 * (JSGPU_SEARCH_CHUNK_BYTES, as jsgpu_search_bytes) through the search's pinned staging buffers, each chunk uploaded once and
 * searched, counted and listed on the device, the running count kept there.  Files of 2^32 bytes or more are refused
 * (JSGPU_EINVAL).  The batch of the context is left untouched.  Synchronous. */
int jsgpu_find_all(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, uint32_t value, uint32_t len, uint64_t* count, uint32_t* pos,
                   uint64_t cap);

/* --- the markers of Extract embedded JPEG / Extract All (JPEGsnoopCore.cpp:913-1088) ---------------------------------------
 * One streaming pass that lists, in ascending order:
 *   soi_pos   every p in [0, n - 3] whose bytes are FF D8 FF: the list jsgpu_find_all(value 0xFFD8FF, len 3) returns, whose
 *             positions from 1 on are the frame starts Extract All's chain of BufSearch calls visits;
 *   term_pos  every PASS-1 scan terminator (CjfifDecode::DecodeMarker, JfifDecode.cpp:5194-5265): p in [0, n - 2] with
 *             byte p == FF and byte p + 1 neither 00 nor D0..D7.  The byte after a stuffed or RST FF is never FF, so the end
 *             of a scan starting at s is the first terminator >= s, whatever the scan holds; with none, the scan runs out of
 *             file ("Ran out of buffer before EOI").  An FF in the last byte ends nothing: Buf() reads the byte past the end
 *             of the file as 0.
 * Both are read with `noverlays` overlays applied as jsgpu_find_value applies them (bytes an overlay puts past the end of the
 * file are not searched).  *nsoi / *nterm receive complete counts; soi_pos / term_pos receive at most soi_cap / term_cap
 * positions.  Each chunk (JSGPU_SEARCH_CHUNK_BYTES) is uploaded once with its next two bytes, so a terminator or an SOI on a
 * chunk's last positions is decided there.  Files of 2^32 bytes or more are refused (JSGPU_EINVAL).  The batch of the
 * context is left untouched.  Synchronous. */
int jsgpu_find_markers(jsgpu_ctx* ctx, const uint8_t* data, uint64_t n, const jsgpu_overlay* overlays, uint32_t noverlays,
                       uint32_t* soi_pos, uint64_t soi_cap, uint64_t* nsoi, uint32_t* term_pos, uint64_t term_cap, uint64_t* nterm);

/* Pinned host memory helpers (for callers that want true async copies). */
void* jsgpu_host_alloc(uint64_t bytes);
void  jsgpu_host_free(void* p);
/* Raw copy rate of this box between pinned host memory and the context's device: `bytes` are copied `reps` times with
 * cudaMemcpyAsync on the context stream and timed with CUDA events; direction 0 = host->device, 1 = device->host.
 * *gbs receives the best repetition in GB/s.  This is the ceiling jsgpu_decode_batch_host can reach (its time is the
 * device->host copy of the reference's outputs); bench.py reports its end-to-end figure as a fraction of it. */
int jsgpu_host_copy_rate(jsgpu_ctx* ctx, int direction, uint64_t bytes, int reps, float* gbs);

#ifdef __cplusplus
}
#endif
#endif /* JSGPU_H */
