/* jsimg.h — flat C shim over the host class CimgDecode (jpegsnoop_b200/csrc/host/ImgDecode.h)
 * for FFI callers (Python ctypes in tests/bench, or any non-C++ host).  One function per public
 * method of the reference class that the scan-decode path uses; names are the reference's method
 * names with a jsimg_ prefix (reference: source/ImgDecode.h:286-356,384-385,407-408,416).
 * Also exports the minimal JFIF marker walk that issues CjfifDecode's setter sequence
 * (reference: source/JfifDecode.cpp:3535-3600, 4576-4651, 5001-5026, 5150-5164, 5291-5330).
 * All functions are exported from libjsgpu.so. */
#ifndef JSIMG_H
#define JSIMG_H
#include <stdint.h>
#include "jsgpu.h"
#ifdef __cplusplus
extern "C" {
#endif

typedef struct jsimg jsimg;   /* {CDocLog, CwindowBuf, CSnoopConfig, CimgDecode} as wired by CJPEGsnoopCore.cpp:38-53 */

jsimg* jsimg_create(void);
void   jsimg_destroy(jsimg*);
/* config (CSnoopConfig fields read at ImgDecode.cpp:2730-2741 + device knobs); device_markers is ignored
 * (jsgpu_options.device_markers) */
void   jsimg_config(jsimg*, int decode_ac, int idct_fixedpt, int cuda_device, int huff_kernel, int idct_kernel, int device_markers);
/* CSnoopConfig::bHistoEn / bStatClipEn / bDumpHistoY (SnoopConfig.cpp:76-82), read at ImgDecode.cpp:2730-2741 */
void   jsimg_config_histo(jsimg*, int histo_en, int statclip_en, int dump_histo_y);
/* CSnoopConfig::nErrMaxDecodeScan (SnoopConfig.cpp:89, default 20), read at ImgDecode.cpp:2732: each kind of capped scan
 * error line is reported while fewer than n were; 0 reports none of them */
void   jsimg_config_scan_err_max(jsimg*, unsigned n);
/* CimgDecode::ScanErrorsDisable / ScanErrorsEnable (ImgDecode.cpp:1014-1030): disabling counts the cap as used up (the count
 * survives Reset(), so a cap raised later lets only the difference through) and drops the "Expected RST marker index" lines;
 * enabling sets the count back to 0.  ResetState() (every marker walk) clears the switch. */
void   jsimg_ScanErrorsDisable(jsimg*);
void   jsimg_ScanErrorsEnable(jsimg*);
/* byte source: CwindowBuf::BufFileSet equivalent on a memory buffer (caller keeps it alive) */
void   jsimg_set_file(jsimg*, const uint8_t* data, uint64_t n);
int    jsimg_overlay_install(jsimg*, uint32_t start, const uint8_t* data, uint32_t n);
void   jsimg_overlay_remove_all(jsimg*);                       /* CwindowBuf::OverlayRemoveAll, WindowBuf.cpp:571 */

void   jsimg_Reset(jsimg*);
void   jsimg_ResetState(jsimg*);
int    jsimg_SetDqtEntry(jsimg*, unsigned nTblDestId, unsigned nCoeffInd, unsigned nCoeffIndZz, unsigned nCoeffVal);
int    jsimg_SetDqtTables(jsimg*, unsigned nCompInd, unsigned nTbl);
unsigned jsimg_GetDqtEntry(jsimg*, unsigned nTblDestId, unsigned nCoeffInd);
int    jsimg_SetDhtTables(jsimg*, unsigned nCompInd, unsigned nTblDc, unsigned nTblAc);
int    jsimg_SetDhtEntry(jsimg*, unsigned nDestId, unsigned nClass, unsigned nInd, unsigned nLen, unsigned nBits, unsigned nMask, unsigned nCode);
int    jsimg_SetDhtSize(jsimg*, unsigned nDestId, unsigned nClass, unsigned nSize);
void   jsimg_SetPrecision(jsimg*, unsigned nPrecision);
void   jsimg_SetSofSampFactors(jsimg*, unsigned nCompInd, unsigned nSampFactH, unsigned nSampFactV);
void   jsimg_SetImageDetails(jsimg*, unsigned nDimX, unsigned nDimY, unsigned nCompsSOF, unsigned nCompsSOS, int bRstEn, unsigned nRstInterval);
void   jsimg_DecodeScanImg(jsimg*, unsigned nStart, int bDisplay, int bQuiet);
int    jsimg_IsPreviewReady(jsimg*);

void   jsimg_GetImageSize(jsimg*, unsigned* nX, unsigned* nY);
void   jsimg_GetPixMapPtrs(jsimg*, const int16_t** pMapY, const int16_t** pMapCb, const int16_t** pMapCr);
const uint8_t*  jsimg_GetBitmapPtr(jsimg*);
void   jsimg_LookupFilePosMcu(jsimg*, unsigned nMcuX, unsigned nMcuY, unsigned* nByte, unsigned* nBit);
void   jsimg_LookupFilePosPix(jsimg*, unsigned nPixX, unsigned nPixY, unsigned* nByte, unsigned* nBit);
void   jsimg_LookupBlkYCC(jsimg*, unsigned nBlkX, unsigned nBlkY, int* nY, int* nCb, int* nCr);
const uint32_t* jsimg_GetMcuFileMap(jsimg*);
const int16_t*  jsimg_GetBlkDcMap(jsimg*, unsigned nChan);
void   jsimg_GetDhtHisto(jsimg*, uint32_t* out /*[2][4][17]*/);
void   jsimg_GetGeometry(jsimg*, unsigned* out8);
void   jsimg_GetStats(jsimg*, int32_t* out12);   /* avgY, avgValid, brightY,Cb,Cr,R,G,B, mcuX, mcuY, nRestartRead, scanBad */
void   jsimg_GetIdctTables(jsimg*, float* lf /*[64*64]*/, int32_t* li /*[64*64]*/);
void   jsimg_GetStageMs(jsimg*, float* ms5);
unsigned jsimg_GetScanStatus(jsimg*);
/* channel preview and colour statistics (ImgDecode.h:304-312; ImgDecode.cpp:631-677, 3764-4012) */
void   jsimg_SetPreviewMode(jsimg*, unsigned nMode);
unsigned jsimg_GetPreviewMode(jsimg*);
void   jsimg_SetPreviewYccOffset(jsimg*, unsigned nMcuX, unsigned nMcuY, int nY, int nCb, int nCr);
void   jsimg_GetPreviewYccOffset(jsimg*, unsigned* nMcuX, unsigned* nMcuY, int* nY, int* nCb, int* nCr);
void   jsimg_GetStatClip(jsimg*, uint32_t* out12);                 /* m_sStatClip: Y/Cb/Cr/R/G/B x under, over     */
void   jsimg_GetHistoRanges(jsimg*, int32_t* out36, uint32_t* nCount);   /* m_sHisto in PixelCcHisto's member order */
void   jsimg_GetCcHisto(jsimg*, unsigned nChan, uint32_t* out128); /* m_anCcHisto_r/g/b                            */
void   jsimg_GetHistoYFull(jsimg*, uint32_t* out2048);             /* m_anHistoYFull                               */
const uint8_t* jsimg_GetHistoDib(jsimg*, int which /*0 RGB (128x90), 1 Y (512x30)*/, int* ready);   /* m_pDibHistRgb / m_pDibHistY */

/* "Detailed Decode" of nLen MCUs from (nX,nY): CimgDecode::SetDetailVlc / GetDetailVlc (ImgDecode.cpp:4880-4904) */
void   jsimg_SetDetailVlc(jsimg*, int bDetail, unsigned nX, unsigned nY, unsigned nLen);
void   jsimg_GetDetailVlc(jsimg*, unsigned* bDetail, unsigned* nX, unsigned* nY, unsigned* nLen);
/* Export-to-TIFF (CJPEGsnoopDoc::OnToolsExporttiff + FileTiff::WriteFile): mode 0 RGB8, 1 RGB16, 2 YCC8; 1 on success */
int    jsimg_ExportTiff(jsimg*, const char* path, unsigned mode);
/* FileTiff::WriteFile on a caller-made sample array (no device involved); 1 on success */
int    jsimg_tiff_write(const char* path, int ycc, int b16, const void* data, unsigned w, unsigned h);

/* Tools -> Search Executable for DQT (CJPEGsnoopDoc::OnToolsSearchexecutablefordqt, JPEGsnoopDoc.cpp:1233-1529) over the n bytes
 * at `data` (exe_path names them in the report).  With `analysed` set, the handle's decoder stands for the analysed JPEG
 * (analysed_path): table 0 as GetDqtEntry(0, .) holds it is searched next to the JPEG standard's.  The report goes to the log,
 * line for line and kind for kind as the reference writes it; every search runs on the GPU (jsgpu_search_bytes) in one pass.
 * Returns 0, or a negative JSGPU_E* code after one error line and no report (no CUDA device; files of 2^32 bytes or more). */
int    jsimg_search_dqt(jsimg*, const uint8_t* data, uint64_t n, const char* exe_path, int analysed, const char* analysed_path);

/* Img Search Fwd / Rev and the offset modes (JPEGsnoopDoc.cpp:829-932; JPEGsnoopCore.cpp:700-756).  Positions are absolute
 * file offsets throughout: a decode at `pos` walks the markers from the SOI at pos, and its scan start, MCU file map, error
 * lines and Detailed Decode report offsets in the whole file.
 * jsimg_buf_search: CwindowBuf::BufSearch over the installed file and overlays, on the GPU (jsgpu_find_value); returns 1 found,
 *   0 not found (*found_pos as the reference leaves it either way) or a negative JSGPU_E* code. */
int    jsimg_buf_search(jsimg*, uint64_t start, uint32_t value, uint32_t len, int fwd, uint64_t* found_pos);
/* ProcessFile with nPosStart = pos: the marker walk from the SOI at pos, then DecodeScanImg.  Returns the absolute scan start
 * or a negative code, as jsimg_decode_jpeg (which is this at pos 0). */
int    jsimg_decode_jpeg_at(jsimg*, const uint8_t* data, uint64_t n, uint64_t pos, int quiet);
/* Tools -> Img Search Fwd (fwd = 1) / Rev (fwd = 0) from `start` over the installed file, as the Doc's handlers do it: search
 * for FF D8 FF; forward, a match becomes the new start and is reprocessed, otherwise nothing changes; reverse (only when
 * start > 0), a match is reprocessed, otherwise the start becomes 0 and the file is reprocessed from there.  *found: the
 * search's answer, *pos: the new start, *decoded: whether a decode at *pos ran.  Returns that decode's result (as
 * jsimg_decode_jpeg), 0 when nothing was decoded, or a negative JSGPU_E* code from the search (with *decoded = 0). */
int    jsimg_img_search(jsimg*, uint64_t start, int fwd, int quiet, int* found, uint64_t* pos, int* decoded);
/* DoAnalyzeOffset's modes (teOffsetMode, snoop.h:166): decode at 0; at 0 unless the walk there reaches no frame header
 * (CjfifDecode::GetDecodeStatus), then at the first FF D8 FF after 0 if there is one; at the first FF D8 FF after 0 if there is
 * one, else at 0; at `pos`.  *pos_used receives the offset decoded at.  Returns as jsimg_decode_jpeg, or a negative JSGPU_E*
 * code when a needed search failed (EINVAL for an unknown mode). */
#define JSIMG_OFFSET_START 0
#define JSIMG_OFFSET_SRCH1 1
#define JSIMG_OFFSET_SRCH2 2
#define JSIMG_OFFSET_POS   3
int    jsimg_decode_offset_mode(jsimg*, const uint8_t* data, uint64_t n, int mode, uint64_t pos, int quiet, uint64_t* pos_used);

/* Tools -> Extract embedded JPEG and its Extract All mode (JPEGsnoopCore.cpp:913-1088; CjfifDecode::ExportJpegPrepare /
 * ExportJpegDo, JfifDecode.cpp:7544-7797) over the installed file and overlays.  One GPU pass (jsgpu_find_markers) lists the
 * FF D8 FF candidates and the PASS-1 scan terminators; the host then walks each frame's markers from its start to the EOI as
 * ProcessFile does (every scan skipped to its first terminator), and copies the frame out of the caller's buffer.  Nothing is
 * decoded.  The bytes are the reference's, quirks included:
 *   - [start, first SOS) and [first SOS, end) are each copied by a loop that stops one byte short of a part of
 *     k * 131072 + 1 bytes (for the second part that byte is the EOI's D9), and writes nothing of a 1-byte part;
 *   - FORCE_SOI writes FF D8 only when the walk met no SOI; FORCE_EOI appends FF D9 always, after a real EOI too;
 *   - with no EOI, FORCE_EOI or IGNORE_EOI end the frame at the end of the file (otherwise the export is refused);
 *   - DHT_AVI inserts the 0x1A4-byte Annex K DHT segment before the first SOS, whatever the frame holds;
 *   - OVERLAY copies the bytes through the overlays; the walk always reads through them.
 * The log receives the reference's lines: the "*** Exporting JPEG ***" header, "Exporting from / to", the Prepare errors and
 * warnings, "Forcing SOI/EOI Marker", "Inserting standard AVI DHT huffman table", "Export done", "Can't overwrite source
 * file" when out_path equals src_name (the names are compared, as the reference does).  Files of 2^32 bytes or more are
 * refused (JSGPU_EINVAL, one error line).
 * jsimg_export_jpeg: the frame at `pos` (which need not hold an SOI) into out_path; 1 written, 0 refused, or a negative
 *   JSGPU_E* code from the search.
 * jsimg_extract_all: frames from offset 0, then from each FF D8 FF after the previous start (thumbnails nested in an APP1
 *   included), written to root.000001.jpg, root.000002.jpg, ... where root is out_name up to its last '.'.  A frame the
 *   Prepare step refuses takes no number.  offsets / numbers receive, for the first `cap` frames analysed, the frame's offset
 *   and its file's number (0: not written).  Returns the number of frames analysed, JSGPU_EINVAL after "ERROR: Invalid
 *   filename" when out_name has no '.', or a negative JSGPU_E* code from the search.  The search runs on `ctx` when given
 *   (a batch resident there is left untouched), else on the handle's own search context. */
#define JSIMG_EXPORT_OVERLAY    1u
#define JSIMG_EXPORT_FORCE_SOI  2u
#define JSIMG_EXPORT_FORCE_EOI  4u
#define JSIMG_EXPORT_IGNORE_EOI 8u
#define JSIMG_EXPORT_DHT_AVI    16u
int     jsimg_export_jpeg(jsimg*, uint64_t pos, const char* src_name, const char* out_path, unsigned flags);
int64_t jsimg_extract_all(jsimg*, jsgpu_ctx* ctx, const char* src_name, const char* out_name, unsigned flags, uint64_t* offsets,
                          uint32_t* numbers, uint64_t cap);
/* log access (error convention: failures are log lines, ImgDecode.cpp:2755-2758 etc.) */
int    jsimg_log_count(jsimg*, int kind /*0 line,1 hdr,2 warn,3 err,4 good,-1 all*/);
const char* jsimg_log_line(jsimg*, int kind, int index);
void   jsimg_log_clear(jsimg*);

/* Marker walk: issues the setter sequence for the first frame/scan of a JPEG, returns the file
 * offset of the first entropy-coded byte (> 0) or a negative code.  jsimg_decode_jpeg then calls
 * DecodeScanImg(start, true, quiet) exactly as JfifDecode.cpp:5299 does. */
int    jsimg_walk_jpeg(jsimg*, const uint8_t* data, uint64_t n);
int    jsimg_decode_jpeg(jsimg*, const uint8_t* data, uint64_t n, int quiet);
/* Same walk, but only export the C-ABI table set + image descriptor (for batch decoding); _at walks the JPEG whose SOI is at
 * `pos`, and the scan start it returns and desc->file_pos are absolute file offsets. */
int    jsimg_parse_jpeg(const uint8_t* data, uint64_t n, jsgpu_tables* tables, jsgpu_image_desc* desc);
int    jsimg_parse_jpeg_at(const uint8_t* data, uint64_t n, uint64_t pos, jsgpu_tables* tables, jsgpu_image_desc* desc);

#ifdef __cplusplus
}
#endif
#endif
