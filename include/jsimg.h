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

/* log access (error convention: failures are log lines, ImgDecode.cpp:2755-2758 etc.) */
int    jsimg_log_count(jsimg*, int kind /*0 line,1 hdr,2 warn,3 err,4 good,-1 all*/);
const char* jsimg_log_line(jsimg*, int kind, int index);
void   jsimg_log_clear(jsimg*);

/* Marker walk: issues the setter sequence for the first frame/scan of a JPEG, returns the file
 * offset of the first entropy-coded byte (> 0) or a negative code.  jsimg_decode_jpeg then calls
 * DecodeScanImg(start, true, quiet) exactly as JfifDecode.cpp:5299 does. */
int    jsimg_walk_jpeg(jsimg*, const uint8_t* data, uint64_t n);
int    jsimg_decode_jpeg(jsimg*, const uint8_t* data, uint64_t n, int quiet);
/* Same walk, but only export the C-ABI table set + image descriptor (for batch decoding). */
int    jsimg_parse_jpeg(const uint8_t* data, uint64_t n, jsgpu_tables* tables, jsgpu_image_desc* desc);

#ifdef __cplusplus
}
#endif
#endif
