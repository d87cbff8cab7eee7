// jsimg_cabi.cpp — include/jsimg.h: flat C shim over CimgDecode for FFI callers.
#include "../../../include/jsimg.h"
#include "ImgDecode.h"
#include "TiffExport.h"
#include "JfifWalk.h"
#include <cstring>

struct jsimg {
    CDocLog log; CwindowBuf wbuf; CSnoopConfig cfg; CimgDecode* dec;
    jsimg() : dec(new CimgDecode(&log, &wbuf, &cfg)) {}
    ~jsimg() { delete dec; }
};

extern "C" {
jsimg* jsimg_create(void) { return new jsimg(); }
void jsimg_destroy(jsimg* h) { delete h; }
void jsimg_config(jsimg* h, int ac, int fixed, int dev, int hk, int ik, int)
{ h->cfg.bDecodeScanImgAc = ac != 0; h->cfg.bIdctFixedPt = fixed != 0; h->cfg.nCudaDevice = dev; h->cfg.nHuffKernel = hk; h->cfg.nIdctKernel = ik; }
void jsimg_config_histo(jsimg* h, int he, int sc, int dy) { h->cfg.bHistoEn = he != 0; h->cfg.bStatClipEn = sc != 0; h->cfg.bDumpHistoY = dy != 0; }
void jsimg_SetPreviewMode(jsimg* h, unsigned m) { h->dec->SetPreviewMode(m); }
unsigned jsimg_GetPreviewMode(jsimg* h) { return h->dec->GetPreviewMode(); }
void jsimg_SetPreviewYccOffset(jsimg* h, unsigned mx, unsigned my, int y, int cb, int cr) { h->dec->SetPreviewYccOffset(mx, my, y, cb, cr); }
void jsimg_GetPreviewYccOffset(jsimg* h, unsigned* mx, unsigned* my, int* y, int* cb, int* cr) { h->dec->GetPreviewYccOffset(*mx, *my, *y, *cb, *cr); }
void jsimg_GetStatClip(jsimg* h, uint32_t* o) { memcpy(o, h->dec->GetStatClip(), 12 * sizeof(uint32_t)); }
void jsimg_GetHistoRanges(jsimg* h, int32_t* o, uint32_t* n) { int t[36]; unsigned c = 0; h->dec->GetHistoRanges(t, c); for (int i = 0; i < 36; i++) o[i] = t[i]; *n = c; }
void jsimg_GetCcHisto(jsimg* h, unsigned c, uint32_t* o) { memcpy(o, h->dec->GetCcHisto(c), JSGPU_CC_HISTO_BINS * sizeof(uint32_t)); }
void jsimg_GetHistoYFull(jsimg* h, uint32_t* o) { memcpy(o, h->dec->GetHistoYFull(), JSGPU_Y_HISTO_BINS * sizeof(uint32_t)); }
const uint8_t* jsimg_GetHistoDib(jsimg* h, int which, int* ready)
{
    if (ready) *ready = which ? h->dec->m_bDibHistYReady : h->dec->m_bDibHistRgbReady;
    return (const uint8_t*)(which ? h->dec->m_pDibHistY.GetDIBBitArray() : h->dec->m_pDibHistRgb.GetDIBBitArray());
}
int  jsimg_ExportTiff(jsimg* h, const char* path, unsigned mode) { return h->dec->ExportTiff(path, mode) ? 1 : 0; }
int  jsimg_tiff_write(const char* path, int ycc, int b16, const void* data, unsigned w, unsigned h) { FileTiff t; return t.WriteFile(path ? path : "", ycc != 0, b16 != 0, data, w, h) ? 1 : 0; }
void jsimg_SetDetailVlc(jsimg* h, int d, unsigned x, unsigned y, unsigned n) { h->dec->SetDetailVlc(d != 0, x, y, n); }
void jsimg_GetDetailVlc(jsimg* h, unsigned* d, unsigned* x, unsigned* y, unsigned* n) { bool b; h->dec->GetDetailVlc(b, *x, *y, *n); *d = b ? 1u : 0u; }
void jsimg_set_file(jsimg* h, const uint8_t* d, uint64_t n) { h->wbuf.BufSet(d, (size_t)n); }
int  jsimg_overlay_install(jsimg* h, uint32_t start, const uint8_t* d, uint32_t n) { return h->wbuf.OverlayInstall(start, d, n) ? 1 : 0; }
void jsimg_overlay_remove_all(jsimg* h) { h->wbuf.OverlayRemoveAll(); }
void jsimg_Reset(jsimg* h) { h->dec->Reset(); }
void jsimg_ResetState(jsimg* h) { h->dec->ResetState(); }
int  jsimg_SetDqtEntry(jsimg* h, unsigned t, unsigned i, unsigned z, unsigned v) { return h->dec->SetDqtEntry(t, i, z, (unsigned short)v); }
int  jsimg_SetDqtTables(jsimg* h, unsigned c, unsigned t) { return h->dec->SetDqtTables(c, t); }
unsigned jsimg_GetDqtEntry(jsimg* h, unsigned t, unsigned i) { return h->dec->GetDqtEntry(t, i); }
int  jsimg_SetDhtTables(jsimg* h, unsigned c, unsigned dc, unsigned ac) { return h->dec->SetDhtTables(c, dc, ac); }
int  jsimg_SetDhtEntry(jsimg* h, unsigned id, unsigned cls, unsigned ind, unsigned len, unsigned bits, unsigned mask, unsigned code) { return h->dec->SetDhtEntry(id, cls, ind, len, bits, mask, code); }
int  jsimg_SetDhtSize(jsimg* h, unsigned id, unsigned cls, unsigned n) { return h->dec->SetDhtSize(id, cls, n); }
void jsimg_SetPrecision(jsimg* h, unsigned p) { h->dec->SetPrecision(p); }
void jsimg_SetSofSampFactors(jsimg* h, unsigned c, unsigned hh, unsigned v) { h->dec->SetSofSampFactors(c, hh, v); }
void jsimg_SetImageDetails(jsimg* h, unsigned x, unsigned y, unsigned nf, unsigned ns, int rst, unsigned ri) { h->dec->SetImageDetails(x, y, nf, ns, rst != 0, ri); }
void jsimg_DecodeScanImg(jsimg* h, unsigned s, int disp, int quiet) { h->dec->DecodeScanImg(s, disp != 0, quiet != 0); }
int  jsimg_IsPreviewReady(jsimg* h) { return h->dec->IsPreviewReady(); }
void jsimg_GetImageSize(jsimg* h, unsigned* x, unsigned* y) { h->dec->GetImageSize(*x, *y); }
void jsimg_GetPixMapPtrs(jsimg* h, const int16_t** y, const int16_t** cb, const int16_t** cr) { short *a, *b, *c; h->dec->GetPixMapPtrs(a, b, c); *y = a; *cb = b; *cr = c; }
const uint8_t* jsimg_GetBitmapPtr(jsimg* h) { unsigned char* p; h->dec->GetBitmapPtr(p); return p; }
void jsimg_LookupFilePosMcu(jsimg* h, unsigned mx, unsigned my, unsigned* by, unsigned* bi) { h->dec->LookupFilePosMcu(mx, my, *by, *bi); }
void jsimg_LookupFilePosPix(jsimg* h, unsigned px, unsigned py, unsigned* by, unsigned* bi) { h->dec->LookupFilePosPix(px, py, *by, *bi); }
void jsimg_LookupBlkYCC(jsimg* h, unsigned bx, unsigned by, int* y, int* cb, int* cr) { h->dec->LookupBlkYCC(bx, by, *y, *cb, *cr); }
const uint32_t* jsimg_GetMcuFileMap(jsimg* h) { return h->dec->GetMcuFileMap(); }
const int16_t* jsimg_GetBlkDcMap(jsimg* h, unsigned ch) { return h->dec->GetBlkDcMap(ch); }
void jsimg_GetDhtHisto(jsimg* h, uint32_t* out) { memcpy(out, h->dec->GetDhtHisto(), 2 * 4 * 17 * sizeof(uint32_t)); }
void jsimg_GetGeometry(jsimg* h, unsigned* out8) { h->dec->GetGeometry(out8); }
void jsimg_GetStats(jsimg* h, int32_t* o)
{
    long avg = 0; bool av = h->dec->GetAvgY(avg);
    int y, cb, cr; unsigned r, g, b, mx, my; h->dec->GetBrightest(y, cb, cr, r, g, b, mx, my);
    o[0] = (int32_t)avg; o[1] = av; o[2] = y; o[3] = cb; o[4] = cr; o[5] = (int32_t)r; o[6] = (int32_t)g; o[7] = (int32_t)b;
    o[8] = (int32_t)mx; o[9] = (int32_t)my; o[10] = (int32_t)h->dec->GetRestartRead(); o[11] = h->dec->GetScanBad();
}
void jsimg_GetIdctTables(jsimg* h, float* lf, int32_t* li) { memcpy(lf, h->dec->GetIdctLookupFloat(), 64 * 64 * 4); memcpy(li, h->dec->GetIdctLookupFixed(), 64 * 64 * 4); }
void jsimg_GetStageMs(jsimg* h, float* ms5) { h->dec->GetStageMs(ms5); }
unsigned jsimg_GetScanStatus(jsimg* h) { return h->dec->GetScanStatus(); }

int jsimg_log_count(jsimg* h, int kind) { if (kind < 0) return (int)h->log.Lines().size(); return (int)h->log.Count((CDocLog::Kind)kind); }
const char* jsimg_log_line(jsimg* h, int kind, int index)
{
    int k = 0;
    for (auto& e : h->log.Lines()) if (kind < 0 || (int)e.kind == kind) { if (k == index) return e.text.c_str(); k++; }
    return "";
}
void jsimg_log_clear(jsimg* h) { h->log.Clear(); }

int jsimg_walk_jpeg(jsimg* h, const uint8_t* d, uint64_t n) { jsimg_set_file(h, d, n); return JfifWalk(h->dec, d, n); }
int jsimg_decode_jpeg(jsimg* h, const uint8_t* d, uint64_t n, int quiet)
{
    int start = jsimg_walk_jpeg(h, d, n);
    if (start < 0) return start;
    h->dec->DecodeScanImg((unsigned)start, true, quiet != 0);       // JfifDecode.cpp:5299
    return start;
}
int jsimg_parse_jpeg(const uint8_t* d, uint64_t n, jsgpu_tables* t, jsgpu_image_desc* desc)
{
    CDocLog log; CwindowBuf wb; CSnoopConfig cfg; wb.BufSet(d, (size_t)n);
    CimgDecode dec(&log, &wb, &cfg);
    int start = JfifWalk(&dec, d, n);
    if (start < 0) return start;
    dec.ExportTables(*t);
    if (!dec.ExportImageDesc(*desc, (unsigned)start)) return JFIFWALK_EMARKER;
    desc->scan_offset = (uint64_t)start; desc->scan_length = n - (uint64_t)start;
    return start;
}
}
