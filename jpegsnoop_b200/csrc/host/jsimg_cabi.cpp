// jsimg_cabi.cpp — include/jsimg.h: flat C shim over CimgDecode for FFI callers.
#include "../../../include/jsimg.h"
#include "ImgDecode.h"
#include "TiffExport.h"
#include "JfifWalk.h"
#include "JpegExport.h"
#include "DqtSearch.h"
#include <cstring>

struct jsimg {
    CDocLog log; CwindowBuf wbuf; CSnoopConfig cfg; CimgDecode* dec;
    jsgpu_ctx* search = nullptr;        // the searches' device context (jsimg_search_dqt, jsimg_buf_search), created on first use
    jsimg() : dec(new CimgDecode(&log, &wbuf, &cfg)) {}
    ~jsimg() { delete dec; if (search) jsgpu_free(search); }
};

extern "C" {
jsimg* jsimg_create(void) { return new jsimg(); }
void jsimg_destroy(jsimg* h) { delete h; }
void jsimg_config(jsimg* h, int ac, int fixed, int dev, int hk, int ik, int)
{ h->cfg.bDecodeScanImgAc = ac != 0; h->cfg.bIdctFixedPt = fixed != 0; h->cfg.nCudaDevice = dev; h->cfg.nHuffKernel = hk; h->cfg.nIdctKernel = ik; }
void jsimg_config_scan_err_max(jsimg* h, unsigned n) { h->cfg.nErrMaxDecodeScan = n; }
void jsimg_ScanErrorsDisable(jsimg* h) { h->dec->ScanErrorsDisable(); }
void jsimg_ScanErrorsEnable(jsimg* h)  { h->dec->ScanErrorsEnable(); }
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
void jsimg_GetDhtHisto(jsimg* h, uint32_t* out) { memcpy(out, h->dec->GetDhtHisto(), JSGPU_HISTO_WORDS * sizeof(uint32_t)); }
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
// ProcessFile with nPosStart = pos over the installed file: the walk, then DecodeScanImg at the scan's absolute offset
static int decode_at(jsimg* h, uint64_t pos, int quiet)
{
    const int start = JfifWalk(h->dec, h->wbuf.BufData(), h->wbuf.GetPosEof(), pos);
    if (start < 0) return start;
    h->dec->DecodeScanImg((unsigned)start, true, quiet != 0);       // JfifDecode.cpp:5299
    return start;
}
int jsimg_decode_jpeg(jsimg* h, const uint8_t* d, uint64_t n, int quiet) { return jsimg_decode_jpeg_at(h, d, n, 0, quiet); }
int jsimg_decode_jpeg_at(jsimg* h, const uint8_t* d, uint64_t n, uint64_t pos, int quiet) { jsimg_set_file(h, d, n); return decode_at(h, pos, quiet); }
int jsimg_buf_search(jsimg* h, uint64_t start, uint32_t value, uint32_t len, int fwd, uint64_t* found_pos)
{
    if (!h->search) {
        const int r = jsgpu_init(h->cfg.nCudaDevice, &h->search);
        if (r != JSGPU_OK) {
            h->search = nullptr;
            h->log.AddLineErr(std::string("*** ERROR: Img Search: GPU search unavailable (") + jsgpu_strerror(r) + ") ***");
            return r;
        }
    }
    std::vector<jsgpu_overlay> ovl;
    for (auto& o : h->wbuf.Overlays()) ovl.push_back({(uint64_t)o.start, (uint64_t)o.data.size(), o.data.data()});
    int found = 0;
    const int r = jsgpu_find_value(h->search, h->wbuf.BufData(), h->wbuf.GetPosEof(), start, value, len, fwd, ovl.data(),
                                   (uint32_t)ovl.size(), &found, found_pos);
    if (r != JSGPU_OK) {
        h->log.AddLineErr(std::string("*** ERROR: Img Search: ") + jsgpu_strerror(r) + " (" + jsgpu_last_error(h->search) + ") ***");
        return r;
    }
    return found;
}
int jsimg_img_search(jsimg* h, uint64_t start, int fwd, int quiet, int* found, uint64_t* pos, int* decoded)
{
    *found = 0; *pos = start; *decoded = 0;
    if (!fwd && start == 0) return 0;                               // "Don't attempt to search past start of file" (JPEGsnoopDoc.cpp:902)
    uint64_t p = 0;
    const int r = jsimg_buf_search(h, start, 0xFFD8FF, 3, fwd, &p);
    if (r < 0) return r;
    *found = r;
    if (r) *pos = p;
    else if (fwd) return 0;                                         // forward: the start stays, nothing is reprocessed
    else *pos = 0;                                                  // reverse: reprocess from the start of the file
    *decoded = 1;
    return decode_at(h, *pos, quiet);
}
int jsimg_decode_offset_mode(jsimg* h, const uint8_t* d, uint64_t n, int mode, uint64_t pos, int quiet, uint64_t* pos_used)
{
    jsimg_set_file(h, d, n);
    *pos_used = 0;
    uint64_t at = 0, p = 0;
    int r = 0;
    switch (mode) {                                                 // CJPEGsnoopCore::DoAnalyzeOffset (JPEGsnoopCore.cpp:700-756)
    case JSIMG_OFFSET_START: break;
    case JSIMG_OFFSET_SRCH1: {                                      // search only when the decode at 0 did not reach a frame header
        bool bImgOK = false;
        JfifWalk(h->dec, d, n, 0, &bImgOK);
        if (bImgOK) break;
        if ((r = jsimg_buf_search(h, 0, 0xFFD8FF, 3, 1, &p)) < 0) return r;
        if (r) at = p;
        break; }
    case JSIMG_OFFSET_SRCH2:                                        // the first SOI after offset 0
        if ((r = jsimg_buf_search(h, 0, 0xFFD8FF, 3, 1, &p)) < 0) return r;
        if (r) at = p;
        break;
    case JSIMG_OFFSET_POS: at = pos; break;
    default: return JSGPU_EINVAL;
    }
    *pos_used = at;
    return decode_at(h, at, quiet);
}
int jsimg_search_dqt(jsimg* h, const uint8_t* d, uint64_t n, const char* exe_path, int analysed, const char* analysed_path)
{
    return DqtSearch(&h->log, &h->search, h->cfg.nCudaDevice, analysed ? h->dec : nullptr, d, n, exe_path, analysed_path);
}
int jsimg_parse_jpeg(const uint8_t* d, uint64_t n, jsgpu_tables* t, jsgpu_image_desc* desc) { return jsimg_parse_jpeg_at(d, n, 0, t, desc); }
int jsimg_parse_jpeg_at(const uint8_t* d, uint64_t n, uint64_t pos, jsgpu_tables* t, jsgpu_image_desc* desc)
{
    CDocLog log; CwindowBuf wb; CSnoopConfig cfg; wb.BufSet(d, (size_t)n);
    CimgDecode dec(&log, &wb, &cfg);
    int start = JfifWalk(&dec, d, n, pos);
    if (start < 0) return start;
    dec.ExportTables(*t);
    if (!dec.ExportImageDesc(*desc, (unsigned)start)) return JFIFWALK_EMARKER;
    desc->scan_offset = (uint64_t)start; desc->scan_length = n - (uint64_t)start;
    return start;
}
}

int jsimg_export_jpeg(jsimg* h, uint64_t pos, const char* src_name, const char* out_path, unsigned flags)
{
    std::vector<uint32_t> soi, term;
    const int r = JpegFindMarkers(&h->log, &h->search, h->cfg.nCudaDevice, h->wbuf, soi, term);
    if (r != JSGPU_OK) return r;
    return JpegExportOne(&h->log, h->wbuf, term, pos, src_name ? src_name : "", out_path ? out_path : "", flags);
}

int64_t jsimg_extract_all(jsimg* h, jsgpu_ctx* ctx, const char* src_name, const char* out_name, unsigned flags, uint64_t* offsets,
                          uint32_t* numbers, uint64_t cap)
{
    std::vector<uint32_t> soi, term;
    const int r = JpegFindMarkers(&h->log, ctx ? &ctx : &h->search, h->cfg.nCudaDevice, h->wbuf, soi, term);
    if (r != JSGPU_OK) return r;
    std::vector<uint64_t> offs;
    std::vector<uint32_t> nums;
    const int64_t k = JpegExtractAll(&h->log, h->wbuf, soi, term, src_name ? src_name : "", out_name ? out_name : "", flags, offs, nums);
    if (k < 0) return JSGPU_EINVAL;
    for (uint64_t i = 0; i < std::min<uint64_t>(cap, offs.size()); i++) { offsets[i] = offs[i]; numbers[i] = nums[i]; }
    return k;
}
