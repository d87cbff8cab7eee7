// ImgDecode.cpp — host side of the H100 scan decoder (see ImgDecode.h).  Reference line
// numbers refer to /root/reference/source/ImgDecode.cpp.  Only table keeping, validation,
// byte shipping and result hosting happen here; all decoding is on the device (jsgpu_*).
#include "ImgDecode.h"
#include "TiffExport.h"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdarg>
#include <vector>

static std::string fmt(const char* f, ...)
{
    char buf[512];
    va_list ap; va_start(ap, f); vsnprintf(buf, sizeof buf, f, ap); va_end(ap);
    return std::string(buf);
}

// The only places where the two build modes differ: how a line reaches the log, how the scan bytes are fetched, and where
// the device knobs (which the reference's CSnoopConfig does not have) come from.
#ifdef JSGPU_HOST_EXTERNAL_TYPES
#include "JPEGsnoop.h"          // CJPEGsnoopApp::m_pAppConfig, as the reference's constructor reads it (ImgDecode.cpp:146-148)
#define JS_LOGSTR(x) CString(std::string(x).c_str())
static void js_copy_scan(CwindowBuf* w, unsigned long off, size_t n, uint8_t* dst) { for (size_t i = 0; i < n; i++) dst[i] = w->Buf(off + (unsigned long)i); }
#ifdef IDCT_FIXEDPT
static const bool kCfgIdctFixed = true;      // the reference's own compile-time switch (ImgDecode.cpp:32)
#else
static const bool kCfgIdctFixed = false;
#endif
#define JS_CFG_IDCT_FIXED(c)   kCfgIdctFixed
#define JS_CFG_DEVICE(c)       0
#define JS_CFG_HUFF(c)         0
#define JS_CFG_IDCTK(c)        0
#else
#define JS_LOGSTR(x) std::string(x)
static void js_copy_scan(CwindowBuf* w, unsigned long off, size_t n, uint8_t* dst) { w->BufCopy(off, n, dst); }
#define JS_CFG_IDCT_FIXED(c)   ((c)->bIdctFixedPt)
#define JS_CFG_DEVICE(c)       ((c)->nCudaDevice)
#define JS_CFG_HUFF(c)         ((c)->nHuffKernel)
#define JS_CFG_IDCTK(c)        ((c)->nIdctKernel)
#endif

CimgDecode::CimgDecode(CDocLog* pLog, CwindowBuf* pWBuf, CSnoopConfig* pConfig)
{
#ifdef JSGPU_HOST_EXTERNAL_TYPES
    m_pAppConfig = pConfig ? pConfig : ((CJPEGsnoopApp*)AfxGetApp())->m_pAppConfig;
#else
    m_pAppConfig = pConfig ? pConfig : &m_sOwnConfig;
#endif
    m_pLog = pLog; m_pWBuf = pWBuf; m_pGpu = nullptr;
    m_bDibTempReady = false; m_bPreviewIsJpeg = false;
    m_pMcuFileMap = nullptr;
    m_pPixValY = m_pPixValCb = m_pPixValCr = nullptr;
    m_pBlkDcValY = m_pBlkDcValCb = m_pBlkDcValCr = nullptr;
    m_pDibBits = nullptr;
    m_bScanErrorsDisable = false; m_nWarnBadScanNum = 0; m_nScanErrMax = 20;
    m_bDecodeScanAc = true; m_bScanBad = false; m_nScanStatus = 0;
    m_nMcuWidth = m_nMcuHeight = 1;          // ref :189-191 (avoid divide-by-zero before the first decode)
    m_nRestartRead = 0;
    for (float& v : m_afStageMs) v = 0.f;
    m_bDetailVlc = false; m_nDetailVlcX = m_nDetailVlcY = 0; m_nDetailVlcLen = 1;      // ref :194-197
    m_bHistEn = m_bStatClipEn = false;
    m_nPreviewMode = 1;                      // PREVIEW_RGB (ref :220)
    m_nPreviewShiftY = m_nPreviewShiftCb = m_nPreviewShiftCr = 0; m_nPreviewShiftMcuX = m_nPreviewShiftMcuY = 0;   // ref :226
    m_nWarnYccClipNum = 0; m_nEndPos = m_nEndAlign = 0; m_bDecodedOnDevice = false;
    m_bDibHistRgbReady = m_bDibHistYReady = false;
    memset(m_anStatClip, 0, sizeof m_anStatClip); memset(m_anHistoMin, 0, sizeof m_anHistoMin); memset(m_anHistoMax, 0, sizeof m_anHistoMax);
    memset(m_anHistoSum, 0, sizeof m_anHistoSum); m_nHistoCount = 0;
    memset(m_anCcHisto, 0, sizeof m_anCcHisto); memset(m_anHistoYFull, 0, sizeof m_anHistoYFull);
    Reset();
    PrecalcIdct();
    ResetState();
}

CimgDecode::~CimgDecode()
{
    FreeOutputs();
    if (m_pGpu) jsgpu_free(m_pGpu);
}

void CimgDecode::FreeOutputs()
{
    delete[] m_pMcuFileMap; m_pMcuFileMap = nullptr;
    delete[] m_pPixValY; delete[] m_pPixValCb; delete[] m_pPixValCr; m_pPixValY = m_pPixValCb = m_pPixValCr = nullptr;
    delete[] m_pBlkDcValY; delete[] m_pBlkDcValCb; delete[] m_pBlkDcValCr; m_pBlkDcValY = m_pBlkDcValCb = m_pBlkDcValCr = nullptr;
    delete[] m_pDibBits; m_pDibBits = nullptr;
}

// ref :49-138
void CimgDecode::Reset()
{
    m_nRestartRead = 0;
    m_nImgSizeX = m_nImgSizeY = 0;
    m_nMcuXMax = m_nMcuYMax = m_nBlkXMax = m_nBlkYMax = 0;
    m_bBrightValid = false; m_nBrightY = m_nBrightCb = m_nBrightCr = -32768;
    m_nBrightR = m_nBrightG = m_nBrightB = 0; m_nBrightMcuX = m_nBrightMcuY = 0;
    m_bAvgYValid = false; m_nAvgY = 0;
    m_bDibTempReady = false;
    m_bScanBad = false; m_nScanStatus = 0;
    FreeOutputs();
    m_bDecodedOnDevice = false;
    if (!m_bScanErrorsDisable) m_nWarnBadScanNum = 0;
    m_nWarnYccClipNum = 0;                   // ref :130
}

// ref :286-306, 343-360, 373-406
void CimgDecode::ResetState()
{
    ResetDhtLookup();
    ResetDqtTables();
    for (unsigned i = 0; i < MAX_SOF_COMP_NF; i++) { m_anSofSampFactH[i] = 0; m_anSofSampFactV[i] = 0; }
    m_bImgDetailsSet = false;
    m_nNumSofComps = 0;
    m_nPrecision = 0;
    m_bScanErrorsDisable = false;
}
void CimgDecode::ResetDqtTables()
{
    for (unsigned i = 0; i < MAX_DQT_COMP; i++) m_anDqtTblSel[i] = -1;
    memset(m_anDqtCoeff, 0, sizeof m_anDqtCoeff);
    memset(m_anDqtCoeffZz, 0, sizeof m_anDqtCoeffZz);
    m_nNumSofComps = 0;
}
void CimgDecode::ResetDhtLookup()
{
    memset(m_anDhtHisto, 0, sizeof m_anDhtHisto);
    memset(m_anDhtLookupSetMax, 0, sizeof m_anDhtLookupSetMax);
    memset(m_anDhtLookupSize, 0, sizeof m_anDhtLookupSize);
    memset(m_anDhtLookup_bitlen, 0, sizeof m_anDhtLookup_bitlen);
    memset(m_anDhtLookup_bits, 0, sizeof m_anDhtLookup_bits);
    memset(m_anDhtLookup_mask, 0, sizeof m_anDhtLookup_mask);
    memset(m_anDhtLookup_code, 0, sizeof m_anDhtLookup_code);
    for (unsigned c = 0; c < MAX_DHT_CLASS; c++) for (unsigned i = 0; i < 1 + MAX_SOS_COMP_NS; i++) m_anDhtTblSel[c][i] = -1;
    m_nNumSosComps = 0;
}

// The IDCT tables depend on the host libm's cosf and on float rounding of the reference's exact
// expression (ref :2313-2351): float constants, argument evaluated in float, cos on a float
// (-> cosf), product of the two cosines first, then Cu*Cv*that, then (int)(x*1024).
void CimgDecode::PrecalcIdct()
{
    const float fPi = (float)3.141592654, fSqrtHalf = (float)0.707106781;
    for (unsigned nY = 0; nY < 8; nY++) for (unsigned nX = 0; nX < 8; nX++) {
        const unsigned nYX = nY * 8 + nX;
        for (unsigned nV = 0; nV < 8; nV++) for (unsigned nU = 0; nU < 8; nU++) {
            const unsigned nVU = nV * 8 + nU;
            const float fCu = (nU == 0) ? fSqrtHalf : 1, fCv = (nV == 0) ? fSqrtHalf : 1;
            const float fCosProd = cosf((2 * nX + 1) * nU * fPi / 16) * cosf((2 * nY + 1) * nV * fPi / 16);
            const float fInside = fCu * fCv * fCosProd;
            m_afIdctLookup[nYX][nVU] = fInside;
            m_anIdctLookup[nYX][nVU] = (int)(fInside * (1 << 10));
        }
    }
}

// ---- setters: same range checks, return values and log lines as the reference ----------------
bool CimgDecode::SetDqtEntry(unsigned nTblDestId, unsigned nCoeffInd, unsigned nCoeffIndZz, unsigned short nCoeffVal)
{
    if (nTblDestId < MAX_DQT_DEST_ID && nCoeffInd < MAX_DQT_COEFF && nCoeffIndZz < MAX_DQT_COEFF) {
        m_anDqtCoeff[nTblDestId][nCoeffInd] = nCoeffVal;
        m_anDqtCoeffZz[nTblDestId][nCoeffIndZz] = nCoeffVal;
        return true;
    }
    return false;      // ref :433-451 (debug string only, no log line)
}
unsigned CimgDecode::GetDqtEntry(unsigned nTblDestId, unsigned nCoeffInd)
{
    if (nTblDestId < MAX_DQT_DEST_ID && nCoeffInd < MAX_DQT_COEFF) return m_anDqtCoeff[nTblDestId][nCoeffInd];
    m_pLog->AddLineErr(JS_LOGSTR(fmt("ERROR: GetDqtEntry(nTblDestId=%u, nCoeffInd=%u) out of indexed range", nTblDestId, nCoeffInd)));
    return 0;
}
bool CimgDecode::SetDqtTables(unsigned nCompId, unsigned nTbl)
{
    if (nCompId < MAX_SOF_COMP_NF && nTbl < MAX_DQT_DEST_ID) { m_anDqtTblSel[nCompId] = (int)nTbl; return true; }
    m_pLog->AddLineErr(JS_LOGSTR(fmt("ERROR: SetDqtTables(Comp ID=%u, Table=%u) out of indexed range", nCompId, nTbl)));
    return false;
}
bool CimgDecode::SetDhtTables(unsigned nCompInd, unsigned nTblDc, unsigned nTblAc)
{
    if (nCompInd >= 1 && nCompInd < MAX_SOS_COMP_NS + 1 && nTblDc < MAX_DHT_DEST_ID && nTblAc < MAX_DHT_DEST_ID) {
        m_anDhtTblSel[DHT_CLASS_DC][nCompInd] = (int)nTblDc;
        m_anDhtTblSel[DHT_CLASS_AC][nCompInd] = (int)nTblAc;
        return true;
    }
    m_pLog->AddLineErr(JS_LOGSTR(fmt("ERROR: SetDhtTables(comp=%u, TblDC=%u TblAC=%u) out of indexed range", nCompInd, nTblDc, nTblAc)));
    return false;
}
bool CimgDecode::SetDhtEntry(unsigned nDestId, unsigned nClass, unsigned nInd, unsigned nLen, unsigned nBits, unsigned nMask, unsigned nCode)
{
    if (nDestId >= MAX_DHT_DEST_ID || nClass >= MAX_DHT_CLASS || nInd >= MAX_DHT_CODES) {
        m_pLog->AddLineErr(JS_LOGSTR("ERROR: Attempt to set DHT entry out of range"));
        return false;
    }
    m_anDhtLookup_bitlen[nClass][nDestId][nInd] = nLen;
    m_anDhtLookup_bits[nClass][nDestId][nInd] = nBits;
    m_anDhtLookup_mask[nClass][nDestId][nInd] = nMask;
    m_anDhtLookup_code[nClass][nDestId][nInd] = nCode;
    if (nDestId > m_anDhtLookupSetMax[nClass]) m_anDhtLookupSetMax[nClass] = nDestId;
    // The reference also fills a 9-bit direct table here (ref :786-818); the device builds its own
    // look-up tables from the entry list in jsgpu_upload_tables().
    return true;
}
bool CimgDecode::SetDhtSize(unsigned nDestId, unsigned nClass, unsigned nSize)
{
    if (nDestId >= MAX_DHT_DEST_ID || nClass >= MAX_DHT_CLASS || nSize >= MAX_DHT_CODES) {
        m_pLog->AddLineErr(JS_LOGSTR("ERROR: Attempt to set DHT table size out of range"));
        return false;
    }
    m_anDhtLookupSize[nClass][nDestId] = nSize;
    return true;
}
void CimgDecode::SetPrecision(unsigned nPrecision) { m_nPrecision = nPrecision; }
void CimgDecode::SetImageDimensions(unsigned, unsigned) {}
void CimgDecode::SetImageDetails(unsigned nDimX, unsigned nDimY, unsigned nCompsSOF, unsigned nCompsSOS, bool bRstEn, unsigned nRstInterval)
{
    m_bImgDetailsSet = true; m_nDimX = nDimX; m_nDimY = nDimY;
    m_nNumSofComps = nCompsSOF; m_nNumSosComps = nCompsSOS;
    m_bRestartEn = bRstEn; m_nRestartInterval = nRstInterval;
}
void CimgDecode::SetSofSampFactors(unsigned nCompInd, unsigned nSampFactH, unsigned nSampFactV)
{
    if (nCompInd >= MAX_SOF_COMP_NF) return;          // the reference does not range-check (ref :619-624 "TODO")
    m_anSofSampFactH[nCompInd] = nSampFactH; m_anSofSampFactV[nCompInd] = nSampFactV;
}
void CimgDecode::ScanErrorsDisable() { m_nWarnBadScanNum = m_nScanErrMax; m_bScanErrorsDisable = true; }
void CimgDecode::ScanErrorsEnable()  { m_nWarnBadScanNum = 0; m_bScanErrorsDisable = false; }

// ---- C-ABI structure export -------------------------------------------------------------------
void CimgDecode::ExportTables(jsgpu_tables& t) const
{
    memset(&t, 0, sizeof t);
    for (unsigned q = 0; q < 4; q++) for (unsigned k = 0; k < 64; k++) t.dqt_zz[q][k] = m_anDqtCoeffZz[q][k];
    for (unsigned c = 0; c < 2; c++) for (unsigned id = 0; id < 4; id++) {
        unsigned n = m_anDhtLookupSize[c][id];
        t.dht_size[c][id] = n;
        for (unsigned i = 0; i < n && i < MAX_DHT_CODES; i++) {
            t.dht_bits[c][id][i] = m_anDhtLookup_bits[c][id][i] & m_anDhtLookup_mask[c][id][i];
            t.dht_len[c][id][i] = (uint8_t)m_anDhtLookup_bitlen[c][id][i];
            t.dht_code[c][id][i] = (uint8_t)m_anDhtLookup_code[c][id][i];
        }
    }
}
bool CimgDecode::ExportImageDesc(jsgpu_image_desc& d, unsigned nStart) const
{
    memset(&d, 0, sizeof d);
    d.dim_x = m_nDimX; d.dim_y = m_nDimY; d.num_sof_comps = m_nNumSofComps; d.num_sos_comps = m_nNumSosComps;
    d.precision = m_nPrecision; d.restart_en = m_bRestartEn ? 1 : 0; d.restart_interval = m_nRestartInterval;
    for (unsigned c = 0; c < 3 && c < m_nNumSosComps; c++) {
        d.samp_h[c] = m_anSofSampFactH[c + 1]; d.samp_v[c] = m_anSofSampFactV[c + 1];
        if (m_anDqtTblSel[c + 1] < 0 || m_anDhtTblSel[0][c + 1] < 0 || m_anDhtTblSel[1][c + 1] < 0) return false;
        d.dqt_sel[c] = (uint32_t)m_anDqtTblSel[c + 1];
        d.dht_dc_sel[c] = (uint32_t)m_anDhtTblSel[0][c + 1]; d.dht_ac_sel[c] = (uint32_t)m_anDhtTblSel[1][c + 1];
    }
    d.file_pos = nStart;
    return true;
}

bool CimgDecode::EnsureDevice()
{
    if (m_pGpu) return true;
    int r = jsgpu_init(JS_CFG_DEVICE(m_pAppConfig), &m_pGpu);
    if (r != JSGPU_OK) {
        // No CPU fallback exists: the decode fails loudly, in the reference's own convention (a log line)
        m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: GPU scan decoder unavailable (%s) — scan not decoded ***", jsgpu_strerror(r))));
        m_pGpu = nullptr;
        return false;
    }
    r = jsgpu_set_idct_tables(m_pGpu, &m_anIdctLookup[0][0], &m_afIdctLookup[0][0]);
    if (r != JSGPU_OK) { m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: GPU scan decoder: %s ***", jsgpu_last_error(m_pGpu)))); return false; }
    return true;
}

// ref :2723-3745.  Order of checks and the log lines for refused inputs follow the reference.
void CimgDecode::DecodeScanImg(unsigned nStart, bool bDisplay, bool bQuiet)
{
    bool bDecodeScanAc = bDisplay ? m_pAppConfig->bDecodeScanImgAc : false;        // ref :2735-2739
    const bool bDumpHistoY = m_pAppConfig->bDumpHistoY;                            // ref :2730
    m_bHistEn = m_pAppConfig->bHistoEn; m_bStatClipEn = m_pAppConfig->bStatClipEn; // ref :2740-2741
    Reset();
    m_nScanErrMax = m_pAppConfig->nErrMaxDecodeScan;
    m_bDecodeScanAc = bDecodeScanAc;
    m_bPreviewIsJpeg = false;

    if (!m_bImgDetailsSet) { m_pLog->AddLineErr(JS_LOGSTR("*** ERROR: Decoding image before Image components defined ***")); return; }
    if (m_nNumSosComps != NUM_CHAN_GRAYSCALE && m_nNumSosComps != NUM_CHAN_YCC) {
        m_pLog->AddLineWarn(JS_LOGSTR(fmt("  NOTE: Number of SOS components not supported [%u]", m_nNumSosComps)));
        return;
    }
    unsigned nHMax = 0, nVMax = 0;
    for (unsigned c = 1; c <= m_nNumSosComps; c++) { if (m_anSofSampFactH[c] > nHMax) nHMax = m_anSofSampFactH[c]; if (m_anSofSampFactV[c] > nVMax) nVMax = m_anSofSampFactV[c]; }
    if (m_nNumSosComps == 1) {                                                     // ref :2805-2817
        if (m_anSofSampFactH[1] != 1 || m_anSofSampFactV[1] != 1) m_pLog->AddLineWarn(JS_LOGSTR("    Altering sampling factor for single component scan to 0x11"));
        m_anSofSampFactH[1] = 1; m_anSofSampFactV[1] = 1; nHMax = nVMax = 1;
    }
    if (nHMax == 0 || nVMax == 0 || nHMax > MAX_SAMP_FACT_H || nVMax > MAX_SAMP_FACT_V) {
        m_pLog->AddLineWarn(JS_LOGSTR(fmt("  NOTE: Degree of subsampling factor not supported [HMax=%u, VMax=%u]", nHMax, nVMax)));
        return;
    }
    m_nMcuWidth = nHMax * 8; m_nMcuHeight = nVMax * 8;
    m_nMcuXMax = m_nDimX / m_nMcuWidth + ((m_nDimX % m_nMcuWidth) ? 1 : 0);
    m_nMcuYMax = m_nDimY / m_nMcuHeight + ((m_nDimY % m_nMcuHeight) ? 1 : 0);
    m_nBlkXMax = m_nMcuXMax * nHMax; m_nBlkYMax = m_nMcuYMax * nVMax;
    if (m_nBlkXMax == 0 || m_nBlkYMax == 0) return;                                // ref :2866-2868
    m_nImgSizeX = m_nMcuXMax * m_nMcuWidth; m_nImgSizeY = m_nMcuYMax * m_nMcuHeight;

    const size_t nMcu = (size_t)m_nMcuXMax * m_nMcuYMax, nBlk = (size_t)m_nBlkXMax * m_nBlkYMax, nPix = (size_t)m_nImgSizeX * m_nImgSizeY;
    m_pMcuFileMap = new unsigned[nMcu]();
    m_pBlkDcValY = new short[nBlk]();
    if (m_nNumSosComps == NUM_CHAN_YCC) { m_pBlkDcValCb = new short[nBlk](); m_pBlkDcValCr = new short[nBlk](); }
    m_pPixValY = new short[nPix]();
    if (m_nNumSosComps == NUM_CHAN_YCC) { m_pPixValCb = new short[nPix](); m_pPixValCr = new short[nPix](); }
    if (bDisplay) m_pDibBits = new unsigned char[nPix * 4]();

    if (!bQuiet) { m_pLog->AddLineHdr(JS_LOGSTR("*** Decoding SCAN Data ***")); m_pLog->AddLine(JS_LOGSTR(fmt("  OFFSET: 0x%08X", nStart))); }
    if (m_nNumSofComps != NUM_CHAN_GRAYSCALE && m_nNumSofComps != NUM_CHAN_YCC) {   // ref :3029-3035
        m_pLog->AddLineWarn(JS_LOGSTR(fmt("  NOTE: Number of Image Components not supported [%u]", m_nNumSofComps)));
        return;
    }
    for (unsigned c = 1; c <= m_nNumSosComps; c++) if (m_anDqtTblSel[c] < 0) {
        m_pLog->AddLineErr(JS_LOGSTR("*** ERROR: Decoding image before DQT Table Selection via JFIF_SOF ***")); return; }
    bool bDhtReady = true;
    for (unsigned k = 0; k < 2; k++) for (unsigned c = 1; c <= m_nNumSosComps; c++) if (m_anDhtTblSel[k][c] < 0) bDhtReady = false;
    if (bDhtReady) for (unsigned c = 1; c <= m_nNumSosComps; c++) {
        if (m_anDhtLookupSize[0][m_anDhtTblSel[0][c]] == 0) bDhtReady = false;
        if (m_anDhtLookupSize[1][m_anDhtTblSel[1][c]] == 0) bDhtReady = false;
    }
    if (!bDhtReady) { m_pLog->AddLineErr(JS_LOGSTR("*** ERROR: Decoding image before DHT Table Selection via JFIF_SOS ***")); return; }
    if (!bQuiet) {
        m_pLog->AddLine(JS_LOGSTR(m_bDecodeScanAc ? "  Scan Decode Mode: Full IDCT (AC + DC)" : "  Scan Decode Mode: No IDCT (DC only)"));
        if (!m_bDecodeScanAc) m_pLog->AddLineWarn(JS_LOGSTR("    NOTE: Low-resolution DC component shown. Can decode full-res with [Options->Scan Segment->Full IDCT]"));
        m_pLog->AddLine(JS_LOGSTR(""));
    }

    if (bDisplay) {                                                                // ref :3144-3156
        memset(m_anStatClip, 0, sizeof m_anStatClip); memset(m_anHistoMin, 0, sizeof m_anHistoMin); memset(m_anHistoMax, 0, sizeof m_anHistoMax);
        memset(m_anHistoSum, 0, sizeof m_anHistoSum); m_nHistoCount = 0;
        memset(m_anCcHisto, 0, sizeof m_anCcHisto); memset(m_anHistoYFull, 0, sizeof m_anHistoYFull);
    }

    // ---- device decode (replaces HOT LOOPS 1-4, ref :3164-3630 and :4619-4821) -----------------
    if (!EnsureDevice()) { m_bScanBad = true; return; }
    jsgpu_options opt; jsgpu_get_options(m_pGpu, &opt);
    opt.idct_mode = JS_CFG_IDCT_FIXED(m_pAppConfig) ? 0 : 1;
    opt.decode_ac = m_bDecodeScanAc ? 1 : 0;
    opt.huff_kernel = JS_CFG_HUFF(m_pAppConfig); opt.idct_kernel = JS_CFG_IDCTK(m_pAppConfig);
    opt.want_histo = 1; opt.want_mcu_map = 1;
    opt.scan_err_max = m_nScanErrMax;
    jsgpu_set_options(m_pGpu, &opt);
    jsgpu_set_scan_error_state(m_pGpu, m_nWarnBadScanNum, m_bScanErrorsDisable ? 1 : 0);
    // CalcChannelPreview() at the end of the decode (ref :3641-3643) with this object's preview settings: the device takes the
    // extra colour pass inside jsgpu_batch_decode only when they differ from the defaults
    jsgpu_preview pv; PreviewSettings(pv);
    if (!bDisplay) { memset(&pv, 0, sizeof pv); pv.mode = 1; }
    jsgpu_set_preview(m_pGpu, &pv);
    jsgpu_detail dtl; memset(&dtl, 0, sizeof dtl);
    dtl.enable = m_bDetailVlc ? 1 : 0; dtl.image = 0; dtl.mcu_x = m_nDetailVlcX; dtl.mcu_y = m_nDetailVlcY; dtl.len = m_nDetailVlcLen;
    jsgpu_set_detail(m_pGpu, &dtl);
    const bool bPreviewPass = pv.hist_en || pv.statclip_en || pv.mode != 1 || pv.shift_y || pv.shift_cb || pv.shift_cr;

    jsgpu_tables* pTables = new jsgpu_tables;
    ExportTables(*pTables);
    jsgpu_image_desc d;
    ExportImageDesc(d, nStart);
    const unsigned long nEof = m_pWBuf->GetPosEof();
    const size_t nScanBytes = (nStart < nEof) ? (size_t)(nEof - nStart) : 0;
    std::vector<uint8_t> scan(nScanBytes + 4, 0);
    js_copy_scan(m_pWBuf, nStart, nScanBytes, scan.data());         // one bulk read instead of Buf() per byte (ref :1398-1399)
    d.table_set = 0; d.scan_offset = 0; d.scan_length = nScanBytes;

    int r = jsgpu_upload_tables(m_pGpu, pTables, 1);
    delete pTables;
    if (r == JSGPU_OK) r = jsgpu_batch_begin(m_pGpu, &d, 1, nScanBytes);
    if (r == JSGPU_OK) r = jsgpu_batch_upload(m_pGpu, scan.data(), nScanBytes);
    if (r == JSGPU_OK) r = jsgpu_batch_decode(m_pGpu);
    if (r == JSGPU_OK) r = jsgpu_sync(m_pGpu);
    jsgpu_image_layout lo; memset(&lo, 0, sizeof lo);
    if (r == JSGPU_OK) r = jsgpu_batch_layout(m_pGpu, &lo, 1);
    if (r != JSGPU_OK) {
        m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: GPU scan decoder failed: %s (%s) ***", jsgpu_strerror(r), jsgpu_last_error(m_pGpu))));
        m_bScanBad = true;
        return;
    }
    m_bDecodedOnDevice = true;
    jsgpu_batch_stage_ms(m_pGpu, m_afStageMs);
    jsgpu_batch_download(m_pGpu, JSGPU_OUT_MCU_MAP, 0, m_pMcuFileMap, nMcu * 4);
    jsgpu_batch_download(m_pGpu, JSGPU_OUT_BLK_Y, 0, m_pBlkDcValY, nBlk * 2);
    {
        // the reference counts into m_anDhtHisto (ref :1191) and clears it only in ResetDhtLookup (ref :375): a second
        // DecodeScanImg without a new marker walk adds to the first one's counts
        unsigned anHisto[JSGPU_HISTO_WORDS];
        jsgpu_batch_download(m_pGpu, JSGPU_OUT_HISTO, 0, anHisto, sizeof anHisto);
        static_assert(sizeof anHisto == sizeof m_anDhtHisto, "histogram layout");
        unsigned* pHisto = &m_anDhtHisto[0][0][0];
        for (unsigned i = 0; i < JSGPU_HISTO_WORDS; i++) pHisto[i] += anHisto[i];
    }
    if (m_nNumSosComps == NUM_CHAN_YCC) {
        jsgpu_batch_download(m_pGpu, JSGPU_OUT_BLK_CB, 0, m_pBlkDcValCb, nBlk * 2);
        jsgpu_batch_download(m_pGpu, JSGPU_OUT_BLK_CR, 0, m_pBlkDcValCr, nBlk * 2);
    }
    int32_t st[JSGPU_STAT_WORDS]; memset(st, 0, sizeof st);
    jsgpu_batch_download(m_pGpu, JSGPU_OUT_STATS, 0, st, sizeof st);
    m_nRestartRead = (unsigned)st[JSGPU_STAT_NRST];
    if (bDisplay) {
        jsgpu_batch_download(m_pGpu, JSGPU_OUT_PIX_Y, 0, m_pPixValY, nPix * 2);
        if (m_nNumSosComps == NUM_CHAN_YCC) {
            jsgpu_batch_download(m_pGpu, JSGPU_OUT_PIX_CB, 0, m_pPixValCb, nPix * 2);
            jsgpu_batch_download(m_pGpu, JSGPU_OUT_PIX_CR, 0, m_pPixValCr, nPix * 2);
        }
        jsgpu_batch_download(m_pGpu, JSGPU_OUT_DIB, 0, m_pDibBits, nPix * 4);
        m_nAvgY = st[JSGPU_STAT_AVGY]; m_bAvgYValid = true;
        m_nBrightY = st[JSGPU_STAT_BRIGHT_Y]; m_nBrightCb = st[JSGPU_STAT_BRIGHT_CB]; m_nBrightCr = st[JSGPU_STAT_BRIGHT_CR];
        m_nBrightR = (unsigned)st[JSGPU_STAT_BRIGHT_R]; m_nBrightG = (unsigned)st[JSGPU_STAT_BRIGHT_G]; m_nBrightB = (unsigned)st[JSGPU_STAT_BRIGHT_B];
        m_nBrightMcuX = (unsigned)st[JSGPU_STAT_BRIGHT_MX]; m_nBrightMcuY = (unsigned)st[JSGPU_STAT_BRIGHT_MY];
        m_bBrightValid = true;
        m_bDibTempReady = true; m_bPreviewIsJpeg = true;                           // ref :3646-3649
    }
    m_nScanStatus = lo.status;
    // What the scan left in the log: the error events of a damaged scan (the device decoded it a second time the way ReadScanVal /
    // BuffAddByte / DecodeScanComp do — one-bit resynchronisation, stray markers, lazy restarts, error cap: ref :1096-1115, 1166-1187,
    // 1257-1282, 1486-1561, 1683-1706, 1737-1797, 2605-2660, 3180-3200 — and kept what the reference would have logged) and, when
    // SetDetailVlc asked for it, the symbol-by-symbol dump of the chosen MCUs, in the order the reference writes them.
    bool bMarkerNoteLogged = false;
    {
        jsgpu_scan_errors* pErr = new jsgpu_scan_errors; memset(pErr, 0, 16);
        uint32_t anDetInfo[4] = { 0, 0, 0, 0 };
        const bool bExact = (lo.status & JSGPU_ST_EXACT) != 0;
        const bool bHaveDet = m_bDetailVlc && jsgpu_batch_detail_info(m_pGpu, anDetInfo) == JSGPU_OK;
        const bool bHaveErr = (bExact || bHaveDet) && jsgpu_batch_errors(m_pGpu, 0, pErr) == JSGPU_OK;
        // every event: the first JSGPU_MAX_EVENTS came with pErr, the rest from an events-only walk on the device
        std::vector<jsgpu_scan_event> vErr;
        if (bHaveErr) {
            vErr.assign(pErr->ev, pErr->ev + (pErr->nevents < JSGPU_MAX_EVENTS ? pErr->nevents : JSGPU_MAX_EVENTS));
            if (pErr->nevents > JSGPU_MAX_EVENTS) {
                vErr.resize(pErr->nevents);
                if (jsgpu_batch_error_events(m_pGpu, 0, 0, pErr->nevents, vErr.data()) != JSGPU_OK) {
                    vErr.resize(JSGPU_MAX_EVENTS);
                    m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: GPU scan decoder: error events past the first %u unavailable: %s ***", JSGPU_MAX_EVENTS, jsgpu_last_error(m_pGpu))));
                }
            }
        }
        const unsigned nEv = (unsigned)vErr.size();
        unsigned iEv = 0;
        if (bHaveDet) {
            // every event and matrix, read in pages (the matrices in the order the events name them)
            const unsigned nDet = anDetInfo[0], nBlk = anDetInfo[1], nPage = 4096, nMatPage = 512;
            std::vector<jsgpu_detail_event> vEv(nPage);
            std::vector<int16_t> vMat((size_t)nMatPage * 64);
            unsigned nMatFirst = 0, nMatHave = 0;
            for (unsigned nFirst = 0; nFirst < nDet; nFirst += nPage) {
                const unsigned n = (nDet - nFirst < nPage) ? nDet - nFirst : nPage;
                if (jsgpu_batch_detail_events(m_pGpu, nFirst, n, vEv.data()) != JSGPU_OK) break;
                for (unsigned i = 0; i < n; i++) {
                    const jsgpu_detail_event& e = vEv[i];
                    for (; iEv < nEv && iEv < e.seq; iEv++) { if (vErr[iEv].code == JSGPU_EV_MARKER_NOTE) bMarkerNoteLogged = true; LogScanEvent(vErr[iEv]); }
                    const int16_t* pMat = nullptr;
                    if (e.kind == JSGPU_DT_MATRIX && e.a < nBlk) {
                        if (e.a < nMatFirst || e.a >= nMatFirst + nMatHave) {
                            nMatFirst = e.a; nMatHave = (nBlk - e.a < nMatPage) ? nBlk - e.a : nMatPage;
                            if (jsgpu_batch_detail_matrices(m_pGpu, nMatFirst, nMatHave, vMat.data()) != JSGPU_OK) nMatHave = 0;
                        }
                        if (e.a >= nMatFirst && e.a < nMatFirst + nMatHave) pMat = &vMat[(size_t)(e.a - nMatFirst) * 64];
                    }
                    LogDetailEvent(e, pMat);
                }
            }
        }
        if (bExact) {
            if (bHaveErr) {
                m_bScanBad = pErr->scan_bad != 0;
                for (; iEv < nEv; iEv++) LogScanEvent(vErr[iEv]);
                m_nRestartRead = pErr->restart_read;
                m_nWarnBadScanNum = pErr->warn_num;                 // what the walk counted: kept across decodes while errors are disabled
            } else {
                m_bScanBad = true;
                m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Bad scan data (device status 0x%08X; error events unavailable: %s) ***", lo.status, jsgpu_last_error(m_pGpu))));
            }
        } else {
            // a healthy image walked only for its detailed decode: the walk stops after the printed MCUs; what it met up to there
            // (the end-of-scan marker, when the range reaches the end of the image) has its place among the dump lines
            for (; iEv < nEv; iEv++) { if (vErr[iEv].code == JSGPU_EV_MARKER_NOTE) bMarkerNoteLogged = true; LogScanEvent(vErr[iEv]); }
            if (lo.status) { m_bScanBad = true; m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Bad scan data (device status 0x%08X) ***", lo.status))); }
        }
        delete pErr;
    }
    if (!(lo.status & JSGPU_ST_EXACT)) {
        // A healthy scan still leaves one line behind: topping the accumulator up past the last data byte meets the marker
        // that ends the scan (ref :1527-1543) — EOI normally; anything else also earns an error line there.
        const unsigned nEndMark = (unsigned)st[JSGPU_STAT_END_MARK];
        if (bMarkerNoteLogged) m_nWarnBadScanNum++;
        else if ((unsigned long)nEndMark + 1 < nEof && m_nWarnBadScanNum < m_nScanErrMax) {
            const unsigned nMarker = m_pWBuf->Buf(nEndMark + 1);
            m_pLog->AddLine(JS_LOGSTR(fmt("  Scan Data encountered marker   0xFF%02X @ 0x%08X.0", nMarker, nEndMark)));
            if (nMarker != 0xD9) m_pLog->AddLineErr(JS_LOGSTR("  NOTE: Marker wasn't EOI (0xFFD9)"));
            m_nWarnBadScanNum++;
            if (m_nWarnBadScanNum >= m_nScanErrMax) m_pLog->AddLineErr(JS_LOGSTR(fmt("    Only reported first %u instances of this message...", m_nScanErrMax)));
        }
    }
    const unsigned nEndPos = (unsigned)st[JSGPU_STAT_END_POS], nEndAlign = (unsigned)st[JSGPU_STAT_END_ALIGN];
    m_nEndPos = nEndPos; m_nEndAlign = nEndAlign;
    if (!bQuiet) m_pLog->AddLine(JS_LOGSTR(""));                                    // ref :3630-3632
    if (bDisplay && bPreviewPass) FetchPreviewResults();                           // what CalcChannelPreview left behind (ref :3641-3643)
    else if (bDisplay && m_bDetailVlc) LogDetailRgb(nullptr);
    if (!bQuiet) {
        // ref :3655-3668 compression statistics: bits of scan data consumed up to where the accumulator stands
        m_pLog->AddLine(JS_LOGSTR("  Compression stats:"));
        const float fRatio = (float)(m_nDimX * m_nDimY * m_nNumSosComps * 8) / (float)((nEndPos - nStart) * 8);
        m_pLog->AddLine(JS_LOGSTR(fmt("    Compression Ratio: %5.2f:1", fRatio)));
        const float fBpp = (float)((nEndPos - nStart) * 8) / (float)(m_nDimX * m_nDimY);
        m_pLog->AddLine(JS_LOGSTR(fmt("    Bits per pixel:    %5.2f:1", fBpp)));
        m_pLog->AddLine(JS_LOGSTR(""));
        // ref :3670-3691 code-length histogram (m_anDhtHisto, counted on the device)
        m_pLog->AddLine(JS_LOGSTR("  Huffman code histogram stats:"));
        for (unsigned nClass = DHT_CLASS_DC; nClass <= DHT_CLASS_AC; nClass++)
            for (unsigned nDestId = 0; nDestId <= m_anDhtLookupSetMax[nClass]; nDestId++) {
                unsigned nTotal = 0;
                for (unsigned nLen = 1; nLen <= 16; nLen++) nTotal += m_anDhtHisto[nClass][nDestId][nLen];
                m_pLog->AddLine(JS_LOGSTR(fmt("    Huffman Table: (Dest ID: %u, Class: %s)", nDestId, nClass ? "AC" : "DC")));
                for (unsigned nLen = 1; nLen <= 16; nLen++)
                    m_pLog->AddLine(JS_LOGSTR(fmt("      # codes of length %02u bits: %8u (%3.0f%%)", nLen, m_anDhtHisto[nClass][nDestId][nLen],
                                                   (m_anDhtHisto[nClass][nDestId][nLen] * 100.0) / nTotal)));
                m_pLog->AddLine(JS_LOGSTR(""));
            }
        ReportColorStats();                                      // ref :3692-3693
    }
    if (bDisplay && m_bHistEn) DrawHistogram(bQuiet, bDumpHistoY);  // ref :3700-3703
    if (bDisplay && m_bAvgYValid) {                              // ref :3702-3708 (also in quiet mode)
        m_pLog->AddLine(JS_LOGSTR("  Average Pixel Luminance (Y):"));
        m_pLog->AddLine(JS_LOGSTR(fmt("    Y=[%3u] (range: 0..255)", (unsigned)m_nAvgY)));
        m_pLog->AddLine(JS_LOGSTR(""));
    }
    if (bDisplay && m_bBrightValid) {                            // ref :3710-3718
        m_pLog->AddLine(JS_LOGSTR("  Brightest Pixel Search:"));
        m_pLog->AddLine(JS_LOGSTR(fmt("    YCC=[%5d,%5d,%5d] RGB=[%3u,%3u,%3u] @ MCU[%3u,%3u]", m_nBrightY, m_nBrightCb, m_nBrightCr, m_nBrightR, m_nBrightG, m_nBrightB, m_nBrightMcuX, m_nBrightMcuY)));
        m_pLog->AddLine(JS_LOGSTR(""));
    }
    if (!bQuiet) {                                               // ref :3723-3731
        m_pLog->AddLine(JS_LOGSTR("  Finished Decoding SCAN Data"));
        m_pLog->AddLine(JS_LOGSTR(fmt("    Number of RESTART markers decoded: %u", m_nRestartRead)));
        m_pLog->AddLine(JS_LOGSTR(fmt("    Next position in scan buffer: Offset 0x%08X.%u", nEndPos, nEndAlign)));
        m_pLog->AddLine(JS_LOGSTR(""));
    }
    if (bDisplay && m_bHistEn && bDumpHistoY) ReportHistogramY();   // ref :3740-3742
}

void CimgDecode::LogScanEvent(const jsgpu_scan_event& e)
{
    switch (e.code) {
    case JSGPU_EV_OVERREAD_BEFORE:     m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Overread scan segment (before nCode)! @ Offset: 0x%08X.%u", e.a, e.b))); break;
    case JSGPU_EV_OVERREAD_AFTER_CODE: m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Overread scan segment (after nCode)! @ Offset: 0x%08X.%u", e.a, e.b))); break;
    case JSGPU_EV_OVERREAD_AFTER_BITS: m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Overread scan segment (after bitstring)! @ Offset: 0x%08X.%u", e.a, e.b))); break;
    case JSGPU_EV_NOCODE:              m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Can't find huffman bitstring @ 0x%08X.%u, table %u, value [0x%08x]", e.a, e.b, e.c, e.d))); break;
    case JSGPU_EV_CAP:                 m_pLog->AddLineErr(JS_LOGSTR(fmt("    Only reported first %u instances of this message...", e.a))); break;
    case JSGPU_EV_RST_MISMATCH:        m_pLog->AddLineErr(JS_LOGSTR(fmt("  ERROR: Expected RST marker index RST%u got RST%u @ 0x%08X.0", e.a, e.b, e.c))); break;
    case JSGPU_EV_MARKER_NOTE:
        m_pLog->AddLine(JS_LOGSTR(fmt("  Scan Data encountered marker   0xFF%02X @ 0x%08X.0", e.a, e.b)));
        if (e.a != 0xD9) m_pLog->AddLineErr(JS_LOGSTR("  NOTE: Marker wasn't EOI (0xFFD9)"));
        break;
    case JSGPU_EV_BADMARK:             m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Bad marker @ 0x%08X.%u", e.a, e.b))); break;
    case JSGPU_EV_BADCODE:             m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Bad huffman code @ 0x%08X.%u", e.a, e.b))); break;
    case JSGPU_EV_NCOEF:               m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: @ 0x%08X.%u, nNumCoeffs>64 [%u]", e.a, e.b, e.c))); break;
    case JSGPU_EV_MCU: {
        const unsigned nComp = e.c & 0xFF, nCssH = (e.c >> 8) & 0xFF, nCssV = (e.c >> 16) & 0xFF;
        std::string strComp = fmt(nComp == 0 ? "Lum CSS(%u,%u)" : nComp == 1 ? "Chr(Cb) CSS(%u,%u)" : "Chr(Cr) CSS(%u,%u)", nCssH, nCssV);
        m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: Bad scan data in MCU(%u,%u): %s @ Offset 0x%08X.%u", e.a, e.b, strComp.c_str(), e.d, e.e)));
        m_pLog->AddLineErr(JS_LOGSTR(fmt("           MCU located at pixel=(%u,%u)", m_nMcuWidth * e.a + nCssH * 8, m_nMcuHeight * e.b + nCssV * 8)));
        break; }
    case JSGPU_EV_RST_MISSING:
        m_pLog->AddLine(JS_LOGSTR(fmt("  Expect Restart interval elapsed @ 0x%08X.%u", e.a, e.b)));
        m_pLog->AddLineErr(JS_LOGSTR("    ERROR: Restart marker not detected"));
        break;
    default: break;
    }
}

// ---- "Detailed Decode" (ref :1859-2232, 4880-4904) -----------------------------------------------------------------------------
void CimgDecode::SetDetailVlc(bool bDetail, unsigned nX, unsigned nY, unsigned nLen) { m_bDetailVlc = bDetail; m_nDetailVlcX = nX; m_nDetailVlcY = nY; m_nDetailVlcLen = nLen; }
void CimgDecode::GetDetailVlc(bool& bDetail, unsigned& nX, unsigned& nY, unsigned& nLen) { bDetail = m_bDetailVlc; nX = m_nDetailVlcX; nY = m_nDetailVlcY; nLen = m_nDetailVlcLen; }

void CimgDecode::LogDetailEvent(const jsgpu_detail_event& e, const int16_t* pMatrix)
{
    switch (e.kind) {
    case JSGPU_DT_MCU: m_pLog->AddLine(JS_LOGSTR("")); break;                                          // ref :3249-3251
    case JSGPU_DT_BLOCK: {                                                                             // ref :1873-1889
        const char* szTbl = e.a == 0 ? "Lum" : e.a == 1 ? "Chr(0)" : e.a == 2 ? "Chr(1)" : "???";
        m_pLog->AddLine(JS_LOGSTR(fmt("    %s (Tbl #%u), MCU=[%u,%u]", szTbl, e.a, e.b, e.c)));
        break; }
    case JSGPU_DT_VLC: {                                                                               // ReportVlc, ref :2152-2232
        const unsigned nVlcPos = e.a, nVlcAlign = e.b, nZrl = e.c, nCoeffStart = e.e & 0xFF, nCoeffEnd = (e.e >> 8) & 0xFF, nBits = e.e >> 16;
        const int nVal = (int)(short)e.d;
        // the four data bytes from the file position on, stuffed zeros skipped the way the reference's look-back does
        unsigned nBufByte[4]; unsigned nInd = nVlcPos;
        const unsigned nPre = m_pWBuf->Buf(nInd - 1);
        nBufByte[0] = m_pWBuf->Buf(nInd++);
        if (nPre == 0xFF && nBufByte[0] == 0x00) nBufByte[0] = m_pWBuf->Buf(nInd++);
        for (unsigned k = 1; k < 4; k++) {
            nBufByte[k] = m_pWBuf->Buf(nInd++);
            if (nBufByte[k - 1] == 0xFF && nBufByte[k] == 0x00) nBufByte[k] = m_pWBuf->Buf(nInd++);
        }
        std::string strBytes;
        for (unsigned k = 0; k < 4; k++) for (int bit = 7; bit >= 0; bit--) strBytes += ((nBufByte[k] >> bit) & 1) ? '1' : '0';
        std::string strBin(nVlcAlign < 32 ? nVlcAlign : 32, '-');
        if (nVlcAlign < 32) strBin += strBytes.substr(nVlcAlign, nBits);
        for (unsigned i = nVlcAlign + nBits; i < 32; i++) strBin += '-';
        for (unsigned at : { 24u, 16u, 8u }) if (strBin.size() >= at) strBin.insert(at, " "); else strBin += " ";
        const std::string strData = fmt("0x %02X %02X %02X %02X = 0b (%s)", nBufByte[0], nBufByte[1], nBufByte[2], nBufByte[3], strBin.c_str());
        static const char* const kSpecial[4] = { "", "EOB", "ERROR", "EOB64" };
        if (nCoeffStart == 0 && nCoeffEnd == 0)
            m_pLog->AddLine(JS_LOGSTR(fmt("      [0x%08X.%u]: ZRL=[%2u] Val=[%5d] Coef=[%02u= DC] Data=[%s] %s", nVlcPos, nVlcAlign, nZrl, nVal, nCoeffStart, strData.c_str(), kSpecial[e.f & 3])));
        else
            m_pLog->AddLine(JS_LOGSTR(fmt("      [0x%08X.%u]: ZRL=[%2u] Val=[%5d] Coef=[%02u..%02u] Data=[%s] %s", nVlcPos, nVlcAlign, nZrl, nVal, nCoeffStart, nCoeffEnd, strData.c_str(), kSpecial[e.f & 3])));
        break; }
    case JSGPU_DT_MATRIX: {                                                                            // ReportDctMatrix, ref :2104-2131
        if (!pMatrix) break;
        for (unsigned nY = 0; nY < 8; nY++) {
            std::string strLine = nY == 0 ? "                      DCT Matrix=[" : "                                 [";
            for (unsigned nX = 0; nX < 8; nX++) { strLine += fmt("%5d", (int)pMatrix[nY * 8 + nX]); if (nX != 7) strLine += " "; }
            strLine += "]";
            m_pLog->AddLine(JS_LOGSTR(strLine));
        }
        m_pLog->AddLine(JS_LOGSTR(""));
        break; }
    default: break;
    }
}

// ---- channel preview, colour statistics, histograms (SURVEY.md §8f N3/N4) --------------------------------------------------
void CimgDecode::PreviewSettings(jsgpu_preview& pv) const
{
    memset(&pv, 0, sizeof pv);
    pv.hist_en = m_bHistEn ? 1 : 0; pv.statclip_en = m_bStatClipEn ? 1 : 0;
    pv.mode = (int32_t)m_nPreviewMode;
    if (pv.mode < 1 || pv.mode > 8) pv.mode = 1;                    // ChannelExtract's final else (ref :4869-4873); PREVIEW_NONE too
    pv.shift_y = m_nPreviewShiftY; pv.shift_cb = m_nPreviewShiftCb; pv.shift_cr = m_nPreviewShiftCr;
    pv.shift_mcu_x = m_nPreviewShiftMcuX; pv.shift_mcu_y = m_nPreviewShiftMcuY;
    pv.ycc_warn_budget = m_nWarnYccClipNum < JSGPU_MAX_YCC_WARN ? JSGPU_MAX_YCC_WARN - m_nWarnYccClipNum : 0;
    pv.detail_en = m_bDetailVlc ? 1u : 0u; pv.detail_mcu_x = m_nDetailVlcX; pv.detail_mcu_y = m_nDetailVlcY;
}

void CimgDecode::SetPreviewMode(unsigned nMode) { m_nPreviewMode = nMode; CalcChannelPreview(); }             // ref :631-639
void CimgDecode::SetPreviewYccOffset(unsigned nMcuX, unsigned nMcuY, int nY, int nCb, int nCr)                  // ref :650-659
{
    m_nPreviewShiftY = nY; m_nPreviewShiftCb = nCb; m_nPreviewShiftCr = nCr;
    m_nPreviewShiftMcuX = nMcuX; m_nPreviewShiftMcuY = nMcuY;
    CalcChannelPreview();
}
void CimgDecode::GetPreviewYccOffset(unsigned& nMcuX, unsigned& nMcuY, int& nY, int& nCb, int& nCr)
{
    nY = m_nPreviewShiftY; nCb = m_nPreviewShiftCb; nCr = m_nPreviewShiftCr; nMcuX = m_nPreviewShiftMcuX; nMcuY = m_nPreviewShiftMcuY;
}

// ref :4967-4990.  No DIB, nothing to do (as there); otherwise the device recomputes it from the pixel maps it still holds.
void CimgDecode::CalcChannelPreview()
{
    if (!m_pDibBits || !m_pGpu || !m_bDecodedOnDevice) return;
    jsgpu_preview pv; PreviewSettings(pv);
    int r = jsgpu_batch_preview(m_pGpu, &pv);
    if (r != JSGPU_OK) {
        m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: GPU channel preview failed: %s (%s) ***", jsgpu_strerror(r), jsgpu_last_error(m_pGpu))));
        return;
    }
    FetchPreviewResults();
}

void CimgDecode::FetchPreviewResults()
{
    const size_t nPix = (size_t)m_nImgSizeX * m_nImgSizeY;
    jsgpu_batch_download(m_pGpu, JSGPU_OUT_DIB, 0, m_pDibBits, nPix * 4);
    int32_t st[JSGPU_STAT_WORDS]; memset(st, 0, sizeof st);
    jsgpu_batch_download(m_pGpu, JSGPU_OUT_STATS, 0, st, sizeof st);
    m_nAvgY = st[JSGPU_STAT_AVGY]; m_bAvgYValid = true;             // ref :4813-4819; the brightest pixel does not depend on the settings
    m_bBrightValid = true;
    jsgpu_colour_stats* cs = new jsgpu_colour_stats;
    if (jsgpu_batch_colour_stats(m_pGpu, 0, cs) == JSGPU_OK) {
        // CalcChannelPreviewFull does not clear the statistics (only DecodeScanImg does, ref :3144-3156): every pass adds to them
        for (unsigned k = 0; k < 12; k++) {
            m_anStatClip[k] += cs->clip[k];
            if (cs->vmin[k] < m_anHistoMin[k]) m_anHistoMin[k] = cs->vmin[k];
            if (cs->vmax[k] > m_anHistoMax[k]) m_anHistoMax[k] = cs->vmax[k];
            m_anHistoSum[k] = (int)((unsigned)m_anHistoSum[k] + (unsigned)(unsigned long long)cs->vsum[k]);     // the reference's sums are `int`
        }
        m_nHistoCount += (unsigned)cs->count;
        for (unsigned c = 0; c < 3; c++) for (unsigned i = 0; i < JSGPU_CC_HISTO_BINS; i++) m_anCcHisto[c][i] += cs->cc_histo[c][i];
        for (unsigned i = 0; i < JSGPU_Y_HISTO_BINS; i++) m_anHistoYFull[i] += cs->y_histo[i];
        if (m_bDetailVlc) LogDetailRgb(cs);                            // the notes, with the RGB dump lines in between
        else for (unsigned i = 0; i < cs->nwarn && i < JSGPU_MAX_YCC_WARN; i++) LogYccNote(cs->warn[i]);
    } else if (m_bDetailVlc) LogDetailRgb(nullptr);
    delete cs;
}

// The reference builds the array from the DIB it displays (whatever the preview mode shows) or from the pixel maps (:2098-2170).
bool CimgDecode::ExportTiffData(unsigned nMode, std::vector<unsigned char>& data)
{
    if (nMode > 2 || !m_pDibBits || !m_pGpu || !m_bDecodedOnDevice) return false;
    if (nMode == 2 && m_nNumSosComps != NUM_CHAN_YCC) return false;           // the reference dereferences all three pixel maps
    data.assign((size_t)m_nImgSizeX * m_nImgSizeY * (nMode == 1 ? 6 : 3), 0);
    const int r = jsgpu_batch_export(m_pGpu, 0, (int)nMode, data.data(), data.size());
    if (r != JSGPU_OK) { m_pLog->AddLineErr(JS_LOGSTR(fmt("*** ERROR: GPU export failed: %s (%s) ***", jsgpu_strerror(r), jsgpu_last_error(m_pGpu)))); return false; }
    return true;
}
bool CimgDecode::ExportTiff(const char* szFnameOut, unsigned nMode)
{
    std::vector<unsigned char> data;
    if (!szFnameOut || !ExportTiffData(nMode, data)) return false;
    FileTiff myTiff;
    return myTiff.WriteFile(szFnameOut, nMode == 2, nMode == 1, data.data(), m_nImgSizeX, m_nImgSizeY);
}

// CapYccRange's notes (ref :4366-4466)
void CimgDecode::LogYccNote(const jsgpu_ycc_warn& w)
{
    static const char* const kKind[6] = { "Y Underflow", "Y Overflow", "Cb Underflow", "Cb Overflow", "Cr Underflow", "Cr Overflow" };
    m_pLog->AddLineWarn(JS_LOGSTR(fmt("*** NOTE: YCC Clipped. MCU=(%4u,%4u) YCC=(%5d,%5d,%5d) %s @ Offset 0x%08X.%u",
                                      w.mcu_x, w.mcu_y, w.y, w.cb, w.cr, kKind[w.kind < 6 ? w.kind : 0], m_nEndPos, m_nEndAlign)));
    m_nWarnYccClipNum++;
    if (m_nWarnYccClipNum == JSGPU_MAX_YCC_WARN)
        m_pLog->AddLineWarn(JS_LOGSTR(fmt("    Only reported first %u instances of this message...", (unsigned)JSGPU_MAX_YCC_WARN)));
}

// ref :4683-4687, 4757-4780, 4797-4799: header, one line per pixel row of MCU (m_nDetailVlcX, m_nDetailVlcY) — written when the raster
// walk leaves the MCU's columns, so a row at the right edge closes on the first pixel of the next row, and the last such row never
// does — then a blank line.  The "YCC Clipped" notes of the same pass appear where the walk met them.
void CimgDecode::LogDetailRgb(const jsgpu_colour_stats* cs)
{
    m_pLog->AddLine(JS_LOGSTR("  Detailed IDCT Dump (RGB):"));
    m_pLog->AddLine(JS_LOGSTR(fmt("    MCU [%3u,%3u]:", m_nDetailVlcX, m_nDetailVlcY)));
    const unsigned W = m_nImgSizeX, H = m_nImgSizeY;
    const unsigned nNotes = cs ? (cs->nwarn < JSGPU_MAX_YCC_WARN ? cs->nwarn : JSGPU_MAX_YCC_WARN) : 0;
    unsigned iNote = 0;
    // the triplet is the pixel BEFORE ChannelExtract (ref :4757-4764): the preview pass kept it for this MCU; without a pass (default
    // settings) the DIB holds exactly it
    const bool bRgbInDib = (cs == nullptr);
    const unsigned long long x0 = (unsigned long long)m_nDetailVlcX * m_nMcuWidth, x1 = x0 + m_nMcuWidth;
    const unsigned long long y0 = (unsigned long long)m_nDetailVlcY * m_nMcuHeight;
    if (x0 < W) for (unsigned long long py = y0; py < y0 + m_nMcuHeight && py < H; py++) {
        const unsigned long long nClose = py * W + (x1 < W ? x1 : W);          // raster index of the pixel that closes this row
        if (nClose >= (unsigned long long)W * H || (nClose / W) / m_nMcuHeight != m_nDetailVlcY) break;   // never closed: not logged
        for (; iNote < nNotes && (unsigned long long)cs->warn[iNote].py * W + cs->warn[iNote].px <= nClose; iNote++) LogYccNote(cs->warn[iNote]);
        std::string strLine = "      [ ";
        for (unsigned long long px = x0; px < x1 && px < W; px++) {
            unsigned nR, nG, nB;
            if (bRgbInDib) { const unsigned char* q = m_pDibBits + ((size_t)(H - 1 - py) * W + px) * 4; nR = q[2]; nG = q[1]; nB = q[0]; }
            else { const unsigned v = cs->detail_rgb[py - y0][px - x0]; nR = (v >> 16) & 0xFF; nG = (v >> 8) & 0xFF; nB = v & 0xFF; }
            strLine += fmt("x%02X%02X%02X ", nR, nG, nB);
        }
        strLine += " ]";
        m_pLog->AddLine(JS_LOGSTR(strLine));
    }
    for (; iNote < nNotes; iNote++) LogYccNote(cs->warn[iNote]);
    m_pLog->AddLine(JS_LOGSTR(""));
}

void CimgDecode::GetHistoRanges(int out[36], unsigned& nCount) const
{
    // PixelCcHisto's order (ImgDecode.h:236-280): pre-ranged YCC, ranged YCC, CLIPPED RGB, pre-clip RGB
    static const int kOrder[12] = { 0, 1, 2, 3, 4, 5, 9, 10, 11, 6, 7, 8 };
    for (int k = 0; k < 12; k++) { out[k * 3] = m_anHistoMin[kOrder[k]]; out[k * 3 + 1] = m_anHistoMax[kOrder[k]]; out[k * 3 + 2] = m_anHistoSum[kOrder[k]]; }
    nCount = m_nHistoCount;
}

// ref :3764-3837
void CimgDecode::ReportColorStats()
{
    static const char* const kYcc[3] = { "Y ", "Cb", "Cr" };
    static const char* const kRgb[3] = { "R ", "G ", "B " };
    m_pLog->AddLine(JS_LOGSTR("  YCC clipping in DC:"));
    for (unsigned c = 0; c < 3; c++) m_pLog->AddLine(JS_LOGSTR(fmt("    %s component: [<0=%5u] [>255=%5u]", kYcc[c], m_anStatClip[c * 2], m_anStatClip[c * 2 + 1])));
    m_pLog->AddLine(JS_LOGSTR(""));
    if (m_bHistEn) {
        struct { const char* title; const char* const* names; unsigned first; } blocks[3] = {
            { "  YCC histogram in DC (DCT sums : pre-ranged:", kYcc, 0 }, { "  YCC histogram in DC:", kYcc, 3 }, { "  RGB histogram in DC (before clip):", kRgb, 6 } };
        for (auto& bl : blocks) {
            m_pLog->AddLine(JS_LOGSTR(bl.title));
            for (unsigned c = 0; c < 3; c++)
                m_pLog->AddLine(JS_LOGSTR(fmt("    %s component histo: [min=%5d max=%5d avg=%7.1f]", bl.names[c], m_anHistoMin[bl.first + c], m_anHistoMax[bl.first + c],
                                              (float)m_anHistoSum[bl.first + c] / (float)m_nHistoCount)));
            m_pLog->AddLine(JS_LOGSTR(""));
        }
    }
    m_pLog->AddLine(JS_LOGSTR("  RGB clipping in DC:"));
    for (unsigned c = 0; c < 3; c++) m_pLog->AddLine(JS_LOGSTR(fmt("    %s component: [<0=%5u] [>255=%5u]", kRgb[c], m_anStatClip[6 + c * 2], m_anStatClip[6 + c * 2 + 1])));
    m_pLog->AddLine(JS_LOGSTR(""));
}

// ref :3846-3859
void CimgDecode::ReportHistogramY()
{
    m_pLog->AddLine(JS_LOGSTR("  Y Histogram in DC: (DCT sums) Full"));
    for (unsigned row = 0; row < JSGPU_Y_HISTO_BINS / 8; row++) {
        std::string strFull = fmt("    Y=%5d..%5d: ", -1024 + (int)(row * 8), -1024 + (int)(row * 8) + 7);
        for (unsigned col = 0; col < 8; col++) strFull += fmt("0x%06x, ", m_anHistoYFull[col + row * 8]);
        m_pLog->AddLine(JS_LOGSTR(strFull));
    }
}

// ref :3870-4012: the after-clip RGB ranges, then the two histogram bitmaps (bars of HISTO_BIN_HEIGHT_MAX = 30 rows, one pixel
// per bin: 128 x 90 for R/G/B stacked, 512 x 30 for the luminance sums taken four bins at a time)
void CimgDecode::DrawHistogram(bool bQuiet, bool bDumpHistoY)
{
    if (!bQuiet) {
        static const char* const kRgb[3] = { "R ", "G ", "B " };
        m_pLog->AddLine(JS_LOGSTR("  RGB histogram in DC (after clip):"));
        for (unsigned c = 0; c < 3; c++)
            m_pLog->AddLine(JS_LOGSTR(fmt("    %s component histo: [min=%5d max=%5d avg=%7.1f]", kRgb[c], m_anHistoMin[9 + c], m_anHistoMax[9 + c],
                                          (float)m_anHistoSum[9 + c] / (float)m_nHistoCount)));
        m_pLog->AddLine(JS_LOGSTR(""));
    }
    const unsigned kBarMax = 30, kSubset = 512;
    m_pDibHistRgb.Kill(); m_bDibHistRgbReady = false;
    m_pDibHistRgb.CreateDIB(JSGPU_CC_HISTO_BINS, 3 * kBarMax, 32);
    if (unsigned char* pBits = (unsigned char*)m_pDibHistRgb.GetDIBBitArray()) {
        const unsigned nRowBytes = JSGPU_CC_HISTO_BINS * 4;
        memset(pBits, 0, (size_t)3 * kBarMax * nRowBytes);
        unsigned nPeak = 1;                                          // across all three channels (ref :3912-3926)
        for (unsigned c = 0; c < 3; c++) for (unsigned i = 0; i < JSGPU_CC_HISTO_BINS; i++) if (m_anCcHisto[c][i] > nPeak) nPeak = m_anCcHisto[c][i];
        for (unsigned c = 0; c < 3; c++) for (unsigned i = 0; i < JSGPU_CC_HISTO_BINS; i++) {
            const unsigned nHeight = kBarMax * m_anCcHisto[c][i] / nPeak;          // 32-bit product, like the reference's
            for (unsigned y = 0; y < nHeight; y++) {
                unsigned char* px = pBits + (size_t)i * 4 + (size_t)((2 - c) * kBarMax + y) * nRowBytes;
                px[3] = 0; px[2] = (c == 0) ? 255 : 0; px[1] = (c == 1) ? 255 : 0; px[0] = (c == 2) ? 255 : 0;
            }
        }
        m_bDibHistRgbReady = true;
    }
    m_bDibHistYReady = false;
    if (bDumpHistoY) {
        m_pDibHistY.Kill();
        m_pDibHistY.CreateDIB(kSubset, kBarMax, 32);
        if (unsigned char* pBits = (unsigned char*)m_pDibHistY.GetDIBBitArray()) {
            const unsigned nRowBytes = kSubset * 4;
            memset(pBits, 0, (size_t)kBarMax * nRowBytes);
            unsigned nPeak = 1;
            for (unsigned i = 0; i < kSubset; i++) { const unsigned v = m_anHistoYFull[i * 4] + m_anHistoYFull[i * 4 + 1] + m_anHistoYFull[i * 4 + 2] + m_anHistoYFull[i * 4 + 3]; if (v > nPeak) nPeak = v; }
            for (unsigned i = 0; i < kSubset; i++) {
                const unsigned v = m_anHistoYFull[i * 4] + m_anHistoYFull[i * 4 + 1] + m_anHistoYFull[i * 4 + 2] + m_anHistoYFull[i * 4 + 3];
                const unsigned nHeight = kBarMax * v / nPeak;
                for (unsigned y = 0; y < nHeight; y++) { unsigned char* px = pBits + (size_t)i * 4 + (size_t)y * nRowBytes; px[3] = 0; px[2] = 255; px[1] = 255; px[0] = 0; }
            }
            m_bDibHistYReady = true;
        }
    }
}

bool CimgDecode::IsPreviewReady() { return m_bPreviewIsJpeg; }
void CimgDecode::ResetImageContent() {}                       // ref :603-605

// ---- getters ----------------------------------------------------------------------------------
void CimgDecode::GetPixMapPtrs(short*& pMapY, short*& pMapCb, short*& pMapCr) { pMapY = m_pPixValY; pMapCb = m_pPixValCb; pMapCr = m_pPixValCr; }
void CimgDecode::GetImageSize(unsigned& nX, unsigned& nY) { nX = m_nImgSizeX; nY = m_nImgSizeY; }
void CimgDecode::GetBitmapPtr(unsigned char*& pBitmap)          // ref :4940: the bits of m_pDibTemp — which a JPEG scan keeps in m_pDibBits here
{ pBitmap = (m_bDibTempReady && !m_bPreviewIsJpeg) ? (unsigned char*)m_pDibTemp.GetDIBBitArray() : m_pDibBits; }
unsigned CimgDecode::PackFileOffset(unsigned nByte, unsigned nBit) { return (nByte << 4) + nBit; }
void CimgDecode::UnpackFileOffset(unsigned nPacked, unsigned& nByte, unsigned& nBit) { nBit = nPacked & 0x7; nByte = nPacked >> 4; }
void CimgDecode::LookupFilePosPix(unsigned nPixX, unsigned nPixY, unsigned& nByte, unsigned& nBit)
{
    nByte = nBit = 0;
    if (!m_pMcuFileMap) return;
    unsigned nMcuX = nPixX / m_nMcuWidth, nMcuY = nPixY / m_nMcuHeight;
    if (nMcuX >= m_nMcuXMax || nMcuY >= m_nMcuYMax) return;
    UnpackFileOffset(m_pMcuFileMap[nMcuX + nMcuY * m_nMcuXMax], nByte, nBit);
}
void CimgDecode::LookupFilePosMcu(unsigned nMcuX, unsigned nMcuY, unsigned& nByte, unsigned& nBit)
{
    nByte = nBit = 0;
    if (!m_pMcuFileMap || nMcuX >= m_nMcuXMax || nMcuY >= m_nMcuYMax) return;
    UnpackFileOffset(m_pMcuFileMap[nMcuX + nMcuY * m_nMcuXMax], nByte, nBit);
}
void CimgDecode::LookupBlkYCC(unsigned nBlkX, unsigned nBlkY, int& nY, int& nCb, int& nCr)
{
    nY = nCb = nCr = 0;
    if (!m_pBlkDcValY || nBlkX >= m_nBlkXMax || nBlkY >= m_nBlkYMax) return;
    nY = m_pBlkDcValY[nBlkX + nBlkY * m_nBlkXMax];
    if (m_nNumSosComps == NUM_CHAN_YCC) { nCb = m_pBlkDcValCb[nBlkX + nBlkY * m_nBlkXMax]; nCr = m_pBlkDcValCr[nBlkX + nBlkY * m_nBlkXMax]; }
}
void CimgDecode::GetGeometry(unsigned o[8]) const
{ o[0] = m_nMcuWidth; o[1] = m_nMcuHeight; o[2] = m_nMcuXMax; o[3] = m_nMcuYMax; o[4] = m_nBlkXMax; o[5] = m_nBlkYMax; o[6] = m_nImgSizeX; o[7] = m_nImgSizeY; }
bool CimgDecode::GetBrightest(int& nY, int& nCb, int& nCr, unsigned& nR, unsigned& nG, unsigned& nB, unsigned& nMcuX, unsigned& nMcuY) const
{ nY = m_nBrightY; nCb = m_nBrightCb; nCr = m_nBrightCr; nR = m_nBrightR; nG = m_nBrightG; nB = m_nBrightB; nMcuX = m_nBrightMcuX; nMcuY = m_nBrightMcuY; return m_bBrightValid; }
