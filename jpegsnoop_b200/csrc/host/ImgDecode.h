// ImgDecode.h — host side of the H100 scan decoder: class CimgDecode with the public surface of
// the reference class (reference: source/ImgDecode.h:284-425) so that CjfifDecode can drive it
// unchanged: the table/geometry setters it calls (JfifDecode.cpp:3577-3600, 4648, 5008-5025, 5161,
// 5291), DecodeScanImg (JfifDecode.cpp:5299) and the getters the rest of JPEGsnoop reads results
// through (JPEGsnoopCore.cpp:1211-1398).  The scan itself is decoded on the GPU through the
// C-ABI in include/jsgpu.h; this class only keeps tables, validates, ships bytes and owns the
// host copies of the results.  GUI members of the reference class (ViewOnDraw, zoom, overlays,
// status bar, histogram drawing: ImgDecode.h:296-298, 319-329, 346-349, 419-425) are outside
// the hot path and are not part of this class (SURVEY.md §2 row 1).
#pragma once
#include <vector>
// Two build modes.  Stand-alone (default): HostCompat.h supplies small stand-ins for CDocLog / CwindowBuf / CSnoopConfig /
// CDIB.  Inside JPEGsnoop (-DJSGPU_HOST_EXTERNAL_TYPES): the application's own DocLog.h, WindowBuf.h, SnoopConfig.h and
// Dib.h are used — this is how oracle/Makefile's `n1` target compiles the reference's unmodified CjfifDecode against this
// class (INTEGRATION.md §1a).
#ifdef JSGPU_HOST_EXTERNAL_TYPES
#include "stdafx.h"
#include "DocLog.h"
#include "WindowBuf.h"
#include "SnoopConfig.h"
#include "Dib.h"
#include "jsgpu.h"                 // found through -I<repo>/include (the application's build decides the include paths)
#else
#include "HostCompat.h"
#include "../../../include/jsgpu.h"
#endif
#include <string>

// Limits and indices — same meaning as the reference's (ImgDecode.h:62-106)
#ifndef MAX_DHT_CLASS
#define MAX_DHT_CLASS     2
#endif
#ifndef MAX_DHT_DEST_ID
#define MAX_DHT_DEST_ID   4
#endif
#ifndef DHT_CLASS_DC
#define DHT_CLASS_DC      0
#endif
#ifndef DHT_CLASS_AC
#define DHT_CLASS_AC      1
#endif
#ifndef MAX_DHT_CODES
#define MAX_DHT_CODES     260
#endif
#ifndef MAX_DQT_DEST_ID
#define MAX_DQT_DEST_ID   4
#endif
#ifndef MAX_DQT_COEFF
#define MAX_DQT_COEFF     64
#endif
#ifndef MAX_DQT_COMP
#define MAX_DQT_COMP      256
#endif
#ifndef MAX_SOF_COMP_NF
#define MAX_SOF_COMP_NF   256
#endif
#ifndef MAX_SOS_COMP_NS
#define MAX_SOS_COMP_NS   4
#endif
#ifndef MAX_SAMP_FACT_H
#define MAX_SAMP_FACT_H   4
#endif
#ifndef MAX_SAMP_FACT_V
#define MAX_SAMP_FACT_V   4
#endif
#ifndef NUM_CHAN_GRAYSCALE
#define NUM_CHAN_GRAYSCALE 1
#endif
#ifndef NUM_CHAN_YCC
#define NUM_CHAN_YCC      3
#endif
#ifndef DCT_SZ_ALL
#define DCT_SZ_ALL        64
#endif

// ... and the ones the reference's OTHER translation units take from ImgDecode.h (JfifDecode.cpp:3465, 4959-4965, 7477)
#ifndef MAX_DHT_CODELEN
#define MAX_DHT_CODELEN   16      // ImgDecode.h:67
#endif
#ifndef SCAN_COMP_Y
#define SCAN_COMP_Y       1       // ImgDecode.h:112-114: component indices of a YCC scan
#define SCAN_COMP_CB      2
#define SCAN_COMP_CR      3
#endif

class CimgDecode
{
public:
    CimgDecode(CDocLog* pLog, CwindowBuf* pWBuf, CSnoopConfig* pConfig = nullptr);
    ~CimgDecode();
    CimgDecode(const CimgDecode&) = delete;
    CimgDecode& operator=(const CimgDecode&) = delete;

    void        Reset();        // start of an SOS decode        (ref ImgDecode.cpp:49-138)
    void        ResetState();   // start of a new JFIF decode    (ref :286-306)

    void        DecodeScanImg(unsigned nStart, bool bDisplay, bool bQuiet);      // ref :2723-3745
    bool        IsPreviewReady();                                                // ref :3753

    // Config — called by the marker parser
    void        SetImageDimensions(unsigned nWidth, unsigned nHeight);           // ref :2706
    void        SetImageDetails(unsigned nDimX, unsigned nDimY, unsigned nCompsSOF, unsigned nCompsSOS, bool bRstEn, unsigned nRstInterval); // ref :590
    void        SetSofSampFactors(unsigned nCompInd, unsigned nSampFactH, unsigned nSampFactV);  // ref :619
    bool        SetDqtEntry(unsigned nTblDestId, unsigned nCoeffInd, unsigned nCoeffIndZz, unsigned short nCoeffVal); // ref :424
    bool        SetDqtTables(unsigned nCompInd, unsigned nTbl);                  // ref :505
    unsigned    GetDqtEntry(unsigned nTblDestId, unsigned nCoeffInd);            // ref :466
    bool        SetDhtTables(unsigned nCompInd, unsigned nTblDc, unsigned nTblAc); // ref :536
    bool        SetDhtEntry(unsigned nDestId, unsigned nClass, unsigned nInd, unsigned nLen,
                            unsigned nBits, unsigned nMask, unsigned nCode);     // ref :748
    bool        SetDhtSize(unsigned nDestId, unsigned nClass, unsigned nSize);   // ref :834
    void        SetPrecision(unsigned nPrecision);                               // ref :564

    // Utilities
    void        LookupFilePosPix(unsigned nPixX, unsigned nPixY, unsigned& nByte, unsigned& nBit);   // ref :5001
    void        LookupFilePosMcu(unsigned nMcuX, unsigned nMcuY, unsigned& nByte, unsigned& nBit);   // ref :5020
    void        LookupBlkYCC(unsigned nBlkX, unsigned nBlkY, int& nY, int& nCb, int& nCr);           // ref :5037
    void        GetImageSize(unsigned& nX, unsigned& nY);                                            // ref :4929
    void        GetPixMapPtrs(short*& pMapY, short*& pMapCb, short*& pMapCr);                        // ref :4913
    void        GetBitmapPtr(unsigned char*& pBitmap);                                               // ref :4940
    unsigned    PackFileOffset(unsigned nByte, unsigned nBit);                                       // ref :5104
    void        UnpackFileOffset(unsigned nPacked, unsigned& nByte, unsigned& nBit);                 // ref :5123
    void        ScanErrorsDisable();                                                                 // ref :1014
    void        ScanErrorsEnable();                                                                  // ref :1026
    void        ResetImageContent();                                                                 // ref :603 (empty there too)
    // Channel preview (SURVEY.md §8f N3/N4): each setter recomputes the DIB on the device (CalcChannelPreview, ref :4967-4990)
    void        SetPreviewMode(unsigned nMode);                                                      // ref :631
    unsigned    GetPreviewMode() const { return m_nPreviewMode; }                                    // ref :600
    void        SetPreviewYccOffset(unsigned nMcuX, unsigned nMcuY, int nY, int nCb, int nCr);       // ref :650
    void        GetPreviewYccOffset(unsigned& nMcuX, unsigned& nMcuY, int& nY, int& nCb, int& nCr);  // ref :669
    void        ReportColorStats();                                                                  // ref :3764
    void        ReportHistogramY();                                                                  // ref :3846
    void        DrawHistogram(bool bQuiet, bool bDumpHistoY);                                        // ref :3870
    // "Detailed Decode": every Huffman symbol and coefficient matrix of nLen MCUs from (nX,nY) goes to the log (ref :4880-4904)
    void        SetDetailVlc(bool bDetail, unsigned nX, unsigned nY, unsigned nLen);
    void        GetDetailVlc(bool& bDetail, unsigned& nX, unsigned& nY, unsigned& nLen);
    // Export-to-TIFF (CJPEGsnoopDoc::OnToolsExporttiff, JPEGsnoopDoc.cpp:2008-2193): nMode 0 RGB 8-bit, 1 RGB 16-bit, 2 YCC 8-bit
    // (the dialog's m_nCtlFmt); the sample array is packed on the device.  ExportTiffData fills the pixel part only.
    bool        ExportTiff(const char* szFnameOut, unsigned nMode);
    bool        ExportTiffData(unsigned nMode, std::vector<unsigned char>& data);
    void        SetStatusBar(void* /* CStatusBar* */) {}                                              // ref ImgDecode.h:296: GUI only

    // Results the reference keeps in private members and reports in its log (ref :3659-3720);
    // exposed read-only so callers and tests do not need `friend` access.
    const unsigned* GetMcuFileMap() const { return m_pMcuFileMap; }
    const short*    GetBlkDcMap(unsigned nChan) const { return nChan == 0 ? m_pBlkDcValY : nChan == 1 ? m_pBlkDcValCb : m_pBlkDcValCr; }
    const unsigned* GetDhtHisto() const { return &m_anDhtHisto[0][0][0]; }
    void        GetGeometry(unsigned out[8]) const;
    bool        GetScanBad() const { return m_bScanBad; }
    unsigned    GetScanStatus() const { return m_nScanStatus; }
    unsigned    GetRestartRead() const { return m_nRestartRead; }
    bool        GetBrightest(int& nY, int& nCb, int& nCr, unsigned& nR, unsigned& nG, unsigned& nB, unsigned& nMcuX, unsigned& nMcuY) const;
    bool        GetAvgY(long& nAvgY) const { nAvgY = m_nAvgY; return m_bAvgYValid; }
    // m_sStatClip (12 counters, PixelCcClip order), m_sHisto as [12 channels][min,max,sum] in PixelCcHisto's order of appearance
    // (pre-ranged YCC, ranged YCC, clipped RGB, pre-clip RGB) + nCount, m_anCcHisto_r/g/b, m_anHistoYFull
    const unsigned* GetStatClip() const { return m_anStatClip; }
    void        GetHistoRanges(int out[36], unsigned& nCount) const;
    const unsigned* GetCcHisto(unsigned nChan) const { return m_anCcHisto[nChan < 3 ? nChan : 0]; }
    const unsigned* GetHistoYFull() const { return m_anHistoYFull; }
    const float* GetIdctLookupFloat() const { return &m_afIdctLookup[0][0]; }
    const int*   GetIdctLookupFixed() const { return &m_anIdctLookup[0][0]; }
    // Fill the C-ABI structures from the current table / geometry state (used for batching).
    void        ExportTables(jsgpu_tables& t) const;
    bool        ExportImageDesc(jsgpu_image_desc& d, unsigned nStart) const;
    // Last per-stage device times (ms): marker scan, Huffman, IDCT+colour, finalise, total.
    void        GetStageMs(float ms[5]) const { for (int i = 0; i < 5; i++) ms[i] = m_afStageMs[i]; }

public:
    // DQT tables are public in the reference too (ImgDecode.h:568-571)
    unsigned short  m_anDqtCoeff[MAX_DQT_DEST_ID][MAX_DQT_COEFF];      // natural order
    unsigned short  m_anDqtCoeffZz[MAX_DQT_DEST_ID][MAX_DQT_COEFF];    // zig-zag order
    int             m_anDqtTblSel[MAX_DQT_COMP];
    bool            m_bDibTempReady;
    bool            m_bPreviewIsJpeg;
    CDIB            m_pDibHistRgb, m_pDibHistY;      // the histogram bitmaps DrawHistogram paints (ref ImgDecode.h:513-517)
    bool            m_bDibHistRgbReady, m_bDibHistYReady;
    CDIB            m_pDibTemp;        // public in the reference (ImgDecode.h:384): CjfifDecode hands it to the PSD decoder
                                       // (JfifDecode.cpp:7369); a JPEG scan's BGRA bits live in m_pDibBits, see GetBitmapPtr()

private:
    void        ResetDqtTables();
    void        ResetDhtLookup();
    void        PrecalcIdct();                    // ref :2313-2351 — must run on the HOST (libm cosf)
    void        FreeOutputs();
    bool        EnsureDevice();
    void        CalcChannelPreview();             // ref :4967-4990 -> CalcChannelPreviewFull :4619-4821, on the device
    void        PreviewSettings(jsgpu_preview& pv) const;
    void        FetchPreviewResults();
    void        LogScanEvent(const jsgpu_scan_event& e);          // one error event of a damaged scan -> the reference's line(s)
    void        LogDetailEvent(const jsgpu_detail_event& e, const int16_t* pMatrix);   // ReportVlc / ReportDctMatrix lines (pMatrix: 64 entries, for JSGPU_DT_MATRIX)
    void        LogYccNote(const jsgpu_ycc_warn& w);
    void        LogDetailRgb(const jsgpu_colour_stats* cs);       // "Detailed IDCT Dump (RGB)" of CalcChannelPreviewFull, with the YCC notes in between            // DIB, average luminance, statistics and "YCC Clipped" notes of the last preview pass

    CSnoopConfig*   m_pAppConfig;
    CSnoopConfig    m_sOwnConfig;
    CDocLog*        m_pLog;
    CwindowBuf*     m_pWBuf;
    jsgpu_ctx*      m_pGpu;

    // outputs (host copies; owned, freed by Reset()/dtor like the reference's new[] buffers)
    unsigned*       m_pMcuFileMap;
    short*          m_pPixValY; short* m_pPixValCb; short* m_pPixValCr;
    short*          m_pBlkDcValY; short* m_pBlkDcValCb; short* m_pBlkDcValCr;
    unsigned char*  m_pDibBits;

    unsigned        m_nMcuWidth, m_nMcuHeight, m_nMcuXMax, m_nMcuYMax, m_nBlkXMax, m_nBlkYMax;
    unsigned        m_nImgSizeX, m_nImgSizeY;

    bool            m_bImgDetailsSet;
    unsigned        m_nDimX, m_nDimY, m_nNumSosComps, m_nNumSofComps, m_nPrecision;
    unsigned        m_anSofSampFactH[MAX_SOF_COMP_NF], m_anSofSampFactV[MAX_SOF_COMP_NF];
    bool            m_bRestartEn; unsigned m_nRestartInterval, m_nRestartRead;

    int             m_anDhtTblSel[MAX_DHT_CLASS][1 + MAX_SOS_COMP_NS];
    unsigned        m_anDhtLookupSetMax[MAX_DHT_CLASS];
    unsigned        m_anDhtLookupSize[MAX_DHT_CLASS][MAX_DHT_DEST_ID];
    unsigned        m_anDhtLookup_bitlen[MAX_DHT_CLASS][MAX_DHT_DEST_ID][MAX_DHT_CODES];
    unsigned        m_anDhtLookup_bits[MAX_DHT_CLASS][MAX_DHT_DEST_ID][MAX_DHT_CODES];
    unsigned        m_anDhtLookup_mask[MAX_DHT_CLASS][MAX_DHT_DEST_ID][MAX_DHT_CODES];
    unsigned        m_anDhtLookup_code[MAX_DHT_CLASS][MAX_DHT_DEST_ID][MAX_DHT_CODES];
    unsigned        m_anDhtHisto[MAX_DHT_CLASS][MAX_DHT_DEST_ID][17];

    float           m_afIdctLookup[DCT_SZ_ALL][DCT_SZ_ALL];
    int             m_anIdctLookup[DCT_SZ_ALL][DCT_SZ_ALL];

    bool            m_bDecodeScanAc, m_bScanBad, m_bScanErrorsDisable;
    unsigned        m_nScanStatus, m_nScanErrMax, m_nWarnBadScanNum;
    int             m_nBrightY, m_nBrightCb, m_nBrightCr;
    unsigned        m_nBrightR, m_nBrightG, m_nBrightB, m_nBrightMcuX, m_nBrightMcuY;
    bool            m_bBrightValid, m_bAvgYValid;
    long            m_nAvgY;
    float           m_afStageMs[5];

    bool            m_bDetailVlc; unsigned m_nDetailVlcX, m_nDetailVlcY, m_nDetailVlcLen;
    bool            m_bHistEn, m_bStatClipEn;
    unsigned        m_nPreviewMode;
    int             m_nPreviewShiftY, m_nPreviewShiftCb, m_nPreviewShiftCr;
    unsigned        m_nPreviewShiftMcuX, m_nPreviewShiftMcuY;
    unsigned        m_nWarnYccClipNum;
    unsigned        m_nEndPos, m_nEndAlign;       // m_anScanBuffPtr_pos[0], m_nScanBuffPtr_align after the scan (GetScanBufPos, ref :2575)
    bool            m_bDecodedOnDevice;           // the device still holds this object's last decode
    unsigned        m_anStatClip[12];
    int             m_anHistoMin[12], m_anHistoMax[12], m_anHistoSum[12];     // jsgpu_colour_stats channel order
    unsigned        m_nHistoCount;
    unsigned        m_anCcHisto[3][JSGPU_CC_HISTO_BINS];
    unsigned        m_anHistoYFull[JSGPU_Y_HISTO_BINS];
};
