// JpegExport.cpp — Extract embedded JPEG and Extract All (see JpegExport.h).  The walk to EOI takes every scan's end from the
// device's terminator list, so the host reads only marker segments; the exported bytes are copied from the caller's buffer.
#include <algorithm>
#include <cstdio>
#include "JpegExport.h"
#include "JfifWalk.h"

int JpegFindMarkers(CDocLog* pLog, jsgpu_ctx** pGpu, int device, const CwindowBuf& wb, std::vector<uint32_t>& soi,
                    std::vector<uint32_t>& term)
{
    if (!*pGpu) {
        const int r = jsgpu_init(device, pGpu);
        if (r != JSGPU_OK) {
            *pGpu = nullptr;
            pLog->AddLineErr(std::string("*** ERROR: Extract: GPU search unavailable (") + jsgpu_strerror(r) + ") ***");
            return r;
        }
    }
    std::vector<jsgpu_overlay> ovl;
    for (auto& o : wb.Overlays()) ovl.push_back({(uint64_t)o.start, (uint64_t)o.data.size(), o.data.data()});
    const uint64_t n = wb.GetPosEof();
    // a first guess that holds a JPEG's markers and random bytes' terminators (about one per 265 bytes); else a second pass
    uint64_t ns = 0, nt = 0;
    soi.resize(n / 4096 + 1024); term.resize(n / 128 + 1024);
    for (int pass = 0; pass < 2; pass++) {
        const int r = jsgpu_find_markers(*pGpu, wb.BufData(), n, ovl.data(), (uint32_t)ovl.size(), soi.data(), soi.size(), &ns,
                                         term.data(), term.size(), &nt);
        if (r != JSGPU_OK) {
            pLog->AddLineErr(std::string("*** ERROR: Extract: ") + jsgpu_strerror(r) + " (" + jsgpu_last_error(*pGpu) + ") ***");
            return r;
        }
        if (ns <= soi.size() && nt <= term.size()) break;
        soi.resize(std::max<uint64_t>(ns, 1)); term.resize(std::max<uint64_t>(nt, 1));
    }
    soi.resize(ns); term.resize(nt);
    return JSGPU_OK;
}

// ExportJpegPrepare (JfifDecode.cpp:7544-7624): its log lines, and whether the export goes ahead; a missing EOI under Force /
// Ignore EOI ends the frame at the end of the file.
static bool Prepare(CDocLog* pLog, JfifEnd& st, uint64_t nPosStart, uint64_t nFileEnd, const std::string& strIn, unsigned flags)
{
    pLog->AddLine("");
    pLog->AddLineHdr("*** Exporting JPEG ***");
    pLog->AddLine("  Exporting from: [" + strIn + "]");
    if (!st.bEoi) {
        if (!(flags & (JPEGEXPORT_FORCE_EOI | JPEGEXPORT_IGNORE_EOI))) {
            pLog->AddLineErr("  ERROR: Missing marker: EOI");
            pLog->AddLineErr("         Aborting export. Consider enabling [Force EOI] or [Ignore Missing EOI] option");
            return false;
        }
        st.nPosEmbedEnd = nFileEnd;
    }
    if (nPosStart == 0 && st.nPosEmbedEnd == 0) {
        pLog->AddLineErr("  No frame found at this position in file. Consider using [Img Search]");
        return false;
    }
    if (!st.bSoi && !(flags & JPEGEXPORT_FORCE_SOI)) {
        pLog->AddLineErr("  ERROR: Missing marker: SOI");
        pLog->AddLineErr("         Aborting export. Consider enabling [Force SOI] option");
        return false;
    }
    if (!st.bSos) {
        pLog->AddLineErr("  ERROR: Missing marker: SOS");
        pLog->AddLineErr("         Aborting export");
        return false;
    }
    std::string strMissing;
    if (!st.bDqt) strMissing += "DQT ";
    if (!st.bDht) strMissing += "DHT ";
    if (!st.bSof) strMissing += "SOF ";
    if (!strMissing.empty()) {
        pLog->AddLineWarn("  NOTE: Missing marker: " + strMissing);
        pLog->AddLineWarn("        Exported JPEG may not be valid");
    }
    if (st.nPosEmbedEnd < nPosStart) {
        pLog->AddLineErr("ERROR: Invalid SOI-EOI order. Export aborted.");
        return false;
    }
    return true;
}

// One part of ExportJpegDo's copy: `while (ind < nCopyEnd)` with nCopyEnd = b - 1 inclusive, in 131 072-byte pieces
// (EXPORT_BUF_SIZE), so a part of k * 131072 + 1 bytes loses its last byte and one of 1 byte is not written.  The bytes are
// Buf(ind, !bOverlayEn): the file's (0 past its end), through the overlays when `ovl`.  A part ending at 0 (nCopyEnd
// wrapping to 2^32 - 1) writes nothing here.
static void CopyPart(FILE* f, const CwindowBuf& wb, uint64_t a, uint64_t b, bool ovl)
{
    const uint32_t kBuf = 131072;
    if (b == 0) return;
    const uint32_t nCopyEnd = (uint32_t)(b - 1);
    const uint64_t n = wb.GetPosEof();
    std::vector<uint8_t> buf(kBuf);
    for (uint32_t ind = (uint32_t)a; ind < nCopyEnd;) {
        const uint32_t nLeft = std::min(nCopyEnd - ind + 1, kBuf);
        const uint64_t nIn = ind < n ? std::min<uint64_t>(nLeft, n - ind) : 0;
        std::copy(wb.BufData() + ind, wb.BufData() + ind + nIn, buf.begin());
        std::fill(buf.begin() + nIn, buf.begin() + nLeft, 0);
        if (ovl)
            for (auto& o : wb.Overlays())
                for (size_t j = 0; j < o.data.size(); j++)
                    if (o.start + j >= ind && o.start + j - ind < nLeft) buf[o.start + j - ind] = o.data[j];
        fwrite(buf.data(), 1, nLeft, f);
        ind += nLeft;
    }
}

// ExportJpegDo (JfifDecode.cpp:7632-7797): [start, first SOS), the AVI DHT, [first SOS, end), around a forced SOI / EOI.
static bool Write(CDocLog* pLog, const CwindowBuf& wb, const JfifEnd& st, uint64_t nPosStart, const std::string& strIn,
                  const std::string& strOut, unsigned flags)
{
    pLog->AddLine("  Exporting to:   [" + strOut + "]");
    if (strIn == strOut) {
        pLog->AddLineErr("ERROR: Can't overwrite source file. Aborting export.");
        return false;
    }
    if (strIn.empty()) {
        pLog->AddLineErr("ERROR: Export but source filename empty");
        return false;
    }
    FILE* f = fopen(strOut.c_str(), "wb");
    if (!f) {
        pLog->AddLineErr("ERROR: Couldn't open file for write [" + strOut + "]: []");
        return false;
    }
    if (!st.bSoi && (flags & JPEGEXPORT_FORCE_SOI)) {
        pLog->AddLine("    Forcing SOI Marker");
        fwrite("\xFF\xD8", 1, 2, f);
    }
    const bool ovl = (flags & JPEGEXPORT_OVERLAY) != 0;
    CopyPart(f, wb, nPosStart, st.nPosSos, ovl);
    if (flags & JPEGEXPORT_DHT_AVI) {
        pLog->AddLine("  Inserting standard AVI DHT huffman table");
        const std::vector<uint8_t>& t = MjpgDhtTables();             // m_abMJPGDHTSeg: the marker, the length, the tables
        const uint8_t hdr[4] = {0xFF, 0xC4, (uint8_t)((t.size() + 2) >> 8), (uint8_t)(t.size() + 2)};
        fwrite(hdr, 1, 4, f);
        fwrite(t.data(), 1, t.size(), f);
    }
    CopyPart(f, wb, st.nPosSos, st.nPosEmbedEnd, ovl);
    if (flags & JPEGEXPORT_FORCE_EOI) {
        pLog->AddLine("    Forcing EOI Marker");
        fwrite("\xFF\xD9", 1, 2, f);
    }
    fclose(f);
    pLog->AddLine("  Export done");
    return true;
}

// The file as the walk reads it: through the overlays (a copy only when there are any)
static const uint8_t* WalkView(const CwindowBuf& wb, std::vector<uint8_t>& tmp)
{
    if (wb.Overlays().empty()) return wb.BufData();
    const uint64_t n = wb.GetPosEof();
    tmp.resize(n);
    wb.BufCopy(0, n, tmp.data());
    return tmp.data();
}

// 0: refused by Prepare; 1: prepared, not written; 2: written
static int ExportFrom(CDocLog* pLog, const CwindowBuf& wb, const uint8_t* d, const std::vector<uint32_t>& term, uint64_t nPosStart,
                      const std::string& strIn, const std::string& strOut, unsigned flags)
{
    const uint64_t n = wb.GetPosEof();
    JfifEnd st;
    JfifWalkToEoi(d, n, nPosStart, term.data(), term.size(), &st);
    if (!Prepare(pLog, st, nPosStart, n, strIn, flags)) return 0;
    return Write(pLog, wb, st, nPosStart, strIn, strOut, flags) ? 2 : 1;
}

int JpegExportOne(CDocLog* pLog, const CwindowBuf& wb, const std::vector<uint32_t>& term, uint64_t nPosStart,
                  const std::string& strIn, const std::string& strOut, unsigned flags)
{
    std::vector<uint8_t> tmp;
    return ExportFrom(pLog, wb, WalkView(wb, tmp), term, nPosStart, strIn, strOut, flags) == 2;
}

int64_t JpegExtractAll(CDocLog* pLog, const CwindowBuf& wb, const std::vector<uint32_t>& soi, const std::vector<uint32_t>& term,
                       const std::string& strIn, const std::string& strOut, unsigned flags, std::vector<uint64_t>& offs,
                       std::vector<uint32_t>& nums)
{
    offs.clear(); nums.clear();
    const size_t nExt = strOut.rfind('.');
    if (nExt == std::string::npos) {
        pLog->AddLineErr("ERROR: Invalid filename [" + strOut + "]");
        return -1;
    }
    const std::string strRoot = strOut.substr(0, nExt);
    std::vector<uint8_t> tmp;
    const uint8_t* d = WalkView(wb, tmp);
    uint32_t nExportCnt = 1;
    uint64_t nPos = 0;
    for (;;) {
        char name[16];
        snprintf(name, sizeof name, ".%06u.jpg", nExportCnt);
        const int r = ExportFrom(pLog, wb, d, term, nPos, strIn, strRoot + name, flags);
        offs.push_back(nPos);
        nums.push_back(r == 2 ? nExportCnt : 0);
        if (r) nExportCnt++;                                      // a frame Prepare refuses keeps the counter (:1026-1047)
        // BufSearch(nPos, 0xFFD8FF, 3, fwd): the first FF D8 FF after nPos (:1054)
        auto it = std::upper_bound(soi.begin(), soi.end(), nPos, [](uint64_t a, uint32_t b) { return a < b; });
        if (it == soi.end()) break;
        nPos = *it;
    }
    return (int64_t)offs.size();
}
