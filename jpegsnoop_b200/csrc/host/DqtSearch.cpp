// DqtSearch.cpp — see DqtSearch.h.  Reference line numbers refer to the reference's source/JPEGsnoopDoc.cpp.
#include "DqtSearch.h"
#include "JfifWalk.h"
#include <cstdio>
#include <cstring>
#include <cstdarg>
#include <map>
#include <vector>

static std::string fmt(const char* f, ...)
{
    char buf[1024];
    va_list ap; va_start(ap, f); vsnprintf(buf, sizeof buf, f, ap); va_end(ap);
    return std::string(buf);
}

// The JPEG standard's luminance table, raster order (T.81 Table K.1; the reference's glb_anStdQuantLum)
static const unsigned kStdQuantLum[64] = {
    16, 11, 10, 16, 24, 40, 51, 61,  12, 12, 14, 19, 26, 58, 60, 55,  14, 13, 16, 24, 40, 57, 69, 56,  14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68,109,103, 77,  24, 35, 55, 64, 81,104,113, 92,  49, 64, 78, 87,103,121,120,101,  72, 92, 95, 98,112,100,103, 99 };

int DqtSearch(CDocLog* pLog, jsgpu_ctx** ppGpu, int nDevice, CimgDecode* pImgDec, const uint8_t* pData, uint64_t nSize,
              const char* szExePath, const char* szAnalysedPath)
{
    if (nSize >> 32) {                       // the reference's offsets and "%08X" are 32-bit (DESIGN.md §7)
        pLog->AddLineErr(fmt("*** ERROR: Search Executable for DQT: file of %llu bytes; files of 4 GiB or more are not searched ***",
                             (unsigned long long)nSize));
        return JSGPU_EINVAL;
    }
    if (!*ppGpu) {
        const int r = jsgpu_init(nDevice, ppGpu);
        if (r != JSGPU_OK) {
            *ppGpu = nullptr;
            pLog->AddLineErr(fmt("*** ERROR: Search Executable for DQT: GPU search unavailable (%s) ***", jsgpu_strerror(r)));
            return r;
        }
    }

    // the analysed table's flags compare entries 1..63 with entry 0 only (:1348-1358)
    unsigned anTbl[64] = {0};
    bool bAllSame = true, bBaseline = true;
    unsigned nSearchSetMax = 1;
    if (pImgDec) {
        for (unsigned i = 0; i < 64; i++) anTbl[i] = pImgDec->GetDqtEntry(0, i);
        for (unsigned i = 1; i < 64; i++) {
            if (anTbl[i] != anTbl[0]) bAllSame = false;
            if (anTbl[i] > 255) bBaseline = false;
        }
        nSearchSetMax = bAllSame ? 1 : 2;
    }

    // every (ordering, set, layout) the loops below visit, and the distinct byte patterns they need
    struct Search { unsigned nZigZag, nSet, nLayout; int nPat; };
    std::vector<Search> searches;
    std::vector<std::vector<uint8_t>> pats;
    std::map<std::vector<uint8_t>, int> patIndex;
    for (unsigned nZigZag = 0; nZigZag < 2; nZigZag++)
        for (unsigned nSet = 0; nSet < nSearchSetMax; nSet++)
            for (unsigned nLayout = 0; nLayout < 5; nLayout++) {
                // layouts (:1388-1414): 1-byte; 2-byte; 2-byte swapped; 4-byte; 4-byte swapped
                const unsigned nWidth = nLayout == 0 ? 1 : nLayout <= 2 ? 2 : 4;
                const bool bSwap = nLayout == 2 || nLayout == 4;
                if (nWidth == 1 && !bBaseline) { searches.push_back({nZigZag, nSet, nLayout, -1}); continue; }
                std::vector<uint8_t> pat(64 * nWidth, 0);
                for (unsigned k = 0; k < 64; k++) {
                    // "pre-zigzag" (nZigZag 0) takes the entries in zig-zag sequence (GetDqtZigZagIndex, JfifDecode.cpp:398-405)
                    const unsigned nInd = nZigZag ? k : kJfifZigZag[k];
                    const unsigned v = nSet == 0 ? kStdQuantLum[nInd] : anTbl[nInd];
                    uint8_t* e = &pat[k * nWidth];
                    // a baseline table writes the low byte only (:1456-1496)
                    if (nWidth == 1) e[0] = (uint8_t)(v & 0xFF);
                    else if (bSwap) { e[0] = (uint8_t)(v & 0xFF); if (!bBaseline) e[1] = (uint8_t)((v >> 8) & 0xFF); }
                    else { e[nWidth - 1] = (uint8_t)(v & 0xFF); if (!bBaseline) e[nWidth - 2] = (uint8_t)((v >> 8) & 0xFF); }
                }
                auto it = patIndex.find(pat);
                int idx;
                if (it != patIndex.end()) idx = it->second;
                else { idx = (int)pats.size(); patIndex[pat] = idx; pats.push_back(pat); }
                searches.push_back({nZigZag, nSet, nLayout, idx});
            }

    // one pass over the file for all patterns; a second one only when the first position buffer was too small
    std::vector<uint8_t> cat; std::vector<uint32_t> lens;
    for (auto& p : pats) { cat.insert(cat.end(), p.begin(), p.end()); lens.push_back((uint32_t)p.size()); }
    std::vector<uint64_t> counts(pats.size(), 0), first(pats.size(), 0);
    std::vector<uint32_t> pos(1u << 16);
    for (int pass = 0; pass < 2 && !pats.empty(); pass++) {
        const int r = jsgpu_search_bytes(*ppGpu, pData, nSize, cat.data(), lens.data(), (uint32_t)pats.size(), counts.data(),
                                         pos.data(), pos.size());
        if (r != JSGPU_OK) {
            pLog->AddLineErr(fmt("*** ERROR: Search Executable for DQT: GPU search failed: %s (%s) ***", jsgpu_strerror(r), jsgpu_last_error(*ppGpu)));
            return r;
        }
        uint64_t total = 0;
        for (size_t k = 0; k < pats.size(); k++) { first[k] = total; total += counts[k]; }
        if (total <= pos.size()) break;
        pos.assign(total, 0);
    }

    // the report (:1305-1519)
    pLog->AddLineHdr("*** Searching Executable for DQT ***");
    pLog->AddLine(fmt("  Filename: [%s]", szExePath ? szExePath : ""));
    pLog->AddLine(fmt("  Size:     [%lu]", (unsigned long)nSize));
    if (pImgDec && bAllSame) {
        // the reference's format strings print the stray ",_T(" and ")" (:1361-1364)
        pLog->AddLineWarn(fmt("  NOTE: Because the JPEG's DQT Luminance table is constant nValue (0x%02X),_T(", anTbl[0]));
        pLog->AddLineWarn(")        matching for this table has been disabled.");
        pLog->AddLineWarn("        Please select a different reference image.");
    }
    pLog->AddLine("  Searching for DQT Luminance tables:");
    for (const Search& s : searches) {
        if (s.nSet == 0 && s.nLayout == 0) pLog->AddLine(fmt("    DQT Ordering: %s", s.nZigZag ? "post-zigzag" : "pre-zigzag"));
        if (s.nLayout == 0) pLog->AddLine(s.nSet == 0 ? std::string("      Matching [JPEG Standard]")
                                                       : fmt("      Matching [%s]", szAnalysedPath ? szAnalysedPath : ""));
        const unsigned nWidth = s.nLayout == 0 ? 1 : s.nLayout <= 2 ? 2 : 4;
        pLog->AddLine(fmt("        Searching patterns with %u-byte DQT entries%s", nWidth, (s.nLayout == 2 || s.nLayout == 4) ? ", endian byteswap" : ""));
        if (s.nPat < 0) { pLog->AddLine("          DQT Table is not baseline, skipping 1-byte search"); continue; }
        for (uint64_t i = 0; i < counts[s.nPat]; i++)
            pLog->AddLineGood(fmt("          Found @ 0x%08X", pos[first[s.nPat] + i]));
    }
    pLog->AddLine("  Done Search");
    return JSGPU_OK;
}
