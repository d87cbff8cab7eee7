// JfifWalk.cpp — the slice of CjfifDecode::DecodeMarker that feeds the scan decoder: walk
// SOI / DQT / SOF0-1 / DHT / DRI / SOS and make the SAME setter calls, in the same order and with
// the same arguments, that the reference parser makes (source/JfifDecode.cpp: DQT 4576-4651,
// SOF 5001-5026, DHT 3535-3600, DRI 5310-5330, SOS 5150-5164 + 5291, the AVI1 Huffman-table
// import 4406-4426).  Everything else the reference parser does (EXIF, signatures, thumbnails,
// logging) is out of scope (SURVEY.md §8f N1).
#include <algorithm>
#include <vector>
#include "ImgDecode.h"
#include "JfifWalk.h"
#include "../annex_k.h"

const unsigned kJfifZigZag[64] = {
     0, 1, 8,16, 9, 2, 3,10, 17,24,32,25,18,11, 4, 5, 12,19,26,33,40,48,41,34, 27,20,13, 6, 7,14,21,28,
    35,42,49,56,57,50,43,36, 29,22,15,23,30,37,44,51, 58,59,52,45,38,31,39,46, 53,60,61,54,47,55,62,63 };

// The tables of one DHT segment, [q, e): canonical codes in the reference's SetDhtEntry / SetDhtSize calls (:3535-3600).
static int WalkDht(CimgDecode* pImgDec, const uint8_t* d, uint64_t q, uint64_t e)
{
    while (q < e) {
        unsigned Tc = d[q] >> 4, Th = d[q] & 15; q++;
        if (q + 16 > e) return JFIFWALK_ETRUNC;
        unsigned Li[17], tot = 0;
        for (unsigned i = 1; i <= 16; i++) { Li[i] = d[q++]; tot += Li[i]; }
        if (q + tot > e) return JFIFWALK_ETRUNC;
        const uint8_t* vals = d + q; q += tot;
        unsigned nCodeVal = 0, nDhtInd = 0, nLookupInd = 0;
        for (unsigned nBitLen = 1; nBitLen <= 16; nBitLen++) {
            for (unsigned j = 0; j < Li[nBitLen]; j++) {
                unsigned nMask = (unsigned)((((uint64_t)1 << nBitLen) - 1) << (32 - nBitLen));
                pImgDec->SetDhtEntry(Th, Tc, nLookupInd, nBitLen, nCodeVal << (32 - nBitLen), nMask, vals[nDhtInd]);   // :3581
                nLookupInd++; nCodeVal++; nDhtInd++;
            }
            nCodeVal <<= 1;
        }
        pImgDec->SetDhtSize(Th, Tc, nLookupInd);                             // :3600
    }
    return 0;
}

// The tables of the DHT segment a Motion-JPEG frame leaves out (OpenDML AVI, "Proposed Data Chunk Format"): the T.81
// Annex K tables in the order DC 0, DC 1, AC 0, AC 1, as the Tc/Th bytes, BITS and HUFFVAL of one DHT segment.
const std::vector<uint8_t>& MjpgDhtTables()
{
    static const std::vector<uint8_t> seg = [] {
        using namespace annex_k;
        std::vector<uint8_t> s;
        auto put = [&](uint8_t tcth, const uint8_t* bits, const uint8_t* vals, unsigned nvals) {
            s.push_back(tcth); s.insert(s.end(), bits, bits + 16); s.insert(s.end(), vals, vals + nvals);
        };
        put(0x00, kDcLumBits, kDcVals, 12); put(0x01, kDcChrBits, kDcVals, 12);
        put(0x10, kAcLumBits, kAcLumVals, 162); put(0x11, kAcChrBits, kAcChrVals, 162);
        return s;
    }();
    return seg;
}

// CjfifDecode reads the APP0 identifier with BufReadStrn (WindowBuf.cpp:984-1007) from just after the length field, whatever
// the length: up to 255 bytes, stopping at a 0 byte and keeping only printable ones, bytes past the end of the file reading
// as 0.  A Motion-JPEG frame is one whose identifier starts with "AVI1" (JfifDecode.cpp:4406).
static bool App0IsAvi1(const uint8_t* d, uint64_t n, uint64_t q)
{
    static const char kAvi1[4] = {'A', 'V', 'I', '1'};
    unsigned k = 0;
    for (uint64_t i = 0; i < 255 && k < 4; i++) {
        const uint8_t c = q + i < n ? d[q + i] : 0;
        if (c == 0) break;
        if (c >= 0x20 && c <= 0x7E) {
            if (c != (uint8_t)kAvi1[k]) return false;
            k++;
        }
    }
    return k == 4;
}

// One walk for both callers.  Without pEnd it is the decode walk: the first frame's setter sequence from an SOI at nPosStart
// to its first SOS.  With pEnd it is ProcessFile's loop to the EOI (JfifDecode.cpp:7430-7451, DecodeMarker :3783-5440),
// recording the export state; pImgDec is then null and no setter is called.  A segment that runs past the end of the file
// stops it there (the reference reads 0s past the end and then stops at "Early EOF").
static int Walk(CimgDecode* pImgDec, const uint8_t* d, uint64_t n, uint64_t nPosStart, bool* pbSof, const uint32_t* term,
                uint64_t nterm, JfifEnd* pEnd)
{
    unsigned unzz[64];
    for (unsigned i = 0; i < 64; i++) unzz[kJfifZigZag[i]] = i;
    const bool bToEoi = pEnd != nullptr;
    if (pImgDec) pImgDec->ResetState();
    bool bSofSeen = false;                                          // CjfifDecode::m_bImgOK (JfifDecode.cpp:96, 5030)
    if (!pbSof) pbSof = &bSofSeen;
    *pbSof = false;
    auto byte = [&](uint64_t q) -> unsigned { return q < n ? d[q] : 0u; };   // Buf(): 0 past the end of the file
    uint64_t p = nPosStart;
    if (!bToEoi) {
        // ProcessFile starts the marker walk at m_pAppConfig->nPosStart and every position stays absolute (JfifDecode.cpp:7338-7341)
        if (nPosStart >= n || n - nPosStart < 4 || d[nPosStart] != 0xFF || d[nPosStart + 1] != 0xD8) return JFIFWALK_ENOTJPEG;
        p = nPosStart + 2;
    }
    unsigned X = 0, Y = 0, Nf = 0, P = 8, nRstInterval = 0;
    bool bRstEn = false, bSof = false;
    while (bToEoi ? p < n : p + 4 <= n) {
        if (d[p] != 0xFF) return JFIFWALK_EMARKER;
        unsigned m = byte(p + 1); p += 2;
        if (m == 0xFF) { p -= 1; continue; }                       // fill byte
        if (bToEoi) {
            if (m == 0xD8) { pEnd->bSoi = true; continue; }
            if (m == 0xD9) { pEnd->bEoi = true; pEnd->nPosEmbedEnd = p; return 0; }     // :5338-5342
            // RSTn outside a scan and the markers DecodeMarker has no case for stop the walk (bRelaxedParsing off, :5350-5430)
            const bool bKnown = (m >= 0xC0 && m <= 0xCF) || (m >= 0xDA && m <= 0xFE) || m == 0x01;
            if (!bKnown) return JFIFWALK_EMARKER;
        } else {
            if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
            if (m == 0xD9) return JFIFWALK_ENOSCAN;
        }
        unsigned L = (byte(p) << 8) | byte(p + 1);
        uint64_t q = p + 2, e = p + L;
        if (bToEoi) {
            if (m == 0xDB) pEnd->bDqt = true;                                       // :4440
            if (m == 0xC4 || (m == 0xE0 && App0IsAvi1(d, n, q))) pEnd->bDht = true;  // :5100, the AVI1 import :4397, 4421
            if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) { pEnd->bSof = bSof = true; *pbSof = true; }   // :4821, 5032
            if (m == 0xDA) {
                pEnd->bSos = true;                                                  // :5108-5116
                if (pEnd->nPosSos == 0) pEnd->nPosSos = p - 2;
                if (!bSof) return JFIFWALK_EMARKER;                                 // "SOS before valid SOF defined"
            }
            if (e > n) return JFIFWALK_ETRUNC;
            if (m == 0xDB) {                                                        // Pq 0..1, Tq 0..3 (:4473-4474)
                while (q < e) {
                    const unsigned Pq = d[q] >> 4, Tq = d[q] & 15;
                    if (Pq > 1 || Tq > 3) return JFIFWALK_EMARKER;
                    q += 1 + 64 * (Pq + 1);
                }
            }
            if (m == 0xDA) {
                // PASS 1 (:5194-5265): the scan ends at the first terminator at or after its start, or runs out of file
                const uint32_t* t = std::lower_bound(term, term + nterm, e, [](uint32_t a, uint64_t b) { return a < b; });
                if (t == term + nterm) return JFIFWALK_ETRUNC;
                p = *t;
                continue;
            }
            p = e;
            continue;
        }
        if (L < 2 || e > n) return JFIFWALK_ETRUNC;
        switch (m) {
        case 0xDB:                                                  // DQT
            while (q < e) {
                unsigned Pq = d[q] >> 4, Tq = d[q] & 15; q++;
                unsigned tbl[64];
                for (unsigned k = 0; k < 64; k++) {                 // file order is zig-zag (JfifDecode.cpp:4576-4584)
                    if (q >= e) return JFIFWALK_ETRUNC;
                    unsigned v = d[q++]; if (Pq) { if (q >= e) return JFIFWALK_ETRUNC; v = (v << 8) | d[q++]; }
                    tbl[kJfifZigZag[k]] = v;
                }
                for (unsigned i = 0; i < 64; i++) pImgDec->SetDqtEntry(Tq, i, unzz[i], (unsigned short)tbl[i]);   // :4648
            }
            break;
        case 0xC0: case 0xC1: {                                     // SOF0 / SOF1 (others unsupported: :4827-4829)
            if (q + 6 > e) return JFIFWALK_ETRUNC;
            P = d[q]; Y = ((unsigned)d[q + 1] << 8) | d[q + 2]; X = ((unsigned)d[q + 3] << 8) | d[q + 4]; Nf = d[q + 5]; q += 6;
            if (q + 3ull * Nf > e) return JFIFWALK_ETRUNC;
            unsigned H[256], V[256], T[256];
            for (unsigned i = 1; i <= Nf; i++) { q++; H[i] = d[q] >> 4; V[i] = d[q] & 15; q++; T[i] = d[q++]; }
            for (unsigned i = 1; i <= Nf; i++) { pImgDec->SetDqtTables(i, T[i]); pImgDec->SetPrecision(P); }       // :5008,5012
            for (unsigned i = 1; i <= Nf; i++) pImgDec->SetSofSampFactors(i, H[i], V[i]);                           // :5025
            bSof = true; *pbSof = true;
            break; }
        case 0xC2: case 0xC3: case 0xC5: case 0xC6: case 0xC7: case 0xC9: case 0xCA: case 0xCB: case 0xCD: case 0xCE: case 0xCF:
            *pbSof = true;                                          // the reference parses these frames too (:4800-4812)
            return JFIFWALK_EUNSUP;
        case 0xC4: {                                                // DHT
            const int r = WalkDht(pImgDec, d, q, e);
            if (r) return r;
            break; }
        case 0xE0:                                                  // APP0: a Motion-JPEG frame imports the tables it omits
            if (App0IsAvi1(d, n, q)) {
                const std::vector<uint8_t>& t = MjpgDhtTables();
                WalkDht(pImgDec, t.data(), 0, t.size());
            }
            break;
        case 0xDD:                                                  // DRI (:5310-5330)
            if (q + 2 > e) return JFIFWALK_ETRUNC;
            nRstInterval = ((unsigned)d[q] << 8) | d[q + 1];
            bRstEn = (nRstInterval != 0);
            break;
        case 0xDA: {                                                // SOS
            if (!bSof) return JFIFWALK_EMARKER;
            unsigned Ns = d[q++];
            if (Ns > MAX_SOS_COMP_NS || q + 2ull * Ns + 3 > e) return JFIFWALK_ETRUNC;
            for (unsigned i = 1; i <= Ns; i++) { q++; unsigned t = d[q++]; pImgDec->SetDhtTables(i, t >> 4, t & 15); }    // :5161
            pImgDec->SetImageDetails(X, Y, Nf, Ns, bRstEn, nRstInterval);                                         // :5291
            if (e > 0x7FFFFFFFull) return JFIFWALK_ETRUNC;          // the scan start is returned as an int (file positions are 32-bit in the reference too)
            return (int)e;
        }
        default: break;                                             // APPn, COM, ...: skipped
        }
        p = e;
    }
    return JFIFWALK_ENOSCAN;
}

int JfifWalk(CimgDecode* pImgDec, const uint8_t* d, uint64_t n, uint64_t nPosStart, bool* pbSof)
{
    return Walk(pImgDec, d, n, nPosStart, pbSof, nullptr, 0, nullptr);
}

void JfifWalkToEoi(const uint8_t* d, uint64_t n, uint64_t nPosStart, const uint32_t* term, uint64_t nterm, JfifEnd* pEnd)
{
    *pEnd = JfifEnd();
    Walk(nullptr, d, n, nPosStart, nullptr, term, nterm, pEnd);
}
