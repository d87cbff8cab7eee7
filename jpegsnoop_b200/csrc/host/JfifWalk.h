#pragma once
#include <cstdint>
#include <vector>
class CimgDecode;
#define JFIFWALK_ENOTJPEG -1
#define JFIFWALK_EMARKER  -2
#define JFIFWALK_ENOSCAN  -3
#define JFIFWALK_ETRUNC   -4
#define JFIFWALK_EUNSUP   -5
// Walk the markers of the first frame of the JPEG whose SOI is at nPosStart and issue CjfifDecode's setter sequence on pImgDec.
// Returns the absolute file offset of the first entropy-coded byte of the first scan (>0) or a JFIFWALK_E* code.
// *pbSof (optional) tells whether the walk reached a frame header: CjfifDecode::GetDecodeStatus() after ProcessFile.
int JfifWalk(CimgDecode* pImgDec, const uint8_t* data, uint64_t n, uint64_t nPosStart = 0, bool* pbSof = nullptr);

// What CjfifDecode's ProcessFile leaves for ExportJpegPrepare / ExportJpegDo (JfifDecode.cpp:7297-7451): the marker flags,
// the first SOS marker's position (m_nPosSos, :5114-5116) and the position just past FF D9 (m_nPosEmbedEnd, :5338).
struct JfifEnd {
    bool bSoi = false, bDqt = false, bDht = false, bSof = false, bSos = false, bEoi = false;
    uint64_t nPosSos = 0, nPosEmbedEnd = 0;
};
// The same walk carried on to the EOI, as ProcessFile runs it from nPosStart whether or not an SOI is there: every scan is
// skipped to the first PASS-1 terminator at or after its start, taken from term[0 .. nterm) (ascending, every terminator
// of the file: jsgpu_find_markers).  The walk stops at EOI, at a marker the reference stops at, or past the end of the
// file.  Nothing is decoded and no setter is called.
void JfifWalkToEoi(const uint8_t* data, uint64_t n, uint64_t nPosStart, const uint32_t* term,
                   uint64_t nterm, JfifEnd* pEnd);
// The Annex K tables a Motion-JPEG frame leaves out, DC 0, DC 1, AC 0, AC 1, as the body of one DHT segment
const std::vector<uint8_t>& MjpgDhtTables();
// zig-zag position -> natural index (T.81 Figure A.6; the permutation of the reference's glb_anZigZag)
extern const unsigned kJfifZigZag[64];
