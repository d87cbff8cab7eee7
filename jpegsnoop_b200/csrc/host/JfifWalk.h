#pragma once
#include <cstdint>
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
// zig-zag position -> natural index (T.81 Figure A.6; the permutation of the reference's glb_anZigZag)
extern const unsigned kJfifZigZag[64];
