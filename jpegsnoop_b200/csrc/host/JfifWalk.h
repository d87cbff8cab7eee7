#pragma once
#include <cstdint>
class CimgDecode;
#define JFIFWALK_ENOTJPEG -1
#define JFIFWALK_EMARKER  -2
#define JFIFWALK_ENOSCAN  -3
#define JFIFWALK_ETRUNC   -4
#define JFIFWALK_EUNSUP   -5
// Walk the markers of the first frame of a JPEG and issue CjfifDecode's setter sequence on pImgDec.
// Returns the file offset of the first entropy-coded byte of the first scan (>0) or a JFIFWALK_E* code.
int JfifWalk(CimgDecode* pImgDec, const uint8_t* data, uint64_t n);
// zig-zag position -> natural index (T.81 Figure A.6; the permutation of the reference's glb_anZigZag)
extern const unsigned kJfifZigZag[64];
