#pragma once
// Tools -> Extract embedded JPEG and its Extract All mode (JPEGsnoopCore.cpp:913-1088): CjfifDecode::ExportJpegPrepare and
// ExportJpegDo (JfifDecode.cpp:7544-7797) over the export state the walk to EOI leaves (JfifWalkToEoi).
#include <cstdint>
#include <string>
#include <vector>
#include "HostCompat.h"
#include "../../../include/jsgpu.h"

#define JPEGEXPORT_OVERLAY    1u    // bOverlayEn: copy the bytes through the overlays (the walk always reads through them)
#define JPEGEXPORT_FORCE_SOI  2u    // bForceSoi
#define JPEGEXPORT_FORCE_EOI  4u    // bForceEoi
#define JPEGEXPORT_IGNORE_EOI 8u    // bIgnoreEoi
#define JPEGEXPORT_DHT_AVI    16u   // bDhtAviInsert

// Every FF D8 FF and every PASS-1 scan terminator of the window buffer's file, through its overlays (jsgpu_find_markers on
// *pGpu, made on first use on `device`).  Returns JSGPU_OK or a JSGPU_E* code after one error line in pLog.
int JpegFindMarkers(CDocLog* pLog, jsgpu_ctx** pGpu, int device, const CwindowBuf& wb, std::vector<uint32_t>& soi,
                    std::vector<uint32_t>& term);
// ProcessFile from nPosStart, ExportJpegPrepare and, if it agrees, ExportJpegDo into strOut.  Returns 1 when the file was
// written, 0 when the export was refused (the reason is in the log).
int JpegExportOne(CDocLog* pLog, const CwindowBuf& wb, const std::vector<uint32_t>& term, uint64_t nPosStart,
                  const std::string& strIn, const std::string& strOut, unsigned flags);
// Extract All: frames from offset 0, then from each FF D8 FF after the last start, named root.NNNNNN.jpg (root: strOut up to
// its last '.').  offs / nums receive, per frame analysed, its offset and the number its file got (0: refused).  Returns the
// number of frames analysed, or -1 after the "Invalid filename" error when strOut has no '.'.
int64_t JpegExtractAll(CDocLog* pLog, const CwindowBuf& wb, const std::vector<uint32_t>& soi, const std::vector<uint32_t>& term,
                       const std::string& strIn, const std::string& strOut, unsigned flags, std::vector<uint64_t>& offs,
                       std::vector<uint32_t>& nums);
