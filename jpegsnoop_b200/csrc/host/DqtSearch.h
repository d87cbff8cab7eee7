// DqtSearch.h — Tools -> Search Executable for DQT (CJPEGsnoopDoc::OnToolsSearchexecutablefordqt, JPEGsnoopDoc.cpp:1233-1529)
// on the GPU: the luminance quantisation tables (the JPEG standard's, and table 0 of the analysed image when there is one)
// in both orderings and five byte layouts are searched in one pass over the file (jsgpu_search_bytes), and the report goes to
// the log line for line as the reference writes it.
#pragma once
#include <cstdint>
#include "ImgDecode.h"

// pImgDec: the decoder that analysed the current JPEG (its GetDqtEntry(0, .) is read), or nullptr when no file has been
// analysed (the Doc's IsAnalyzed()).  *ppGpu is the device context, created on first use on device nDevice and kept by
// the caller.  Returns JSGPU_OK, or a negative JSGPU_E* code after an error line (no search lines are written then).
int DqtSearch(CDocLog* pLog, jsgpu_ctx** ppGpu, int nDevice, CimgDecode* pImgDec, const uint8_t* pData, uint64_t nSize,
              const char* szExePath, const char* szAnalysedPath);
