// HostCompat.h — the three collaborators CimgDecode talks to, reduced to what the scan-decode
// path uses, for building the host class outside MFC.  In a real JPEGsnoop build these names are
// provided by the application's own DocLog.h / WindowBuf.h / SnoopConfig.h (see INTEGRATION.md);
// here they are small, self-contained stand-ins written for this repo (not copies).
#pragma once
#include <cstdint>
#include <cstddef>
#include <string>
#include <vector>

// Line log.  CimgDecode reports problems as log lines, never as exceptions
// (reference convention: ImgDecode.cpp:2755-2758, 2764-2769, 3050-3054, 3098-3102).
class CDocLog {
public:
    enum Kind { LINE, HDR, WARN, ERR, GOOD };
    struct Entry { Kind kind; std::string text; };
    void AddLine(const std::string& s)     { if (m_en) m_lines.push_back({LINE, s}); }
    void AddLineHdr(const std::string& s)  { if (m_en) m_lines.push_back({HDR, s}); }
    void AddLineWarn(const std::string& s) { if (m_en) m_lines.push_back({WARN, s}); }
    void AddLineErr(const std::string& s)  { if (m_en) m_lines.push_back({ERR, s}); }
    void AddLineGood(const std::string& s) { if (m_en) m_lines.push_back({GOOD, s}); }
    void Enable() { m_en = true; }
    void Disable() { m_en = false; }
    void Clear() { m_lines.clear(); }
    size_t Count(Kind k) const { size_t n = 0; for (auto& e : m_lines) if (e.kind == k) n++; return n; }
    const std::vector<Entry>& Lines() const { return m_lines; }
private:
    std::vector<Entry> m_lines;
    bool m_en = true;
};

// Byte source.  The reference reads the file through a 128 KiB sliding window one byte at a time
// (WindowBuf.cpp:639-713); the GPU path wants the whole entropy-coded segment at once, so the only
// operations kept are "byte at offset" (0 past EOF, as WindowBuf.cpp:704-711), the EOF position and
// a bulk view.  Overlays (WindowBuf.cpp:516-560) are honoured by BufCopy() when installed.
class CwindowBuf {
public:
    void BufSet(const uint8_t* data, size_t n) { m_p = data; m_n = n; }
    uint8_t Buf(unsigned long off, bool bClean = false) const {
        uint8_t v = (off < m_n) ? m_p[off] : 0;
        if (!bClean) for (auto& o : m_ovl) if (off >= o.start && off < o.start + o.data.size()) v = o.data[off - o.start];   // the last overlay installed wins (WindowBuf.cpp:659-670)
        return v;
    }
    void BufLoadWindow(unsigned long) {}
    unsigned long GetPosEof() const { return (unsigned long)m_n; }
    bool GetBufOk() const { return m_p != nullptr; }
    // copy [off, off+n) through Buf() semantics (overlays applied, zero past EOF)
    void BufCopy(unsigned long off, size_t n, uint8_t* dst) const {
        for (size_t i = 0; i < n; i++) dst[i] = (off + i < m_n) ? m_p[off + i] : 0;
        for (auto& o : m_ovl) for (size_t j = 0; j < o.data.size(); j++) { unsigned long a = o.start + (unsigned long)j; if (a >= off && a < off + n) dst[a - off] = o.data[j]; }
    }
    bool OverlayInstall(unsigned long start, const uint8_t* d, size_t n) { m_ovl.push_back({start, std::vector<uint8_t>(d, d + n)}); return true; }
    void OverlayRemoveAll() { m_ovl.clear(); }
private:
    struct Ovl { unsigned long start; std::vector<uint8_t> data; };
    const uint8_t* m_p = nullptr; size_t m_n = 0;
    std::vector<Ovl> m_ovl;
};

// Stand-in for the reference's CDIB (Dib.h:32-55) as far as the decode path needs it: a w*h*4-byte BGRA buffer.
class CDIB {
public:
    void  Kill() { m_bits.clear(); m_bits.shrink_to_fit(); }
    bool  CreateDIB(unsigned w, unsigned h, unsigned short) { m_bits.assign((size_t)w * h * 4, 0); return true; }
    void* GetDIBBitArray() const { return m_bits.empty() ? nullptr : (void*)m_bits.data(); }
private:
    std::vector<uint8_t> m_bits;
};

// The configuration fields DecodeScanImg reads (SnoopConfig.h:72-142, read at
// ImgDecode.cpp:448, 2730-2741) plus this port's device knobs.
struct CSnoopConfig {
    bool     bInteractive = false;
    bool     bDumpHistoY = false;
    bool     bDecodeScanImg = true;
    bool     bDecodeScanImgAc = true;     // reference default is false (DC-only preview, SnoopConfig.cpp:70)
    bool     bHistoEn = false;
    bool     bStatClipEn = false;
    unsigned nErrMaxDecodeScan = 20;      // SnoopConfig.cpp:89
    // --- port additions ---
    bool     bIdctFixedPt = true;         // true = the IDCT_FIXEDPT build's arithmetic (ImgDecode.cpp:32)
    int      nCudaDevice = 0;
    int      nHuffKernel = 0;             // jsgpu_options.huff_kernel
    int      nIdctKernel = 0;             // jsgpu_options.idct_kernel
};
