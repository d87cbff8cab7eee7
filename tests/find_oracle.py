"""TEST INFRASTRUCTURE: JPEGsnoop's Img Search and offset decoding on the CPU, for tests/test_image_search.py and
tools/find_probe.py.

* bufsearch_model(...): CwindowBuf::BufSearch (WindowBuf.cpp:149-212) restated in numpy: the positions its loop tests, in
  order, the big-endian value of the `length` bytes at each (overlays applied, 0 past EOF), the first match.
* ref_bufsearch(...): the reference's own compiled CwindowBuf::BufSearch, called on the window buffer of a fresh
  oracle/_ref/liboracle_ref_fixed.so context (the same one tests/dqt_oracle.py uses), overlays installed with the
  reference's CwindowBuf::OverlayInstall.
* RefN1: the reference's CjfifDecode + CimgDecode (oracle/_ref/libn1_ref.so) with CSnoopConfig::nPosStart set before
  ProcessFile, as JPEGsnoopCore.cpp:700-756 and the Doc's handlers set it; GetDecodeStatus, SetDetailVlc and the per-MCU /
  per-block lookups are the reference's exported member functions called on the harness's objects.
* ref_doc_search / ref_offset_mode: the Doc's OnToolsSearchforward / OnToolsSearchreverse (JPEGsnoopDoc.cpp:829-932) and
  DoAnalyzeOffset (JPEGsnoopCore.cpp:700-756) restated over ref_bufsearch and RefN1.
All but the model need the compiled reference (ref_available()).
"""
import ctypes as C
import os
import numpy as np

import dqt_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
SOI3 = 0xFFD8FF

ref_available = dqt_oracle.ref_available


def tested_positions(n, start, length, forward):
    """The positions BufSearch's loop tests, in order: forward start + 1 .. the first p with p + length - 1 >= n (or start + 1
    alone); reverse start - 1 .. 0, and 0 alone from 0."""
    if forward:
        first = start + 1
        return np.arange(first, max(first, n - length + 1) + 1, dtype=np.int64)
    return np.arange(start - 1, -1, -1, dtype=np.int64) if start else np.zeros(1, np.int64)


def bufsearch_model(data, start, value, length, forward, overlays=()):
    """(found, position): what BufSearch(start, value, length, forward) returns; not found -> the last position tested."""
    src = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data
    pos = tested_positions(src.size, start, length, forward)
    top = int(pos.max()) + length
    for o, b in overlays:
        top = max(top, o + len(b))
    buf = np.zeros(max(top, src.size), np.uint8)
    buf[:src.size] = src
    for o, b in overlays:                              # installed order: the last one wins (WindowBuf.cpp:659-670)
        buf[o:o + len(b)] = np.frombuffer(bytes(b), np.uint8)
    v = np.zeros(pos.size, np.uint64)
    for i in range(length):
        v = (v << np.uint64(8)) | buf[pos + i].astype(np.uint64)
    hit = np.flatnonzero(v == np.uint64(value))
    return (True, int(pos[hit[0]])) if hit.size else (False, int(pos[-1]))


class _RefSearch:
    def __init__(self):
        R = dqt_oracle._lib()
        L = self.L = R.L
        self.wbuf_off = R.wbuf_off
        # bool CwindowBuf::BufSearch(unsigned long nStartPos, unsigned nSearchVal, unsigned nSearchLen, bool bDirFwd,
        #                            unsigned long& nFoundPos)
        self.search = L._ZN10CwindowBuf9BufSearchEmjjbRm
        self.search.argtypes = [C.c_void_p, C.c_ulong, C.c_uint, C.c_uint, C.c_bool, C.POINTER(C.c_ulong)]
        self.search.restype = C.c_bool
        # bool CwindowBuf::OverlayInstall(unsigned nOvrInd, BYTE* pOverlay, unsigned nLen, unsigned nBegin, unsigned nMcuX,
        #                                 unsigned nMcuY, unsigned nMcuLen, unsigned nMcuLenIns, int nAdjY, int nAdjCb, int nAdjCr)
        self.install = L._ZN10CwindowBuf14OverlayInstallEjPhjjjjjjiii
        self.install.argtypes = [C.c_void_p, C.c_uint, C.c_void_p] + [C.c_uint] * 5 + [C.c_int] * 3
        self.install.restype = C.c_bool


_rs = None


def ref_bufsearch(data, start, value, length, forward, overlays=()):
    """(found, position) from the reference's compiled BufSearch over `data` with `overlays` [(offset, bytes)] installed."""
    global _rs
    if _rs is None:
        _rs = _RefSearch()
    R = _rs
    buf = np.frombuffer(bytes(data), np.uint8).copy() if not isinstance(data, np.ndarray) else data
    keep = [np.frombuffer(bytes(b), np.uint8).copy() for _, b in overlays]
    c = R.L.ref_create()
    try:
        R.L.ref_set_file(c, buf.ctypes.data, buf.size)
        for k, ((o, _), a) in enumerate(zip(overlays, keep)):
            assert R.install(c + R.wbuf_off, k, a.ctypes.data, a.size, o, 0, 0, 0, 0, 0, 0, 0)
        pos = C.c_ulong(0)
        found = R.search(c + R.wbuf_off, start, value, length, bool(forward), C.byref(pos))
        return bool(found), int(pos.value)
    finally:
        R.L.ref_destroy(c)


class RefN1:
    """The reference's parser and decoder (libn1_ref.so, float IDCT) processing a file from a start offset."""

    def __init__(self):
        L = self.L = C.CDLL(os.path.join(REF_DIR, "libn1_ref.so"), mode=os.RTLD_LOCAL | os.RTLD_DEEPBIND)
        L.n1_create.restype = C.c_void_p
        L.n1_destroy.argtypes = [C.c_void_p]
        L.n1_process.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.n1_num_lines.argtypes = [C.c_void_p]
        L.n1_line.restype = C.c_char_p; L.n1_line.argtypes = [C.c_void_p, C.c_int]
        L.n1_image_size.argtypes = [C.c_void_p, C.c_void_p]
        L.n1_pix.restype = C.POINTER(C.c_int16); L.n1_pix.argtypes = [C.c_void_p, C.c_int]
        L.n1_dib.restype = C.POINTER(C.c_uint8); L.n1_dib.argtypes = [C.c_void_p]
        L.n1_preview_ready.argtypes = [C.c_void_p]
        L.n1_config.argtypes = [C.c_int, C.c_int]
        self.status = L._ZN11CjfifDecode15GetDecodeStatusEv
        self.status.argtypes = [C.c_void_p]; self.status.restype = C.c_bool
        self.detail = L._ZN10CimgDecode12SetDetailVlcEbjjj
        self.detail.argtypes = [C.c_void_p, C.c_bool, C.c_uint, C.c_uint, C.c_uint]; self.detail.restype = None
        self.mcu_pos = L._ZN10CimgDecode16LookupFilePosMcuEjjRjS0_
        self.mcu_pos.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.POINTER(C.c_uint), C.POINTER(C.c_uint)]; self.mcu_pos.restype = None
        self.blk = L._ZN10CimgDecode12LookupBlkYCCEjjRiS0_S0_
        self.blk.argtypes = [C.c_void_p, C.c_uint, C.c_uint] + [C.POINTER(C.c_int)] * 3; self.blk.restype = None
        self.c = C.c_void_p(L.n1_create())
        # theApp.m_pAppConfig (oracle/compat_n1/JPEGsnoop.h: after CWinApp's vtable pointer) -> the harness's CSnoopConfig;
        # bDecodeScanImg / bDecodeScanImgAc are its bytes 2 and 3, nPosStart (unsigned long) its bytes 24..31
        # (oracle/compat_n1/SnoopConfig.h).  Both offsets are checked here and by the "Start Offset" line of every process().
        app = C.addressof(C.c_uint8.in_dll(L, "theApp"))
        self.cfg = C.c_void_p.from_address(app + 8).value
        L.n1_config(0, 1)
        ok = C.c_uint8.from_address(self.cfg + 2).value == 0 and C.c_uint8.from_address(self.cfg + 3).value == 1
        L.n1_config(1, 1)
        ok = ok and C.c_uint8.from_address(self.cfg + 2).value == 1
        assert ok, "CSnoopConfig layout changed: nPosStart is not where RefN1 expects it"
        self.pos_start = C.c_ulong.from_address(self.cfg + 24)
        self.img = self.jfif = None
        self._detail = None

    def close(self):
        if self.c:
            self.L.n1_destroy(self.c); self.c = None

    def _locate(self, buf):
        # N1 is {CDocLog, CwindowBuf, CFile, CimgDecode* img, CjfifDecode* jfif, std::vector<uint8_t> data}: the vector's
        # begin/end pair is the one that spans a copy of the file just processed; the two pointers precede it.
        # The window buffer's 500 overlay pointers put the pair near word 530; words are read in order up to it.
        words = np.ctypeslib.as_array(C.cast(self.c, C.POINTER(C.c_uint64)), shape=(1024,))
        for k in range(2, 1023):
            b, e = int(words[k]), int(words[k + 1])
            if b and e - b == buf.size and C.string_at(b, min(buf.size, 64)) == buf[:64].tobytes():
                self.img, self.jfif = int(words[k - 2]), int(words[k - 1])
                return
        raise AssertionError("N1 layout changed: the parser and decoder pointers were not found")

    def set_detail(self, x, y, n):
        self._detail = (x, y, n)

    def process(self, data, pos=0):
        """ProcessFile with nPosStart = pos; returns the log lines."""
        buf = np.frombuffer(bytes(data), np.uint8).copy() if not isinstance(data, np.ndarray) else data
        if self.img is None:
            self.pos_start.value = 0
            self.L.n1_process(self.c, buf.ctypes.data, buf.size)
            self._locate(buf)
        if self._detail:
            self.detail(self.img, True, *self._detail)
        self.pos_start.value = pos
        self.L.n1_process(self.c, buf.ctypes.data, buf.size)
        self.pos_start.value = 0
        lines = [self.L.n1_line(self.c, i).decode("latin-1") for i in range(self.L.n1_num_lines(self.c))]
        assert ("Start Offset: 0x%08X" % pos) in lines, "nPosStart was not applied"
        return lines

    def decode_status(self):
        return bool(self.status(self.jfif))

    def outputs(self):
        """Everything of the last process the tests compare: padded size, pixel maps, DIB, per-MCU file positions (byte, bit)
        and per-block DC values, through the reference's getters."""
        xy = np.zeros(2, np.uint32); self.L.n1_image_size(self.c, xy.ctypes.data)
        W, H = int(xy[0]), int(xy[1])
        out = {"size": (W, H), "ready": bool(self.L.n1_preview_ready(self.c))}
        for k, name in enumerate(("y", "cb", "cr")):
            p = self.L.n1_pix(self.c, k)
            out[name] = np.ctypeslib.as_array(p, shape=(H, W)).copy() if p and W and H else None
        p = self.L.n1_dib(self.c)
        out["dib"] = np.ctypeslib.as_array(p, shape=(H, W, 4)).copy() if p and W and H else None
        return out

    def mcu_map(self, mx, my):
        a, b = C.c_uint(), C.c_uint()
        out = np.zeros((my, mx, 2), np.uint32)
        for y in range(my):
            for x in range(mx):
                self.mcu_pos(self.img, x, y, C.byref(a), C.byref(b)); out[y, x] = (a.value, b.value)
        return out

    def blk_dc(self, bx, by):
        y, cb, cr = C.c_int(), C.c_int(), C.c_int()
        out = np.zeros((by, bx, 3), np.int32)
        for j in range(by):
            for i in range(bx):
                self.blk(self.img, i, j, C.byref(y), C.byref(cb), C.byref(cr)); out[j, i] = (y.value, cb.value, cr.value)
        return out


def scan_lines(lines):
    """The lines DecodeScanImg wrote into a ProcessFile log: from its header to its trailing blank line."""
    i = lines.index("*** Decoding SCAN Data ***")
    return lines[i:]


def ref_doc_search(data, start, forward, search=None):
    """OnToolsSearchforward / OnToolsSearchreverse over BufSearch: (found, new start, reprocess?)."""
    search = search or ref_bufsearch
    if not forward and start == 0:
        return False, 0, False
    found, pos = search(data, start, SOI3, 3, forward)
    if found:
        return True, pos, True
    return (False, start, False) if forward else (False, 0, True)


def ref_offset_mode(data, mode, pos, n1, search=None):
    """DoAnalyzeOffset: the offset the reference decodes at last; n1 is a RefN1 (SRCH1 asks its GetDecodeStatus at 0)."""
    search = search or ref_bufsearch
    if mode == 0:
        return 0
    if mode == 3:
        return pos
    if mode == 1:
        n1.process(data, 0)
        if n1.decode_status():
            return 0
    found, p = search(data, 0, SOI3, 3, True)
    return p if found else 0
