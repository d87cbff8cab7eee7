"""TEST INFRASTRUCTURE: the reference's "Search Executable for DQT" on the CPU, for tests/test_dqt_search.py and
tools/dqt_search_probe.py.

* ref_bufsearch_all(data, pat): the Doc's repeated search loop (JPEGsnoopDoc.cpp:1500-1512) -- start at 0, report the find,
  start again one past it -- over the reference's own CwindowBuf::BufSearchX (WindowBuf.cpp:243-331) as oracle/Makefile
  compiled it, unmodified, into oracle/_ref/liboracle_ref_fixed.so.  The window buffer is the one of a fresh harness
  context (oracle/ref_harness.cpp: RefCtx, filled by ref_set_file); the exported member function is called on it directly.
* ref_search_dqt(...): the rest of OnToolsSearchexecutablefordqt (:1305-1519) restated line for line over that search,
  the reference's compiled glb_anZigZag / glb_anStdQuantLum (General.cpp) and, for an analysed JPEG, GetDqtEntry(0, .) of
  the reference's CimgDecode after the reference's own CjfifDecode parsed it (oracle/_ref/libn1_ref.so).
Both need the compiled reference (ref_available()).
"""
import ctypes as C
import os
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")

_ref = None


def ref_available():
    return all(os.path.exists(os.path.join(REF_DIR, f)) for f in ("liboracle_ref_fixed.so", "libn1_ref.so"))


class _Ref:
    def __init__(self):
        L = C.CDLL(os.path.join(REF_DIR, "liboracle_ref_fixed.so"))
        L.ref_create.restype = C.c_void_p
        L.ref_destroy.argtypes = [C.c_void_p]
        L.ref_set_file.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        # bool CwindowBuf::BufSearchX(unsigned long nStartPos, BYTE* anSearchVal, unsigned nSearchLen, bool bDirFwd,
        #                             unsigned long& nFoundPos)  and  unsigned long CwindowBuf::GetPosEof()
        self.search = L._ZN10CwindowBuf10BufSearchXEmPhjbRm
        self.search.argtypes = [C.c_void_p, C.c_ulong, C.c_void_p, C.c_uint, C.c_bool, C.POINTER(C.c_ulong)]
        self.search.restype = C.c_bool
        self.eof = L._ZN10CwindowBuf9GetPosEofEv
        self.eof.argtypes = [C.c_void_p]; self.eof.restype = C.c_ulong
        self.zigzag = list((C.c_uint * 64).in_dll(L, "glb_anZigZag"))
        self.std_lum = list((C.c_uint * 64).in_dll(L, "glb_anStdQuantLum"))
        self.L = L
        # RefCtx is {CDocLog log; CwindowBuf wbuf; ...}: the window buffer follows the 80-byte log stand-in
        # (oracle/compat/DocLog.h: three vectors and two flags).  Checked here against the file size the buffer reports.
        self.wbuf_off = 80
        probe = np.zeros(12345, np.uint8)
        c = L.ref_create()
        L.ref_set_file(c, probe.ctypes.data, probe.size)
        ok = self.eof(c + self.wbuf_off) == probe.size
        L.ref_destroy(c)
        assert ok, "RefCtx layout changed: the window buffer is not where ref_search expects it"
        N = C.CDLL(os.path.join(REF_DIR, "libn1_ref.so"))
        N.n1_create.restype = C.c_void_p
        N.n1_destroy.argtypes = [C.c_void_p]
        N.n1_process.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        N.n1_dqt.argtypes = [C.c_void_p, C.c_uint, C.c_uint]; N.n1_dqt.restype = C.c_uint
        self.N = N


def _lib():
    global _ref
    if _ref is None:
        _ref = _Ref()
    return _ref


def ref_bufsearch_all(data, pat):
    """Positions the Doc's loop reports for `pat` in `data`, from the compiled BufSearchX."""
    R = _lib()
    buf = np.frombuffer(bytes(data), np.uint8).copy() if not isinstance(data, np.ndarray) else data
    p = np.frombuffer(bytes(pat), np.uint8).copy()
    c = R.L.ref_create()
    try:
        R.L.ref_set_file(c, buf.ctypes.data, buf.size)
        out, start, found = [], 0, C.c_ulong(0)
        while R.search(c + R.wbuf_off, start, p.ctypes.data, p.size, True, C.byref(found)):
            out.append(found.value)
            start = found.value + 1
        return out
    finally:
        R.L.ref_destroy(c)


def ref_analysed_table(jpeg):
    """GetDqtEntry(0, 0..63) of the reference's CimgDecode after the reference's CjfifDecode analysed `jpeg`."""
    R = _lib()
    buf = np.frombuffer(bytes(jpeg), np.uint8).copy()
    c = R.N.n1_create()
    try:
        R.N.n1_process(c, buf.ctypes.data, buf.size)
        return [int(R.N.n1_dqt(c, 0, i)) for i in range(64)]
    finally:
        R.N.n1_destroy(c)


def dqt_pattern(values, width, swap, baseline):
    """The search matrix of one layout (JPEGsnoopDoc.cpp:1456-1496): `values` in search order."""
    out = bytearray(64 * width)
    for i, v in enumerate(values):
        e = i * width
        if width == 1:
            out[e] = v & 0xFF
        elif swap:
            out[e] = v & 0xFF
            if not baseline:
                out[e + 1] = (v & 0xFF00) >> 8
        else:
            out[e + width - 1] = v & 0xFF
            if not baseline:
                out[e + width - 2] = (v & 0xFF00) >> 8
    return bytes(out)


LAYOUTS = [(1, False), (2, False), (2, True), (4, False), (4, True)]


def ref_search_dqt(data, exe_path, analysed_jpeg=None, analysed_path="", search=None):
    """(kind, line) of every log line the Doc writes; kind is the CDocLog call: hdr, line, warn or good.
    `search(data, pattern)` defaults to ref_bufsearch_all."""
    R = _lib()
    search = search or ref_bufsearch_all
    n = len(data)
    out = [("hdr", "*** Searching Executable for DQT ***"), ("line", f"  Filename: [{exe_path}]"), ("line", f"  Size:     [{n}]")]
    set_max, all_same, baseline, tbl = 1, True, True, None
    if analysed_jpeg is not None:
        tbl = ref_analysed_table(analysed_jpeg)
        for i in range(1, 64):
            if tbl[i] != tbl[0]:
                all_same = False
            if tbl[i] > 255:
                baseline = False
        if all_same:
            out += [("warn", "  NOTE: Because the JPEG's DQT Luminance table is constant nValue (0x%02X),_T(" % tbl[0]),
                    ("warn", ")        matching for this table has been disabled."),
                    ("warn", "        Please select a different reference image.")]
        else:
            set_max = 2
    out.append(("line", "  Searching for DQT Luminance tables:"))
    for zz in range(2):
        out.append(("line", "    DQT Ordering: %s" % ("post-zigzag" if zz else "pre-zigzag")))
        for s in range(set_max):
            out.append(("line", "      Matching [JPEG Standard]" if s == 0 else f"      Matching [{analysed_path}]"))
            for width, swap in LAYOUTS:
                if width == 1:
                    out.append(("line", "        Searching patterns with 1-byte DQT entries"))
                    if not baseline:
                        out.append(("line", "          DQT Table is not baseline, skipping 1-byte search"))
                        continue
                else:
                    out.append(("line", "        Searching patterns with %u-byte DQT entries%s" % (width, ", endian byteswap" if swap else "")))
                idx = [k if zz else R.zigzag[k] for k in range(64)]
                vals = [R.std_lum[i] if s == 0 else tbl[i] for i in idx]
                for p in search(data, dqt_pattern(vals, width, swap, baseline)):
                    out.append(("good", "          Found @ 0x%08X" % p))
    out.append(("line", "  Done Search"))
    return out
