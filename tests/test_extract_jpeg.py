"""Extract embedded JPEG and Extract All against the compiled reference.

The reference side is CjfifDecode's own ProcessFile, ExportJpegPrepare and ExportJpegDo (oracle/_ref/libn1_ref.so), called
as JPEGsnoopCore.cpp:913-961 calls them: nPosStart set, the file processed, then the two export members on the harness's
parser with the window buffer attached again (the harness detaches it after ProcessFile).  Extract All is the loop of
JPEGsnoopCore.cpp:963-1088 restated over those calls and the reference's BufSearch.

* CPU: the terminator rule (mjpg_corpus.scan_end_marker, extended to the last byte) against the position where the
  reference's PASS 1 stops, on crafted scans; the oracle's own bookkeeping.
* GPU: jsgpu_find_markers against the model (chunk edges, halo, unaligned buffers, overlays, many terminators, caps, the
  2^32 limit); every exported file and its log lines against the reference's for the corpus and option combinations;
  Extract All over a 2 000-frame AVI; a resident batch left untouched.
"""
import ctypes as C
import os

import numpy as np
import pytest

import jpeg_cases as JC
import mjpg_corpus as MC
from find_oracle import RefN1, ref_available, ref_bufsearch

pytestmark = pytest.mark.skipif(not ref_available(), reason="compiled reference not available")

OPTS = ("overlay", "force_soi", "force_eoi", "ignore_eoi", "dht_avi_insert")
SRC = "source.bin"


# ---- the model --------------------------------------------------------------------------------------------------------
def term_model(data, overlays=()):
    """Every p in [0, n - 2] with byte p == FF and byte p + 1 neither 00 nor D0..D7 (overlays applied inside the file)."""
    d = np.frombuffer(bytes(data), np.uint8).copy()
    for o, b in overlays:
        b = np.frombuffer(bytes(b), np.uint8)[:max(0, d.size - o)]
        d[o:o + b.size] = b
    if d.size < 2:
        return np.zeros(0, np.int64)
    nxt = d[1:]
    return np.flatnonzero((d[:-1] == 0xFF) & (nxt != 0) & ((nxt & 0xF8) != 0xD0))


def soi_model(data, overlays=()):
    d = np.frombuffer(bytes(data), np.uint8).copy()
    for o, b in overlays:
        b = np.frombuffer(bytes(b), np.uint8)[:max(0, d.size - o)]
        d[o:o + b.size] = b
    return MC.find_all_model(d)


# ---- the reference ----------------------------------------------------------------------------------------------------
class RefExport(RefN1):
    """RefN1 plus the reference's export members and overlays on the harness's window buffer."""

    WBUF = 80                                  # N1 = {CDocLog (three vectors, two flags: 80 bytes), CwindowBuf, CFile, ...}
    CFILE = 40                                 # oracle/compat/mfc_stub.h CFile: vtable, m_p, m_n, m_pos, m_f

    def __init__(self):
        super().__init__()
        L = self.L
        self.prep = L._ZN11CjfifDecode17ExportJpegPrepareE7CStringbbb
        self.prep.argtypes = [C.c_void_p, C.c_void_p, C.c_bool, C.c_bool, C.c_bool]; self.prep.restype = C.c_bool
        self.do = L._ZN11CjfifDecode12ExportJpegDoE7CStringS0_mbbbb
        self.do.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_ulong] + [C.c_bool] * 4; self.do.restype = C.c_bool
        self.fset = L._ZN10CwindowBuf10BufFileSetEP5CFile
        self.fset.argtypes = [C.c_void_p, C.c_void_p]; self.fset.restype = None
        self.install = L._ZN10CwindowBuf14OverlayInstallEjPhjjjjjjiii
        self.install.argtypes = [C.c_void_p, C.c_uint, C.c_void_p] + [C.c_uint] * 5 + [C.c_int] * 3
        self.install.restype = C.c_bool
        self.remove = L._ZN10CwindowBuf16OverlayRemoveAllEv
        self.remove.argtypes = [C.c_void_p]; self.remove.restype = None
        self.cstr = L._ZN7CStringC1EPKc
        self.cstr.argtypes = [C.c_void_p, C.c_char_p]; self.cstr.restype = None
        self._keep = []

    def _cstring(self, s):
        buf = C.create_string_buffer(64)       # a std::string (32 bytes); never destroyed, the test's lifetime holds it
        self.cstr(buf, s.encode())
        self._keep.append(buf)
        return buf

    def _file(self, buf):
        words = np.ctypeslib.as_array(C.cast(self.c, C.POINTER(C.c_uint64)), shape=(1024,))
        k = int(np.flatnonzero(words == self.img)[0])
        f = self.c.value + 8 * k - self.CFILE
        assert C.c_uint64.from_address(f + 16).value == buf.size, "N1 layout changed: the CFile is not where expected"
        return f

    def lines(self):
        return [self.L.n1_line(self.c, i).decode("latin-1") for i in range(self.L.n1_num_lines(self.c))]

    def export(self, data, pos, out, opts=(), overlays=(), src=SRC):
        """ProcessFile at pos, ExportJpegPrepare, ExportJpegDo: (written?, the export's log lines)."""
        buf = np.frombuffer(bytes(data), np.uint8).copy()
        wbuf = self.c.value + self.WBUF
        keep = [np.frombuffer(bytes(b), np.uint8).copy() for _, b in overlays]
        self.remove(wbuf)
        for k, ((o, _), a) in enumerate(zip(overlays, keep)):
            assert self.install(wbuf, k, a.ctypes.data, a.size, o, 0, 0, 0, 0, 0, 0, 0)
        # the scan decode does not touch the export state: skip it, then restore the library-wide setting RefN1 leaves
        self.L.n1_config(0, 1)
        try:
            self.process(buf, pos)
            self.fset(wbuf, self._file(buf))
            o = dict.fromkeys(OPTS, False); o.update(dict.fromkeys(opts, True))
            n0 = len(self.lines())
            ok = self.prep(self.jfif, self._cstring(src), o["force_soi"], o["force_eoi"], o["ignore_eoi"])
            if ok:
                ok = self.do(self.jfif, self._cstring(src), self._cstring(str(out)), buf.size, o["overlay"],
                             o["dht_avi_insert"], o["force_soi"], o["force_eoi"])
            return bool(ok), self.lines()[n0:]
        finally:
            self.remove(wbuf)
            self.L.n1_config(1, 1)

    def extract_all(self, data, out_name, opts=(), overlays=(), src=SRC):
        """JPEGsnoopCore.cpp:963-1088 over the reference's calls: ([(offset, path or None)], log lines)."""
        if "." not in out_name:
            return [], ["ERROR: Invalid filename [%s]" % out_name]
        root = out_name[:out_name.rfind(".")]
        frames, lines, cnt, pos = [], [], 1, 0
        while True:
            name = "%s.%06u.jpg" % (root, cnt)
            ok, ln = self.export(data, pos, name, opts, overlays, src)
            lines += ln
            prepared = any(s.startswith("  Exporting to:") for s in ln)
            frames.append((pos, name if ok else None))
            cnt += prepared
            found, nxt = ref_bufsearch(data, pos, 0xFFD8FF, 3, True, overlays)
            if not found:
                return frames, lines
            pos = nxt


@pytest.fixture(scope="module")
def ref(built):
    r = RefExport()
    yield r
    r.close()


# ---- corpus -----------------------------------------------------------------------------------------------------------
def _progressive():
    return JC.enc(JC.synth_rgb(64, 48, 5), quality=80, progressive=True)


def _scan_start(j):
    return MC.segments(j)[-1][2]


def _pad_to(j, which, k):
    """j with a COM segment (header part) or stuffed bytes (scan part) so that part has k * 131072 + 1 bytes."""
    sos = MC.segments(j)[-1][1]
    if which == "head":
        need = k * 131072 + 1 - sos
        parts = []
        while need > 0:
            L = min(need, 65535 + 2)
            if need - L in (1, 2, 3):          # a segment is at least 4 bytes
                L -= 4
            parts.append(b"\xff\xfe" + (L - 2).to_bytes(2, "big") + bytes(L - 4))
            need -= L
        return j[:2] + b"".join(parts) + j[2:]
    need = k * 131072 + 1 - (len(j) - sos)
    s = _scan_start(j)                         # zero bytes are 8 zero bits of the last code: pad after the scan's first byte
    return j[:s + 1] + bytes(need) + j[s + 1:]


def corpus():
    """(name, data, offset, [option sets], overlays)"""
    base = MC.frame(3, "420")
    ex, thumb = MC.exif_jpeg(9)
    mj = MC.to_mjpg(MC.frame(4, "422_dri"))
    avi, offs = MC.avi(MC.mjpg_frames(6, 5))
    trunc = base[:_scan_start(base) + 40]
    dqt = [a for m, a, _ in MC.segments(base) if m == 0xDB][0]
    sos = MC.segments(base)[-1][1]
    none, f_eoi, i_eoi = (), ("force_eoi",), ("ignore_eoi",)
    out = [
        ("baseline", base, 0, [none, f_eoi, ("force_soi",), ("dht_avi_insert",)], ()),
        ("exif", ex, 0, [none], ()),
        ("exif_thumb", ex, thumb, [none], ()),
        ("progressive", _progressive(), 0, [none, f_eoi], ()),
        ("mjpg", mj, 0, [none, ("dht_avi_insert",)], ()),
        ("avi_frame", avi, offs[2], [none, ("dht_avi_insert",)], ()),
        ("avi_offset0", avi, 0, [none, f_eoi, i_eoi, ("force_soi", "ignore_eoi")], ()),
        ("truncated", trunc, 0, [none, f_eoi, i_eoi], ()),
        ("truncated_ff_last", trunc[:-1] + b"\xff", 0, [none, f_eoi, i_eoi], ()),
        ("fill_before_eoi", base[:-2] + b"\xff\xff\xff\xd9", 0, [none, f_eoi], ()),
        ("at_dqt", base, dqt, [none, ("force_soi",), ("force_soi", "force_eoi")], ()),
        ("head_131073", _pad_to(base, "head", 1), 0, [none, ("force_soi",)], ()),
        ("scan_131073", _pad_to(base, "scan", 1), 0, [none, f_eoi], ()),
        ("overlay_marker", base, 0, [none, ("overlay",)], [(sos - 20, b"\x12\x34\x56")]),
        ("overlay_kills_eoi", base, 0, [none, ("overlay", "ignore_eoi"), ("ignore_eoi",)], [(len(base) - 2, b"\x00")]),
    ]
    return out


def _cases():
    for name, data, pos, optsets, ovl in corpus():
        for o in optsets:
            yield name, data, pos, o, ovl


# ---- CPU --------------------------------------------------------------------------------------------------------------
def _crafted_scans():
    base = MC.frame(11, "420_dri")
    s = _scan_start(base)
    body = base[s:-2]
    return [
        ("rst_and_stuffing", base),
        ("fill_before_eoi", base[:-2] + b"\xff\xff\xff\xd9"),
        ("ff00_run", base[:s] + b"\xff\x00" * 8 + body + b"\xff\xd9"),
        ("ff_last_byte", base[:s] + body + b"\xff"),
        ("runs_to_eof", base[:s] + body),
        ("rst_then_com", base[:s] + body + b"\xff\xd3\xff\xfe\x00\x04ab\xff\xd9"),
    ]


def _ref_scan_end(lines):
    """Where the reference's PASS 1 stopped: the marker after the SOS, at its OFFSET less its pad bytes; None when the walk
    ran out of buffer."""
    i = max(k for k, s in enumerate(lines) if s.startswith("*** Marker: SOS"))
    if any("Ran out of buffer" in s for s in lines[i:]):
        return None
    pad = 0
    for s in lines[i + 1:]:
        if s.startswith("*** Skipped "):
            pad = int(s.split()[2])
        if s.startswith("*** Marker: ") and "SOS" not in s:
            j = lines.index(s, i + 1)
            off = next(t for t in lines[j:] if t.startswith("  OFFSET: 0x"))
            return int(off.split("0x")[1], 16) - pad
    return None


@pytest.mark.parametrize("name,data", _crafted_scans(), ids=[n for n, _ in _crafted_scans()])
def test_terminator_model_is_where_pass1_stops(ref, name, data):
    lines = ref.process(np.frombuffer(data, np.uint8).copy(), 0)
    t = term_model(data)
    s = _scan_start(data)
    after = t[t >= s]
    want = _ref_scan_end(lines)
    assert (int(after[0]) if after.size else None) == want, name


def test_reference_export_runs_and_reports(ref, tmp_path):
    base = MC.frame(3, "420")
    ok, lines = ref.export(base, 0, tmp_path / "a.jpg")
    assert ok and (tmp_path / "a.jpg").read_bytes() == base
    assert lines[1] == "*** Exporting JPEG ***" and lines[-1] == "  Export done"
    ok, lines = ref.export(base, 0, SRC)
    assert not ok and "ERROR: Can't overwrite source file. Aborting export." in lines


def test_reference_copy_loses_the_last_byte_of_a_131073_byte_scan_part(ref, tmp_path):
    j = _pad_to(MC.frame(3, "420"), "scan", 1)
    assert len(j) - MC.segments(j)[-1][1] == 131073
    ok, _ = ref.export(j, 0, tmp_path / "b.jpg")
    assert ok and (tmp_path / "b.jpg").read_bytes() == j[:-1]


# ---- GPU --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bd(built):
    from jpegsnoop_b200 import BatchDecoder
    b = BatchDecoder(device=0)
    yield b
    b.close()


def find_markers(bd, data, overlays=(), soi_cap=None, term_cap=None):
    from jpegsnoop_b200 import _lib as B
    buf = data if isinstance(data, np.ndarray) else np.frombuffer(bytes(data), np.uint8)
    keep = [np.frombuffer(bytes(b), np.uint8) for _, b in overlays]
    ov = (B.jsgpu_overlay * max(len(keep), 1))(*[B.jsgpu_overlay(int(o), a.size, a.ctypes.data) for (o, _), a in zip(overlays, keep)])
    sc = buf.size if soi_cap is None else soi_cap
    tc = buf.size if term_cap is None else term_cap
    soi = np.zeros(max(sc, 1), np.uint32); term = np.zeros(max(tc, 1), np.uint32)
    ns, nt = C.c_uint64(), C.c_uint64()
    r = bd.L.jsgpu_find_markers(bd.ctx, buf.ctypes.data, buf.size, ov, len(keep), soi.ctypes.data, sc, C.byref(ns),
                                term.ctypes.data, tc, C.byref(nt))
    return r, int(ns.value), soi[:min(sc, ns.value)], int(nt.value), term[:min(tc, nt.value)]


def _check(bd, data, overlays=()):
    r, ns, soi, nt, term = find_markers(bd, data, overlays)
    assert r == 0
    ws, wt = soi_model(data, overlays), term_model(data, overlays)
    assert ns == ws.size and np.array_equal(soi, ws)
    assert nt == wt.size and np.array_equal(term, wt)


@pytest.mark.gpu
def test_gpu_find_markers_crafted(bd):
    for _, data in _crafted_scans():
        _check(bd, data)
    for data in (b"", b"\xff", b"\xff\xd9", b"\xff\xd8\xff", b"\xff\xff\xff", b"\xff\x00\xff\xd0\xff\xd7\xff\xd8\xff\xc0"):
        _check(bd, data)


@pytest.mark.gpu
def test_gpu_find_markers_chunk_edges_halo_and_unaligned(built, monkeypatch):
    from jpegsnoop_b200 import BatchDecoder
    monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", "4096")
    b = BatchDecoder(device=0)
    try:
        rng = np.random.default_rng(3)
        for n in (4095, 4096, 4097, 8192, 8193, 3 * 4096 + 2):
            d = rng.integers(0, 0xC0, n + 64, dtype=np.uint8)
            for e in (4093, 4094, 4095, 4096, 8190, 8191, n - 3, n - 2, n - 1):
                if 0 <= e and e + 3 <= d.size:
                    d[e:e + 3] = (0xFF, 0xD8, 0xFF)
            for off in (0, 1, 3, 7):           # unaligned host buffers
                _check(b, d[off:off + n])
        # overlays that create and remove terminators across a chunk edge
        d = rng.integers(0, 0xC0, 3 * 4096, dtype=np.uint8)
        d[4095:4097] = (0xFF, 0xC4)
        _check(b, d, [(4095, b"\x00"), (8191, b"\xff\xda"), (100, b"\xff\xd8\xff")])
    finally:
        b.close()


@pytest.mark.gpu
def test_gpu_find_markers_many_terminators_caps_and_limit(bd):
    d = np.tile(np.array([0xFF, 0xC4, 0x11], np.uint8), 500_000)        # 500 000 terminators ...
    d = np.concatenate([d, np.tile(np.array([0xFF, 0xD8, 0xFF, 0xE0], np.uint8), 300_000)])   # ... and 900 000 more
    _check(bd, d)
    r, ns, soi, nt, term = find_markers(bd, d, soi_cap=1000, term_cap=12345)
    wt, ws = term_model(d), soi_model(d)
    assert r == 0 and nt == wt.size > 10 ** 6 and ns == ws.size
    assert np.array_equal(term, wt[:12345]) and np.array_equal(soi, ws[:1000])
    r, ns, _, nt, _ = find_markers(bd, d, soi_cap=0, term_cap=0)
    assert r == 0 and (ns, nt) == (ws.size, wt.size)
    big = np.zeros(1, np.uint8)
    ns, nt = C.c_uint64(), C.c_uint64()
    assert bd.L.jsgpu_find_markers(bd.ctx, big.ctypes.data, 1 << 32, None, 0, None, 0, C.byref(ns), None, 0, C.byref(nt)) != 0


def _ours(data, pos, out, opts, overlays):
    from jpegsnoop_b200 import CimgDecode
    dec = CimgDecode(device=0)
    try:
        return dec.export_jpeg(data, out, offset=pos, overlays=overlays, src_name=SRC, **dict.fromkeys(opts, True))
    finally:
        dec.close()


def _read(p):
    return open(p, "rb").read() if os.path.exists(p) else None


@pytest.mark.gpu
@pytest.mark.parametrize("name,data,pos,opts,ovl", list(_cases()), ids=[f"{c[0]}-{'+'.join(c[3]) or 'none'}" for c in _cases()])
def test_gpu_export_equals_the_reference(ref, tmp_path, name, data, pos, opts, ovl):
    want_ok, want_lines = ref.export(data, pos, tmp_path / "ref.jpg", opts, ovl)
    got_ok, got_lines = _ours(data, pos, tmp_path / "ours.jpg", opts, ovl)
    assert bool(got_ok) == want_ok
    assert [s.replace("ref.jpg", "ours.jpg") for s in want_lines] == got_lines
    assert _read(tmp_path / "ours.jpg") == _read(tmp_path / "ref.jpg")


@pytest.mark.gpu
def test_gpu_export_refuses_to_overwrite_the_source(ref, tmp_path):
    base = MC.frame(3, "420")
    want_ok, want_lines = ref.export(base, 0, SRC)
    got_ok, got_lines = _ours(base, 0, SRC, (), ())
    assert not want_ok and not got_ok and want_lines == got_lines


def _extract_check(ref, bd, data, tmp_path, opts=(), overlays=(), name="out.log"):
    (tmp_path / "r").mkdir(); (tmp_path / "o").mkdir()
    want, wl = ref.extract_all(data, str(tmp_path / "r" / name), opts, overlays)
    got, gl = bd.extract_all(data, str(tmp_path / "o" / name), overlays=overlays, src_name=SRC, **dict.fromkeys(opts, True))
    fix = lambda p: p and os.path.basename(p)
    assert [(o, fix(p)) for o, p in got] == [(o, fix(p)) for o, p in want]
    assert [s.replace(str(tmp_path / "r"), "") for s in wl] == [s.replace(str(tmp_path / "o"), "") for s in gl]
    assert sorted(os.listdir(tmp_path / "o")) == sorted(os.listdir(tmp_path / "r"))
    for f in os.listdir(tmp_path / "r"):
        assert _read(tmp_path / "o" / f) == _read(tmp_path / "r" / f), f
    return got


@pytest.mark.gpu
def test_gpu_extract_all_exif_yields_both_images(ref, bd, tmp_path):
    ex, thumb = MC.exif_jpeg(9)
    got = _extract_check(ref, bd, ex, tmp_path)
    assert [o for o, p in got if p] == [0, thumb]


@pytest.mark.gpu
@pytest.mark.parametrize("opts", [(), ("dht_avi_insert",), ("force_eoi", "force_soi")])
def test_gpu_extract_all_small_containers(ref, bd, tmp_path, opts):
    name, data = MC.corpus()[1]
    _extract_check(ref, bd, data, tmp_path, opts)


@pytest.mark.gpu
def test_gpu_extract_all_name_without_dot(ref, bd, tmp_path):
    got, lines = bd.extract_all(MC.frame(3, "420"), str(tmp_path / "noext"), src_name=SRC)
    want, wl = ref.extract_all(MC.frame(3, "420"), str(tmp_path / "noext"))
    assert got == want == [] and lines == wl and os.listdir(tmp_path) == []


@pytest.mark.gpu
def test_gpu_extract_all_large_avi_and_batch_untouched(ref, bd, tmp_path):
    # a resident decoded batch is left as it was
    j = MC.frame(5, "420")
    bd.set_batch([j]); bd.decode(); bd.sync()
    before = bd.fetch(0)
    data, offs = MC.avi(MC.mjpg_frames(21, 2000))
    got = _extract_check(ref, bd, data, tmp_path, ("dht_avi_insert",), name="movie.avi")
    assert [o for o, p in got if p] == offs
    after = bd.fetch(0)
    assert not JC.compare(before, after)
