"""The damaged-scan error report at every error cap, under ScanErrorsDisable and past 256 events.

JPEGsnoop reports each kind of capped scan error while fewer than CSnoopConfig::nErrMaxDecodeScan were reported
(ImgDecode.cpp:1100-1110 and its copies); four kinds of line are never capped (the RST-index mismatch :1414-1424, the missing
restart marker :3180-3200, the two "Overread ... (after ...)" lines).  ScanErrorsDisable (:1014-1018) counts the cap as used
up, Reset() keeps that count (:127), DecodeScanImg reloads the cap after Reset() (:2748-2750) and the RST-index line is dropped
while errors are disabled (:1417).  The device keeps the first 256 events of an image in jsgpu_scan_errors and walks the image
again for the others (jsgpu_batch_error_events).

The corpus reaches the edges of all of that: exactly 255, 256 and 257 events, more than 1 000 events, more capped errors than
any cap below 300, capped and uncapped lines on both sides of the cap line.  CPU tests pin the reference's behaviour on it;
GPU tests compare the CUDA path with the compiled reference: every output buffer, stats[10:12], the full log and the error
lines, at caps 0 .. 2^32 - 1, with each Huffman kernel, in ScanErrorsDisable / Enable sequences, in Detailed Decode ranges and
in mixed batches."""
import ctypes as C
import functools
import re

import numpy as np
import pytest

import jpeg_cases as JC
from oracle_util import Oracle, ref_available

needs_ref = pytest.mark.skipif(not ref_available("fixed"), reason="needs oracle/_ref (the compiled reference)")

CAPS = [0, 1, 2, 19, 20, 21, 255, 256, 257, 1000, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1]

# jsgpu.h JSGPU_EV_*
EV_OVR_BEFORE, EV_OVR_CODE, EV_OVR_BITS, EV_NOCODE, EV_CAP, EV_RST_MISMATCH, EV_MARKER, EV_BADMARK, EV_BADCODE, EV_NCOEF, \
    EV_MCU, EV_RST_MISSING = range(1, 13)
UNCAPPED = (EV_OVR_CODE, EV_OVR_BITS, EV_RST_MISMATCH, EV_RST_MISSING)

_H = r"0x([0-9A-F]{8})\.(\d+)"
_LINE_EVENTS = [          # the first line of each event as ImgDecode.cpp prints it -> (code, its numbers in jsgpu_scan_event order)
    (re.compile(r"^\*\*\* ERROR: Overread scan segment \(before nCode\)! @ Offset: " + _H + "$"), EV_OVR_BEFORE),
    (re.compile(r"^\*\*\* ERROR: Overread scan segment \(after nCode\)! @ Offset: " + _H + "$"), EV_OVR_CODE),
    (re.compile(r"^\*\*\* ERROR: Overread scan segment \(after bitstring\)! @ Offset: " + _H + "$"), EV_OVR_BITS),
    (re.compile(r"^\*\*\* ERROR: Can't find huffman bitstring @ " + _H + r", table (\d+), value \[0x([0-9a-f]{8})\]$"), EV_NOCODE),
    (re.compile(r"^    Only reported first (\d+) instances of this message\.\.\.$"), EV_CAP),
    (re.compile(r"^  ERROR: Expected RST marker index RST(\d+) got RST(\d+) @ 0x([0-9A-F]{8})\.0$"), EV_RST_MISMATCH),
    (re.compile(r"^  Scan Data encountered marker   0xFF([0-9A-F]{2}) @ 0x([0-9A-F]{8})\.0$"), EV_MARKER),
    (re.compile(r"^\*\*\* ERROR: Bad marker @ " + _H + "$"), EV_BADMARK),
    (re.compile(r"^\*\*\* ERROR: Bad huffman code @ " + _H + "$"), EV_BADCODE),
    (re.compile(r"^\*\*\* ERROR: @ " + _H + r", nNumCoeffs>64 \[(\d+)\]$"), EV_NCOEF),
    (re.compile(r"^\*\*\* ERROR: Bad scan data in MCU\((\d+),(\d+)\): (Lum|Chr\(Cb\)|Chr\(Cr\)) CSS\((\d+),(\d+)\) @ Offset " + _H + "$"), EV_MCU),
    (re.compile(r"^  Expect Restart interval elapsed @ " + _H + "$"), EV_RST_MISSING),
]
_HEX = {EV_NOCODE: (0, 3), EV_CAP: (), EV_RST_MISMATCH: (2,), EV_MARKER: (0, 1)}     # groups printed in hex (default: the offset)


def ref_events(lines):
    """The scan error events behind a reference log: [(code, a, b, c, d, e)], the columns of jsgpu_scan_event."""
    out = []
    for s in lines:
        for rx, code in _LINE_EVENTS:
            m = rx.match(s)
            if not m:
                continue
            g = list(m.groups())
            if code == EV_MCU:
                comp = ("Lum", "Chr(Cb)", "Chr(Cr)").index(g[2])
                v = [int(g[0]), int(g[1]), comp | int(g[3]) << 8 | int(g[4]) << 16, int(g[5], 16), int(g[6])]
            else:
                v = [int(x, 16) if i in _HEX.get(code, (0,)) else int(x) for i, x in enumerate(g)]
            out.append(tuple([code] + v + [0] * (5 - len(v))))
            break
    return out


def _capped(ev):
    return [e for e in ev if e[0] not in UNCAPPED and e[0] != EV_CAP]


# --- corpus -----------------------------------------------------------------------------------------------------------------

def _rst_positions(j):
    lo = j.index(b"\xff\xda") + 14
    return [i for i in range(lo, len(j) - 1) if j[i] == 0xFF and 0xD0 <= j[i + 1] <= 0xD7]


def _relabel_rst0(j, idx):
    a = bytearray(j); rp = _rst_positions(j)
    for i in idx:
        a[rp[i] + 1] = 0xD0
    return bytes(a)


def _flipped(j, n, seed, upto=1.0):
    """n random bit flips in the scan, within its first `upto` part."""
    r = np.random.default_rng(seed)
    a = bytearray(j); lo = j.index(b"\xff\xda") + 14
    for p in r.integers(lo, lo + int((len(j) - 2 - lo) * upto), n):
        a[p] ^= 1 << int(r.integers(0, 8))
    return bytes(a)


@functools.lru_cache(maxsize=1)
def corpus():
    """name -> jpeg bytes.  The base image is small_cases()[2]: 1920x1080 4:2:0, DRI = 4, 2 039 RST markers."""
    small = JC.small_cases()
    good = small[2][1]
    rp = _rst_positions(good)
    n = len(rp)
    removed = bytearray(); prev = 0
    for p in rp[10:]:                               # every marker from the 11th on taken out
        removed += good[prev:p]; prev = p + 2
    removed = bytes(removed + good[prev:])
    nodri = small[3][1]
    body = nodri.index(b"\xff\xda") + 14
    gray = small[4][1]
    assert gray.endswith(b"\xff\xd9")
    return {
        # every marker relabelled RST0: 2 038 uncapped RST-index lines (one of them is RST0 where RST0 is due)
        "all_rst0": _relabel_rst0(good, range(n)),
        # the last k relabelled: k - 1 or k RST-index lines (none for a marker that already was RST0) and the EOI note, so at the
        # default cap 254 -> 255 events, 256 -> 257, and at cap 1 254 -> 256 (note + cap line); test_corpus_reaches_the_edges
        # shows the counts on the reference's own log
        "last254_rst0": _relabel_rst0(good, range(n - 254, n)),
        "last255_rst0": _relabel_rst0(good, range(n - 255, n)),
        "last256_rst0": _relabel_rst0(good, range(n - 256, n)),
        # intervals run together: capped errors, an uncapped "Restart marker not detected" pair per interval
        "rst_removed_from_11th": removed,
        "flip_dense": _flipped(good, 1500, 11),                                 # 1 000 capped errors and an overread
        # capped errors up front, RST-index lines all along: uncapped lines on both sides of the cap line
        "flip_then_rst0": _flipped(_relabel_rst0(good, range(n)), 400, 13, upto=0.2),
        # the scan cut short by an EOI: the note mid-scan, then capped errors on the zeros read past it
        "cut_eoi": nodri[: body + (len(nodri) - body) // 2 + 1] + b"\xff\xd9",
        "long_interval_flip": _flipped(JC.long_cases()[2][1], 40, 12),          # no DRI: the self-synchronising path flags it
        "healthy_app1_end": gray[:-2] + b"\xff\xe1\x00\x04ab\xff\xd9",          # a healthy scan that ends in a non-EOI marker
    }


DAMAGED = ["all_rst0", "last254_rst0", "last255_rst0", "last256_rst0", "rst_removed_from_11th", "flip_dense", "flip_then_rst0", "cut_eoi",
           "long_interval_flip"]


# --- the reference ----------------------------------------------------------------------------------------------------------

class Ref:
    """The compiled reference with the process-wide CSnoopConfig and the decoder's error switch in reach.

    ScanErrorsDisable / ScanErrorsEnable are the reference's own members, exported from the oracle library, called on the
    harness's CimgDecode* (RefCtx = {CDocLog, CwindowBuf, CFile, CimgDecode* dec}, oracle/ref_harness.cpp: dec at byte 4184,
    checked below through the reference's GetDetailVlc)."""
    DEC_OFF = 4184

    def __init__(self):
        self.o = Oracle("ref_fixed")
        L = self.o.lib
        L.ref_config.argtypes = [C.c_int, C.c_int, C.c_uint]
        L.ref_setup_jpeg.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        L.ref_DecodeScanImg.argtypes = [C.c_void_p, C.c_uint, C.c_int, C.c_int]
        L.ref_log_clear.argtypes = [C.c_void_p]
        self._disable, self._enable = L._ZN10CimgDecode17ScanErrorsDisableEv, L._ZN10CimgDecode16ScanErrorsEnableEv
        for f in (self._disable, self._enable):
            f.argtypes = [C.c_void_p]; f.restype = None
        self.dec = C.c_void_p.from_address(self.o.ctx.value + self.DEC_OFF).value
        get = L._ZN10CimgDecode12GetDetailVlcERbRjS1_S1_
        get.argtypes = [C.c_void_p, C.POINTER(C.c_bool)] + [C.POINTER(C.c_uint)] * 3; get.restype = None
        self.o.set_detail_vlc(True, 12345, 23456, 34567)
        d, x, y, n = C.c_bool(), C.c_uint(), C.c_uint(), C.c_uint()
        get(self.dec, C.byref(d), C.byref(x), C.byref(y), C.byref(n))
        self.o.set_detail_vlc(False, 0, 0, 1)
        assert (d.value, x.value, y.value, n.value) == (True, 12345, 23456, 34567), "RefCtx layout changed: dec is not at DEC_OFF"
        self._buf = None

    def cap(self, n):
        self.o.lib.ref_config(1, 0, n)

    def decode(self, j):
        """Marker walk (ResetState clears the error switch) + DecodeScanImg(start, true, false)."""
        d = self.o.decode(j, quiet=False)
        return d, self.o.log_lines()

    def walk(self, j):
        self._buf = np.frombuffer(j, np.uint8).copy()
        start = self.o.lib.ref_setup_jpeg(self.o.ctx, self._buf.ctypes.data, self._buf.size)
        assert start > 0
        return start

    def decode_scan(self, start):
        """DecodeScanImg(start, true, false) on the state the last walk left, as the reference's own callers issue it."""
        self.o.lib.ref_log_clear(self.o.ctx)
        self.o.lib.ref_DecodeScanImg(self.o.ctx, start, 1, 0)
        return self.o.collect(), self.o.log_lines()

    def disable(self): self._disable(self.dec)
    def enable(self): self._enable(self.dec)

    def close(self):
        self.cap(20)
        self.o.close()


@pytest.fixture
def ref():
    r = Ref()
    r.cap(20)
    yield r
    r.close()                  # the process-wide configuration back to the defaults: cap 20 (errors are per decoder)


@functools.lru_cache(maxsize=None)
def _ref_run(name, cap):
    """(Decoded, log lines, error lines) of the reference decoding corpus()[name] at `cap`, computed once per process."""
    r = Ref()
    try:
        r.cap(cap)
        d, lines = r.decode(corpus()[name])
        return d, lines, r.o.err_lines()
    finally:
        r.close()


# --- CPU: the reference on the corpus ----------------------------------------------------------------------------------------

@needs_ref
def test_log_parser_reads_every_event_line(built):
    """The parser behind every event comparison below accounts for every scan error line of the reference's log."""
    for name in DAMAGED + ["healthy_app1_end"]:
        for cap in (0, 1, 20, 1000):
            _, lines, errs = _ref_run(name, cap)
            ev = ref_events(lines)
            nerr = sum(2 if e[0] == EV_MCU else 1 for e in ev if e[0] not in (EV_MARKER, EV_RST_MISSING))
            nerr += sum(1 for e in ev if e[0] == EV_RST_MISSING) + sum(1 for e in ev if e[0] == EV_MARKER and e[1] != 0xD9)
            assert nerr == len(errs), (name, cap, nerr, len(errs))


@needs_ref
def test_reference_counts_at_each_cap(built):
    """Error lines of the reference (liboracle_ref_fixed.so) at caps 20, 0, 1 and 1000."""
    want = {"all_rst0": (2038, 2038, 2039, 2038), "rst_removed_from_11th": (29, 1, 3, 1413), "last256_rst0": (256, 256, 257, 256),
            "last254_rst0": (254, 254, 255, 254), "last255_rst0": (254, 254, 255, 254)}
    for name, counts in want.items():
        got = tuple(len(_ref_run(name, cap)[2]) for cap in (20, 0, 1, 1000))
        assert got == counts, (name, got, counts)


@needs_ref
def test_corpus_reaches_the_edges(built):
    """Exactly 255, 256 and 257 events; more than 1 000; more capped errors than any cap below 300; capped and uncapped
    lines on both sides of the cap line."""
    n_ev = lambda name, cap: len(ref_events(_ref_run(name, cap)[1]))
    assert n_ev("last254_rst0", 20) == 255 and n_ev("last254_rst0", 1) == 256 and n_ev("last254_rst0", 0) == 254
    assert n_ev("last256_rst0", 20) == 257 and n_ev("last256_rst0", 0) == 256
    assert n_ev("all_rst0", 20) > 1000 and n_ev("rst_removed_from_11th", 1000) > 1000
    assert len(_capped(ref_events(_ref_run("flip_dense", 1000)[1]))) >= 300
    assert any(e[0] in (EV_OVR_CODE, EV_OVR_BITS) for e in ref_events(_ref_run("flip_dense", 20)[1]))      # an uncapped overread
    assert [e[0] for e in ref_events(_ref_run("cut_eoi", 20)[1])].index(EV_MARKER) < 20
    assert any(e[0] == EV_MARKER and e[1] != 0xD9 for e in ref_events(_ref_run("healthy_app1_end", 20)[1]))
    for name, cap, uncapped_before, uncapped_after in (("rst_removed_from_11th", 20, True, False), ("cut_eoi", 20, False, False),
                                                       ("flip_then_rst0", 1, True, True)):
        ev = ref_events(_ref_run(name, cap)[1])
        k = [i for i, e in enumerate(ev) if e[0] == EV_CAP]
        assert len(k) == 1 and ev[k[0]][1] == cap, (name, cap)
        before, after = ev[:k[0]], ev[k[0] + 1:]
        assert len(_capped(before)) == cap and not _capped(after), (name, cap)
        assert any(e[0] in UNCAPPED for e in before) == uncapped_before, (name, cap)
        assert any(e[0] in UNCAPPED for e in after) == uncapped_after, (name, cap)


@needs_ref
def test_reference_scan_errors_disable(ref):
    """ScanErrorsDisable: the count it sets persists over two decodes, a cap raised afterwards lets cap - old cap lines
    through, RST-index lines are dropped meanwhile, and ScanErrorsEnable resets the count."""
    j = corpus()["rst_removed_from_11th"]
    start = ref.walk(j)
    _, base = ref.decode_scan(start)
    base_ev = ref_events(base)
    ref.disable()
    for _ in range(2):
        _, lines = ref.decode_scan(start)
        ev = ref_events(lines)
        assert not _capped(ev) and not any(e[0] == EV_CAP for e in ev)
        assert [e for e in ev if e[0] in UNCAPPED] == [e for e in base_ev if e[0] in UNCAPPED and e[0] != EV_RST_MISMATCH]
    ref.cap(27)                                   # 7 more than the count the switch set (the cap in force then, 20)
    _, lines = ref.decode_scan(start)
    ev = ref_events(lines)
    assert len(_capped(ev)) == 7 and [e[1] for e in ev if e[0] == EV_CAP] == [27]
    assert _capped(ev) == _capped(base_ev)[:7]
    ref.enable()
    _, lines = ref.decode_scan(start)
    ev = ref_events(lines)
    assert len(_capped(ev)) == 27 and [e[1] for e in ev if e[0] == EV_CAP] == [27]
    # RST-index lines: present at once with errors enabled, absent while disabled
    r0 = corpus()["all_rst0"]
    s0 = ref.walk(r0)
    ref.cap(20); ref.disable()
    _, lines = ref.decode_scan(s0)
    assert not any(e[0] == EV_RST_MISMATCH for e in ref_events(lines))
    ref.enable()
    _, lines = ref.decode_scan(s0)
    assert sum(e[0] == EV_RST_MISMATCH for e in ref_events(lines)) == 2038


# --- GPU: the CUDA path against the reference -------------------------------------------------------------------------------

def _same(name, want, wlines, got, glines, gerr, werr):
    bad = JC.compare(want, got)
    assert not bad, f"{name}: mismatch in {bad}"
    assert np.array_equal(np.asarray(want.stats)[10:12], np.asarray(got.stats)[10:12]), (name, want.stats[10:12], got.stats[10:12])
    assert gerr == werr, (name, len(gerr), len(werr), [(i, a, b) for i, (a, b) in enumerate(zip(gerr, werr)) if a != b][:3])
    assert glines == wlines, (name, len(glines), len(wlines), [(i, a, b) for i, (a, b) in enumerate(zip(glines, wlines)) if a != b][:3])


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("huff", [0, 1, 2], ids=["auto", "warp", "lane"])
def test_every_cap_matches_the_reference(built, huff):
    from jpegsnoop_b200 import CimgDecode
    dec = CimgDecode(idct_fixedpt=True, huff_kernel=huff, idct_kernel=0)
    for cap in CAPS:
        dec.config_scan_err_max(cap)
        for name, j in corpus().items():
            want, wlines, werr = _ref_run(name, cap)
            got = dec.decode(j, quiet=False)
            _same(f"{name} cap={cap}", want, wlines, got, dec.log_lines(-1), dec.log_lines(3), werr)
    dec.close()


def _seq(ref, dec, j, steps):
    """The same sequence of calls on both decoders after one marker walk each; every decode compared."""
    sr = ref.walk(j); sd = dec.walk(j)
    assert sr == sd
    for k, step in enumerate(steps):
        if step == "decode":
            want, wlines = ref.decode_scan(sr)
            dec.L.jsimg_log_clear(dec.h)
            dec.DecodeScanImg(sd, True, False)
            got = dec.collect()
            _same(f"step {k}", want, wlines, got, dec.log_lines(-1), dec.log_lines(3), ref.o.err_lines())
        elif step == "disable":
            ref.disable(); dec.ScanErrorsDisable()
        elif step == "enable":
            ref.enable(); dec.ScanErrorsEnable()
        else:
            ref.cap(step); dec.config_scan_err_max(step)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("huff", [0, 2], ids=["auto", "lane"])
def test_scan_errors_disable_sequences_match_the_reference(built, ref, huff):
    from jpegsnoop_b200 import CimgDecode
    dec = CimgDecode(idct_fixedpt=True, huff_kernel=huff, idct_kernel=0)
    # every sequence decodes once before ScanErrorsDisable: the reference's constructor leaves m_nScanErrMax unset, and the
    # switch copies it (ImgDecode.cpp:1016); from the first DecodeScanImg on it is the configured cap (:2750)
    seq = ["decode", "disable", "decode", "decode", 27, "decode", "enable", "decode"]
    for name in ("rst_removed_from_11th", "all_rst0", "flip_dense", "healthy_app1_end", "long_interval_flip"):
        ref.cap(20); dec.config_scan_err_max(20)
        _seq(ref, dec, corpus()[name], seq)
    ref.cap(1); dec.config_scan_err_max(1)
    _seq(ref, dec, corpus()["healthy_app1_end"], ["decode", "disable", 3, "decode", "decode", 0, "decode", "enable", 2, "decode"])
    ref.cap(0); dec.config_scan_err_max(0)
    _seq(ref, dec, corpus()["last256_rst0"], ["decode", "disable", "decode", 300, "decode", "enable", "decode"])
    dec.close()


@pytest.mark.gpu
@needs_ref
def test_detailed_decode_past_the_256th_event(built, ref):
    """A range placed after the first 256 events of the all-RST0 image keeps the error lines between its dump lines, and a
    healthy image's range that reaches the end-of-scan note reports it as the reference does at caps 0 and 1."""
    from jpegsnoop_b200 import CimgDecode
    dec = CimgDecode(idct_fixedpt=True)
    j = corpus()["all_rst0"]
    _, _, werr = _ref_run("all_rst0", 20)
    try:
        for cap, (x, y, n) in ((20, (0, 40, 240)), (0, (100, 60, 30)), (1000, (0, 66, 240))):   # MCU 4800 on: past RST 1200
            ref.cap(cap); dec.config_scan_err_max(cap)
            ref.o.set_detail_vlc(True, x, y, n); dec.SetDetailVlc(True, x, y, n)
            want, wlines = ref.decode(j)
            got = dec.decode(j, quiet=False)
            _same(f"all_rst0 detail {(x, y, n)} cap={cap}", want, wlines, got, dec.log_lines(-1), dec.log_lines(3), ref.o.err_lines())
            assert sum("Expected RST marker index" in s for s in wlines) > 1000
        g = corpus()["healthy_app1_end"]
        for cap in (0, 1, 2):
            ref.cap(cap); dec.config_scan_err_max(cap)
            ref.o.set_detail_vlc(True, 20, 12, 40); dec.SetDetailVlc(True, 20, 12, 40)      # through the last MCU
            want, wlines = ref.decode(g)
            got = dec.decode(g, quiet=False)
            _same(f"healthy_app1_end detail cap={cap}", want, wlines, got, dec.log_lines(-1), dec.log_lines(3), ref.o.err_lines())
    finally:
        ref.o.set_detail_vlc(False)
        dec.close()
    assert len(werr) == 2038


@pytest.mark.gpu
@needs_ref
def test_batch_reports_every_event(built):
    """Damaged images between healthy ones in one batch: nerr_lines equals the reference's count, scan_error_events equals
    the events behind the reference's lines (all of them), and the neighbours stay untouched."""
    from jpegsnoop_b200 import BatchDecoder
    small = JC.small_cases()
    healthy = [("ok_444", small[0][1]), ("ok_422", small[1][1]), ("ok_gray", small[4][1])]
    c = corpus()
    items = [healthy[0]] + [(k, c[k]) for k in DAMAGED[:4]] + [healthy[1]] + [(k, c[k]) for k in DAMAGED[4:]] + [healthy[2]]
    WHAT = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "mcu_map", "blk_dc", "dht_histo")
    for huff in (0, 2):
        bd = BatchDecoder(huff_kernel=huff, idct_kernel=0)
        bd.set_batch([j for _, j in items]); bd.decode(); bd.sync()
        orc = Oracle("ref_fixed")
        for i, (name, j) in enumerate(items):
            got = bd.fetch(i)
            if name.startswith("ok"):
                assert got.status == 0, (name, hex(got.status))
                assert not JC.compare(orc.decode(j), got, what=WHAT), name
                continue
            want, wlines, werr = _ref_run(name, 20)
            assert not JC.compare(want, got, what=WHAT), (name, huff)
            assert got.status & 0x40000000, (name, hex(got.status))
            e = bd.scan_errors(i)
            assert e.nerr_lines == len(werr) and e.scan_bad == int(want.stats[11]), (name, e.nerr_lines, len(werr))
            ev = bd.scan_error_events(i)
            want_ev = ref_events(wlines)
            assert ev.shape[0] == e.nevents == len(want_ev), (name, ev.shape, e.nevents, len(want_ev))
            got_ev = [tuple(int(v) for v in r[:6]) for r in ev]
            assert got_ev == want_ev, (name, [(k, a, b) for k, (a, b) in enumerate(zip(got_ev, want_ev)) if a != b][:3])
            first = np.frombuffer(bytes(e), np.uint32)[8:].reshape(256, 8)[:min(256, ev.shape[0])]
            assert np.array_equal(first, ev[:256]), name
            if ev.shape[0] > 300:                            # a range across the 256th event, from the events-only walk
                part = np.zeros((20, 8), np.uint32)
                assert bd.L.jsgpu_batch_error_events(bd.ctx, i, 250, 20, part.ctypes.data) == 0
                assert np.array_equal(part, ev[250:270]), name
            assert bd.L.jsgpu_batch_error_events(bd.ctx, i, ev.shape[0], 1, np.zeros(8, np.uint32).ctypes.data) != 0
        orc.close(); bd.close()
