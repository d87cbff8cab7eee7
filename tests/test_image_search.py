"""Tools -> Img Search Fwd / Rev and decoding from any file offset (jsgpu_find_value, jsimg_buf_search, jsimg_img_search,
jsimg_decode_jpeg_at, jsimg_decode_offset_mode, jsimg_parse_jpeg_at; CimgDecode.search_forward / search_reverse /
decode(offset, mode), parse_jpeg(offset), BatchDecoder.prepare((bytes, offset)), BatchDecoder.find_value).

CPU: the numpy model of CwindowBuf::BufSearch equals the reference's compiled BufSearch on crafted buffers (tests/find_oracle.py);
the marker walk from an offset gives the cut-out JPEG's tables and descriptor with absolute positions.
GPU: the device search equals the model and the reference on crafted buffers, containers, chunk edges, overlays and unaligned
buffers; decodes at an offset, the Fwd/Rev handlers and the four offset modes equal the reference's CjfifDecode with nPosStart
set (oracle/_ref/libn1_ref.so); a batch of (container, offset) pairs equals the per-image decodes and the cut-out batch.
"""
import ctypes as C

import numpy as np
import pytest

import jpeg_cases as JC
import find_oracle as F

needs_ref = pytest.mark.skipif(not F.ref_available(), reason="needs oracle/_ref (the compiled reference)")
SOI3 = F.SOI3


def crafted():
    """(name, data, [(start, value, length, forward)]) covering the reference loop's edges."""
    out = []
    rng = np.random.default_rng(7)
    base = rng.integers(0, 255, 64, dtype=np.uint8)          # no 0xFF: the only matches are the planted ones
    vals = {1: 0xD8, 2: 0xFFD8, 3: SOI3, 4: 0xFFD8FFE0}

    def be(v, L):
        return bytes((v >> (8 * (L - 1 - i))) & 0xFF for i in range(L))
    for L, v in vals.items():
        n = base.size
        for name, at in (("at0", 0), ("at_end", n - L), ("mid", 29)):
            d = base.copy(); d[at:at + L] = np.frombuffer(be(v, L), np.uint8)
            q = [(s, v, L, f) for s in (0, 1, at - 1 if at else 0, at, at + 1, n - L, n - 2, n - 1, n, n + 3) for f in (True, False) if s >= 0]
            out.append((f"len{L}_{name}", d, q))
        # straddling EOF: the first k bytes of the value at the end, the rest read as 0
        for k in range(1, L):
            v0 = v & ~((1 << (8 * (L - k))) - 1)
            d = base.copy(); d[n - k:] = np.frombuffer(be(v0, L)[:k], np.uint8)
            out.append((f"len{L}_eof{k}", d, [(s, v0, L, f) for s in (0, n - L, n - k - 1, n - 1, n + 2) for f in (True, False)]))
        # value 0: every position past EOF matches
        out.append((f"len{L}_zero", base.copy(), [(s, 0, L, f) for s in (0, 10, n - 1, n, n + 5) for f in (True, False)]))
        # a value wider than len bytes never matches
        out.append((f"len{L}_wide", base.copy(), [(s, 1 << (8 * L), L, f) for s in (0, 30, n) for f in (True, False)] if L < 4 else []))
    runs = bytes([1, 2, 0xFF, 0xD8, 0xFF, 0xD8, 0xFF, 3, 0xFF, 0xD8, 0xFF, 0xD8, 0xFF, 0xD8])
    out.append(("runs", np.frombuffer(runs, np.uint8).copy(),
                [(s, v, L, f) for s in range(len(runs) + 2) for f in (True, False) for L, v in ((3, SOI3), (2, 0xFFD8), (2, 0xD8FF))]))
    out.append(("not_found", base.copy(), [(s, v, L, f) for s in (0, 5, 63, 64) for f in (True, False) for L, v in vals.items()]))
    tiny = [bytes([0xFF]), bytes([0xFF, 0xD8]), bytes([0xFF, 0xD8, 0xFF])]
    for t in tiny:
        out.append((f"tiny{len(t)}", np.frombuffer(t, np.uint8).copy(),
                    [(s, v, L, f) for s in range(5) for f in (True, False) for L, v in ((3, SOI3), (2, 0xFFD8), (1, 0xFF), (4, 0xFFD8FF00))]))
    return out


def _jpegs(seed, count):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(count):
        w, h = int(rng.integers(3, 9)) * 16 + int(rng.integers(0, 9)), int(rng.integers(2, 6)) * 16 + int(rng.integers(0, 9))
        out.append(JC.enc(JC.synth_rgb(w, h, seed * 10 + k), quality=int(rng.integers(60, 95)), subsampling=k % 3,
                          restart_marker_blocks=int(rng.integers(0, 4))))
    return out


def container(seed, count=5, lead=None):
    """`count` JPEGs, each behind random junk, and a junk tail: (bytes, [SOI offsets])."""
    rng = np.random.default_rng(seed)
    parts, offs, at = [], [], 0
    for k, j in enumerate(_jpegs(seed, count)):
        junk = rng.integers(0, 256, int(rng.integers(1, 3000)) if (lead is None or k) else lead, dtype=np.uint8).tobytes()
        parts += [junk, j]; offs.append(at + len(junk)); at += len(junk) + len(j)
    parts.append(rng.integers(0, 256, 777, dtype=np.uint8).tobytes())
    return b"".join(parts), offs


# --- CPU ----------------------------------------------------------------------------------------------------------------

@needs_ref
def test_model_equals_the_reference_bufsearch():
    n = 0
    for name, d, qs in crafted():
        for (s, v, L, f) in qs:
            assert F.bufsearch_model(d, s, v, L, f) == F.ref_bufsearch(d, s, v, L, f), (name, s, hex(v), L, f)
            n += 1
    assert n > 500


@needs_ref
def test_model_equals_the_reference_with_overlays():
    d = np.frombuffer(bytes(range(1, 200)), np.uint8).copy()
    d[100:103] = (0xFF, 0xD8, 0xFF)
    cases = [[(50, b"\xff\xd8\xff")], [(101, b"\x00")], [(60, b"\xff\xd8\xff"), (60, b"\x01")], [(197, b"\xff\xd8\xff\xd8")],
             [(250, b"\xff\xd8\xff")], [(99, b"\x07\xff\xd8\xff"), (100, b"\x05")]]
    for ov in cases:
        for s in (0, 40, 99, 100, 101, 150, 199, 260):
            for f in (True, False):
                assert F.bufsearch_model(d, s, SOI3, 3, f, ov) == F.ref_bufsearch(d, s, SOI3, 3, f, ov), (ov, s, f)


def test_walk_from_an_offset_is_the_cut_out_walk_with_absolute_positions(built):
    from jpegsnoop_b200.host import parse_jpeg
    cont, offs = container(3)
    for o in offs:
        t0, d0, s0 = parse_jpeg(cont[o:])
        t1, d1, s1 = parse_jpeg(cont, o)
        assert bytes(t0) == bytes(t1) and s1 == s0 + o and d1.file_pos == d0.file_pos + o
        d0.file_pos += o; d0.scan_offset = s1; d0.scan_length = len(cont) - s1
        assert bytes(d0) == bytes(d1)
    for bad in (offs[0] - 1, offs[0] + 1, len(cont) - 2, len(cont) + 5):
        with pytest.raises(ValueError):
            parse_jpeg(cont, bad)


# --- GPU: the search ----------------------------------------------------------------------------------------------------

def _both(bd, d, s, v, L, f, ov=(), ref=True):
    want = F.bufsearch_model(d, s, v, L, f, ov)
    got = bd.find_value(d, s, v, L, f, ov)
    assert got == want, (s, hex(v), L, f, ov, got, want)
    if ref and F.ref_available():
        assert F.ref_bufsearch(d, s, v, L, f, ov) == want, (s, hex(v), L, f, ov)


@pytest.mark.gpu
def test_gpu_crafted(built):
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    bd = BatchDecoder()
    for name, d, qs in crafted():
        for q in qs:
            _both(bd, d, *q)
    # the same through the decoder's window buffer (jsimg_buf_search)
    dec = CimgDecode()
    for name, d, qs in crafted()[:6]:
        dec.set_file(d)
        for (s, v, L, f) in qs:
            assert dec.buf_search(s, v, L, f) == F.bufsearch_model(d, s, v, L, f), (name, s, L, f)


@pytest.mark.gpu
def test_gpu_containers(built):
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder()
    for seed in (1, 2):
        cont, offs = container(seed, lead=0 if seed == 2 else None)
        d = np.frombuffer(cont, np.uint8)
        starts = sorted({0, 1, len(cont) - 1, len(cont)} | {o + k for o in offs for k in (-1, 0, 1) if o + k >= 0})
        for s in starts:
            for f in (True, False):
                _both(bd, d, s, SOI3, 3, f, ref=(s in (0, len(cont)) or s in offs))
        # the Fwd chain visits every SOI in order (and nothing in the junk), the Rev chain comes back
        pos, seen = 0, []
        while True:
            found, pos = bd.find_value(d, pos, SOI3, 3, True)
            if not found:
                break
            seen.append(pos)
        truth = [p for p in range(1, len(cont) - 2) if cont[p:p + 3] == b"\xff\xd8\xff"]
        assert seen == truth and set(offs) - {0} <= set(seen)
        pos, back = len(cont), []
        while pos > 0:
            found, pos = bd.find_value(d, pos, SOI3, 3, False)
            if found:
                back.append(pos)
        assert back == [p for p in reversed(range(len(cont))) if cont[p:p + 3] == b"\xff\xd8\xff"]


@pytest.mark.gpu
def test_gpu_chunk_edges(built, monkeypatch):
    """4 KiB chunks: matches across, in the halo of, and at the first position of a chunk, in both directions, from starts
    that put a chunk edge on every side of them."""
    from jpegsnoop_b200 import BatchDecoder
    monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", "4096")
    bd = BatchDecoder()
    rng = np.random.default_rng(11)
    base = rng.integers(0, 255, 5 * 4096 + 123, dtype=np.uint8)
    n = base.size
    for L, v in ((3, SOI3), (4, 0xFFD8FFE1), (2, 0xFFD8), (1, 0xFF)):
        pat = np.frombuffer(bytes((v >> (8 * (L - 1 - i))) & 0xFF for i in range(L)), np.uint8)
        for f in (True, False):
            for s in (0, 1, 4095, 4096, 4097, 2 * 4096 - 1, n - 1, n):
                if f:
                    edges = [s + 1 + k * 4096 for k in (1, 2)]
                else:
                    hi = min(s - 1, n - L)
                    edges = [hi + 1 - k * 4096 for k in (1, 2)]
                for e in edges:
                    for p in range(e - L - 1, e + 2):           # the match's first byte before, across and after the edge
                        if not 0 <= p <= n - L:
                            continue
                        d = base.copy(); d[p:p + L] = pat
                        _both(bd, d, s, v, L, f, ref=False)
            # two matches in consecutive chunks: the first in search order wins
            d = base.copy(); d[5000:5000 + L] = pat; d[9000:9000 + L] = pat
            _both(bd, d, 0 if f else n, v, L, f, ref=False)


@pytest.mark.gpu
def test_gpu_files_past_one_default_chunk(built):
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder()
    rng = np.random.default_rng(5)
    n = (64 << 20) + (3 << 20) + 17
    d = rng.integers(0, 255, n, dtype=np.uint8)                     # no 0xFF anywhere
    assert bd.find_value(d, 0, SOI3, 3, True) == (False, n - 2)
    assert bd.find_value(d, n, SOI3, 3, False) == (False, 0)
    d[n - 1000:n - 997] = (0xFF, 0xD8, 0xFF)                        # in the last chunk forward
    d[700:703] = (0xFF, 0xD8, 0xFF)                                 # in the last chunk backward
    assert bd.find_value(d, 800, SOI3, 3, True) == (True, n - 1000)
    assert bd.find_value(d, n - 1100, SOI3, 3, False) == (True, 700)
    assert bd.find_value(d, 0, SOI3, 3, True) == (True, 700)
    assert bd.find_value(d, n, SOI3, 3, False) == (True, n - 1000)


@pytest.mark.gpu
def test_gpu_overlays(built, monkeypatch):
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    cont, offs = container(4)
    d = np.frombuffer(cont, np.uint8)
    o1, o2 = offs[1], offs[2]
    cases = [[(o1, b"\x00")],                                        # removes the second SOI: Fwd jumps to the third
             [(o1 + 1, b"\xd9\xff\xd8")],                            # removes one and creates another two bytes later
             [(o1 - 500, b"\xff\xd8\xff")],                          # creates one in the junk
             [(o1 - 10, b"\xff\xd8\xff"), (o1 - 10, b"\x11")],       # ... that a later overlay removes again
             [(len(cont) - 1, b"\xd8\xff")]]                         # reaches past EOF
    monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", "4096")
    bd = BatchDecoder()
    dec = CimgDecode()
    dec.set_file(cont)
    for ov in cases:
        dec.L.jsimg_overlay_remove_all(dec.h)
        keep = [np.frombuffer(b, np.uint8).copy() for _, b in ov]
        for (o, _), a in zip(ov, keep):
            dec.L.jsimg_overlay_install(dec.h, o, a.ctypes.data, a.size)
        for s in (offs[0], o1 - 600, o1 - 11, o1, o2, len(cont) - 2, len(cont) + 1):
            for f in (True, False):
                _both(bd, d, s, SOI3, 3, f, ov, ref=True)
                assert dec.buf_search(s, SOI3, 3, f) == F.bufsearch_model(d, s, SOI3, 3, f, ov), (ov, s, f)
    # an overlay changes the answer
    assert bd.find_value(d, offs[0], SOI3, 3, True) == (True, o1)
    assert bd.find_value(d, offs[0], SOI3, 3, True, [(o1, b"\x00")]) == (True, o2)
    assert bd.find_value(d, offs[0], SOI3, 3, True, [(o1 - 500, b"\xff\xd8\xff")]) == (True, o1 - 500)


@pytest.mark.gpu
def test_gpu_unaligned_host_buffers(built, monkeypatch):
    from jpegsnoop_b200 import BatchDecoder
    monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", "8192")
    bd = BatchDecoder()
    cont, offs = container(6)
    raw = np.zeros(len(cont) + 16, np.uint8)
    for a in (1, 3, 7, 13):
        d = raw[a:a + len(cont)]; d[:] = np.frombuffer(cont, np.uint8)
        for s in (0, offs[1], offs[3] + 1, len(cont)):
            for f in (True, False):
                _both(bd, d, s, SOI3, 3, f, ref=False)


@pytest.mark.gpu
def test_gpu_strided_views_search_their_own_bytes(built):
    """A strided uint8 view is searched element by element, not as the memory under its first elements: find_value and
    search_bytes give what they give for its contiguous copy."""
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder()
    cont, offs = container(9)
    pat = np.random.default_rng(9).integers(0, 256, 64, dtype=np.uint8)
    planted = [100, len(cont) // 2, len(cont) - 300]
    raw = np.zeros(2 * len(cont), np.uint8)                     # the view's bytes interleaved with zeros in memory
    view = raw[::2]
    view[:] = np.frombuffer(cont, np.uint8)
    for p in planted:
        view[p:p + pat.size] = pat
    flat = view.copy()
    assert not view.flags.c_contiguous
    counts, (pos,) = bd.search_bytes(view, [pat.tobytes()])
    counts0, (pos0,) = bd.search_bytes(flat, [pat.tobytes()])
    assert counts.tolist() == counts0.tolist() == [len(planted)]
    assert pos.tolist() == pos0.tolist() == planted
    for s in (0, offs[1], offs[3] + 1, len(cont)):
        for f in (True, False):
            assert bd.find_value(view, s, SOI3, 3, f) == bd.find_value(flat, s, SOI3, 3, f) == F.bufsearch_model(flat, s, SOI3, 3, f)


@pytest.mark.gpu
def test_gpu_size_limit(built):
    from jpegsnoop_b200 import BatchDecoder, CimgDecode, JsgpuError
    big = np.zeros(1 << 32, np.uint8)                          # pages never touched
    bd = BatchDecoder()
    with pytest.raises(JsgpuError):
        bd.find_value(big, 0, SOI3, 3, True)
    with pytest.raises(JsgpuError):
        bd.find_value(big[:100], (1 << 32) - 1, SOI3, 3, False)
    with pytest.raises(JsgpuError):
        bd.find_value(big[:100], 0, SOI3, 5, True)
    dec = CimgDecode()
    dec.L.jsimg_set_file(dec.h, big.ctypes.data, big.size)
    with pytest.raises(JsgpuError):
        dec.buf_search(0, SOI3, 3, True)
    assert len(dec.log_lines(3)) == 1


# --- GPU: decoding at an offset -----------------------------------------------------------------------------------------

def _lookups(dec, geom):
    mx, my, bx, by = int(geom[2]), int(geom[3]), int(geom[4]), int(geom[5])
    m = np.array([[dec.LookupFilePosMcu(x, y) for x in range(mx)] for y in range(my)], np.uint32)
    b = np.array([[dec.LookupBlkYCC(x, y) for x in range(bx)] for y in range(by)], np.int32)
    return m, b


def _check_at(ref, dec, cont, off, what):
    rl = ref.process(cont, off)
    d = dec.decode(cont, offset=off, quiet=False)
    gl = dec.log_lines(-1)
    i = rl.index("*** Decoding SCAN Data ***")
    assert gl == rl[i:i + len(gl)], (what, [(k, a, b) for k, (a, b) in enumerate(zip(gl, rl[i:])) if a != b][:3])
    assert gl[-1] == "" and not rl[i + len(gl)].startswith("  "), (what, rl[i + len(gl) - 2:i + len(gl) + 2])
    want = ref.outputs()
    assert want["ready"] and want["size"] == (d.pix_y.shape[1], d.pix_y.shape[0]), what
    for k, got in (("y", d.pix_y), ("cb", d.pix_cb), ("cr", d.pix_cr), ("dib", d.dib)):
        assert np.array_equal(want[k], got), (what, k)
    m, b = _lookups(dec, d.geom)
    assert np.array_equal(ref.mcu_map(m.shape[1], m.shape[0]), m), what
    assert np.array_equal(ref.blk_dc(b.shape[1], b.shape[0]), b), what
    assert m[0, 0, 0] >= off and d.mcu_map[0] >> 4 == m[0, 0, 0]
    return d, gl


def _damaged(j, seed):
    from jpegsnoop_b200.host import parse_jpeg
    start = parse_jpeg(j)[2]
    b = bytearray(j)
    rng = np.random.default_rng(seed)
    for p in rng.integers(start + 20, len(j) - 40, 6):
        b[p] ^= 0x5A
    return bytes(b)


@pytest.mark.gpu
@needs_ref
def test_gpu_decode_at_offset_matches_the_reference(built):
    from jpegsnoop_b200 import CimgDecode
    ref, dec = F.RefN1(), CimgDecode(idct_fixedpt=False)
    try:
        cont, offs = container(8)
        for o in offs:
            _check_at(ref, dec, cont, o, ("healthy", o))
        # a damaged image inside the container: its error lines carry absolute offsets
        js = _jpegs(9, 2)
        junk = np.random.default_rng(9).integers(0, 256, 4321, dtype=np.uint8).tobytes()
        bad = _damaged(js[1], 3)
        cont2 = junk + js[0] + junk + bad + junk
        o = len(junk) * 2 + len(js[0])
        d, gl = _check_at(ref, dec, cont2, o, "damaged")
        errs = [l for l in gl if "@ 0x" in l and ("ERROR" in l or "Expect" in l)]
        assert errs and d.nerr > 0
        assert all(int(l.split("@ 0x")[1][:8], 16) >= o for l in errs)
        # a Detailed Decode range inside the embedded image
        ref.set_detail(1, 0, 3); dec.SetDetailVlc(True, 1, 0, 3)
        d, gl = _check_at(ref, dec, cont, offs[2], "detail")
        vlc = [l for l in gl if l.startswith("      [0x")]
        assert vlc and all(int(l[9:17], 16) >= offs[2] for l in vlc)
    finally:
        dec.SetDetailVlc(False); ref.close()


@pytest.mark.gpu
@needs_ref
def test_gpu_search_and_reprocess_follows_the_doc_handlers(built):
    from jpegsnoop_b200 import CimgDecode
    ref, dec = F.RefN1(), CimgDecode(idct_fixedpt=False)
    try:
        cont, offs = container(12)
        dec.set_file(cont)
        steps = [True] * 6 + [False] * 7 + [True, False, False]
        start, visited = 0, []
        for fwd in steps:
            want = F.ref_doc_search(cont, start, fwd)
            found, pos = dec.search_forward(start) if fwd else dec.search_reverse(start)
            assert (found, pos, dec.reprocessed is not None) == want, (start, fwd)
            if want[2]:
                rl = ref.process(cont, pos)
                if dec.reprocessed >= 0:
                    gl = dec.log_lines(-1)
                    i = rl.index("*** Decoding SCAN Data ***")
                    assert gl == rl[i:i + len(gl)], (start, fwd, pos)
                    want_px = ref.outputs()["y"]
                    assert np.array_equal(dec.collect().pix_y, want_px), (start, fwd, pos)
                    visited.append(pos)
                else:
                    assert not ref.decode_status() and pos == 0
            start = pos
        assert visited[:5] == offs and visited[5:9] == offs[3::-1] and start == 0
    finally:
        ref.close()


@pytest.mark.gpu
@needs_ref
def test_gpu_offset_modes_pick_the_reference_position(built):
    from jpegsnoop_b200 import CimgDecode
    from jpegsnoop_b200 import _lib as B
    from PIL import Image
    import io
    js = _jpegs(21, 2)
    junk = np.random.default_rng(21).integers(0, 256, 999, dtype=np.uint8).tobytes()
    prog = io.BytesIO(); Image.fromarray(JC.synth_rgb(64, 48, 5)).save(prog, "JPEG", progressive=True, quality=80)
    sof = js[0].index(b"\xff\xc0")
    sof_end = sof + 2 + (js[0][sof + 2] << 8 | js[0][sof + 3])
    files = {"soi_at_0": js[0] + junk + js[1], "junk_first": junk + js[0] + junk + js[1], "no_soi": junk * 3,
             "sof_no_scan_at_0": js[0][:sof_end] + junk + js[1], "progressive_at_0": prog.getvalue() + junk + js[1]}
    ref, dec = F.RefN1(), CimgDecode(idct_fixedpt=False)
    try:
        for name, f in files.items():
            buf = np.frombuffer(f, np.uint8).copy()
            for mode in range(4):
                for pos in ((0, 999, len(f) - len(js[1])) if mode == 3 else (0,)):
                    want = F.ref_offset_mode(f, mode, pos, ref)
                    used = C.c_uint64(0)
                    r = dec.L.jsimg_decode_offset_mode(dec.h, buf.ctypes.data, buf.size, mode, pos, 0, C.byref(used))
                    assert used.value == want, (name, mode, pos)
                    ref.process(f, want)
                    # the reference's status is "a frame header was decoded"; there is no scan to decode in these two at 0
                    ok = ref.decode_status() and not (want == 0 and name in ("sof_no_scan_at_0", "progressive_at_0"))
                    assert (r >= 0) == ok, (name, mode, pos, r)
        # the public face
        d = dec.decode(files["junk_first"], mode=B.OFFSET_SRCH1)
        assert d.pos == len(junk) and d.scan_start > d.pos
    finally:
        ref.close()


# --- GPU: batches of (container, offset) pairs ---------------------------------------------------------------------------

_M1, _M2 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xD6E8FEB86659FD93)


def host_ck(a):
    """The device checksum of a host buffer (include/jsgpu.h: jsgpu_batch_checksums)."""
    if a is None:
        return 0
    b = np.ascontiguousarray(a).tobytes()
    b += bytes(-len(b) % 4)
    w = np.frombuffer(b, "<u4").astype(np.uint64)
    with np.errstate(over="ignore"):
        x = w + (np.arange(w.size, dtype=np.uint64) + np.uint64(1)) * _M1
        x ^= x >> np.uint64(32); x *= _M2; x ^= x >> np.uint64(29)
        return int(x.sum(dtype=np.uint64))


@pytest.mark.gpu
def test_gpu_batch_of_offsets(built):
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    cont, offs = container(31)
    bd = BatchDecoder()
    bd.set_batch([(cont, o) for o in offs]); bd.decode(); bd.sync()
    ck = bd.checksums()
    dec = CimgDecode()
    for i, o in enumerate(offs):
        d = dec.decode(cont, offset=o)
        want = [host_ck(x) for x in (d.pix_y, d.pix_cb, d.pix_cr, d.dib, *d.blk_dc, d.mcu_map, d.dht_histo)]
        assert [int(v) for v in ck[i, :9]] == want, i
        if i in (1, 3):
            assert not JC.compare(d, bd.fetch(i), what=("geom", "pix_y", "pix_cb", "pix_cr", "dib", "mcu_map", "blk_dc", "dht_histo")), i
    # the same JPEGs cut out of the container: equal but for the absolute positions
    cut = BatchDecoder()
    cut.set_batch([cont[o:o + len(j)] for o, j in zip(offs, _jpegs(31, 5))]); cut.decode(); cut.sync()
    ck2 = cut.checksums()
    keep = [c for c in range(12) if c != 7]
    assert np.array_equal(ck[:, keep], ck2[:, keep])
    for i, o in enumerate(offs):
        a, b = bd.fetch(i), cut.fetch(i)
        assert np.array_equal(a.mcu_map, b.mcu_map + (o << 4)), i
        s = b.stats.copy(); s[12] += o; s[14] += o if s[14] else 0
        assert np.array_equal(a.stats, s), (i, a.stats, b.stats)
        assert not JC.compare(a, b, what=("geom", "pix_y", "pix_cb", "pix_cr", "dib", "blk_dc", "dht_histo")), i
