"""Every JPEG a file holds in one GPU batch: the Motion-JPEG Huffman-table import of the marker walk (an "AVI1" APP0 brings
in the T.81 Annex K tables), jsgpu_find_all / BatchDecoder.find_all, the scan windows of plan_windows and
BatchDecoder.decode_all.

CPU: on the compiled reference, an AVI1 frame without DHT decodes as the same frame with an explicit Annex K DHT, and a
frame's own DHT after AVI1 wins; parse_jpeg gives the same tables; near-miss identifiers import nothing; the numpy model of
find_all equals the reference's chained BufSearch; every healthy frame's scan ends well inside its planned window and the
windows add up to about the container's size.
GPU: find_all equals the model (crafted buffers, chunk edges, unaligned buffers, > 10^6 matches, a partial cap, the 2^32
limit); single MJPG frames decode and step as the reference does; decode_all equals the per-offset decodes on every corpus
container and on a 2 000-frame AVI, and leaves a batch decoded before a find_all call intact.
"""
import numpy as np
import pytest

import find_oracle as F
import mjpg_corpus as M

needs_ref = pytest.mark.skipif(not F.ref_available(), reason="needs oracle/_ref (the compiled reference)")
SLACK = 64


def _pairs():
    """(name, MJPG frame without DHT, the same frame with its explicit Annex K DHT) for every layout, with and without DRI."""
    out = []
    for k, kind in enumerate(M.KINDS):
        j = M.frame(500 + k, kind)
        out.append((kind, M.to_mjpg(j), M.to_mjpg(j, keep_dht=True)))
    return out


def _ref_outputs(ref, data, pos=0):
    ref.process(data, pos)
    o = ref.outputs()
    assert o["ready"] and ref.decode_status()
    return o


# --- CPU ----------------------------------------------------------------------------------------------------------------

@needs_ref
def test_reference_avi1_import_equals_an_explicit_annex_k_dht():
    ref = F.RefN1()
    try:
        for kind, mj, explicit in _pairs():
            a, b = _ref_outputs(ref, mj), _ref_outputs(ref, explicit)
            for k in ("y", "cb", "cr", "dib"):
                assert (a[k] is None and b[k] is None) or np.array_equal(a[k], b[k]), (kind, k)
    finally:
        ref.close()


@needs_ref
def test_reference_own_dht_after_avi1_wins():
    ref = F.RefN1()
    try:
        for k, kind in enumerate(("420_opt", "444_dri_opt", "gray_opt")):
            j = M.frame(600 + k, kind)
            mj = M.to_mjpg(j, keep_dht=True)
            a, b = _ref_outputs(ref, mj), _ref_outputs(ref, j)
            for c in ("y", "cb", "cr", "dib"):
                assert (a[c] is None and b[c] is None) or np.array_equal(a[c], b[c]), (kind, c)
    finally:
        ref.close()


def test_walk_imports_annex_k_for_avi1_only(built):
    from jpegsnoop_b200.host import parse_jpeg
    for kind, mj, explicit in _pairs():
        assert bytes(parse_jpeg(mj)[0]) == bytes(parse_jpeg(explicit)[0]), kind
    j = M.frame(601, "444_dri_opt")
    own = M.to_mjpg(j, keep_dht=True)
    assert bytes(parse_jpeg(own)[0]) == bytes(parse_jpeg(j)[0])
    # an identifier that is not AVI1 imports nothing: the tables are those of the frame without any DHT
    j = M.frame(602, "420")
    none = bytes(parse_jpeg(M.to_mjpg(j, ident=b"JFXX\x00"))[0])
    assert bytes(parse_jpeg(M.to_mjpg(j))[0]) != none
    for ident in (b"AVI\x00", b"AVI2", b"JFIF\x00", b"AV\x00I1", b"avi1"):
        assert bytes(parse_jpeg(M.to_mjpg(j, ident=ident))[0]) == none, ident
    # the identifier is read as the reference's BufReadStrn reads it: unprintable bytes are skipped
    assert bytes(parse_jpeg(M.to_mjpg(j, ident=b"AV\x01I1"))[0]) == bytes(parse_jpeg(M.to_mjpg(j))[0])


def _crafted_buffers():
    from test_image_search import crafted
    out = [(name, np.asarray(d)) for name, d, _ in crafted()]
    out += [("overlap", np.frombuffer(b"\x00\xff\xd8\xff\xd8\xff\xd8\xff\x01\xff\xd8\xff", np.uint8)),
            ("soi_at_0_and_end", np.frombuffer(b"\xff\xd8\xff\x10\x20\xff\xd8\xff", np.uint8))]
    out += [(name, np.frombuffer(c, np.uint8)) for name, c in M.corpus()]
    return out


@needs_ref
def test_find_all_model_equals_the_chained_reference_bufsearch():
    for name, d in _crafted_buffers():
        chain, pos = [], 0
        while True:
            found, pos = F.ref_bufsearch(d, pos, F.SOI3, 3, True)
            if not found:
                break
            chain.append(pos)
        model = M.find_all_model(d)
        assert chain == [int(p) for p in model if p >= 1], name


def test_window_planner_on_the_corpus(built):
    from jpegsnoop_b200.host import plan_windows
    for name, c in M.corpus():
        plan = plan_windows(c, M.find_all_model(c))
        walked = [(p, s, w) for p, s, w in plan if s > 0]
        assert walked, name
        for p, s, w in walked:
            e = M.scan_end_marker(c, s)
            if e is not None and c[e + 1] == 0xD9:                 # a healthy scan, ended by its EOI
                assert w == len(c) or e + SLACK <= w, (name, p, e, w)
        if name != "exif":                                         # a thumbnail's window runs on through its host's scan
            planned = sum((w - s + 15) // 16 * 16 for p, s, w in walked)
            assert planned <= len(c) + 96 * len(walked), (name, planned, len(c))


# --- GPU: find_all ------------------------------------------------------------------------------------------------------

def _model_check(bd, d, value=0xFFD8FF, length=3, cap=None):
    want = M.find_all_model(d, value, length)
    n, got = bd.find_all(d, value, length, cap)
    assert n == want.size, (n, want.size)
    k = want.size if cap is None else min(cap, want.size)
    assert np.array_equal(got, want[:k].astype(np.uint32))


def _be(v, L):
    return np.frombuffer(bytes((v >> (8 * (L - 1 - i))) & 0xFF for i in range(L)), np.uint8)


@pytest.mark.gpu
def test_gpu_find_all_crafted(built):
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder()
    for name, d in _crafted_buffers():
        for L, v in ((3, 0xFFD8FF), (2, 0xFFD8), (1, 0xFF), (4, 0xFFD8FFE0), (2, 0xD8FF), (1, 0x00)):
            _model_check(bd, d, v, L)
    assert bd.find_all(b"\xff\xd8\xff\xd8\xff")[1].tolist() == [0, 2]
    assert bd.find_all(b"\xff\xd8")[0] == 0 and bd.find_all(b"")[0] == 0
    assert bd.find_all(b"\xff\xff", 0x1FF, 1)[0] == 0                # wider than one byte: never matches


@pytest.mark.gpu
def test_gpu_find_all_chunk_edges_and_unaligned(built, monkeypatch):
    from jpegsnoop_b200 import BatchDecoder
    monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", "4096")
    bd = BatchDecoder()
    rng = np.random.default_rng(13)
    base = rng.integers(0, 255, 6 * 4096 + 77, dtype=np.uint8)     # no 0xFF
    for L, v in ((3, 0xFFD8FF), (4, 0xFFD8FFE1), (2, 0xFFD8), (1, 0xFF)):
        for delta in range(-L - 1, 2):                              # the match before, across and after each chunk edge
            d = base.copy()
            for e in (4096, 2 * 4096, 3 * 4096, 5 * 4096):
                d[e + delta:e + delta + L] = _be(v, L)
            d[-L:] = _be(v, L)
            _model_check(bd, d, v, L)
        raw = np.zeros(d.size + 16, np.uint8)
        for a in (1, 3, 7, 13):
            u = raw[a:a + d.size]; u[:] = d
            _model_check(bd, u, v, L)
    cont = M.corpus()[0][1]
    for a in (1, 5):
        raw = np.zeros(len(cont) + 8, np.uint8); u = raw[a:a + len(cont)]; u[:] = np.frombuffer(cont, np.uint8)
        _model_check(bd, u)


@pytest.mark.gpu
def test_gpu_find_all_many_matches_and_cap(built):
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder()
    rng = np.random.default_rng(17)
    d = rng.integers(0, 255, (64 << 20) + 12345, dtype=np.uint8)    # past one default chunk
    d[rng.integers(0, d.size - 3, 3_000_000)] = 0xFF
    d[np.flatnonzero(d == 0xFF)[::2] + 1] = 0xD8
    want = M.find_all_model(d, 0xFFD8, 2)
    assert want.size > 10 ** 6
    _model_check(bd, d, 0xFFD8, 2)
    for cap in (0, 1, 777, want.size - 1, want.size + 5):
        _model_check(bd, d, 0xFFD8, 2, cap)
    _model_check(bd, d, 0xFF, 1)


@pytest.mark.gpu
def test_gpu_find_all_size_limit_and_batch_untouched(built):
    from jpegsnoop_b200 import BatchDecoder, JsgpuError
    bd = BatchDecoder()
    cont = M.corpus()[0][1]
    bd.set_batch([M.frame(3, "420"), M.frame(4, "444_dri")]); bd.decode(); bd.sync()
    before = bd.checksums()
    big = np.zeros(1 << 32, np.uint8)                               # pages never touched
    with pytest.raises(JsgpuError):
        bd.find_all(big)
    with pytest.raises(JsgpuError):
        bd.find_all(cont, 0xFFD8FF, 5)
    assert bd.find_all(cont)[0] == M.find_all_model(cont).size
    assert np.array_equal(bd.checksums(), before)


# --- GPU: single MJPG frames --------------------------------------------------------------------------------------------

@pytest.mark.gpu
@needs_ref
def test_gpu_mjpg_frames_decode_and_step_as_the_reference(built):
    from jpegsnoop_b200 import CimgDecode
    from test_image_search import _check_at
    avi, offs = M.avi(M.mjpg_frames(3, 10))
    ref, dec = F.RefN1(), CimgDecode(idct_fixedpt=False)
    try:
        for o in offs:
            _check_at(ref, dec, avi, o, ("mjpg", o))
        dec.set_file(avi)
        start, seen = 0, []
        while True:
            want = F.ref_doc_search(avi, start, True)
            found, pos = dec.search_forward(start, quiet=True)
            assert (found, pos, dec.reprocessed is not None) == want, start
            if not found:
                break
            assert dec.reprocessed > pos
            seen.append(pos); start = pos
        assert seen == offs
    finally:
        ref.close()


# --- GPU: decode_all ----------------------------------------------------------------------------------------------------

def _same(a, b, what):
    for k in ("pix_y", "pix_cb", "pix_cr", "dib", "mcu_map", "dht_histo"):
        x, y = getattr(a, k), getattr(b, k)
        assert (x is None and y is None) or np.array_equal(x, y), (what, k)
    for x, y in zip(a.blk_dc, b.blk_dc):
        assert (x is None and y is None) or np.array_equal(x, y), (what, "blk_dc")
    assert np.array_equal(a.geom, b.geom), (what, "geom")


@pytest.mark.gpu
@pytest.mark.parametrize("fixed", [True, False])
def test_gpu_decode_all_equals_the_per_offset_decodes(built, fixed):
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    from jpegsnoop_b200.host import walk_jpeg
    bd, one, dec = BatchDecoder(idct_fixedpt=fixed), BatchDecoder(idct_fixedpt=fixed), CimgDecode(idct_fixedpt=fixed)
    windowed = redone = 0
    for name, c in M.corpus():
        res, info = bd.decode_all(c)
        assert [p for p, _, _ in res] == M.find_all_model(c).tolist(), name
        walked = 0
        for p, s, img in res:
            r = walk_jpeg(c, p)[2]
            assert s == r, (name, p)
            if r < 0:
                assert img is None, (name, p)
                continue
            walked += 1
            d = dec.decode(c, offset=p)
            _same(img, d, (name, p))
            assert img.status == d.status and img.scan_start == d.scan_start and img.pos == p, (name, p, img.status, d.status)
            one.set_batch([(c, p)]); one.decode(); one.sync()
            full = one.fetch(0)
            assert np.array_equal(img.stats, full.stats) and img.status == full.status, (name, p)
        assert info["uploaded"] >= sum(1 for _, s, _ in res if s > 0)
        redone += info["redone"]
        windowed += walked - info["redone"]
    assert redone >= 1 and windowed >= 1


@pytest.mark.gpu
def test_gpu_decode_all_large_avi(built):
    from jpegsnoop_b200 import BatchDecoder
    frames = M.mjpg_frames(5, 40)
    seq = [frames[k % len(frames)] for k in range(2000)]
    avi, offs = M.avi(seq)
    bd = BatchDecoder()
    res, info = bd.decode_all(avi)
    assert [p for p, _, _ in res] == offs and info["redone"] == 0
    assert info["uploaded"] <= len(avi) + 96 * len(offs), (info, len(avi))
    cut = BatchDecoder()
    cut.set_batch(frames); cut.decode(); cut.sync()
    ref = [cut.fetch(i) for i in range(len(frames))]
    for k, (p, s, img) in enumerate(res):
        b = ref[k % len(frames)]
        for f in ("pix_y", "pix_cb", "pix_cr", "dib"):
            x, y = getattr(img, f), getattr(b, f)
            assert (x is None and y is None) or np.array_equal(x, y), (k, f)
        assert np.array_equal(img.mcu_map, b.mcu_map + (p << 4)), k
