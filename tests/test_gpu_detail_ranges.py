"""The "Detailed Decode" of MCU ranges of any length (CimgDecode::SetDetailVlc, ImgDecode.cpp:4880-4904): every ReportVlc line and
every coefficient matrix of the range (:1859-2232), however many there are.  Healthy images are decoded one GPU thread per MCU
(jsgpu_detail.cu), damaged ones by the serial walk (jsgpu_exact.cu); both are compared with the compiled reference line for line,
and with each other word for word.

The CPU tests check, on the reference's own log, that the corpus reaches what the GPU tests rely on: more than 8192 detail lines
and 512 matrices in one range, ranges across restart intervals and MCU-row ends, symbols and MCU starts in the FF byte of a
stuffed FF 00 pair, and ranges that end at and run past the last MCU (where the end-of-scan marker note falls among the lines)."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import coef_jpeg as CJ
import jpeg_cases as JC
import mini_jpeg as MJ
from oracle_util import Oracle, ref_available

needs_ref = pytest.mark.skipif(not ref_available("fixed"), reason="needs oracle/_ref (the compiled reference)")
S420, S422, GREY = ((2, 2), (1, 1), (1, 1)), ((2, 1), (1, 1), (1, 1)), ((1, 1),)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _blocks(rng, W, H, samp, density, smax):
    out = []
    for c in range(len(samp)):
        R, C = CJ.block_shape(W, H, samp, c)
        b = np.zeros((R, C, 64), np.int64)
        s = rng.integers(0, 12, (R, C))
        b[..., 0] = (rng.random((R, C)) * (1 << s)).astype(np.int64) * rng.choice([-1, 1], (R, C))
        sz = rng.integers(1, smax + 1, (R, C, 63))
        mag = (1 << (sz - 1)) + (rng.random((R, C, 63)) * (1 << (sz - 1))).astype(np.int64)
        b[..., 1:] = np.where(rng.random((R, C, 63)) < density, mag * rng.choice([-1, 1], (R, C, 63)), 0)
        out.append(b)
    return out


def _flipped(j, n, seed):
    r = np.random.default_rng(seed)
    a = bytearray(j); lo = j.index(b"\xff\xda") + 14
    for p in r.integers(lo, len(j) - 2, n):
        a[p] ^= 1 << int(r.integers(0, 8))
    return bytes(a)


@functools.lru_cache(maxsize=None)
def corpus():
    """name -> (jpeg bytes, [(mcu x, mcu y, len)]) — healthy images and the ranges the GPU tests print."""
    sc = dict(JC.small_cases())
    rng = np.random.default_rng(20261016)
    q16 = lambda lo, hi: rng.integers(lo, hi + 1, 64)
    p12, _ = CJ.encode_coefs(_blocks(rng, 328, 72, S420, 0.12, 15), 328, 72, S420, [q16(1, 300), q16(1, 300)], [0, 1, 1],
                             precision=12, dri=4, force_pq16=True)
    q255 = np.full(64, 255)
    wrap, _ = CJ.encode_coefs(_blocks(rng, 264, 72, S422, 0.10, 10), 264, 72, S422, [q255, q255], [0, 1, 1], dri=2)
    exotic = MJ.encode(JC.synth_rgb(96, 64, 61), quality=80, samp=((4, 4), (4, 4), (4, 4)), dri=1)      # 48 blocks per MCU
    return {
        # a whole MCU row of a 1920x1080 4:2:0 frame (DRI = 4: 30 intervals), the last row, and across a row end
        "420_dri4_1080p": (sc["420_dri4_1080p"], [(0, 20, 120), (0, 67, 120), (117, 30, 6)]),
        "444_tiny_whole": (sc["444_q100_tiny"], [(0, 0, 48), (0, 0, 100)]),
        "422_whole": (sc["422_opt_dri5"], [(0, 0, 40 * 60)]),
        "gray_whole": (sc["gray_dri3"], [(0, 0, 25 * 13), (24, 12, 1), (20, 12, 3)]),
        "exotic_48blk": (exotic, [(0, 0, 6), (1, 0, 5)]),
        # no DRI: one interval, the self-synchronising Huffman path
        "420_norst_odd": (sc["420_norst_odd"], [(0, 6, 21), (15, 13, 10), (0, 0, 21 * 14)]),
        "p12_420_dri4": (p12, [(0, 0, 21 * 5), (18, 4, 9)]),
        "wrap_q255_422_dri2": (wrap, [(0, 0, 17 * 9), (10, 8, 20)]),
    }


def _vlc_lines(lines):
    return [l for l in lines if l.startswith("      [0x")]


def _pos(line):
    return int(line[9:17], 16), int(line[18])


# --- CPU: what the corpus reaches, from the reference's own log ------------------------------------------------------

@needs_ref
def test_corpus_reaches_the_edges():
    ref = Oracle("ref_fixed")
    seen = {"big": False, "rst": False, "row": False, "ff_sym": False, "ff_mcu": False, "ends_at_last": False, "past_last": False}
    try:
        for name, (j, ranges) in corpus().items():
            for (x, y, n) in ranges:
                ref.set_detail_vlc(True, x, y, n)
                d = ref.decode(j, quiet=False)
                mxm, mym = int(d.geom[2]), int(d.geom[3])
                lines = ref.log_lines()
                vlc = _vlc_lines(lines)
                nmat = sum(1 for l in lines if "DCT Matrix=[" in l)
                if len(vlc) + 2 * nmat > 8192 and nmat > 512:
                    seen["big"] = True
                pos = [_pos(l)[0] for l in vlc]
                if pos and any(j[p] == 0xFF and 0xD0 <= j[p + 1] <= 0xD7 for p in range(min(pos), max(pos))):
                    seen["rst"] = True
                rows = {l.split("MCU=[")[1].split(",")[1] for l in lines if "MCU=[" in l}
                if len(rows) > 1:
                    seen["row"] = True
                stuffed = [i for i, l in enumerate(lines) if l.startswith("      [0x") and j[_pos(l)[0]] == 0xFF and j[_pos(l)[0] + 1] == 0]
                if stuffed:
                    seen["ff_sym"] = True
                if any(lines[i - 1].startswith("    ") and "MCU=[" in lines[i - 1] and lines[i - 2] == "" for i in stuffed):
                    seen["ff_mcu"] = True
                last = min(y * mxm + x + n, mxm * mym) == mxm * mym and y * mxm + x < mxm * mym
                if last and any("Scan Data encountered marker" in l for l in lines):
                    seen["past_last" if y * mxm + x + n > mxm * mym else "ends_at_last"] = True
    finally:
        ref.set_detail_vlc(False); ref.close()
    assert all(seen.values()), seen


# --- GPU: line for line against the reference -------------------------------------------------------------------------

def _check(ref, dec, name, j, what):
    want = ref.decode(j, quiet=False); got = dec.decode(j, quiet=False)
    bad = JC.compare(want, got)
    assert not bad, f"{name} {what}: mismatch in {bad}"
    wl, gl = ref.log_lines(), dec.log_lines(-1)
    assert wl == gl, (name, what, [(i, a, b) for i, (a, b) in enumerate(zip(wl, gl)) if a != b][:3], len(wl), len(gl))
    return want


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("decode_ac", [True, False], ids=["full_idct", "dc_only"])
def test_ranges_match_the_reference(built, decode_ac):
    from jpegsnoop_b200 import CimgDecode
    ref = Oracle("ref_fixed", decode_ac=decode_ac)
    dec = CimgDecode(decode_ac=decode_ac)
    try:
        for name, (j, ranges) in corpus().items():
            for (x, y, n) in ranges if decode_ac else ranges[:1]:
                ref.set_detail_vlc(True, x, y, n); dec.SetDetailVlc(True, x, y, n)
                _check(ref, dec, name, j, (x, y, n))
    finally:
        ref.set_detail_vlc(False); ref.close()


@pytest.mark.gpu
@pytest.mark.skipif(not ref_available("float"), reason="needs oracle/_ref (the compiled reference)")
def test_range_matches_the_float_reference(built):
    from jpegsnoop_b200 import CimgDecode
    ref = Oracle("ref_float"); dec = CimgDecode(idct_fixedpt=False)
    j, ranges = corpus()["420_dri4_1080p"]
    try:
        ref.set_detail_vlc(True, *ranges[0]); dec.SetDetailVlc(True, *ranges[0])
        _check(ref, dec, "420_dri4_1080p/float", j, ranges[0])
    finally:
        ref.set_detail_vlc(False); ref.close()


@pytest.mark.gpu
@needs_ref
def test_damaged_range_beyond_the_old_caps(built):
    """A damaged image takes the serial walk; a whole MCU row of it is more than 8192 events and 512 matrices."""
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    import jpegsnoop_b200._lib as B
    j = _flipped(corpus()["420_dri4_1080p"][0], 200, 3)
    ref = Oracle("ref_fixed"); dec = CimgDecode()
    try:
        ref.set_detail_vlc(True, 0, 20, 120); dec.SetDetailVlc(True, 0, 20, 120)
        _check(ref, dec, "flip200/3", j, (0, 20, 120))
    finally:
        ref.set_detail_vlc(False); ref.close()
    bd = BatchDecoder(); bd.set_batch([j]); bd.set_detail(0, 0, 20, 120); bd.decode(); bd.sync()
    nev, nblk, path = bd.detail_info()
    assert path == B.DETAIL_SERIAL and nev > 8192 and nblk > 512, (nev, nblk, path)
    bd.close()


# --- GPU: the two paths, the fixed-size dump and the rest of the batch --------------------------------------------------

_CHILD = r"""
import sys, numpy as np
sys.path.insert(0, sys.argv[1])
from jpegsnoop_b200 import BatchDecoder
import jpegsnoop_b200._lib as B
jpegs = [open(p, "rb").read() for p in sys.argv[4:]]
x, y, n = (int(v) for v in sys.argv[3].split(","))
out = {}
for i in range(len(jpegs)):
    for ac in (1, 0):
        bd = BatchDecoder(decode_ac=bool(ac)); bd.set_batch([jpegs[i]]); bd.set_detail(0, x, y, n); bd.decode(); bd.sync()
        ev, mat = bd.detail(); out[f"ev{i}_{ac}"] = ev; out[f"mat{i}_{ac}"] = mat; out[f"path{i}_{ac}"] = bd.detail_info()[2]
        out[f"ck{i}_{ac}"] = bd.checksums(); e = np.frombuffer(bytes(bd.scan_errors(0)), np.uint32)
        out[f"err{i}_{ac}"] = np.concatenate([e[:5], e[8:8 + 8 * int(e[1])]])      # what the walk writes for a healthy image
        bd.close()
np.savez(sys.argv[2], **out)
"""


def _run_child(tmp_path, tag, walk, jpegs, rng):
    files = []
    for i, j in enumerate(jpegs):
        p = tmp_path / f"{tag}_{i}.jpg"; p.write_bytes(j); files.append(str(p))
    env = dict(os.environ)
    env.pop("JSGPU_DETAIL_WALK", None)
    if walk:
        env["JSGPU_DETAIL_WALK"] = "1"
    out = tmp_path / f"{tag}.npz"
    r = subprocess.run([sys.executable, "-c", _CHILD, ROOT, str(out), ",".join(map(str, rng))] + files, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return np.load(out)


@pytest.mark.gpu
def test_parallel_and_serial_paths_agree_word_for_word(built, tmp_path):
    """JSGPU_DETAIL_WALK=1 forces the serial walk on healthy images: the same events and matrices, word for word, the same
    end-of-scan note and the same outputs (DC-only rows included), on DRI, no-DRI, 12-bit and exotic images."""
    import jpegsnoop_b200._lib as B
    c = corpus()
    cases = [(c["420_dri4_1080p"][0], (0, 67, 120)), (c["420_norst_odd"][0], (0, 0, 21 * 14)), (c["p12_420_dri4"][0], (0, 0, 21 * 5)),
             (c["gray_whole"][0], (20, 12, 9)), (c["exotic_48blk"][0], (0, 0, 6))]
    for k, (j, rng) in enumerate(cases):
        par = _run_child(tmp_path, f"par{k}", False, [j], rng)
        ser = _run_child(tmp_path, f"ser{k}", True, [j], rng)
        for ac in (1, 0):
            assert int(par[f"path0_{ac}"]) == B.DETAIL_PARALLEL and int(ser[f"path0_{ac}"]) == B.DETAIL_SERIAL
            for key in ("ev", "mat", "ck", "err"):
                a, b = par[f"{key}0_{ac}"], ser[f"{key}0_{ac}"]
                assert a.shape == b.shape and np.array_equal(a, b), (k, ac, key, a.shape, b.shape,
                                                                      np.argwhere(a != b)[:3].tolist() if a.shape == b.shape else None)


@pytest.mark.gpu
def test_fixed_size_dump_keeps_the_first_events(built):
    """jsgpu_batch_detail still returns the full counts and the first 8192 events / 512 matrices."""
    import ctypes as C
    from jpegsnoop_b200 import BatchDecoder
    j = corpus()["420_dri4_1080p"][0]
    bd = BatchDecoder(); bd.set_batch([j]); bd.set_detail(0, 0, 20, 120); bd.decode(); bd.sync()
    ev, mat = bd.detail()
    assert ev.shape[0] > 8192 and mat.shape[0] > 512
    size = 16 + 8192 * 32 + 512 * 128
    buf = np.zeros(size, np.uint8)
    assert bd.L.jsgpu_batch_detail(bd.ctx, C.c_void_p(buf.ctypes.data)) == 0
    hdr = buf[:16].view(np.uint32)
    assert (int(hdr[0]), int(hdr[1]), int(hdr[2]), int(hdr[3])) == (ev.shape[0], mat.shape[0], 0, 0)
    assert np.array_equal(buf[16:16 + 8192 * 32].view(np.uint32).reshape(8192, 8), ev[:8192])
    assert np.array_equal(buf[16 + 8192 * 32:].view(np.int16).reshape(512, 64), mat[:512])
    bd.close()


@pytest.mark.gpu
@needs_ref
def test_mixed_batch_with_the_detail_image_in_the_middle(built):
    """Images of other layouts, precisions and Huffman paths around the detail image: every image's checksums equal the
    reference's, the detail image takes the parallel path, and its detailed decode equals the one it gets alone."""
    from jpegsnoop_b200 import BatchDecoder
    import jpegsnoop_b200._lib as B
    c = corpus()
    jpegs = [c["444_tiny_whole"][0], c["gray_whole"][0], c["420_dri4_1080p"][0], c["420_norst_odd"][0], c["p12_420_dri4"][0]]
    bd = BatchDecoder(); bd.set_batch(jpegs); bd.set_detail(2, 0, 20, 120); bd.decode(); bd.sync()
    got = bd.checksums(); ev, mat = bd.detail(); path = bd.detail_info()[2]
    bd.close()
    _, _, want = Oracle("ref_fixed").bench_ck(jpegs)
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, [(int(i), np.flatnonzero(got[i] != want[i]).tolist()) for i in bad[:5]]
    assert path == B.DETAIL_PARALLEL
    one = BatchDecoder(); one.set_batch([jpegs[2]]); one.set_detail(0, 0, 20, 120); one.decode(); one.sync()
    ev1, mat1 = one.detail(); one.close()
    assert np.array_equal(ev, ev1) and np.array_equal(mat, mat1)
