"""The decoder at its numeric edges: 12-bit scans (SOF1, ReadScanVal's divide by 1 << (P-8)), 16-bit quantisers,
coefficients, DC predictors and samples that wrap in 16 bits, 31-bit code + value steps, samples whose y>>3 / cb>>3 / cr>>3
land on both sides of every clamp, and every (cb, cr) pair of the colour conversion.  The corpus is written at coefficient
level by tests/coef_jpeg.py from fixed seeds; tests/coef_jpeg.expected restates the reference's arithmetic for it.

CPU: the compiled reference decodes every corpus image exactly as restated, and the C port agrees with it.
GPU: every kernel form against the reference (and the restatement) on every output buffer, in both IDCT builds; a batch
mixing 8- and 12-bit images; DC-only mode; damaged 12-bit / wrapping scans with their error lines; the clip / histogram
statistics; the colour sweep; and the device checksums bench.py relies on against the reference's."""
import functools

import numpy as np
import pytest

import coef_jpeg as CJ
import jpeg_cases as JC
from oracle_util import Oracle, ref_available

FIELDS = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "blk_dc")
BATCH_FIELDS = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "mcu_map", "blk_dc", "dht_histo")
S420, S422, S444, GREY = ((2, 2), (1, 1), (1, 1)), ((2, 1), (1, 1), (1, 1)), ((1, 1), (1, 1), (1, 1)), ((1, 1),)


# --- corpus -----------------------------------------------------------------------------------------------------------

def _shapes(W, H, samp):
    return [CJ.block_shape(W, H, samp, c) for c in range(len(samp))]


def _rand_ac(rng, shape, density, smin, smax, pin=None, pin_frac=0.0):
    """Random AC values: each position non-zero with probability `density`, size uniform in smin..smax (any sign); a
    fraction pin_frac of the non-zero values is replaced by +-pin."""
    s = rng.integers(smin, smax + 1, shape + (63,))
    mag = (1 << (s - 1)) + (rng.random(shape + (63,)) * (1 << (s - 1))).astype(np.int64)
    if pin is not None:
        mag = np.where(rng.random(shape + (63,)) < pin_frac, pin, mag)
    val = mag * rng.choice([-1, 1], shape + (63,))
    return np.where(rng.random(shape + (63,)) < density, val, 0)


def _rand_dc(rng, shape, smax=14):
    """Absolute DC values of mixed magnitude (|v| < 2^14): every difference fits in 15 bits, sizes 0..15 all occur."""
    s = rng.integers(0, smax + 1, shape)
    return (rng.random(shape) * (1 << s)).astype(np.int64) * rng.choice([-1, 1], shape)


def _blocks(rng, W, H, samp, ac_density, smin, smax, **kw):
    out = []
    for R, C in _shapes(W, H, samp):
        b = np.zeros((R, C, 64), np.int64)
        b[..., 0] = _rand_dc(rng, (R, C))
        b[..., 1:] = _rand_ac(rng, (R, C), ac_density, smin, smax, **kw)
        out.append(b)
    return out


def _dc_from_targets(W, H, samp, dri, targets):
    """Absolute written DC values (quantiser 1, P = 8) that make the reference's running short predictor equal `targets`
    (one int array per component, block grid shaped).  Each written difference is the wrapped step, so it fits 15 bits."""
    out = [np.zeros(t.shape, np.int64) for t in targets]
    pred = [0] * len(samp); wr = [0] * len(samp)
    for n, mcu in enumerate(CJ._mcu_order(W, H, samp)):
        if dri and n and n % dri == 0:
            pred = [0] * len(samp); wr = [0] * len(samp)
        for c, r, k in mcu:
            t = int(targets[c][r, k])
            d = ((t - pred[c] + 32768) & 0xFFFF) - 32768
            if d == -32768:                     # one step short of the other end: move the target by one
                d += 1; t += 1; targets[c][r, k] = t
            pred[c] = ((pred[c] + d + 32768) & 0xFFFF) - 32768
            wr[c] += d; out[c][r, k] = wr[c]
    return out


def _clamp_case(rng, W, H, samp, dri, low_ac):
    """DC-only (and, with low_ac, a few small AC) blocks whose samples sit at y>>3 = -4096, -129, -128, 127, 128, 4095 ... in
    every component: both sides of every clamp of the colour conversion and of the clip statistics."""
    T = np.array([-4096, -4095, -1000, -130, -129, -128, -127, -1, 0, 1, 126, 127, 128, 129, 1000, 4095])
    shapes = _shapes(W, H, samp)
    targets = [T[rng.integers(0, T.size, s)] * 8 + rng.integers(0, 8, s) for s in shapes]
    dc = _dc_from_targets(W, H, samp, dri, targets)
    blocks = []
    for c, (R, C) in enumerate(shapes):
        b = np.zeros((R, C, 64), np.int64); b[..., 0] = dc[c]
        if low_ac:
            b[..., 1:10] = np.where(rng.random((R, C, 9)) < 0.3, rng.integers(-3, 4, (R, C, 9)), 0)
        blocks.append(b)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(blocks, W, H, samp, [q1, q1], [0, 1, 1][:len(samp)], dri=dri)


def _colour_sweep():
    """4:2:0, 4096 x 4112.  MCU (mx, my < 256) carries the DC-only chroma pair (cb, cr) = (my - 128, mx - 128), at 8c + 0..7,
    and luma blocks with random AC whose samples span y>>3 = -128..127 and beyond.  The last MCU row gives the three pairs the
    table path hands to the exact routine -- (0, 0), (-100, 100), (100, -100) -- every y in -128..127 (DC-only luma)."""
    rng = np.random.default_rng(20261015)
    W, H = 4096, 4112
    (Ry, Cy), (Rc, Cc), _ = _shapes(W, H, S420)
    y = np.zeros((Ry, Cy, 64), np.int64)
    y[:512, :, 0] = rng.integers(-1100, 1100, (512, Cy))
    pos = CJ.ZZ[1:10]
    y[:512, :, pos] = np.where(rng.random((512, Cy, 9)) < 0.6, rng.integers(-60, 61, (512, Cy, 9)), 0)
    cb = np.zeros((Rc, Cc, 64), np.int64); cr = np.zeros((Rc, Cc, 64), np.int64)
    ci = np.arange(256)
    cb[:256, :, 0] = 8 * (ci[:, None] - 128) + rng.integers(0, 8, (256, Cc))
    cr[:256, :, 0] = 8 * (ci[None, :] - 128) + rng.integers(0, 8, (256, Cc))
    flagged = [(0, 0), (-100, 100), (100, -100)]
    for k in range(Cc):                                   # last MCU row: 64 MCUs per flagged pair, 4 luma blocks each
        p = flagged[min(k // 64, 2)] if k < 192 else flagged[k % 3]
        cb[256, k, 0] = 8 * p[0] + rng.integers(0, 8); cr[256, k, 0] = 8 * p[1] + rng.integers(0, 8)
        for j in range(4):
            yv = ((k % 64) * 4 + j) - 128 if k < 192 else int(rng.integers(-128, 128))
            y[512 + j // 2, 2 * k + j % 2, 0] = 8 * yv + int(rng.integers(0, 8))
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs([y, cb, cr], W, H, S420, [q1, q1], [0, 1, 1], dri=8)


@functools.lru_cache(maxsize=None)
def corpus():
    """[(name, jpeg bytes, spec)]: the healthy edge-case images (the colour sweep is separate)."""
    out = []
    rng = np.random.default_rng(12_2026)
    q16 = lambda lo, hi: rng.integers(lo, hi + 1, 64)
    # P = 12, 16-bit DQT, DC differences and AC values over the whole size range (size-15 DC / size-14 and -15 AC behind
    # 16-bit codes); widths are not a multiple of 32 blocks
    for samp, tag, W, H in ((S420, "420", 328, 72), (S422, "422", 344, 40), (S444, "444", 264, 40)):
        for dri in (1, 4):
            qt = [q16(1, 300), q16(1, 300)]
            bl = _blocks(rng, W, H, samp, 0.12, 1, 15)
            out.append((f"p12_{tag}_dri{dri}", *CJ.encode_coefs(bl, W, H, samp, qt, [0, 1, 1], precision=12, dri=dri, force_pq16=True)))
    bl = _blocks(rng, 200, 56, GREY, 0.15, 1, 15)
    out.append(("p12_grey_dri3", *CJ.encode_coefs(bl, 200, 56, GREY, [q16(1, 255)], [0], precision=12, dri=3, force_pq16=True)))
    bl = _blocks(rng, 496, 128, S420, 0.08, 1, 15)          # one interval of 1488 blocks: the self-synchronising passes
    out.append(("p12_420_nodri", *CJ.encode_coefs(bl, 496, 128, S420, [q16(1, 64), q16(1, 64)], [0, 1, 1], precision=12, force_pq16=True)))
    # P = 8: dequantised coefficients, DC predictors and samples wrap in 16 bits
    q255 = np.full(64, 255); q65535 = np.full(64, 65535)
    bl = _blocks(rng, 264, 72, S420, 0.10, 1, 10, pin=1023, pin_frac=0.3)
    out.append(("wrap_q255_420_dri2", *CJ.encode_coefs(bl, 264, 72, S420, [q255, q255], [0, 1, 1], dri=2)))
    bl = _blocks(rng, 200, 48, S444, 0.10, 1, 15)
    out.append(("wrap_q65535_444_dri3", *CJ.encode_coefs(bl, 200, 48, S444, [q65535, q65535], [0, 1, 1], dri=3)))
    mixed = np.where(rng.random(64) < 0.5, q16(256, 65535), q16(1, 40)); mixed[0] = 3
    bl = _blocks(rng, 328, 40, S422, 0.12, 1, 12, pin=1023, pin_frac=0.2)
    out.append(("wrap_mixed_422_dri5", *CJ.encode_coefs(bl, 328, 40, S422, [mixed, q255], [0, 1, 1], dri=5)))
    bl = _blocks(rng, 400, 160, S420, 0.06, 1, 10, pin=1023, pin_frac=0.3)   # no restart markers: wrapping DC sums through k_ph_scan
    out.append(("wrap_q255_420_nodri", *CJ.encode_coefs(bl, 400, 160, S420, [q255, mixed], [0, 1, 1])))
    bl = _blocks(rng, 136, 40, GREY, 0.15, 1, 15)
    out.append(("wrap_q65535_grey_dri1", *CJ.encode_coefs(bl, 136, 40, GREY, [q65535], [0], dri=1)))
    # clamps of the colour conversion
    out.append(("clamp_444_dri2", *_clamp_case(rng, 264, 56, S444, 2, False)))
    out.append(("clamp_420_lowac", *_clamp_case(rng, 328, 96, S420, 3, True)))
    out.append(("clamp_422_lowac_nodri", *_clamp_case(rng, 296, 48, S422, 0, True)))
    out.append(("clamp_grey_lowac", *_clamp_case(rng, 120, 40, GREY, 0, True)))
    return out


@functools.lru_cache(maxsize=None)
def colour_sweep():
    return _colour_sweep()


@functools.lru_cache(maxsize=None)
def damaged():
    """[(name, jpeg bytes)]: a truncated 12-bit scan and a wrapping scan with bit flips."""
    c = {n: j for n, j, _ in corpus()}
    p12 = c["p12_420_dri4"]; wrap = c["wrap_q255_420_dri2"]
    lo = wrap.index(b"\xff\xda") + 14
    r = np.random.default_rng(77); a = bytearray(wrap)
    for p in r.integers(lo, len(wrap) - 2, 12):
        a[p] ^= 1 << int(r.integers(0, 8))
    body = p12.index(b"\xff\xda") + 14
    return [("p12_trunc", p12[: body + (len(p12) - body) * 3 // 5] + b"\xff\xd9"), ("wrap_flip12", bytes(a))]


def _oracle(fixed, decode_ac=True):
    if ref_available("fixed" if fixed else "float"):
        return Oracle("ref_fixed" if fixed else "ref_float", decode_ac=decode_ac)
    return Oracle("port", idct_fixed=fixed, decode_ac=decode_ac)


@functools.lru_cache(maxsize=None)
def tables():
    return Oracle("port").idct_tables()


@functools.lru_cache(maxsize=None)
def oracle_out(fixed):
    """name -> the oracle's decode, for the corpus and the 8-bit Pillow images mixed into the batch test."""
    o = _oracle(fixed)                       # decoded right away: the compiled reference's configuration is process-wide
    return {name: o.decode(j) for name, j in [(n, j) for n, j, _ in corpus()] + _mixed_in()}


@functools.lru_cache(maxsize=None)
def expected_out(fixed):
    lf, li = tables()
    return {name: CJ.expected(spec, fixed, li, lf) for name, _, spec in corpus()}


def _mixed_in():
    s = JC.small_cases()
    return [s[3], s[7]]


# --- CPU ----------------------------------------------------------------------------------------------------------------

def test_corpus_reaches_the_edges(built):
    """The corpus really exercises what it is for: 16-bit codes, pixel maps and DC predictors at both ends of int16,
    y>>3 on both sides of the clamps, every (cb, cr) pair, and the three flagged pairs with every y."""
    names = [n for n, _, _ in corpus()]
    assert len(names) == len(set(names))
    ex = expected_out(True)
    lo_hi = lambda a: (int(a.min()), int(a.max()))
    ymin, ymax = zip(*[lo_hi(ex[n].pix_y) for n in names if n.startswith("wrap")])
    assert min(ymin) == -32768 and max(ymax) >= 32760
    dcs = np.concatenate([np.asarray(ex[n].blk_dc[0], np.int64) for n in names if n.startswith("wrap")])
    assert dcs.min() < -30000 and dcs.max() > 30000
    for n in names:
        if n.startswith("clamp"):
            y3 = ex[n].pix_y.astype(np.int64) >> 3
            for v in (-4096, -129, -128, 127, 128, 4095):
                assert (y3 == v).any(), (n, v)
    d = Oracle("port").decode(dict((n, j) for n, j, _ in corpus())["p12_420_dri1"])
    assert d.dht_histo[0, 0, 16] > 0 and d.dht_histo[1, 0, 16] > 0           # 16-bit DC and AC codes
    j, spec = colour_sweep()
    lf, li = tables()
    e = CJ.expected(spec, True, li, lf)
    cb3 = e.pix_cb[:4096].astype(np.int64) >> 3; cr3 = e.pix_cr[:4096].astype(np.int64) >> 3
    assert np.unique((cb3 + 128) * 256 + (cr3 + 128)).size == 65536
    y3 = e.pix_y[:4096].astype(np.int64) >> 3
    assert y3.min() < -128 and y3.max() > 127
    last = (e.pix_y[4096:].astype(np.int64) >> 3, e.pix_cb[4096:].astype(np.int64) >> 3, e.pix_cr[4096:].astype(np.int64) >> 3)
    for p in ((0, 0), (-100, 100), (100, -100)):
        sel = (last[1] == p[0]) & (last[2] == p[1])
        assert np.array_equal(np.unique(last[0][sel]), np.arange(-128, 128)), p


@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_reference_decodes_the_corpus_as_restated(built, fixed):
    """The compiled reference's pixel maps, DIB and block-DC maps equal coef_jpeg.expected() for every corpus image."""
    if not ref_available("fixed" if fixed else "float"):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    o = Oracle("ref_fixed" if fixed else "ref_float")
    lf, li = o.idct_tables()
    for name, j, spec in corpus() + [("colour_sweep",) + colour_sweep()]:
        got = o.decode(j)
        assert got.nerr == 0, (name, o.err_lines()[:3])
        bad = JC.compare(CJ.expected(spec, fixed, li, lf), got, what=FIELDS)
        assert not bad, f"{name}: mismatch in {bad}"


@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_port_matches_the_reference_on_the_corpus(built, fixed):
    """The C port equals the compiled reference on every output (the restatement alone where the reference is not built)."""
    port = Oracle("port", idct_fixed=fixed)
    have_ref = ref_available("fixed" if fixed else "float")
    ref = Oracle("ref_fixed" if fixed else "ref_float") if have_ref else None
    lf, li = port.idct_tables()
    for name, j, spec in corpus() + [("colour_sweep",) + colour_sweep()]:
        got = port.decode(j)
        assert got.nerr == 0, name
        if have_ref:
            want = ref.decode(j)
            assert not JC.compare(want, got), name
            assert np.array_equal(want.stats, got.stats), (name, want.stats, got.stats)
        else:
            assert not JC.compare(CJ.expected(spec, fixed, li, lf), got, what=FIELDS), name


# --- GPU ----------------------------------------------------------------------------------------------------------------

def _check(want, got, name, exp=None, what=None):
    bad = JC.compare(want, got, what=what) if what else JC.compare(want, got)
    assert not bad, f"{name}: mismatch with the oracle in {bad}"
    if exp is not None:
        bad = JC.compare(exp, got, what=FIELDS)
        assert not bad, f"{name}: mismatch with the restatement in {bad}"


@pytest.mark.gpu
@pytest.mark.parametrize("idct", [0, 1, 2, 3], ids=["idct_auto", "idct_simple", "idct_tma", "idct_ldg"])
@pytest.mark.parametrize("huff", [0, 1, 2], ids=["huff_auto", "huff_warp", "huff_lane"])
@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_single_image_dropin_at_the_edges(built, fixed, huff, idct):
    from jpegsnoop_b200 import CimgDecode
    want = oracle_out(fixed); exp = expected_out(fixed)
    dec = CimgDecode(idct_fixedpt=fixed, huff_kernel=huff, idct_kernel=idct)
    for name, j, _ in corpus():
        got = dec.decode(j)
        assert got.nerr == 0 and want[name].nerr == 0, (name, dec.log_lines(3))
        _check(want[name], got, name, exp[name])
        assert np.array_equal(np.asarray(want[name].stats), np.asarray(got.stats)), (name, want[name].stats, got.stats)
    dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("huff", [0, 2], ids=["huff_auto", "huff_lane"])
@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_batch_mixing_8_and_12_bit_images(built, fixed, huff):
    """One 12-bit image switches the whole batch to the GENERIC lane kernel (any_p12): the 8-bit images next to it must not change."""
    from jpegsnoop_b200 import BatchDecoder
    want = oracle_out(fixed); exp = expected_out(fixed)
    named = [(n, j) for n, j, _ in corpus()] + _mixed_in()
    named = named[::2] + named[1::2]                         # 8- and 12-bit images interleaved
    bd = BatchDecoder(idct_fixedpt=fixed, huff_kernel=huff, idct_kernel=0)
    bd.set_batch([j for _, j in named]); bd.decode(); bd.sync()
    for i, (name, j) in enumerate(named):
        got = bd.fetch(i)
        assert got.status == 0, (name, hex(got.status))
        _check(want[name], got, name, exp.get(name), what=BATCH_FIELDS)
    bd.close()


@pytest.mark.gpu
@pytest.mark.parametrize("huff", [0, 1, 2], ids=["huff_auto", "huff_warp", "huff_lane"])
def test_dc_only_mode_at_the_edges(built, huff):
    from jpegsnoop_b200 import CimgDecode
    todo = [(n, j, s) for n, j, s in corpus() if n.startswith(("p12", "wrap"))]
    o = _oracle(True, decode_ac=False)
    want = {n: o.decode(j) for n, j, _ in todo}
    o.close()
    lf, li = tables()
    dec = CimgDecode(decode_ac=False, idct_fixedpt=True, huff_kernel=huff, idct_kernel=0)
    for name, j, spec in todo:
        got = dec.decode(j)
        assert got.nerr == 0 and want[name].nerr == 0, (name, dec.log_lines(3))
        _check(want[name], got, name, CJ.expected(spec, True, li, lf, decode_ac=False))
    dec.close()


@pytest.mark.gpu
@pytest.mark.parametrize("huff", [0, 1, 2], ids=["huff_auto", "huff_warp", "huff_lane"])
def test_damaged_edge_scans_match_the_reference(built, huff):
    """A truncated 12-bit scan and a wrapping scan with bit flips go through the serial exact walk (k_huff_exact) with the
    divide and the 16-bit wraps: every buffer and every error line equal the reference's."""
    if not ref_available("fixed"):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    from jpegsnoop_b200 import CimgDecode
    orc = Oracle("ref_fixed")
    dec = CimgDecode(idct_fixedpt=True, huff_kernel=huff, idct_kernel=0)
    for name, j in damaged():
        want = orc.decode(j); want_lines = orc.err_lines()
        got = dec.decode(j)
        assert want.nerr > 0, name
        _check(want, got, name)
        assert np.array_equal(np.asarray(want.stats)[10:12], np.asarray(got.stats)[10:12]), (name, want.stats, got.stats)
        got_lines = dec.log_lines(3)
        assert got_lines == want_lines, (name, len(got_lines), len(want_lines), [(a, b) for a, b in zip(got_lines, want_lines) if a != b][:3])
    dec.close()


@pytest.mark.gpu
def test_clip_and_histogram_statistics_at_the_clamps(built):
    """bHistoEn + bStatClipEn on wrapping and clamp-edge images: DIB, m_sHisto, m_sStatClip, both histograms, the histogram
    bitmaps and the whole non-quiet log (including the "YCC Clipped" notes) equal the reference's."""
    if not ref_available("fixed"):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    from jpegsnoop_b200 import CimgDecode
    c = {n: j for n, j, _ in corpus()}
    ref = Oracle("ref_fixed")
    try:
        ref.config_histo(True, True, False)
        dec = CimgDecode(); dec.config_histo(True, True, False)
        for name in ("wrap_q255_420_dri2", "clamp_444_dri2", "clamp_420_lowac"):
            want = ref.decode(c[name], quiet=False); got = dec.decode(c[name], quiet=False)
            _check(want, got, name)
            assert np.array_equal(np.asarray(want.stats), np.asarray(got.stats)), (name, want.stats, got.stats)
            ws, gs = ref.colour_stats(), dec.colour_stats()
            for k in ("clip", "ranges", "cc_histo", "y_histo"):
                assert np.array_equal(ws[k], gs[k]), (name, k, ws[k][:16], gs[k][:16])
            assert ws["count"] == gs["count"], name
            for which in (0, 1):
                w, g = ref.histo_dib(which), dec.histo_dib(which)
                assert (w is None) == (g is None), (name, which)
                if w is not None:
                    assert np.array_equal(w, g), (name, "histogram bitmap", which)
            wl, gl = ref.log_lines(), dec.log_lines(-1)
            assert any("YCC Clipped" in ln for ln in wl), name
            assert wl == gl, (name, [(a, b) for a, b in zip(wl, gl) if a != b][:4], len(wl), len(gl))
        dec.close()
    finally:
        ref.config_histo(False, False, False); ref.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_colour_sweep(built, fixed):
    """Every (cb, cr) pair under luma that spans the clamp range, and the pairs the table path hands to the exact routine
    with every y: the DIB (and the maps) equal the restatement and the oracle."""
    from jpegsnoop_b200 import CimgDecode
    j, spec = colour_sweep()
    lf, li = tables()
    exp = CJ.expected(spec, fixed, li, lf)
    want = _oracle(fixed).decode(j)
    got = CimgDecode(idct_fixedpt=fixed).decode(j)
    assert got.nerr == 0 and want.nerr == 0
    _check(want, got, "colour_sweep", exp)


@pytest.mark.gpu
def test_device_checksums_equal_the_reference_checksums(built):
    """bench.py's bit-exactness verdict compares jsgpu_batch_checksums with the reference harness's ref_bench_ck: the two
    must agree word for word on healthy images (odd block counts, greyscale, 12-bit, wrapping and Pillow images)."""
    if not ref_available("fixed"):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    from jpegsnoop_b200 import BatchDecoder
    jpegs = [j for _, j, _ in corpus()] + [colour_sweep()[0]] + [j for _, j in JC.small_cases()] + [j for _, j in JC.mini_cases()]
    bd = BatchDecoder()
    bd.set_batch(jpegs); bd.decode(); bd.sync()
    got = bd.checksums()
    bd.close()
    _, errs, want = Oracle("ref_fixed").bench_ck(jpegs)
    assert errs == 0
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, [(int(i), np.flatnonzero(got[i] != want[i]).tolist()) for i in bad[:5]]
