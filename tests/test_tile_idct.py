"""Stage B: the fused tile kernel k_idct_tile<P1, EHS> (jsgpu_idct.cu, phase 2 in jsgpu_idct_common.cuh), the literal kernels
next to it and the brightest-pixel / average-luma statistics (k_color_simple, k_finalize_stats, k_preview_stats).

The corpus is written at coefficient level by tests/coef_jpeg.py from fixed seeds:
  * one image in each of the 35 three-component layouts whose chroma components are identical and have factors of 1 or the
    maximum, with Hmax in 1, 2, 4 (28 take the fused kernel, 8 of them at its 192-block tile limit; 7 go past the limit to
    k_idct_simple), and greyscale; random AC, DRI 3.  Per chroma class (EHS 0, 1, 2) and tile width, the last tile of a row
    holds 1, 2, tile_mcus - 1 and tile_mcus MCUs; there are images one MCU row high and one tile wide;
  * statistics images: tied maxima whose raster-first occurrence is processed after the other one -- by the same thread in
    the next tile of its run, by another warp, by another CTA --; first occurrences at k = 3 and k = 7 of a thread's 8-pixel
    group under full-resolution chroma; a maximum that exists only in padded columns or rows; Y = 32767; Y = -32768
    everywhere; greyscale; and a white 4112 x 4104 image whose 32-bit luma sum wraps.

CPU: the corpus reaches those edges, by the images and by a restatement of plan_image's layout rule, the tile list and the CTA
partition of launch_tiles (at 132 SMs); the compiled reference equals coef_jpeg.expected / expected_stats on every image in
both IDCT builds, and the C port equals the reference.
GPU: every image through every kernel form against the reference and the restatement, the launch count of each layout, a
batch whose CTA runs cross images of different layouts of one class (checksums of every image, full comparison of a sample),
and the preview / histogram pass over the new MCU sizes."""
import functools
import os

import numpy as np
import pytest

import coef_jpeg as CJ
import jpeg_cases as JC
from oracle_util import Oracle, ref_available

FIELDS = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "blk_dc")
WHAT = FIELDS + ("mcu_map", "dht_histo")
H100_SMS = 132
TILE_BLOCK_LIMIT = 48 * 1024 // (128 * 2)          # 192: the sample planes are double-buffered in 48 KB of shared memory
GREY = ((1, 1),)
S420 = ((2, 2), (1, 1), (1, 1))
S444 = ((1, 1), (1, 1), (1, 1))
S440F = ((1, 2), (1, 2), (1, 2))
AT_LIMIT = {((1, 2),) * 3, ((2, 2),) * 3, ((4, 2),) * 3, ((1, 4), (1, 1), (1, 1)), ((2, 3), (1, 3), (1, 3)),
            ((2, 4), (2, 1), (2, 1)), ((4, 4), (1, 4), (1, 4)), ((4, 4), (4, 1), (4, 1))}
OVER_LIMIT = {((1, 3),) * 3, ((1, 4),) * 3, ((2, 3),) * 3, ((2, 4), (1, 4), (1, 4)), ((2, 4),) * 3, ((4, 3),) * 3, ((4, 4),) * 3}
WHITE = "white_420_4112x4104"
needs_ref = pytest.mark.skipif(not ref_available("fixed"), reason="needs the compiled reference (oracle/_ref)")


# --- plan_image, the tile list and launch_tiles, restated (jsgpu_api.cu, jsgpu_idct.cu) -------------------------------------

def geometry(W, H, samp):
    """(hmax, vmax, mcu_xmax, mcu_ymax)"""
    if len(samp) == 1:
        return 1, 1, -(-W // 8), -(-H // 8)
    return CJ._geometry(W, H, samp)


def tile_mcus(samp):
    return 32 // geometry(8, 8, samp)[0]


def tile_blocks(samp):
    return sum(h * v for h, v in samp) * tile_mcus(samp) if len(samp) == 3 else tile_mcus(samp)


def fused(samp):
    """plan_image's std_layout: component 0 carries Hmax and Vmax, Hmax is 1, 2 or 4, the chroma components are identical
    with factors of 1 or the maximum, and a tile has at most 192 blocks."""
    if len(samp) == 1:
        return True
    hmax, vmax = max(h for h, _ in samp), max(v for _, v in samp)
    ok = samp[0] == (hmax, vmax) and hmax in (1, 2, 4)
    ok = ok and samp[1] == samp[2] and samp[1][0] in (1, hmax) and samp[1][1] in (1, vmax)
    return ok and tile_blocks(samp) <= TILE_BLOCK_LIMIT


def chroma_class(samp):
    """EHS of the launch: chroma replication 1, 2 or 4 horizontally -> 0, 1, 2 (greyscale: 0)."""
    if len(samp) == 1:
        return 0
    return {1: 0, 2: 1, 4: 2}[geometry(8, 8, samp)[0] // samp[1][0]]


def evc(samp):
    return 1 if len(samp) == 1 else geometry(8, 8, samp)[1] // samp[1][1]


def tile_lists(images):
    """images: [(W, H, samp)] in batch order -> per class the tiles (image, mcu row, first mcu col, mcus in tile)."""
    out = [[], [], []]
    for i, (W, H, samp) in enumerate(images):
        if not fused(samp):
            continue
        U = tile_mcus(samp)
        _, _, mx, my = geometry(W, H, samp)
        for r in range(my):
            for t in range(-(-mx // U)):
                out[chroma_class(samp)].append((i, r, t * U, min(U, mx - t * U)))
    return out


def grid_of(cnt, sms, fixed):
    return min(sms * (5 if fixed else 4), cnt)


def runs(cnt, grid):
    """CTA b walks tiles [cnt * b / grid, cnt * (b + 1) / grid) of its class."""
    return [(cnt * b // grid, cnt * (b + 1) // grid) for b in range(grid)]


def run_of(cnt, grid, t):
    return next(b for b, (s, e) in enumerate(runs(cnt, grid)) if s <= t < e)


# --- the corpus -------------------------------------------------------------------------------------------------------------

def layouts():
    """The 35 layouts with identical chroma whose factors are 1 or the maximum, Hmax in 1, 2, 4."""
    return [((hm, vm), (hc, vc), (hc, vc)) for hm in (1, 2, 4) for vm in (1, 2, 3, 4)
            for hc in sorted({1, hm}) for vc in sorted({1, vm})]


def lname(samp):
    return "grey" if len(samp) == 1 else "_".join("%dx%d" % hv for hv in samp[:2])


def _zero_blocks(W, H, samp):
    return [np.zeros(CJ.block_shape(W, H, samp, c) + (64,), np.int64) for c in range(len(samp))]


def _layout_images():
    """[(name, W, H, samp, seed)]: per (class, tile width) group, the k-th fused image's last tile holds (1, 2, U-1, U)[k % 4]
    MCUs; rows of tiles alternate between one tile and two, heights between one MCU row and two or three."""
    groups = {}
    out = []
    for k, samp in enumerate(layouts() + [GREY]):
        U = tile_mcus(samp)
        key = (chroma_class(samp), U) if fused(samp) else ("over",)
        n = groups.get(key, 0); groups[key] = n + 1
        nmt = (1, 2, U - 1, U)[n % 4]
        tiles = 1 + (n // 2) % 2
        rows = (1, 2, 1, 3)[n % 4]
        hmax, vmax, _, _ = geometry(8, 8, samp)
        mw, mh = 8 * hmax, 8 * vmax
        W = ((tiles - 1) * U + nmt) * mw - (5 * k) % mw
        H = rows * mh - (3 * k) % mh
        out.append((lname(samp), W, H, samp, 1000 + k))
    return out


def _random_image(W, H, samp, seed):
    rng = np.random.default_rng(seed)
    bl = []
    for c in range(len(samp)):
        shape = CJ.block_shape(W, H, samp, c)
        b = np.zeros(shape + (64,), np.int64)
        b[..., 0] = rng.integers(-700, 700, shape)
        b[..., 1:] = np.where(rng.random(shape + (63,)) < 0.15, rng.integers(-40, 41, shape + (63,)), 0)
        bl.append(b)
    q = [rng.integers(1, 6, 64), rng.integers(1, 6, 64)]
    return CJ.encode_coefs(bl, W, H, samp, q, [0, 1, 1][:len(samp)], dri=3)


@functools.lru_cache(maxsize=None)
def idct_tables():
    return Oracle("port").idct_tables()           # (lf, li): the port's PrecalcIdct equals the reference's (test_oracle)


def n8(n, a, fixed):
    """The 8x8 samples (before the DC level shift) of a block whose only AC coefficient is natural index n = a (quantiser 1)."""
    lf, li = idct_tables()
    coef = np.zeros((1, 64), np.int64); coef[0, n] = a
    if fixed:
        s = CJ._i16(CJ._idct_fixed(coef, li)) * 8
    else:
        s = CJ._i16(CJ._f2i_trunc(CJ._idct_float(coef, lf) * np.float32(8)))
    return s.reshape(8, 8)


def cosine(n, first):
    """(a, peak): the smallest |a| >= 40 for which a block with only coefficient n = a has its raster-first maximum at
    `first` (y, x) and the same peak in both IDCT builds."""
    for mag in range(40, 400):
        for a in (mag, -mag):
            p = [n8(n, a, f) for f in (True, False)]
            if all(np.unravel_index(np.argmax(s), s.shape) == first for s in p) and p[0].max() == p[1].max():
                return a, int(p[0].max())
    raise AssertionError(("no coefficient value", n, first))


def _peak(blk, r, c, dc):
    blk[r, c, :] = 0; blk[r, c, 0] = dc


def _tie_thread():
    """4:2:0, 4096 x 688: 688 tiles (16 per MCU row), more than the grid of either IDCT build at 132 SMs, so a CTA walks two
    tiles in a row.  A flat block of 900 sits in block row 1 of tile c, another in block row 0 of tile c + 1 at the same
    column of its tile: the second one is raster-first (row 0 < row 8) and reaches the same lane of the same warp (rows 0 and 8
    are both warp 0's) one tile later.  c is chosen so that c and c + 1 share an MCU row and a CTA run in both builds."""
    W, H = 4096, 688
    cnt = 16 * 43
    for c in range(cnt - 1):
        if c % 16 != 15 and all(run_of(cnt, grid_of(cnt, H100_SMS, f), c) == run_of(cnt, grid_of(cnt, H100_SMS, f), c + 1)
                                for f in (True, False)):
            break
    else:
        raise AssertionError("no tile pair inside one run")
    bl = _zero_blocks(W, H, S420)
    row, col = c // 16, c % 16
    j = 5                                                  # block column inside the tile = the lane
    _peak(bl[0], 2 * row + 1, 32 * col + j, 900)
    _peak(bl[0], 2 * row, 32 * (col + 1) + j, 900)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, W, H, S420, [q1, q1], [0, 1, 1], dri=16)


def _tie_warp():
    """1x2 for all three components (16-row MCUs, one row group per pixel row), one tile (256 x 16): a block with a negative
    v = 1 coefficient peaks only in its row 7 (warp 3); a flat block of the same value starts at row 8 (warp 0) further
    left: the raster-first occurrence is warp 3's."""
    W, H = 256, 16
    a, pk = cosine(8, (7, 0))
    bl = _zero_blocks(W, H, S440F)
    bl[0][0, 20, 0] = 100; bl[0][0, 20, 8] = a             # natural order: index 8 is (v, u) = (1, 0)
    _peak(bl[0], 1, 3, 100 + pk)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, W, H, S440F, [q1, q1], [0, 1, 1], dri=4)


def _tie_cta():
    """4:2:0, two tiles in one MCU row (512 x 16): one CTA each.  A flat block in block row 1 of tile 0, one of the same
    value in block row 0 of tile 1: the raster-first occurrence is the other CTA's."""
    bl = _zero_blocks(512, 16, S420)
    _peak(bl[0], 1, 10, 640)
    _peak(bl[0], 0, 40, 640)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, 512, 16, S420, [q1, q1], [0, 1, 1], dri=2)


def _first_at(k):
    """4:4:4 (full-resolution chroma: every pixel of a group has its own Cb, Cr), 128 x 16.  A block whose only AC
    coefficient (u = 2 for k = 3, u = 1 for k = 7) puts its raster-first maximum at x = k of its 8-pixel group, and further
    on a flat block of the same value (k = 0).  Cb and Cr ramp across the group, so the brightest pixel's Cb / Cr / RGB
    tell k = 0 from k."""
    W, H = 128, 16
    a, pk = cosine(2 if k == 3 else 1, (0, k))
    bl = _zero_blocks(W, H, S444)
    bl[0][0, 3, 0] = 50; bl[0][0, 3, 2 if k == 3 else 1] = a
    _peak(bl[0], 1, 9, 50 + pk)
    bl[1][0, 3, 1] = 300; bl[2][0, 3, 1] = -300              # u = 1 ramps of +-37 in cb >> 3, cr >> 3 across the group
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, W, H, S444, [q1, q1], [0, 1, 1], dri=3)


def _pad_cols():
    """4:2:0, 81 x 32 (Wp = 96): the maximum is a flat block at x = 88..95, all padding."""
    bl = _zero_blocks(81, 32, S420)
    bl[0][..., 0] = np.arange(bl[0].shape[1])[None, :] * 8
    _peak(bl[0], 2, 11, 700)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, 81, 32, S420, [q1, q1], [0, 1, 1], dri=3)


def _pad_rows():
    """4:4:0 (1x2 + 1x1), 40 x 33 (Hp = 48): the maximum is a flat block at y = 40..47, all padding."""
    samp = ((1, 2), (1, 1), (1, 1))
    bl = _zero_blocks(40, 33, samp)
    bl[0][..., 0] = np.arange(bl[0].shape[0])[:, None] * 16
    _peak(bl[0], 5, 2, 900)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, 40, 33, samp, [q1, q1], [0, 1, 1], dri=2)


def _y_max():
    """4:2:2 with random content and one flat block of Y = 32767."""
    samp = ((2, 1), (1, 1), (1, 1))
    j, spec = _random_image(96, 24, samp, 77)
    bl = [b.copy() for b in spec["blocks"]]
    qt = [q.copy() for q in spec["qtabs"]]; qt[0][0] = 1
    _peak(bl[0], 1, 6, 0); _peak(bl[0], 1, 7, 32767); _peak(bl[0], 1, 8, 0)     # DC steps of +-32767
    return CJ.encode_coefs(bl, 96, 24, samp, qt, [0, 1, 1], dri=3)


def _all_min():
    """4:4:4, every sample -32768 (DC -16384 dequantised by 2): no pixel beats the initial brightest value."""
    bl = _zero_blocks(48, 24, S444)
    for b in bl:
        b[..., 0] = -16384
    q2 = np.full(64, 2)
    return CJ.encode_coefs(bl, 48, 24, S444, [q2, q2], [0, 1, 1], dri=4)


def _grey_stats():
    """Greyscale, random content with two flat blocks at a new maximum in consecutive block rows, the raster-first one
    further right."""
    j, spec = _random_image(200, 40, GREY, 78)
    bl = [spec["blocks"][0].copy()]
    qt = spec["qtabs"][0].copy(); qt[0] = 1
    _peak(bl[0], 2, 3, 20000); _peak(bl[0], 3, 1, 20000)
    return CJ.encode_coefs(bl, 200, 40, GREY, [qt], [0], dri=3)


def _white():
    """4:2:0, 4112 x 4104 (padded 4112 x 4112), DC-only, Y = 1020 everywhere: Y8 = 255, so the luma sum is
    255 x 4112 x 4112 = 4 311 744 960 and wraps past 2^32 in the reference's 32-bit unsigned."""
    W, H = 4112, 4104
    bl = _zero_blocks(W, H, S420)
    bl[0][..., 0] = 1020
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, W, H, S420, [q1, q1], [0, 1, 1])


@functools.lru_cache(maxsize=None)
def layout_corpus():
    """[(name, jpeg, spec)]"""
    return [(n, *_random_image(W, H, samp, seed)) for n, W, H, samp, seed in _layout_images()]


@functools.lru_cache(maxsize=None)
def stats_corpus():
    return [("tie_thread_420", *_tie_thread()), ("tie_warp_440", *_tie_warp()), ("tie_cta_420", *_tie_cta()),
            ("first_k3_444", *_first_at(3)), ("first_k7_444", *_first_at(7)), ("pad_cols_420", *_pad_cols()),
            ("pad_rows_440", *_pad_rows()), ("y32767_422", *_y_max()), ("all_min_444", *_all_min()),
            ("grey_stats", *_grey_stats())]


@functools.lru_cache(maxsize=None)
def white():
    return _white()


def corpus(with_white=False):
    return layout_corpus() + stats_corpus() + ([(WHITE, *white())] if with_white else [])


@functools.lru_cache(maxsize=None)
def expected(name, fixed):
    spec = {n: s for n, _, s in corpus(True)}[name]
    lf, li = idct_tables()
    e = CJ.expected(spec, fixed, li, lf)
    return e, CJ.expected_stats(e)


def _samp(spec):
    return spec["samp"] if len(spec["samp"]) == 3 else GREY


# --- CPU: the corpus reaches its edges ----------------------------------------------------------------------------------------

def test_every_layout_is_on_its_side_of_the_rule():
    L = layouts()
    assert len(L) == len(set(L)) == 35
    assert sum(fused(s) for s in L) == 28
    assert {s for s in L if tile_blocks(s) == TILE_BLOCK_LIMIT} == AT_LIMIT and all(fused(s) for s in AT_LIMIT)
    assert {s for s in L if not fused(s)} == OVER_LIMIT
    assert fused(GREY) and not fused(((3, 1), (1, 1), (1, 1)))
    names = {lname(_samp(spec)) for _, _, spec in layout_corpus()}
    assert names == {lname(s) for s in L + [GREY]}
    # full resolution in one direction only: phase 2 with EHS = 0 and evc > 1, or EHS > 0 and evc = 1
    one_dir = {(chroma_class(s), evc(s) > 1) for s in L if fused(s)}
    assert (0, True) in one_dir and (1, False) in one_dir and (2, False) in one_dir


def test_last_tiles_cover_every_width():
    """Per class and tile width: the last tile of a row holds 1, 2, tile_mcus - 1 and tile_mcus MCUs; one-MCU-row images and
    images one tile wide in every class."""
    seen, one_row, one_tile = {}, set(), set()
    for name, j, spec in layout_corpus():
        samp = _samp(spec)
        if not fused(samp):
            continue
        U = tile_mcus(samp); cls = chroma_class(samp)
        _, _, mx, my = geometry(spec["W"], spec["H"], samp)
        last = tile_lists([(spec["W"], spec["H"], samp)])[cls][-1][3]
        seen.setdefault((cls, U), set()).add(last)
        if my == 1:
            one_row.add(cls)
        if mx <= U:
            one_tile.add(cls)
    assert set(seen) == {(0, 32), (0, 16), (0, 8), (1, 16), (2, 8)}, seen
    for (cls, U), s in seen.items():
        assert {1, 2, U - 1, U} <= s, (cls, U, s)
    assert one_row == one_tile == {0, 1, 2}


def _first_max(name, fixed=True):
    e, st = expected(name, fixed)
    y = np.asarray(e.pix_y, np.int64)
    idx = np.flatnonzero(y.ravel() == y.max())
    Wp = y.shape[1]
    return e, st, [(int(i) // Wp, int(i) % Wp) for i in idx]


def _thread(samp, yx, mcu_h):
    """(tile-local lane, warp) that handles pixel (y, x) in phase 2; rows of an MCU row go to warps by row group."""
    y, x = yx
    U = tile_mcus(samp); mw = 256 // U
    rg = (y % mcu_h) // evc(samp)
    return ((x % 256) // 8, rg % 4), (y // mcu_h, x // 256), rg


@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_statistics_images_reach_their_edges(fixed):
    """The ties are processed in the stated order (132 SMs), the first maxima sit at k = 3 and 7 under a chroma ramp, the
    padding, 32767, -32768 and wrap images are what they say."""
    spec = {n: s for n, _, s in corpus()}
    # same thread, next tile of its run: raster-first occurrence in tile c + 1, the other in tile c, same lane and warp
    e, st, occ = _first_max("tie_thread_420", fixed)
    s = spec["tie_thread_420"]
    firsts = [p for p in occ if p[0] % 8 == 0 and p[1] % 8 == 0]      # block corners
    (la, wa), (ra, ta), _ = _thread(S420, firsts[1], 16)
    (lb, wb), (rb, tb), _ = _thread(S420, firsts[0], 16)
    assert firsts[0][0] < firsts[1][0] and (la, wa) == (lb, wb) and ra == rb and tb == ta + 1, firsts
    cnt = len(tile_lists([(s["W"], s["H"], S420)])[1])
    grid = grid_of(cnt, H100_SMS, fixed)
    ti = lambda p: (p[0] // 16) * 16 + p[1] // 256
    assert cnt > grid and run_of(cnt, grid, ti(firsts[0])) == run_of(cnt, grid, ti(firsts[1]))
    assert (st[8], st[9]) == (firsts[0][1] // 16, firsts[0][0] // 16)
    # another warp of the same CTA: the raster-first occurrence is warp 3's (row 7), the flat block's first row is warp 0's
    e, st, occ = _first_max("tie_warp_440", fixed)
    (l0, w0), (r0, t0), _ = _thread(S440F, occ[0], 16)
    later = [_thread(S440F, p, 16) for p in occ[1:]]
    assert occ[0][0] == 7 and w0 == 3 and all(t == t0 for _, (_, t), _ in later)
    rest = [p for p in occ if p[0] != 7]
    assert all(p[0] >= 8 for p in rest) and _thread(S440F, rest[0], 16)[0][1] == 0, rest[:3]
    # another CTA
    e, st, occ = _first_max("tie_cta_420", fixed)
    assert occ[0][1] >= 256 and any(p[1] < 256 and p[0] > occ[0][0] for p in occ)
    # k = 3 / 7 of the 8-pixel group; an equal value at k = 0 further on; Cb and Cr at k differ from those at k = 0
    for name, k in (("first_k3_444", 3), ("first_k7_444", 7)):
        e, st, occ = _first_max(name, fixed)
        y0, x0 = occ[0]
        assert x0 % 8 == k and any(p[1] % 8 == 0 and p > occ[0] for p in occ), (name, occ[:4])
        g = x0 - k
        assert (e.pix_cb[y0, g] >> 3) != (e.pix_cb[y0, x0] >> 3) and (e.pix_cr[y0, g] >> 3) != (e.pix_cr[y0, x0] >> 3)
        assert tuple(CJ.ycc_to_bgra(e.pix_y[y0, x0], e.pix_cb[y0, g], e.pix_cr[y0, g])) != tuple(CJ.ycc_to_bgra(e.pix_y[y0, x0], e.pix_cb[y0, x0], e.pix_cr[y0, x0]))
    # the maximum exists only in padding
    e, st, occ = _first_max("pad_cols_420", fixed)
    assert all(x >= spec["pad_cols_420"]["W"] for _, x in occ)
    e, st, occ = _first_max("pad_rows_440", fixed)
    assert all(y >= spec["pad_rows_440"]["H"] for y, _ in occ)
    e, st = expected("y32767_422", fixed)
    assert e.pix_y.max() == 32767 and st[2] == 32767
    e, st = expected("all_min_444", fixed)
    assert (e.pix_y == -32768).all() and (e.pix_cb == -32768).all() and tuple(st[2:10]) == (-32768, -32768, -32768, 0, 135, 0, 0, 0)
    assert len(spec["grey_stats"]["samp"]) == 1
    if fixed:
        e, st = expected(WHITE, True)
        Wp, Hp = int(e.geom[6]), int(e.geom[7])
        assert 255 * Wp * Hp >= 1 << 32 and (e.pix_y >> 3 >= 127).all() and st[0] == 0


# --- the batch whose CTA runs cross images -----------------------------------------------------------------------------------

BIG_TILES_PER_ROW = 15


def _big(tie):
    """4:2:0, 3840 x 2160 (2025 tiles, 15 per MCU row), random DC and some AC: flat blocks of 1000 in block row 1 of tile
    tie - 1 and in block row 0 of tile tie (same MCU row), the latter raster-first."""
    W, H = 3840, 2160
    rng = np.random.default_rng(4242)
    bl = _zero_blocks(W, H, S420)
    for b in bl:
        b[..., 0] = rng.integers(-300, 300, b.shape[:2])
    band = bl[0][:40]
    band[..., 1:12] = np.where(rng.random(band.shape[:2] + (11,)) < 0.3, rng.integers(-20, 21, band.shape[:2] + (11,)), 0)
    r, c = divmod(tie, BIG_TILES_PER_ROW)
    _peak(bl[0], 2 * r + 1, 32 * (c - 1) + 9, 1000)
    _peak(bl[0], 2 * r, 32 * c + 9, 1000)
    q1 = np.ones(64, np.int64)
    return CJ.encode_coefs(bl, W, H, S420, [q1, q1], [0, 1, 1], dri=8)


@functools.lru_cache(maxsize=None)
def big(tie):
    return _big(tie)


def _exotic():
    """3x1 + 1x1: Hmax 3, the literal kernels."""
    return _random_image(72, 16, ((3, 1), (1, 1), (1, 1)), 99)


@functools.lru_cache(maxsize=None)
def exotic():
    return _exotic()


@functools.lru_cache(maxsize=None)
def batch_pool():
    """[(name, jpeg, spec)]: one image per fused layout and greyscale, all padded to 256 x 192 (one tile wide, 6 to 24 tiles
    high), ragged inside the last MCU."""
    out = []
    for k, samp in enumerate([s for s in layouts() if fused(s)] + [GREY]):
        hmax, vmax, _, _ = geometry(8, 8, samp)
        W, H = 256 - (3 * k) % (8 * hmax), 192 - (5 * k) % (8 * vmax)
        out.append(("pool_" + lname(samp), *_random_image(W, H, samp, 3000 + k)))
    return out


def _npix(s):
    _, _, mx, my = geometry(s["W"], s["H"], _samp(s))
    hmax, vmax, _, _ = geometry(8, 8, _samp(s))
    return mx * my * 64 * hmax * vmax


@functools.lru_cache(maxsize=None)
def batch(sms, fixed):
    """[(name, jpeg, spec)] of one batch.  Per class the pool images of that class in turn (neighbours differ in layout)
    until the class has 3 x grid tiles; in class 1 the 3840 x 2160 image last, its tied tiles on both sides of a run
    boundary; an over-limit or the 3x1 image after every 16 images.  Every fused image has more tiles than a run is long and
    padded sizes never decrease along a class: a run that carried one image's statistics into the next would show as a
    wrong value in an image that holds the carried pixel index."""
    pools = [[], [], []]
    for n, j, s in batch_pool():
        pools[chroma_class(_samp(s))].append((n, j, s))
    over = [(n, j, s) for n, j, s in layout_corpus() if not fused(_samp(s))] + [("exotic_3x1", *exotic())]
    g = sms * (5 if fixed else 4)
    ntiles = lambda s: len(sum(tile_lists([(s["W"], s["H"], _samp(s))]), []))
    per = [[], [], []]
    for cls in (0, 2):
        k = 0
        while sum(ntiles(s) for _, _, s in per[cls]) < 3 * g:
            per[cls].append(pools[cls][k % len(pools[cls])]); k += 1
    per[1] = [pools[1][k % len(pools[1])] for k in range(2 * len(pools[1]))]
    off = sum(ntiles(s) for _, _, s in per[1])
    cnt = off + 2025
    tie = next(s - off for s, _ in runs(cnt, min(g, cnt))
               if 67 * BIG_TILES_PER_ROW <= s - off < 2025 and (s - off) % BIG_TILES_PER_ROW)
    per[1].append((f"big_420_3840x2160_tie{tie}", *big(tie)))
    out = []
    n = max(len(p) for p in per)
    for i in range(n):
        for cls in (0, 1, 2):
            if i < len(per[cls]):
                out.append(per[cls][i])
        if i % 16 == 15:
            out.append(over[(i // 16) % len(over)])
    return out


def batch_reach(items, sms, fixed):
    """Per class: tile count, grid, shortest and longest run, runs that cross a boundary between two different layouts, the
    kinds of such boundaries, the fewest runs an image spans, whether padded sizes never decrease; and the runs that hold
    the big image's tied tiles."""
    images = [(s["W"], s["H"], _samp(s)) for _, _, s in items]
    tl = tile_lists(images)
    out = {}
    tie_runs = set()
    for cls in range(3):
        cnt = len(tl[cls]); grid = grid_of(cnt, sms, fixed)
        rr = runs(cnt, grid)
        run_at = np.repeat(np.arange(grid), [e - s for s, e in rr])
        cross, kinds = 0, set()
        for s, e in rr:
            hit = False
            for t in range(s + 1, e):
                a, b = tl[cls][t - 1][0], tl[cls][t][0]
                la, lb = images[a][2], images[b][2]
                if a != b and la != lb:
                    hit = True
                    if len(la) != len(lb):
                        kinds.add("grey_colour")
                    if TILE_BLOCK_LIMIT in (tile_blocks(la), tile_blocks(lb)) and min(tile_blocks(la), tile_blocks(lb)) <= 96:
                        kinds.add("limit_small")
            cross += hit
        spans, order = {}, []
        for t, (i, r, c0, nmt) in enumerate(tl[cls]):
            spans.setdefault(i, set()).add(int(run_at[t]))
            if not order or order[-1] != i:
                order.append(i)
            name = items[i][0]
            if name.startswith("big"):
                tie = int(name.rsplit("tie", 1)[1])
                if r * BIG_TILES_PER_ROW + c0 // 16 in (tie - 1, tie):
                    tie_runs.add(int(run_at[t]))
        sizes = [_npix(items[i][2]) for i in order]
        out[cls] = dict(cnt=cnt, grid=grid, shortest=min(e - s for s, e in rr), longest=max(e - s for s, e in rr),
                        cross=cross, kinds=kinds, fewest_runs=min(len(v) for v in spans.values()),
                        sizes_ascend=all(a <= b for a, b in zip(sizes, sizes[1:])))
    return out, tie_runs


@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_batch_partition_at_132_sms(fixed):
    _check_partition(batch(H100_SMS, fixed), H100_SMS, fixed)


def _check_partition(items, sms, fixed):
    reach, tie_runs = batch_reach(items, sms, fixed)
    print(reach, tie_runs)
    for cls, r in reach.items():
        assert r["cnt"] >= 3 * sms * (5 if fixed else 4) and r["shortest"] >= 2, (cls, r)
        assert r["fewest_runs"] >= 2 and r["sizes_ascend"], (cls, r)
    assert sum(r["cross"] for r in reach.values()) >= 100, reach
    assert "grey_colour" in reach[0]["kinds"] and any("limit_small" in r["kinds"] for r in reach.values()), reach
    assert len(tie_runs) == 2, tie_runs
    names = {n for n, _, _ in items}
    assert "exotic_3x1" in names and any(lname(_samp(s)) in {lname(o) for o in OVER_LIMIT} for _, _, s in items)


# --- CPU: the reference equals the restatement; the port equals the reference -------------------------------------------------

@needs_ref
@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_reference_decodes_the_corpus_as_restated(built, fixed):
    """Maps, DIB, block-DC maps and stats[0:10] of the compiled reference equal expected() / expected_stats() on every image
    (the 4112 x 4104 image in the integer build only)."""
    if not ref_available("fixed" if fixed else "float"):
        pytest.skip("needs the compiled reference (oracle/_ref)")
    o = Oracle("ref_fixed" if fixed else "ref_float")
    extra = [(WHITE, *white())] if fixed else []
    batch_images = list({n: (n, j, s) for n, j, s in batch(H100_SMS, fixed) if n.startswith(("pool", "big"))}.values())
    for name, j, spec in corpus() + extra + batch_images:
        got = o.decode(j)
        assert got.nerr == 0, (name, o.err_lines()[:3])
        lf, li = idct_tables()
        e = CJ.expected(spec, fixed, li, lf)
        bad = JC.compare(e, got, what=FIELDS)
        assert not bad, (name, bad)
        assert np.array_equal(CJ.expected_stats(e), got.stats[:10]), (name, CJ.expected_stats(e), got.stats)


@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_port_matches_the_reference_on_the_corpus(built, fixed):
    port = Oracle("port", idct_fixed=fixed)
    have_ref = ref_available("fixed" if fixed else "float")
    ref = Oracle("ref_fixed" if fixed else "ref_float") if have_ref else None
    for name, j, spec in corpus():
        got = port.decode(j)
        assert got.nerr == 0, name
        if have_ref:
            want = ref.decode(j)
            assert not JC.compare(want, got), name
            assert np.array_equal(want.stats, got.stats), (name, want.stats, got.stats)
        else:
            e, st = expected(name, fixed)
            assert not JC.compare(e, got, what=FIELDS) and np.array_equal(st, got.stats[:10]), name


# --- GPU ------------------------------------------------------------------------------------------------------------------------

def _oracle(fixed):
    return Oracle("ref_fixed" if fixed else "ref_float")


@functools.lru_cache(maxsize=None)
def ref_out(fixed):
    """name -> the reference's decode (the 4112 x 4104 image in the integer build only)."""
    o = _oracle(fixed)
    return {n: o.decode(j) for n, j, _ in corpus(fixed)}


def _check(want, got, name, exp=None, what=WHAT):
    bad = JC.compare(want, got, what=what)
    assert not bad, f"{name}: mismatch with the reference in {bad}"
    if exp is not None:
        e, st = exp
        bad = JC.compare(e, got, what=FIELDS)
        assert not bad, f"{name}: mismatch with the restatement in {bad}"


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("idct", [0, 1], ids=["fused", "simple"])
@pytest.mark.parametrize("build", ["int_immediates", "int_smem", "float"])
def test_single_image_in_every_kernel_form(built, build, idct, monkeypatch):
    """Every corpus image through CimgDecode: every buffer and the whole stats row against the reference, the maps against
    expected() and stats[0:10] against expected_stats()."""
    from jpegsnoop_b200 import CimgDecode
    fixed = build != "float"
    if build == "int_smem":
        monkeypatch.setenv("JSGPU_IDCT_TABLE", "0")
    with_white = build == "int_immediates"
    want = ref_out(fixed)
    dec = CimgDecode(idct_fixedpt=fixed, huff_kernel=0, idct_kernel=idct)
    for name, j, _ in corpus(with_white):
        got = dec.decode(j)
        assert got.nerr == 0, (name, dec.log_lines(3))
        _check(want[name], got, name, expected(name, fixed))
        assert np.array_equal(np.asarray(want[name].stats), np.asarray(got.stats)), (name, want[name].stats, got.stats)
        assert np.array_equal(expected(name, fixed)[1], np.asarray(got.stats)[:10]), (name, expected(name, fixed)[1], got.stats)
    dec.close()


@pytest.mark.gpu
def test_launch_counts_follow_the_layout_rule(built):
    """Decoded alone, a fused layout takes one IDCT launch fewer with idct_kernel 0 (one k_idct_tile) than with 1
    (k_idct_simple + k_color_simple); an over-limit layout takes the same number either way."""
    from jpegsnoop_b200 import BatchDecoder
    for name, j, spec in layout_corpus():
        n = []
        for idct in (0, 1):
            bd = BatchDecoder(huff_kernel=0, idct_kernel=idct)
            bd.set_batch([j]); bd.decode(); bd.sync()
            n.append(bd.launches())
            assert bd.fetch(0).status == 0, name
            bd.close()
        assert n[1] - n[0] == (1 if fused(_samp(spec)) else 0), (name, n)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_cta_runs_cross_images(built, fixed):
    """One batch per IDCT build in which every class has at least 3 x grid tiles (grid from the device's SM count): every
    CTA walks two tiles or more, runs cross images of different layouts of one class, and the 3840 x 2160 image's tied
    maximum lies in two runs.  Checksums of every image against the reference; one image per layout, both images at
    sampled boundaries inside runs and the large image compared in full."""
    import torch
    from jpegsnoop_b200 import BatchDecoder
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    items = batch(sms, fixed)
    _check_partition(items, sms, fixed)
    jpegs = [j for _, j, _ in items]
    distinct = {}
    for n, j, s in items:
        distinct.setdefault(n, (j, s))
    o = _oracle(fixed)
    names = list(distinct)
    _, errs, ck = o.bench_ck([distinct[n][0] for n in names])
    assert errs == 0
    want_ck = dict(zip(names, ck))
    bd = BatchDecoder(idct_fixedpt=fixed, huff_kernel=0, idct_kernel=0)
    bd.set_batch(jpegs); bd.decode(); bd.sync()
    got = bd.checksums()
    bad = [(i, items[i][0], np.flatnonzero(got[i] != want_ck[items[i][0]]).tolist()) for i in range(len(items))
           if not np.array_equal(got[i], want_ck[items[i][0]])]
    assert not bad, (len(bad), bad[:8])
    # full comparison: the first image of every name and both images of sampled boundaries inside runs
    pick = {}
    for i, (n, _, _) in enumerate(items):
        pick.setdefault(n, i)
    images = [(s["W"], s["H"], _samp(s)) for _, _, s in items]
    tl = tile_lists(images)
    bnd = set()
    for cls in range(3):
        cnt = len(tl[cls]); rr = runs(cnt, grid_of(cnt, sms, fixed))
        hits = [(tl[cls][t - 1][0], tl[cls][t][0]) for s, e in rr for t in range(s + 1, e)
                if tl[cls][t - 1][0] != tl[cls][t][0] and images[tl[cls][t - 1][0]][2] != images[tl[cls][t][0]][2]]
        for a, b in hits[::max(1, len(hits) // 12)]:
            bnd.update((a, b))
    want = {}
    for i in sorted(set(pick.values()) | bnd):
        n, j, spec = items[i]
        if n not in want:
            want[n] = o.decode(j)
        g = bd.fetch(i)
        assert g.status == 0, (i, n)
        _check(want[n], g, f"{n} (image {i})")
        assert np.array_equal(CJ.device_stats(g.stats), np.asarray(want[n].stats)[:10]), (i, n, g.stats, want[n].stats)
        if n != "exotic_3x1":
            lf, li = idct_tables()
            e = CJ.expected(spec, fixed, li, lf)
            assert not JC.compare(e, g, what=FIELDS), (i, n)
            assert np.array_equal(CJ.expected_stats(e), CJ.device_stats(g.stats)), (i, n)
    bd.close()


def _preview_ref(ref, j, mx, my):
    ref.set_preview_mode(1); ref.set_ycc_offset(0, 0, 0, 0, 0)
    ref.set_ycc_offset(mx, my, 40, -30, 25); ref.set_preview_mode(6)
    return ref.decode(j)


@pytest.mark.gpu
@needs_ref
def test_preview_over_the_new_layouts(built):
    """hist_en + statclip_en, preview mode 6 and a YCC shift from an MCU in the middle of a row (k_preview, pv_shifted with
    MCUs of 8 to 32 pixels): the batch pass and the single-image drop-in against the reference -- DIB, stats and the colour
    statistics.  Then the 4112 x 4104 image with the histogram on: k_preview_stats' average wraps like the reference's."""
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    items = layout_corpus()
    ref = Oracle("ref_fixed")
    order = (0, 1, 2, 3, 4, 5, 9, 10, 11, 6, 7, 8)          # PixelCcHisto's member order -> jsgpu_colour_stats channel order
    try:
        ref.config_histo(True, True, False)
        shift = []
        for n, j, spec in items:
            _, _, mx, my = geometry(spec["W"], spec["H"], _samp(spec))
            shift.append((mx // 2, my // 2))
        want = []
        for (n, j, spec), (mx, my) in zip(items, shift):
            w = _preview_ref(ref, j, mx, my)
            want.append((w, ref.colour_stats(), ref.bitmap()))
        # single-image drop-in
        dec = CimgDecode(); dec.config_histo(True, True, False)
        for (n, j, spec), (mx, my), (w, ws, wd) in zip(items, shift, want):
            dec.SetPreviewMode(1); dec.SetPreviewYccOffset(0, 0, 0, 0, 0)
            dec.SetPreviewYccOffset(mx, my, 40, -30, 25); dec.SetPreviewMode(6)
            g = dec.decode(j)
            assert np.array_equal(wd, dec.bitmap()), n
            assert np.array_equal(np.asarray(w.stats), np.asarray(g.stats)), (n, w.stats, g.stats)
            gs = dec.colour_stats()
            for k in ("clip", "ranges", "cc_histo", "y_histo"):
                assert np.array_equal(ws[k], gs[k]), (n, k)
            assert ws["count"] == gs["count"], n
        dec.close()
        # batch: one image at a time shares nothing, so the shift MCU is per image: one batch per distinct shift
        by_shift = {}
        for i, s in enumerate(shift):
            by_shift.setdefault(s, []).append(i)
        for (mx, my), idx in by_shift.items():
            bd = BatchDecoder()
            bd.set_preview(hist_en=1, statclip_en=1, mode=6, shift_y=40, shift_cb=-30, shift_cr=25, shift_mcu_x=mx, shift_mcu_y=my)
            bd.set_batch([items[i][1] for i in idx]); bd.decode(); bd.sync()
            for b, i in enumerate(idx):
                n = items[i][0]; w, ws, wd = want[i]
                g = bd.fetch(b)
                assert np.array_equal(wd, g.dib), n
                assert np.array_equal(CJ.device_stats(g.stats), np.asarray(w.stats)[:10]), (n, g.stats, w.stats)
                s = bd.colour_stats(b)
                assert np.array_equal(ws["clip"], np.array(s.clip[:], np.uint32)), (n, ws["clip"], s.clip[:])
                assert np.array_equal(ws["y_histo"], np.array(s.y_histo[:], np.uint32)), n
                assert np.array_equal(ws["cc_histo"], np.array([list(r) for r in s.cc_histo], np.uint32)), n
                assert ws["count"] == s.count, n
                rng = np.array([[s.vmin[k], s.vmax[k], np.int64(s.vsum[k]).astype(np.int32)] for k in order], np.int32).ravel()
                assert np.array_equal(ws["ranges"], rng), n
            bd.close()
        # the wrapping luma sum through k_preview_stats
        ref.set_preview_mode(1); ref.set_ycc_offset(0, 0, 0, 0, 0)
        ref.config_histo(True, False, False)
        j = white()[0]
        w = ref.decode(j)
        dec = CimgDecode(); dec.config_histo(True, False, False)
        g = dec.decode(j)
        assert np.array_equal(np.asarray(w.stats), np.asarray(g.stats)), (w.stats, g.stats)
        assert g.stats[0] == 0 and expected(WHITE, True)[1][0] == 0
        gs, ws = dec.colour_stats(), ref.colour_stats()
        for k in ("clip", "ranges", "cc_histo", "y_histo"):
            assert np.array_equal(ws[k], gs[k]), k
        dec.close()
        bd = BatchDecoder()
        bd.set_preview(hist_en=1)
        bd.set_batch([j]); bd.decode(); bd.sync()
        assert np.array_equal(CJ.device_stats(bd.fetch(0).stats), np.asarray(w.stats)[:10]), bd.fetch(0).stats
        bd.close()
    finally:
        ref.set_preview_mode(1); ref.set_ycc_offset(0, 0, 0, 0, 0)
        ref.config_histo(False, False, False); ref.close()
