"""TEST INFRASTRUCTURE: a coefficient-level JPEG writer and a plain numpy restatement of what the reference decoder
computes from such a file, with every fixed-width wrap written out.

`encode_coefs` writes baseline (SOF0) or extended (SOF1, P = 12) files from given quantised coefficients, with any
quantiser 1..65535 (16-bit DQT entries where needed), DC and AC sizes up to 15 and optional 16-bit codes for the largest
sizes, so that a code plus its value bits is a 30-31-bit step.  Neither Pillow nor tests/mini_jpeg.py can write these.

`expected` is the decode of such a file by the reference's arithmetic (ImgDecode.cpp ReadScanVal, DecodeIdctSet,
DecodeIdctCalcFixedpt / DecodeIdctCalcFloat, SetFullRes, ConvertYCCtoRGBFastFloat, the block-DC maps) for every layout
whose components each have a sampling factor of 1 or the maximum in each direction (4:4:4, 4:2:2, 4:2:0, 4:1:1, 4:4:0,
2x4 + 2x1, 4x3 + 1x3 ... and greyscale): there no two blocks of a component overlap.  It uses the IDCT tables the oracle
hands out, nothing else from the reference.  `expected_stats` restates the brightest-pixel and average-luma statistics
CalcChannelPreviewFull derives from those maps."""
import numpy as np

from mini_jpeg import ZZ, BitWriter, bits_from_lengths, canonical_codes, _seg


# --- Huffman tables --------------------------------------------------------------------------------------------------

# DC symbols with a run nibble: (r << 4) | s carries a size-s value that lands at zig-zag position r (ImgDecode.cpp
# DecodeIdctSet stores it at num_coeffs + zrl); the block goes on at 1 + r and its DC difference is 0.
DC_RUN_SYMBOLS = [(r << 4) | (r * 7 % 15 + 1) for r in range(1, 16)]


def dc_table(long_codes=True, runs=False):
    """DC sizes 0..15; with long_codes the sizes 14 and 15 have 16-bit codes (a 16 + 15 = 31-bit step).  runs adds the
    DC_RUN_SYMBOLS behind 14-bit codes."""
    extra = DC_RUN_SYMBOLS if runs else []
    lengths = [2, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9, 12, 12] + [14] * len(extra) + ([16, 16] if long_codes else [13, 13])
    return bits_from_lengths(lengths), list(range(14)) + extra + [14, 15]


def ac_table(long_codes=True, variant=0):
    """Every run/size symbol with sizes 1..15, EOB and ZRL.  Sizes 14 and 15 sit behind 16-bit codes with long_codes
    (one 10-bit prefix: the second-level look-up stays small enough for the lane kernel's shared-memory copy).
    variant 1 swaps the two shortest codes, so that luma and chroma tables differ."""
    short = [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x21, 0x05, 0x12, 0x31]
    if variant:
        short[0], short[1] = short[1], short[0]
    short_len = [2, 3, 3, 4, 4, 5, 5, 6, 6, 6]
    rest = [0xF0] + [(r << 4) | s for s in range(1, 14) for r in range(16)]
    rest = [s for s in rest if s not in short]
    big = [(r << 4) | s for s in (14, 15) for r in range(16)]
    syms = short + rest + big
    lengths = short_len + [10] * len(rest) + [16 if long_codes else 13] * len(big)
    return bits_from_lengths(lengths), syms


# --- writer ----------------------------------------------------------------------------------------------------------

def _geometry(W, H, samp):
    hmax = max(h for h, v in samp); vmax = max(v for h, v in samp)
    mcu_w, mcu_h = 8 * hmax, 8 * vmax
    return hmax, vmax, (W + mcu_w - 1) // mcu_w, (H + mcu_h - 1) // mcu_h


def block_shape(W, H, samp, c):
    """(block rows, block cols) of component c: what `blocks[c]` must be shaped as (plus the trailing 64)."""
    _, _, mx, my = _geometry(W, H, samp)
    h, v = samp[c]
    return my * v, mx * h


def _mcu_order(W, H, samp):
    """Blocks in scan order: list over MCUs of [(component, block row, block col)], the reference's loop nest."""
    _, _, mxn, myn = _geometry(W, H, samp)
    order = []
    for my in range(myn):
        for mx in range(mxn):
            order.append([(c, my * v + by, mx * h + bx) for c, (h, v) in enumerate(samp) for by in range(v) for bx in range(h)])
    return order


def encode_coefs(blocks, W, H, samp, qtabs, qsel, precision=8, dri=0, long_codes=True, force_pq16=False,
                 shared_tables=False, dc_runs=None, trace=None):
    """A JPEG whose scan carries exactly these coefficients.

    blocks: one int array per component, (block rows, block cols, 64) in natural order, holding the values as written
            into the bitstream (for P = 12 the reference divides them by 16 when it reads them).  DC is the absolute
            value; the writer codes differences, reset at each restart, like any encoder.
    samp:   (H, V) per component (one entry = greyscale).
    qtabs:  quantisation tables, 64 values 1..65535 in natural order; a table is written with Pq = 1 when an entry
            exceeds 255 or force_pq16 is set.  qsel: table index per component.
    shared_tables: every component uses DC/AC table 0 (else luma 0, chroma 1).
    dc_runs: per component, block-grid shaped run nibbles r (0..15): a block with r > 0 writes its zig-zag value r with the
            DC symbol (r << 4) | size (the DC table then holds DC_RUN_SYMBOLS); its DC must equal the previous block's and
            its zig-zag values 1 .. r-1 must be 0.  `expected` does not model this.
    trace:  a list that receives, per restart interval, a dict of the unstuffed bit position of every MCU start
            ("mcu_bits") and block start ("blk_bits", per MCU), the reference's int16 DC predictors at every MCU start
            ("dc", per MCU one value per component) and the interval's unstuffed length in bits ("nbits", before padding).
    Returns (jpeg bytes, spec): spec is what `expected` needs."""
    ncomp = len(samp)
    assert ncomp in (1, 3) and precision in (8, 12)
    if ncomp == 1:
        assert tuple(samp[0]) == (1, 1)
    blocks = [np.asarray(b, np.int64) for b in blocks]
    for c in range(ncomp):
        assert blocks[c].shape == block_shape(W, H, samp, c) + (64,), (c, blocks[c].shape)
        assert np.all(np.abs(blocks[c][..., 1:]) <= 32767)
    qtabs = [np.asarray(q, np.int64) for q in qtabs]
    for q in qtabs:
        assert q.shape == (64,) and q.min() >= 1 and q.max() <= 65535
    ntab = 1 if (ncomp == 1 or shared_tables) else 2
    dc_tabs = [dc_table(long_codes, runs=dc_runs is not None)] * ntab
    ac_tabs = [ac_table(long_codes, variant=t) for t in range(ntab)]
    dcc = [canonical_codes(*t) for t in dc_tabs]; acc = [canonical_codes(*t) for t in ac_tabs]
    zz = [b[..., ZZ] for b in blocks]                         # zig-zag order, so a block's symbols are a left-to-right walk
    bw = BitWriter(); out = bytearray(); pred = [0] * ncomp; rst = 0
    div = 1 << (precision - 8)
    cdiv = lambda a: -(-a // div) if a < 0 else a // div
    i16 = lambda a: ((a + 32768) & 0xFFFF) - 32768
    nbits = [0]; dcp = [0] * ncomp                          # bits of the current interval; the reference's short predictors
    new_iv = lambda: {"mcu_bits": [], "blk_bits": [], "dc": [], "nbits": 0}
    cur = new_iv()

    def put(code, length):
        bw.put(code, length); nbits[0] += length

    def put_val(code_len, a, s):
        code, length = code_len
        put((code << s) | ((a if a > 0 else a + (1 << s) - 1) & ((1 << s) - 1)), length + s)

    for n, mcu in enumerate(_mcu_order(W, H, samp)):
        if dri and n and n % dri == 0:
            cur["nbits"] = nbits[0]
            if trace is not None:
                trace.append(cur)
            bw.flush(); out += bw.out; out += bytes([0xFF, 0xD0 + (rst & 7)]); rst += 1
            bw = BitWriter(); pred = [0] * ncomp; nbits[0] = 0; dcp = [0] * ncomp; cur = new_iv()
        cur["mcu_bits"].append(nbits[0]); cur["blk_bits"].append([]); cur["dc"].append(list(dcp))
        for c, br, bc in mcu:
            cur["blk_bits"][-1].append(nbits[0])
            t = 0 if (c == 0 or shared_tables) else 1
            z = zz[c][br, bc]
            diff = int(z[0]) - pred[c]; pred[c] = int(z[0])
            assert abs(diff) <= 32767, ("DC difference needs more than 15 bits", c, br, bc, diff)
            r = int(dc_runs[c][br, bc]) if dc_runs is not None else 0
            k = 1
            if r:
                assert diff == 0 and not z[1:r].any() and z[r], ("a DC run symbol needs DC difference 0 and zig-zag values", c, br, bc)
                a = int(z[r]); s = abs(a).bit_length()
                assert (r << 4) | s in dcc[t], ("no DC run symbol", hex((r << 4) | s))
                put_val(dcc[t][(r << 4) | s], a, s)
                k = r + 1
            else:
                s = abs(diff).bit_length()
                put_val(dcc[t][s], diff, s)
                dcp[c] = i16(dcp[c] + i16(cdiv(diff) * int(qtabs[qsel[c]][0])))
            nz = np.flatnonzero(z[k:]) + k
            for p in nz.tolist():
                run = p - k
                while run > 15:
                    put(*acc[t][0xF0]); run -= 16
                a = int(z[p]); s = abs(a).bit_length()
                put_val(acc[t][(run << 4) | s], a, s)
                k = p + 1
            if k < 64:
                put(*acc[t][0x00])
    cur["nbits"] = nbits[0]
    if trace is not None:
        trace.append(cur)
    bw.flush(); out += bw.out
    f = bytearray(b"\xFF\xD8")
    for i, q in enumerate(qtabs):
        pq = 1 if (force_pq16 or q.max() > 255) else 0
        body = b"".join(int(v).to_bytes(2 if pq else 1, "big") for v in q[ZZ])
        f += _seg(0xDB, bytes([(pq << 4) | i]) + body)
    f += _seg(0xC1 if precision != 8 else 0xC0, bytes([precision]) + H.to_bytes(2, "big") + W.to_bytes(2, "big") + bytes([ncomp]) +
              b"".join(bytes([c + 1, (samp[c][0] << 4) | samp[c][1], qsel[c]]) for c in range(ncomp)))
    for i in range(ntab):
        f += _seg(0xC4, bytes([0x00 | i]) + bytes(dc_tabs[i][0]) + bytes(dc_tabs[i][1]))
        f += _seg(0xC4, bytes([0x10 | i]) + bytes(ac_tabs[i][0]) + bytes(ac_tabs[i][1]))
    if dri:
        f += _seg(0xDD, dri.to_bytes(2, "big"))
    f += _seg(0xDA, bytes([ncomp]) + b"".join(bytes([c + 1, 0x00 if (c == 0 or shared_tables) else 0x11]) for c in range(ncomp)) + bytes([0, 63, 0]))
    spec = dict(blocks=blocks, W=W, H=H, samp=tuple(tuple(s) for s in samp), qtabs=qtabs, qsel=tuple(qsel), precision=precision, dri=dri)
    return bytes(f + out + b"\xFF\xD9"), spec


# --- the reference's arithmetic, restated --------------------------------------------------------------------------

def _i16(x):
    """C conversion to short of an integer value: the low 16 bits, two's complement."""
    return ((np.asarray(x, np.int64) + 32768) & 0xFFFF) - 32768


def _i32(x):
    return ((np.asarray(x, np.int64) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def _cdiv(a, d):
    """C integer division (truncates toward zero)."""
    a = np.asarray(a, np.int64)
    return np.sign(a) * (np.abs(a) // d)


def _idct_fixed(coef, li):
    """DecodeIdctCalcFixedpt: s = sum over vu >= 1 of Li[yx][vu] * c[vu] in int, C `/4`, then `>>10`.
    |Li| <= 1024 and |c| <= 32768, so the float64 product sum is exact; the int wrap is applied explicitly."""
    s = np.rint(coef[:, 1:].astype(np.float64) @ li[:, 1:].T.astype(np.float64)).astype(np.int64)
    return _cdiv(_i32(s), 4) >> 10


def _idct_float(coef, lf):
    """DecodeIdctCalcFloat: one fp32 multiply and one fp32 add per term, in natural index order, then * 0.25.
    A term whose coefficient is zero in every block adds +-0 to a sum that is never -0: skipping it is exact."""
    s = np.zeros((coef.shape[0], 64), np.float32)
    cf = coef.astype(np.float32)
    for vu in range(1, 64):
        if not cf[:, vu].any():
            continue
        s = s + lf[:, vu][None, :] * cf[:, vu][:, None]
    return s * np.float32(0.25)


def _f2i_trunc(f):
    """x86 cvttss2si: float -> int32 truncating (0x80000000 when out of range)."""
    f = np.asarray(f, np.float64)
    ok = np.abs(f) < 2.0 ** 31
    return np.where(ok, np.trunc(np.where(ok, f, 0)), -(2 ** 31)).astype(np.int64)


def ycc_to_bgra(py, pcb, pcr):
    """ConvertYCCtoRGBFastFloat (ImgDecode.cpp:4086-4139) over whole maps: float32, one rounding per operation."""
    f32 = np.float32
    y = np.clip(np.asarray(py, np.int64) >> 3, -128, 127)
    cb = np.clip(np.asarray(pcb, np.int64) >> 3, -128, 127)
    cr = np.clip(np.asarray(pcr, np.int64) >> 3, -128, 127)
    cR, cG, cB = f32(0.299), f32(0.587), f32(0.114)
    kR = f32(2) - f32(2) * cR; kB = f32(2) - f32(2) * cB
    fy = y.astype(f32)
    vr = cr.astype(f32) * kR + fy
    vb = cb.astype(f32) * kB + fy
    vg = (fy - cB * vb - cR * vr) / cG
    vr = vr + f32(128); vb = vb + f32(128); vg = vg + f32(128)
    to8 = lambda v: np.where(v < 0, 0, np.where(v > 255, 255, np.trunc(np.clip(v, 0, 255)))).astype(np.uint8)
    return np.stack([to8(vb), to8(vg), to8(vr), np.zeros(y.shape, np.uint8)], -1)


class Expected:
    """What the reference leaves behind for a file from `encode_coefs`: the fields JC.compare reads."""
    def __init__(self):
        self.geom = self.pix_y = self.pix_cb = self.pix_cr = self.dib = self.blk_dc = None


def expected(spec, idct_fixed, li, lf, decode_ac=True):
    """The reference's decode of `spec` (from encode_coefs): Y/Cb/Cr pixel maps, the bottom-up BGRA DIB, the block-DC maps.
    li / lf: the IDCT tables, from Oracle.idct_tables() or CimgDecode.idct_tables()."""
    W, H, samp, P, dri = spec["W"], spec["H"], spec["samp"], spec["precision"], spec["dri"]
    ncomp = len(samp)
    hmax, vmax, mxn, myn = _geometry(W, H, samp)
    mcu_w, mcu_h = 8 * hmax, 8 * vmax
    img_x, img_y = mxn * mcu_w, myn * mcu_h
    blk_xmax, blk_ymax = mxn * hmax, myn * vmax
    for h, v in samp:
        assert h in (1, hmax) and v in (1, vmax), "expected() covers layouts whose factors are 1 or the maximum only"
    div = 1 << (P - 8)
    e = Expected()
    e.geom = np.array([mcu_w, mcu_h, mxn, myn, blk_xmax, blk_ymax, img_x, img_y], np.uint32)
    maps, dcmaps = [], []
    for c in range(ncomp):
        h, v = samp[c]
        blk = spec["blocks"][c]
        q = spec["qtabs"][spec["qsel"][c]]
        R, Cn = blk.shape[:2]
        # ReadScanVal: value / (1 << (P-8)), C division.  DecodeIdctSet: (short)(val * q).
        val = _cdiv(blk, div) if div > 1 else blk.copy()
        # DC: the written differences in scan order (reset at each restart), divided and dequantised one by one; the running
        # predictor is a short.  Blocks of component c in scan order: MCU-major, then (by, bx) inside the MCU.
        mcu_r = np.arange(R)[:, None] // v; mcu_c = np.arange(Cn)[None, :] // h
        mcu_idx = (mcu_r * mxn + mcu_c)
        inner = (np.arange(R)[:, None] % v) * h + (np.arange(Cn)[None, :] % h)
        order = np.lexsort((inner.ravel(), mcu_idx.ravel()))     # scan order of the flat (R*Cn) blocks
        dc_written = blk[..., 0].ravel()[order]
        seg = (mcu_idx.ravel()[order] // dri) if dri else np.zeros(order.size, np.int64)
        prev = np.concatenate([[0], dc_written[:-1]])
        first = np.concatenate([[True], seg[1:] != seg[:-1]])
        diff = np.where(first, dc_written, dc_written - prev)
        dval = _cdiv(diff, div) if div > 1 else diff
        ddq = _i16(dval * int(q[0]))
        cs = np.cumsum(ddq)
        start = np.maximum.accumulate(np.where(first, np.arange(order.size), 0))
        base = np.concatenate([[0], cs[:-1]])[start]
        dc_run = _i16(cs - base)                                   # (short)(dc + d) each step == the sum modulo 2^16
        dc_blk = np.empty(order.size, np.int64); dc_blk[order] = dc_run
        dc_blk = dc_blk.reshape(R, Cn)
        # AC: (short)(val * q) at the natural index, then the IDCT over the 63 AC terms; DC enters as the level shift
        coef = _i16(val.reshape(-1, 64) * q[None, :])
        coef[:, 0] = 0
        if not decode_ac:
            n8 = np.zeros((R * Cn, 64), np.int64)
        elif idct_fixed:
            n8 = _i16(_idct_fixed(coef, li)) * 8                  # nv = (short)iidct; nv = (short)(nv*8 + dcoff)
        else:
            n8 = _i16(_f2i_trunc(_idct_float(coef, lf) * np.float32(8)))    # (short)(f*8), then + dcoff
        pix = _i16(n8.reshape(R, Cn, 8, 8) + dc_blk[:, :, None, None]).astype(np.int16)
        # SetFullRes: block (r, c) covers rows r*8*ev.. and columns c*8*eh.., each sample replicated ev x eh
        eh, ev = hmax // h, vmax // v
        plane = pix.transpose(0, 2, 1, 3).reshape(R * 8, Cn * 8)
        maps.append(np.repeat(np.repeat(plane, ev, 0), eh, 1))
        # block-DC maps (ImgDecode.cpp:3524-3608): luma cell = (my*ev + v)*blk_xmax + mx*eh + h with Y's expand factors,
        # chroma cell = (my*ev + v)*blk_xmax + (mx*eh + h); in MCU order, later writes win, cells past the end are dropped
        nb = blk_xmax * blk_ymax
        my_, mx_ = np.divmod(np.arange(mxn * myn), mxn)
        cells, seqs, vals = [], [], []
        for by in range(v):
            for bx in range(h):
                cells.append((my_ * ev + by) * blk_xmax + mx_ * eh + bx)
                seqs.append((my_ * mxn + mx_) * 16 + by * 4 + bx)
                vals.append(dc_blk[my_ * v + by, mx_ * h + bx])
        cells = np.concatenate(cells); seqs = np.concatenate(seqs); vals = np.concatenate(vals)
        keep = cells < nb
        cells, seqs, vals = cells[keep], seqs[keep], vals[keep]
        o = np.argsort(seqs, kind="stable")[::-1]
        u, firsts = np.unique(cells[o], return_index=True)
        m = np.zeros(nb, np.int16); m[u] = vals[o][firsts]
        dcmaps.append(m)
    e.pix_y = maps[0]
    if ncomp == 3:
        e.pix_cb, e.pix_cr = maps[1], maps[2]
        e.blk_dc = (dcmaps[0], dcmaps[1], dcmaps[2])
        e.dib = ycc_to_bgra(maps[0], maps[1], maps[2])[::-1].copy()
    else:
        z = np.zeros_like(maps[0])
        e.blk_dc = (dcmaps[0], None, None)
        e.dib = ycc_to_bgra(maps[0], z, z)[::-1].copy()
    return e


def expected_stats(e):
    """The reference's stats[0:10] (avgY, avgY valid, brightest Y, Cb, Cr, R, G, B, its MCU x, y) for an `expected` result:
    CalcChannelPreviewFull (ImgDecode.cpp:4693-4730, 4813-4819) walks the padded maps in raster order and keeps the first
    strict maximum of raw Y, starting from -32768, so an image whose Y is -32768 everywhere keeps the initial values at pixel 0;
    the luma sum is a 32-bit unsigned and the divisor is (Wp + 1)(Hp + 1)."""
    mcu_w, mcu_h, Wp, Hp = int(e.geom[0]), int(e.geom[1]), int(e.geom[6]), int(e.geom[7])
    y = np.asarray(e.pix_y, np.int64).ravel()
    idx = int(np.argmax(y))
    if y[idx] == -32768:
        by = bcb = bcr = -32768; idx = 0
    else:
        by = int(y[idx])
        bcb = int(np.asarray(e.pix_cb).ravel()[idx]) if e.pix_cb is not None else 0
        bcr = int(np.asarray(e.pix_cr).ravel()[idx]) if e.pix_cr is not None else 0
    b, g, r, _ = (int(v) for v in ycc_to_bgra(by, bcb, bcr))
    s = int((np.clip(y >> 3, -128, 127) + 128).sum()) & 0xFFFFFFFF
    avg = s // ((Wp + 1) * (Hp + 1))
    return np.array([avg, 1, by, bcb, bcr, r, g, b, (idx % Wp) // mcu_w, (idx // Wp) // mcu_h], np.int32)


def device_stats(st):
    """The reference's stats[0:10] layout from the device's 16-word stats row (include/jsgpu.h: [2] m_nAvgY, [3:11] the
    brightest pixel's Y, Cb, Cr, R, G, B and its MCU x, y); the valid flag is set by every decode."""
    st = np.asarray(st, np.int64)
    return np.concatenate([[st[2], 1], st[3:11]]).astype(np.int32)
