"""TEST INFRASTRUCTURE: greyscale baseline files in which chosen bytes land at chosen raw scan offsets.

Stage A of the decoder (marker scan, unstuffing, and the map from unstuffed bit positions back to file positions) works on
fixed byte grids: 4-byte words, 16-byte loads and pieces, 64-byte thread spans, 128-byte rows, 512-byte warp rows, 4096-byte
chunks, 32 KB passes.  Natural content puts an RST marker or a stuffed FF 00 pair on a grid edge only by chance; this writer
puts them there on purpose.

The file is built from restart intervals of `dri` 8x8 blocks.  Its length is steered by the coefficients:
* a filler interval of exactly L raw bytes holds no 0xFF byte (a DC difference of size 0..5 gives one-bit control, AC values
  of sizes 1..13 at zig-zag positions 1.. make up the rest, so the interval needs no pad bits);
* a stuffed pair is an AC value of +32767 (size 15): its fifteen one-bits after the code cover at least one whole byte, and
  the filler coefficients in front of it move that byte onto the wanted unstuffed index;
* an RST marker lands at offset t when the intervals before it add up to t bytes.
The coefficients go through coef_jpeg.encode_coefs, so coef_jpeg.expected is the reference decode of every healthy file.

Offsets count from the first byte after the SOS segment.  The record returned with a file (`Placed`) lists every RST, every
stuffed pair, every MCU start (interval, unstuffed bit) and every spliced byte string as they are in the bytes; the tests
recompute the boundaries they care about from the bytes themselves."""
import numpy as np

import coef_jpeg as CJ
from mini_jpeg import ZZ, BitWriter, canonical_codes

DC = canonical_codes(*CJ.dc_table(True))
AC = canonical_codes(*CJ.ac_table(True, 0))
Q1 = np.ones(64, np.int64)
MAX_FILL = 150                                   # longest filler interval (bytes); a block of 63 size-13 values is ~180


def _val_bits(a, s):
    return (a if a > 0 else a + (1 << s) - 1) & ((1 << s) - 1)


def _low_ones(s, k=0):
    """A negative value of size s whose bits are 0 1 0 1 ... (k odd: 0 0 1 1 0 0 ...): short runs of ones, no 0xFF byte."""
    pat = ("01" * 8) if k % 2 == 0 else ("0011" * 4)
    return int(pat[:s], 2) - ((1 << s) - 1)


def block_items(zz):
    """(code, length) items of one block, zz = 64 values in zig-zag order, zz[0] = the DC difference."""
    out = []
    d = int(zz[0]); s = abs(d).bit_length()
    code, n = DC[s]; out.append(((code << s) | _val_bits(d, s), n + s))
    nz = [p for p in range(1, 64) if zz[p]]
    k = 1
    for p in nz:
        run = p - k
        while run > 15:
            out.append(AC[0xF0]); run -= 16
        a = int(zz[p]); s = abs(a).bit_length()
        code, n = AC[(run << 4) | s]; out.append(((code << s) | _val_bits(a, s), n + s))
        k = p + 1
    if k < 64:
        out.append(AC[0x00])
    return out


def interval_bytes(blocks):
    bw = BitWriter()
    for zz in blocks:
        for c, n in block_items(zz):
            bw.put(c, n)
    bw.flush()
    return bytes(bw.out)


def _bits(zz):
    return sum(n for _, n in block_items(zz))


_DC_SIZES = [(s, DC[s][1] + s) for s in range(0, 6)]                   # DC size -> bits: 2, 4, 5, 6, 7, 8
_AC_COST = {s: AC[s][1] + s for s in range(1, 14)}                      # run 0, size s -> bits


def _ways(limit=1600):
    """way[r]: AC sizes (run 0) whose codes and values add up to exactly r bits, fewest values first."""
    way = {0: []}
    for r in range(1, limit):
        best = None
        for sz, c in _AC_COST.items():
            if r - c in way and (best is None or len(way[r - c]) + 1 < len(best)):
                best = way[r - c] + [sz]
        if best is not None:
            way[r] = best
    return way


_WAY = _ways()


def _fill_zz(nbits, k=0):
    """zig-zag values of one block whose code is exactly nbits long, or None."""
    for ds, db in _DC_SIZES[::-1] if k % 2 else _DC_SIZES:
        for eob in (2, 0):
            sizes = _WAY.get(nbits - db - eob)
            if sizes is not None and len(sizes) <= 63 and (len(sizes) == 63) == (eob == 0):
                zz = np.zeros(64, np.int64)
                zz[0] = _low_ones(ds, k) if ds else 0
                for p, sz in enumerate(sizes, 1):
                    zz[p] = _low_ones(sz, k + p)
                return zz
    return None


def filler(L, nblk, k=0):
    """nblk blocks (zig-zag) whose interval is exactly L raw bytes with no 0xFF in it."""
    rest = [np.zeros(64, np.int64) for _ in range(nblk - 1)]            # DC 0 + EOB: 4 bits each
    need = 8 * L - 4 * (nblk - 1)
    for kk in range(k, k + 40):
        z = _fill_zz(need, kk)
        if z is None:
            break
        bl = [z] + rest
        b = interval_bytes(bl)
        if len(b) == L and 0xFF not in b:
            return bl
    raise ValueError(f"no filler interval of {L} bytes with {nblk} blocks")


def with_pairs(us, nblk):
    """Blocks of one interval whose unstuffed bytes us[0] < us[1] < ... are 0xFF (each then stuffed) and no other byte is:
    a +32767 (size 15) per pair, filler values in front of it moving its first whole byte of ones onto u."""
    zz = np.zeros(64, np.int64); p = 1; bits = 2                         # DC difference 0
    cl = AC[0x0F][1]
    for i, u in enumerate(us):
        tries = [(start, alt) for start in range(8 * u, 8 * u - 8, -1) for alt in (0, 1)]   # value bits from `start`: byte u is all ones
        for start, alt in tries:
            gap = start - cl - bits
            lead = [1] if i else []                                       # behind a run of ones: a code that starts with 0
            if gap - 4 * len(lead) not in _WAY or p + len(lead) + len(_WAY[gap - 4 * len(lead)]) >= 63:
                continue
            t = zz.copy(); q = p
            for sz in lead + sorted(_WAY[gap - 4 * len(lead)]):
                t[q] = _low_ones(sz, q + alt); q += 1
            t[q] = 32767; q += 1
            b = interval_bytes([t])
            ff = [j for j in range(len(b)) if b[j] == 0xFF]
            want = [uu + n for n, uu in enumerate(us[:i + 1])]           # raw offsets: one stuffed zero behind each earlier FF
            if ff == want:
                zz, p, bits = t, q, start + 15
                break
        else:
            raise ValueError(f"cannot put a lone stuffed pair at unstuffed byte {u}")
    return [zz] + [np.zeros(64, np.int64) for _ in range(nblk - 1)]


def dense_pairs(n, nblk):
    """One interval of n consecutive +32767 values: runs of adjacent pairs FF 00 FF 00 ..."""
    zz = np.zeros(64, np.int64); zz[1:1 + n] = 32767
    return [zz] + [np.zeros(64, np.int64) for _ in range(nblk - 1)]


def _ffs(out, lo=0):
    return [j for j in range(max(0, lo), len(out)) if out[j] == 0xFF]


def _clone(bw):
    c = BitWriter(); c.out = bytearray(bw.out); c.acc = bw.acc; c.n = bw.n
    return c


def long_interval(targets, nblk, length):
    """Blocks of one interval of exactly `length` raw bytes, spread over nblk blocks, whose 0xFF bytes are exactly the raw
    offsets in `targets` (increasing, at least 6 apart; each then stuffed).  For intervals longer than one block can carry:
    the long intervals of the self-synchronising path, thousands of bytes each."""
    blocks, zz, p = [], np.zeros(64, np.int64), 1
    bw = BitWriter(); bw.put(*DC[0]); bits = DC[0][1]; after_pair = False
    cl = AC[0x0F][1]

    def close():                                   # EOB, next block with a DC difference of 0
        nonlocal zz, p, bits
        bw.put(*AC[0x00]); bits += 2
        blocks.append(zz); zz, p = np.zeros(64, np.int64), 1
        bw.put(*DC[0]); bits += DC[0][1]

    def put_val(v):
        nonlocal p, bits
        s = abs(int(v)).bit_length(); code, n = AC[s]
        bw.put((code << s) | _val_bits(int(v), s), n + s); zz[p] = v; p += 1; bits += n + s

    def fill_to(goal, then_pair):
        """filler values until the next item starts at unstuffed bit goal(); True when it worked without a stray 0xFF"""
        nonlocal bw, zz, p, bits, after_pair
        while True:
            gap = goal() - bits
            lead = [1] if after_pair else []
            rest = gap - 4 * len(lead)
            if rest in _WAY and p + len(lead) + len(_WAY[rest]) + (1 if then_pair else 0) < 63 and rest < 700:
                break
            if gap < 700 + 64 and p + 40 >= 63 or p >= 60:
                if gap < 8:
                    return False
                close(); after_pair = False
                continue
            if gap < 60:
                return False
            # a big filler value, its pattern chosen so that no 0xFF appears
            for alt in (0, 1, 2, 3):
                save = (_clone(bw), zz.copy(), p, bits)
                lo = len(bw.out)
                for sz in lead + [13]:
                    put_val(_low_ones(sz, p + alt))
                if not _ffs(bw.out, lo):
                    break
                bw, zz, p, bits = save
            else:
                return False
            after_pair = False
        for alt in (0, 1):
            save = (_clone(bw), zz.copy(), p, bits)
            lo = len(bw.out)
            for sz in lead + sorted(_WAY[rest]):
                put_val(_low_ones(sz, p + alt))
            if not _ffs(bw.out, lo):
                after_pair = False
                return True
            bw, zz, p, bits = save
        return False

    for i, t in enumerate(targets):
        u = t - i                                              # unstuffed index: one stuffed zero behind each earlier FF
        for start in range(8 * u, 8 * u - 8, -1):
            save = (_clone(bw), zz.copy(), p, bits, list(blocks), after_pair)
            if fill_to(lambda: start - cl, True):
                lo = len(bw.out)
                put_val(32767)
                if _ffs(bw.out, lo - 1) == [t]:
                    after_pair = True
                    break
            bw, zz, p, bits, blocks, after_pair = save
        else:
            raise ValueError(f"cannot put a stuffed pair at raw offset {t}")
    # the tail: exactly `length` bytes, then DC-only blocks up to nblk
    nstuff = len(targets)
    goal = lambda: 8 * (length - nstuff) - 2 - 4 * (nblk - len(blocks) - 1)     # EOB, then DC-only blocks of 4 bits
    if not (fill_to(goal, False) and bits == goal()):
        raise ValueError("cannot end the interval at the wanted length")
    blocks.append(zz)
    blocks += [np.zeros(64, np.int64) for _ in range(nblk - len(blocks))]
    assert len(blocks) == nblk, (len(blocks), nblk)
    b = interval_bytes(blocks)
    assert len(b) == length and _ffs(b) == list(targets), (len(b), length, _ffs(b)[:8], targets[:8])
    return blocks


class Placed:
    """What a writer put where (scan offsets).  rst: FF offsets of the RST markers; pairs: offsets of the FF of every stuffed
    pair; intervals: (start, end) raw bounds; splices: (offset, bytes) inserted after encoding; nrst: RSTs of the healthy scan;
    mcu_bits: per interval, (unstuffed start bit of each MCU, bits of the interval's data)."""
    def __init__(self):
        self.rst, self.pairs, self.intervals, self.splices, self.mcu_bits = [], [], [], [], []
        self.scan_start = 0; self.nrst = 0


class Writer:
    """Greyscale baseline file, DRI = dri, one 8-pixel-high MCU row (or more when the interval count asks for it)."""
    def __init__(self, dri=1):
        self.dri = dri; self.iv = []; self.pos = 0

    def add(self, blocks):
        b = interval_bytes(blocks)
        self.iv.append(blocks)
        self.pos += len(b) + 2                    # + the RST marker behind it (the last one becomes EOI)
        return len(b)

    def advance_to(self, x):
        """Filler intervals until the next interval starts at raw offset x (x - pos must be 0 or >= 3 per interval)."""
        g = x - self.pos
        if g == 0:
            return
        assert g >= 3, (x, self.pos)
        n = -(-g // (MAX_FILL + 2))
        while g - 2 * n < n * max(1, (4 * self.dri + 7) // 8):
            n -= 1
        assert n >= 1, g
        base, extra = divmod(g - 2 * n, n)
        for i in range(n):
            self.add(filler(base + (i < extra), self.dri, k=len(self.iv)))

    def rst_at(self, t):
        """The next RST marker's FF at offset t: one interval ends there."""
        lo = max(1, (4 * self.dri + 7) // 8)
        if t - self.pos < lo:
            raise ValueError((t, self.pos))
        if t - self.pos > MAX_FILL:
            self.advance_to(t - min(MAX_FILL, 40 + (t - self.pos) % 40))
        self.add(filler(t - self.pos, self.dri, k=len(self.iv)))

    def pairs_at(self, ts, slack=24):
        """Stuffed pairs whose FF is at each offset in ts (one interval; ts increasing, at least 2 bytes apart)."""
        start = ts[0] - slack
        self.advance_to(start)
        us, shift = [], 0
        for t in ts:
            us.append(t - start - shift); shift += 1
        self.add(with_pairs(us, self.dri))

    def finish(self, min_mcus=0, width_mcus=None):
        """(jpeg bytes, coef_jpeg spec, Placed).  Adds DC-only intervals to fill the last MCU row."""
        nmcu = max(len(self.iv) * self.dri, min_mcus)
        wm = width_mcus or min(nmcu, 4096)
        rows = -(-nmcu // wm)
        while len(self.iv) * self.dri < wm * rows:
            self.iv.append([np.zeros(64, np.int64)] * self.dri)
        zz_all = [z for blocks in self.iv for z in blocks][: wm * rows]
        # coefficients in natural order, absolute DC (the predictor restarts at every interval)
        nat = np.zeros((rows, wm, 64), np.int64)
        for i, z in enumerate(zz_all):
            v = np.zeros(64, np.int64); v[ZZ] = z
            dc = int(z[0]) if i % self.dri == 0 else int(nat.reshape(-1, 64)[i - 1][0]) + int(z[0])
            v[0] = dc
            nat[i // wm, i % wm] = v
        j, spec = CJ.encode_coefs([nat], 8 * wm, 8 * rows, ((1, 1),), [Q1], [0], dri=self.dri)
        rec = Placed()
        s = j.index(b"\xff\xda"); rec.scan_start = s + 2 + int.from_bytes(j[s + 2:s + 4], "big")
        scan = j[rec.scan_start:]
        rec.rst = [i for i in range(len(scan) - 1) if scan[i] == 0xFF and 0xD0 <= scan[i + 1] <= 0xD7]
        rec.pairs = [i for i in range(len(scan) - 1) if scan[i] == 0xFF and scan[i + 1] == 0]
        bounds = [-2] + rec.rst + [len(scan) - 2]
        rec.intervals = [(a + 2, b) for a, b in zip(bounds[:-1], bounds[1:])]
        rec.nrst = len(rec.rst)
        # unstuffed start bit of every MCU inside its interval (MCU = one block)
        rec.mcu_bits = []
        for blocks in self.iv:
            b, starts = 0, []
            for zz in blocks:
                starts.append(b); b += _bits(zz)
            rec.mcu_bits.append((starts, b))
        rec.mcu_bits = rec.mcu_bits[:len(rec.intervals)]
        return j, spec, rec


def splice(j, rec, t, data):
    """Insert `data` at scan offset t (after encoding): a terminator, a stray marker or fill bytes.  Returns (bytes, Placed)."""
    import copy
    r = copy.deepcopy(rec)
    p = rec.scan_start + t
    out = j[:p] + bytes(data) + j[p:]
    scan = out[r.scan_start:]
    r.rst = [i for i in range(len(scan) - 1) if scan[i] == 0xFF and 0xD0 <= scan[i + 1] <= 0xD7]
    r.pairs = [i for i in range(len(scan) - 1) if scan[i] == 0xFF and scan[i + 1] == 0]
    r.splices = rec.splices + [(t, bytes(data))]
    return out, r
