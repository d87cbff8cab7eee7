"""TEST INFRASTRUCTURE: coefficient-level files whose MCU starts, block starts and chosen symbols land on given bit offsets of
a restart interval.

The self-synchronising Huffman passes (jpegsnoop_b200/csrc/jsgpu_phuff_core.cuh) cut the unstuffed copy of a long interval
into 4096-bit slots and decode every slot from its first bit.  Natural content puts an MCU start, a 31-bit code + value step
or a slot-spanning MCU on a slot edge only by chance; this writer puts them there on purpose.  Offsets count in the interval's
unstuffed copy: bit 0 is the first byte after the SOS segment or after an RST marker, the coordinates the slots use.  The
writer works in those bits, so stuffed zeros do not move anything.

An MCU is a list of blocks in zig-zag order with zz[0] = the DC difference (written as such, the predictor restarts at every
interval).  Its cost in bits follows from the Huffman tables coef_jpeg.encode_coefs writes; `goto` and `end` pad with MCUs of
exactly computed cost (DC sizes and run-0 AC values whose codes add up to the gap).  `finish` writes the file through
coef_jpeg.encode_coefs and checks that its trace (bit position of every MCU and block start, the reference's int16 DC
predictors at every MCU start, the interval's length) equals the plan: that trace is the truth map the tests compare with."""
import numpy as np

import coef_jpeg as CJ
from mini_jpeg import ZZ, canonical_codes

SLOT = 4096
CHUNK = 1300                                       # most extra bits one padding block absorbs (62 AC values of 10-bit codes)


def value(s, sign=1):
    """A value of size s (0 for s = 0)."""
    return 0 if s == 0 else sign * (1 << (s - 1))


class SlotWriter:
    """samp: (H, V) per component (one entry = greyscale).  ri: MCUs per restart interval; dri=False writes no DRI (ri None:
    the one interval takes as many MCUs as are written, `end` rounds them up to whole rows).  width: MCUs per row.
    qtabs / qsel / precision as coef_jpeg.encode_coefs; shared_tables: every component decodes with table 0; dc_runs: the DC tables carry coef_jpeg.DC_RUN_SYMBOLS."""

    def __init__(self, samp, ri, width, dri=True, precision=8, qtabs=None, qsel=None, shared_tables=False, dc_runs=False, seed=0):
        self.samp = tuple(tuple(s) for s in samp); self.ncomp = len(samp)
        self.comp = [c for c, (h, v) in enumerate(self.samp) for _ in range(h * v)]
        assert dri or ri is None
        self.bpm = len(self.comp); self.ri = ri if ri else 1 << 30; self.width = width; self.dri = dri
        self.precision = precision; self.shared = shared_tables; self.use_runs = dc_runs
        self.qtabs = qtabs if qtabs is not None else [np.ones(64, np.int64)] * 2
        self.qsel = qsel if qsel is not None else [0, 1, 1][:self.ncomp]
        self.dcc = canonical_codes(*CJ.dc_table(True, runs=dc_runs))
        ntab = 1 if (self.ncomp == 1 or shared_tables) else 2
        self.acc = [canonical_codes(*CJ.ac_table(True, variant=t)) for t in range(ntab)]
        self.tab = [0 if (c == 0 or shared_tables) else 1 for c in self.comp]
        self.rng = np.random.default_rng(seed)
        self.mcus = []                              # [(blocks, runs)]
        self.plan = [[]]                            # per interval: planned MCU start bits
        self.blk_plan = [[]]                        # ... block start bits, per MCU
        self.across = [[]]                          # ... symbols across a slot edge: (start bit, kind, code length, length)
        self.pos = 0                                # bit position in the current interval
        self.n_in = 0                               # MCUs in the current interval
        self.way = [self._ways(t) for t in range(ntab)]

    # --- costs ---------------------------------------------------------------------------------------------------------
    def _ways(self, t):
        """AC run-0 sizes whose codes + values add up to exactly r bits, fewest values first."""
        cost = {s: self.acc[t][s][1] + s for s in range(1, 14)}
        way = {0: []}
        for r in range(1, CHUNK + 64):
            best = None
            for s, c in cost.items():
                if r - c in way and (best is None or len(way[r - c]) + 1 < len(best)):
                    best = way[r - c] + [s]
            if best is not None:
                way[r] = best
        return way

    def block_items(self, b, zz, run=0):
        """(length, kind, code length) of every symbol of block b of an MCU: kind 'dc', 'ac', 'eob' or 'zrl'; the value bits
        are the length less the code length."""
        t = self.tab[b]
        out = []
        if run:
            a = int(zz[run]); s = abs(a).bit_length(); n = self.dcc[(run << 4) | s][1]; out.append((n + s, "dc", n)); k = run + 1
        else:
            d = int(zz[0]); s = abs(d).bit_length(); n = self.dcc[s][1]; out.append((n + s, "dc", n)); k = 1
        for p in range(k, 64):
            if not zz[p]:
                continue
            r = p - k
            while r > 15:
                out.append((self.acc[t][0xF0][1], "zrl", self.acc[t][0xF0][1])); r -= 16
            a = int(zz[p]); s = abs(a).bit_length(); n = self.acc[t][(r << 4) | s][1]
            out.append((n + s, "ac", n)); k = p + 1
        if k < 64:
            out.append((self.acc[t][0x00][1], "eob", self.acc[t][0x00][1]))
        return out

    def block_cost(self, b, zz, run=0):
        return sum(n for n, _, _ in self.block_items(b, zz, run))

    def mcu_cost(self, blocks, runs=None):
        return sum(self.block_cost(b, z, runs[b] if runs else 0) for b, z in enumerate(blocks))

    def min_block(self, b):
        return self.block_cost(b, np.zeros(64, np.int64))

    def exact_block(self, b, extra):
        """A block that costs min_block(b) + extra bits (extra = 0 or >= 2), DC difference and run-0 AC values."""
        t = self.tab[b]
        for ds in (0, 1, 2, 3, 4, 5, 6, 7, 8):
            de = (self.dcc[ds][1] + ds) - self.dcc[0][1]
            if de > extra or (extra - de) not in self.way[t] or len(self.way[t][extra - de]) > 62:
                continue
            zz = np.zeros(64, np.int64)
            zz[0] = value(ds, int(self.rng.choice([-1, 1])))
            for p, s in enumerate(self.way[t][extra - de], 1):
                zz[p] = value(s, int(self.rng.choice([-1, 1])))
            assert self.block_cost(b, zz) == self.min_block(b) + extra
            return zz
        raise ValueError(f"no block of {extra} extra bits")

    # --- placement -----------------------------------------------------------------------------------------------------
    def _roll(self):
        if self.n_in == self.ri:                    # the current interval is full: the next MCU starts the next one
            self.pos = 0; self.n_in = 0; self.plan.append([]); self.blk_plan.append([]); self.across.append([])

    def left(self):
        """MCUs the current interval still takes."""
        self._roll()
        return self.ri - self.n_in

    def mcu(self, blocks, runs=None):
        """Append one MCU (bpm zig-zag blocks, zz[0] = DC difference); returns its start bit."""
        assert len(blocks) == self.bpm
        self._roll()
        self.n_in += 1
        start = self.pos
        self.plan[-1].append(start)
        blocks = [np.asarray(z, np.int64).copy() for z in blocks]
        self.mcus.append((blocks, list(runs) if runs else None))
        starts = []
        for b, z in enumerate(blocks):
            starts.append(self.pos)
            for n, kind, code in self.block_items(b, z, runs[b] if runs else 0):
                if self.pos // SLOT != (self.pos + n - 1) // SLOT:
                    self.across[-1].append((self.pos, kind, code, n))
                self.pos += n
        self.blk_plan[-1].append(starts)
        return start

    def pad(self, nbits, n):
        """n MCUs of exactly nbits bits in all."""
        mn = [self.min_block(b) for b in range(self.bpm)]
        extra = nbits - n * sum(mn)
        assert extra >= 0 and extra != 1, (nbits, n, extra)
        chunks = []
        while extra:
            c = min(extra, CHUNK)
            if extra - c == 1:
                c -= 2
            chunks.append(c); extra -= c
        nblk = n * self.bpm
        assert len(chunks) <= nblk, ("padding needs more blocks", nbits, n)
        # spread the chunks over the blocks evenly
        ex = [0] * nblk
        for i, c in enumerate(chunks):
            ex[(i * nblk) // max(1, len(chunks))] = c
        for m in range(n):
            self.mcu([self.exact_block(b, ex[m * self.bpm + b]) for b in range(self.bpm)])

    def _count_for(self, gap, most):
        mn = sum(self.min_block(b) for b in range(self.bpm))
        n = max(1, min(most, gap // (mn + 600)))
        while n > 1 and (gap - n * mn < 0 or gap - n * mn == 1):
            n -= 1
        while gap - n * mn > CHUNK * n * self.bpm and n < most:
            n += 1
        return n

    def goto(self, bit):
        """Pad the current interval so that the next MCU starts at `bit` (keeps at least one MCU for the rest)."""
        most = self.left() - 1
        gap = bit - self.pos
        if gap == 0:
            return
        n = self._count_for(gap, most)
        self.pad(gap, n)
        assert self.pos == bit

    def end(self, nbits):
        """Pad the rest of the current interval so that its data end at bit nbits."""
        n = self.left()
        if not self.dri:                            # the one open interval: whole MCU rows
            mn = sum(self.min_block(b) for b in range(self.bpm))
            n = (-len(self.mcus)) % self.width
            while True:
                extra = nbits - self.pos - n * mn
                if n == 0 and extra == 0 or n and extra >= 0 and extra != 1 and extra <= CHUNK * n * self.bpm:
                    break
                assert extra >= 0, ("the interval is already longer", nbits, self.pos)
                n += self.width
        if n == 0:
            assert self.pos == nbits
            return
        self.pad(nbits - self.pos, n)
        assert self.pos == nbits

    def random_mcu(self, density=0.1, smin=1, smax=10, dc_smax=10):
        blocks = []
        for b in range(self.bpm):
            zz = np.zeros(64, np.int64)
            zz[0] = value(int(self.rng.integers(0, dc_smax + 1)), int(self.rng.choice([-1, 1]))) + (int(self.rng.integers(0, 2)) if dc_smax > 1 else 0)
            for p in range(1, 64):
                if self.rng.random() < density:
                    s = int(self.rng.integers(smin, smax + 1))
                    zz[p] = value(s, int(self.rng.choice([-1, 1])))
            blocks.append(zz)
        return blocks

    # --- the file ------------------------------------------------------------------------------------------------------
    def finish(self):
        """(jpeg bytes, coef_jpeg spec, truth): truth is the trace of coef_jpeg.encode_coefs, one dict per interval."""
        nmcu = len(self.mcus)
        if not self.dri:
            self.ri = nmcu
        assert nmcu % self.ri == 0 and nmcu % self.width == 0, (nmcu, self.ri, self.width)
        rows = nmcu // self.width
        hmax = max(h for h, v in self.samp); vmax = max(v for h, v in self.samp)
        W, H = 8 * hmax * self.width, 8 * vmax * rows
        grids = [np.zeros(CJ.block_shape(W, H, self.samp, c) + (64,), np.int64) for c in range(self.ncomp)]
        rgrids = [np.zeros(CJ.block_shape(W, H, self.samp, c), np.int64) for c in range(self.ncomp)]
        order = CJ._mcu_order(W, H, self.samp)
        pred = [0] * self.ncomp
        for n, ((blocks, runs), pos) in enumerate(zip(self.mcus, order)):
            if n % self.ri == 0:
                pred = [0] * self.ncomp
            for b, (c, br, bc) in enumerate(pos):
                z = blocks[b]; r = runs[b] if runs else 0
                pred[c] += 0 if r else int(z[0])
                nat = np.zeros(64, np.int64); nat[ZZ] = z; nat[0] = pred[c]
                grids[c][br, bc] = nat; rgrids[c][br, bc] = r
        trace = []
        j, spec = CJ.encode_coefs(grids, W, H, self.samp, self.qtabs, self.qsel, precision=self.precision,
                                  dri=self.ri if self.dri else 0, shared_tables=self.shared,
                                  dc_runs=rgrids if self.use_runs else None, trace=trace)
        assert [t["mcu_bits"] for t in trace] == self.plan, "the file does not follow the plan"
        assert [t["blk_bits"] for t in trace] == self.blk_plan, "the file does not follow the plan"
        for t, a in zip(trace, self.across):
            t["across"] = a                         # the plan's symbols across a slot edge (its block starts are the file's)
        return j, spec, trace
