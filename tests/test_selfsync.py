"""The self-synchronising Huffman passes (K1s: k_ph_sync, k_ph_fix_cta, k_ph_scan, then k_huff_lane<VSEG>) on bit-placed scans.

The corpus comes from tests/slot_jpeg.py, built in memory from fixed seeds; every file takes the self-synchronising path
(ri * bpm >= JS_PSYNC_MIN_BLOCKS) except one short-interval file for the lane and warp kernels.  Slot i of an interval is
bits [4096 i, 4096 (i + 1)) of its unstuffed copy.  The corpus puts MCU starts on slot edges and one bit either side,
31-bit code + value steps across them, settled exit states at every block of a 4:2:0 MCU, at zig-zag 1, 63 and before an
EOB, MCUs that span three slots next to slots with hundreds of MCU starts, last slots of 0, 1, 2047-2049 and 4095 data bits,
511-513-byte intervals, unstuffed copies that end on and beside a 512-byte boundary of ph_slot_base's addressing,
ph_nslots of 255, 256 and 257 (k_ph_scan's passes and a one-slot vitem), int16 DC sums that wrap (DQT 255 / 65535, 12-bit), DC symbols with a run nibble, the largest MCU
(three components at 4x4) and a file whose block phase no decoder can observe, so the fix rounds run past PH_MAX_ROUNDS.

CPU: the corpus reaches those edges, by the writer's truth map and by the kernels' own per-slot code run on the host
(tests/native/phuff_model.cpp); that code's virtual intervals equal the truth map for every slot order and guess length;
the compiled reference equals coef_jpeg.expected where it applies and the C port equals the reference.
GPU: every file with every Huffman kernel against the reference, alone and batched (a K1x rescue counts as a failure),
the fix-round counts, DC-only mode, damaged scans line by line, and a batch large enough that a CTA of k_ph_sync meets
several images that share their decode tables but not their MCU layout."""
import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np
import pytest

import coef_jpeg as CJ
import jpeg_cases as JC
import slot_jpeg as SJ
from oracle_util import Oracle, ref_available

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "jpegsnoop_b200", "csrc")
WHAT = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "mcu_map", "blk_dc", "dht_histo")
FIELDS = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "blk_dc")
needs_ref = pytest.mark.skipif(not ref_available("fixed"), reason="needs the compiled reference (oracle/_ref)")


def _const(name, header):
    src = open(os.path.join(CSRC, header)).read()
    return int(re.search(r"#define\s+%s\s+(\d+)" % name, src).group(1))


PSYNC_MIN = _const("JS_PSYNC_MIN_BLOCKS", "jsgpu_internal.h")
USLACK = _const("JS_USLACK", "jsgpu_internal.h")
LANE_SEGS = _const("JS_LANE_SEGS", "jsgpu_internal.h")
MAX_ROUNDS = _const("PH_MAX_ROUNDS", "jsgpu_phuff_core.cuh")
MAX_BPM = _const("PH_MAX_BPM", "jsgpu_phuff_core.cuh")
GUESS_BITS = _const("PH_GUESS_BITS", "jsgpu_phuff_core.cuh")
S420, S422, S444, GREY = ((2, 2), (1, 1), (1, 1)), ((2, 1), (1, 1), (1, 1)), ((1, 1), (1, 1), (1, 1)), ((1, 1),)
S48 = ((4, 4), (4, 4), (4, 4))


def ph_nslots(scan_len, nseg):
    """jsgpu_api.cu: uregion = align_up(scan_len + JS_USLACK * nseg + 128, 256); ph_nslots = (uregion >> 9) + nseg + 2."""
    uregion = (scan_len + USLACK * nseg + 128 + 255) // 256 * 256
    return (uregion >> 9) + nseg + 2


# --- the corpus ----------------------------------------------------------------------------------------------------------

def _z(*vals, dc=0):
    """zig-zag block: DC difference dc, then the values at zig-zag 1, 2, ..."""
    z = np.zeros(64, np.int64); z[0] = dc
    z[1:1 + len(vals)] = vals
    return z


def _edges_420():
    """4:2:0, no DRI.  One placement per slot edge e = 4096 i: MCU starts at e, e - 1 and e + 1; a 31-bit DC step (16-bit
    code, size 15) with its code and then its value across e; the same for an AC step; a block start of every index 1..5
    one bit past e; a block whose zig-zag 63 value starts at e; an EOB at e.  Then MCUs of 58 values of sizes 12..15 per block
    (each spans three slots) next to MCUs of 26 bits (157 MCU starts per slot).  The data end 2047 bits into the last slot."""
    w = SJ.SlotWriter(S420, ri=None, width=40, dri=False, seed=1)
    e = [SJ.SLOT * i for i in range(1, 40)]
    flat = [np.zeros(64, np.int64)] * 6
    big_dc = _z(dc=SJ.value(15)); big_ac = _z(SJ.value(15, -1))
    k = 0

    def at(bit, blocks):
        w.goto(bit); w.mcu(blocks)

    for d in (0, -1, 1):
        at(e[k] + d, w.random_mcu()); k += 1
    for back in (1, 8, 20):                                # DC: code across the edge (exit 30 bits past it), then the value
        at(e[k] - back, [big_dc] + flat[1:]); k += 1
    for back in (8, 20):                                   # AC (behind a 2-bit DC): code, then value across the edge
        at(e[k] - 2 - back, [big_ac] + flat[1:]); k += 1
    for b in range(1, 6):                                  # the first symbol at/after the edge opens block b
        pre = sum(w.block_cost(i, flat[i]) for i in range(b))
        at(e[k] + 1 - pre, flat); k += 1
    z63 = np.zeros(64, np.int64); z63[1:64] = 1            # DC 0 (2 bits) + 63 values of 4 bits: zig-zag 63 at +250
    at(e[k] - 250, [z63] + flat[1:]); k += 1
    zeob = _z(1, 1, 1, 1, 1)                               # DC 0 + five 4-bit values: the EOB at +22
    at(e[k] - 22, [zeob] + flat[1:]); k += 1
    w.goto(e[k] + 100)
    for _ in range(2):
        dense = []                                         # 58 values of sizes 12..15 per block: ~9.5 kbit per MCU
        for b in range(6):
            z = np.zeros(64, np.int64)
            z[1:59] = [SJ.value(int(s), int(g)) for s, g in zip(w.rng.integers(12, 16, 58), w.rng.choice([-1, 1], 58))]
            dense.append(z)
        w.mcu(dense)
        for _ in range(200):
            w.mcu(flat)                                    # 26 bits each
    nb = (w.pos // SJ.SLOT + 3) * SJ.SLOT + 2047
    w.end(nb)
    return w.finish()


def _flat_grey():
    """Greyscale, no DRI: slots of 682 6-bit MCUs next to slots without an MCU start (blocks of 63 values of sizes 12..15);
    the data end on a slot edge (L mod 4096 = 0)."""
    w = SJ.SlotWriter(GREY, ri=None, width=256, dri=False, seed=2)
    for r in range(6):
        for i in range(1500):
            w.mcu([_z(dc=1 - 2 * (i & 1))])               # 6 bits: a DC difference of +-1 and an EOB
        for _ in range(6):
            z = np.zeros(64, np.int64)
            z[1:64] = [SJ.value(int(s), int(g)) for s, g in zip(w.rng.integers(12, 16, 63), w.rng.choice([-1, 1], 63))]
            w.mcu([z])
    w.end((w.pos // SJ.SLOT + 2) * SJ.SLOT)
    return w.finish()


def _lengths_420():
    """4:2:0, DRI 32 (192 blocks: the self-synchronising path): intervals whose data end at L = 8192 + 0, 1, 2047, 2048, 2049,
    4095 bits, and intervals of 511, 512 and 513 unstuffed bytes."""
    w = SJ.SlotWriter(S420, ri=32, width=32, seed=3)
    ends = [8192 + r for r in (0, 1, 2047, 2048, 2049, 4095)] + [8 * 511, 8 * 512, 8 * 513]
    for nb in ends:
        for _ in range(4):
            w.mcu(w.random_mcu(0.05))
        w.end(nb)
    return w.finish()


def _wrap(samp, q, precision, seed, name_dc_smax):
    """No DRI, random content whose DC differences make the int16 predictor sums wrap (or, for P = 12, truncate toward zero
    on negative values), with an MCU start on every slot edge."""
    bpm = sum(h * v for h, v in samp)
    n = -(-PSYNC_MIN // bpm) * 4
    w = SJ.SlotWriter(samp, ri=None, width=16, dri=False, precision=precision, qtabs=[q, q], seed=seed)
    for i in range(n):
        if i % 40 == 39:
            w.goto((w.pos // SJ.SLOT + 1) * SJ.SLOT)
        w.mcu(w.random_mcu(0.08, 1, 12, dc_smax=name_dc_smax))
    w.end(w.pos + 1500)
    return w.finish()


def _runs(samp, ri, width, dri, seed):
    """DC symbols with a run nibble: about one block in four carries its zig-zag value r (1..15) with the DC symbol r|size."""
    w = SJ.SlotWriter(samp, ri=ri if dri else None, width=width, dri=dri, dc_runs=True, seed=seed)
    rng = np.random.default_rng(seed)
    bpm = w.bpm
    total = ri * (1 if not dri else 24)
    for m in range(total):
        blocks, runs = [], []
        for b in range(bpm):
            z = w.random_mcu(0.1, 1, 9)[0]
            r = 0
            if rng.random() < 0.25:
                r = int(rng.integers(1, 16))
                z[0] = 0; z[1:r] = 0
                z[r] = SJ.value(r * 7 % 15 + 1, int(rng.choice([-1, 1])))
            blocks.append(z); runs.append(r)
        w.mcu(blocks, runs)
    return w.finish()


def _bpm48():
    """Three components at 4x4: 48 blocks per MCU (PH_MAX_BPM), no DRI."""
    w = SJ.SlotWriter(S48, ri=None, width=4, dri=False, seed=6)
    for _ in range(8):
        w.mcu(w.random_mcu(0.06, 1, 11))
    return w.finish()


def _rounds():
    """4:2:2 with one shared table pair (the block phase cannot be observed) and every block exactly 1024 bits: a guess
    starts at a block start PH_GUESS_BITS before its slot's end, two blocks off the MCU grid, so its exit state is wrong in
    every slot and each fix round repairs one more slot.  48 slots: more than PH_MAX_ROUNDS + 2."""
    w = SJ.SlotWriter(S422, ri=None, width=48, dri=False, shared_tables=True, seed=7)
    for _ in range(48):
        w.mcu([w.exact_block(b, 1024 - w.min_block(b)) for b in range(4)])
    return w.finish()


def _scan(j):
    s = j.index(b"\xff\xda")
    return j[s + 2 + int.from_bytes(j[s + 2:s + 4], "big"):]


def interval_starts(j):
    """Raw scan offset s0 of every restart interval: 0, then 2 past every RST marker."""
    sc = _scan(j)
    return [0] + [i + 2 for i in range(len(sc) - 1) if sc[i] == 0xFF and 0xD0 <= sc[i + 1] <= 0xD7]


def copy_end(s0, k, ulen):
    """Where the unstuffed copy of interval k ends in the image's region: ph_slot_base's (s0 & ~15) + JS_USLACK * k, + ulen."""
    return (s0 & ~15) + USLACK * k + ulen


def _nslots_grey(want, seed):
    """Greyscale, no DRI, one interval sized so that ph_nslots = want (the scan length is steered through the restated
    formula, by the bytes the writer produced)."""
    target = ((want - 3) << 9) - USLACK - 128              # the middle of the scan lengths that give `want`
    nbits = 8 * target
    for _ in range(6):
        w = SJ.SlotWriter(GREY, ri=None, width=64, dri=False, seed=seed)
        w.end(nbits)
        f = w.finish()
        n = len(_scan(f[0]))
        if ph_nslots(n, 1) == want and abs(n - target) < 200:
            return f
        nbits -= 8 * (n - target)
    raise AssertionError(("cannot size the scan", want, n))


def _copy_ends(wants, seed):
    """Greyscale, DRI 256 (ri * bpm >= JS_PSYNC_MIN_BLOCKS): one long interval per entry of `wants`, whose unstuffed copy ends
    at that residue mod 512 of ph_slot_base's addressing; then one more interval."""
    ulen = [3000 + 700 * k for k in range(len(wants) + 1)]

    def build():
        w = SJ.SlotWriter(GREY, ri=256, width=256, seed=seed)
        for u in ulen:
            w.end(8 * u)
        return w.finish()

    f = build()
    for k, want in enumerate(wants):
        s0 = interval_starts(f[0])[k]                          # does not depend on this interval or the later ones
        ulen[k] += (want - copy_end(s0, k, ulen[k])) % 512
        f = build()
    return f


@functools.lru_cache(maxsize=None)
def corpus():
    """[(name, jpeg, spec, truth)]"""
    q255, q65535 = np.full(64, 255), np.full(64, 65535)
    out = [("edges_420",) + _edges_420(), ("flat_grey",) + _flat_grey(), ("lengths_420_dri32",) + _lengths_420(),
           ("wrap_q255_420",) + _wrap(S420, q255, 8, 11, 10), ("wrap_q65535_grey",) + _wrap(GREY, q65535, 8, 12, 6),
           ("p12_422",) + _wrap(S422, np.arange(1, 65), 12, 13, 14),
           ("runs_444",) + _runs(S444, 96, 32, False, 21), ("runs_420_dri1",) + _runs(S420, 1, 8, True, 22),
           ("bpm48",) + _bpm48(), ("rounds_422_shared",) + _rounds(),
           ("copy_ends_grey_dri256",) + _copy_ends([511, 0, 1], 41)]
    out += [(f"nslots{n}_grey",) + _nslots_grey(n, 50 + n) for n in (255, 256, 257)]
    return out


def _psync(spec):
    bpm = sum(h * v for h, v in spec["samp"])
    nmcu = spec["blocks"][0].shape[0] * spec["blocks"][0].shape[1] // (spec["samp"][0][0] * spec["samp"][0][1])
    ri = spec["dri"] or nmcu
    return ri * bpm >= PSYNC_MIN


def _restated(name):
    return not name.startswith(("runs", "bpm48"))


# --- CPU: the host model -----------------------------------------------------------------------------------------------

def _model_lib(tmp_path_factory, guess_bits):
    so = str(tmp_path_factory.mktemp(f"phm{guess_bits}") / "libphuff_model.so")
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I/usr/local/cuda/include", "-o", so,
           os.path.join(HERE, "native", "phuff_model.cpp")]
    if guess_bits != GUESS_BITS:
        cmd.insert(1, f"-DPH_GUESS_BITS={guess_bits}u")
    subprocess.run(cmd, check=True)
    L = C.CDLL(so)
    L.phm_check.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    L.phm_walk.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    return L


@pytest.fixture(scope="module")
def models(built, tmp_path_factory):
    return {g: _model_lib(tmp_path_factory, g) for g in (64, 512, GUESS_BITS, 4096)}


def _run_model(L, j, order):
    from jpegsnoop_b200.host import parse_jpeg
    t, d, start = parse_jpeg(j)
    scan = np.frombuffer(j, np.uint8)[start:].copy()
    out = np.zeros(32, np.uint32)
    r = L.phm_check(C.byref(t), C.byref(d), scan.ctypes.data, scan.size, order, out.ctypes.data)
    assert r == 0, r
    return [int(v) for v in out]


def test_truth_map_is_what_a_sequential_walk_reads(models):
    """The writer's truth map (MCU start bits, int16 DC predictors, interval lengths) equals the host model's walk."""
    from jpegsnoop_b200.host import parse_jpeg
    L = models[GUESS_BITS]
    for name, j, spec, truth in corpus():
        t, d, start = parse_jpeg(j)
        scan = np.frombuffer(j, np.uint8)[start:].copy()
        nm = sum(len(tr["mcu_bits"]) for tr in truth)
        bits = np.zeros(nm + 8, np.uint32); dc = np.zeros((nm + 8) * 3, np.int16); ulen = np.zeros(len(truth) + 8, np.uint32)
        m = L.phm_walk(C.byref(t), C.byref(d), scan.ctypes.data, scan.size, bits.ctypes.data, dc.ctypes.data, nm + 8,
                       ulen.ctypes.data, len(truth) + 8)
        assert m == nm, (name, m, nm)
        assert bits[:nm].tolist() == [b for tr in truth for b in tr["mcu_bits"]], name
        ncomp = len(spec["samp"])
        want = np.array([p for tr in truth for p in tr["dc"]], np.int64).reshape(nm, ncomp)
        assert np.array_equal(dc.reshape(-1, 3)[:nm, :ncomp], want), name
        assert ulen[:len(truth)].tolist() == [(tr["nbits"] + 7) // 8 for tr in truth], name


def reach():
    """name -> count over the corpus, from the truth map and the slot formulas."""
    hits = {}
    add = lambda k, n=1: hits.__setitem__(k, hits.get(k, 0) + int(n))
    for name, j, spec, truth in corpus():
        scan_len = len(_scan(j))
        if not _psync(spec):
            add("short_interval_file")
            continue
        ns = ph_nslots(scan_len, len(truth))
        add(f"nslots_mod256_{ns % 256}", ns >= 255)
        add("vitem_with_one_slot", ns % LANE_SEGS == 1)
        for k, (s0, tr) in enumerate(zip(interval_starts(j), truth)):
            add(f"copy_end_mod512_{copy_end(s0, k, (tr['nbits'] + 7) // 8) % 512}", len(truth) > 1)
        for tr in truth:
            for pos, kind, code, n in tr["across"]:
                e = (pos // SJ.SLOT + 1) * SJ.SLOT
                add(f"{kind}_code_across_edge", pos < e < pos + code)
                add(f"{kind}_value_across_edge", pos + code < e < pos + n)
                add("step31_across_edge", n == 31)
            mb = tr["mcu_bits"]; L = tr["nbits"]; ub = (L + 7) // 8
            for b in mb[1:]:
                for d, k in ((0, "mcu_on_edge"), (-1, "mcu_one_before_edge"), (1, "mcu_one_after_edge")):
                    add(k, (b - d) % SJ.SLOT == 0)
            for blks in tr["blk_bits"]:
                for i, b in enumerate(blks[1:], 1):
                    add(f"block{i}_one_after_edge", b % SJ.SLOT == 1 and i < 6 and len(blks) == 6)
            nsub = (ub + 511) // 512
            per = np.bincount(np.array(mb) // SJ.SLOT, minlength=nsub)[:nsub]
            add("slot_without_mcu_start", (per == 0).sum())
            add("slot_with_over_150_mcu_starts", (per > 150).sum())
            ends = mb[1:] + [L]
            add("mcu_spans_three_slots", sum(1 for a, b in zip(mb, ends) if b // SJ.SLOT - a // SJ.SLOT >= 2))
            add(f"last_slot_data_bits_{L % SJ.SLOT}")
            last = ub * 8 - (nsub - 1) * SJ.SLOT                          # lim - s0 of the last slot
            add("last_slot_guess_from_start", nsub > 1 and last <= GUESS_BITS)
            add("last_slot_guess_inside", nsub > 1 and last > GUESS_BITS)
            add(f"interval_bytes_{ub}", ub in (511, 512, 513))
            add("several_long_intervals", len(truth) > 1)
        add(f"bpm_{sum(h * v for h, v in spec['samp'])}")
        add("dc_run_symbols_psync", spec is not None and name.startswith("runs"))
        dcs = np.array([p for tr in truth for p in tr["dc"]], np.int64)
        add("dc_predictor_below_minus_30000", (dcs < -30000).any()); add("dc_predictor_above_30000", (dcs > 30000).any())
        add("p12_psync", spec["precision"] == 12)
    return hits


REQUIRED = (["mcu_on_edge", "mcu_one_before_edge", "mcu_one_after_edge", "slot_without_mcu_start", "slot_with_over_150_mcu_starts",
             "mcu_spans_three_slots", "last_slot_guess_from_start", "last_slot_guess_inside", "several_long_intervals",
             "dc_predictor_below_minus_30000", "dc_predictor_above_30000", "p12_psync", "dc_run_symbols_psync",
             "short_interval_file", f"bpm_{MAX_BPM}"]
            + [f"block{i}_one_after_edge" for i in range(1, 6)]
            + [f"last_slot_data_bits_{r}" for r in (0, 1, 2047, 2048, 2049, 4095)]
            + [f"interval_bytes_{b}" for b in (511, 512, 513)]
            + [f"nslots_mod256_{r}" for r in (255, 0, 1)] + ["vitem_with_one_slot"]
            + [f"copy_end_mod512_{r}" for r in (511, 0, 1)]
            + ["dc_code_across_edge", "dc_value_across_edge", "ac_code_across_edge", "ac_value_across_edge", "step31_across_edge"])


def test_corpus_reaches_the_slot_edges(models):
    """By the truth map, and by the kernels' own per-slot code on the settled exit states (host model)."""
    hits = reach()
    print("\n".join(f"{k:36s} {hits.get(k, 0)}" for k in REQUIRED))
    missing = [k for k in REQUIRED if not hits.get(k)]
    assert not missing, missing
    L = models[GUESS_BITS]
    tot = {}
    blk_mask = zz_mask = 0
    for name, j, spec, truth in corpus():
        if not _psync(spec):
            continue
        o = _run_model(L, j, 0)
        for i, k in ((6, "no_mcu_start"), (7, "exit_blk_nonzero"), (8, "exit_zz_nonzero"), (9, "exit_past_end"), (11, "exit_before_eob")):
            tot[k] = tot.get(k, 0) + o[i]
        tot["max_overshoot"] = max(tot.get("max_overshoot", 0), o[10])
        tot["max_mcu_starts_per_slot"] = max(tot.get("max_mcu_starts_per_slot", 0), o[12])
        if name.startswith("edges"):
            blk_mask |= o[13]; zz_mask |= o[15] | (o[16] << 32)
        if name == "rounds_422_shared":
            assert o[1] > MAX_ROUNDS + 1 and o[18] > 0 and o[17] > 0, o[:19]
        else:
            assert o[1] <= MAX_ROUNDS - 1, (name, o[1])
        print(name, "fix rounds", o[1])
    print(tot, hex(blk_mask), hex(zz_mask))
    for k in ("no_mcu_start", "exit_blk_nonzero", "exit_zz_nonzero", "exit_past_end", "exit_before_eob"):
        assert tot[k] > 0, k
    assert tot["max_overshoot"] == 30 and tot["max_mcu_starts_per_slot"] >= 600
    assert blk_mask & 0x3F == 0x3F, hex(blk_mask)                       # 4:2:0 exits at every block index 0..5
    assert zz_mask & (1 << 1) and zz_mask & (1 << 63), hex(zz_mask)


@pytest.mark.parametrize("guess_bits", [64, 512, GUESS_BITS, 4096])
@pytest.mark.parametrize("order", [0, 1, 2], ids=["descending", "ascending", "shuffled"])
def test_virtual_intervals_match_the_truth_map(models, order, guess_bits):
    """The kernels' per-slot code (guess, fix rounds, prefix sums, virtual intervals) lands every virtual interval on a true MCU
    start with the true DC predictors, and the intervals tile every real interval.  A different guess length may change
    the number of rounds, never the result."""
    L = models[guess_bits]
    for name, j, spec, truth in corpus():
        if not _psync(spec):
            continue
        o = _run_model(L, j, order)
        nm = sum(len(tr["mcu_bits"]) for tr in truth)
        assert o[0] == 0 and o[5] == nm, (name, o[:6])


@needs_ref
def test_reference_decodes_the_corpus_as_restated(built):
    o = Oracle("ref_fixed")
    lf, li = o.idct_tables()
    for name, j, spec, truth in corpus():
        d = o.decode(j)
        assert d.nerr == 0, (name, o.err_lines()[:3])
        if _restated(name):
            bad = JC.compare(CJ.expected(spec, True, li, lf), d, what=FIELDS)
            assert not bad, (name, bad)


def test_port_matches_the_reference_on_the_corpus(built):
    port = Oracle("port", idct_fixed=True)
    have_ref = ref_available("fixed")
    ref = Oracle("ref_fixed") if have_ref else None
    lf, li = port.idct_tables()
    for name, j, spec, truth in corpus():
        got = port.decode(j)
        assert got.nerr == 0, name
        if have_ref:
            want = ref.decode(j)
            assert not JC.compare(want, got), name
            assert np.array_equal(want.stats, got.stats), (name, want.stats, got.stats)
        elif _restated(name):
            assert not JC.compare(CJ.expected(spec, True, li, lf), got, what=FIELDS), name


# --- damaged scans -----------------------------------------------------------------------------------------------------

def _raw_of(scan, u):
    """raw offset in `scan` of unstuffed byte u of its first interval"""
    kept = 0
    for r in range(len(scan)):
        if scan[r] == 0 and r > 0 and scan[r - 1] == 0xFF:
            continue
        if kept == u:
            return r
        kept += 1
    return len(scan)


@functools.lru_cache(maxsize=None)
def damaged():
    """[(name, jpeg)]: the edges file truncated on a slot edge, at an MCU start inside a slot and inside a slot-spanning MCU,
    and with surplus bytes behind its last MCU."""
    name, j, spec, truth = corpus()[0]
    s = j.index(b"\xff\xda"); s0 = s + 2 + int.from_bytes(j[s + 2:s + 4], "big")
    scan = j[s0:-2]
    mb = truth[0]["mcu_bits"]
    cut = lambda u: j[:s0] + scan[:_raw_of(scan, u)] + b"\xff\xd9"
    inside = next(b for b in mb if b % SJ.SLOT > 1000 and b % 8 == 0 and b > 3 * SJ.SLOT)
    ends = mb[1:] + [truth[0]["nbits"]]
    span = next(a for a, b in zip(mb, ends) if b - a > 2 * SJ.SLOT)
    return [("trunc_on_slot_edge", cut(512 * 6)), ("trunc_at_mcu_start", cut(inside // 8)),
            ("trunc_in_spanning_mcu", cut((span + SJ.SLOT + 300) // 8)),
            ("surplus_after_last_mcu", j[:-2] + bytes([0x5A, 0xC3] * 700) + b"\xff\xd9")]


# --- GPU -----------------------------------------------------------------------------------------------------------------

def _check(want, got, name, what=WHAT):
    bad = JC.compare(want, got, what=what)
    assert not bad, f"{name}: mismatch with the reference in {bad}"


@functools.lru_cache(maxsize=None)
def _ref_out():
    o = Oracle("ref_fixed")
    return {n: (o.decode(j, quiet=False), o.log_lines()) for n, j, _, _ in corpus()}


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("huff", [0, 1, 2], ids=["huff_selfsync", "huff_warp", "huff_lane"])
def test_corpus_matches_the_reference(built, huff):
    """Every file as a single drop-in (every buffer, the stats row, the full log) and in one batch (status 0: a K1x rescue
    of a healthy file is a failure)."""
    from jpegsnoop_b200 import BatchDecoder, CimgDecode
    want = _ref_out()
    dec = CimgDecode(idct_fixedpt=True, huff_kernel=huff, idct_kernel=0)
    for name, j, _, _ in corpus():
        got = dec.decode(j, quiet=False)
        _check(want[name][0], got, name)
        assert np.array_equal(np.asarray(want[name][0].stats), np.asarray(got.stats)[:12]), (name, want[name][0].stats, got.stats)
        gl = dec.log_lines(-1)
        assert gl == want[name][1], (name, [(a, b) for a, b in zip(want[name][1], gl) if a != b][:3])
    dec.close()
    bd = BatchDecoder(huff_kernel=huff, idct_kernel=0)
    bd.set_batch([j for _, j, _, _ in corpus()]); bd.decode(); bd.sync()
    for i, (name, j, _, _) in enumerate(corpus()):
        got = bd.fetch(i)
        assert got.status == 0, (name, hex(got.status))
        _check(want[name][0], got, name)
    bd.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fixed", [True, False], ids=["idct_fixed", "idct_float"])
def test_restated_files_in_both_idct_builds(built, fixed):
    from jpegsnoop_b200 import CimgDecode
    o = Oracle("ref_fixed" if fixed else "ref_float") if ref_available("fixed" if fixed else "float") else Oracle("port", idct_fixed=fixed)
    lf, li = o.idct_tables()
    dec = CimgDecode(idct_fixedpt=fixed, huff_kernel=0, idct_kernel=0)
    for name, j, spec, _ in corpus():
        if not _restated(name):
            continue
        got = dec.decode(j)
        _check(o.decode(j), got, name)
        bad = JC.compare(CJ.expected(spec, fixed, li, lf), got, what=FIELDS)
        assert not bad, (name, bad)
    dec.close()


@pytest.mark.gpu
def test_fix_round_counts(built):
    """Alone in a batch, every file settles before fix round PH_MAX_ROUNDS except the one whose block phase cannot be observed:
    its round PH_MAX_ROUNDS still changes slots, and k_ph_fix_cta finishes the job (the pixels are checked above)."""
    from jpegsnoop_b200 import BatchDecoder
    for name, j, spec, _ in corpus():
        bd = BatchDecoder(huff_kernel=0, idct_kernel=0)
        bd.set_batch([j]); bd.decode(); bd.sync()
        nimg, nslots, chg = bd.selfsync_info()
        assert nimg == (1 if _psync(spec) else 0), (name, nimg)
        if _psync(spec):
            assert len(chg) >= MAX_ROUNDS, (name, chg)
            if name == "rounds_422_shared":
                assert chg[MAX_ROUNDS - 1] > 0, (name, chg)
            else:
                assert chg[MAX_ROUNDS - 1] == 0, (name, chg)
        assert bd.fetch(0).status == 0, name
        bd.close()


def _dc_only(huff, names):
    from jpegsnoop_b200 import CimgDecode
    o = Oracle("ref_fixed", decode_ac=False)
    todo = [(n, j) for n, j, _, _ in corpus() if n in names]
    want = {n: o.decode(j) for n, j in todo}
    o.close()
    dec = CimgDecode(decode_ac=False, idct_fixedpt=True, huff_kernel=huff, idct_kernel=0)
    for name, j in todo:
        got = dec.decode(j)
        assert got.nerr == 0, (name, dec.log_lines(3))
        _check(want[name], got, name, what=FIELDS)
    dec.close()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("huff", [0, 1, 2], ids=["huff_selfsync", "huff_warp", "huff_lane"])
def test_dc_only_mode(built, huff):
    """The reference runs no IDCT in DC-only mode: a run-nibble DC symbol's value (stored at zig-zag r) must not reach the
    pixels, in the self-synchronising, warp and lane kernels alike."""
    _dc_only(huff, [n for n, _, _, _ in corpus()])


@pytest.mark.gpu
@needs_ref
def test_damaged_scans_match_the_reference_line_for_line(built):
    """Truncations and surplus data in a long interval: ph_vseg's run-on (fewer MCUs than expected) and the final lane's end
    and leftover report; every buffer, the stats row and every log line equal the reference's."""
    from jpegsnoop_b200 import CimgDecode
    o = Oracle("ref_fixed")
    dec = CimgDecode(idct_fixedpt=True, huff_kernel=0, idct_kernel=0)
    for name, j in damaged():
        want = o.decode(j, quiet=False); wl = o.log_lines()
        got = dec.decode(j, quiet=False)
        _check(want, got, name)
        assert np.array_equal(np.asarray(want.stats), np.asarray(got.stats)[:12]), (name, want.stats, got.stats)
        gl = dec.log_lines(-1)
        assert gl == wl, (name, [(a, b) for a, b in zip(wl, gl) if a != b][:3], len(wl), len(gl))
    dec.close()


# --- a CTA of k_ph_sync meets images that share their decode tables but not their MCU layout ------------------------------

def _reuse_files():
    """Four one-vitem psync files with the same Huffman and quantisation tables and the same selectors (one table set, one
    tab_sig): 4:2:0, 4:4:4 and 4:2:2 at 8 bits, and 4:2:0 at 12 bits.  Each spans several slots and has non-zero DC
    differences, so a wrong layout or a wrong divide shows in the exit states and the DC sums."""
    q = np.arange(1, 65) % 23 + 1
    out = {}
    for key, samp, P, seed in (("420", S420, 8, 31), ("444", S444, 8, 32), ("422", S422, 8, 33), ("420p12", S420, 12, 34)):
        bpm = sum(h * v for h, v in samp)
        n = 16 * (-(-PSYNC_MIN // bpm // 16) + 1)
        w = SJ.SlotWriter(samp, ri=None, width=16, dri=False, precision=P, qtabs=[q, q], seed=seed)
        for _ in range(n):
            w.mcu(w.random_mcu(0.12, 1, 10, dc_smax=12 if P == 12 else 8))
        out[key] = w.finish()[0]
    return out


def _reuse_order(grid):
    """Image i is visited by CTA i % grid on pass i // grid.  CTA b meets, pass by pass: (b % 3 == 0) 4:2:0, 4:4:4, 4:2:2;
    (1) 8-bit 4:2:0, 12-bit 4:2:0, 8-bit 4:2:0; (2) the control, 4:2:0 three times."""
    seq = {0: ("420", "444", "422"), 1: ("420", "420p12", "420"), 2: ("420", "420", "420")}
    return [seq[b % 3][p] for p in range(3) for b in range(grid)]


@pytest.mark.gpu
@needs_ref
def test_cta_reuse_restages_each_image_layout(built):
    """N = 3 x (8 x SMs) one-vitem images, more than twice k_ph_sync's grid: every CTA decodes three images in turn that share
    (table_set, tab_sig) but differ in sampling or precision (or, as a control, do not).  Every image's checksums equal the
    reference's for its file and every status is 0."""
    import torch
    from jpegsnoop_b200 import BatchDecoder
    from jpegsnoop_b200.host import parse_jpeg
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = 8 * sms
    files = _reuse_files()
    keys = _reuse_order(grid)
    jpegs = [files[k] for k in keys]
    # preconditions, from the host preparation: one table set, one tab_sig, one vitem per image, nvitems > 2 x grid
    tarr, darr, _ = BatchDecoder.prepare(jpegs)
    assert len(tarr) == 1
    sel = {tuple((d.dht_dc_sel[c], d.dht_ac_sel[c], d.dqt_sel[c]) for c in range(d.num_sos_comps)) for d in darr}
    assert len(sel) == 1 and {d.num_sos_comps for d in darr} == {3}
    assert {(int(d.precision), tuple(d.samp_h[:3]), tuple(d.samp_v[:3])) for d in darr} == {
        (8, (2, 1, 1), (2, 1, 1)), (8, (1, 1, 1), (1, 1, 1)), (8, (2, 1, 1), (1, 1, 1)), (12, (2, 1, 1), (2, 1, 1))}
    for k, j in files.items():
        t, d, start = parse_jpeg(j)
        hm, vm = max(d.samp_h[:3]), max(d.samp_v[:3])
        nmcu = -(-d.dim_x // (8 * hm)) * -(-d.dim_y // (8 * vm))
        assert not d.restart_interval and nmcu * sum(h * v for h, v in zip(d.samp_h[:3], d.samp_v[:3])) >= PSYNC_MIN, k
        assert ph_nslots(len(j) - start, 1) <= LANE_SEGS, k              # one vitem
    assert len(jpegs) > 2 * grid
    _, errs, ck = Oracle("ref_fixed").bench_ck(list(files.values()))
    assert errs == 0
    want = dict(zip(files.keys(), ck))
    bd = BatchDecoder(huff_kernel=0, idct_kernel=0)
    bd.set_batch(jpegs); bd.decode(); bd.sync()
    assert bd.selfsync_info()[0] == len(jpegs)
    got = bd.checksums()
    st = np.array([int(l.status) for l in bd.refresh_layout()])
    bd.close()
    bad = [(i, keys[i], hex(int(st[i]))) for i in range(len(jpegs)) if st[i] != 0 or not np.array_equal(got[i], want[keys[i]])]
    summary = {}
    for i, k, s in bad:
        summary.setdefault((k, i // grid, s), 0)
        summary[(k, i // grid, s)] += 1
    assert not bad, summary
