"""Stage A (marker scan, unstuffing, the MCU file map's raw positions) on byte-placed scans and on both sides of the rules
that choose its kernel forms.

The placed corpus comes from tests/byte_jpeg.py: RST markers, terminators and stuffed FF 00 pairs on the last byte of
16-byte pieces, 64-byte spans, 512-byte rows, 4096-byte chunks and 32 KB passes; intervals with 6, 7 and more than 40 stuffed
zeros; MCU starts on both bytes of a stuffed pair.  The forms are
  marker scan:  k_marker_scan (CTA per image) when nimg >= 2 * JS_H100_SMS and the batch is not uneven, else k_marker_scan2;
  unstuff:      k_unstuff (warp per interval) when max_nseg < 256, else k_unstuff_lane; k_unstuff_long on the
                self-synchronising path (ri * bpm >= JS_PSYNC_MIN_BLOCKS);
  huff_kernel:  auto = lane kernel when the batch has 4096 or more short intervals.
JSGPU_MARKER / JSGPU_UNSTUFF force a form; the library reads them once per process, so forced forms run in a child process
(tests/stage_a_child.py).  Batch-size cases are derived below from the launch formulas, not from timing."""
import ctypes
import functools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import byte_jpeg as BJ
import coef_jpeg as CJ
import jpeg_cases as JC
from oracle_util import Oracle, effective_cores, ref_available

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "jpegsnoop_b200", "csrc")
WHAT = ("geom", "pix_y", "pix_cb", "pix_cr", "dib", "mcu_map", "blk_dc", "dht_histo")
needs_ref = pytest.mark.skipif(not ref_available("fixed"), reason="needs the compiled reference (oracle/_ref)")


def _const(name):
    src = open(os.path.join(CSRC, "jsgpu_internal.h")).read()
    return int(re.search(r"#define\s+%s\s+(\d+)" % name, src).group(1))


SMS = _const("JS_H100_SMS")
PSYNC_MIN = _const("JS_PSYNC_MIN_BLOCKS")
STUFF_LIST = _const("JS_STUFF_LIST")


# --- the placed corpus -----------------------------------------------------------------------------------------------

def _edges_file():
    """DRI 1, 34 chunks (> 128 KB: look-backs cross more than one 32-chunk window).  In every chunk: an RST on a piece end,
    a stuffed pair at a varying residue, an RST on a 64-byte span end, a pair on a 128-byte row end, an RST on a 512-byte row
    end, and an RST (or, every fifth chunk, a stuffed pair) on the chunk's last byte; chunk ends 8k - 1 are 32 KB pass ends."""
    w = BJ.Writer(dri=1)
    for c in range(34):
        base = 4096 * c
        w.rst_at(base + 16 * (2 + c % 4) - 1)
        w.pairs_at([base + 300 + c % 16])
        w.rst_at(base + 64 * (8 + c % 6) - 1)
        w.pairs_at([base + 128 * (9 + c % 3) - 1])
        w.rst_at(base + 512 * (3 + c % 3) - 1)
        w.pairs_at([base + 3000 + 7 * (c % 9), base + 3010 + 7 * (c % 9)])
        if c % 5 == 4:
            w.pairs_at([base + 4095])
        else:
            w.rst_at(base + 4095)
    return w.finish()


def _dense_file():
    """DRI 1: intervals with exactly 6 and exactly 7 lone stuffed pairs, with 45 values of +32767 (runs of adjacent pairs,
    more than 40 stuffed zeros), starting with an FF (DC difference of size 15), of 1..3 bytes, and lone pairs whose
    interval starts at every residue mod 16."""
    w = BJ.Writer(dri=1)
    for k in range(48):
        w.add(BJ.filler(1 + k % 3, 1, k))                       # fewer than 4 unstuffed bytes
        w.add(BJ.filler(5 + k, 1, k))                            # moves the next interval's start through every residue
        n = (6, 7)[k % 2]
        w.add(BJ.with_pairs([4 + 5 * i + (k % 3) for i in range(n)], 1))
        if k % 8 == 0:
            w.add(BJ.dense_pairs(45, 1))
        if k % 4 == 1:
            z = np.zeros(64, np.int64); z[0] = 16384 + k; w.add([z])
        w.add(BJ.with_pairs([3 + k % 13], 1))
    # for every s0 & 15: one interval with a pair split across a k_unstuff row edge ((s0 & ~3) + 128 r) -- also a word edge --
    # and one split across a 16-byte load
    for r in range(16):
        start = w.pos + 3 + (r - (w.pos + 3)) % 16
        p1 = (start & ~3) + 127
        p2 = p1 + 6 + (15 - (p1 + 6)) % 16
        w.advance_to(start)
        w.pairs_at([p1, p2], slack=p1 - start)
    return w.finish()


def _mcu_file(rng):
    """DRI 4: blocks ending in +32767 at zig-zag 63 (no EOB behind it), so that the next MCU starts inside or right behind a
    run of ones: MCU starts on the FF of a stuffed pair and on the byte after its 00, in intervals with at most and with
    more than JS_STUFF_LIST stuffed zeros."""
    w = BJ.Writer(dri=4)
    for k in range(600):
        blocks = []
        for b in range(4):
            z = np.zeros(64, np.int64)
            z[0] = int(rng.integers(-40, 41))
            n = int(rng.integers(0, 12))
            z[1:1 + n] = [BJ._low_ones(int(s), int(s) + k) for s in rng.integers(1, 9, n)]
            if rng.random() < 0.7:
                z[63] = 32767
            if rng.random() < 0.1:
                z[1 + n:1 + n + 8] = 32767
            blocks.append(z)
        w.add(blocks)
    return w.finish()


def _long_file():
    """DRI 256 (ri * bpm >= JS_PSYNC_MIN_BLOCKS: the self-synchronising path, k_unstuff_long), four intervals of ~8.8 KB whose
    starts s0 have s0 & 3 = 0, 1, 2, 3.  k_unstuff_long cuts an interval into 4096-byte chunks from s0 - (s0 & 3): each interval
    has stuffed pairs split across both of its chunk edges, in the last and the first 16-byte group of a chunk, and in the
    first group of the interval."""
    w = BJ.Writer(dri=256)
    for r in range(4):
        mis = w.pos & 3
        assert mis == r
        e1, e2 = 4096 - mis, 8192 - mis                       # chunk edges, interval-relative
        length = 8800 + ((r + 1 - (w.pos + 8800 + 2)) % 4)    # the next interval starts at residue r + 1
        w.add(BJ.long_interval([6, e1 - 12, e1 - 1, e1 + 5, e2 - 9, e2 - 1, e2 + 9], 256, length))
    return w.finish()


@functools.lru_cache(maxsize=None)
def corpus():
    """[(name, jpeg, spec, Placed)]: the healthy placed files."""
    rng = np.random.default_rng(20261015)
    return [("edges_dri1",) + _edges_file(), ("dense_dri1",) + _dense_file(), ("mcu_dri4",) + _mcu_file(rng),
            ("long_dri256",) + _long_file()]


@functools.lru_cache(maxsize=None)
def damaged():
    """[(name, jpeg, Placed)]: the edges file with a terminator, a stray marker or fill bytes spliced in on a grid edge."""
    _, j, _, rec = corpus()[0]
    r = rec.rst
    on = lambda m: next(t for t in r if t % m == m - 1 and t > 8192)         # an RST whose FF ends a piece / chunk ...
    out = []
    out.append(("eoi_chunk_end",) + BJ.splice(j, rec, on(4096), b"\xff\xd9"))           # terminator FF on a chunk's last byte
    out.append(("eoi_pass_end",) + BJ.splice(j, rec, on(32768), b"\xff\xd9"))           # ... on a 32 KB pass end
    out.append(("app1_row_end",) + BJ.splice(j, rec, on(512), b"\xff\xe1"))             # stray marker on a 512-byte row end
    out.append(("app1_span_end",) + BJ.splice(j, rec, on(64), b"\xff\xe1"))             # ... on a 64-byte span end
    piece = next(t for t in r if t % 16 == 15 and t % 64 != 63 and t > 8192)
    out.append(("eoi_piece_end",) + BJ.splice(j, rec, piece, b"\xff\xd9"))             # terminator FF on a piece's last byte
    out.append(("app1_piece_end",) + BJ.splice(j, rec, piece, b"\xff\xe1"))            # stray marker on a piece's last byte
    out.append(("fill_piece_edge",) + BJ.splice(j, rec, on(16), b"\xff"))               # FF FF Dn across a piece edge
    t = on(4096)
    out.append(("rst_oos_chunk_end",) + BJ.splice(j, rec, t, bytes([0xFF, 0xD0 + (r.index(t) + 3) % 8])))   # out-of-sequence RST
    out.append(("ff_last_byte", j[:-3] + b"\xff", rec))                                       # no EOI, an FF as the scan's last byte
    return out


def _stuffed(scan, a, b):
    return [i for i in range(a, b - 1) if scan[i] == 0xFF and scan[i + 1] == 0]


def boundary_hits():
    """name -> number of places in the corpus that reach it, computed from the bytes.  Grid edges are taken from each kernel's
    own origin: scan offsets for the marker scans and k_unstuff_lane's 16-byte loads (scans are 16-byte aligned), s0 & ~3 for
    k_unstuff's 128-byte rows, s0 - (s0 & 3) for k_unstuff_long's 4096-byte chunks (s0 = the interval's first byte)."""
    hits = {}
    add = lambda k, n=1: hits.__setitem__(k, hits.get(k, 0) + int(n))
    for name, j, spec, rec in corpus():
        scan = j[rec.scan_start:]
        long_iv = spec["dri"] >= PSYNC_MIN                       # greyscale: ri * bpm = dri
        for t in rec.rst:
            for m, k in ((16, "rst_piece_end"), (64, "rst_span64_end"), (512, "rst_row512_end"), (4096, "rst_chunk_end"), (32768, "rst_pass_end")):
                add(k, t % m == m - 1)
        add("scan_over_128KB", len(scan) > 32 * 4096)
        for (s0, e), (starts, nbits) in zip(rec.intervals, rec.mcu_bits):
            pairs = _stuffed(scan, s0, e)
            if long_iv:
                c0 = s0 - (s0 & 3)
                for p in pairs:
                    add(f"long_pair_split_chunk_mis{s0 & 3}", (p - c0) % 4096 == 4095 and p + 1 < e)
                    add("long_pair_in_first_group", (p - c0) % 4096 < 16 and p - c0 >= 4096)
                    add("long_pair_in_last_group", (p - c0) % 4096 >= 4080)
                continue
            if e - s0 - len(pairs) < 4:
                add("interval_under_4_bytes")
            if nbits % 8 == 0:
                add("interval_consumed_to_last_bit")
            if e > s0 and scan[s0] == 0xFF:
                add("ff_first_byte_of_interval")
            add("stuffed_6", len(pairs) == 6); add("stuffed_7", len(pairs) == 7); add("stuffed_over_40", len(pairs) > 40)
            r = s0 & 15
            for p in pairs:
                add(f"pair_split_word_s0mod16_{r}", p % 4 == 3)
                add(f"pair_split_load16_s0mod16_{r}", p % 16 == 15)
                add(f"pair_split_row128_s0mod16_{r}", (p - (s0 & ~3)) % 128 == 127)
            add("adjacent_pairs", any(b - a == 2 for a, b in zip(pairs, pairs[1:])))
            # MCU starts: unstuffed byte u -> raw; on the FF of a pair, or on the byte after its 00
            form = "overflow" if len(pairs) > STUFF_LIST else "list"
            for m, bit in enumerate(starts):
                if m == 0:
                    continue
                raw = _raw_of(scan, s0, e, bit >> 3)
                add(f"mcu_on_ff_{form}", raw + 1 < e and scan[raw] == 0xFF and scan[raw + 1] == 0)
                add(f"mcu_after_00_{form}", raw - 2 >= s0 and scan[raw - 2] == 0xFF and scan[raw - 1] == 0)
    for name, j, rec in damaged():
        scan = j[rec.scan_start:]
        marks = [(i, scan[i + 1]) for i in range(len(scan) - 1) if scan[i] == 0xFF and scan[i + 1] != 0]
        term = next((i for i, m in marks if not 0xD0 <= m <= 0xD7 and m != 0xFF), None)
        if term is not None and not name.startswith("ff_"):
            for m, k in ((16, "term_piece_end"), (64, "term_span64_end"), (512, "term_row512_end"), (4096, "term_chunk_end"), (32768, "term_pass_end")):
                add(k, term % m == m - 1)
            add("rst_after_term_in_later_chunk", any(0xD0 <= m <= 0xD7 and i // 4096 > term // 4096 for i, m in marks))
        rsts = [i for i, m in marks if 0xD0 <= m <= 0xD7 and (term is None or i < term)]
        add("rst_out_of_sequence_on_chunk_end", any(i % 4096 == 4095 and scan[i + 1] != 0xD0 + k % 8 for k, i in enumerate(rsts)))
        add("fill_ff_ff_dn_across_piece_edge", any(i % 16 == 15 and scan[i + 1] == 0xFF and 0xD0 <= scan[i + 2] <= 0xD7 for i, m in marks if m == 0xFF))
        add("ff_last_byte_of_scan", scan[-1] == 0xFF)
    return hits


def _raw_of(scan, s0, e, u):
    """raw offset of unstuffed byte u of the interval [s0, e)"""
    kept = 0
    for r in range(s0, e):
        if scan[r] == 0 and r > s0 and scan[r - 1] == 0xFF:
            continue
        if kept == u:
            return r
        kept += 1
    return e


REQUIRED = (["rst_piece_end", "rst_span64_end", "rst_row512_end", "rst_chunk_end", "rst_pass_end", "scan_over_128KB",
             "interval_under_4_bytes", "interval_consumed_to_last_bit", "ff_first_byte_of_interval", "stuffed_6", "stuffed_7",
             "stuffed_over_40", "adjacent_pairs", "mcu_on_ff_list", "mcu_on_ff_overflow", "mcu_after_00_list", "mcu_after_00_overflow"]
            + [f"pair_split_{g}_s0mod16_{r}" for g in ("word", "load16", "row128") for r in range(16)]
            + [f"long_pair_split_chunk_mis{m}" for m in range(4)] + ["long_pair_in_first_group", "long_pair_in_last_group"]
            + ["term_piece_end", "term_span64_end", "term_row512_end", "term_chunk_end", "term_pass_end", "rst_after_term_in_later_chunk",
               "rst_out_of_sequence_on_chunk_end", "fill_ff_ff_dn_across_piece_edge", "ff_last_byte_of_scan"])


# --- CPU ---------------------------------------------------------------------------------------------------------------

def test_corpus_reaches_the_boundaries(built):
    hits = boundary_hits()
    print("\n".join(f"{k:32s} {hits.get(k, 0)}" for k in REQUIRED))
    missing = [k for k in REQUIRED if not hits.get(k)]
    assert not missing, missing
    # the record matches the bytes: every placed RST is where the writer said, and the healthy files carry nmcu/dri - 1 RSTs
    for name, j, spec, rec in corpus():
        scan = j[rec.scan_start:]
        assert all(scan[t] == 0xFF and 0xD0 <= scan[t + 1] <= 0xD7 for t in rec.rst), name
        assert rec.nrst == len(rec.intervals) - 1 == spec["blocks"][0].shape[1] * spec["blocks"][0].shape[0] // spec["dri"] - 1, name
    for name, j, rec in damaged():
        for t, data in rec.splices:
            assert j[rec.scan_start + t: rec.scan_start + t + len(data)] == data, name


@needs_ref
def test_reference_decodes_the_placed_corpus(built):
    """No error lines, m_nRestartRead = the placed RSTs, pixels as coef_jpeg.expected restates them."""
    o = Oracle("ref_fixed")
    lf, li = o.idct_tables()
    for name, j, spec, rec in corpus():
        d = o.decode(j)
        assert d.nerr == 0, (name, o.err_lines()[:3])
        assert int(d.stats[10]) == rec.nrst, (name, d.stats)
        bad = JC.compare(CJ.expected(spec, True, li, lf), d, what=("geom", "pix_y", "dib", "blk_dc"))
        assert not bad, (name, bad)


def test_port_matches_the_reference_on_the_placed_corpus(built):
    port = Oracle("port", idct_fixed=True)
    have_ref = ref_available("fixed")
    ref = Oracle("ref_fixed") if have_ref else None
    lf, li = port.idct_tables()
    for name, j, spec, rec in corpus():
        got = port.decode(j)
        assert got.nerr == 0, name
        if have_ref:
            want = ref.decode(j)
            assert not JC.compare(want, got), name
            assert np.array_equal(want.stats, got.stats), (name, want.stats, got.stats)
        else:
            assert not JC.compare(CJ.expected(spec, True, li, lf), got, what=("geom", "pix_y", "dib", "blk_dc")), name


# --- GPU: placed files, every buffer and line ----------------------------------------------------------------------------

def _all_jpegs():
    return [(n, j) for n, j, _, _ in corpus()] + [(n, j) for n, j, _ in damaged()]


@pytest.mark.gpu
@needs_ref
def test_placed_files_match_the_reference_line_for_line(built):
    """Single-image decodes: every buffer, the whole stats row, the whole non-quiet log (scan-position and compression-ratio
    lines included) and, for damaged files, every error line."""
    from jpegsnoop_b200 import CimgDecode
    o = Oracle("ref_fixed")
    dec = CimgDecode(idct_fixedpt=True)
    for name, j in _all_jpegs():
        want = o.decode(j, quiet=False); wl = o.log_lines(); we = o.err_lines()
        got = dec.decode(j, quiet=False)
        bad = JC.compare(want, got, what=WHAT)
        assert not bad, (name, bad)
        assert np.array_equal(np.asarray(want.stats), np.asarray(got.stats)[:12]), (name, want.stats, got.stats)
        gl = dec.log_lines(-1)
        assert gl == wl, (name, [(a, b) for a, b in zip(wl, gl) if a != b][:3], len(wl), len(gl))
        assert dec.log_lines(3) == we, name
    dec.close()


FORMS = [(m, u) for m in (0, 1) for u in (0, 1)]


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("marker,unstuff", FORMS, ids=[f"marker{m}-unstuff{u}" for m, u in FORMS])
def test_forced_forms_match_the_reference(built, tmp_path, marker, unstuff):
    """JSGPU_MARKER x JSGPU_UNSTUFF, each with huff_kernel 0, 1, 2, in a child process: the placed corpus, its damaged
    variants and the parity suite's damaged scans, batched; fetched buffers against the reference, checksums against its
    checksums (healthy files)."""
    import test_gpu_parity as TP
    named = _all_jpegs() + [(k, v[0]) for k, v in TP._damaged_cases(JC.small_cases()).items() if not v[1]]
    src, dst = tmp_path / "in.npz", tmp_path / "out.npz"
    np.savez(src, jpegs=np.array([j for _, j in named], dtype=object))
    env = dict(os.environ, JSGPU_MARKER=str(marker), JSGPU_UNSTUFF=str(unstuff))
    r = subprocess.run([sys.executable, os.path.join(HERE, "stage_a_child.py"), str(src), str(dst), "0", "1", "2"],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(dst)
    o = Oracle("ref_fixed")
    healthy = {n for n, _, _, _ in corpus()}
    _, errs, want_ck = o.bench_ck([j for n, j in named if n in healthy])
    assert errs == 0
    for h in (0, 1, 2):
        ck = got[f"ck_{h}"]
        for k, (name, j) in enumerate(named):
            want = o.decode(j)
            for f in ("pix_y", "dib", "mcu_map", "dht_histo"):
                assert np.array_equal(np.asarray(getattr(want, f)), got[f"{f}_{h}_{k}"]), (name, h, f)
            assert np.array_equal(np.asarray(want.blk_dc[0]), got[f"blk_y_{h}_{k}"]), (name, h)
            # the batch stats row: sum of Y (2 words), m_nAvgY, brightest pixel Y/Cb/Cr/R/G/B, its MCU, m_nRestartRead, ...
            ws, gs = np.asarray(want.stats), got[f"stats_{h}_{k}"]
            assert gs[2] == ws[0] and np.array_equal(gs[3:12], ws[2:11]), (name, h, ws, gs)
        hk = [k for k, (n, _) in enumerate(named) if n in healthy]
        assert np.array_equal(ck[hk], want_ck), h


# --- GPU: both sides of every rule, persistent loops -----------------------------------------------------------------------

def _gray(W, H, dri, seed, q=80):
    return JC.enc(JC.synth_rgb(W, H, seed)[:, :, 0], quality=q, restart_marker_blocks=dri) if dri else \
        JC.enc(JC.synth_rgb(W, H, seed)[:, :, 0], quality=q)


def _nseg(j):
    from jpegsnoop_b200.host import parse_jpeg
    _, d, _ = parse_jpeg(j)
    hm = max(d.samp_h[c] for c in range(d.num_sos_comps)); vm = max(d.samp_v[c] for c in range(d.num_sos_comps))
    if d.num_sos_comps == 1:
        hm = vm = 1
    nmcu = -(-d.dim_x // (8 * hm)) * -(-d.dim_y // (8 * vm))
    ri = d.restart_interval if (d.restart_en and d.restart_interval) else nmcu
    bpm = sum(d.samp_h[c] * d.samp_v[c] for c in range(d.num_sos_comps)) if d.num_sos_comps > 1 else 1
    return -(-nmcu // ri), ri, bpm


def _marker_form(jpegs):
    """js_launch_marker_scan: 'per_image' (k_marker_scan) or 'chunked' (k_marker_scan2)."""
    from jpegsnoop_b200 import BatchDecoder
    _, darr, bits = BatchDecoder.prepare(jpegs)
    n = len(jpegs); mx = max(int(d.scan_length) for d in darr)
    uneven = mx * n > 2 * bits.size
    return "chunked" if (n < 2 * SMS or uneven) else "per_image"


def _check_batch(jpegs, **opts):
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder(**opts)
    bd.set_batch(jpegs); bd.decode(); bd.sync()
    got = bd.checksums(); bd.close()
    uniq, inv = {}, []
    for j in jpegs:
        inv.append(uniq.setdefault(j, len(uniq)))
    _, errs, want = Oracle("ref_fixed").bench_ck(list(uniq), threads=effective_cores()[0])
    assert errs == 0
    want = want[np.array(inv)]
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, [(int(i), np.flatnonzero(got[i] != want[i]).tolist()) for i in bad[:5]]


@functools.lru_cache(maxsize=None)
def _small_set():
    return [_gray(64 + 8 * (k % 4), 48, 1 + k % 3, k) for k in range(8)] + [JC.enc(JC.synth_rgb(48, 32, 40 + k), quality=85, subsampling=2, restart_marker_blocks=2) for k in range(4)]


@pytest.mark.gpu
@needs_ref
def test_marker_scan_threshold(built):
    """263 against 264 images of similar size, and 264 with one large image (uneven)."""
    s = _small_set()
    big = _gray(1024, 512, 4, 99)
    cases = {"n263": [s[k % len(s)] for k in range(2 * SMS - 1)], "n264": [s[k % len(s)] for k in range(2 * SMS)]}
    cases["n264_uneven"] = cases["n264"][:-1] + [big]
    assert [_marker_form(v) for v in cases.values()] == ["chunked", "per_image", "chunked"]
    for v in cases.values():
        _check_batch(v)


@pytest.mark.gpu
@needs_ref
def test_unstuff_threshold_and_persistent_loops(built):
    """max_nseg 255 (k_unstuff) against 256 (k_unstuff_lane), with enough images that k_unstuff's `k += kstep` and
    k_unstuff_lane's k0 loop take a second turn."""
    a = [_gray(8 * 255, 8, 1, k) for k in range(4)]
    b = [_gray(8 * 256, 8, 1, k) for k in range(4)]
    assert max(_nseg(j)[0] for j in a) == 255 and max(_nseg(j)[0] for j in b) == 256
    # k_unstuff: grid.x = min(ceil(max_nseg / 4), ceil(SMS*16*8 / nimg)), four warps per CTA, kstep = 4 * grid.x
    batch = [a[k % 4] for k in range(300)]
    gx = min(-(-255 // 4), -(-SMS * 16 * 8 // len(batch)))
    assert 4 * gx < 255
    _check_batch(batch)
    # k_unstuff_lane: grid.x = min(ceil(max_nseg / 256), ceil(SMS*8*4 / nimg)), 256 intervals per CTA and turn
    c = [_gray(512, 512, 1, k) for k in range(2)]
    batch = [c[k % 2] for k in range(290)] + b
    gx = min(-(-4096 // 256), -(-SMS * 8 * 4 // len(batch)))
    assert _nseg(c[0])[0] == 4096 and 256 * gx < 4096
    _check_batch(batch)


@pytest.mark.gpu
@needs_ref
def test_huffman_auto_and_selfsync_thresholds(built):
    """4095 against 4096 short intervals per batch (huff_kernel auto), ri*bpm 191 against 192 (self-synchronising path)."""
    base = [_gray(8 * 255, 8, 1, k) for k in range(16)]
    for tail_mcus, n in ((15, 4095), (16, 4096)):
        batch = base + [_gray(8 * tail_mcus, 8, 1, 50)]
        assert sum(_nseg(j)[0] for j in batch) == n
        _check_batch(batch)
    for dri in (PSYNC_MIN - 1, PSYNC_MIN):
        j = _gray(1536, 64, dri, 60 + dri)
        nseg, ri, bpm = _nseg(j)
        assert ri * bpm == dri
        _check_batch([j, _gray(1536, 64, dri, 61 + dri), base[0]])


@pytest.mark.gpu
@needs_ref
def test_long_unstuff_and_marker_ticket_loops(built):
    """16 no-DRI 4K images (more than 8 * SMS * 8 chunks: k_marker_scan2's ticket loop wraps) next to 60 tiny ones
    (k_unstuff_long's grid shrinks to ceil(SMS*8*4 / nimg) CTAs per image: its cs loop takes a second turn)."""
    from jpegsnoop_b200 import BatchDecoder
    big = [JC.enc(JC.synth_rgb(3840, 2160, 41 + k % 2), quality=85, subsampling=2) for k in range(2)]
    tiny = _small_set()
    batch = [big[k % 2] for k in range(16)] + [tiny[k % len(tiny)] for k in range(60)]
    _, darr, _ = BatchDecoder.prepare(batch)
    chunks = sum(max(1, -(-int(d.scan_length) // 4096)) for d in darr)
    assert chunks > 8 * SMS * 8
    n = len(batch)
    cs = max((int(d.scan_length) >> 12) + 2 * 1 + 2 for d in darr[:16])
    gx = min(-(-cs // 8), -(-SMS * 8 * 4 // n))
    assert 8 * gx < cs
    assert _nseg(big[0])[1] >= PSYNC_MIN
    _check_batch(batch)


# --- GPU: more than 65,535 images ------------------------------------------------------------------------------------------

@pytest.mark.gpu
@needs_ref
def test_batch_of_65537_images(built):
    """grid.y is limited to 65,535: the per-image kernels stride over blockIdx.y.  One batch of 65,537 tiny images (16x16
    4:2:0 and 8x8 grey, eight distinct files cycled), decoded with MCU maps, then with the simple IDCT kernels, then
    recoloured by jsgpu_batch_preview with a non-default mode and the histograms on."""
    from jpegsnoop_b200 import BatchDecoder
    from jpegsnoop_b200 import _lib as B
    files = [JC.enc(JC.synth_rgb(16, 16, k), quality=70 + k, subsampling=2, **({"restart_marker_blocks": 1} if k % 2 else {})) for k in range(4)]
    files += [JC.enc(JC.synth_rgb(8, 8, 10 + k)[:, :, 0], quality=60 + 5 * k) for k in range(4)]
    N, U = 65537, len(files)
    tarr, darr, bits = BatchDecoder.prepare(files)
    reps = -(-N // U)
    sz = ctypes.sizeof(B.jsgpu_image_desc)
    raw = np.frombuffer(bytes(darr), np.uint8).reshape(U, sz)
    big = np.tile(raw, (reps, 1))[:N].copy()
    off = B.jsgpu_image_desc.scan_offset.offset
    so = big[:, off:off + 8].copy().view(np.uint64).ravel() + np.repeat(np.arange(reps, dtype=np.uint64) * np.uint64(bits.size), U)[:N]
    big[:, off:off + 8] = so.view(np.uint8).reshape(N, 8)
    dbig = (B.jsgpu_image_desc * N).from_buffer_copy(big.tobytes())
    bbig = np.tile(bits, reps)
    o = Oracle("ref_fixed")
    _, errs, want = o.bench_ck(files)
    assert errs == 0
    pick = sorted({0, N - 3, N - 2, N - 1} | set(np.random.default_rng(5).integers(0, N, 24).tolist()))
    bd = BatchDecoder()
    bd.set_tables(tarr); bd.plan(dbig, bbig.size); bd.upload(bbig)
    for idct in (0, 1):
        bd.set_options(idct_kernel=idct)
        bd.decode(); bd.sync()
        ck = bd.checksums()
        for i in pick:
            assert np.array_equal(ck[i], want[i % U]), (idct, i, ck[i], want[i % U])
    bd.preview(mode=2, hist_en=1, statclip_en=1)
    bd.sync()
    o.config_histo(True, True, False)
    try:
        for i in pick[:4] + pick[-4:]:
            w = o.decode(files[i % U]); ws = o.colour_stats()
            s = bd.colour_stats(i)
            assert np.array_equal(ws["clip"], np.array(s.clip[:], np.uint32)), i
            assert np.array_equal(ws["y_histo"], np.array(s.y_histo[:], np.uint32)), i
            assert ws["count"] == s.count, i
            o.set_preview_mode(2)
            assert np.array_equal(o.bitmap(), bd.fetch(i).dib), i
            o.set_preview_mode(1)
    finally:
        o.config_histo(False, False, False)
    bd.close()
