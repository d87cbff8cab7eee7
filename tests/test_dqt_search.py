"""Tools -> Search Executable for DQT on the GPU (jsgpu_search_bytes, jsimg_search_dqt, CimgDecode.search_dqt).

CPU: the reporting rule below equals the reference's repeated BufSearchX loop (tests/dqt_oracle.py) on a seeded corpus;
the restated Doc loop writes the lines of every quirk; without a device the tool fails loudly.
GPU: every corpus file's report equals the reference's line for line and kind for kind; large, dense and unaligned
inputs equal the rule; the 2^32-byte limit; a resident decoded batch is left alone.
"""
import numpy as np
import pytest

import jpeg_cases as JC
import dqt_oracle as D

STD_LUM = [16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
           18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99]
ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
          35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]
WINDOW = 131072                                   # the reference's window size (WindowBuf.h: MAX_BUF_WINDOW)


def rule_positions(data, pat):
    """What the reference's loop reports: every byte-exact match p with 1 <= p <= N - 2L + 2 whose p - 1 was not reported
    (in a run of consecutive matches: the first, the third, ...)."""
    d = data if isinstance(data, np.ndarray) else np.frombuffer(bytes(data), np.uint8)
    p = np.frombuffer(bytes(pat), np.uint8)
    L, last = p.size, d.size - 2 * p.size + 2
    if last < 1:
        return np.zeros(0, np.int64)
    cand = np.flatnonzero(d[1:last + 1] == p[0]) + 1
    for j in range(1, L):
        cand = cand[d[cand + j] == p[j]]
    if cand.size == 0:
        return cand
    idx = np.arange(cand.size)
    start = np.maximum.accumulate(np.where(np.r_[True, np.diff(cand) != 1], idx, 0))
    return cand[(idx - start) % 2 == 0]


def all_forms(tbl):
    """The 20 search patterns of a table: 2 orderings x 5 layouts, baseline and not."""
    out = []
    for zz in range(2):
        vals = [tbl[k if zz else ZIGZAG[k]] for k in range(64)]
        for w, sw in D.LAYOUTS:
            out.append(D.dqt_pattern(vals, w, sw, True))
            if w > 1:
                out.append(D.dqt_pattern(vals, w, sw, False))
    return out


def q75_table():
    return [max(1, (v * 50 + 50) // 100) for v in STD_LUM]


def corpus():
    """(name, data, pattern): seeded files on a 4-letter alphabet (dense partial matches) with planted copies."""
    rng = np.random.default_rng(20261016)
    cases = []
    for L in (8, 64, 128, 256):
        pat = bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), L))
        noise = lambda n: rng.choice(np.frombuffer(b"ACGT", np.uint8), n).astype(np.uint8)
        cases += [(f"empty_L{L}", b"", pat), (f"one_L{L}", b"A", pat), (f"short_L{L}", pat[:-1], pat), (f"exact_L{L}", pat, pat)]
        for N in (3 * L, 4 * L + 17, 5000):
            if N < 2 * L + 4:
                continue
            for at in (0, 1, N - 2 * L + 1, N - 2 * L + 2, N - 2 * L + 3, N - L):
                d = noise(N); d[at:at + L] = np.frombuffer(pat, np.uint8)
                cases.append((f"edge_L{L}_N{N}_at{at}", d.tobytes(), pat))
        # overlapping copies of a periodic pattern, copies exactly L apart, and a constant pattern over a zero run
        per = (pat[:3] * L)[:L]
        d = noise(20000); d[100:100 + 3 * L] = np.frombuffer((per * 4)[:3 * L], np.uint8)
        cases.append((f"periodic_L{L}", d.tobytes(), per))
        d = noise(20000); d[500:500 + 4 * L] = np.frombuffer(pat * 4, np.uint8)
        cases.append((f"adjacent_L{L}", d.tobytes(), pat))
        d = noise(20000); d[300:300 + 5 * L] = 0
        cases.append((f"zeros_L{L}", d.tobytes(), bytes(L)))
        # partial matches that rewind across the 128 KiB window reload, and full copies straddling it
        d = noise(3 * WINDOW + 1000)
        for k, at in enumerate((WINDOW - L // 2, 2 * WINDOW - 3, WINDOW - 5)):
            d[at:at + L] = np.frombuffer(pat, np.uint8)
            if k == 2:
                d[at + L - 2] ^= 1                             # a partial match over the boundary
        cases.append((f"window_L{L}", d.tobytes(), pat))
    # the 20 forms of the standard table and of a q75 table, planted in both orderings, with truncated copies
    for name, tbl in (("std", STD_LUM), ("q75", q75_table())):
        for i, pat in enumerate(all_forms(tbl)):
            d = rng.integers(0, 256, 6000).astype(np.uint8)
            d[777:777 + len(pat)] = np.frombuffer(pat, np.uint8)
            d[3000:3000 + len(pat) - 1] = np.frombuffer(pat[:-1], np.uint8)
            d[6000 - 2 * len(pat) + 2:6000 - len(pat) + 2] = np.frombuffer(pat, np.uint8)
            cases.append((f"form_{name}_{i}", d.tobytes(), pat))
    return cases


def make_jpeg(tables, base=None):
    """A Pillow JPEG whose DQT segments are replaced by `tables` {Tq: 64 natural-order values} (16-bit when any is > 255)."""
    j = base or JC.enc(JC.synth_rgb(48, 32, 3), quality=80)
    out, p = bytearray(j[:2]), 2
    for tq, tbl in tables.items():
        pq = int(max(tbl) > 255)
        body = bytes([(pq << 4) | tq]) + b"".join(int(tbl[ZIGZAG[k]]).to_bytes(2 if pq else 1, "big") for k in range(64))
        out += b"\xff\xdb" + (len(body) + 2).to_bytes(2, "big") + body
    while p < len(j):
        m, L = j[p + 1], int.from_bytes(j[p + 2:p + 4], "big")
        if m == 0xDA:
            out += j[p:]
            break
        if m != 0xDB:
            out += j[p:p + 2 + L]
        p += 2 + L
    return bytes(out)


def harness_cases():
    """(name, analysed JPEG or None, file): the four quirks and an ordinary analysed table."""
    rng = np.random.default_rng(7)
    q75 = q75_table()
    big0 = list(q75); big0[0] = 0x1234                    # only entry 0 above 255: still baseline
    bigac = list(q75); bigac[9] = 300                     # a large AC entry: 1-byte searches skipped for both sets
    const = [5] * 64
    cases = []
    for name, tables in (("standard_only", None), ("q75", {0: q75, 1: STD_LUM}), ("entry0_16bit", {0: big0}),
                         ("ac_16bit", {0: bigac}), ("constant", {0: const}), ("no_table0", {1: q75})):
        jp = None if tables is None else make_jpeg(tables)
        tbl = q75 if tables is None or 0 not in tables else tables[0]
        d = rng.integers(0, 256, 40000).astype(np.uint8)
        at = 1000
        for pat in all_forms(STD_LUM) + all_forms(tbl):
            if at + len(pat) > d.size - 600:
                break
            d[at:at + len(pat)] = np.frombuffer(pat, np.uint8); at += len(pat) + 37
        if name == "q75":
            d[40000 - 64:] = np.frombuffer(bytes(all_forms(STD_LUM)[0]), np.uint8)        # past the reference's reach
        cases.append((name, jp, d.tobytes()))
    return cases


ref = pytest.mark.skipif(not D.ref_available(), reason="compiled reference (oracle/_ref) not built")


# ---------------------------------------------------------------------------------------------------------------- CPU
@ref
def test_rule_equals_reference_loop(built):
    n = 0
    for name, data, pat in corpus():
        want = D.ref_bufsearch_all(data, pat)
        got = rule_positions(data, pat).tolist()
        assert got == want, name
        n += len(want)
    assert n > 100


@ref
def test_reference_lines_cover_the_quirks(built):
    got = {name: D.ref_search_dqt(data, "/fw/cam.bin", jp, "/img/a.jpg") for name, jp, data in harness_cases()}
    text = {k: [s for _, s in v] for k, v in got.items()}
    for k, v in got.items():
        assert v[0] == ("hdr", "*** Searching Executable for DQT ***") and v[-1] == ("line", "  Done Search"), k
        assert ("line", "  Size:     [40000]") in v
    assert not any("Matching [/img/a.jpg]" in s for s in text["standard_only"])
    assert sum(s.startswith("      Matching [") for s in text["standard_only"]) == 2
    assert sum(s == "      Matching [/img/a.jpg]" for s in text["q75"]) == 2
    assert sum(k == "good" for k, _ in got["q75"]) >= 20                  # 5 layouts x 2 orderings x 2 tables
    assert "          DQT Table is not baseline, skipping 1-byte search" not in text["entry0_16bit"]
    assert sum(s == "          DQT Table is not baseline, skipping 1-byte search" for s in text["ac_16bit"]) == 4
    note = "  NOTE: Because the JPEG's DQT Luminance table is constant nValue (0x05),_T("
    assert [s for k, s in got["constant"] if k == "warn"] == [note, ")        matching for this table has been disabled.",
                                                             "        Please select a different reference image."]
    assert [s for k, s in got["no_table0"] if k == "warn"][0].endswith("(0x00),_T(")
    assert not any("Matching [/img/a.jpg]" in s for s in text["constant"] + text["no_table0"])
    # the rule gives the same lines
    for name, jp, data in harness_cases():
        assert D.ref_search_dqt(data, "x", jp, "y", search=lambda d, p: rule_positions(d, p).tolist()) == \
            D.ref_search_dqt(data, "x", jp, "y"), name


def _no_gpu():
    try:
        import torch
        return not torch.cuda.is_available()
    except Exception:
        return True


@pytest.mark.skipif(not _no_gpu(), reason="only meaningful without a GPU")
def test_search_fails_loudly_without_gpu(built):
    from jpegsnoop_b200 import CimgDecode, JsgpuError
    dec = CimgDecode()
    with pytest.raises(JsgpuError):
        dec.search_dqt(bytes(4096), "/fw/cam.bin")
    lines = dec.log_lines()
    assert len(dec.log_lines(3)) == 1 and "GPU search unavailable" in dec.log_lines(3)[0]
    assert not any("Found @" in s or s == "  Done Search" for s in lines)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@ref
def test_gpu_report_equals_reference(built):
    from jpegsnoop_b200 import CimgDecode
    for name, jp, data in harness_cases():
        dec = CimgDecode()
        if jp is not None:
            dec.walk(jp)
        dec.L.jsimg_log_clear(dec.h)
        found = dec.search_dqt(data, "/fw/cam.bin", analysed=jp is not None, analysed_path="/img/a.jpg")
        want = D.ref_search_dqt(data, "/fw/cam.bin", jp, "/img/a.jpg")
        assert dec.log_lines() == [s for _, s in want], name
        for kind, label in ((1, "hdr"), (2, "warn"), (3, "err"), (4, "good")):
            assert dec.log_lines(kind) == [s for k, s in want if k == label], (name, label)
        assert sum(len(v) for v in found.values()) == sum(k == "good" for k, _ in want), name


@pytest.mark.gpu
def test_gpu_report_equals_rule(built):
    """The report's positions against the rule, with the tables restated here (no compiled reference needed)."""
    from jpegsnoop_b200 import CimgDecode
    for name, jp, data in harness_cases():
        if name not in ("standard_only", "q75", "ac_16bit"):
            continue
        dec = CimgDecode()
        tables = [STD_LUM]
        if jp is not None:
            dec.walk(jp)
            tables.append([dec.GetDqtEntry(0, i) for i in range(64)])
        found = dec.search_dqt(data, "f", analysed=jp is not None, analysed_path="a")
        baseline = max(tables[-1][1:]) <= 255
        keys = []
        for zz in range(2):
            for s, tbl in enumerate(tables):
                vals = [tbl[k if zz else ZIGZAG[k]] for k in range(64)]
                for lay, (w, sw) in enumerate(D.LAYOUTS):
                    if w == 1 and not baseline:
                        continue
                    keys.append((zz, s, lay))
                    assert found[(zz, s, lay)] == rule_positions(data, D.dqt_pattern(vals, w, sw, baseline)).tolist(), (name, zz, s, lay)
        assert sorted(found) == sorted(keys), name
        assert sum(map(len, found.values())) >= 10, name


@pytest.mark.gpu
def test_gpu_corpus_equals_rule(built):
    from jpegsnoop_b200 import BatchDecoder
    bd = BatchDecoder()
    for name, data, pat in corpus():
        if len(pat) < 8:
            continue
        counts, pos = bd.search_bytes(data, [pat])
        want = rule_positions(data, pat)
        assert int(counts[0]) == want.size and np.array_equal(pos[0], want), name


def _planted_file(n, pats, rng, chunk):
    """Random bytes with patterns planted across every chunk edge (one byte before, on, after it, and ending on it),
    across CTA tile edges, at the last reportable offset and one byte either side of it."""
    d = rng.integers(0, 256, n, dtype=np.uint8)
    L = len(pats[0])
    spots = [c * chunk + (-1, 0, 1, -L)[c % 4] for c in range(1, n // chunk + 1)]
    spots += [4096 - 1, 6 * 4096, 9 * 4096 + 1, 12 * 4096 - L]
    for i, s in enumerate(spots):
        p = pats[i % len(pats)]
        d[s:s + len(p)] = np.frombuffer(p, np.uint8)
    d[n - 2 * L + 1:n - L + 1] = np.frombuffer(pats[0], np.uint8)
    return d, spots + [n - 2 * L + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [None, 1 << 20])
def test_gpu_large_files_equal_rule(built, chunk, monkeypatch):
    from jpegsnoop_b200 import BatchDecoder
    if chunk:
        monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", str(chunk))
    size = chunk or (64 << 20)
    n = (4 if chunk else 2) * size + size // 2 + 12345
    rng = np.random.default_rng(5)
    pats = [all_forms(STD_LUM)[i] for i in (0, 1, 5)] + [all_forms(q75_table())[i] for i in (0, 2, 7)]
    d, spots = _planted_file(n, pats, rng, size)
    want = [rule_positions(d, p) for p in pats]
    reported = set(np.concatenate(want).tolist())
    assert {s for s in spots if s <= n - 2 * len(pats[0]) + 2} <= reported and n - 2 * len(pats[0]) + 1 in reported
    bd = BatchDecoder()
    for shift in (0, 3):                                       # an unaligned host buffer
        buf = np.zeros(n + 16, np.uint8)[shift:shift + n]
        buf[:] = d
        counts, pos = bd.search_bytes(buf, pats)
        for k in range(len(pats)):
            assert int(counts[k]) == want[k].size and np.array_equal(pos[k], want[k]), (k, shift)


@pytest.mark.gpu
def test_gpu_dense_matches_and_cap(built, monkeypatch):
    from jpegsnoop_b200 import BatchDecoder
    monkeypatch.setenv("JSGPU_SEARCH_CHUNK_BYTES", str(1 << 20))
    rng = np.random.default_rng(11)
    n = 9 << 20
    d = np.zeros(n, np.uint8)
    for a, b in ((4 << 20, (4 << 20) + 777), ((6 << 20) + 5, (6 << 20) + 6)):   # breaks in the zero run
        d[a:b] = rng.integers(1, 256, b - a)
    pats = [bytes(64), bytes(8), bytes([0] * 63 + [1])]
    bd = BatchDecoder()
    counts, pos = bd.search_bytes(d, pats)
    for k, p in enumerate(pats):
        want = rule_positions(d, p)
        assert int(counts[k]) == want.size and np.array_equal(pos[k], want), k
    assert int(counts[0]) > 10 ** 6 // 2 and int(counts[0]) + int(counts[1]) > 10 ** 6
    # a small cap: complete counts, the first cap positions in order
    cap = int(counts[0]) + 1000
    c2, p2 = bd.search_bytes(d, pats, cap=cap)
    assert np.array_equal(c2, counts) and np.array_equal(p2[0], pos[0]) and np.array_equal(p2[1], pos[1][:1000]) and p2[2].size == 0


@pytest.mark.gpu
def test_gpu_size_limit(built):
    from jpegsnoop_b200 import BatchDecoder, CimgDecode, JsgpuError
    big = np.zeros(1 << 32, np.uint8)                          # pages never touched
    bd = BatchDecoder()
    with pytest.raises(JsgpuError):
        bd.search_bytes(big, [bytes(64)], cap=16)
    dec = CimgDecode()
    with pytest.raises(JsgpuError):
        dec.search_dqt(big, "/disk.img")
    assert len(dec.log_lines(3)) == 1 and not any("Found @" in s for s in dec.log_lines())


@pytest.mark.gpu
def test_gpu_search_leaves_the_batch_alone(built):
    from jpegsnoop_b200 import BatchDecoder
    jpegs = [JC.enc(JC.synth_rgb(320, 240, s), quality=85, subsampling=2) for s in range(3)]
    bd = BatchDecoder()
    bd.set_batch(jpegs); bd.decode(); bd.sync()
    before = bd.checksums()
    data = np.frombuffer(b"".join(jpegs) * 50, np.uint8)
    counts, pos = bd.search_bytes(data, [bytes(all_forms(STD_LUM)[0])])
    assert np.array_equal(pos[0], rule_positions(data, all_forms(STD_LUM)[0]))
    assert np.array_equal(bd.checksums(), before)
