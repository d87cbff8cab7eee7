"""Host model of k_unstuff_lane's per-lane arithmetic (jsgpu_huff.cu) against a byte-by-byte unstuffing: the stuffed-zero nibble,
the big-endian PRMT packing, the 64-bit shift register, the 0xFF pad and the stuffed-byte list.  Run: python tools/models/unstuff_lane_model.py"""
import random

M32 = 0xFFFFFFFF


def popc(x): return bin(x).count("1")


def byte_perm(a, b, sel):
    by = [(a >> (8 * i)) & 0xFF for i in range(4)] + [(b >> (8 * i)) & 0xFF for i in range(4)]
    r = 0
    for i in range(4):
        r |= by[(sel >> (4 * i)) & 7] << (8 * i)
    return r


def us_selector(rm, big_endian):
    sel = 0; n = 0
    for i in range(4):
        j = 3 - i if big_endian else i
        if not (rm >> j) & 1:
            sel |= j << (4 * n); n += 1
    for n in range(n, 4):
        sel |= 4 << (4 * n)
    return sel


SELBE = [us_selector(t, True) for t in range(16)]


def us_classify(prev, word, rel0, length):
    vlo = max(0, -rel0); vhi = min(4, length - rel0)
    vn = (((1 << vhi) - 1) & ~((1 << vlo) - 1)) & 15 if vhi > vlo else 0
    an = (vn & ~(1 << (-rel0))) if (rel0 <= 0 and rel0 > -4) else vn
    pw = byte_perm(prev, word, 0x6543); npw = (~pw) & M32
    z = (~((((word & 0x7F7F7F7F) + 0x7F7F7F7F) | word | 0x7F7F7F7F))) & M32
    f = (~((((npw & 0x7F7F7F7F) + 0x7F7F7F7F) | npw | 0x7F7F7F7F))) & M32
    dn = (((((z & f) >> 7) * 0x00204081) & M32) >> 21) & an
    return dn, dn | (vn ^ 15)


def lane_unstuff(buf, s0, length):
    mis = s0 & 15; base = s0 - mis
    nwords = (mis + length + 3) >> 2
    acc = 0; nacc = 0; wr = 0; nstuff = 0; prevw = 0; out = []; stuff = []
    for j in range(nwords):
        word = int.from_bytes(bytes(buf[base + 4 * j + i] if base + 4 * j + i < len(buf) else 0 for i in range(4)), "little")
        dn, rm = us_classify(prevw, word, 4 * j - mis, length)
        cnt = 4 - popc(rm)
        d = dn
        while d:
            jj = (d & -d).bit_length() - 1; d &= d - 1
            if nstuff < 6:
                stuff.append(wr + popc((~rm) & ((1 << jj) - 1)) - 1)
            nstuff += 1
        acc = ((acc << (8 * cnt)) | byte_perm(word, 0, SELBE[rm])) & 0xFFFFFFFFFFFFFFFF
        nacc += cnt; wr += cnt
        if nacc >= 4:
            out.append((acc >> (8 * (nacc - 4))) & M32); nacc -= 4
        prevw = word
    total = ((wr + 16 + 15) & ~15) >> 2; pad = 16
    while len(out) < total:
        n = min(4, pad); v = M32 if n == 4 else (0 if n == 0 else (M32 << (8 * (4 - n))) & M32); pad -= n
        acc = ((acc << 32) | v) & 0xFFFFFFFFFFFFFFFF; nacc += 4
        out.append((acc >> (8 * (nacc - 4))) & M32); nacc -= 4
    return out, wr, nstuff, stuff


def ref_unstuff(buf, s0, length):
    seg = buf[s0:s0 + length]; o = []; stuff = []; n = 0
    for i, x in enumerate(seg):
        if i >= 1 and x == 0 and seg[i - 1] == 0xFF:
            if n < 6:
                stuff.append(len(o) - 1)
            n += 1; continue
        o.append(x)
    wr = len(o); by = o + [0xFF] * 16
    while len(by) % 16:
        by.append(0)
    return [int.from_bytes(bytes(by[i:i + 4]), "big") for i in range(0, len(by), 4)], wr, n, stuff


if __name__ == "__main__":
    random.seed(1); bad = 0
    for t in range(40000):
        n = random.randint(80, 240)
        buf = [random.choice([0, 0xFF, 0xFF, 0, random.randint(0, 255), random.randint(0, 255)]) for _ in range(n)]
        s0 = random.randint(0, 40); length = random.choice([0, 1, 2, 3, 4, 5, random.randint(0, n - s0)])
        if lane_unstuff(buf, s0, length) != ref_unstuff(buf, s0, length):
            bad += 1
    print("mismatches:", bad)
