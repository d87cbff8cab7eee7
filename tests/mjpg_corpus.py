"""TEST INFRASTRUCTURE: Motion-JPEG frames, a minimal RIFF/AVI writer and the containers tests/test_decode_all.py decodes.

Frames are Pillow JPEGs made with libjpeg's default tables, which are the T.81 Annex K ones; to_mjpg turns one into an
MJPG frame the way AVI writers store them: the JFIF APP0 replaced by an "AVI1" APP0, the DHT segments left out.
"""
import struct

import numpy as np

import jpeg_cases as JC

SOI3 = b"\xff\xd8\xff"


def segments(j):
    """[(marker, start, end)] of the segments before the first SOS (end: one past the segment)."""
    out, p = [], 2
    while p + 4 <= len(j):
        m = j[p + 1]
        L = j[p + 2] << 8 | j[p + 3]
        out.append((m, p, p + 2 + L))
        if m == 0xDA:
            break
        p += 2 + L
    return out


def app0(ident):
    body = ident + bytes(max(0, 14 - len(ident)))
    return b"\xff\xe0" + struct.pack(">H", len(body) + 2) + body


def to_mjpg(j, keep_dht=False, ident=b"AVI1\x00"):
    """The frame with its JFIF APP0 replaced by an APP0 carrying `ident` and, unless keep_dht, no DHT segment."""
    parts = [j[:2], app0(ident)]
    segs = segments(j)
    for m, a, e in segs:
        if m == 0xE0 or (m == 0xC4 and not keep_dht):
            continue
        parts.append(j[a:e])
    parts.append(j[segs[-1][2]:])
    return b"".join(parts)


def frame(seed, kind):
    """One Pillow JPEG of the corpus: kind is '420', '422', '444', 'gray', each optionally with '_dri' or '_opt'."""
    rng = np.random.default_rng(seed)
    w, h = int(rng.integers(2, 7)) * 16 + int(rng.integers(0, 16)), int(rng.integers(2, 5)) * 16 + int(rng.integers(0, 16))
    img = JC.synth_rgb(w, h, seed)
    kw = {"quality": int(rng.integers(60, 95))}
    if kind.startswith("gray"):
        img = img[:, :, 0]
    else:
        kw["subsampling"] = {"444": 0, "422": 1, "420": 2}[kind[:3]]
    if "_dri" in kind:
        kw["restart_marker_blocks"] = int(rng.integers(1, 5))
    if "_opt" in kind:
        kw["optimize"] = True
    return JC.enc(img, **kw)


KINDS = ("420", "422", "444", "gray", "420_dri", "422_dri", "444_dri", "gray_dri")


def mjpg_frames(seed, count):
    """`count` MJPG frames cycling through every layout, with and without DRI; every fifth keeps its own optimised DHT."""
    out = []
    for k in range(count):
        if k % 5 == 4:
            out.append(to_mjpg(frame(seed * 1000 + k, KINDS[k % len(KINDS)] + "_opt"), keep_dht=True))
        else:
            out.append(to_mjpg(frame(seed * 1000 + k, KINDS[k % len(KINDS)])))
    return out


def _chunk(fourcc, data):
    return fourcc + struct.pack("<I", len(data)) + data + (b"\x00" if len(data) & 1 else b"")


def _list(kind, *chunks):
    body = kind + b"".join(chunks)
    return b"LIST" + struct.pack("<I", len(body)) + body


def avi(frames, width=64, height=48):
    """A minimal RIFF AVI: hdrl (avih, one video strl with strh/strf), movi with one '00dc' chunk per frame, idx1.
    Returns (bytes, [offset of each frame's SOI])."""
    n = len(frames)
    avih = struct.pack("<10I4I", 40000, 0, 0, 0x10, n, 0, 1, max(len(f) for f in frames), width, height, 0, 0, 0, 0)
    strh = b"vidsMJPG" + struct.pack("<IHHIIIIIIIIhhhh", 0, 0, 0, 0, 1, 25, 0, n, max(len(f) for f in frames), 0xFFFFFFFF, 0,
                                     0, 0, width, height)
    strf = struct.pack("<IiiHH4sIiiII", 40, width, height, 1, 24, b"MJPG", width * height * 3, 0, 0, 0, 0)
    hdrl = _list(b"hdrl", _chunk(b"avih", avih), _list(b"strl", _chunk(b"strh", strh), _chunk(b"strf", strf)))
    movi_start = 12 + len(hdrl) + 8                          # 'RIFF' size 'AVI ' hdrl, then 'LIST' size
    body, offs, idx = b"movi", [], []
    for f in frames:
        idx.append(struct.pack("<4sIII", b"00dc", 0x10, len(body), len(f)))
        offs.append(movi_start + len(body) + 8)
        body += _chunk(b"00dc", f)
    movi = b"LIST" + struct.pack("<I", len(body)) + body
    riff = b"AVI " + hdrl + movi + _chunk(b"idx1", b"".join(idx))
    return b"RIFF" + struct.pack("<I", len(riff)) + riff, offs


def exif_jpeg(seed):
    """A camera-style JPEG: an APP1 Exif segment whose IFD1 carries a JPEG thumbnail, then the main image.
    Returns (bytes, offset of the thumbnail's SOI)."""
    main = frame(seed, "420_dri")
    thumb = frame(seed + 1, "420")
    # TIFF header, IFD0 with no entries, IFD1 with JPEGInterchangeFormat / ...Length, then the thumbnail
    ifd1 = 8 + 2 + 4
    tiff = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<HI", 0, ifd1)
    tiff += struct.pack("<H", 2) + struct.pack("<HHII", 0x0201, 4, 1, ifd1 + 2 + 24 + 4) + struct.pack("<HHII", 0x0202, 4, 1, len(thumb))
    tiff += struct.pack("<I", 0) + thumb
    body = b"Exif\x00\x00" + tiff
    app1 = b"\xff\xe1" + struct.pack(">H", len(body) + 2) + body
    j = main[:2] + app1 + main[2:]
    return j, 2 + 4 + 6 + ifd1 + 2 + 24 + 4


def scan_end_marker(data, start):
    """Where a scan that starts at `start` meets its terminating marker: the first FF followed by neither 00 nor an RST
    (None when the data ends first)."""
    d = np.frombuffer(data, np.uint8)
    ff = np.flatnonzero(d[start:-1] == 0xFF) + start
    nxt = d[ff + 1]
    hit = ff[(nxt != 0) & ((nxt < 0xD0) | (nxt > 0xD7)) & (nxt != 0xFF)]
    return int(hit[0]) if hit.size else None


def find_all_model(data, value=0xFFD8FF, length=3):
    """Every p in [0, n - length] whose big-endian `length` bytes equal `value`."""
    d = np.frombuffer(bytes(data), np.uint8) if not isinstance(data, np.ndarray) else data
    if d.size < length:
        return np.zeros(0, np.int64)
    v = np.zeros(d.size - length + 1, np.uint64)
    for i in range(length):
        v = (v << np.uint64(8)) | d[i:d.size - length + 1 + i].astype(np.uint64)
    return np.flatnonzero(v == np.uint64(value))


def _scan_start(j):
    return segments(j)[-1][2]


def damaged(j, seed):
    """The frame with six bytes of its scan flipped."""
    b = bytearray(j)
    s = _scan_start(j)
    for p in np.random.default_rng(seed).integers(s + 10, len(j) - 20, 6):
        b[p] ^= 0x5A
    return bytes(b)


def corpus():
    """(name, container bytes) for decode_all: MJPG AVIs, damaged frames, an Exif thumbnail, junk with stray and overlapping
    SOIs, and the junk containers of the image-search tests."""
    from test_image_search import container
    rng = np.random.default_rng(77)
    out = [("avi", avi(mjpg_frames(1, 12))[0])]
    f = mjpg_frames(2, 6)
    trunc = f[1][:_scan_start(f[1]) + (len(f[1]) - _scan_start(f[1])) // 2]
    out.append(("avi_damaged", avi([f[0], damaged(f[2], 5), f[3][:-2], f[4]])[0]))
    out.append(("truncated_into_next_soi", f[0] + trunc + f[2] + f[5][:-2]))
    ex, _ = exif_jpeg(9)
    out.append(("exif", ex + rng.integers(0, 256, 300, dtype=np.uint8).tobytes() + f[3]))
    junk = rng.integers(0, 256, 2000, dtype=np.uint8).tobytes()
    out.append(("stray_sois", junk[:500] + SOI3 + junk[500:900] + b"\xff\xd8\xff\xd8\xff" + junk[900:1200] + f[4]
                + junk[1200:] + f[0] + b"\x11\xff\xd8\xff"))
    for seed in (1, 2, 3):
        out.append((f"junk{seed}", container(seed, lead=0 if seed == 2 else None)[0]))
    return out
