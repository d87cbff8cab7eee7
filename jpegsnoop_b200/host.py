"""Python faces of the host API.

* `CimgDecode`   — one-image drop-in: mirrors the reference class's method names 1:1 over the C
                   shim (include/jsimg.h), so parity tests read like calls on the reference class.
* `BatchDecoder` — many images per call through the C-ABI (include/jsgpu.h): the form the
                   bench and the multi-GPU path use.
Neither contains decode logic; both fail loudly when libjsgpu.so or a CUDA device is missing.
"""
import ctypes as C
import numpy as np
from . import _lib as B


class JsgpuError(RuntimeError):
    pass


class DecodedImage:
    """numpy copies of everything DecodeScanImg leaves behind (same fields as tests/oracle_util.Decoded)."""
    def __init__(self):
        self.geom = None; self.pix_y = self.pix_cb = self.pix_cr = None; self.dib = None
        self.mcu_map = None; self.blk_dc = None; self.dht_histo = None; self.stats = None
        self.nerr = 0; self.scan_start = 0; self.status = 0; self.stage_ms = None; self.pos = 0


class CimgDecode:
    """Mirror of the reference class (source/ImgDecode.h:284-425) driven through jsimg_*."""

    def __init__(self, decode_ac=True, idct_fixedpt=True, device=0, huff_kernel=0, idct_kernel=0):
        self.L = B.load()
        self.h = C.c_void_p(self.L.jsimg_create())
        self.L.jsimg_config(self.h, int(decode_ac), int(idct_fixedpt), device, huff_kernel, idct_kernel, 1)
        self._file = None
        self.reprocessed = None

    def close(self):
        if self.h:
            self.L.jsimg_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- byte source -------------------------------------------------------------------------
    def set_file(self, data):
        self._file = np.frombuffer(bytes(data), np.uint8).copy()
        self.L.jsimg_set_file(self.h, self._file.ctypes.data, self._file.size)

    # --- the reference's method names --------------------------------------------------------
    def Reset(self): self.L.jsimg_Reset(self.h)
    def ResetState(self): self.L.jsimg_ResetState(self.h)
    def SetDqtEntry(self, t, i, izz, v): return bool(self.L.jsimg_SetDqtEntry(self.h, t, i, izz, v))
    def SetDqtTables(self, comp, t): return bool(self.L.jsimg_SetDqtTables(self.h, comp, t))
    def GetDqtEntry(self, t, i): return int(self.L.jsimg_GetDqtEntry(self.h, t, i))
    def SetDhtTables(self, comp, dc, ac): return bool(self.L.jsimg_SetDhtTables(self.h, comp, dc, ac))
    def SetDhtEntry(self, dest, cls, ind, length, bits, mask, code):
        return bool(self.L.jsimg_SetDhtEntry(self.h, dest, cls, ind, length, bits & 0xFFFFFFFF, mask & 0xFFFFFFFF, code))
    def SetDhtSize(self, dest, cls, n): return bool(self.L.jsimg_SetDhtSize(self.h, dest, cls, n))
    def SetPrecision(self, p): self.L.jsimg_SetPrecision(self.h, p)
    def SetSofSampFactors(self, comp, h, v): self.L.jsimg_SetSofSampFactors(self.h, comp, h, v)
    def SetImageDetails(self, x, y, nf, ns, rst_en, ri): self.L.jsimg_SetImageDetails(self.h, x, y, nf, ns, int(rst_en), ri)
    def DecodeScanImg(self, start, bDisplay=True, bQuiet=True): self.L.jsimg_DecodeScanImg(self.h, start, int(bDisplay), int(bQuiet))
    def IsPreviewReady(self): return bool(self.L.jsimg_IsPreviewReady(self.h))

    def GetImageSize(self):
        x, y = C.c_uint32(), C.c_uint32(); self.L.jsimg_GetImageSize(self.h, C.byref(x), C.byref(y)); return x.value, y.value

    def LookupFilePosMcu(self, mx, my):
        a, b = C.c_uint32(), C.c_uint32(); self.L.jsimg_LookupFilePosMcu(self.h, mx, my, C.byref(a), C.byref(b)); return a.value, b.value

    def LookupFilePosPix(self, px, py):
        a, b = C.c_uint32(), C.c_uint32(); self.L.jsimg_LookupFilePosPix(self.h, px, py, C.byref(a), C.byref(b)); return a.value, b.value

    def LookupBlkYCC(self, bx, by):
        y, cb, cr = C.c_int(), C.c_int(), C.c_int()
        self.L.jsimg_LookupBlkYCC(self.h, bx, by, C.byref(y), C.byref(cb), C.byref(cr)); return y.value, cb.value, cr.value

    # --- channel preview, colour statistics, histograms (ImgDecode.cpp:631-677, 3764-4012) -------
    def config_histo(self, histo_en=False, statclip_en=False, dump_histo_y=False):
        self.L.jsimg_config_histo(self.h, int(histo_en), int(statclip_en), int(dump_histo_y))

    def config_scan_err_max(self, n):
        """CSnoopConfig::nErrMaxDecodeScan: how many of each capped scan error line a decode reports (0: none; default 20)."""
        self.L.jsimg_config_scan_err_max(self.h, n)

    def ScanErrorsDisable(self): self.L.jsimg_ScanErrorsDisable(self.h)
    def ScanErrorsEnable(self): self.L.jsimg_ScanErrorsEnable(self.h)

    def SetPreviewMode(self, mode): self.L.jsimg_SetPreviewMode(self.h, mode)
    def GetPreviewMode(self): return int(self.L.jsimg_GetPreviewMode(self.h))
    def SetPreviewYccOffset(self, mx, my, y, cb, cr): self.L.jsimg_SetPreviewYccOffset(self.h, mx, my, y, cb, cr)

    def GetPreviewYccOffset(self):
        mx, my = C.c_uint32(), C.c_uint32(); y, cb, cr = C.c_int(), C.c_int(), C.c_int()
        self.L.jsimg_GetPreviewYccOffset(self.h, C.byref(mx), C.byref(my), C.byref(y), C.byref(cb), C.byref(cr))
        return mx.value, my.value, y.value, cb.value, cr.value

    def colour_stats(self):
        """m_sStatClip [12], m_sHisto ([36] min/max/sum in PixelCcHisto order, nCount), m_anCcHisto_r/g/b [3][128], m_anHistoYFull [2048]."""
        clip = np.zeros(12, np.uint32); self.L.jsimg_GetStatClip(self.h, clip.ctypes.data)
        rng = np.zeros(36, np.int32); n = C.c_uint32(); self.L.jsimg_GetHistoRanges(self.h, rng.ctypes.data, C.byref(n))
        cc = np.zeros((3, 128), np.uint32)
        for c in range(3):
            self.L.jsimg_GetCcHisto(self.h, c, cc[c].ctypes.data)
        yh = np.zeros(2048, np.uint32); self.L.jsimg_GetHistoYFull(self.h, yh.ctypes.data)
        return {"clip": clip, "ranges": rng, "count": int(n.value), "cc_histo": cc, "y_histo": yh}

    def histo_dib(self, which):
        """The histogram bitmap DrawHistogram painted (0: R/G/B 128x90, 1: Y 512x30), or None when it is not ready."""
        ready = C.c_int(0); p = self.L.jsimg_GetHistoDib(self.h, which, C.byref(ready))
        if not ready.value or not p:
            return None
        shape = (30, 512, 4) if which else (90, 128, 4)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=shape).copy()

    def SetDetailVlc(self, detail, x=0, y=0, n=1): self.L.jsimg_SetDetailVlc(self.h, int(detail), x, y, n)

    def ExportTiff(self, path, mode=0):
        """Export-to-TIFF of the decoded image (mode 0 RGB 8-bit, 1 RGB 16-bit, 2 YCC 8-bit), JPEGsnoopDoc.cpp:2008-2193."""
        return bool(self.L.jsimg_ExportTiff(self.h, str(path).encode(), mode))

    def search_dqt(self, data, exe_path, analysed=False, analysed_path=""):
        """Tools -> Search Executable for DQT over `data` (JPEGsnoopDoc.cpp:1233-1529), on the GPU.  With `analysed`, this
        decoder's table 0 (from the last walk/decode) is searched next to the JPEG standard's.  The report goes to the log
        (log_lines()); returns {(ordering, set, layout): [positions]} for every search the report lists: ordering 0
        pre-zigzag / 1 post-zigzag, set 0 the standard table / 1 the analysed one, layout 0..4 = 1-byte, 2-byte,
        2-byte swapped, 4-byte, 4-byte swapped (a skipped 1-byte search is absent).  Raises JsgpuError on failure."""
        buf = np.frombuffer(data, np.uint8) if isinstance(data, np.ndarray) else np.frombuffer(bytes(data), np.uint8)
        n0 = self.L.jsimg_log_count(self.h, -1)
        r = self.L.jsimg_search_dqt(self.h, buf.ctypes.data, buf.size, str(exe_path).encode(), int(analysed), str(analysed_path).encode())
        lines = self.log_lines()[n0:]
        if r != 0:
            raise JsgpuError(f"jsimg_search_dqt failed ({r}): {lines}")
        found, key, zz, ts = {}, None, -1, -1
        for s in lines:
            if s.startswith("    DQT Ordering: "):
                zz += 1; ts = -1
            elif s.startswith("      Matching ["):
                ts += 1
            elif s.startswith("        Searching patterns with "):
                w = int(s.split("with ")[1].split("-byte")[0]); swap = s.endswith("byteswap")
                key = (zz, ts, {1: 0, 2: 1, 4: 3}[w] + int(swap)); found[key] = []
            elif s.startswith("          DQT Table is not baseline"):
                del found[key]
            elif s.startswith("          Found @ 0x"):
                found[key].append(int(s.split("0x")[1], 16))
        return found

    def bitmap(self):
        g = np.zeros(8, np.uint32); self.L.jsimg_GetGeometry(self.h, g.ctypes.data)
        p = self.L.jsimg_GetBitmapPtr(self.h)
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(int(g[7]), int(g[6]), 4)).copy() if p else None

    def log_lines(self, kind=-1):
        n = self.L.jsimg_log_count(self.h, kind)
        return [self.L.jsimg_log_line(self.h, kind, i).decode() for i in range(n)]

    def num_err_lines(self): return self.L.jsimg_log_count(self.h, 3)

    def idct_tables(self):
        lf = np.zeros((64, 64), np.float32); li = np.zeros((64, 64), np.int32)
        self.L.jsimg_GetIdctTables(self.h, lf.ctypes.data, li.ctypes.data); return lf, li

    # --- convenience ---------------------------------------------------------------------------
    def walk(self, jpeg_bytes):
        self.set_file(jpeg_bytes)
        return self.L.jsimg_walk_jpeg(self.h, self._file.ctypes.data, self._file.size)

    def collect(self):
        """Copy out everything the getters expose after DecodeScanImg."""
        d = DecodedImage()
        g = np.zeros(8, np.uint32); self.L.jsimg_GetGeometry(self.h, g.ctypes.data); d.geom = g
        Wp, Hp = int(g[6]), int(g[7]); nblk = int(g[4]) * int(g[5]); nmcu = int(g[2]) * int(g[3])

        def arr(ptr, ctype, shape):
            if not ptr:
                return None
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape=shape).copy()
        py, pcb, pcr = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self.L.jsimg_GetPixMapPtrs(self.h, C.byref(py), C.byref(pcb), C.byref(pcr))
        d.pix_y = arr(py.value, C.c_int16, (Hp, Wp)); d.pix_cb = arr(pcb.value, C.c_int16, (Hp, Wp)); d.pix_cr = arr(pcr.value, C.c_int16, (Hp, Wp))
        d.dib = arr(self.L.jsimg_GetBitmapPtr(self.h), C.c_uint8, (Hp, Wp, 4))
        d.mcu_map = arr(self.L.jsimg_GetMcuFileMap(self.h), C.c_uint32, (nmcu,))
        d.blk_dc = tuple(arr(self.L.jsimg_GetBlkDcMap(self.h, c), C.c_int16, (nblk,)) for c in range(3))
        h = np.zeros((2, 4, 17), np.uint32); self.L.jsimg_GetDhtHisto(self.h, h.ctypes.data); d.dht_histo = h
        s = np.zeros(12, np.int32); self.L.jsimg_GetStats(self.h, s.ctypes.data); d.stats = s
        ms = np.zeros(5, np.float32); self.L.jsimg_GetStageMs(self.h, ms.ctypes.data); d.stage_ms = ms
        d.nerr = self.num_err_lines(); d.status = int(self.L.jsimg_GetScanStatus(self.h))
        return d

    def decode(self, jpeg_bytes, quiet=True, offset=0, mode=None):
        """Marker walk (CjfifDecode's setter sequence) from the SOI at `offset`, then DecodeScanImg(start, True, quiet).
        With `mode` (B.OFFSET_START / SRCH1 / SRCH2 / POS, DoAnalyzeOffset's modes) the offset is chosen as the reference's
        command line does; `offset` is then the position of OFFSET_POS.  Every position is absolute in `jpeg_bytes`;
        d.pos is the offset decoded at."""
        self.set_file(jpeg_bytes)
        self.L.jsimg_log_clear(self.h)
        if mode is None:
            r = self.L.jsimg_decode_jpeg_at(self.h, self._file.ctypes.data, self._file.size, offset, int(quiet))
            pos = offset
        else:
            used = C.c_uint64(0)
            r = self.L.jsimg_decode_offset_mode(self.h, self._file.ctypes.data, self._file.size, mode, offset, int(quiet), C.byref(used))
            pos = used.value
        if r < 0:
            raise ValueError(f"marker walk failed ({r}) at offset {pos}: {self.log_lines(3)}")
        d = self.collect(); d.scan_start = r; d.pos = pos
        return d

    def buf_search(self, start, value, length, forward=True):
        """CwindowBuf::BufSearch over the file set last and its overlays, on the GPU: (found, position)."""
        p = C.c_uint64(0)
        r = self.L.jsimg_buf_search(self.h, start, value, length, int(forward), C.byref(p))
        if r < 0:
            raise JsgpuError(f"jsimg_buf_search failed ({r}): {self.log_lines(3)}")
        return bool(r), p.value

    def export_jpeg(self, data, out_path, offset=0, overlay=False, force_soi=False, force_eoi=False, ignore_eoi=False,
                    dht_avi_insert=False, overlays=(), src_name="input.bin"):
        """Tools -> Extract embedded JPEG (JPEGsnoopCore.cpp:913-961): the frame at `offset` of `data` (bytes or a uint8 array)
        walked to its EOI, its scans skipped on the GPU, written to out_path as ExportJpegPrepare / ExportJpegDo write it.
        `overlays` [(start, bytes), ...] are installed for the walk; `overlay` copies the bytes through them too.  src_name is
        the source file's name (the log names it, and an out_path equal to it is refused).  Returns (written, the export's
        log lines); raises JsgpuError when the GPU search fails."""
        return self._export(data, overlays, lambda f: self.L.jsimg_export_jpeg(self.h, offset, str(src_name).encode(),
                                                                                str(out_path).encode(), f),
                            overlay, force_soi, force_eoi, ignore_eoi, dht_avi_insert)

    def _export(self, data, overlays, run, *opts):
        self._file = _u8(data)
        self.L.jsimg_set_file(self.h, self._file.ctypes.data, self._file.size)
        self.L.jsimg_overlay_remove_all(self.h)
        keep = [np.frombuffer(bytes(b), np.uint8) for _, b in overlays]
        for (o, _), a in zip(overlays, keep):
            self.L.jsimg_overlay_install(self.h, int(o), a.ctypes.data, a.size)
        self.L.jsimg_log_clear(self.h)
        flags = sum(1 << k for k, v in enumerate(opts) if v)
        try:
            r = run(flags)
        finally:
            self.L.jsimg_overlay_remove_all(self.h)
        lines = self.log_lines()
        if r < 0 and not (r == -2 and lines and lines[-1].startswith("ERROR: Invalid filename")):
            raise JsgpuError(f"export failed ({r}): {lines[-3:]}")
        return r, lines

    def _img_search(self, start, forward, quiet):
        found, pos, decoded = C.c_int(0), C.c_uint64(0), C.c_int(0)
        self.L.jsimg_log_clear(self.h)
        r = self.L.jsimg_img_search(self.h, start, int(forward), int(quiet), C.byref(found), C.byref(pos), C.byref(decoded))
        if r < 0 and not decoded.value:
            raise JsgpuError(f"jsimg_img_search failed ({r}): {self.log_lines(3)}")
        # the scan start of the reprocessed image (negative: its marker walk failed), or None when nothing was reprocessed
        self.reprocessed = r if decoded.value else None
        return bool(found.value), pos.value

    def search_forward(self, start, quiet=False):
        """Tools -> Img Search Fwd from `start` over the file set last (JPEGsnoopDoc.cpp:828-873): (found, new start).  A match
        is reprocessed (self.reprocessed is its scan start; collect() returns its outputs); otherwise nothing changes.  The
        reprocess writes the scan-decode lines the reference's Reprocess writes (DecodeScanImg with bQuiet false)."""
        return self._img_search(start, True, quiet)

    def search_reverse(self, start, quiet=False):
        """Tools -> Img Search Rev (JPEGsnoopDoc.cpp:878-932): (found, new start).  From start > 0 a match is reprocessed, and
        without one the file is reprocessed from 0; from start 0 nothing happens (self.reprocessed is None)."""
        return self._img_search(start, False, quiet)


def _u8(data):
    """`data` as a uint8 array, without a copy where it already is one (bytes are viewed in place)."""
    if isinstance(data, np.ndarray) and data.dtype == np.uint8 and data.ndim == 1 and data.flags.c_contiguous:
        return data
    return np.frombuffer(bytes(data), np.uint8)


def walk_jpeg(jpeg_bytes, offset=0):
    """Marker walk from the SOI at `offset` -> (jsgpu_tables, jsgpu_image_desc, scan start, or the walk's negative error code)."""
    buf = _u8(jpeg_bytes)
    t = B.jsgpu_tables(); d = B.jsgpu_image_desc()
    r = B.load().jsimg_parse_jpeg_at(buf.ctypes.data, buf.size, offset, C.byref(t), C.byref(d))
    return t, d, r


def parse_jpeg(jpeg_bytes, offset=0):
    """Marker walk only, from the SOI at `offset` -> (jsgpu_tables, jsgpu_image_desc, scan_start); the scan start and
    desc.file_pos are absolute offsets in `jpeg_bytes`."""
    t, d, r = walk_jpeg(jpeg_bytes, offset)
    if r < 0:
        raise ValueError(f"marker walk failed ({r}) at offset {offset}")
    return t, d, r


SOI3 = 0xFFD8FF
WINDOW_SLACK = 64     # bytes a scan window reads past the next SOI candidate; an accepted scan ends at least this far inside it


def plan_windows(data, candidates):
    """The first pass of BatchDecoder.decode_all: for every SOI candidate p (ascending) -> (p, scan start or the walk's error
    code, window end w).  A walked image reads [scan start, w), w = min(n, q + WINDOW_SLACK) with q the first candidate past
    its scan start (FF D8 is a marker, so a healthy scan ends by q); w is None for a failed walk."""
    buf = _u8(data)
    cands = np.asarray(candidates, np.int64)
    out = []
    for p in cands.tolist():
        _, _, r = walk_jpeg(buf, p)
        if r < 0:
            out.append((p, r, None))
            continue
        k = int(np.searchsorted(cands, r, side="right"))
        out.append((p, r, buf.size if k == cands.size else min(buf.size, int(cands[k]) + WINDOW_SLACK)))
    return out


def tables_key(t):
    return bytes(t)


class BatchDecoder:
    """Batch decode through the C-ABI.  Typical use:
        bd = BatchDecoder(device=0)
        bd.set_batch(list_of_jpeg_bytes)       # parse, dedupe tables, plan, upload bitstream
        bd.decode(); bd.sync()
        img = bd.fetch(i)                      # numpy copies of image i's outputs
    """

    def __init__(self, device=0, idct_fixedpt=True, decode_ac=True, huff_kernel=0, idct_kernel=0,
                 want_histo=True, want_mcu_map=True):
        self.L = B.load()
        ctx = C.c_void_p()
        r = self.L.jsgpu_init(device, C.byref(ctx))
        if r != 0:
            raise JsgpuError(f"jsgpu_init failed: {self.L.jsgpu_strerror(r).decode()} (no CPU fallback)")
        self.ctx = ctx
        self.device = device
        # IDCT tables come from the host class (PrecalcIdct on the host libm)
        h = C.c_void_p(self.L.jsimg_create())
        lf = np.zeros((64, 64), np.float32); li = np.zeros((64, 64), np.int32)
        self.L.jsimg_GetIdctTables(h, lf.ctypes.data, li.ctypes.data)
        self.L.jsimg_destroy(h)
        self.idct_lf, self.idct_li = lf, li
        self._ck(self.L.jsgpu_set_idct_tables(self.ctx, li.ctypes.data, lf.ctypes.data))
        self.opt = B.jsgpu_options(idct_mode=0 if idct_fixedpt else 1, decode_ac=int(decode_ac), huff_kernel=huff_kernel,
                                   idct_kernel=idct_kernel, want_histo=int(want_histo), want_mcu_map=int(want_mcu_map),
                                   scan_err_max=20)
        self._ck(self.L.jsgpu_set_options(self.ctx, C.byref(self.opt)))
        self.n = 0; self.layout = None; self.descs = None; self.bitstream = None; self.nsof_pixels = 0
        self._jsimg = None                    # extract_all's host walker and log, made on first use

    def _ck(self, r):
        if r != 0:
            raise JsgpuError(f"{self.L.jsgpu_strerror(r).decode()}: {self.L.jsgpu_last_error(self.ctx).decode()}")

    def close(self):
        if self._jsimg is not None:
            self._jsimg.close(); self._jsimg = None
        if self.ctx:
            self.L.jsgpu_free(self.ctx); self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_options(self, **kw):
        for k, v in kw.items():
            setattr(self.opt, k, int(v))
        self._ck(self.L.jsgpu_set_options(self.ctx, C.byref(self.opt)))

    @staticmethod
    def prepare(jpegs):
        """Host-side preparation: marker walk of every JPEG, table-set dedupe, concatenation of the
        scan bytes.  Returns (table_sets array, descs array, bitstream uint8 array).  An entry may be a
        (file bytes, offset) pair: the JPEG whose SOI is at that offset, decoded as CimgDecode.decode(offset=...)
        decodes it (its scan runs to the end of the file, and its MCU file map holds absolute positions).
        An (file bytes, offset, length) triple reads the file as if it ended at offset + length: only the scan bytes
        before that point are copied, and positions stay absolute."""
        sets, keys, descs, chunks, off = [], {}, [], [], 0
        for j in jpegs:
            j, at, *length = j if isinstance(j, tuple) else (j, 0)
            j = _u8(j)
            if length:
                j = j[:at + length[0]]
            t, d, start = parse_jpeg(j, at)
            k = tables_key(t)
            if k not in keys:
                keys[k] = len(sets); sets.append(t)
            d.table_set = keys[k]
            scan = j[start:]
            d.scan_offset = off; d.scan_length = scan.size; d.file_pos = start
            chunks.append(scan); off += (scan.size + 15) // 16 * 16
            descs.append(d)
        bits = np.zeros(off, np.uint8)
        for d, c in zip(descs, chunks):
            bits[d.scan_offset:d.scan_offset + c.size] = c
        tarr = (B.jsgpu_tables * len(sets))(*sets)
        darr = (B.jsgpu_image_desc * len(descs))(*descs)
        return tarr, darr, bits

    def set_tables(self, tarr):
        self._tables = tarr
        self._ck(self.L.jsgpu_upload_tables(self.ctx, C.byref(tarr), len(tarr)))

    def plan(self, darr, bitstream_bytes):
        self.descs = darr; self.n = len(darr)
        self._ck(self.L.jsgpu_batch_begin(self.ctx, C.byref(darr), self.n, bitstream_bytes))
        self.layout = (B.jsgpu_image_layout * self.n)()
        self._ck(self.L.jsgpu_batch_layout(self.ctx, C.byref(self.layout), self.n))
        self.nsof_pixels = sum(int(d.dim_x) * int(d.dim_y) for d in darr)
        self.npadded_pixels = sum(int(l.img_x) * int(l.img_y) for l in self.layout)

    def upload(self, bits):
        self.bitstream = bits
        self._ck(self.L.jsgpu_batch_upload(self.ctx, bits.ctypes.data, bits.size))

    def set_batch(self, jpegs):
        tarr, darr, bits = self.prepare(jpegs)
        self.set_tables(tarr); self.plan(darr, bits.size); self.upload(bits)

    def decode(self): self._ck(self.L.jsgpu_batch_decode(self.ctx))
    def sync(self): self._ck(self.L.jsgpu_sync(self.ctx))
    def stream(self): return self.L.jsgpu_stream(self.ctx)
    def launches(self): return int(self.L.jsgpu_batch_launches(self.ctx))

    def host_copy_rate(self, direction=1, nbytes=1 << 30, reps=3):
        """GB/s of a plain cudaMemcpyAsync between pinned host memory and this GPU (1 = device->host)."""
        g = C.c_float(0); self._ck(self.L.jsgpu_host_copy_rate(self.ctx, direction, nbytes, reps, C.byref(g))); return float(g.value)

    def search_bytes(self, data, patterns, cap=None):
        """jsgpu_search_bytes: every position the reference's repeated BufSearchX loop reports for each pattern (8..256 bytes,
        at most 32) in `data` (bytes or a uint8 array).  Returns (counts uint64 [npat], [positions uint32 array per pattern]);
        with `cap`, at most cap positions are returned in all (counts stay complete)."""
        buf = _u8(data)
        pats = [np.frombuffer(bytes(p), np.uint8) for p in patterns]
        cat = np.concatenate(pats) if pats else np.zeros(0, np.uint8)
        lens = np.array([p.size for p in pats], np.uint32)
        counts = np.zeros(len(pats), np.uint64)
        if cap is None:                       # count first, then fetch everything
            self._ck(self.L.jsgpu_search_bytes(self.ctx, buf.ctypes.data, buf.size, cat.ctypes.data, lens.ctypes.data, len(pats),
                                               counts.ctypes.data, None, 0))
            cap = int(counts.sum())
        pos = np.zeros(max(int(cap), 1), np.uint32)
        self._ck(self.L.jsgpu_search_bytes(self.ctx, buf.ctypes.data, buf.size, cat.ctypes.data, lens.ctypes.data, len(pats),
                                           counts.ctypes.data, pos.ctypes.data, int(cap)))
        first = np.concatenate([[0], np.cumsum(counts.astype(np.int64))])
        return counts, [pos[min(first[k], cap):min(first[k + 1], cap)].copy() for k in range(len(pats))]

    def find_value(self, data, start, value, length, forward=True, overlays=()):
        """jsgpu_find_value: what CwindowBuf::BufSearch(start, value, length, forward) returns over `data` (bytes or a uint8
        array) with `overlays` [(start, bytes), ...] applied, the last one winning: (found, position)."""
        buf = _u8(data)
        keep = [np.frombuffer(bytes(b), np.uint8) for _, b in overlays]
        ov = (B.jsgpu_overlay * max(len(keep), 1))(*[B.jsgpu_overlay(int(o), a.size, a.ctypes.data) for (o, _), a in zip(overlays, keep)])
        found, pos = C.c_int(0), C.c_uint64(0)
        self._ck(self.L.jsgpu_find_value(self.ctx, buf.ctypes.data, buf.size, start, value, length, int(forward), ov, len(keep),
                                         C.byref(found), C.byref(pos)))
        return bool(found.value), pos.value

    def find_all(self, data, value=SOI3, length=3, cap=None):
        """jsgpu_find_all: every position of the big-endian `length`-byte `value` in `data` (bytes or a uint8 array), overlapping
        ones included -> (count, positions uint32 ascending).  With `cap`, at most cap positions are returned (count stays
        complete); without it, all of them (a second pass runs only when there are more than one per 2 KiB of file)."""
        buf = _u8(data)
        count = C.c_uint64(0)
        want = cap if cap is not None else buf.size // 2048 + 1024
        pos = np.zeros(max(int(want), 1), np.uint32)
        self._ck(self.L.jsgpu_find_all(self.ctx, buf.ctypes.data, buf.size, value, length, C.byref(count), pos.ctypes.data, int(want)))
        if cap is None and count.value > want:
            want = count.value; pos = np.zeros(want, np.uint32)
            self._ck(self.L.jsgpu_find_all(self.ctx, buf.ctypes.data, buf.size, value, length, C.byref(count), pos.ctypes.data, want))
        return int(count.value), pos[:min(int(count.value), int(want))]

    def extract_all(self, data, out_name, overlay=False, force_soi=False, force_eoi=False, ignore_eoi=False,
                    dht_avi_insert=False, overlays=(), src_name="input.bin"):
        """Extract All (JPEGsnoopCore.cpp:963-1088; the command line's -ext_all): every frame from offset 0 and from each FF D8 FF
        after the last start, written to root.000001.jpg, root.000002.jpg, ... (root: out_name up to its last '.').  The search
        runs on this context; a resident batch is left untouched.  Options as CimgDecode.export_jpeg.  Returns
        ([(offset, path or None)] per frame analysed, the export log lines); with no '.' in out_name, ([], the error line)."""
        if self._jsimg is None:
            self._jsimg = CimgDecode(device=self.device)
        d = self._jsimg
        want = _u8(data).size // 4096 + 1024          # frames analysed: one more than the FF D8 FF after offset 0
        offs = np.zeros(want, np.uint64); nums = np.zeros(want, np.uint32)

        def run(flags):
            nonlocal offs, nums
            a = (C.c_char_p(str(src_name).encode()), C.c_char_p(str(out_name).encode()), flags)
            k = self.L.jsimg_extract_all(d.h, self.ctx, *a, offs.ctypes.data, nums.ctypes.data, offs.size)
            if k > offs.size:                         # more frames than the guess holds: run again with room for all
                d.L.jsimg_log_clear(d.h)
                offs = np.zeros(k, np.uint64); nums = np.zeros(k, np.uint32)
                k = self.L.jsimg_extract_all(d.h, self.ctx, *a, offs.ctypes.data, nums.ctypes.data, k)
            offs, nums = offs[:max(k, 0)], nums[:max(k, 0)]
            return k

        r, lines = d._export(data, overlays, run, overlay, force_soi, force_eoi, ignore_eoi, dht_avi_insert)
        if r < 0:
            return [], lines
        root = str(out_name)[:str(out_name).rfind(".")]
        return [(int(o), f"{root}.{int(m):06d}.jpg" if m else None) for o, m in zip(offs, nums)], lines

    def decode_all(self, data, redo_budget=1 << 30):
        """Every JPEG in `data` in one batch: the SOI candidates of find_all(), each walked from its offset, each walked image
        decoded from a window of its scan (plan_windows), so that a file of K images uploads about its own size rather than
        K times it.  An image keeps its windowed outputs when its window runs to the end of the file, or when it decoded
        without error and the marker ending its scan lies at least WINDOW_SLACK bytes inside the window; every other image is
        decoded again from its scan start to the end of the file, as the reference reads a damaged scan on through markers,
        in batches of at most `redo_budget` scan bytes (an image longer than that alone).
        Returns ([(offset, scan start or the walk's error code, DecodedImage or None)] in file order,
                 {"redone": images decoded again, "uploaded": bitstream bytes uploaded in all}).
        Every image equals CimgDecode.decode(data, offset=p) but for nerr: positions absolute, status included."""
        buf = _u8(data)
        n = buf.size
        _, cands = self.find_all(buf)
        plan = plan_windows(buf, cands)
        imgs = [None] * len(plan)
        walked = [k for k, (_, r, _) in enumerate(plan) if r >= 0]
        uploaded = 0

        def run(entries, ks, accept):
            nonlocal uploaded
            tarr, darr, bits = self.prepare(entries)
            self.set_tables(tarr); self.plan(darr, bits.size); self.upload(bits); self.decode(); self.sync()
            uploaded += bits.size
            self.refresh_layout()
            for i, k in enumerate(ks):
                d = self.fetch(i, refresh=False)
                d.pos, d.scan_start = plan[k][0], plan[k][1]
                if accept(d, plan[k][2]):
                    imgs[k] = d

        if walked:
            run([(buf, plan[k][0], plan[k][2] - plan[k][0]) for k in walked], walked,
                lambda d, w: w == n or (d.status == 0 and d.scan_start <= (int(d.stats[14]) & 0xFFFFFFFF) <= w - WINDOW_SLACK))
        redo = [k for k in walked if imgs[k] is None]
        group, size = [], 0
        for k in redo + [None]:
            tail = None if k is None else n - plan[k][1]
            if group and (k is None or size + tail > redo_budget):
                run([(buf, plan[g][0]) for g in group], group, lambda d, w: True)
                group, size = [], 0
            if k is not None:
                group.append(k); size += tail
        return [(p, r, imgs[k]) for k, (p, r, _) in enumerate(plan)], {"redone": len(redo), "uploaded": uploaded}

    def scan_errors(self, i):
        """jsgpu_scan_errors of image i (only for images whose status carries JSGPU_ST_EXACT = 0x40000000)."""
        e = B.jsgpu_scan_errors(); self._ck(self.L.jsgpu_batch_errors(self.ctx, i, C.byref(e))); return e

    def scan_error_events(self, i):
        """Every error event of image i (jsgpu_batch_error_events), not only the first 256: uint32 [nevents, 8] with the
        columns of jsgpu_scan_event (code, a, b, c, d, e, pad0, pad1)."""
        n = int(self.scan_errors(i).nevents)
        ev = np.zeros((n, 8), np.uint32)
        self._ck(self.L.jsgpu_batch_error_events(self.ctx, i, 0, n, ev.ctypes.data)); return ev

    def checksums(self):
        """uint64 [n][12]: device-side checksums of every output buffer of every image (include/jsgpu.h)."""
        a = np.zeros((self.n, 12), np.uint64); self._ck(self.L.jsgpu_batch_checksums(self.ctx, a.ctypes.data, self.n)); return a

    def set_preview(self, **kw):
        """jsgpu_set_preview: hist_en, statclip_en, mode, shift_y/cb/cr, shift_mcu_x/y, ycc_warn_budget (default 10)."""
        p = B.jsgpu_preview(); p.mode = 1; p.ycc_warn_budget = 10
        for k, v in kw.items():
            setattr(p, k, v)
        self._ck(self.L.jsgpu_set_preview(self.ctx, C.byref(p)))

    def preview(self, **kw):
        """jsgpu_batch_preview: recolour the current batch's DIBs with these settings."""
        p = B.jsgpu_preview(); p.mode = 1; p.ycc_warn_budget = 10
        for k, v in kw.items():
            setattr(p, k, v)
        self._ck(self.L.jsgpu_batch_preview(self.ctx, C.byref(p)))

    def colour_stats(self, i):
        s = B.jsgpu_colour_stats(); self._ck(self.L.jsgpu_batch_colour_stats(self.ctx, i, C.byref(s))); return s

    def export(self, i, mode=0):
        """jsgpu_batch_export: the top-down 3-samples-per-pixel array of image i (uint8; RGB16 as big-endian byte pairs)."""
        lo = self.layout[i]
        out = np.zeros(int(lo.img_x) * int(lo.img_y) * (6 if mode == 1 else 3), np.uint8)
        self._ck(self.L.jsgpu_batch_export(self.ctx, i, mode, out.ctypes.data, out.size)); return out

    def selfsync_info(self):
        """(images on the self-synchronising path, slots, [slots changed in fix round 1, 2, ...])"""
        a = np.zeros(16, np.uint32); self._ck(self.L.jsgpu_batch_selfsync_info(self.ctx, a.ctypes.data, 16))
        return int(a[0]), int(a[1]), [int(v) for v in a[3:3 + int(a[2])]]

    def set_detail(self, image, x=0, y=0, n=1, enable=True):
        """jsgpu_set_detail: the next decode also reports the "Detailed Decode" of `n` MCUs of image `image` from MCU (x, y)."""
        d = B.jsgpu_detail(enable=int(enable), image=image, mcu_x=x, mcu_y=y, len=n)
        self._ck(self.L.jsgpu_set_detail(self.ctx, C.byref(d)))

    def detail_info(self):
        """(events, blocks, path) of the last decode's detailed decode; path is B.DETAIL_SERIAL or B.DETAIL_PARALLEL."""
        a = np.zeros(4, np.uint32); self._ck(self.L.jsgpu_batch_detail_info(self.ctx, a.ctypes.data))
        return int(a[0]), int(a[1]), int(a[2])

    def detail(self):
        """The last decode's detailed decode in full: (events uint32 [n, 8] — columns B.DETAIL_EVENT_FIELDS, kind JSGPU_DT_* —,
        matrices int16 [blocks, 64], natural order, [0] = the DC difference)."""
        nev, nblk, _ = self.detail_info()
        ev = np.zeros((nev, 8), np.uint32); mat = np.zeros((nblk, 64), np.int16)
        self._ck(self.L.jsgpu_batch_detail_events(self.ctx, 0, nev, ev.ctypes.data))
        self._ck(self.L.jsgpu_batch_detail_matrices(self.ctx, 0, nblk, mat.ctypes.data))
        return ev, mat

    def timer_start(self): self._ck(self.L.jsgpu_timer_start(self.ctx))

    def timer_stop(self):
        ms = C.c_float(0); self._ck(self.L.jsgpu_timer_stop(self.ctx, C.byref(ms))); return float(ms.value)

    def decode_host(self, darr, bits, outs):
        """One-call end-to-end form (jsgpu_decode_batch_host): host bitstream in, host buffers out.
        outs: dict name -> numpy array (pinned or pageable) for any of the jsgpu_host_outputs fields."""
        ho = B.jsgpu_host_outputs()
        for k, a in outs.items():
            setattr(ho, k, a.ctypes.data)
        self.descs = darr; self.n = len(darr)
        self._ck(self.L.jsgpu_decode_batch_host(self.ctx, C.byref(darr), self.n, bits.ctypes.data, bits.size, C.byref(ho)))

    def stage_ms(self):
        ms = np.zeros(5, np.float32); self._ck(self.L.jsgpu_batch_stage_ms(self.ctx, ms.ctypes.data)); return ms

    def pools(self):
        p = B.jsgpu_pools(); self._ck(self.L.jsgpu_batch_pools(self.ctx, C.byref(p))); return p

    def refresh_layout(self):
        self._ck(self.L.jsgpu_batch_layout(self.ctx, C.byref(self.layout), self.n)); return self.layout

    @staticmethod
    def _outputs(lo, i):
        """The ten per-image outputs: (name, JSGPU_OUT_* selector, dtype, shape, element offset of image i in its host pool,
        absent from a one-component scan).  blk_y/cb/cr become DecodedImage.blk_dc."""
        W, H = int(lo.img_x), int(lo.img_y); nblk = int(lo.blk_xmax) * int(lo.blk_ymax); nmcu = int(lo.mcu_xmax) * int(lo.mcu_ymax)
        po, bo = int(lo.pix_off), int(lo.blk_off)
        return [("pix_y", B.OUT_PIX_Y, np.int16, (H, W), po, False), ("pix_cb", B.OUT_PIX_CB, np.int16, (H, W), po, True),
                ("pix_cr", B.OUT_PIX_CR, np.int16, (H, W), po, True), ("dib", B.OUT_DIB, np.uint8, (H, W, 4), int(lo.dib_off), False),
                ("blk_y", B.OUT_BLK_Y, np.int16, (nblk,), bo, False), ("blk_cb", B.OUT_BLK_CB, np.int16, (nblk,), bo, True),
                ("blk_cr", B.OUT_BLK_CR, np.int16, (nblk,), bo, True),
                ("mcu_map", B.OUT_MCU_MAP, np.uint32, (nmcu,), int(lo.mcu_off), False),
                ("dht_histo", B.OUT_HISTO, np.uint32, (2, 4, 17), i * 136, False), ("stats", B.OUT_STATS, np.int32, (16,), i * 16, False)]

    def _image(self, i, get, refresh=True):
        """DecodedImage of image i, each output from get(name, selector, dtype, shape, offset)."""
        if refresh:
            self.refresh_layout()
        lo = self.layout[i]; d = DecodedImage()
        d.geom = np.array([lo.mcu_w, lo.mcu_h, lo.mcu_xmax, lo.mcu_ymax, lo.blk_xmax, lo.blk_ymax, lo.img_x, lo.img_y], np.uint32)
        ns = self.descs[i].num_sos_comps
        v = {name: None if chroma and ns != 3 else get(name, sel, dtype, shape, off)
             for name, sel, dtype, shape, off, chroma in self._outputs(lo, i)}
        d.blk_dc = (v.pop("blk_y"), v.pop("blk_cb"), v.pop("blk_cr"))
        d.__dict__.update(v)
        d.status = int(lo.status)
        return d

    def fetch_host(self, i, outs):
        """The same DecodedImage as fetch(), cut out of the host buffers a decode_host() call filled."""
        return self._image(i, lambda name, sel, dtype, shape, off: np.array(outs[name][off:off + int(np.prod(shape))]).reshape(shape))

    def fetch(self, i, refresh=True):
        """DecodedImage of image i; refresh=False reuses the layout read after the last decode (one read for a whole batch)."""
        def dl(name, sel, dtype, shape, off):
            a = np.zeros(shape, dtype)
            self._ck(self.L.jsgpu_batch_download(self.ctx, sel, i, a.ctypes.data, a.nbytes)); return a
        return self._image(i, dl, refresh)
