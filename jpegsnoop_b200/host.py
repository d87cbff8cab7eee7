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
        self.nerr = 0; self.scan_start = 0; self.status = 0; self.stage_ms = None


class CimgDecode:
    """Mirror of the reference class (source/ImgDecode.h:284-425) driven through jsimg_*."""

    def __init__(self, decode_ac=True, idct_fixedpt=True, device=0, huff_kernel=0, idct_kernel=0):
        self.L = B.load()
        self.h = C.c_void_p(self.L.jsimg_create())
        self.L.jsimg_config(self.h, int(decode_ac), int(idct_fixedpt), device, huff_kernel, idct_kernel, 1)
        self._file = None

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

    def decode(self, jpeg_bytes, quiet=True):
        """Marker walk (CjfifDecode's setter sequence) then DecodeScanImg(start, True, quiet)."""
        self.set_file(jpeg_bytes)
        self.L.jsimg_log_clear(self.h)
        r = self.L.jsimg_decode_jpeg(self.h, self._file.ctypes.data, self._file.size, int(quiet))
        if r < 0:
            raise ValueError(f"marker walk failed ({r})")
        d = self.collect(); d.scan_start = r
        return d


def parse_jpeg(jpeg_bytes):
    """Marker walk only -> (jsgpu_tables, jsgpu_image_desc, scan_start)."""
    L = B.load()
    buf = np.frombuffer(bytes(jpeg_bytes), np.uint8)
    t = B.jsgpu_tables(); d = B.jsgpu_image_desc()
    r = L.jsimg_parse_jpeg(buf.ctypes.data, buf.size, C.byref(t), C.byref(d))
    if r < 0:
        raise ValueError(f"marker walk failed ({r})")
    return t, d, r


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
                                   scan_err_max=0)
        self._ck(self.L.jsgpu_set_options(self.ctx, C.byref(self.opt)))
        self.n = 0; self.layout = None; self.descs = None; self.bitstream = None; self.nsof_pixels = 0

    def _ck(self, r):
        if r != 0:
            raise JsgpuError(f"{self.L.jsgpu_strerror(r).decode()}: {self.L.jsgpu_last_error(self.ctx).decode()}")

    def close(self):
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
        scan bytes.  Returns (table_sets array, descs array, bitstream uint8 array)."""
        sets, keys, descs, chunks, off = [], {}, [], [], 0
        for j in jpegs:
            t, d, start = parse_jpeg(j)
            k = tables_key(t)
            if k not in keys:
                keys[k] = len(sets); sets.append(t)
            d.table_set = keys[k]
            scan = np.frombuffer(bytes(j), np.uint8)[start:]
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

    def scan_errors(self, i):
        """jsgpu_scan_errors of image i (only for images whose status carries JSGPU_ST_EXACT = 0x40000000)."""
        e = B.jsgpu_scan_errors(); self._ck(self.L.jsgpu_batch_errors(self.ctx, i, C.byref(e))); return e

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

    def _dl(self, which, i, dtype, shape):
        a = np.zeros(shape, dtype)
        self._ck(self.L.jsgpu_batch_download(self.ctx, which, i, a.ctypes.data, a.nbytes)); return a

    def fetch_host(self, i, outs):
        """The same DecodedImage as fetch(), cut out of the host buffers a decode_host() call filled."""
        self.refresh_layout()
        lo = self.layout[i]; d = DecodedImage()
        d.geom = np.array([lo.mcu_w, lo.mcu_h, lo.mcu_xmax, lo.mcu_ymax, lo.blk_xmax, lo.blk_ymax, lo.img_x, lo.img_y], np.uint32)
        Wp, Hp = int(lo.img_x), int(lo.img_y); nblk = int(lo.blk_xmax) * int(lo.blk_ymax); nmcu = int(lo.mcu_xmax) * int(lo.mcu_ymax)
        ns = self.descs[i].num_sos_comps
        po, do, bo, mo = int(lo.pix_off), int(lo.dib_off), int(lo.blk_off), int(lo.mcu_off)
        cut = lambda a, off, n, shape: np.array(a[off:off + n]).reshape(shape)
        d.pix_y = cut(outs["pix_y"], po, Wp * Hp, (Hp, Wp))
        d.pix_cb = cut(outs["pix_cb"], po, Wp * Hp, (Hp, Wp)) if ns == 3 else None
        d.pix_cr = cut(outs["pix_cr"], po, Wp * Hp, (Hp, Wp)) if ns == 3 else None
        d.dib = cut(outs["dib"], do, Wp * Hp * 4, (Hp, Wp, 4))
        d.mcu_map = cut(outs["mcu_map"], mo, nmcu, (nmcu,))
        d.blk_dc = (cut(outs["blk_y"], bo, nblk, (nblk,)),
                    cut(outs["blk_cb"], bo, nblk, (nblk,)) if ns == 3 else None,
                    cut(outs["blk_cr"], bo, nblk, (nblk,)) if ns == 3 else None)
        d.dht_histo = cut(outs["dht_histo"], i * 136, 136, (2, 4, 17))
        d.stats = cut(outs["stats"], i * 16, 16, (16,))
        d.status = int(lo.status)
        return d

    def fetch(self, i):
        self.refresh_layout()
        lo = self.layout[i]; d = DecodedImage()
        d.geom = np.array([lo.mcu_w, lo.mcu_h, lo.mcu_xmax, lo.mcu_ymax, lo.blk_xmax, lo.blk_ymax, lo.img_x, lo.img_y], np.uint32)
        Wp, Hp = lo.img_x, lo.img_y; nblk = lo.blk_xmax * lo.blk_ymax; nmcu = lo.mcu_xmax * lo.mcu_ymax
        ns = self.descs[i].num_sos_comps
        d.pix_y = self._dl(B.OUT_PIX_Y, i, np.int16, (Hp, Wp))
        d.pix_cb = self._dl(B.OUT_PIX_CB, i, np.int16, (Hp, Wp)) if ns == 3 else None
        d.pix_cr = self._dl(B.OUT_PIX_CR, i, np.int16, (Hp, Wp)) if ns == 3 else None
        d.dib = self._dl(B.OUT_DIB, i, np.uint8, (Hp, Wp, 4))
        d.mcu_map = self._dl(B.OUT_MCU_MAP, i, np.uint32, (nmcu,))
        d.blk_dc = (self._dl(B.OUT_BLK_Y, i, np.int16, (nblk,)),
                    self._dl(B.OUT_BLK_CB, i, np.int16, (nblk,)) if ns == 3 else None,
                    self._dl(B.OUT_BLK_CR, i, np.int16, (nblk,)) if ns == 3 else None)
        d.dht_histo = self._dl(B.OUT_HISTO, i, np.uint32, (2, 4, 17))
        d.stats = self._dl(B.OUT_STATS, i, np.int32, (16,))
        d.status = int(lo.status)
        return d
