"""TEST INFRASTRUCTURE: ctypes front-end to the CPU oracles.

Two oracles share one API shape:
  * "port"          -> oracle/liboracle_port.so      (our plain-C restatement, oracle/port/)
  * "ref_fixed/float" -> oracle/_ref/liboracle_ref_*.so (the UNMODIFIED reference compiled in place)
Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this.
"""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")


def build_oracles(quiet=True):
    """Build the port always; the reference oracle only where /root/reference exists."""
    out = subprocess.run(["make", "-C", ORACLE_DIR, "port", "ref", "n1"], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout[-2000:] + out.stderr[-2000:])
    return out.stdout if not quiet else ""


def ref_available(mode="fixed"):
    return os.path.exists(os.path.join(ORACLE_DIR, "_ref", f"liboracle_ref_{mode}.so"))


class Decoded:
    """Plain container of one decode's outputs (numpy copies)."""
    def __init__(self):
        self.geom = None       # mcu_w, mcu_h, mcu_xmax, mcu_ymax, blk_xmax, blk_ymax, img_x, img_y
        self.pix_y = self.pix_cb = self.pix_cr = None   # int16 [Hp, Wp]
        self.dib = None        # uint8 [Hp, Wp, 4] BGRA bottom-up (row 0 = bottom image row)
        self.mcu_map = None    # uint32 [mcu_ymax*mcu_xmax]
        self.blk_dc = None     # tuple of int16 [blk_ymax*blk_xmax]
        self.dht_histo = None  # uint32 [2,4,17]
        self.stats = None      # int32[12]: avgY, avgValid, brightY,Cb,Cr,R,G,B, mcuX, mcuY, nRst, scanBad
        self.nerr = 0
        self.scan_start = 0


class Oracle:
    """One decoder instance of either oracle.  kind: 'port' | 'ref_fixed' | 'ref_float'.
    For 'port', idct_fixed selects the arithmetic (True = -DIDCT_FIXEDPT semantics)."""

    def __init__(self, kind="port", idct_fixed=True, decode_ac=True):
        self.kind = kind
        if kind == "port":
            path = os.path.join(ORACLE_DIR, "liboracle_port.so")
            self.p = "op_"
        else:
            path = os.path.join(ORACLE_DIR, "_ref", f"liboracle_{kind}.so")
            self.p = "ref_"
            idct_fixed = (kind == "ref_fixed")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.idct_fixed = idct_fixed
        self.lib = L = C.CDLL(path)
        f = self._f
        f("create").restype = C.c_void_p
        for n in ("pix_y", "pix_cb", "pix_cr", "blk_dc_y", "blk_dc_cb", "blk_dc_cr"):
            f(n).restype = C.POINTER(C.c_int16)
            f(n).argtypes = [C.c_void_p]
        f("dib").restype = C.POINTER(C.c_uint8); f("dib").argtypes = [C.c_void_p]
        f("mcu_file_map").restype = C.POINTER(C.c_uint32); f("mcu_file_map").argtypes = [C.c_void_p]
        f("decode_jpeg").argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int]
        f("setup_jpeg").argtypes = [C.c_void_p, C.c_void_p, C.c_uint64]
        for n in ("geometry", "dht_histo", "stats"):
            f(n).argtypes = [C.c_void_p, C.c_void_p]
        f("idct_tables").argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        f("num_err_lines").argtypes = [C.c_void_p]
        f("destroy").argtypes = [C.c_void_p]
        f("bench").restype = C.c_double
        self.ctx = C.c_void_p(f("create")())
        if kind == "port":
            L.op_config.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint]
            L.op_config(self.ctx, int(idct_fixed), int(decode_ac), 20)
        else:
            assert bool(L.ref_is_fixedpt()) == idct_fixed
            L.ref_config(int(decode_ac), 0, 20)
        self._keep = None

    def _f(self, name):
        return getattr(self.lib, self.p + name)

    def close(self):
        if self.ctx:
            self._f("destroy")(self.ctx)
            self.ctx = None

    def idct_tables(self):
        lf = np.zeros((64, 64), np.float32); li = np.zeros((64, 64), np.int32)
        self._f("idct_tables")(self.ctx, lf.ctypes.data, li.ctypes.data)
        return lf, li

    def err_lines(self):
        """Error log lines (AddLineErr) of the last decode — compiled reference only."""
        assert self.kind != "port"
        self.lib.ref_err_line.restype = C.c_char_p; self.lib.ref_err_line.argtypes = [C.c_void_p, C.c_int]
        return [self.lib.ref_err_line(self.ctx, i).decode("latin-1") for i in range(self._f("num_err_lines")(self.ctx))]

    # --- channel preview / colour statistics (both oracles; the histogram bitmaps and log lines: compiled reference only) ------
    def config_histo(self, histo_en=False, statclip_en=False, dump_histo_y=False):
        if self.kind == "port":
            self.lib.op_config_histo.argtypes = [C.c_void_p, C.c_int, C.c_int]; self.lib.op_config_histo(self.ctx, int(histo_en), int(statclip_en))
        else:
            self.lib.ref_config_histo(int(histo_en), int(statclip_en), int(dump_histo_y))

    def set_detail_vlc(self, detail, x=0, y=0, n=1):
        assert self.kind != "port"
        self.lib.ref_SetDetailVlc.argtypes = [C.c_void_p, C.c_int, C.c_uint, C.c_uint, C.c_uint]; self.lib.ref_SetDetailVlc(self.ctx, int(detail), x, y, n)

    def set_preview_mode(self, mode):
        f = self._f("SetPreviewMode"); f.argtypes = [C.c_void_p, C.c_uint]; f(self.ctx, mode)

    def set_ycc_offset(self, mx, my, y, cb, cr):
        f = self._f("SetPreviewYccOffset"); f.argtypes = [C.c_void_p, C.c_uint, C.c_uint, C.c_int, C.c_int, C.c_int]
        f(self.ctx, mx, my, y, cb, cr)

    def colour_stats(self):
        clip = np.zeros(12, np.uint32); f = self._f("GetStatClip"); f.argtypes = [C.c_void_p, C.c_void_p]; f(self.ctx, clip.ctypes.data)
        rng = np.zeros(36, np.int32); n = C.c_uint32()
        f = self._f("GetHistoRanges"); f.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32)]; f(self.ctx, rng.ctypes.data, C.byref(n))
        cc = np.zeros((3, 128), np.uint32); f = self._f("GetCcHisto"); f.argtypes = [C.c_void_p, C.c_uint, C.c_void_p]
        for c in range(3):
            f(self.ctx, c, cc[c].ctypes.data)
        yh = np.zeros(2048, np.uint32); f = self._f("GetHistoYFull"); f.argtypes = [C.c_void_p, C.c_void_p]; f(self.ctx, yh.ctypes.data)
        return {"clip": clip, "ranges": rng, "count": int(n.value), "cc_histo": cc, "y_histo": yh}

    def histo_dib(self, which):
        L = self.lib; ready = C.c_int(0)
        L.ref_GetHistoDib.restype = C.POINTER(C.c_uint8); L.ref_GetHistoDib.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        p = L.ref_GetHistoDib(self.ctx, which, C.byref(ready))
        if not ready.value or not p:
            return None
        return np.ctypeslib.as_array(p, shape=(30, 512, 4) if which else (90, 128, 4)).copy()

    def bitmap(self):
        g = np.zeros(8, np.uint32); self._f("geometry")(self.ctx, g.ctypes.data)
        p = self._f("dib")(self.ctx)
        return np.ctypeslib.as_array(p, shape=(int(g[7]), int(g[6]), 4)).copy() if p else None

    def log_lines(self):
        """Every log line of the last decode, in order — compiled reference only."""
        assert self.kind != "port"
        self.lib.ref_line.restype = C.c_char_p; self.lib.ref_line.argtypes = [C.c_void_p, C.c_int]
        return [self.lib.ref_line(self.ctx, i).decode("latin-1") for i in range(self.lib.ref_num_lines(self.ctx))]

    def decode(self, jpeg_bytes, overlays=(), quiet=True):
        """Marker walk + DecodeScanImg(start, bDisplay=true, bQuiet=quiet); returns Decoded.
        overlays: [(file offset, bytes)] installed in the reference's CwindowBuf before the decode (reference only)."""
        buf = np.frombuffer(jpeg_bytes, np.uint8).copy()
        self._keep = buf
        if self.kind != "port":
            self.lib.ref_log_clear.argtypes = [C.c_void_p]; self.lib.ref_log_clear(self.ctx)      # nerr counts THIS decode
            self.lib.ref_overlay_remove_all.argtypes = [C.c_void_p]; self.lib.ref_overlay_remove_all(self.ctx)
            for off, data in overlays:
                ob = np.frombuffer(bytes(data), np.uint8).copy()
                self.lib.ref_overlay_install.argtypes = [C.c_void_p, C.c_uint, C.c_void_p, C.c_uint]
                self.lib.ref_overlay_install(self.ctx, int(off), ob.ctypes.data, ob.size)
        r = self._f("decode_jpeg")(self.ctx, buf.ctypes.data, buf.size, 1 if quiet else 0)
        if r < 0:
            raise ValueError(f"marker walk failed ({r})")
        d = self.collect(); d.scan_start = r
        return d

    def collect(self):
        """Decoded copy of everything the last DecodeScanImg left behind (scan_start not set)."""
        d = Decoded()
        g = np.zeros(8, np.uint32); self._f("geometry")(self.ctx, g.ctypes.data); d.geom = g
        Wp, Hp = int(g[6]), int(g[7])
        nblk = int(g[4]) * int(g[5]); nmcu = int(g[2]) * int(g[3])

        def arr(ptr, shape):
            if not ptr:
                return None
            return np.ctypeslib.as_array(ptr, shape=shape).copy()
        d.pix_y = arr(self._f("pix_y")(self.ctx), (Hp, Wp))
        d.pix_cb = arr(self._f("pix_cb")(self.ctx), (Hp, Wp))
        d.pix_cr = arr(self._f("pix_cr")(self.ctx), (Hp, Wp))
        d.dib = arr(self._f("dib")(self.ctx), (Hp, Wp, 4))
        d.mcu_map = arr(self._f("mcu_file_map")(self.ctx), (nmcu,))
        d.blk_dc = tuple(arr(self._f(n)(self.ctx), (nblk,)) for n in ("blk_dc_y", "blk_dc_cb", "blk_dc_cr"))
        h = np.zeros((2, 4, 17), np.uint32); self._f("dht_histo")(self.ctx, h.ctypes.data); d.dht_histo = h
        s = np.zeros(12, np.int32); self._f("stats")(self.ctx, s.ctypes.data); d.stats = s
        d.nerr = self._f("num_err_lines")(self.ctx)
        return d

    def bench_ck(self, jpegs, threads=1):
        """Decode every JPEG once on `threads` host threads; returns (wall seconds, error lines, uint64 [n][12] checksums
        of every output buffer — the layout of jsgpu_batch_checksums, include/jsgpu.h).  Compiled reference only."""
        assert self.kind != "port"
        bufs = [np.frombuffer(j, np.uint8) for j in jpegs]
        n = len(bufs)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        lens = (C.c_uint64 * n)(*[b.size for b in bufs])
        ck = np.zeros((n, 12), np.uint64); errs = C.c_int(0)
        self.lib.ref_bench_ck.restype = C.c_double
        t = self.lib.ref_bench_ck(ptrs, lens, n, threads, C.c_void_p(ck.ctypes.data), C.byref(errs))
        return float(t), int(errs.value), ck

    def bench(self, jpegs, threads=1, reps=1):
        """Wall seconds to decode every JPEG in `jpegs` `reps` times on `threads` host threads."""
        bufs = [np.frombuffer(j, np.uint8).copy() for j in jpegs]
        n = len(bufs)
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        lens = (C.c_uint64 * n)(*[b.size for b in bufs])
        errs = C.c_int(0)
        if self.kind == "port":
            t = self.lib.op_bench(ptrs, lens, n, threads, reps, int(self.idct_fixed), C.byref(errs))
        else:
            t = self.lib.ref_bench(ptrs, lens, n, threads, reps, C.byref(errs))
        return float(t), int(errs.value)


def effective_cores():
    """Host threads this process can really use: the affinity mask, capped by the cgroup CPU quota (a container on a
    128-thread box may be limited to a handful of cores: os.cpu_count() says nothing about that)."""
    import math
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    quota = None
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            quota = float(q) / float(p)
    except Exception:
        try:
            q = float(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read()); p = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / p
        except Exception:
            pass
    eff = n if quota is None else max(1, min(n, int(math.ceil(quota))))
    return eff, {"os_cpu_count": os.cpu_count(), "affinity": n, "cgroup_quota_cores": quota}


def dib_to_rgb(dib):
    """BGRA bottom-up DIB [Hp,Wp,4] -> top-down RGB [Hp,Wp,3]."""
    return dib[::-1, :, 2::-1]
