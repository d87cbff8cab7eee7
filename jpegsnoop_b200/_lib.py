"""ctypes bindings of libjsgpu.so (include/jsgpu.h + include/jsimg.h).

The library is built in-tree by `jpegsnoop_b200.build.build()` (nvcc, sm_90a).  There is no
Python or CPU implementation of the decode path behind these bindings: if the shared library
is missing, importing a decoder raises; if no CUDA device is present, jsgpu_init() fails.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("JSGPU_LIB") or os.path.join(HERE, "libjsgpu.so")   # JSGPU_LIB: kernel-variant experiments only

MAX_DHT_CODES = 260


class jsgpu_tables(C.Structure):
    _fields_ = [("dqt_zz", (C.c_uint16 * 64) * 4),
                ("dht_size", (C.c_uint32 * 4) * 2),
                ("dht_bits", ((C.c_uint32 * MAX_DHT_CODES) * 4) * 2),
                ("dht_len", ((C.c_uint8 * MAX_DHT_CODES) * 4) * 2),
                ("dht_code", ((C.c_uint8 * MAX_DHT_CODES) * 4) * 2)]


class jsgpu_image_desc(C.Structure):
    _fields_ = [("dim_x", C.c_uint32), ("dim_y", C.c_uint32),
                ("num_sof_comps", C.c_uint32), ("num_sos_comps", C.c_uint32),
                ("precision", C.c_uint32),
                ("restart_en", C.c_uint32), ("restart_interval", C.c_uint32),
                ("samp_h", C.c_uint32 * 4), ("samp_v", C.c_uint32 * 4),
                ("dqt_sel", C.c_uint32 * 4),
                ("dht_dc_sel", C.c_uint32 * 4), ("dht_ac_sel", C.c_uint32 * 4),
                ("table_set", C.c_uint32), ("file_pos", C.c_uint32),
                ("scan_offset", C.c_uint64), ("scan_length", C.c_uint64)]


class jsgpu_image_layout(C.Structure):
    _fields_ = [("mcu_w", C.c_uint32), ("mcu_h", C.c_uint32), ("mcu_xmax", C.c_uint32), ("mcu_ymax", C.c_uint32),
                ("blk_xmax", C.c_uint32), ("blk_ymax", C.c_uint32), ("img_x", C.c_uint32), ("img_y", C.c_uint32),
                ("num_segments", C.c_uint32), ("status", C.c_uint32),
                ("pix_off", C.c_uint64), ("dib_off", C.c_uint64), ("blk_off", C.c_uint64), ("mcu_off", C.c_uint64)]


class jsgpu_options(C.Structure):
    _fields_ = [("idct_mode", C.c_int32), ("decode_ac", C.c_int32), ("huff_kernel", C.c_int32),
                ("idct_kernel", C.c_int32), ("want_histo", C.c_int32), ("want_mcu_map", C.c_int32),
                ("device_markers", C.c_int32), ("scan_err_max", C.c_int32)]


class jsgpu_scan_event(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("code", "a", "b", "c", "d", "e", "pad0", "pad1")]


class jsgpu_scan_errors(C.Structure):
    _fields_ = [("nerr_lines", C.c_uint32), ("nevents", C.c_uint32), ("scan_bad", C.c_uint32), ("restart_read", C.c_uint32),
                ("done", C.c_uint32), ("end_pos", C.c_uint32), ("end_align", C.c_uint32), ("pad", C.c_uint32), ("ev", jsgpu_scan_event * 256)]


class jsgpu_pools(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("pix_y", "pix_cb", "pix_cr", "dib", "blk_y", "blk_cb", "blk_cr",
                                          "mcu_map", "dht_histo", "stats", "coef", "bitstream")]


class jsgpu_host_outputs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("pix_y", "pix_cb", "pix_cr", "dib", "blk_y", "blk_cb", "blk_cr",
                                          "mcu_map", "dht_histo", "stats")]


class jsgpu_preview(C.Structure):
    """include/jsgpu.h: CalcChannelPreviewFull settings (histogram/clip conversion, preview mode, YCC shift)."""
    _fields_ = [("hist_en", C.c_int32), ("statclip_en", C.c_int32), ("mode", C.c_int32),
                ("shift_y", C.c_int32), ("shift_cb", C.c_int32), ("shift_cr", C.c_int32),
                ("shift_mcu_x", C.c_uint32), ("shift_mcu_y", C.c_uint32), ("ycc_warn_budget", C.c_uint32),
                ("detail_en", C.c_uint32), ("detail_mcu_x", C.c_uint32), ("detail_mcu_y", C.c_uint32), ("pad", C.c_uint32)]


class jsgpu_ycc_warn(C.Structure):
    _fields_ = [("mcu_x", C.c_uint32), ("mcu_y", C.c_uint32), ("y", C.c_int32), ("cb", C.c_int32), ("cr", C.c_int32), ("kind", C.c_uint32), ("px", C.c_uint32), ("py", C.c_uint32)]


class jsgpu_colour_stats(C.Structure):
    _fields_ = [("cc_histo", (C.c_uint32 * 128) * 3), ("y_histo", C.c_uint32 * 2048),
                ("vmin", C.c_int32 * 12), ("vmax", C.c_int32 * 12), ("vsum", C.c_int64 * 12), ("count", C.c_uint64),
                ("clip", C.c_uint32 * 12), ("nwarn", C.c_uint32), ("pad", C.c_uint32), ("warn", jsgpu_ycc_warn * 10),
                ("detail_rgb", (C.c_uint32 * 32) * 32)]


class jsgpu_detail(C.Structure):
    _fields_ = [("enable", C.c_int32), ("image", C.c_uint32), ("mcu_x", C.c_uint32), ("mcu_y", C.c_uint32), ("len", C.c_uint32)]


# jsgpu_detail_event as a numpy record (kind JSGPU_DT_*, seq, a..f: include/jsgpu.h)
DETAIL_EVENT_FIELDS = ("kind", "seq", "a", "b", "c", "d", "e", "f")
DT_MCU, DT_BLOCK, DT_VLC, DT_MATRIX = 1, 2, 3, 4
DETAIL_SERIAL, DETAIL_PARALLEL = 0, 1

OUT_PIX_Y, OUT_PIX_CB, OUT_PIX_CR, OUT_DIB, OUT_BLK_Y, OUT_BLK_CB, OUT_BLK_CR, OUT_MCU_MAP, OUT_HISTO, OUT_STATS = range(10)

# every symbol include/jsgpu.h and include/jsimg.h declare (tests check they are all exported)
JSGPU_SYMBOLS = [
    "jsgpu_init", "jsgpu_free", "jsgpu_last_error", "jsgpu_strerror", "jsgpu_version", "jsgpu_stream", "jsgpu_sync",
    "jsgpu_set_idct_tables", "jsgpu_set_options", "jsgpu_get_options", "jsgpu_upload_tables", "jsgpu_bcast_tables",
    "jsgpu_batch_begin", "jsgpu_batch_layout", "jsgpu_batch_pools", "jsgpu_batch_upload", "jsgpu_batch_decode",
    "jsgpu_batch_download", "jsgpu_batch_stage_ms", "jsgpu_timer_start", "jsgpu_timer_stop", "jsgpu_batch_launches", "jsgpu_batch_selfsync_info", "jsgpu_batch_checksums", "jsgpu_batch_errors", "jsgpu_decode_batch_host",
    "jsgpu_host_alloc", "jsgpu_host_free", "jsgpu_host_copy_rate", "jsgpu_set_preview", "jsgpu_batch_preview", "jsgpu_batch_colour_stats", "jsgpu_batch_export", "jsgpu_set_detail", "jsgpu_batch_detail",
    "jsgpu_batch_detail_info", "jsgpu_batch_detail_events", "jsgpu_batch_detail_matrices"]
JSIMG_SYMBOLS = [
    "jsimg_create", "jsimg_destroy", "jsimg_config", "jsimg_set_file", "jsimg_overlay_install", "jsimg_overlay_remove_all", "jsimg_Reset", "jsimg_ResetState",
    "jsimg_SetDqtEntry", "jsimg_SetDqtTables", "jsimg_GetDqtEntry", "jsimg_SetDhtTables", "jsimg_SetDhtEntry",
    "jsimg_SetDhtSize", "jsimg_SetPrecision", "jsimg_SetSofSampFactors", "jsimg_SetImageDetails",
    "jsimg_DecodeScanImg", "jsimg_IsPreviewReady", "jsimg_GetImageSize", "jsimg_GetPixMapPtrs", "jsimg_GetBitmapPtr",
    "jsimg_LookupFilePosMcu", "jsimg_LookupFilePosPix", "jsimg_LookupBlkYCC", "jsimg_GetMcuFileMap", "jsimg_GetBlkDcMap",
    "jsimg_GetDhtHisto", "jsimg_GetGeometry", "jsimg_GetStats", "jsimg_GetIdctTables", "jsimg_GetStageMs", "jsimg_GetScanStatus",
    "jsimg_log_count", "jsimg_log_line", "jsimg_log_clear", "jsimg_walk_jpeg", "jsimg_decode_jpeg", "jsimg_parse_jpeg",
    "jsimg_config_histo", "jsimg_SetPreviewMode", "jsimg_GetPreviewMode", "jsimg_SetPreviewYccOffset", "jsimg_GetPreviewYccOffset",
    "jsimg_GetStatClip", "jsimg_GetHistoRanges", "jsimg_GetCcHisto", "jsimg_GetHistoYFull", "jsimg_GetHistoDib", "jsimg_ExportTiff", "jsimg_tiff_write", "jsimg_SetDetailVlc", "jsimg_GetDetailVlc"]

_lib = None


def load():
    """Load libjsgpu.so (raises if it has not been built — there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(the decode path has no Python/CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.jsgpu_init.argtypes = [i32, C.POINTER(vp)]
    L.jsgpu_free.argtypes = [vp]; L.jsgpu_free.restype = None
    L.jsgpu_last_error.argtypes = [vp]; L.jsgpu_last_error.restype = C.c_char_p
    L.jsgpu_strerror.argtypes = [i32]; L.jsgpu_strerror.restype = C.c_char_p
    L.jsgpu_stream.argtypes = [vp]; L.jsgpu_stream.restype = vp
    L.jsgpu_sync.argtypes = [vp]
    L.jsgpu_set_idct_tables.argtypes = [vp, vp, vp]
    L.jsgpu_set_options.argtypes = [vp, C.POINTER(jsgpu_options)]
    L.jsgpu_get_options.argtypes = [vp, C.POINTER(jsgpu_options)]
    L.jsgpu_upload_tables.argtypes = [vp, vp, u32]
    L.jsgpu_bcast_tables.argtypes = [vp, vp, u32, vp, i32]
    L.jsgpu_batch_begin.argtypes = [vp, vp, u32, u64]
    L.jsgpu_batch_layout.argtypes = [vp, vp, u32]
    L.jsgpu_batch_pools.argtypes = [vp, C.POINTER(jsgpu_pools)]
    L.jsgpu_batch_upload.argtypes = [vp, vp, u64]
    L.jsgpu_batch_decode.argtypes = [vp]
    L.jsgpu_batch_download.argtypes = [vp, i32, u32, vp, u64]
    L.jsgpu_batch_stage_ms.argtypes = [vp, vp]
    L.jsgpu_batch_launches.argtypes = [vp]
    L.jsgpu_batch_selfsync_info.argtypes = [vp, vp, u32]
    L.jsgpu_batch_checksums.argtypes = [vp, vp, u32]
    L.jsgpu_batch_errors.argtypes = [vp, u32, C.POINTER(jsgpu_scan_errors)]
    L.jsgpu_timer_start.argtypes = [vp]
    L.jsgpu_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
    L.jsgpu_decode_batch_host.argtypes = [vp, vp, u32, vp, u64, C.POINTER(jsgpu_host_outputs)]
    L.jsgpu_host_alloc.argtypes = [u64]; L.jsgpu_host_alloc.restype = vp
    L.jsgpu_host_free.argtypes = [vp]; L.jsgpu_host_free.restype = None
    L.jsgpu_host_copy_rate.argtypes = [vp, i32, u64, i32, C.POINTER(C.c_float)]
    L.jsgpu_set_preview.argtypes = [vp, C.POINTER(jsgpu_preview)]
    L.jsgpu_batch_preview.argtypes = [vp, C.POINTER(jsgpu_preview)]
    L.jsgpu_batch_colour_stats.argtypes = [vp, u32, C.POINTER(jsgpu_colour_stats)]
    L.jsgpu_batch_export.argtypes = [vp, u32, i32, vp, u64]
    L.jsimg_ExportTiff.argtypes = [vp, C.c_char_p, u32]
    L.jsimg_tiff_write.argtypes = [C.c_char_p, i32, i32, vp, u32, u32]
    L.jsgpu_set_detail.argtypes = [vp, vp]
    L.jsgpu_batch_detail.argtypes = [vp, vp]
    L.jsgpu_batch_detail_info.argtypes = [vp, vp]
    L.jsgpu_batch_detail_events.argtypes = [vp, u32, u32, vp]
    L.jsgpu_batch_detail_matrices.argtypes = [vp, u32, u32, vp]
    L.jsimg_SetDetailVlc.argtypes = [vp, i32, u32, u32, u32]; L.jsimg_SetDetailVlc.restype = None
    L.jsimg_GetDetailVlc.argtypes = [vp] + [C.POINTER(u32)] * 4; L.jsimg_GetDetailVlc.restype = None
    L.jsimg_config_histo.argtypes = [vp, i32, i32, i32]; L.jsimg_config_histo.restype = None
    L.jsimg_SetPreviewMode.argtypes = [vp, u32]; L.jsimg_SetPreviewMode.restype = None
    L.jsimg_GetPreviewMode.argtypes = [vp]; L.jsimg_GetPreviewMode.restype = u32
    L.jsimg_SetPreviewYccOffset.argtypes = [vp, u32, u32, i32, i32, i32]; L.jsimg_SetPreviewYccOffset.restype = None
    L.jsimg_GetPreviewYccOffset.argtypes = [vp] + [C.POINTER(u32)] * 2 + [C.POINTER(i32)] * 3; L.jsimg_GetPreviewYccOffset.restype = None
    L.jsimg_GetStatClip.argtypes = [vp, vp]; L.jsimg_GetStatClip.restype = None
    L.jsimg_GetHistoRanges.argtypes = [vp, vp, C.POINTER(u32)]; L.jsimg_GetHistoRanges.restype = None
    L.jsimg_GetCcHisto.argtypes = [vp, u32, vp]; L.jsimg_GetCcHisto.restype = None
    L.jsimg_GetHistoYFull.argtypes = [vp, vp]; L.jsimg_GetHistoYFull.restype = None
    L.jsimg_GetHistoDib.argtypes = [vp, i32, C.POINTER(i32)]; L.jsimg_GetHistoDib.restype = vp
    L.jsimg_create.restype = vp
    L.jsimg_destroy.argtypes = [vp]; L.jsimg_destroy.restype = None
    L.jsimg_config.argtypes = [vp] + [i32] * 6; L.jsimg_config.restype = None
    L.jsimg_set_file.argtypes = [vp, vp, u64]; L.jsimg_set_file.restype = None
    L.jsimg_overlay_install.argtypes = [vp, u32, vp, u32]
    L.jsimg_overlay_remove_all.argtypes = [vp]; L.jsimg_overlay_remove_all.restype = None
    for n in ("jsimg_Reset", "jsimg_ResetState", "jsimg_log_clear"):
        getattr(L, n).argtypes = [vp]; getattr(L, n).restype = None
    L.jsimg_SetDqtEntry.argtypes = [vp, u32, u32, u32, u32]
    L.jsimg_SetDqtTables.argtypes = [vp, u32, u32]
    L.jsimg_GetDqtEntry.argtypes = [vp, u32, u32]; L.jsimg_GetDqtEntry.restype = u32
    L.jsimg_SetDhtTables.argtypes = [vp, u32, u32, u32]
    L.jsimg_SetDhtEntry.argtypes = [vp] + [u32] * 7
    L.jsimg_SetDhtSize.argtypes = [vp, u32, u32, u32]
    L.jsimg_SetPrecision.argtypes = [vp, u32]; L.jsimg_SetPrecision.restype = None
    L.jsimg_SetSofSampFactors.argtypes = [vp, u32, u32, u32]; L.jsimg_SetSofSampFactors.restype = None
    L.jsimg_SetImageDetails.argtypes = [vp, u32, u32, u32, u32, i32, u32]; L.jsimg_SetImageDetails.restype = None
    L.jsimg_DecodeScanImg.argtypes = [vp, u32, i32, i32]; L.jsimg_DecodeScanImg.restype = None
    L.jsimg_IsPreviewReady.argtypes = [vp]
    L.jsimg_GetImageSize.argtypes = [vp, C.POINTER(u32), C.POINTER(u32)]; L.jsimg_GetImageSize.restype = None
    L.jsimg_GetPixMapPtrs.argtypes = [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]; L.jsimg_GetPixMapPtrs.restype = None
    L.jsimg_GetBitmapPtr.argtypes = [vp]; L.jsimg_GetBitmapPtr.restype = vp
    L.jsimg_LookupFilePosMcu.argtypes = [vp, u32, u32, C.POINTER(u32), C.POINTER(u32)]; L.jsimg_LookupFilePosMcu.restype = None
    L.jsimg_LookupFilePosPix.argtypes = [vp, u32, u32, C.POINTER(u32), C.POINTER(u32)]; L.jsimg_LookupFilePosPix.restype = None
    L.jsimg_LookupBlkYCC.argtypes = [vp, u32, u32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]; L.jsimg_LookupBlkYCC.restype = None
    L.jsimg_GetMcuFileMap.argtypes = [vp]; L.jsimg_GetMcuFileMap.restype = vp
    L.jsimg_GetBlkDcMap.argtypes = [vp, u32]; L.jsimg_GetBlkDcMap.restype = vp
    for n in ("jsimg_GetDhtHisto", "jsimg_GetGeometry", "jsimg_GetStats", "jsimg_GetStageMs"):
        getattr(L, n).argtypes = [vp, vp]; getattr(L, n).restype = None
    L.jsimg_GetIdctTables.argtypes = [vp, vp, vp]; L.jsimg_GetIdctTables.restype = None
    L.jsimg_GetScanStatus.argtypes = [vp]; L.jsimg_GetScanStatus.restype = u32
    L.jsimg_log_count.argtypes = [vp, i32]
    L.jsimg_log_line.argtypes = [vp, i32, i32]; L.jsimg_log_line.restype = C.c_char_p
    L.jsimg_walk_jpeg.argtypes = [vp, vp, u64]
    L.jsimg_decode_jpeg.argtypes = [vp, vp, u64, i32]
    L.jsimg_parse_jpeg.argtypes = [vp, u64, C.POINTER(jsgpu_tables), C.POINTER(jsgpu_image_desc)]
    _lib = L
    return L
