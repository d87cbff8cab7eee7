"""What each batch state of a jsgpu context allows (include/jsgpu.h): after jsgpu_decode_batch_host cut a batch into image
ranges the context holds its layout only; after the single-stream form, and after jsgpu_batch_begin + jsgpu_batch_decode,
the decoded batch is resident and every query works."""
import ctypes as C

import numpy as np
import pytest

import jpeg_cases as JC

pytestmark = pytest.mark.gpu

ESTATE = -5


def _jpegs(n):
    return [JC.enc(JC.synth_rgb(48 + 8 * (i % 5), 40 + 8 * (i % 3), 500 + i), quality=80, subsampling=i % 3) for i in range(n)]


def _host_outputs(lay, n):
    tot = lambda f, a: sum((f(l) + a - 1) // a * a for l in lay)
    pix = tot(lambda l: int(l.img_x) * int(l.img_y), 64); blk = tot(lambda l: int(l.blk_xmax) * int(l.blk_ymax), 64)
    return {"pix_y": np.zeros(pix, np.int16), "pix_cb": np.zeros(pix, np.int16), "pix_cr": np.zeros(pix, np.int16),
            "dib": np.zeros(tot(lambda l: int(l.img_x) * int(l.img_y) * 4, 256), np.uint8),
            "blk_y": np.zeros(blk, np.int16), "blk_cb": np.zeros(blk, np.int16), "blk_cr": np.zeros(blk, np.int16),
            "mcu_map": np.zeros(tot(lambda l: int(l.mcu_xmax) * int(l.mcu_ymax), 32), np.uint32),
            "dht_histo": np.zeros(n * 136, np.uint32), "stats": np.zeros(n * 16, np.int32)}


def _queries(bd):
    """Return code of every batch query on bd's context (image 0), by name."""
    from jpegsnoop_b200 import _lib as B
    L, ctx = bd.L, bd.ctx
    lo = bd.layout[0]
    px = np.zeros(int(lo.img_x) * int(lo.img_y) * 2, np.int16)
    ex = np.zeros(int(lo.img_x) * int(lo.img_y) * 3, np.uint8)
    ck = np.zeros((bd.n, 12), np.uint64); ms = np.zeros(5, np.float32)
    lay = (B.jsgpu_image_layout * bd.n)()
    pv = B.jsgpu_preview(mode=1, ycc_warn_budget=10)
    return {"layout": L.jsgpu_batch_layout(ctx, C.byref(lay), bd.n),
            "download": L.jsgpu_batch_download(ctx, B.OUT_PIX_Y, 0, px.ctypes.data, int(lo.img_x) * int(lo.img_y) * 2),
            "pools": L.jsgpu_batch_pools(ctx, C.byref(B.jsgpu_pools())),
            "checksums": L.jsgpu_batch_checksums(ctx, ck.ctypes.data, bd.n),
            "errors": L.jsgpu_batch_errors(ctx, 0, C.byref(B.jsgpu_scan_errors())),
            "export": L.jsgpu_batch_export(ctx, 0, 0, ex.ctypes.data, ex.size),
            "preview": L.jsgpu_batch_preview(ctx, C.byref(pv)),
            "stage_ms": L.jsgpu_batch_stage_ms(ctx, ms.ctypes.data)}


def test_chunked_host_decode_leaves_the_layout_only(built):
    """After a device decode (so that the context has recorded stage events) a host decode of 24 images runs as image
    ranges on the chunk contexts: the layout and its statuses stay readable, every query of device-resident data answers
    JSGPU_ESTATE (stage_ms included: the context's events belong to the earlier decode), and a new batch_begin + decode
    restores them all."""
    from jpegsnoop_b200 import BatchDecoder
    jpegs = _jpegs(24)
    bd = BatchDecoder()
    tarr, darr, bits = bd.prepare(jpegs)
    bd.set_tables(tarr); bd.plan(darr, bits.size); bd.upload(bits); bd.decode(); bd.sync()
    assert bd.stage_ms()[4] > 0
    outs = _host_outputs(bd.layout, len(jpegs))
    bd.decode_host(darr, bits, outs)
    q = _queries(bd)
    assert q.pop("layout") == 0
    assert all(int(l.status) == 0 for l in bd.refresh_layout())
    assert q == dict.fromkeys(q, ESTATE), q
    msg = bd.L.jsgpu_last_error(bd.ctx).decode()
    assert "nothing decoded" in msg, msg
    bd.plan(darr, bits.size); bd.upload(bits); bd.decode(); bd.sync()
    q = _queries(bd)
    errors = q.pop("errors")
    assert q == dict.fromkeys(q, 0), q
    assert errors == ESTATE and "did not take the serial error path" in bd.L.jsgpu_last_error(bd.ctx).decode()


def test_single_stream_host_decode_keeps_the_batch(built):
    """Fewer than 16 images take one stream on the context itself: the decoded batch stays resident and downloadable."""
    from jpegsnoop_b200 import BatchDecoder
    jpegs = _jpegs(6)
    bd = BatchDecoder()
    tarr, darr, bits = bd.prepare(jpegs)
    bd.set_tables(tarr); bd.plan(darr, bits.size)
    outs = _host_outputs(bd.layout, len(jpegs))
    bd.decode_host(darr, bits, outs)
    for i in range(len(jpegs)):
        got, host = bd.fetch(i), bd.fetch_host(i, outs)
        assert np.array_equal(got.pix_y, host.pix_y) and np.array_equal(got.dib, host.dib), i
        assert np.array_equal(got.dht_histo, host.dht_histo) and np.array_equal(got.stats, host.stats), i
    q = _queries(bd)
    assert q.pop("errors") == ESTATE
    assert q == dict.fromkeys(q, 0), q
