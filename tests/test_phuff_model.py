"""CPU: the self-synchronising Huffman passes (long restart intervals, BASELINE config 5).  The per-slot code of the
CUDA kernels (jpegsnoop_b200/csrc/jsgpu_phuff_core.cuh) is compiled for the host together with an independent
sequential walk (tests/native/phuff_model.cpp) and must produce virtual restart intervals that start at the true MCU
bit positions with the true DC predictors and tile every real interval — for every execution order of the slots."""
import ctypes as C
import os
import subprocess
import numpy as np
import pytest

import jpeg_cases as JC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def model(built, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("phm") / "libphuff_model.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I/usr/local/cuda/include", "-o", so,
                    os.path.join(ROOT, "tests", "native", "phuff_model.cpp")], check=True)
    L = C.CDLL(so)
    L.phm_check.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p]
    return L


def _cases():
    import mini_jpeg as MJ
    ac_fit = MJ.long_code_table(MJ.all_ac_symbols(), n11=8)
    return [
        ("420_norst_1080p", JC.enc(JC.synth_rgb(1920, 1080, 31), quality=85, subsampling=2)),
        ("444_norst_q95", JC.enc(JC.synth_rgb(640, 480, 32), quality=95, subsampling=0)),
        ("422_opt_norst", JC.enc(JC.synth_rgb(800, 600, 33), quality=60, subsampling=1, optimize=True)),
        ("gray_norst_q30", JC.enc(JC.synth_rgb(1024, 768, 34)[:, :, 0], quality=30)),
        ("420_rst_2rows_4kstrip", JC.enc(JC.synth_rgb(3840, 128, 35), quality=85, subsampling=2, restart_marker_rows=2)),
        ("420_norst_odd", JC.enc(JC.synth_rgb(333, 211, 4), quality=92, subsampling=2)),
        ("mini_411_norst", MJ.encode(JC.synth_rgb(400, 304, 36), quality=75, samp=((4, 1), (1, 1), (1, 1)))),
        ("mini_longcodes_fit_420_norst", MJ.encode(JC.synth_rgb(320, 176, 22), quality=90, samp=((2, 2), (1, 1), (1, 1)), ac_tabs=[ac_fit, ac_fit])),
        ("420_norst_flat", JC.enc(np.full((480, 640, 3), 128, np.uint8), quality=85, subsampling=2)),           # ~10 bits per MCU: hundreds of MCUs per slot
        ("444_q100_noise", JC.enc(np.random.default_rng(7).integers(0, 256, (96, 128, 3), dtype=np.uint8).astype(np.uint8), quality=100, subsampling=0)),   # MCUs longer than a slot? (close)
    ]


@pytest.mark.parametrize("order", [0, 1, 2], ids=["descending", "ascending", "shuffled"])
def test_virtual_intervals_match_a_sequential_walk(model, order):
    from jpegsnoop_b200.host import parse_jpeg
    for name, j in _cases():
        t, d, start = parse_jpeg(j)
        scan = np.frombuffer(j, np.uint8)[start:].copy()
        out = np.zeros(32, np.uint32)
        r = model.phm_check(C.byref(t), C.byref(d), scan.ctypes.data, scan.size, order, out.ctypes.data)
        assert r == 0, (name, r)
        bad, rounds, used, nv, guessed, covered = [int(v) for v in out[:6]]
        hmax = max(d.samp_h[:d.num_sos_comps]) if d.num_sos_comps == 3 else 1
        vmax = max(d.samp_v[:d.num_sos_comps]) if d.num_sos_comps == 3 else 1
        nmcu = -(-d.dim_x // (8 * hmax)) * -(-d.dim_y // (8 * vmax))
        assert bad == 0, (name, bad)
        assert covered == nmcu, (name, covered, nmcu)
        # typical content settles in a couple of rounds; components that share their Huffman tables (the block phase is
        # not observable, "mini_*") or near-random data at q100 settle slowly: correct, but through k_ph_fix_cta
        if not name.startswith("mini_") and "q100" not in name:
            assert rounds <= 4, (name, rounds)
        print(f"{name}: {used} slots, {nv} virtual intervals, guess right for {guessed}, {rounds} fix rounds")
