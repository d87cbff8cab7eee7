"""CPU test of the build-time IDCT table generator (jpegsnoop_b200/csrc/tools/gen_idct_table.cpp): the literal
multiply-add / butterfly / correction sequence compiled into k_idct_tile<JS_TILE_INT_BAKED,*> equals the plain integer sums of the
reference's table, and the table itself equals the one the compiled reference computes (golden fixture)."""
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_baked_idct_sequence_equals_plain_sums(built, tmp_path):
    hdr_dir = os.path.join(ROOT, "jpegsnoop_b200", "csrc", "build")
    assert os.path.exists(os.path.join(hdr_dir, "idct_baked.h")), "build() writes build/idct_baked.h"
    exe = str(tmp_path / "check_idct_baked")
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", hdr_dir, "-o", exe, os.path.join(ROOT, "tests", "native", "check_idct_baked.cpp")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    lines = out.stdout.splitlines()
    assert out.returncode == 0 and lines[0].startswith("bad=0"), lines[0]
    li = np.array([int(x) for x in lines[1:4097]], np.int32).reshape(64, 64)
    gold = np.load(os.path.join(ROOT, "tests", "golden", "idct_tables.npz"))["li"].reshape(64, 64)
    # same libm here as where the fixture was made: the baked copy must match (elsewhere the runtime check in
    # jsgpu_set_idct_tables() selects the shared-memory-table kernel instead)
    assert np.array_equal(li, gold)
