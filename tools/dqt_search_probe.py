"""Measure the GPU "Search Executable for DQT" (jsgpu_search_bytes) on an H100.

One run records, as one JSON line (and in --out):
  * the GPU's name and power limit (nvidia-smi --query-gpu, read only);
  * the search kernels' device time from CUDA activity records (torch.profiler) for one call over a seeded 2 GiB file with
    planted tables and all 20 DQT search patterns: bytes/s and its share of the 3.35 TB/s data-sheet HBM bandwidth;
  * end-to-end bytes/s of the call from pageable host memory, next to jsgpu_host_copy_rate's pinned host-to-device ceiling;
  * the compiled reference's BufSearchX loop on a 64 MiB prefix, one pattern (where oracle/_ref exists).
Usage: python tools/dqt_search_probe.py [--gib 2] [--out dqt_search_probe.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_TBS = 3.35          # H100 SXM data sheet


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    import dqt_oracle as D
    from jpegsnoop_b200 import BatchDecoder
    from test_dqt_search import all_forms, q75_table, STD_LUM

    n = int(a.gib * (1 << 30))
    rng = np.random.default_rng(2026)
    data = rng.integers(0, 256, n, dtype=np.uint8)
    pats = [p for p in all_forms(STD_LUM) + all_forms(q75_table())]
    pats = list(dict.fromkeys(pats))[:20]
    for i, at in enumerate(rng.integers(1, n - 1024, 200)):
        p = pats[i % len(pats)]
        data[at:at + len(p)] = np.frombuffer(p, np.uint8)
    bd = BatchDecoder()
    torch.cuda.init()
    counts, _ = bd.search_bytes(data[: 64 << 20], pats, cap=1 << 16)           # warm-up: buffers, pinned staging
    walls = []
    for _ in range(3):
        t0 = time.perf_counter(); counts, _ = bd.search_bytes(data, pats, cap=1 << 16); walls.append(time.perf_counter() - t0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bd.search_bytes(data, pats, cap=1 << 16)
    kern = {}
    for e in prof.events():
        if "k_search" in e.name:                                # kernel records (device time in microseconds)
            name = e.name.split("(")[0]
            kern[name] = kern.get(name, 0.0) + e.device_time_total / 1e6
    tiles = sum(v for k, v in kern.items() if "k_search_tiles" in k)
    ktot = sum(kern.values())
    h2d = bd.host_copy_rate(direction=0, nbytes=1 << 30, reps=3)
    res = {"gpu": gpu_info(), "bytes": n, "patterns": len(pats), "matches": int(counts.sum()),
           "kernel_s": ktot, "kernel_gbs": n / ktot / 1e9 if ktot else None,
           "kernel_frac_hbm": (n / ktot / 1e12) / HBM_TBS if ktot else None,
           "tile_kernel_s": tiles, "kernels": {k: round(v, 6) for k, v in kern.items()},
           "e2e_s_best": min(walls), "e2e_gbs": n / min(walls) / 1e9, "h2d_pinned_gbs": h2d}
    if D.ref_available():
        pre = data[: 64 << 20].copy()
        t0 = time.perf_counter(); r = D.ref_bufsearch_all(pre, pats[0]); t = time.perf_counter() - t0
        res["ref_64mib_one_pattern_s"] = t
        res["ref_bytes_per_s_per_pattern"] = pre.size / t
        res["ref_matches"] = len(r)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
