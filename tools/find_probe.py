"""Measure Img Search Fwd / Rev (jsgpu_find_value) on an H100.

One run records, as one JSON line (and in --out):
  * the GPU's name and power limit (nvidia-smi --query-gpu, read only);
  * forward and reverse searches for FF D8 FF over a seeded 2 GiB buffer whose only match is at the far end of the search
    (forward from 0 to a match 100 bytes before the end, reverse from the end to a match at byte 100), from pageable and
    from pinned host memory: the median wall time of --runs calls each and the bytes searched per second;
  * the search kernel's device time for one forward call from CUDA activity records (torch.profiler);
  * jsgpu_host_copy_rate's pinned host-to-device ceiling.
Usage: python tools/find_probe.py [--gib 2] [--runs 5] [--out find_probe.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SOI3 = 0xFFD8FF


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
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    from jpegsnoop_b200 import BatchDecoder
    from jpegsnoop_b200 import _lib as B

    n = int(a.gib * (1 << 30))
    rng = np.random.default_rng(2026)
    pageable = rng.integers(0, 255, n, dtype=np.uint8)               # no 0xFF: the planted SOI is the only match
    L = B.load()
    pp = L.jsgpu_host_alloc(n)
    if not pp:
        raise RuntimeError("pinned allocation failed")
    pinned = np.ctypeslib.as_array(C.cast(pp, C.POINTER(C.c_uint8)), shape=(n,))
    pinned[:] = pageable
    bd = BatchDecoder()
    torch.cuda.init()
    bd.find_value(pageable[: 64 << 20], 0, SOI3, 3, True)              # warm-up: streams, staging buffers
    res = {"gpu": gpu_info(), "bytes": n, "runs": a.runs}
    try:
        for direction, fwd, at, start in (("forward", True, n - 100, 0), ("reverse", False, 100, n)):
            for buf_name, buf in (("pageable", pageable), ("pinned", pinned)):
                buf[at:at + 3] = (0xFF, 0xD8, 0xFF)
                walls = []
                for _ in range(a.runs):
                    t0 = time.perf_counter()
                    found, pos = bd.find_value(buf, start, SOI3, 3, fwd)
                    walls.append(time.perf_counter() - t0)
                    assert found and pos == at, (direction, buf_name, found, pos)
                buf[at:at + 3] = 0
                med = float(np.median(walls))
                searched = (at - start) if fwd else (start - at)
                res[f"{direction}_{buf_name}_s_median"] = med
                res[f"{direction}_{buf_name}_s_all"] = [round(w, 4) for w in walls]
                res[f"{direction}_{buf_name}_gbs"] = searched / med / 1e9
        pageable[n - 100:n - 97] = (0xFF, 0xD8, 0xFF)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            bd.find_value(pageable, 0, SOI3, 3, True)
        kern = sum(e.device_time_total for e in prof.events() if "k_find_value" in e.name) / 1e6
        res["kernel_s_forward"] = kern
        res["kernel_gbs_forward"] = (n - 100) / kern / 1e9 if kern else None
        res["h2d_pinned_gbs"] = bd.host_copy_rate(direction=0, nbytes=1 << 30, reps=3)
    finally:
        del pinned
        L.jsgpu_host_free(pp)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
