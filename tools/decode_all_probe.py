"""Measure finding and decoding every JPEG in a Motion-JPEG AVI (jsgpu_find_all, BatchDecoder.decode_all) on an H100.

One run builds a seeded MJPG AVI (--distinct Pillow frames of --size pixels, 4:2:0, turned into AVI1 frames without DHT and
repeated to --frames frames, tests/mjpg_corpus.py) and records, as one JSON line (and in --out):
  * the GPU's name and power limit (nvidia-smi --query-gpu, read only);
  * the find_all kernels' device time for one call over the container (torch.profiler CUDA activity, every k_find_all*
    kernel), the bytes searched per second and that rate over the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s;
  * the end-to-end find_all rate: the median wall time of --runs calls from pageable memory;
  * decode_all: the median wall time of --runs calls, frames/s and GPix/s (SOF pixels), images redone, bytes uploaded.
Usage: python tools/decode_all_probe.py [--frames 3000] [--distinct 64] [--size 640x480] [--runs 3] [--out probe.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from find_probe import gpu_info  # noqa: E402

HBM_TBS = 3.35


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3000)
    ap.add_argument("--distinct", type=int, default=64)
    ap.add_argument("--size", default="640x480")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    import jpeg_cases as JC
    import mjpg_corpus as M
    from jpegsnoop_b200 import BatchDecoder

    W, H = (int(v) for v in a.size.split("x"))
    frames = [M.to_mjpg(JC.enc(JC.synth_rgb(W, H, 4000 + k), quality=85, subsampling=2)) for k in range(a.distinct)]
    avi, offs = M.avi([frames[k % a.distinct] for k in range(a.frames)], W, H)
    buf = np.frombuffer(avi, np.uint8)
    n = buf.size
    bd = BatchDecoder()
    torch.cuda.init()
    count, _ = bd.find_all(buf)                                         # warm-up: streams, staging buffers
    assert count == len(offs), (count, len(offs))
    res = {"gpu": gpu_info(), "bytes": n, "frames": a.frames, "frame_size": a.size, "runs": a.runs}

    walls = []
    for _ in range(a.runs):
        t0 = time.perf_counter(); bd.find_all(buf); walls.append(time.perf_counter() - t0)
    res["find_all_s_median"] = float(np.median(walls))
    res["find_all_e2e_gbs"] = n / res["find_all_s_median"] / 1e9
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bd.find_all(buf)
    kern = sum(e.device_time_total for e in prof.events() if "k_find_all" in e.name) / 1e6
    res["find_all_kernel_s"] = kern
    res["find_all_kernel_gbs"] = n / kern / 1e9 if kern else None
    res["find_all_kernel_of_hbm_datasheet"] = (n / kern / 1e12) / HBM_TBS if kern else None

    entries, info = bd.decode_all(buf)                                  # warm-up
    assert len(entries) == len(offs) and all(img is not None for _, _, img in entries)
    walls = []
    for _ in range(a.runs):
        t0 = time.perf_counter(); entries, info = bd.decode_all(buf); walls.append(time.perf_counter() - t0)
    med = float(np.median(walls))
    res["decode_all_s_median"] = med
    res["decode_all_s_all"] = [round(w, 4) for w in walls]
    res["decode_all_frames_per_s"] = len(offs) / med
    res["decode_all_gpix_per_s"] = len(offs) * W * H / med / 1e9
    res["redone"] = info["redone"]
    res["uploaded_bytes"] = info["uploaded"]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
