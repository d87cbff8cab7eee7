"""Measure Extract All (jsgpu_find_markers, BatchDecoder.extract_all) on an H100, next to the compiled reference's walk.

One run builds two seeded inputs: a Motion-JPEG AVI of --frames 640x480 frames (tests/mjpg_corpus.py) and a --gib GiB container
of random bytes with one such frame every 64 MiB.  It records, as one JSON line (and in --out):
  * the GPU's name and power limit (nvidia-smi --query-gpu, read only);
  * per input: jsgpu_find_markers end to end from pageable memory (median of --runs calls), its k_find_all* kernels' device
    time for one call (torch.profiler CUDA activity) and that rate over the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s,
    the SOI and terminator counts, and extract_all end to end (median of --runs calls, the files written to a temporary
    directory and deleted);
  * jsgpu_host_copy_rate's pinned host-to-device ceiling;
  * the compiled reference (oracle/_ref/libn1_ref.so, when built): ProcessFile with the scan decode off (the marker walk and
    PASS 1) over each of the first --ref-frames frames of the AVI, passed on its own (the harness copies what it is given), and BufSearch for FF D8 FF over the first 64 MiB of the
    container, as bytes per second.
Usage: python tools/extract_all_probe.py [--frames 3000] [--gib 2] [--runs 3] [--ref-frames 200] [--out probe.json]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from find_probe import gpu_info  # noqa: E402

HBM_TBS = 3.35


def _median_wall(f, runs):
    walls = []
    for _ in range(runs):
        t0 = time.perf_counter(); f(); walls.append(time.perf_counter() - t0)
    return float(np.median(walls))


def measure(bd, buf, runs, name):
    from torch.profiler import profile, ProfilerActivity
    from test_extract_jpeg import find_markers
    n = buf.size
    r, ns, _, nt, _ = find_markers(bd, buf, soi_cap=n // 4096 + 1024, term_cap=n // 128 + 1024)   # warm-up
    assert r == 0
    res = {"bytes": n, "soi": ns, "terminators": nt}
    s = _median_wall(lambda: find_markers(bd, buf, soi_cap=n // 4096 + 1024, term_cap=n // 128 + 1024), runs)
    res["find_markers_s_median"] = s
    res["find_markers_e2e_gbs"] = n / s / 1e9
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        find_markers(bd, buf, soi_cap=n // 4096 + 1024, term_cap=n // 128 + 1024)
    kern = sum(e.device_time_total for e in prof.events() if "k_find_all" in e.name) / 1e6
    res["kernel_s"] = kern
    res["kernel_gbs"] = n / kern / 1e9 if kern else None
    res["kernel_of_hbm_datasheet"] = (n / kern / 1e12) / HBM_TBS if kern else None
    tmp = tempfile.mkdtemp(prefix=f"extract_{name}_")
    written = []

    def run():
        frames, _ = bd.extract_all(buf, os.path.join(tmp, "out.log"))
        written.append(sum(p is not None for _, p in frames))
    try:
        run()
        res["extract_all_s_median"] = _median_wall(run, runs)
        res["extract_all_frames_written"] = written[-1]
        res["extract_all_e2e_gbs"] = n / res["extract_all_s_median"] / 1e9
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return res


def reference(avi, offs, box, nframes):
    from find_oracle import RefN1, ref_available, ref_bufsearch
    if not ref_available():
        return "not measured (compiled reference not built)"
    r = RefN1()
    r.L.n1_config(0, 1)
    k = min(nframes, len(offs) - 1)
    chunks = [np.frombuffer(avi[offs[i]:offs[i + 1]], np.uint8).copy() for i in range(k)]   # each frame walked from its SOI
    t0 = time.perf_counter()
    for c in chunks:
        r.process(c, 0)
    walk = time.perf_counter() - t0
    pre = np.frombuffer(bytes(box[:64 << 20]), np.uint8).copy()
    pre[pre == 0xD8] = 0xD9                   # no FF D8 FF: the search runs to the end
    t0 = time.perf_counter()
    ref_bufsearch(pre, 0, 0xFFD8FF, 3, True)
    srch = time.perf_counter() - t0
    r.close()
    return {"process_file_frames": k, "process_file_bytes": int(offs[k] - offs[0]),
            "process_file_gbs": (offs[k] - offs[0]) / walk / 1e9, "bufsearch_bytes": pre.size, "bufsearch_gbs": pre.size / srch / 1e9}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3000)
    ap.add_argument("--gib", type=float, default=2.0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--ref-frames", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    import torch
    import jpeg_cases as JC
    import mjpg_corpus as M
    from jpegsnoop_b200 import BatchDecoder

    frames = [M.to_mjpg(JC.enc(JC.synth_rgb(640, 480, 4000 + k), quality=85, subsampling=2)) for k in range(64)]
    avi, offs = M.avi([frames[k % 64] for k in range(a.frames)], 640, 480)
    n = int(a.gib * (1 << 30))
    box = np.random.default_rng(7).integers(0, 256, n, dtype=np.uint8)
    for k, p in enumerate(range(1 << 20, n - (1 << 20), 64 << 20)):
        f = np.frombuffer(frames[k % 64], np.uint8)
        box[p:p + f.size] = f
    torch.cuda.init()
    bd = BatchDecoder()
    res = {"gpu": gpu_info(), "runs": a.runs}
    res["avi"] = measure(bd, np.frombuffer(avi, np.uint8), a.runs, "avi")
    res["container"] = measure(bd, box, a.runs, "box")
    res["host_copy_h2d_gbs"] = bd.host_copy_rate(direction=0, nbytes=1 << 30, reps=3)
    res["reference"] = reference(avi, offs, box, a.ref_frames)
    bd.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
