"""Time of jsgpu_batch_decode with a "Detailed Decode" of the LAST MCU row of a 3840x2160 4:2:0 frame (240 MCUs), without restart
markers and with DRI = 8, on the parallel path (one thread per MCU, jsgpu_detail.cu) and on the serial walk (JSGPU_DETAIL_WALK=1,
jsgpu_exact.cu), next to the same decode without the detailed decode.  Each configuration runs in a child process (the variable
is read once per process); the decode is timed with the context's CUDA events around decode + sync, after warm-up.

    python tools/detail_probe.py [--reps 20] [--out detail_probe.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import numpy as np
from jpegsnoop_b200 import BatchDecoder, synth
ri, detail, reps = int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4])
j = synth.encode(3840, 2160, "420", 85, ri, False, seed=7)
bd = BatchDecoder(); bd.set_batch([j])
if detail:
    bd.set_detail(0, 0, 134, 240)                       # the last MCU row (2160 / 16 = 135 rows)
ms = []
for i in range(reps + 3):
    bd.timer_start(); bd.decode(); bd.sync(); t = bd.timer_stop()
    if i >= 3:
        ms.append(t)
out = {"ri": ri, "detail": detail, "ms": ms, "median_ms": float(np.median(ms)), "min_ms": float(np.min(ms))}
if detail:
    nev, nblk, path = bd.detail_info(); out.update(events=nev, blocks=nblk, path=path)
print(json.dumps(out))
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "runs": []}
    for ri in (0, 8):
        for mode in ("none", "parallel", "serial"):
            env = dict(os.environ)
            env.pop("JSGPU_DETAIL_WALK", None)
            if mode == "serial":
                env["JSGPU_DETAIL_WALK"] = "1"
            r = subprocess.run([sys.executable, "-c", CHILD, ROOT, str(ri), str(int(mode != "none")), str(a.reps)],
                               env=env, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(r.stderr[-3000:])
            o = json.loads(r.stdout.strip().splitlines()[-1]); o["mode"] = mode
            res["runs"].append(o)
            print(f"DRI={ri} {mode:9s} median {o['median_ms']:8.3f} ms  min {o['min_ms']:8.3f} ms"
                  + (f"  events {o['events']} blocks {o['blocks']} path {o['path']}" if mode != "none" else ""))
    print("GPU:", gpu)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
