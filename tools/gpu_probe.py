"""Scratch GPU probe: small batch timing across kernel variants (not a bench)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
from jpegsnoop_b200 import BatchDecoder, synth
n = int(sys.argv[1]) if len(sys.argv) > 1 else 16
variants = [tuple(int(x) for x in v.split(",")) for v in sys.argv[2:]] or [(1, 1), (2, 3)]
t = time.time()
specs = [dict(width=1920, height=1080, subsampling="420", quality=85, restart_interval=4, optimize=False, seed=2000 + i) for i in range(n)]
buf, offs = synth.encode_batch(specs)
jpegs = [buf[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]
print("encode s %.2f" % (time.time() - t), "bytes/img", len(jpegs[0]))
for hk, ik in variants:
    bd = BatchDecoder(huff_kernel=hk, idct_kernel=ik, want_histo=False)
    t = time.time(); bd.set_batch(jpegs); print("set_batch s %.2f" % (time.time() - t))
    for it in range(3):
        bd.decode(); bd.sync()
        ms = bd.stage_ms()
        mpix = bd.nsof_pixels / 1e6
    print(f"huff={hk} idct={ik} stage ms {np.round(ms,3)}  -> {mpix/(ms[4]/1e3)/1e3:.2f} GPix/s  launches {bd.launches()}  idct GB/s {bd.npadded_pixels*13/ms[2]/1e6:.0f}")
    st = [l.status for l in bd.refresh_layout()]
    print("status", set(st))
    bd.close()
