"""TEST INFRASTRUCTURE: decode a batch in a process of its own, so that the stage-A form variables (JSGPU_MARKER,
JSGPU_UNSTUFF), which the library reads once per process, can be set for it.

    python stage_a_child.py IN.npz OUT.npz HUFF...

IN.npz holds the JPEGs (`jpegs`, an object array of bytes).  For each huff_kernel in HUFF the batch is decoded once, with
the MCU file map, and OUT.npz receives `ck_<huff>` (jsgpu_batch_checksums) and, per image i, `<field>_<huff>_<i>` for the
fetched buffers and the status word."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402


def main(argv):
    from jpegsnoop_b200 import BatchDecoder
    src, dst, huffs = argv[0], argv[1], [int(h) for h in argv[2:]]
    jpegs = [bytes(j) for j in np.load(src, allow_pickle=True)["jpegs"]]
    out = {}
    for h in huffs:
        bd = BatchDecoder(huff_kernel=h, idct_kernel=0)
        bd.set_batch(jpegs); bd.decode(); bd.sync()
        out[f"ck_{h}"] = bd.checksums()
        for i in range(len(jpegs)):
            d = bd.fetch(i)
            for f in ("pix_y", "dib", "mcu_map", "dht_histo", "stats"):
                out[f"{f}_{h}_{i}"] = getattr(d, f)
            out[f"blk_y_{h}_{i}"] = d.blk_dc[0]
            out[f"status_{h}_{i}"] = np.array([d.status], np.uint32)
        bd.close()
    np.savez(dst, **out)


if __name__ == "__main__":
    main(sys.argv[1:])
