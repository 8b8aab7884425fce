#!/usr/bin/env python
"""Generate tests/golden/model_skeletons.npz: the reference's own model files (two Caffe .caffemodel, one OpenVINO IR
.bin + .xml), 14 MB each, reduced to what the weights in gpd_b200/weights/lenet_{15,3,12}ch.npz do not already hold.

Almost every byte of such a file is the eight weight arrays as packed float32 in the framework's order. For each file the
fixture stores the remaining bytes (the protobuf records around the payloads, ~850 B; the IR .xml), where each payload goes,
and the SHA-256 of the original file, so that tests/test_weights_io.py can rebuild the file exactly and parse the real thing.
Needs the reference's model directory (REF below)."""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from test_weights_io import MODEL_FILES, NAMES, framework_order  # noqa: E402

REF = "/root/reference/models"
OUT = os.path.join(ROOT, "tests", "golden", "model_skeletons.npz")


def main():
    out = {}
    for key, (ch, rel) in MODEL_FILES.items():
        data = open(os.path.join(REF, rel), "rb").read()
        z = np.load(os.path.join(ROOT, "gpd_b200", "weights", f"lenet_{ch}ch.npz"))
        skeleton, offsets, pos = bytearray(), [], 0
        for a in framework_order([z[n] for n in NAMES]):  # the payloads lie in this order in all three files
            b = a.tobytes()
            i = data.find(b, pos)
            assert i >= 0 and data.find(b, i + 1) < 0, (rel, "payload not found exactly once, in order")
            skeleton += data[pos:i]
            offsets.append(len(skeleton))  # where the payload goes in the skeleton
            pos = i + len(b)
        skeleton += data[pos:]
        out[key + "_skeleton"] = np.frombuffer(bytes(skeleton), np.uint8)
        out[key + "_offsets"] = np.array(offsets, np.int64)
        out[key + "_sha256"] = np.array(hashlib.sha256(data).hexdigest())
        if rel.endswith(".bin"):
            out[key + "_xml"] = np.frombuffer(open(os.path.join(REF, rel[:-4] + ".xml"), "rb").read(), np.uint8)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
