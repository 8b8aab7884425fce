"""gpdb_preprocess_depth_organized against gpdb_preprocess_depth on depth views in device memory: time per call (CUDA
events around the call, median of the timed repeats after warm-up), the fallback fraction, and the card's power limit
and SM clock read in the same run. Workloads: B = 16 / 64 / 256 views of one 640 x 480 camera, B = 16 views of two
cameras, and a single view (latency). Usage: python tools/bench_organized.py [out.jsonl]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def main():
    import torch

    import depth_reference as dr
    from gpd_b200 import lib
    out = sys.argv[1] if len(sys.argv) > 1 else None
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = lib.Context(lib.default_params())
    pp = lib.preprocess_params()
    rows = []
    for B, K in [(1, 1), (16, 1), (64, 1), (256, 1), (16, 2)]:
        view = dr.render_views([7], [K], 0, n_points=200000, width=640, height=480, f=520.0)[0]
        cams = [c for _, c in view] * B
        depth = torch.from_numpy(np.concatenate([img.ravel() for img, _ in view] * B).view(np.int16)).cuda()
        res = {}
        for name, fn in (("depth", lambda: ctx.preprocess_depth_tensors([K] * B, cams, depth, pp)),
                         ("organized", lambda: ctx.preprocess_depth_organized_tensors([K] * B, cams, depth, pp))):
            r = fn()  # warm-up: module load, scratch growth
            ts = []
            for _ in range(5):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                r = fn()
                b.record()
                torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
            res[name] = float(np.median(ts))
            if name == "organized":
                poff, fb = r
                res["fallback_fraction"] = float(fb.sum()) / max(int(poff[-1]), 1)
        row = {"views": B, "cameras": K, "image": "640x480", "ms_depth": round(res["depth"], 3),
               "ms_organized": round(res["organized"], 3), "fallback_fraction": round(res["fallback_fraction"], 4),
               "gpu": gpu}
        print(json.dumps(row), flush=True)
        rows.append(row)
    if out:
        with open(out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in rows))
    ctx.close()


if __name__ == "__main__":
    main()
