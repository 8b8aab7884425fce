"""Throughput of many small clouds: one gpdb_detect_batch call against a loop of gpdb_set_cloud + gpdb_detect.

Workload (the reference's data generation and labelling: one view at a time, 500 samples per view): B synthetic table
scenes of 20 000 voxelised points, 500 samples each, 15-channel images, the shipped 15-channel LeNet. For B in
{1, 16, 64, 256} it prints one JSON line per B with samples/s of
  - resident: the detect calls alone (the batch already installed; in the loop, the gpdb_detect calls only),
  - e2e: installing the clouds as well (gpdb_set_clouds + gpdb_detect_batch, or every gpdb_set_cloud + gpdb_detect),
the median over --reps repetitions after one warm-up, and the GPU name and power limit. Needs a GPU.

    python tools/bench_batch.py [--sizes 1 16 64 256] [--reps 3]
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

from gpd_b200 import abi, lib, scenes  # noqa: E402

N_POINTS, N_SAMPLES = 20000, 500


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def weights():
    z = np.load(os.path.join(ROOT, "gpd_b200", "weights", "lenet_15ch.npz"))
    return [z[n] for n in ("conv1_weights", "conv1_biases", "conv2_weights", "conv2_biases", "ip1_weights", "ip1_biases",
                                        "ip2_weights", "ip2_biases")], int(z["relu_after_conv"])


def run_batch(ctx, clouds, offsets, sidx, install):
    res, coff = abi.Result(), np.zeros(len(offsets), np.int32)
    t0 = time.perf_counter()
    if install:
        ctx.set_clouds(clouds)
    ctx.detect_batch_raw(offsets, sidx, res, coff)
    t = time.perf_counter() - t0
    lib.free_result(res)
    return t


def run_loop(ctx, clouds, samples):
    """(time of the gpdb_detect calls, time of the whole loop)."""
    t_det = 0.0
    t0 = time.perf_counter()
    for c, s in zip(clouds, samples):
        ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        res = abi.Result()
        t1 = time.perf_counter()
        ctx.detect_raw(s, res)
        t_det += time.perf_counter() - t1
        lib.free_result(res)
    return t_det, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    w, relu = weights()
    ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    ctx.set_weights(w)
    pool = [scenes.synthetic_table_scene(1000 + i, n_points=N_POINTS) for i in range(max(a.sizes))]
    gpu = gpu_info()
    for B in a.sizes:
        clouds = pool[:B]
        samples = [np.random.default_rng(i).choice(N_POINTS, N_SAMPLES, replace=False).astype(np.int32) for i in range(B)]
        offsets, sidx = lib.pack_samples(samples)
        n = B * N_SAMPLES
        ctx.set_clouds(clouds)
        run_batch(ctx, clouds, offsets, sidx, False)  # warm-up of every shape
        run_loop(ctx, clouds, samples)
        rb, eb, rl, el = [], [], [], []
        for _ in range(a.reps):
            eb.append(run_batch(ctx, clouds, offsets, sidx, True))
            rb.append(run_batch(ctx, clouds, offsets, sidx, False))
            d, e = run_loop(ctx, clouds, samples)
            rl.append(d)
            el.append(e)
        med = lambda v: float(np.median(v))  # noqa: E731
        print(json.dumps({"B": B, "samples": n, "batch_resident_sps": round(n / med(rb)), "loop_resident_sps": round(n / med(rl)),
                          "batch_e2e_sps": round(n / med(eb)), "loop_e2e_sps": round(n / med(el)),
                          "batch_resident_ms": round(1e3 * med(rb), 2), "loop_resident_ms": round(1e3 * med(rl), 2),
                          "batch_e2e_ms": round(1e3 * med(eb), 2), "loop_e2e_ms": round(1e3 * med(el), 2), "gpu": gpu}),
              flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
