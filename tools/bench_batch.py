"""Throughput of many small clouds: one gpdb_detect_batch call against a loop of gpdb_set_cloud + gpdb_detect.

Workload (the reference's data generation and labelling: one view at a time, 500 samples per view): B synthetic table
scenes of 20 000 voxelised points, 500 samples each, 15-channel images, the shipped 15-channel LeNet. For B in
{1, 16, 64, 256} it prints one JSON line per B with samples/s of
  - resident: the detect calls alone (the batch already installed; in the loop, the gpdb_detect calls only),
  - e2e: installing the clouds as well (gpdb_set_clouds + gpdb_detect_batch, or every gpdb_set_cloud + gpdb_detect),
the median over --reps repetitions after one warm-up, and the GPU name and power limit. Needs a GPU.

--raw starts from raw views instead: B views of synthetic_raw_scene(1000 + i, n_points=20000), default preprocessing
parameters, 500 samples per view (fewer when a view keeps fewer points), and times three routes per B:
  (a) loop: gpdb_preprocess + gpdb_detect per view,
  (b) today's batch route: gpdb_preprocess + gpdb_get_cloud per view, then gpdb_set_clouds + gpdb_detect_batch,
  (c) gpdb_preprocess_clouds + gpdb_detect_batch,
with the preprocessing alone of (a) and (c) and the device stage times of (c)'s gpdb_preprocess_clouds
(gpdb_preprocess_timings). It checks once, outside the timed region, that (a) and (c) give identical flags and scores.

    python tools/bench_batch.py [--sizes 1 16 64 256] [--reps 3] [--raw]
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


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def raw_loop(ctx, views, pp, samples, keep=False):
    """Route (a): (preprocessing time, whole time[, per-view (flags, scores)])."""
    t_pre, out = 0.0, []
    t0 = time.perf_counter()
    for v, s in zip(views, samples):
        t1 = time.perf_counter()
        ctx.preprocess(v["xyz"], v["cam_source"], v["view_points"], pp, read_back=False)
        t_pre += time.perf_counter() - t1
        res = abi.Result()
        ctx.detect_raw(s, res)
        if keep:
            r = abi.result_to_numpy(res, 0)
            out.append((r["pose_flags"], r["pose_scores"]))
        lib.free_result(res)
    return t_pre, time.perf_counter() - t0, out


def raw_roundtrip(ctx, views, pp, offsets, sidx):
    """Route (b): preprocess + read back every view, then install the batch and detect."""
    t0 = time.perf_counter()
    clouds = []
    for v in views:
        n = ctx.preprocess(v["xyz"], v["cam_source"], v["view_points"], pp, read_back=False)
        k = len(v["view_points"])
        c = {"xyz": np.empty((n, 3), np.float32), "normals": np.empty((n, 3)), "cam_source": np.empty((n, k), np.int32),
             "view_points": v["view_points"]}
        lib.lib().gpdb_get_cloud(ctx.h, _p(c["xyz"]), _p(c["normals"]), _p(c["cam_source"]))
        clouds.append(c)
    ctx.set_clouds(clouds)
    res, coff = abi.Result(), np.zeros(len(offsets), np.int32)
    ctx.detect_batch_raw(offsets, sidx, res, coff)
    t = time.perf_counter() - t0
    lib.free_result(res)
    return t


def raw_batch(ctx, views, pp, offsets, sidx, keep=False):
    """Route (c): (preprocessing time, whole time[, per-view (flags, scores)])."""
    t0 = time.perf_counter()
    ctx.preprocess_clouds(views, pp, read_back=False)
    t_pre = time.perf_counter() - t0
    res, coff = abi.Result(), np.zeros(len(offsets), np.int32)
    ctx.detect_batch_raw(offsets, sidx, res, coff)
    t = time.perf_counter() - t0
    out = []
    if keep:
        r = abi.result_to_numpy(res, 0)
        out = [(v["pose_flags"], v["pose_scores"]) for v in lib.split_batch_result(r, offsets, coff)]
    lib.free_result(res)
    return t_pre, t, out


def main_raw(a, ctx, gpu):
    pp = lib.preprocess_params()
    pool = []
    for i in range(max(a.sizes)):
        s = scenes.synthetic_raw_scene(1000 + i, n_points=N_POINTS)
        pool.append({"xyz": s["xyz"], "cam_source": s["cam_source"], "view_points": s["view_points"]})
    med = lambda v: float(np.median(v))  # noqa: E731
    for B in a.sizes:
        views = pool[:B]
        poff = ctx.preprocess_clouds(views, pp, read_back=False)
        samples = [np.random.default_rng(i).choice(int(poff[i + 1] - poff[i]), min(N_SAMPLES, int(poff[i + 1] - poff[i])),
                                                   replace=False).astype(np.int32) for i in range(B)]
        offsets, sidx = lib.pack_samples(samples)
        n = int(offsets[-1])
        # warm-up of every shape, and the one check that routes (a) and (c) compute the same
        _, _, ra = raw_loop(ctx, views, pp, samples, keep=True)
        _, _, rc = raw_batch(ctx, views, pp, offsets, sidx, keep=True)
        for (fa, sa), (fc, sc) in zip(ra, rc):
            assert np.array_equal(fa, fc) and sa.tobytes() == sc.tobytes(), "routes (a) and (c) differ"
        raw_roundtrip(ctx, views, pp, offsets, sidx)
        ta, tap, tb, tc, tcp, stages = [], [], [], [], [], []
        for _ in range(a.reps):
            pa, wa, _ = raw_loop(ctx, views, pp, samples)
            tb.append(raw_roundtrip(ctx, views, pp, offsets, sidx))
            pc, wc, _ = raw_batch(ctx, views, pp, offsets, sidx)
            stages.append(ctx.preprocess_timings())
            ta.append(wa)
            tap.append(pa)
            tc.append(wc)
            tcp.append(pc)
        st = np.median(np.array(stages), axis=0)
        print(json.dumps({"mode": "raw", "B": B, "raw_points": sum(len(v["xyz"]) for v in views), "processed_points": int(poff[-1]), "samples": n,
                          "a_loop_ms": round(1e3 * med(ta), 2), "b_roundtrip_ms": round(1e3 * med(tb), 2),
                          "c_batch_ms": round(1e3 * med(tc), 2), "a_pre_ms": round(1e3 * med(tap), 2),
                          "c_pre_ms": round(1e3 * med(tcp), 2), "a_sps": round(n / med(ta)), "b_sps": round(n / med(tb)),
                          "c_sps": round(n / med(tc)),
                          "c_pre_stages_ms": dict(zip(("upload", "filter", "voxelise", "grid", "normals", "device_total"),
                                                      [round(float(x), 3) for x in st])),
                          "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--raw", action="store_true", help="start from raw views: three preprocessing + detection routes")
    a = ap.parse_args()
    w, relu = weights()
    if a.raw:
        ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
        ctx.set_weights(w)
        main_raw(a, ctx, gpu_info())
        ctx.close()
        return
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
