"""The statistical outlier removal (gpdb_remove_outliers_clouds / gpdb_remove_outliers) on the device, against the
preprocessing of the same views and the numpy restatement on the CPU.

Workload: B in {16, 64, 256} raw views synthetic_raw_scene(1000 + i, n_points=20000) (the views of tools/bench_refine.py
and tools/bench_plane.py), preprocessed once with preprocess_clouds_tensors (default parameters), then
remove_outliers_clouds; and the config-3 cloud (synthetic_raw_scene(0)) through gpdb_preprocess + gpdb_remove_outliers;
each at mean_k = 50, stddev_mul = 1.0. The call removes points from the store it reads, so every timed call first
reinstalls the processed clouds (outside the timed window). Each JSON line gives, for one workload: the median (and
min / max) device time of the whole call and of preprocessing over --reps runs (CUDA events, after one warm-up), the
device time of each kernel from a separate torch.profiler run (the kNN is k_refine_knn, the scan cub's), the kept
fraction, the numpy restatement (tests/outliers_reference.py) on the first --cpu-views views (scaled to B; checked equal
to the device's kept bytes; not run on the config-3 cloud), and the GPU name and power limit read in the same run.
Needs a GPU.

    python tools/bench_outliers.py [--sizes 16 64 256] [--mean-k 50] [--reps 3] [--cpu-views 2] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import outliers_reference as orf  # noqa: E402
from bench_refine import gpu_info, timed  # noqa: E402
from gpd_b200 import lib, scenes  # noqa: E402

KERNELS = ("k_refine_knn", "k_outlier_mean", "k_outlier_stats", "k_outlier_mark", "DeviceScan", "k_outlier_gather",
           "k_batch_")  # k_batch_*: the grid rebuild of the reinstall


def kernel_ms(fn, setup):
    """Device milliseconds per kernel in one call (summed over its launches), median over 3 calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    per = {k: [] for k in KERNELS}
    per["all"] = []
    for _ in range(3):
        setup()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.events() if e.device_type.name == "CUDA"]
        for k in KERNELS:
            per[k].append(sum(e.device_time for e in ev if k in e.name))
        per["all"].append(sum(e.device_time for e in ev))
    return {k: round(statistics.median(v) / 1000.0, 4) for k, v in per.items()}


def batch_line(B, mean_k, reps, cpu_views, raws):
    ctx = lib.Context(lib.default_params(channels=15))
    off = np.concatenate([[0], np.cumsum([len(r["xyz"]) for r in raws[:B]])]).astype(np.int32)
    xyz = torch.from_numpy(np.concatenate([r["xyz"] for r in raws[:B]])).cuda()
    cam = torch.from_numpy(np.concatenate([r["cam_source"].ravel() for r in raws[:B]]).astype(np.int32)).cuda()
    kc = np.array([len(r["view_points"]) for r in raws[:B]], np.int32)
    vps = np.concatenate([r["view_points"] for r in raws[:B]])
    pp = lib.preprocess_params()
    pre = timed(lambda: ctx.preprocess_clouds_tensors(off, xyz, kc, vps, cam_source=cam, pp=pp), reps)
    poff = ctx.preprocess_clouds_tensors(off, xyz, kc, vps, cam_source=cam, pp=pp)
    clouds = ctx.get_clouds()
    pxyz = torch.from_numpy(np.concatenate([c["xyz"] for c in clouds])).cuda()
    pnrm = torch.from_numpy(np.concatenate([c["normals"] for c in clouds])).cuda()
    pk = np.array([c["cam_source"].shape[1] for c in clouds], np.int32)
    pvp = np.concatenate([c["view_points"] for c in clouds])
    pcam = torch.from_numpy(np.concatenate([c["cam_source"].ravel() for c in clouds]).astype(np.int32)).cuda()

    def reinstall():
        ctx.set_clouds_tensors(poff, pxyz, pnrm, pk, pvp, cam_source=pcam)

    reinstall()
    r = ctx.remove_outliers_clouds(mean_k, 1.0)
    call = timed(lambda: ctx.remove_outliers_clouds(mean_k, 1.0), reps, reinstall)
    kms = kernel_ms(lambda: ctx.remove_outliers_clouds(mean_k, 1.0), reinstall)
    nv = min(cpu_views, B)
    t0 = time.perf_counter()
    same = True
    for b in range(nv):
        kept = orf.remove(clouds[b]["xyz"], mean_k, 1.0)[0]
        same = same and np.array_equal(kept.astype(np.uint8), r["kept"][poff[b]:poff[b + 1]])
    cpu_s = (time.perf_counter() - t0) / nv
    ctx.close()
    return {"workload": f"B={B} synthetic_raw_scene(1000+i, n_points=20000), mean_k={mean_k}, stddev_mul=1.0", "B": B,
            "mean_k": mean_k, "points": int(poff[-1]), "points_per_view_mean": int(np.diff(poff).mean()),
            "kept_fraction": round(float(r["offsets"][-1]) / float(poff[-1]), 4), "call_ms": call, "preprocess_ms": pre,
            "call_over_preprocess": round(call["median"] / pre["median"], 4), "kernel_ms": kms,
            "numpy_s_per_view": round(cpu_s, 3), "numpy_s_batch_estimate": round(cpu_s * B, 1),
            "numpy_views_same_kept": bool(same), "gpu": gpu_info()}


def single_line(mean_k, reps):
    raw = scenes.synthetic_raw_scene(0)
    ctx = lib.Context(lib.default_params(channels=15))
    pp = lib.preprocess_params()
    pre = timed(lambda: ctx.preprocess(raw["xyz"], raw["cam_source"], raw["view_points"], pp=pp, read_back=False), reps)
    pc = ctx.preprocess(raw["xyz"], raw["cam_source"], raw["view_points"], pp=pp)

    def reinstall():
        ctx.set_cloud(pc["xyz"], pc["normals"], pc["cam_source"], pc["view_points"])

    reinstall()
    r = ctx.remove_outliers(mean_k, 1.0)
    call = timed(lambda: ctx.remove_outliers(mean_k, 1.0), reps, reinstall)
    kms = kernel_ms(lambda: ctx.remove_outliers(mean_k, 1.0), reinstall)
    ctx.close()
    return {"workload": f"config 3: synthetic_raw_scene(0), gpdb_preprocess + gpdb_remove_outliers, mean_k={mean_k}",
            "B": 1, "mean_k": mean_k, "points": len(pc["xyz"]), "kept_fraction": round(r["n_kept"] / len(pc["xyz"]), 4),
            "call_ms": call, "preprocess_ms": pre, "call_over_preprocess": round(call["median"] / pre["median"], 4),
            "kernel_ms": kms, "numpy_s": None, "gpu": gpu_info()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--mean-k", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-views", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_outliers: needs a CUDA device")
    raws = [scenes.synthetic_raw_scene(1000 + i, n_points=20000) for i in range(max(a.sizes))]
    lines = [single_line(a.mean_k, a.reps)]
    print(json.dumps(lines[-1]), flush=True)
    for B in a.sizes:
        lines.append(batch_line(B, a.mean_k, a.reps, a.cpu_views, raws))
        print(json.dumps(lines[-1]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
