"""The normal refinement (gpdb_refine_normals_clouds / gpdb_refine_normals) on the device, against the preprocessing of
the same views and the C++ oracle on the CPU.

Workload: B in {16, 64, 256} raw views synthetic_raw_scene(1000 + i, n_points=20000) (the views of tools/bench_plane.py),
preprocessed once with preprocess_clouds_tensors (default parameters), then refine_normals_clouds; and the 300 k-point
config-3 cloud (synthetic_raw_scene(0)) through gpdb_preprocess + gpdb_refine_normals; each at k = 10 and 50. The
refinement rewrites the normals it reads, so every timed call first reinstalls the processed clouds' normals (that
install is outside the timed window). Each JSON line gives, for one workload: the median (and min / max) device time of
the whole call and of preprocessing over --reps runs (CUDA events, after one warm-up), the device time of each kernel
from a separate torch.profiler run (kNN and cast once per call, iterate and stop summed over the call's 15 launches
each), the iterations run, the C++ oracle (tests/refine_oracle.cpp, brute-force lists) on the first --cpu-views views
over every host thread (scaled to B; not run on the config-3 cloud, whose N^2 lists take hours), and the GPU name and
power limit read in the same run. Needs a GPU.

    python tools/bench_refine.py [--sizes 16 64 256] [--ks 10 50] [--reps 3] [--cpu-views 2] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import refine_oracle as ro  # noqa: E402
from gpd_b200 import lib, scenes  # noqa: E402

KERNELS = ("k_refine_knn", "k_refine_cast", "k_refine_iter", "k_refine_stop", "k_refine_commit")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def timed(fn, reps, setup=None):
    """Median / min / max device milliseconds of fn() over reps runs after one warm-up; setup() runs before each, untimed."""
    ms = []
    for i in range(reps + 1):
        if setup:
            setup()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        if i:
            ms.append(a.elapsed_time(b))
    return {"median": round(statistics.median(ms), 3), "min": round(min(ms), 3), "max": round(max(ms), 3)}


def kernel_ms(fn, setup):
    """Device milliseconds per kernel in one call (summed over its launches), median over 3 calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    per = {k: [] for k in KERNELS}
    for _ in range(3):
        setup()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        for k in KERNELS:
            per[k].append(sum(e.device_time for e in prof.events() if k in e.name and e.device_type.name == "CUDA"))
    return {k: round(statistics.median(v) / 1000.0, 4) for k, v in per.items()}


def batch_lines(B, ks, reps, cpu_views, raws):
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

    lines = []
    for k in ks:
        reinstall()
        its = ctx.refine_normals_clouds(k)
        call = timed(lambda: ctx.refine_normals_clouds(k), reps, reinstall)
        kms = kernel_ms(lambda: ctx.refine_normals_clouds(k), reinstall)
        nv = min(cpu_views, B)
        ro.refine(clouds[0]["xyz"][:100], clouds[0]["normals"][:100], k)  # builds the oracle
        t0 = time.perf_counter()
        same = True
        for b in range(nv):
            _, it = ro.refine(clouds[b]["xyz"], clouds[b]["normals"], k)
            same = same and it == its[b]
        oracle_s = (time.perf_counter() - t0) / nv
        npts = np.diff(poff)
        lines.append({"workload": f"B={B} synthetic_raw_scene(1000+i, n_points=20000), k={k}", "B": B, "k": k,
                      "points": int(poff[-1]), "points_per_view_mean": int(npts.mean()),
                      "iterations": {"min": int(its.min()), "max": int(its.max()), "mean": round(float(its.mean()), 2)},
                      "refine_ms": call, "preprocess_ms": pre, "refine_over_preprocess": round(call["median"] / pre["median"], 4),
                      "kernel_ms": kms, "oracle_s_per_view": round(oracle_s, 3),
                      "oracle_s_batch_estimate": round(oracle_s * B, 1), "oracle_threads": os.cpu_count(),
                      "oracle_views_same_iterations": bool(same), "gpu": gpu_info()})
    ctx.close()
    return lines


def single_lines(ks, reps):
    raw = scenes.synthetic_raw_scene(0)
    ctx = lib.Context(lib.default_params(channels=15))
    pp = lib.preprocess_params()
    pre = timed(lambda: ctx.preprocess(raw["xyz"], raw["cam_source"], raw["view_points"], pp=pp, read_back=False), reps)
    pc = ctx.preprocess(raw["xyz"], raw["cam_source"], raw["view_points"], pp=pp)

    def reinstall():
        ctx.set_cloud(pc["xyz"], pc["normals"], pc["cam_source"], pc["view_points"])

    lines = []
    for k in ks:
        reinstall()
        it = ctx.refine_normals(k)
        call = timed(lambda: ctx.refine_normals(k), reps, reinstall)
        kms = kernel_ms(lambda: ctx.refine_normals(k), reinstall)
        lines.append({"workload": f"config 3: synthetic_raw_scene(0), gpdb_preprocess + gpdb_refine_normals, k={k}", "B": 1,
                      "k": k, "points": len(pc["xyz"]), "iterations": it, "refine_ms": call, "preprocess_ms": pre,
                      "refine_over_preprocess": round(call["median"] / pre["median"], 4), "kernel_ms": kms,
                      "oracle_s": None, "gpu": gpu_info()})
    ctx.close()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--ks", type=int, nargs="+", default=[10, 50])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-views", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_refine: needs a CUDA device")
    raws = [scenes.synthetic_raw_scene(1000 + i, n_points=20000) for i in range(max(a.sizes))]
    lines = single_lines(a.ks, a.reps)
    for B in a.sizes:
        lines += batch_lines(B, a.ks, a.reps, a.cpu_views, raws)
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
