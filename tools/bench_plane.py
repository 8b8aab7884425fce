"""The support-plane segmentation (gpdb_segment_planes_device / gpdb_segment_plane) on the device, against the
preprocessing of the same views and the numpy restatement on the CPU.

Workload: B in {16, 64, 256} raw views synthetic_raw_scene(1000 + i, n_points=20000) (about 57 k raw points each,
about 32 k after preprocessing), preprocessed once with preprocess_clouds_tensors (default parameters), then
segment_planes_tensors with the default plane parameters; and one 300 k-point config-3 cloud (synthetic_raw_scene(0))
through gpdb_preprocess + gpdb_segment_plane. Each JSON line gives, for one workload: the median (and min / max) device
time of the whole segmentation call and of preprocessing over --reps runs (CUDA events, after one warm-up), the device
time of each plane kernel from a separate torch.profiler run (median over its launches), the counts of the work (points,
hypotheses evaluated, distance tests), the CPU time of the numpy restatement (tests/plane_reference.py) on the first
--cpu-views views (one host thread; scaled to B) and of the C++ oracle (tests/plane_oracle.cpp) on all B views over
every host thread, and the GPU name and power limit read in the same run. No PCL baseline
is built. Needs a GPU.

    python tools/bench_plane.py [--sizes 16 64 256] [--reps 5] [--cpu-views 4] [--out FILE]
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

import plane_oracle as po  # noqa: E402
import plane_reference as pr  # noqa: E402
from gpd_b200 import lib, scenes  # noqa: E402

KERNELS = ("k_plane_hyp", "k_plane_count", "k_plane_pick", "k_plane_refit", "k_plane_mark")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def timed(fn, reps):
    """Median / min / max device milliseconds of fn() over reps runs after one warm-up (events on torch's stream)."""
    fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return {"median": round(statistics.median(ms), 3), "min": round(min(ms), 3), "max": round(max(ms), 3)}


def kernel_ms(fn):
    """Median device time per plane kernel over 3 calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
    out = {}
    for k in KERNELS:
        t = [e.device_time for e in prof.events() if k in e.name and e.device_type.name == "CUDA"]
        out[k] = round(statistics.median(t) / 1000.0, 4) if t else None
    return out


def batch_line(B, reps, cpu_views, raws):
    ctx = lib.Context(lib.default_params(channels=15))
    off = np.concatenate([[0], np.cumsum([len(r["xyz"]) for r in raws[:B]])]).astype(np.int32)
    xyz = torch.from_numpy(np.concatenate([r["xyz"] for r in raws[:B]])).cuda()
    cam = torch.from_numpy(np.concatenate([r["cam_source"].ravel() for r in raws[:B]]).astype(np.int32)).cuda()
    ks = np.array([len(r["view_points"]) for r in raws[:B]], np.int32)
    vps = np.concatenate([r["view_points"] for r in raws[:B]])
    pp = lib.preprocess_params()
    pre = timed(lambda: ctx.preprocess_clouds_tensors(off, xyz, ks, vps, cam_source=cam, pp=pp), reps)
    poff = ctx.preprocess_clouds_tensors(off, xyz, ks, vps, cam_source=cam, pp=pp)
    seg = timed(lambda: ctx.segment_planes_tensors(), reps)
    r = ctx.segment_planes_tensors()
    kms = kernel_ms(lambda: ctx.segment_planes_tensors())
    clouds = ctx.get_clouds()
    t0 = time.perf_counter()
    for b in range(min(cpu_views, B)):
        pr.segment(clouds[b]["xyz"], key=b)
    cpu_s = (time.perf_counter() - t0) / min(cpu_views, B)
    allxyz = np.concatenate([c["xyz"] for c in clouds])
    po.segment_batch(poff, allxyz)  # builds the oracle
    t0 = time.perf_counter()
    o = po.segment_batch(poff, allxyz)
    oracle_s = time.perf_counter() - t0
    same = bool(np.array_equal(o["n_hypotheses"], r["n_hypotheses"]))
    npts = np.diff(poff)
    H = int(lib.plane_params().max_iterations) + 1
    line = {"workload": f"B={B} synthetic_raw_scene(1000+i, n_points=20000)", "B": B, "points": int(poff[-1]),
            "points_per_view_mean": int(npts.mean()), "hypotheses_evaluated_mean": float(np.mean(r["n_hypotheses"])),
            "distance_tests_counted": int(npts.sum() * H), "inlier_share_mean": float(np.mean(r["n_inliers"] / npts)),
            "segment_ms": seg, "preprocess_ms": pre, "segment_over_preprocess": round(seg["median"] / pre["median"], 4),
            "kernel_ms": kms, "numpy_restatement_s_per_view": round(cpu_s, 4),
            "numpy_restatement_s_batch_estimate": round(cpu_s * B, 2), "oracle_s_batch": round(oracle_s, 3),
            "oracle_threads": os.cpu_count(), "oracle_same_hypotheses_evaluated": same, "gpu": gpu_info()}
    ctx.close()
    return line


def single_line(reps):
    raw = scenes.synthetic_raw_scene(0)
    ctx = lib.Context(lib.default_params(channels=15))
    pp = lib.preprocess_params()
    pre = timed(lambda: ctx.preprocess(raw["xyz"], raw["cam_source"], raw["view_points"], pp=pp, read_back=False), reps)
    seg = timed(lambda: ctx.segment_plane(), reps)
    plane, n_inl, elig = ctx.segment_plane()
    kms = kernel_ms(lambda: ctx.segment_plane())
    xyz = ctx.get_cloud()["xyz"]
    t0 = time.perf_counter()
    pr.segment(xyz, key=0)
    cpu_s = time.perf_counter() - t0
    po.segment(xyz, key=0)
    t0 = time.perf_counter()
    po.segment(xyz, key=0)
    oracle_s = time.perf_counter() - t0
    line = {"workload": "config 3: synthetic_raw_scene(0), gpdb_preprocess + gpdb_segment_plane", "B": 1,
            "points": len(xyz), "inlier_share": round(n_inl / len(xyz), 4), "segment_ms": seg, "preprocess_ms": pre,
            "segment_over_preprocess": round(seg["median"] / pre["median"], 4), "kernel_ms": kms,
            "numpy_restatement_s": round(cpu_s, 3), "oracle_s": round(oracle_s, 3), "gpu": gpu_info()}
    ctx.close()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-views", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_plane: needs a CUDA device")
    raws = [scenes.synthetic_raw_scene(1000 + i, n_points=20000) for i in range(max(a.sizes))]
    lines = [batch_line(B, a.reps, a.cpu_views, raws) for B in a.sizes] + [single_line(a.reps)]
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
