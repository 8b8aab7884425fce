"""Depth images to clustered grasps on the device: the depth route against the same work done with today's calls.

Workload: B views of 640 x 480 uint16 depth images (millimetres) from K pinhole cameras (f = 525 px), rendered with a
z-buffer from synthetic_raw_scene tables (4 distinct scenes, tiled to B views; tests/depth_reference.py), default
preprocessing, 100 samples per view, the 20 best candidates of every view and their clustering (min_inliers 1),
15-channel images and the shipped 15-channel LeNet. The images start as one CUDA tensor.
  depth route: preprocess_depth_tensors -> subsample_clouds_tensors -> detect_batch_select_tensors ->
               find_clusters_batch_tensors;
  today:       torch back-projection of every pixel (float32, NaN for holes) and the one-hot cam_source blocks ->
               preprocess_clouds_tensors -> per-view torch.randperm sample indices -> detect_batch_select_tensors ->
               find_clusters_batch_tensors.
Both routes preprocess the same raw clouds; their sample draws differ (different generators). Each JSON line gives the
median wall time of each route and step over --reps repetitions (after one warm-up), its min / max, the peak memory torch
allocated for the caller's tensors, the device memory the route held at its high-water mark (library arenas and torch's
cache, over what was in use before it), and the GPU name and power limit read in the same run. Needs a GPU.

    python tools/bench_depth.py [--sizes 16 64 256] [--cameras 1 2] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import depth_reference as dr  # noqa: E402
from gpd_b200 import lib  # noqa: E402

W, H, F = 640, 480, 525.0
N_SAMPLES, NUM_SELECTED, MIN_INLIERS, SCENES = 100, 20, 1, 4


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def weights():
    z = np.load(os.path.join(ROOT, "gpd_b200", "weights", "lenet_15ch.npz"))
    return [z[n] for n in ("conv1_weights", "conv1_biases", "conv2_weights", "conv2_biases", "ip1_weights", "ip1_biases",
                           "ip2_weights", "ip2_biases")], int(z["relu_after_conv"])


def context():
    w, relu = weights()
    ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    ctx.set_weights(w)
    return ctx


def sync_ms(t0):
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def depth_route(ctx, B, ks, cams, d_depth, steps):
    t = time.perf_counter()
    ctx.preprocess_depth_tensors(ks, cams, d_depth)
    steps["preprocess"] = sync_ms(t)
    t = time.perf_counter()
    soff, idx = ctx.subsample_clouds_tensors(N_SAMPLES, 7)
    steps["samples"] = sync_ms(t)
    t = time.perf_counter()
    rec, roff = ctx.detect_batch_select_tensors(soff, idx, NUM_SELECTED)
    cl, coff = ctx.find_clusters_batch_tensors(roff, rec, MIN_INLIERS)
    steps["select_cluster"] = sync_ms(t)
    return int(roff[-1]), int(coff[-1])


def torch_route(ctx, B, K, cams, d_depth, steps):
    t = time.perf_counter()
    dev = d_depth.device
    img = (d_depth.view(B, K, H * W).to(torch.int32) & 0xFFFF).to(torch.float32)
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32),
                          indexing="ij")
    u, v = u.reshape(-1), v.reshape(-1)
    xyz = torch.empty((B, K, H * W, 3), dtype=torch.float32, device=dev)
    for k in range(K):
        c = cams[k]
        P = torch.tensor(np.array(c.pose[:]).reshape(3, 4), dtype=torch.float32, device=dev)
        z = img[:, k] * c.depth_scale
        pc = torch.stack([(u - c.cx) * z / c.fx, (v - c.cy) * z / c.fy, z], -1)
        pw = pc @ P[:, :3].T + P[:, 3]
        pw[img[:, k] == 0] = float("nan")
        xyz[:, k] = pw
    cam = torch.zeros((B, K, H * W, K), dtype=torch.int32, device=dev)
    for k in range(K):
        cam[:, k, :, k] = 1
    off = np.arange(B + 1, dtype=np.int64) * K * H * W
    vps = np.array([[c.pose[3], c.pose[7], c.pose[11]] for c in cams[:K]] * B)
    steps["back_project"] = sync_ms(t)
    t = time.perf_counter()
    poff = ctx.preprocess_clouds_tensors(off.astype(np.int32), xyz.view(-1, 3), np.full(B, K, np.int32), vps,
                                         cam_source=cam.view(-1))
    del xyz, cam
    steps["preprocess"] = sync_ms(t)
    t = time.perf_counter()
    lists = [torch.randperm(int(poff[b + 1] - poff[b]), device=dev)[:N_SAMPLES].sort().values for b in range(B)]
    soff = np.zeros(B + 1, np.int32)
    soff[1:] = np.cumsum([len(x) for x in lists])
    idx = torch.cat(lists).to(torch.int32)
    steps["samples"] = sync_ms(t)
    t = time.perf_counter()
    rec, roff = ctx.detect_batch_select_tensors(soff, idx, NUM_SELECTED)
    cl, coff = ctx.find_clusters_batch_tensors(roff, rec, MIN_INLIERS)
    steps["select_cluster"] = sync_ms(t)
    return int(roff[-1]), int(coff[-1])


def run(route, reps):
    """(median total, min / max, median steps, selected, clusters, torch peak MiB, device high-water MiB)."""
    torch.cuda.empty_cache()
    free0, total = torch.cuda.mem_get_info()
    torch.cuda.reset_peak_memory_stats()
    times, all_steps = [], []
    for r in range(reps + 1):
        steps = {}
        t = time.perf_counter()
        sel, ncl = route(steps)
        ms = sync_ms(t)
        if r:
            times.append(ms)
            all_steps.append(steps)
    free1, _ = torch.cuda.mem_get_info()
    med = {k: round(float(np.median([s[k] for s in all_steps])), 2) for k in all_steps[0]}
    return (round(float(np.median(times)), 2), [round(min(times), 2), round(max(times), 2)], med, sel, ncl,
            round(torch.cuda.max_memory_allocated() / 2**20, 1), round((free0 - free1) / 2**20, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    gpu = gpu_info()
    for K in a.cameras:
        cams = dr.default_cameras(K, width=W, height=H, f=F, scale=0.001)
        base = [np.stack([dr.render(pts, c, 0) for c in cams]) for pts in
                (dr.scenes.synthetic_raw_scene(500 + s)["xyz"] for s in range(SCENES))]
        for B in a.sizes:
            host = np.stack([base[b % SCENES] for b in range(B)])  # [B, K, H, W]
            d_depth = torch.from_numpy(host.view(np.int16)).cuda().reshape(-1)
            ks, cam_list = [K] * B, cams * B
            rec = {"B": B, "K": K, "width": W, "height": H, "pixels": int(host.size),
                   "valid_pixels": int(np.count_nonzero(host)), "samples_per_view": N_SAMPLES, "num_selected": NUM_SELECTED}
            ctx = context()
            r = run(lambda st: depth_route(ctx, B, ks, cam_list, d_depth, st), a.reps)
            rec["points"] = int(ctx._batch[0][-1])
            ctx.close()
            ctx = context()
            q = run(lambda st: torch_route(ctx, B, K, cams, d_depth, st), a.reps)
            ctx.close()
            for name, v in (("depth", r), ("today", q)):
                rec[f"{name}_ms"], rec[f"{name}_ms_min_max"], rec[f"{name}_steps_ms"] = v[0], v[1], v[2]
                rec[f"{name}_selected"], rec[f"{name}_clusters"] = v[3], v[4]
                rec[f"{name}_torch_peak_mib"], rec[f"{name}_device_high_water_mib"] = v[5], v[6]
            rec["gpu"] = gpu
            line = json.dumps(rec)
            print(line, flush=True)
            if a.out:
                with open(a.out, "a") as f:
                    f.write(line + "\n")
            del d_depth
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
