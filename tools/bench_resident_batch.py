"""detectGrasps over a batch of views that live in GPU memory: the host route against the device-resident route.

Workload: B raw views of synthetic_raw_scene(1000 + i, n_points=20000) (one camera, cam_source included), default
preprocessing, 500 samples per view (fewer when a view keeps fewer points), the 100 best candidates of every view and
their clustering (min_inliers 1), 15-channel images and the shipped 15-channel LeNet. Every view, and its sample
indices, starts as CUDA tensors, as a simulated depth camera or a GPU depth-to-cloud step leaves them:
  host route:   .cpu() of every view and sample list, gpdb_preprocess_clouds, gpdb_detect_batch_select,
                gpdb_find_clusters_batch (lib.Context.preprocess_clouds / detect_batch_select / find_clusters_batch);
  device route: torch.cat of the views on the device, gpdb_preprocess_clouds_device, gpdb_detect_batch_select_device,
                gpdb_find_clusters_batch_device (the *_tensors methods; records stay in CUDA tensors).
For each B it checks once, outside the timed region, that both routes return identical selected records and clusters,
then prints one JSON line with the median wall time per step and of the whole route over --reps repetitions, the
samples/s of each route, and the GPU name and power limit. Needs a GPU.

--search: a learned sampler's loop instead. The B views are installed once (default preprocessing); every view gets 500
positions drawn by torch on the device (Gaussian offsets, sigma 2 mm, around random points of the processed view), and
the samples are exactly those positions (local indices N_b .. N_b + 499):
  host route:   .cpu() of the positions, gpdb_set_clouds_samples, gpdb_detect_batch (records, flags and scores to the host);
  device route: gpdb_set_clouds_samples_device, gpdb_detect_batch_device (records, flags and scores stay in CUDA tensors).
It checks once, outside the timed region, that both routes return the same records, offsets, flags and score bits, and
also times gpdb_hand_search_batch_device + gpdb_images_batch_device (the grasp images of every hand, for a classifier of
the caller's) on their own. Each JSON line gives the median and the min / max over --reps repetitions.

    python tools/bench_resident_batch.py [--sizes 16 64 256] [--reps 5] [--search]
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

from gpd_b200 import lib, scenes  # noqa: E402

N_POINTS, N_SAMPLES, NUM_SELECTED, MIN_INLIERS = 20000, 500, 100, 1


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


class Steps:
    """Wall time per named step (every step ends in a library call that returns after its device work)."""

    def __init__(self):
        self.t = {}
        self.t0 = time.perf_counter()

    def __call__(self, name):
        now = time.perf_counter()
        self.t[name] = self.t.get(name, 0.0) + now - self.t0
        self.t0 = now


def host_route(ctx, views, samples, vps, pp):
    st = Steps()
    raws = [{"xyz": v["xyz"].cpu().numpy(), "cam_source": v["cam_source"].cpu().numpy(), "view_points": vp}
            for v, vp in zip(views, vps)]
    sidx = [s.cpu().numpy() for s in samples]
    st("to_host")
    ctx.preprocess_clouds(raws, pp, read_back=False)
    st("preprocess")
    sel = ctx.detect_batch_select(sidx, NUM_SELECTED)
    st("select")
    cl = ctx.find_clusters_batch(sel, MIN_INLIERS)
    st("cluster")
    return st.t, (b"".join(s.tobytes() for s in sel), b"".join(c.tobytes() for c in cl))


def device_route(ctx, views, samples, vps, pp):
    st = Steps()
    poff = np.zeros(len(views) + 1, np.int32)
    poff[1:] = np.cumsum([len(v["xyz"]) for v in views])
    soff = np.zeros(len(views) + 1, np.int32)
    soff[1:] = np.cumsum([len(s) for s in samples])
    xyz = torch.cat([v["xyz"] for v in views])
    cam = torch.cat([v["cam_source"].reshape(-1) for v in views])
    sidx = torch.cat(samples)
    st("pack")
    ctx.preprocess_clouds_tensors(poff, xyz, np.ones(len(views), np.int32), np.concatenate(vps), cam_source=cam, pp=pp)
    st("preprocess")
    rec, sel_off = ctx.detect_batch_select_tensors(soff, sidx, NUM_SELECTED)
    st("select")
    cl, _ = ctx.find_clusters_batch_tensors(sel_off, rec, MIN_INLIERS)
    torch.cuda.current_stream().synchronize()
    st("cluster")
    return st.t, (lib.poses_from_tensor(rec).tobytes(), lib.poses_from_tensor(cl).tobytes())


SIGMA = 0.002


def draw_positions(xyz, poff, gen):
    """N_SAMPLES positions per view on the device: Gaussian offsets around uniformly drawn points of the view."""
    counts = torch.from_numpy(np.diff(poff)).cuda().repeat_interleave(N_SAMPLES)
    first = torch.from_numpy(poff[:-1]).cuda().repeat_interleave(N_SAMPLES)
    pick = first + (torch.rand(len(counts), device="cuda", generator=gen, dtype=torch.float64) * counts).long()
    return xyz[pick].double() + SIGMA * torch.randn((len(counts), 3), device="cuda", generator=gen, dtype=torch.float64)


def search_host(ctx, pos, B):
    st = Steps()
    p = pos.cpu().numpy()
    st("to_host")
    first = ctx.set_clouds_samples([p[b * N_SAMPLES:(b + 1) * N_SAMPLES] for b in range(B)])
    st("install")
    res = ctx.detect_batch(first)
    st("detect")
    out = (b"".join(r["candidates"].tobytes() for r in res), [r["n_candidates"] for r in res],
           np.concatenate([r["pose_flags"] for r in res]).tobytes(), np.concatenate([r["pose_scores"] for r in res]).tobytes())
    return st.t, out


def search_device(ctx, pos, soff, sidx):
    st = Steps()
    ctx.set_clouds_samples_tensors(soff, pos)
    st("install")
    rec, flags, scores, coff = ctx.detect_batch_tensors(soff, sidx)
    st("detect")
    return st.t, (rec, flags, scores, coff)


def search_images(ctx, soff, sidx):
    st = Steps()
    rec, _, coff = ctx.hand_search_batch_tensors(soff, sidx)
    st("hand_search")
    img = ctx.images_batch_tensors(coff, rec)
    st("images")
    return st.t, len(img)


def main_search(ctx, a, pool, pp, gpu):
    spread = lambda v: [round(1e3 * min(v), 2), round(1e3 * max(v), 2)]  # noqa: E731
    med = lambda v: float(np.median(v))  # noqa: E731
    for B in a.sizes:
        poff = ctx.preprocess_clouds([{"xyz": r["xyz"], "cam_source": r["cam_source"], "view_points": r["view_points"]}
                                      for r in pool[:B]], pp, read_back=False)
        xyz = torch.from_numpy(np.concatenate([c["xyz"] for c in ctx.get_clouds()])).cuda()
        gen = torch.Generator(device="cuda").manual_seed(B)
        pos = draw_positions(xyz, poff, gen)
        soff = np.arange(B + 1, dtype=np.int32) * N_SAMPLES
        sidx = (torch.from_numpy(np.diff(poff)).cuda().int().repeat_interleave(N_SAMPLES)
                + torch.arange(N_SAMPLES, device="cuda", dtype=torch.int32).repeat(B)).contiguous()
        n = B * N_SAMPLES
        torch.cuda.synchronize()
        # warm-up of every shape, and the one check that both routes agree bit for bit
        _, h = search_host(ctx, pos, B)
        _, (rec, flags, scores, coff) = search_device(ctx, pos, soff, sidx)
        assert h[0] == lib.poses_from_tensor(rec).tobytes(), "records differ"
        assert list(np.diff(coff)) == h[1], "offsets differ"
        assert h[2] == flags.cpu().numpy().tobytes() and h[3] == scores.cpu().numpy().tobytes(), "flags or scores differ"
        del rec, flags, scores
        _, n_img = search_images(ctx, soff, sidx)
        th, td, ti = [], [], []
        for _ in range(a.reps):
            th.append(search_host(ctx, pos, B)[0])
            td.append(search_device(ctx, pos, soff, sidx)[0])
            ti.append(search_images(ctx, soff, sidx)[0])
        tot = lambda ts: [sum(t.values()) for t in ts]  # noqa: E731
        host_ms, dev_ms, img_ms = med(tot(th)), med(tot(td)), med(tot(ti))
        print(json.dumps({"mode": "search", "B": B, "processed_points": int(poff[-1]), "samples": n,
                          "candidates": int(coff[-1]), "images": n_img,
                          "host_ms": round(1e3 * host_ms, 2), "device_ms": round(1e3 * dev_ms, 2),
                          "host_ms_min_max": spread(tot(th)), "device_ms_min_max": spread(tot(td)),
                          "host_sps": round(n / host_ms), "device_sps": round(n / dev_ms),
                          "host_steps_ms": {s: round(1e3 * med([t[s] for t in th]), 2) for s in th[0]},
                          "device_steps_ms": {s: round(1e3 * med([t[s] for t in td]), 2) for s in td[0]},
                          "search_images_ms": round(1e3 * img_ms, 2), "search_images_ms_min_max": spread(tot(ti)),
                          "search_images_sps": round(n / img_ms), "images_per_s": round(n_img / img_ms),
                          "search_images_steps_ms": {s: round(1e3 * med([t[s] for t in ti]), 2) for s in ti[0]},
                          "gpu": gpu}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--search", action="store_true", help="positions drawn on the device: the host against the device route")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resident_batch.py needs a CUDA device")
    w, relu = weights()
    ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    ctx.set_weights(w)
    pp = lib.preprocess_params()
    gpu = gpu_info()
    pool = [scenes.synthetic_raw_scene(1000 + i, n_points=N_POINTS) for i in range(max(a.sizes))]
    if a.search:
        main_search(ctx, a, pool, pp, gpu)
        ctx.close()
        return
    med = lambda v: float(np.median(v))  # noqa: E731
    for B in a.sizes:
        raw = pool[:B]
        poff = ctx.preprocess_clouds([{"xyz": r["xyz"], "cam_source": r["cam_source"], "view_points": r["view_points"]}
                                      for r in raw], pp, read_back=False)
        rng = np.random.default_rng(B)
        views = [{"xyz": torch.from_numpy(r["xyz"]).cuda(), "cam_source": torch.from_numpy(r["cam_source"]).cuda()}
                 for r in raw]
        vps = [r["view_points"] for r in raw]
        samples = [torch.from_numpy(rng.choice(nb, min(N_SAMPLES, nb), replace=False).astype(np.int32)).cuda()
                   for nb in np.diff(poff)]
        n = int(sum(len(s) for s in samples))
        torch.cuda.synchronize()
        # warm-up of every shape, and the one check that both routes return the same records
        _, rh = host_route(ctx, views, samples, vps, pp)
        _, rd = device_route(ctx, views, samples, vps, pp)
        assert rh == rd, "the host and the device route differ"
        th, td = [], []
        for _ in range(a.reps):
            th.append(host_route(ctx, views, samples, vps, pp)[0])
            td.append(device_route(ctx, views, samples, vps, pp)[0])
        host_ms, dev_ms = med([sum(t.values()) for t in th]), med([sum(t.values()) for t in td])
        print(json.dumps({"B": B, "raw_points": int(sum(len(r["xyz"]) for r in raw)), "processed_points": int(poff[-1]),
                          "samples": n, "selected": len(rh[0]) // lib.POSE_BYTES, "clusters": len(rh[1]) // lib.POSE_BYTES,
                          "host_ms": round(1e3 * host_ms, 2), "device_ms": round(1e3 * dev_ms, 2),
                          "host_sps": round(n / host_ms), "device_sps": round(n / dev_ms),
                          "host_steps_ms": {s: round(1e3 * med([t[s] for t in th]), 2) for s in th[0]},
                          "device_steps_ms": {s: round(1e3 * med([t[s] for t in td]), 2) for s in td[0]},
                          "gpu": gpu}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
