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

    python tools/bench_resident_batch.py [--sizes 16 64 256] [--reps 5]
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


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resident_batch.py needs a CUDA device")
    w, relu = weights()
    ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    ctx.set_weights(w)
    pp = lib.preprocess_params()
    gpu = gpu_info()
    pool = [scenes.synthetic_raw_scene(1000 + i, n_points=N_POINTS) for i in range(max(a.sizes))]
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
