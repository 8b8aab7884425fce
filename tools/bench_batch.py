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

--sis times cem_detect_grasps' device steps over B processed views (synthetic_raw_scene(1000 + i, n_points=20000) after
default preprocessing) with the default SIS parameters: 50 initial samples, 5 rounds of 50 positions, the final
classification at every position that carried a hand and the clustering (min_inliers 1). The per-view loop of
single-cloud calls (gpdb_set_cloud, gpdb_hand_search, gpdb_set_samples + gpdb_hand_search per round, gpdb_set_samples +
gpdb_detect, gpdb_find_clusters) runs against one batch call per step (gpdb_set_clouds, gpdb_hand_search_batch,
gpdb_set_clouds_samples + gpdb_hand_search_batch per round, gpdb_set_clouds_samples + gpdb_detect_batch,
gpdb_find_clusters_batch), both through lib.py. The round positions come from one seeded numpy generator (Gaussians around
the initial hand-set positions and uniform cloud points) and are shared by both routes, so the timing measures the device
path and not a host RNG. --detect-full times detectGrasps from raw views: preprocessing, the selection of the 100 best
candidates at 500 samples per view and their clustering, looped (gpdb_preprocess, gpdb_detect_select, gpdb_find_clusters)
against batched (gpdb_preprocess_clouds, gpdb_detect_batch_select, gpdb_find_clusters_batch). Both modes check once,
outside the timed region, that the two routes return identical records, and print per step the median wall time of each
route and the samples/s of the whole route.

--sis-device adds, in the same command and on the same views and initial samples, one gpdb_sis_batch_device call per step
(the whole of cem_detect_grasps with its draws on the device, default SIS parameters, initial indices in a CUDA tensor) and
prints its median wall time and samples/s (initial samples + evaluated round positions + classified kept positions) next
to the --sis batch route. The two routes draw different round positions, so their records are not compared; the device
call is checked once to equal gpdb_sis_batch bit for bit.

    python tools/bench_batch.py [--sizes 1 16 64 256] [--reps 3] [--raw | --sis | --sis-device | --detect-full]
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


SIS_INIT, SIS_ROUNDS, SIS_PER_ROUND, SIS_SIGMA, MIN_INLIERS, NUM_SELECTED = 50, 5, 50, 0.02, 1, 100


class Steps:
    """Wall time per named step (each step ends in a call that returns host results, i.e. after a device synchronise)."""

    def __init__(self):
        self.t = {}
        self.t0 = time.perf_counter()

    def __call__(self, name):
        now = time.perf_counter()
        self.t[name] = self.t.get(name, 0.0) + now - self.t0
        self.t0 = now


def hand_set_positions(view):
    """Positions of the samples that carried at least one hand (candidates are in sample-slot order)."""
    c = view["candidates"]
    _, first = np.unique(c["sample_slot"], return_index=True)
    return c["sample"][first].astype(np.float64)


def sis_loop(ctx, clouds, init, rounds):
    st, kept, out = Steps(), [], []
    for b, c in enumerate(clouds):
        ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        st("install")
        k = [hand_set_positions(ctx.hand_search(init[b]))]
        st("init_search")
        for r in rounds:
            k.append(hand_set_positions(ctx.hand_search(ctx.set_samples(r[b]))))
            st("rounds")
        kept.append(np.concatenate(k))
        det = ctx.detect(ctx.set_samples(kept[-1]))["candidates"]
        st("classify")
        out.append((det, ctx.find_clusters(det, MIN_INLIERS)))
        st("cluster")
    return st.t, sum(len(k) for k in kept), out


def sis_batch(ctx, clouds, init, rounds):
    st = Steps()
    ctx.set_clouds(clouds)
    st("install")
    kept = [[hand_set_positions(v)] for v in ctx.hand_search_batch(init)]
    st("init_search")
    for r in rounds:
        for k, v in zip(kept, ctx.hand_search_batch(ctx.set_clouds_samples(r))):
            k.append(hand_set_positions(v))
        st("rounds")
    kept = [np.concatenate(k) for k in kept]
    det = [v["candidates"] for v in ctx.detect_batch(ctx.set_clouds_samples(kept))]
    st("classify")
    clusters = ctx.find_clusters_batch(det, MIN_INLIERS)
    st("cluster")
    return st.t, sum(len(k) for k in kept), list(zip(det, clusters))


def sis_device(ctx, clouds, offsets, d_init):
    """gpdb_set_clouds + one gpdb_sis_batch_device call: (wall time, samples evaluated, records on the device)."""
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()  # the install is timed, as the batch route's install step is
    ctx.set_clouds(clouds)
    rec, hoff, stats = ctx.sis_batch_tensors(offsets, d_init, min_inliers=MIN_INLIERS)
    t = time.perf_counter() - t0
    rounds = ctx.sis_positions()["round_counts"]
    return t, int(offsets[-1]) + int(rounds.sum()) + stats["n_samples"], (rec, hoff)


def sis_device_check(ctx, clouds, init):
    """The device call's arguments, after the one check that it equals gpdb_sis_batch on the same views."""
    import torch
    offsets, idx = lib.pack_samples(init)
    d_init = torch.from_numpy(idx).cuda()
    ctx.set_clouds(clouds)
    host = ctx.sis_batch(init, min_inliers=MIN_INLIERS)["hands"]
    _, _, (rec, hoff) = sis_device(ctx, clouds, offsets, d_init)
    recs = lib.poses_from_tensor(rec)
    assert all(recs[hoff[b]:hoff[b + 1]].tobytes() == h.tobytes() for b, h in enumerate(host)), "device SIS != host SIS"
    return offsets, d_init


def full_loop(ctx, views, pp, samples):
    st, out = Steps(), []
    for v, s in zip(views, samples):
        ctx.preprocess(v["xyz"], v["cam_source"], v["view_points"], pp, read_back=False)
        st("preprocess")
        sel = ctx.detect_select(s, NUM_SELECTED)["candidates"]
        st("select")
        out.append((sel, ctx.find_clusters(sel, MIN_INLIERS)))
        st("cluster")
    return st.t, 0, out


def full_batch(ctx, views, pp, samples):
    st = Steps()
    ctx.preprocess_clouds(views, pp, read_back=False)
    st("preprocess")
    sel = ctx.detect_batch_select(samples, NUM_SELECTED)
    st("select")
    clusters = ctx.find_clusters_batch(sel, MIN_INLIERS)
    st("cluster")
    return st.t, 0, list(zip(sel, clusters))


def same_records(ra, rb):
    return len(ra) == len(rb) and all(x.tobytes() == y.tobytes() for a, b in zip(ra, rb) for x, y in zip(a, b))


def main_steps(a, ctx, gpu):
    """--sis / --detect-full: the per-view loop against one batch call per step."""
    pp = lib.preprocess_params()
    pool = []
    for i in range(max(a.sizes)):
        s = scenes.synthetic_raw_scene(1000 + i, n_points=N_POINTS)
        pool.append({"xyz": s["xyz"], "cam_source": s["cam_source"], "view_points": s["view_points"]})
    med = lambda v: float(np.median(v))  # noqa: E731
    for B in a.sizes:
        views = pool[:B]
        clouds = ctx.preprocess_clouds(views, pp)
        n = [len(c["xyz"]) for c in clouds]
        rng = np.random.default_rng(B)
        if a.sis or a.sis_device:
            init = [rng.choice(nb, min(SIS_INIT, nb), replace=False).astype(np.int32) for nb in n]
            # round positions of every view from one generator, shared by both routes: Gaussians around the initial
            # hand-set positions (70 %) and cloud points (30 %), as the default prob_rand_samples = 0.3 mixes them
            ctx.set_clouds(clouds)
            start = [hand_set_positions(v) for v in ctx.hand_search_batch(init)]
            rounds = []
            for _ in range(SIS_ROUNDS):
                r = []
                for c, s0 in zip(clouds, start):
                    ng = SIS_PER_ROUND - int(0.3 * SIS_PER_ROUND)
                    centre = s0[rng.integers(0, len(s0), ng)] if len(s0) else c["xyz"][rng.integers(0, len(c["xyz"]), ng)]
                    pts = c["xyz"][rng.integers(0, len(c["xyz"]), SIS_PER_ROUND - ng)].astype(np.float64)
                    r.append(np.vstack([centre + rng.normal(0.0, SIS_SIGMA, centre.shape), pts]))
                rounds.append(r)
            loop, batch, args = sis_loop, sis_batch, (clouds, init, rounds)
            n_search = sum(len(i) for i in init) + SIS_ROUNDS * SIS_PER_ROUND * B
        else:
            samples = [rng.choice(nb, min(N_SAMPLES, nb), replace=False).astype(np.int32) for nb in n]
            loop, batch, args = full_loop, full_batch, (views, pp, samples)
            n_search = sum(len(s) for s in samples)
        # warm-up of every shape, and the one check that both routes return the same records
        _, kl, rl = loop(ctx, *args)
        _, kb, rb = batch(ctx, *args)
        assert kl == kb and same_records(rl, rb), "the loop and the batch route differ"
        dev = sis_device_check(ctx, clouds, init) if a.sis_device else None
        tl, tb, td = [], [], []
        for _ in range(a.reps):
            tl.append(loop(ctx, *args)[0])
            tb.append(batch(ctx, *args)[0])
            if dev:
                td.append(sis_device(ctx, clouds, *dev)[0])
        n_total = n_search + kl  # hand-search samples + classified positions (--sis)
        steps = list(tl[0])
        line = {"mode": "sis_device" if a.sis_device else "sis" if a.sis else "detect_full", "B": B, "processed_points": int(sum(n)), "samples": n_total,
                "loop_ms": round(1e3 * med([sum(t.values()) for t in tl]), 2),
                "batch_ms": round(1e3 * med([sum(t.values()) for t in tb]), 2),
                "loop_sps": round(n_total / med([sum(t.values()) for t in tl])),
                "batch_sps": round(n_total / med([sum(t.values()) for t in tb])),
                "loop_steps_ms": {s: round(1e3 * med([t[s] for t in tl]), 2) for s in steps},
                "batch_steps_ms": {s: round(1e3 * med([t[s] for t in tb]), 2) for s in steps},
                "clusters": int(sum(len(c) for _, c in rb)), "gpu": gpu}
        if dev:
            n_dev = sis_device(ctx, clouds, *dev)[1]
            line.update({"device_ms": round(1e3 * med(td), 2), "device_samples": n_dev, "device_sps": round(n_dev / med(td))})
        print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--sizes", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--reps", type=int, default=3)
    mode = ap.add_mutually_exclusive_group()
    mode.add_argument("--raw", action="store_true", help="start from raw views: three preprocessing + detection routes")
    mode.add_argument("--sis", action="store_true", help="cem_detect_grasps' steps: per-view loop against batch calls")
    mode.add_argument("--sis-device", action="store_true", help="--sis plus one gpdb_sis_batch_device call per step")
    mode.add_argument("--detect-full", action="store_true", help="detectGrasps from raw views: loop against batch calls")
    a = ap.parse_args()
    w, relu = weights()
    if a.sis or a.sis_device or a.detect_full:
        ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
        ctx.set_weights(w)
        main_steps(a, ctx, gpu_info())
        ctx.close()
        return
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
