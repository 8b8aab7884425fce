"""Labelling the candidates of a batch of views against their ground-truth clouds (HandSearch::reevaluateHypotheses,
the evalGroundTruth step of the reference's generate_data): one gpdb_reevaluate per view with its ground truth installed
in turn (the loop), gpdb_reevaluate_batch (host records) and gpdb_reevaluate_batch_device (a CUDA tensor of records),
against the CPU oracle.

Workload: S distinct scenes (--scenes, default 16); view i of a batch of B is scene 3000 + i % S. A view is
synthetic_raw_scene(seed, n_points=20000) seen by one camera, preprocessed with the default parameters, with
num_samples = 400 drawn by subsample_clouds (cfg/generate_data.cfg's value) and its candidates found by
hand_search_batch. Its ground truth is the same seed seen by four cameras, every seeing camera marked
(mark_all_cameras), at the 2 mm lattice, installed twice: voxelised (preprocess_clouds, default parameters) and
unvoxelised (voxelize = 0, normals estimated at 3 cm). B in {16, 64, 256}.

Each JSON line gives, for one ground truth and one B: the hands labelled, the wall milliseconds and labelled hands/s of
the loop (set_cloud of each ground truth + gpdb_reevaluate; also the gpdb_reevaluate calls alone), of the host batch
call and of the device batch call (CUDA events), each the median (min / max) over --reps runs after one warm-up; path
counter 15 (hands whose Antipodal passes walked the grid); the oracle's CPU time for the first --cpu-views views, scaled to
B and checked equal to the device's labels; and the GPU name and power limit read in the same run.

--ab LIB runs the loop mode alone at two builds of the library, this one and LIB (e.g. the parent commit's
libgpd_b200.so), alternating --ab-rounds times in fresh processes on the same prepared workload, and writes one line with
both spreads and whether their labels are identical. Needs a GPU.

    python tools/bench_label.py [--sizes 16 64 256] [--reps 3] [--cpu-views 2] [--ab LIB] [--out FILE]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CAMS4 = np.array([[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.6, 0.0, 0.0], [0.0, 0.6, 0.0]])
GTS = ("voxelised", "unvoxelised")


def prepare(n_scenes, path):
    """Candidates of every scene's view and both ground truths, saved to path (npz)."""
    from gpd_b200 import lib, scenes
    views = [scenes.synthetic_raw_scene(3000 + s, n_points=20000) for s in range(n_scenes)]
    raws = [scenes.synthetic_raw_scene(3000 + s, n_points=20000, cameras=CAMS4, mark_all_cameras=True) for s in range(n_scenes)]
    ctx = lib.Context(lib.default_params(channels=15))
    ctx.preprocess_clouds([{"xyz": v["xyz"], "cam_source": v["cam_source"], "view_points": v["view_points"]} for v in views],
                          read_back=False)
    res = ctx.hand_search_batch(ctx.subsample_clouds(400, 0))
    out = {}
    for s, r in enumerate(res):
        out[f"hands{s}"] = r["candidates"].view(np.uint8)
    for g, pp in zip(GTS, (lib.preprocess_params(), lib.preprocess_params(voxelize=0))):
        for s, c in enumerate(ctx.preprocess_clouds(raws, pp=pp)):
            for k in ("xyz", "normals", "cam_source", "view_points"):
                out[f"{g}{s}_{k}"] = c[k]
    ctx.close()
    np.savez(path, n_scenes=n_scenes, **out)


def load(path):
    from gpd_b200 import abi
    z = np.load(path)
    S = int(z["n_scenes"])
    hands = [z[f"hands{s}"].view(abi.POSE_DTYPE) for s in range(S)]
    gts = {g: [{k: z[f"{g}{s}_{k}"] for k in ("xyz", "normals", "cam_source", "view_points")} for s in range(S)] for g in GTS}
    return hands, gts


def spread(ms):
    return {"median": round(statistics.median(ms), 3), "min": round(min(ms), 3), "max": round(max(ms), 3)}


def loop_mode(hands, gts, B, reps):
    """One gpdb_reevaluate per view with its ground truth installed in turn: wall ms of the loop, of the reevaluate calls
    alone, and a digest of the labels and records."""
    from gpd_b200 import lib
    ctx = lib.Context(lib.default_params(channels=15))
    S = len(hands)
    total, only = [], []
    for rep in range(reps + 1):
        t_re, dig = 0.0, hashlib.sha256()
        t0 = time.perf_counter()
        for i in range(B):
            c, h = gts[i % S], hands[i % S]
            ctx.set_cloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
            t1 = time.perf_counter()
            lb, rec = ctx.reevaluate(h)
            t_re += time.perf_counter() - t1
            dig.update(lb.tobytes())
            dig.update(rec.tobytes())
        if rep:
            total.append(1e3 * (time.perf_counter() - t0))
            only.append(1e3 * t_re)
    ctx.close()
    return {"loop_ms": spread(total), "reevaluate_ms": spread(only), "digest": dig.hexdigest()[:16]}


def batch_line(hands, gts, g, B, reps, cpu_views, info):
    import torch
    from bench_refine import timed
    from gpd_b200 import lib
    from oracle import oracle
    S = len(hands)
    p = lib.default_params(channels=15)
    ctx = lib.Context(p)
    ctx.set_clouds([gts[i % S] for i in range(B)])
    groups = [hands[i % S] for i in range(B)]
    n = sum(len(h) for h in groups)
    host = []
    for rep in range(reps + 1):
        t0 = time.perf_counter()
        labels, recs = ctx.reevaluate_batch(groups)
        if rep:
            host.append(1e3 * (time.perf_counter() - t0))
    hoff = np.concatenate([[0], np.cumsum([len(h) for h in groups])]).astype(np.int32)
    src = torch.from_numpy(np.concatenate(groups).view(np.uint8).reshape(n, lib.POSE_BYTES)).cuda()
    t = src.clone()
    dev = timed(lambda: ctx.reevaluate_batch_tensors(hoff, t), reps, setup=lambda: t.copy_(src))
    t.copy_(src)
    ctx.phase_cycles(1)
    dl = ctx.reevaluate_batch_tensors(hoff, t).cpu().numpy()
    walks = ctx.path_counts()["label_walk"]
    ctx.phase_cycles(0)
    assert np.array_equal(dl, np.concatenate(labels))
    assert lib.poses_from_tensor(t).tobytes() == np.concatenate(recs).tobytes()
    loop = loop_mode(hands, gts, B, reps)
    cpu_s, cpu_n = 0.0, 0
    for i in range(min(cpu_views, B)):
        c = gts[i % S]
        oc = oracle.OracleCloud(c["xyz"], c["normals"], c["cam_source"], c["view_points"])
        t0 = time.perf_counter()
        lo, _ = oc.reevaluate(p, groups[i])
        cpu_s += time.perf_counter() - t0
        cpu_n += len(groups[i])
        assert np.array_equal(lo, labels[i]), i
    ctx.close()
    rate = lambda ms: round(n / (ms["median"] * 1e-3))  # noqa: E731
    return {"bench": "label", "ground_truth": g, "B": B, "hands": n,
            "gt_points_per_cloud": int(np.mean([len(gts[i % S]["xyz"]) for i in range(B)])),
            "positive": int(sum(int(x.sum()) for x in labels)),
            "loop": {**loop, "hands_per_s": rate(loop["loop_ms"])},
            "batch_host": {"ms": spread(host), "hands_per_s": rate(spread(host))},
            "batch_device": {"ms": dev, "hands_per_s": rate(dev)},
            "grid_walks_slot15": int(walks), "grid_walk_share": round(walks / max(n, 1), 4),
            "oracle_cpu_ms_scaled": round(1e3 * cpu_s * n / max(cpu_n, 1), 1), "oracle_views": min(cpu_views, B),
            "gpu": info}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--scenes", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-views", type=int, default=2)
    ap.add_argument("--ab", default=None, help="another build of libgpd_b200.so for the loop-mode comparison")
    ap.add_argument("--ab-rounds", type=int, default=3)
    ap.add_argument("--loop-only", default=None, help=argparse.SUPPRESS)  # a prepared workload: print loop_mode's JSON
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "results", "bench_label_h100.jsonl"))
    a = ap.parse_args()
    if a.loop_only:
        import ctypes
        from gpd_b200 import abi, lib
        so = ctypes.CDLL(lib.SO_PATH)  # an older build lacks the later entry points; the loop needs none of them
        for name in [n for n in abi.PROTOTYPES if not hasattr(so, n)]:
            del abi.PROTOTYPES[name]
        hands, gts = load(a.loop_only)
        print(json.dumps({g: {B: loop_mode(hands, gts[g], B, a.reps) for B in a.sizes} for g in GTS}))
        return
    from bench_refine import gpu_info
    info = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "workload.npz")
        prepare(a.scenes, path)
        hands, gts = load(path)
        lines = [batch_line(hands, gts[g], g, B, a.reps, a.cpu_views, info) for g in GTS for B in a.sizes]
        if a.ab:
            runs = {"this": [], "other": []}
            for _ in range(a.ab_rounds):
                for k, lib_path in (("other", os.path.abspath(a.ab)), ("this", None)):
                    env = dict(os.environ)
                    env.pop("GPD_B200_LIB", None)
                    if lib_path:
                        env["GPD_B200_LIB"] = lib_path
                    cmd = [sys.executable, os.path.abspath(__file__), "--loop-only", path, "--reps", str(a.reps),
                           "--sizes", *map(str, a.sizes)]
                    runs[k].append(json.loads(subprocess.check_output(cmd, env=env).decode().strip().splitlines()[-1]))
            ab = {"bench": "label_loop_ab", "other_lib": os.path.basename(os.path.dirname(os.path.abspath(a.ab))),
                  "rounds": a.ab_rounds, "gpu": info}
            for g in GTS:
                for B in map(str, a.sizes):
                    d = {k: [r[g][B] for r in runs[k]] for k in runs}
                    ab[f"{g}_B{B}"] = {
                        k: {"reevaluate_ms_medians": [x["reevaluate_ms"]["median"] for x in v],
                            "loop_ms_medians": [x["loop_ms"]["median"] for x in v]} for k, v in d.items()}
                    ab[f"{g}_B{B}"]["labels_identical"] = len({x["digest"] for v in d.values() for x in v}) == 1
            lines.append(ab)
    with open(a.out, "w") as f:
        for ln in lines:
            print(json.dumps(ln))
            f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
