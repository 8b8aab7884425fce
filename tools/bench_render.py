"""gpdb_render_depth_device and gpdb_sample_meshes_device on mesh_table_scene tabletops held in device memory: render time
per call, the time gpdb_preprocess_depth_device then takes on the same images (where a view's time goes), sampled
points per second, and the fallback fraction of gpdb_preprocess_depth_organized_device on these dense surface renders.
Times are CUDA events around the call, the median of 5 timed windows after a warm-up call; the card's name, power
limit and clocks are read in the same run. Workloads: B = 1, 16, 64, 256 views of 640 x 480 at K = 1 and 2 cameras, on
scenes of about 20 k and about 200 k faces (four distinct scenes, cycled over the views).
Usage: python tools/bench_render.py [out.jsonl]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

# (label, n_objects, segments): about 20 k and about 200 k faces per scene
SCENES = [("20k", 24, 24), ("200k", 40, 60)]
DENSITY = 1e5  # points per square metre of the ground truth: a 3 mm spacing


def cameras(K):
    """K 640 x 480 cameras looking at the table (z ~ 0.9) from about 0.9 m, tilted a little"""
    from gpd_b200 import lib
    out = []
    for k in range(K):
        a = 0.15 * k
        R = np.array([[np.cos(a), 0.0, np.sin(a)], [0.0, 1.0, 0.0], [-np.sin(a), 0.0, np.cos(a)]])
        t = np.array([-0.9 * np.sin(a), 0.0, 0.9 * (1 - np.cos(a))])
        out.append(lib.depth_camera(640, 480, 520.0, 520.0, 319.5, 239.5, np.hstack([R, t[:, None]]), 0.001))
    return out


def timed(fn):
    import torch
    r = fn()
    ts = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), r


def main():
    import torch

    from gpd_b200 import lib, scenes
    out = sys.argv[1] if len(sys.argv) > 1 else None
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = lib.Context(lib.default_params())
    pp = lib.preprocess_params()
    rows = []
    for label, n_obj, seg in SCENES:
        base = [scenes.mesh_table_scene(s, n_objects=n_obj, segments=seg)[:2] for s in range(4)]
        faces = int(np.mean([len(f) for _, f in base]))
        for B in (1, 16, 64, 256):
            meshes = [base[b % 4] for b in range(B)]
            m = lib.pack_meshes(meshes)
            dv, df = torch.from_numpy(m["vertices"]).cuda(), torch.from_numpy(m["faces"]).cuda()
            for K in (1, 2):
                cams = cameras(K) * B
                ms_render, depth = timed(lambda: ctx.render_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df,
                                                                          [K] * B, cams, torch.uint16))
                ms_pre, _ = timed(lambda: ctx.preprocess_depth_tensors([K] * B, cams, depth, pp))
                row = {"scene": label, "faces_per_view": faces, "views": B, "cameras": K, "image": "640x480",
                       "ms_render": round(ms_render, 3), "ms_preprocess_depth": round(ms_pre, 3),
                       "returns": int((depth.view(torch.int16) != 0).sum().item())}
                if B <= 16:
                    poff, fb = ctx.preprocess_depth_organized_tensors([K] * B, cams, depth, pp)
                    row["organized_fallback_fraction"] = round(float(fb.sum()) / max(int(poff[-1]), 1), 4)
                if K == 1:
                    ms_s, (poff, _, _) = timed(lambda: ctx.sample_meshes_tensors(m["vertex_offsets"], dv, m["face_offsets"],
                                                                              df, DENSITY, 0))
                    row.update({"ms_sample": round(ms_s, 3), "sampled_points": int(poff[-1]),
                                "sampled_points_per_s": round(poff[-1] / (ms_s * 1e-3))})
                row["gpu"] = gpu
                print(json.dumps(row), flush=True)
                rows.append(row)
    if out:
        with open(out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in rows))
    ctx.close()


if __name__ == "__main__":
    main()
