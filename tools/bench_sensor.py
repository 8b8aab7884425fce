"""gpdb_render_sensor_depth_device against gpdb_render_depth_device on the workloads of tools/bench_render.py: B = 1, 16,
64, 256 views of 640 x 480 at K = 1 and 2 cameras, mesh_table_scene tabletops of about 20 k and about 200 k faces. The
two calls alternate; each time is the median of 5 windows of CUDA events around one call, after a warm-up call of each.
The sensor runs the example model of INTEGRATION §5e (with a baseline, so the projector is a second render) and once
without a baseline (lateral jitter and dropout only). The card's name, power limit and clocks are read in the same run.
Usage: python tools/bench_sensor.py [out.jsonl]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]

from bench_render import SCENES, cameras  # noqa: E402

EXAMPLE = dict(baseline=0.075, lateral_sigma=0.5, disparity_sigma=0.05, disparity_step=0.125, min_cos_incidence=0.2,
               shadow_tolerance=0.01, dropout=0.01)


def main():
    import torch

    from gpd_b200 import lib, scenes
    out = sys.argv[1] if len(sys.argv) > 1 else None
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    ctx = lib.Context(lib.default_params())
    models = {"example": lib.sensor_params(**EXAMPLE), "no_baseline": lib.sensor_params(lateral_sigma=0.5, dropout=0.01)}
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
                calls = {"render": lambda: ctx.render_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [K] * B,
                                                                    cams, torch.uint16)}
                for name, sp in models.items():
                    calls[name] = (lambda sp=sp: ctx.render_sensor_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df,
                                                                                 [K] * B, cams, sp, 0, torch.uint16))
                res = {name: fn() for name, fn in calls.items()}  # warm-up
                ts = {name: [] for name in calls}
                for _ in range(5):
                    for name, fn in calls.items():
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        res[name] = fn()
                        b.record()
                        torch.cuda.synchronize()
                        ts[name].append(a.elapsed_time(b))
                med = {name: float(np.median(t)) for name, t in ts.items()}
                row = {"scene": label, "faces_per_view": faces, "views": B, "cameras": K, "image": "640x480",
                       "ms_render": round(med["render"], 3), "ms_sensor": round(med["example"], 3),
                       "ms_sensor_no_baseline": round(med["no_baseline"], 3),
                       "sensor_over_render": round(med["example"] / med["render"], 2),
                       "returns_render": int((res["render"].view(torch.int16) != 0).sum().item()),
                       "returns_sensor": int((res["example"].view(torch.int16) != 0).sum().item()),
                       "sensor": EXAMPLE, "gpu": gpu}
                print(json.dumps(row), flush=True)
                rows.append(row)
                del res
    if out:
        with open(out, "w") as f:
            f.write("".join(json.dumps(r) + "\n" for r in rows))
    ctx.close()


if __name__ == "__main__":
    main()
