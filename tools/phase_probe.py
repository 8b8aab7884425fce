#!/usr/bin/env python
"""Phase breakdown of k_images on the bench workload (development aid)."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gpd_b200 import lib, scenes
import bench
cloud, sidx = bench.make_workload(1, 20000)
p = lib.default_params(channels=15)
ctx = lib.Context(p)
ctx.set_weights(bench.load_weights())
ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
ctx.detect(sidx)
ctx.phase_cycles(1)
r = ctx.detect(sidx)
c = ctx.phase_cycles(1).astype(np.float64)
names = {2: "ball scan 1", 3: "point channels", 4: "shadow setup", 5: "shadow casting", 6: "shadow bitmap pass", 7: "shadow channels", 8: "flush"}
# sub-phases of the shadow half: slot, or (phase, slots) for "the phase minus those sub-phases"
subs = {5: [("cull + append", 16), ("window test", 17), ("draw evaluation", (5, [16, 17]))],
        6: [("intersect + expand", 18), ("eval_voxel", (6, [18]))],
        7: [("shadow_channel passes", 19), ("projection-2 stash sum", 20), ("tile clears", 21),
            ("(profiling scan only)", 22)]}
tot = c[2:9].sum()
nc = r["n_candidates"]
print("candidates", nc, "cycles per image", tot / nc)
for k, v in names.items():
    print(f"  {v:26s} {c[k] / tot:6.1%}  {c[k] / nc:10.0f} cycles/image")
    for sname, s in subs.get(k, []):
        val = c[s] if isinstance(s, int) else c[s[0]] - sum(c[j] for j in s[1])
        print(f"    {sname:24s} {val / tot:6.1%}  {val / nc:10.0f} cycles/image")
print(f"per image: ball points {c[13]/nc:.0f}, box points {c[12]/nc:.0f}, shadow work-list points {c[9]/nc:.0f}, "
      f"draws passing the window {c[10]/nc:.0f} of {33*c[9]/nc:.0f}, unique voxels evaluated {c[11]/nc:.0f}, "
      f"shadow cell-sum entries sharing their cell with another lane of the warp {c[23]/nc:.0f}")
