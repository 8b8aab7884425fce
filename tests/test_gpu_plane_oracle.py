"""The device (gpdb_segment_planes) against the C++ oracle of include/gpd_b200_plane.h (tests/plane_oracle.cpp) on a batch
of 32 preprocessed table views and mixed small clouds: hypotheses evaluated exactly; planes, inlier counts and masks
bit-equal wherever the refined planes are bit-equal, and the planes within the normals' float32 bound elsewhere."""
import numpy as np
import pytest

import plane_oracle as po
from gpd_b200 import lib, scenes

pytestmark = pytest.mark.gpu


def test_device_equals_the_oracle_on_preprocessed_views():
    raws = [scenes.synthetic_raw_scene(1000 + i, n_points=20000) for i in range(32)]
    ctx = lib.Context(lib.default_params(channels=12))
    ctx.preprocess_clouds([{"xyz": r["xyz"], "cam_source": r["cam_source"], "view_points": r["view_points"]} for r in raws])
    r = ctx.segment_planes(lib.plane_params(seed=5))
    clouds = ctx.get_clouds()
    off = np.concatenate([[0], np.cumsum([len(c["xyz"]) for c in clouds])]).astype(np.int32)
    o = po.segment_batch(off, np.concatenate([c["xyz"] for c in clouds]), seed=5)
    assert np.array_equal(r["n_hypotheses"], o["n_hypotheses"])
    same = [r["planes"][b].tobytes() == o["planes"][b].tobytes() for b in range(len(clouds))]
    for b in range(len(clouds)):
        if same[b]:
            assert r["n_inliers"][b] == o["n_inliers"][b]
            assert np.array_equal(r["eligible"][off[b]:off[b + 1]], o["eligible"][off[b]:off[b + 1]])
        else:
            n0, n1 = r["planes"][b][:3].astype(np.float64), o["planes"][b][:3].astype(np.float64)
            assert np.arccos(min(1.0, abs(float(n0 @ n1)))) < 1e-4
    print("clouds with bit-equal planes:", sum(same), "of", len(same))
    ctx.close()
