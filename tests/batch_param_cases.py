"""Inputs of the batch tests off the defaults (test_gpu_batch_params.py, test_gpu_preprocess_batch_params.py on the device;
test_batch_param_cases.py proves on the CPU that each reaches the path it names).

- Grown grid cells: a cloud whose bounding box would need more than 48e6 cells of 2 cm gets cells of 3 cm, then 4.5 cm
  (k_batch_desc). A few outlier points 8 m (one growth step) or 12 m (two steps) away on each axis do
  that to any table scene.
- The batch-wide cell guard: two-point clouds spanning 7.2 m on each axis need just under 48e6 cells each (no growth);
  46 of them need more than INT_MAX - 1 together, so gpdb_set_clouds refuses them with GPDB_ERR_CAPACITY.
- Ties in selection: the shipped weights with both rows of ip2 and both ip2 biases equal give two logits computed by
  the same operations, so every score is exactly +0.0. With the weight of one ip1 unit raised in row 1 only, the logits
  still agree wherever that unit is 0 after the ReLU: exact zeros beside distinct scores.
"""
import numpy as np

from gpd_b200 import scenes
from preprocess_cases import CAMS

GUARD_SPAN = 7.2        # m per axis of each cloud of the cell-guard batch
GUARD_CLOUDS = 46       # clouds of that batch: the first count whose cells exceed INT_MAX - 1
PARTIAL_TIE_UNIT = 290  # ip1 unit whose ip2 weights differ between the two logits: 0 on about half the table images


def table(seed, n=20000, **kw):
    return scenes.synthetic_table_scene(seed, n_points=n, **kw)


def cam_scene(k, seed=5, n=30000, mark_all=False, zero_rows=0.0):
    """A table scene seen by the first k cameras of CAMS; a fraction zero_rows of the cam_source rows is zeroed."""
    s = scenes.synthetic_table_scene(seed, n_points=n, cameras=CAMS[:k], mark_all_cameras=mark_all)
    if zero_rows > 0:
        s["cam_source"][np.random.default_rng(seed + k).random(n) < zero_rows] = 0
    return s


def with_outliers(cloud, dist):
    """The cloud plus one point `dist` metres from its mean along each axis (normal -z, seen by every camera)."""
    c = dict(cloud)
    far = (c["xyz"].astype(np.float64).mean(0) + dist * np.eye(3)).astype(np.float32)
    c["xyz"] = np.ascontiguousarray(np.vstack([c["xyz"], far]))
    c["normals"] = np.ascontiguousarray(np.vstack([c["normals"], np.tile([0.0, 0.0, -1.0], (3, 1))]))
    if c.get("cam_source") is not None:
        k = c["cam_source"].shape[1]
        c["cam_source"] = np.ascontiguousarray(np.vstack([c["cam_source"], np.ones((3, k), np.int32)]))
    return c


def guard_clouds(n=GUARD_CLOUDS):
    """n clouds of two points, the corners of a GUARD_SPAN cube (each cloud shifted a little, so no two are equal)."""
    out = []
    for b in range(n):
        o = np.float32(0.01 * b)
        xyz = np.array([[o, o, o], [o + GUARD_SPAN] * 3], np.float32)
        out.append({"xyz": xyz, "normals": np.tile([0.0, 0.0, -1.0], (2, 1)), "cam_source": None,
                    "view_points": np.zeros((1, 3))})
    return out


def tie_weights(w):
    """ip2 rows (W(o, k) at o + 2 k in the .bin layout) and biases made equal: both logits by the same operations."""
    w = [a.copy() for a in w]
    w[6] = w[6].reshape(-1).copy()
    w[6][1::2] = w[6][0::2]
    w[7] = np.full(2, w[7].reshape(-1)[0], np.float32)
    return w


def partial_tie_weights(w, unit=PARTIAL_TIE_UNIT, delta=1.0):
    """tie_weights, then row 1's weight of one ip1 unit raised by delta: score = 0 exactly where that unit is 0."""
    w = tie_weights(w)
    w[6][2 * unit + 1] = np.float32(w[6][2 * unit] + np.float32(delta))
    return w
