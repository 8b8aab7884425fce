"""CPU checks of the inputs of test_gpu_preprocess_params.py (preprocess_cases.py): the clusters are what the tier cases
need, the lattices are exact, the numpy references agree with the oracle, and the path names hold for the inputs."""
import numpy as np

from gpd_b200 import abi
from oracle import oracle
from preprocess_cases import (Q, TABLE_WS, TIER0_CAP, TIER1_CAP, ball_counts, clusters, filter_mask, grid_rows,
                              lattice, pca_check, raw_table, voxel_reference)


def test_clusters_are_isolated_and_mutually_inside_the_ball():
    r = 0.03
    sizes = [TIER0_CAP, TIER0_CAP + 1, 7, TIER1_CAP]
    pts = clusters(sizes, r)
    start = np.cumsum([0] + sizes)
    boxes = []
    for a, b in zip(start[:-1], start[1:]):
        p = pts[a:b].astype(np.float64)
        assert np.linalg.norm(p.max(0) - p.min(0)) < 0.5 * r  # diameter: every pair well inside r
        boxes.append((p.min(0), p.max(0)))
    for i in range(len(boxes)):
        for j in range(i + 1, len(boxes)):
            gap = np.maximum(boxes[j][0] - boxes[i][1], boxes[i][0] - boxes[j][1]).max()
            assert gap > 2 * r
    assert (ball_counts(pts, start[:-1], r) == sizes).all()
    assert (ball_counts(pts, start[1:] - 1, r) == sizes).all()


def test_lattices_are_exact_and_full_of_distance_ties():
    tilted = lattice((-100, -100, 480), (4, 0, 1), (0, 4, 2), 60, 60)
    i, j = np.meshgrid(np.arange(60), np.arange(60), indexing="ij")
    k = np.stack([-100 + 4 * i, -100 + 4 * j, 480 + i + 2 * j], -1).reshape(-1, 3)
    assert np.array_equal(tilted.astype(np.float64), k * Q)
    # float32 squared distances between lattice points are exact integers in units of Q^2
    d = tilted[1830] - tilted
    d2 = (d * d).sum(1, dtype=np.float32).astype(np.float64)
    assert np.array_equal(d2, ((k[1830] - k) ** 2).sum(1) * Q * Q)
    oc = oracle.OracleCloud(tilted, np.zeros((len(tilted), 3)))
    _, dist = oc.radius_search(tilted[1830], 0.03)
    assert len(dist) > 100 and len(dist) - len(np.unique(dist)) > len(dist) // 2


def test_grid_rows_reach_a_second_row_pass_only_from_r_005():
    s = raw_table(seed=7)
    pp = abi.default_preprocess_params(workspace=TABLE_WS, estimate_normals=0)
    xyz = oracle.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp, normals=np.zeros((len(s["xyz"]), 3)))["xyz"]
    # the table (most of the points) lies at the cloud's largest z: its balls are cut by the grid's last z row
    assert grid_rows(xyz, 0.03).max() <= 32 and grid_rows(xyz, 0.01).max() <= 32
    assert (grid_rows(xyz, 0.05) > 32).sum() > 10000 and (grid_rows(xyz, 0.08) > 32).mean() > 0.9


def test_numpy_references_agree_with_the_oracle():
    """Filter mask, voxel set and PCA normals of preprocess_cases.py against the oracle on the raw table scene with
    three cameras, NaN coordinates and zeroed camera rows."""
    s = raw_table(seed=5, n_cams=3, mark_all=True, zero_rows=0.03, nan_fraction=0.01)
    s["xyz"] = s["xyz"][:30000]
    s["cam_source"] = s["cam_source"][:30000]
    pp = abi.default_preprocess_params(workspace=TABLE_WS)
    r = oracle.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
    src, pts = voxel_reference(s["xyz"], TABLE_WS, 0.003)
    assert np.array_equal(r["src"], src) and np.array_equal(r["xyz"], pts)
    assert filter_mask(s["xyz"], TABLE_WS)[r["src"]].all() and (~filter_mask(s["xyz"], TABLE_WS)).sum() > 200
    checked, worst = pca_check(r, 0.03, np.arange(0, len(r["xyz"]), 97))
    assert checked > 50 and worst <= 1.0
    pp0 = abi.default_preprocess_params(workspace=TABLE_WS, voxelize=0, estimate_normals=0)
    r0 = oracle.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp0, normals=np.zeros((30000, 3)))
    assert np.array_equal(r0["src"], np.nonzero(filter_mask(s["xyz"], TABLE_WS))[0])
