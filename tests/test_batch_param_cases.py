"""The inputs of the batch tests off the defaults reach what they claim (CPU, float32 numpy and the oracle): grids whose
cell grew past 2 cm, the batch-wide cell guard, camera counts and all_seen per cloud, and the tie weights."""
import numpy as np

from batch_param_cases import (GUARD_CLOUDS, cam_scene, guard_clouds, partial_tie_weights, table, tie_weights,
                               with_outliers)
from conftest import load_weights
from gpd_b200 import lib, scenes
from oracle import oracle
from preprocess_cases import grid_of
from test_gpu_parity import _lattice_cloud

INT_MAX = 2 ** 31 - 1


def test_outliers_grow_the_cell_once_and_twice():
    c15, c225 = np.float32(np.float32(0.02) * np.float32(1.5)), None
    c225 = np.float32(c15 * np.float32(1.5))
    for base in (table(7, n=30000), table(4), table(6, two_cameras=True), _lattice_cloud(0.0012)[0]):
        assert grid_of(base["xyz"])[4] == 0
        for dist, steps, cell in ((8.0, 1, c15), (12.0, 2, c225)):
            xyz = with_outliers(base, dist)["xyz"]
            lo, dim, got_cell, cells, got_steps = grid_of(xyz)
            assert got_steps == steps and got_cell == cell and cells <= 48e6
            # one step less would need more than 48e6 cells
            prev = cell / np.float32(1.5)
            ext = xyz.max(0) - xyz.min(0)
            assert np.prod((np.floor(ext / np.float32(prev)) + 2).astype(np.float64)) > 48e6
            assert np.array_equal(dim, np.floor(ext / cell).astype(np.int64) + 2)
    assert abs(float(c15) - 0.03) < 1e-8 and abs(float(c225) - 0.045) < 1e-8


def test_guard_batch_exceeds_int_max_only_together():
    clouds = guard_clouds()
    grids = [grid_of(c["xyz"]) for c in clouds]
    assert all(g[4] == 0 and g[3] <= 48e6 for g in grids)
    assert all(g[3] > 47e6 for g in grids)  # just under 48e6 each
    total = sum(g[3] for g in grids)
    assert total + 1 > INT_MAX
    assert total - grids[-1][3] + 1 <= INT_MAX  # GUARD_CLOUDS - 1 clouds would pass the guard
    assert len(clouds) == GUARD_CLOUDS


def test_camera_mixes_and_all_seen():
    for k in (1, 2, 3, 4, 6, 8):
        assert len(cam_scene(k, seed=4 + k)["view_points"]) == k
    for k in (1, 2):
        s = cam_scene(k, seed=5 + 2 * (k == 1), mark_all=True, zero_rows=0.1)
        bits = s["cam_source"].sum(1)
        assert not (bits == k).all() and 0.05 < (bits == 0).mean() < 0.2
        assert k == 1 or (bits >= 2).mean() > 0.2
        plain = cam_scene(k, seed=6 + 2 * (k == 1))
        assert (plain["cam_source"].sum(1) >= 1).all()  # seen by one camera, not all: all_seen only without cam_source
        assert k == 1 or not (plain["cam_source"] > 0).all()


def test_tie_weights_give_identical_and_partly_identical_logits():
    """On the images of the selection tests (the table scene, 200 samples): equal ip2 rows give bit-equal logits and
    scores of +0.0; the partial tie gives exact zeros on at least a fifth of the images and distinct scores on a fifth."""
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu, keep_images=1)
    t = table(3)
    oc = oracle.OracleCloud(t["xyz"], t["normals"], t["cam_source"], t["view_points"])
    imgs = oc.detect(p, oracle.WeightPack(w), scenes.sample_indices(1, 20000, 200))["images"]
    assert len(imgs) > 150
    s, lg = oracle.classify(p, oracle.WeightPack(tie_weights(w)), imgs)
    assert np.array_equal(lg[:, 0].view(np.uint32), lg[:, 1].view(np.uint32)) and (s.view(np.uint32) == 0).all()
    s0, _ = oracle.classify(p, oracle.WeightPack(w), imgs)
    assert len(np.unique(s0)) > 0.9 * len(s0)  # the shipped weights do not tie
    s, lg = oracle.classify(p, oracle.WeightPack(partial_tie_weights(w)), imgs)
    zero = s == 0
    assert zero.sum() >= 0.2 * len(s) and len(np.unique(s[~zero])) >= 0.2 * len(s)
    assert np.array_equal(lg[zero, 0], lg[zero, 1]) and (s[~zero] > 0).all()


def test_grown_normals_grid_of_the_preprocessing_case():
    s = scenes.synthetic_raw_scene(6, n_points=20000)
    far = (s["xyz"].astype(np.float64).mean(0) + 8.0 * np.eye(3)).astype(np.float32)
    xyz = np.vstack([s["xyz"], far])
    assert grid_of(s["xyz"])[4] == 0 and grid_of(xyz)[4] == 1
