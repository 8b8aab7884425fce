"""GPU parity tests (-m gpu) of gpdb_preprocess (SURVEY.md 8(f).1): the device NaN / workspace filter, voxelisation
and normal estimation against the CPU restatement (oracle/gpd_oracle.cpp) on identical inputs, through the C-ABI.

Bars: point coordinates, camera sources, source indices, voxel-averaged normals: bit-exact. Estimated normals:
every float32 operation follows the oracle's order (rank-sorted float32 sums, -fmad=false); the three libm calls of
pcl::computeRoots (atan2f, cosf, sinf) are correctly rounded on the device and glibc's on the host; a last-bit
difference there moves the smallest eigenvalue by one float32 ulp and the normal by ~1e-7 / (eigenvalue gap).
Bar: 1e-5 absolute (north_star: 1e-4),
>= 90 % bit-equal, no sign flips.
"""
import os

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from oracle import oracle

pytestmark = pytest.mark.gpu


def ctx15():
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    return p, ctx, oracle.WeightPack(w)


def assert_cloud_parity(ro, rg):
    assert len(ro["xyz"]) == len(rg["xyz"])
    assert np.array_equal(ro["src"], rg["src"])
    assert np.array_equal(ro["xyz"], rg["xyz"])
    assert np.array_equal(ro["cam_source"], rg["cam_source"])
    no, ng = ro["normals"], rg["normals"]
    assert np.array_equal(np.isnan(no), np.isnan(ng))
    d = np.abs(np.nan_to_num(no) - np.nan_to_num(ng))
    assert d.max() <= 1e-5
    assert (d.max(axis=1) == 0).mean() >= 0.90 or len(no) < 50
    assert (np.nan_to_num((no * ng).sum(1)) >= 0).all()


def test_krylon_raw_matches_oracle_and_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "krylon_preprocess.npz"))
    p, ctx, w = ctx15()
    pp = lib.preprocess_params()
    rg = ctx.preprocess(g["raw"], None, np.zeros((1, 3)), pp)
    ro = oracle.preprocess(g["raw"], None, np.zeros((1, 3)), pp)
    assert_cloud_parity(ro, rg)
    assert np.array_equal(rg["xyz"], g["xyz"]) and np.abs(rg["normals"] - g["normals"]).max() <= 1e-5
    # the path runs on the cloud the preprocessing installed: same results as uploading the oracle's cloud
    sidx = scenes.sample_indices(2, len(rg["xyz"]), 64)
    r1 = ctx.detect(sidx)
    ctx.set_cloud(rg["xyz"], rg["normals"], rg["cam_source"], rg["view_points"])
    r2 = ctx.detect(sidx)
    assert np.array_equal(r1["pose_flags"], r2["pose_flags"]) and np.array_equal(r1["pose_scores"], r2["pose_scores"], equal_nan=True)
    ctx.close()


def test_two_view_raw_scene_with_nans_matches_oracle():
    s = scenes.synthetic_raw_scene(7, n_points=60000, two_cameras=True, nan_fraction=0.01)
    p, ctx, w = ctx15()
    pp = lib.preprocess_params(workspace=[-0.6, 0.6, -0.5, 0.5, 0.2, 1.0])
    rg = ctx.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
    ro = oracle.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
    assert 0 < len(rg["xyz"]) < len(s["xyz"])
    assert_cloud_parity(ro, rg)
    ctx.close()


def test_supplied_normals_are_voxel_averaged_bit_exactly_and_no_voxelise_mode():
    rng = np.random.default_rng(11)
    s = scenes.synthetic_raw_scene(9, n_points=20000)
    nrm = rng.standard_normal((len(s["xyz"]), 3))
    p, ctx, w = ctx15()
    for vox in (1, 0):
        pp = lib.preprocess_params(estimate_normals=0, voxelize=vox, voxel_size=0.004)
        rg = ctx.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp, normals=nrm)
        ro = oracle.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp, normals=nrm)
        assert np.array_equal(ro["normals"], rg["normals"])
        assert_cloud_parity(ro, rg)
    ctx.close()


def test_edge_cases():
    p, ctx, w = ctx15()
    vp = np.zeros((1, 3))
    # everything filtered out -> 0 points, and the context has no cloud
    far = np.full((10, 3), 5.0, np.float32)
    assert ctx.preprocess(far, None, vp, lib.preprocess_params(), read_back=False) == 0
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect(np.zeros(1, np.int32))
    assert e.value.code == -3
    # isolated point: fewer than 3 neighbours -> NaN normal (pcl::computePointNormal)
    iso = np.array([[0.3, 0.3, 0.3], [0.0, 0.0, 0.5], [0.001, 0.0, 0.5], [0.0, 0.001, 0.5], [0.001, 0.001, 0.5]], np.float32)
    pp = lib.preprocess_params(voxelize=0)
    rg = ctx.preprocess(iso, None, vp, pp)
    ro = oracle.preprocess(iso, None, vp, pp)
    assert_cloud_parity(ro, rg)
    assert np.isnan(rg["normals"][0]).all()
    # bad arguments
    with pytest.raises(lib.GpdbError):
        ctx.preprocess(iso, None, vp, lib.preprocess_params(estimate_normals=0))
    with pytest.raises(lib.GpdbError):
        ctx.preprocess(iso, None, vp, lib.preprocess_params(voxel_size=0.0))
    # dense blob: more than the tier-1 capacity of neighbours per point -> the large-tile tier, same result
    rng = np.random.default_rng(3)
    blob = (rng.uniform(-0.02, 0.02, (3000, 3)) + [0, 0, 0.5]).astype(np.float32)
    pp = lib.preprocess_params(voxelize=0)
    assert_cloud_parity(oracle.preprocess(blob, None, vp, pp), ctx.preprocess(blob, None, vp, pp))
    ctx.close()


def test_full_size_raw_cloud_properties_and_parity():
    """BASELINE-size raw cloud (~0.9 M points -> ~0.5 M voxels): parity against the oracle at full size plus the
    size-independent properties (one point per voxel at its corner, unit normals facing the camera)."""
    s = scenes.synthetic_raw_scene(3)
    p, ctx, w = ctx15()
    pp = lib.preprocess_params()
    rg = ctx.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
    ro = oracle.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
    assert_cloud_parity(ro, rg)
    n = rg["normals"]
    assert not np.isnan(n).any() and np.abs(np.linalg.norm(n, axis=1) - 1).max() < 1e-5
    assert (((rg["xyz"].astype(np.float64) - s["view_points"][0]) * n).sum(1) < 0).all()
    # voxel semantics: one point per occupied voxel (all distinct), each the corner of the voxel that holds its
    # source point: 0 <= raw[src] - voxel < cell (up to float32 rounding of the corner)
    assert len(np.unique(rg["xyz"], axis=0)) == len(rg["xyz"])
    off = s["xyz"][rg["src"]].astype(np.float64) - rg["xyz"].astype(np.float64)
    assert off.min() > -1e-6 and off.max() < 0.003 + 1e-6
    # the path runs on the installed cloud
    r = ctx.detect(scenes.sample_indices(3, len(rg["xyz"]), 2000))
    assert r["n_candidates"] > 0 and np.isfinite(r["candidates"]["score"]).all()
    ctx.close()
