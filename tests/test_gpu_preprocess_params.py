"""GPU parity of gpdb_preprocess off its defaults (-m gpu): normals radius, voxel size, camera sets, the two neighbour
tiers of k_normals and the capacity error, degenerate neighbourhoods, filter edges, the voxel index range, repeated use of
one context, and the grasp path on a preprocessed cloud, each against the CPU oracle on identical inputs.

Bars (assert_cloud_parity, as test_gpu_preprocess.py): coordinates, source indices, camera sources and voxel-averaged
normals bit-equal; estimated normals within 1e-5, >= 90 % bit-equal, no sign flips; NaN only against NaN. Each case
also checks from its inputs that it reaches the path it names (oracle radius-search counts, grid rows from the 2 cm cell,
camera bits), and the radius, camera and lattice cases are checked against plain numpy as well (preprocess_cases.py):
the filter mask, the voxel set and its order, and a float64 PCA of each ball.
"""
import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from oracle import oracle
from preprocess_cases import (TABLE_WS, TIER0_CAP, TIER1_CAP, Q, ball_counts, clusters, filter_mask, grid_rows,
                              lattice, pca_check, raw_table, voxel_reference)
from test_gpu_parity import assert_parity
from test_gpu_preprocess import assert_cloud_parity

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    w, relu = load_weights(15)
    c = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    c.set_weights(w)
    c.weights = oracle.WeightPack(w)
    yield c
    c.close()


def run_both(ctx, xyz, cam, vp, pp, normals=None):
    rg = ctx.preprocess(xyz, cam, vp, pp, normals=normals)
    ro = oracle.preprocess(xyz, cam, vp, pp, normals=normals)
    assert_cloud_parity(ro, rg)
    return ro, rg


def check_numpy(raw, pp, rg, n_pca=300):
    """The device result against the numpy references: filter mask, voxel set and order, float64 PCA normals."""
    ws = list(pp.workspace)
    if pp.voxelize:
        src, pts = voxel_reference(raw, ws, pp.voxel_size)
        assert np.array_equal(rg["src"], src) and np.array_equal(rg["xyz"], pts)
    else:
        keep = np.nonzero(filter_mask(raw, ws))[0]
        assert np.array_equal(rg["src"], keep) and np.array_equal(rg["xyz"], np.asarray(raw, np.float32)[keep])
    if pp.estimate_normals:
        idx = np.unique(np.linspace(0, len(rg["xyz"]) - 1, min(n_pca, len(rg["xyz"]))).astype(int))
        checked, worst = pca_check(rg, pp.normals_radius, idx)
        assert worst <= 1.0, worst
        return checked
    return 0


# ---- normals radius -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [0.005, 0.01, 0.05, 0.08])
def test_normals_radius_sweep(ctx, r):
    """0.005 / 0.01: balls of a few voxels (points with < 3 neighbours get NaN normals); 0.05 / 0.08: more than 32 grid
    rows per ball, so k_normals' row loop takes a second pass; 0.08: interior balls hold more than 1 024 neighbours and
    run in the second tier."""
    s = raw_table(seed=7, nan_fraction=0.01)
    pp = lib.preprocess_params(workspace=TABLE_WS, normals_radius=r)
    ro, rg = run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], pp)
    rows = grid_rows(rg["xyz"], r)
    if r >= 0.05:
        assert (rows > 32).sum() > 10000
    else:
        assert rows.max() <= 32
    probe = np.linspace(0, len(rg["xyz"]) - 1, 200).astype(int)
    cnt = ball_counts(rg["xyz"], probe, r)
    if r == 0.005:
        assert np.isnan(rg["normals"][:, 0]).sum() > 0 and cnt.min() < 3
    if r == 0.08:
        assert cnt.max() > TIER0_CAP
    assert check_numpy(s["xyz"], pp, rg) > 100


# ---- voxel size -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("supplied", [False, True])
@pytest.mark.parametrize("cell", [0.001, 0.005, 0.02])
def test_voxel_size_sweep(ctx, cell, supplied):
    s = raw_table(seed=9)
    nrm = np.random.default_rng(1).standard_normal((len(s["xyz"]), 3)) if supplied else None
    pp = lib.preprocess_params(workspace=TABLE_WS, voxel_size=cell, estimate_normals=0 if supplied else 1)
    ro, rg = run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], pp, normals=nrm)
    if supplied:
        assert np.array_equal(ro["normals"], rg["normals"])
    check_numpy(s["xyz"], pp, rg, n_pca=100)
    # several raw points per voxel at 5 and 20 mm, about one at 1 mm
    assert len(rg["xyz"]) < filter_mask(s["xyz"], TABLE_WS).sum()


def test_lattice_on_voxel_boundaries(ctx):
    """An exact plane lattice whose step is the voxel size: every (p - min) / cell is an integer. Copies shifted by one
    and three quarters of a cell land in the same voxels (three points per voxel, in shuffled order)."""
    step = 4
    base = lattice((-100 * step, -80 * step, 512), (step, 0, 0), (0, step, 0), 120, 100)
    pts = np.vstack([base, base + np.float32([Q, Q, 0]), base + np.float32([3 * Q, 3 * Q, 0])])
    pts = pts[np.random.default_rng(2).permutation(len(pts))]
    for est in (1, 0):
        pp = lib.preprocess_params(voxel_size=step * Q, estimate_normals=est)
        nrm = None if est else np.random.default_rng(3).standard_normal((len(pts), 3))
        ro, rg = run_both(ctx, pts, None, np.zeros((1, 3)), pp, normals=nrm)
        assert len(rg["xyz"]) == len(base) and np.array_equal(np.sort(rg["xyz"], 0), np.sort(base, 0))
        check_numpy(pts, pp, rg)


# ---- cameras --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vox", [1, 0])
@pytest.mark.parametrize("k", [3, 4, 8])
def test_camera_sets(ctx, k, vox):
    """Every camera that sees a point is marked, and 3 % of the rows are zeroed (no camera: zero normal). The flip uses
    the first camera that sees the point (vp[2..7] included), reverseNormals every camera that sees it."""
    s = raw_table(seed=5, n_cams=k, mark_all=True, zero_rows=0.03)
    pp = lib.preprocess_params(workspace=TABLE_WS, voxelize=vox)
    ro, rg = run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], pp)
    cs = rg["cam_source"]
    assert cs.shape[1] == k and (cs.sum(1) >= 2).mean() > 0.2 and (cs.sum(1) == 0).any()
    assert (np.bincount(np.argmax(cs[cs.any(1)], axis=1), minlength=k)[2:] > 0).any()
    assert (rg["normals"][cs.sum(1) == 0] == 0).all()
    check_numpy(s["xyz"], pp, rg)


def test_viewpoint_flip_and_reverse_use_the_right_cameras(ctx):
    """Exact plane z = 0, so every normal is exactly (0, 0, +-1); camera 0 lies in the plane (flip test exactly 0, it never
    decides), camera 1 below, camera 2 above. Expected: seen by {0, 2} -> +z (only camera 2 keeps it), {1, 2} -> -z (the
    flip is towards camera 1, which keeps it), {0, 1} -> -z, {1} -> -z, {2} -> +z."""
    pts = lattice((-50 * 4, -50 * 4, 0), (4, 0, 0), (0, 4, 0), 100, 100)
    vp = np.array([[0.75, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 0.0, 1.0]])
    sets = [(0, 2), (1, 2), (0, 1), (1,), (2,), (0,), ()]
    want = [1.0, -1.0, -1.0, -1.0, 1.0, None, 0.0]
    which = np.arange(len(pts)) % len(sets)
    cam = np.zeros((len(pts), 3), np.int32)
    for w, st in enumerate(sets):
        for c in st:
            cam[which == w, c] = 1
    pp = lib.preprocess_params(voxelize=0)
    ro, rg = run_both(ctx, pts, cam, vp, pp)
    n = rg["normals"]
    assert np.array_equal(ro["normals"], n) and (n[:, :2] == 0).all()
    for w, z in enumerate(want):
        if z is not None:
            assert (n[which == w, 2] == z).all(), sets[w]


@pytest.mark.parametrize("vox", [1, 0])
def test_cam_source_value_two(ctx, vox):
    """Entries other than 0 / 1: with voxelisation a camera sees a point only at exactly 1, like the reference and the
    oracle. Without it the reference keeps the raw values, so the device rejects them (GPDB_ERR_INVALID)."""
    s = raw_table(seed=5, n_cams=3, mark_all=True)
    cs = s["cam_source"].copy()
    cs[(np.random.default_rng(4).random(cs.shape) < 0.3) & (cs == 1)] = 2
    if vox:
        pp = lib.preprocess_params(workspace=TABLE_WS)
        ro, rg = run_both(ctx, s["xyz"], cs, s["view_points"], pp)
        assert (cs[rg["src"]] == 2).any()
        assert np.array_equal(rg["cam_source"], (cs[rg["src"]] == 1).astype(np.int32))
        return
    pp = lib.preprocess_params(workspace=TABLE_WS, voxelize=0, estimate_normals=0)
    nrm = np.zeros((len(cs), 3))
    assert (oracle.preprocess(s["xyz"], cs, s["view_points"], pp, normals=nrm)["cam_source"] == 2).any()
    with pytest.raises(lib.GpdbError) as e:
        ctx.preprocess(s["xyz"], cs, s["view_points"], pp, normals=nrm)
    assert e.value.code == -1 and "0 or 1" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect(np.zeros(1, np.int32))
    assert e.value.code == -3
    run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], pp, normals=nrm)


# ---- neighbour tiers ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [TIER0_CAP, TIER0_CAP + 1, TIER1_CAP])
def test_normal_tier_boundaries(ctx, n):
    """An isolated cluster whose points all lie in each other's ball: exactly n neighbours per point (the oracle's radius
    search counts them), the most the first tier holds (1 024), one more (second tier), and the most the second tier
    holds (8 192)."""
    pts = np.vstack([clusters([n], 0.03), clusters([5, 40], 0.03, seed=8) + np.float32([0, 0.3, 0])])
    pp = lib.preprocess_params(voxelize=0)
    ro, rg = run_both(ctx, pts, None, np.zeros((1, 3)), pp)
    assert (ball_counts(pts, [0, n // 2, n - 1], 0.03) == n).all()
    assert not np.isnan(rg["normals"]).any()


def test_capacity_error_then_recovery(ctx):
    """8 193 neighbours: GPDB_ERR_CAPACITY naming the radius; no cloud is left, and the same context then preprocesses and
    runs the grasp path with oracle parity."""
    pts = clusters([TIER1_CAP + 1], 0.03)
    with pytest.raises(lib.GpdbError) as e:
        ctx.preprocess(pts, None, np.zeros((1, 3)), lib.preprocess_params(voxelize=0))
    assert e.value.code == -5 and "normals_radius 0.03" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect(np.zeros(1, np.int32))
    assert e.value.code == -3
    s = raw_table(seed=7)
    ro, rg = run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], lib.preprocess_params(workspace=TABLE_WS))
    detect_against_oracle(ctx, rg, scenes.sample_indices(5, len(rg["xyz"]), 300))
    run_both(ctx, clusters([TIER1_CAP], 0.03), None, np.zeros((1, 3)), lib.preprocess_params(voxelize=0))


# ---- degenerate neighbourhoods --------------------------------------------------------------------------------------
def test_degenerate_neighbourhoods(ctx):
    """Exact plane (pcl_roots2), tilted exact lattice (distance ties everywhere: the (dist, index) sort key decides the
    float32 sum order), collinear points, coincident points (zero covariance: 0 / 0 normal), 1- and 2-point clouds."""
    vp = np.zeros((1, 3))
    pp = lib.preprocess_params(voxelize=0)
    plane = lattice((-30 * 4, -30 * 4, 512), (4, 0, 0), (0, 4, 0), 60, 60)
    tilted = lattice((-100, -100, 480), (4, 0, 1), (0, 4, 2), 60, 60)
    for pts in (plane, tilted):
        ro, rg = run_both(ctx, pts, None, vp, pp)
        assert not np.isnan(rg["normals"]).any()
        check_numpy(pts, pp, rg)
    assert (run_both(ctx, plane, None, vp, pp)[1]["normals"][:, :2] == 0).all()
    # ties: many neighbours at exactly equal float32 distances (exact lattice: distances are integers in Q^2)
    oc = oracle.OracleCloud(tilted, np.zeros((len(tilted), 3)))
    _, d = oc.radius_search(tilted[1830], 0.03)
    assert len(d) - len(np.unique(d)) > len(d) // 2
    line = lattice((-100 * 4, 100, 500), (4, 0, 0), (0, 0, 0), 200, 1)
    run_both(ctx, line, None, vp, pp)
    coinc = np.vstack([np.tile(np.float32([0.2, 0.2, 0.6]), (5, 1)), lattice((-40, -40, 512), (4, 0, 0), (0, 4, 0), 20, 20)])
    ro, rg = run_both(ctx, coinc, None, vp, pp)
    assert np.isnan(rg["normals"][:5]).all() and not np.isnan(rg["normals"][5:]).any()
    for k in (1, 2):
        ro, rg = run_both(ctx, plane[:k], None, vp, pp)
        assert len(rg["xyz"]) == k and np.isnan(rg["normals"]).all()


# ---- filter edges ---------------------------------------------------------------------------------------------------
def test_filter_edges(ctx):
    """Coordinates equal to each of the six bounds (dropped: strict inequalities), one float32 step inside and outside
    them, a bound that float32 cannot represent (0.1), and NaN / +inf / -inf in each axis."""
    ws = [-0.5, 0.5, -0.25, 0.1, 0.25, 1.0]
    base = lattice((-60 * 4, -40 * 4, 600), (4, 0, 0), (0, 4, 0), 120, 80)
    inside = np.float32([0.0, 0.0, 0.6])
    extra, on_bound = [], []
    for a in range(3):
        for side in (0, 1):
            b = np.float32(ws[2 * a + side])
            for v in (b, np.nextafter(b, np.float32(0.6 if a == 2 else 0.0)), np.nextafter(b, np.float32(9 if side else -9))):
                p = inside.copy()
                p[a] = v
                extra.append(p)
                on_bound.append(float(v) == ws[2 * a + side])
        for bad in (np.nan, np.inf, -np.inf):
            p = inside.copy()
            p[a] = bad
            extra.append(p)
            on_bound.append(False)
    pts = np.vstack([base, np.array(extra, np.float32)])
    mask = filter_mask(pts, ws)
    assert sum(on_bound) == 5 and not mask[len(base):][np.array(on_bound)].any()
    for vox in (1, 0):
        pp = lib.preprocess_params(workspace=ws, voxelize=vox)
        ro, rg = run_both(ctx, pts, None, np.zeros((1, 3)), pp)
        check_numpy(pts, pp, rg, n_pca=50)
        assert set(rg["src"]) <= set(np.nonzero(mask)[0])


def test_workspace_of_one_voxel_and_translated_cloud(ctx):
    s = raw_table(seed=9)
    q = s["xyz"][1234].astype(np.float64)
    ws = [q[0] - 5e-4, q[0] + 5e-4, q[1] - 5e-4, q[1] + 5e-4, q[2] - 5e-4, q[2] + 5e-4]
    pp = lib.preprocess_params(workspace=ws)
    ro, rg = run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], pp)
    assert len(rg["xyz"]) == 1 and filter_mask(s["xyz"], ws).sum() >= 1
    check_numpy(s["xyz"], pp, rg)
    off = np.array([-3.0, 2.0, -1.5])
    xyz = (s["xyz"].astype(np.float64) + off).astype(np.float32)
    ws = [TABLE_WS[i] + off[i // 2] for i in range(6)]
    pp = lib.preprocess_params(workspace=ws)
    ro, rg = run_both(ctx, xyz, s["cam_source"], s["view_points"] + off, pp)
    assert len(rg["xyz"]) > 10000
    check_numpy(xyz, pp, rg, n_pca=100)


# ---- voxel index range ----------------------------------------------------------------------------------------------
def test_voxel_index_range(ctx):
    """Cell 2^-20 over 2 m: the largest voxel index 2^21 - 1 still matches the oracle; one point at 2^21 is
    GPDB_ERR_INVALID and leaves no cloud."""
    cell = 2.0 ** -20
    rng = np.random.default_rng(6)
    k = np.concatenate([[0, 1, 2 ** 20, 2 ** 21 - 2, 2 ** 21 - 1], rng.integers(0, 2 ** 21, 600)])
    pts = np.stack([0.25 + k * cell, 0.1 + rng.integers(0, 64, len(k)) * Q, 0.5 + rng.integers(0, 64, len(k)) * Q], 1)
    pts = pts.astype(np.float32)
    assert np.array_equal(pts[:, 0].astype(np.float64), 0.25 + k * cell)
    pp = lib.preprocess_params(workspace=[-1, 3, -1, 1, -1, 1], voxel_size=cell)
    ro, rg = run_both(ctx, pts, None, np.zeros((1, 3)), pp)
    check_numpy(pts, pp, rg, n_pca=50)
    over = np.vstack([pts, np.float32([[0.25 + 2.0, 0.1, 0.5]])])
    with pytest.raises(lib.GpdbError) as e:
        ctx.preprocess(over, None, np.zeros((1, 3)), pp)
    assert e.value.code == -1 and "2^21" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx.detect(np.zeros(1, np.int32))
    assert e.value.code == -3


# ---- repeated use ---------------------------------------------------------------------------------------------------
def test_repeated_use_matches_fresh_contexts(ctx, golden_dir):
    """Large, small, large on one context (grow-only cloud arena and scratch slots reused at a smaller size): byte-equal
    to a fresh context each time."""
    import os
    big = raw_table(seed=11, n_cams=2, mark_all=True)
    small = {"xyz": np.load(os.path.join(golden_dir, "krylon_preprocess.npz"))["raw"], "cam_source": None,
             "view_points": np.zeros((1, 3))}
    for s, ws in ((big, TABLE_WS), (small, [-1, 1, -1, 1, -1, 1]), (big, TABLE_WS)):
        pp = lib.preprocess_params(workspace=ws)
        r1 = ctx.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
        fresh = lib.Context(ctx.params)
        r2 = fresh.preprocess(s["xyz"], s["cam_source"], s["view_points"], pp)
        fresh.close()
        for key in ("xyz", "normals", "cam_source", "src"):
            assert r1[key].shape == r2[key].shape and r1[key].tobytes() == r2[key].tobytes(), key


# ---- preprocess, then detect ----------------------------------------------------------------------------------------
def detect_against_oracle(ctx, rg, sidx):
    rd = ctx.detect(sidx)
    oc = oracle.OracleCloud(rg["xyz"], rg["normals"], rg["cam_source"], rg["view_points"])
    ro = oc.detect(ctx.params, ctx.weights, sidx)
    assert_parity(ro, rd, 15, equal_nan=True)
    return ro, rd


def detect_scene(ctx, zero_rows):
    """Raw table scene plus isolated pairs of points 5 mm apart (two neighbours each: NaN normals); a fraction zero_rows
    of the camera rows is zeroed (zero normals). Returns the device's processed cloud and samples that include both
    kinds of points."""
    s = raw_table(seed=13, n_cams=2, mark_all=True, zero_rows=zero_rows)
    g = np.stack(np.meshgrid(np.arange(-4, 5) * 0.1, np.arange(-3, 4) * 0.1, indexing="ij"), -1).reshape(-1, 2)
    pairs = np.vstack([np.c_[g, np.full(len(g), 0.45)], np.c_[g + [0.005, 0.0], np.full(len(g), 0.45)]]).astype(np.float32)
    xyz = np.vstack([s["xyz"], pairs])
    cam = np.vstack([s["cam_source"], np.tile([1, 0], (len(pairs), 1)).astype(np.int32)])
    ro, rg = run_both(ctx, xyz, cam, s["view_points"], lib.preprocess_params(workspace=TABLE_WS))
    nan_pts = np.nonzero(np.isnan(rg["normals"][:, 0]))[0]
    zero_pts = np.nonzero(~rg["cam_source"].any(1))[0]
    assert len(nan_pts) >= len(pairs) and (len(zero_pts) > 100) == (zero_rows > 0)
    sidx = np.unique(np.concatenate([nan_pts, zero_pts[:300], scenes.sample_indices(5, len(rg["xyz"]), 400)])).astype(np.int32)
    return rg, sidx


def test_preprocessed_cloud_detect_matches_oracle(ctx):
    """NaN normals reach k_frames (NaN frames at the pairs, compared NaN against NaN), k_hands and k_images."""
    rg, sidx = detect_scene(ctx, 0.0)
    ro, rd = detect_against_oracle(ctx, rg, sidx)
    assert np.isnan(rd["frames"]).any() and rd["n_candidates"] > 100


def test_zero_normals_grasp_images_match_oracle(ctx):
    """Points no camera sees carry zero normals into the grasp images. createNormalsImage folds every writer of a cell into
    it, v += (|n| - v) / ||v||; a zero normal after a unit one leaves v near 1e-8, and the next writer is scaled by about
    1e8 and sets the image maximum. Such images replay the fold in (dist, index) order."""
    rg, sidx = detect_scene(ctx, 0.02)
    ro, rd = detect_against_oracle(ctx, rg, sidx)
    assert rd["n_candidates"] > 100


def test_supplied_normals_voxel_averages_detect_matches_oracle(ctx):
    """estimate_normals = 0: the voxel-averaged supplied normals are not of unit length, in every image."""
    s = raw_table(seed=13, n_cams=2)
    rng = np.random.default_rng(5)
    nrm = rng.standard_normal((len(s["xyz"]), 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pp = lib.preprocess_params(workspace=TABLE_WS, estimate_normals=0)
    ro, rg = run_both(ctx, s["xyz"], s["cam_source"], s["view_points"], pp, normals=nrm)
    l2 = (rg["normals"] ** 2).sum(1)
    assert (np.abs(l2 - 1) > 1e-3).mean() > 0.5
    ro, rd = detect_against_oracle(ctx, rg, scenes.sample_indices(5, len(rg["xyz"]), 400))
    assert rd["n_candidates"] > 50
