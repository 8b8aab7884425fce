"""gpdb_preprocess_clouds off the defaults, on the GPU: one batch per parameter set of test_gpu_preprocess_params.py.

Every processed cloud must be bit-equal to gpdb_preprocess on that raw cloud alone, and the batch's gpdb_detect_batch
bit-equal to gpdb_preprocess + gpdb_detect per cloud (test_gpu_preprocess_batch's contract). Each batch holds one cloud
against the CPU oracle at the bars of test_gpu_preprocess.assert_cloud_parity, and checks from its inputs that it reaches
the path it names (ball sizes, voxel counts, camera bits, the grown normals grid).
"""
import numpy as np
import pytest

from batch_param_cases import CAMS
from gpd_b200 import lib, scenes
from oracle import oracle
from preprocess_cases import Q, TIER0_CAP, ball_counts, filter_mask, grid_of, lattice
from test_gpu_preprocess import assert_cloud_parity
from test_gpu_preprocess_batch import check, context, detect_equals_singles, raw, raw_scene, samples_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = context()
    yield c
    c.close()


def run(ctx, clouds, pp, o=0, n_samples=60):
    """The batch against single calls (clouds and detection), and cloud o against the oracle."""
    got = check(ctx, clouds, pp)
    detect_equals_singles(ctx, clouds, got, pp, samples_of(got, n_samples))
    c = clouds[o]
    assert_cloud_parity(oracle.preprocess(c["xyz"], c["cam_source"], c["view_points"], pp, normals=c["normals"]), got[o])
    return got


def cams_raw(seed, k, n=20000, mark_all=True, zero_rows=0.03):
    s = scenes.synthetic_raw_scene(seed, n_points=n, cameras=CAMS[:k], mark_all_cameras=mark_all)
    if zero_rows > 0:
        s["cam_source"][np.random.default_rng(seed + 77).random(len(s["xyz"])) < zero_rows] = 0
    return raw(s["xyz"], s["cam_source"], s["view_points"])


@pytest.mark.parametrize("r", [0.005, 0.08])
def test_normals_radius(ctx, r):
    """0.005: balls of a few voxels (NaN normals below 3 neighbours); 0.08: balls beyond the first neighbour tier."""
    clouds = [raw_scene(7, n=20000, nan_fraction=0.01), raw_scene(8, n=15000, two_cameras=True)]
    got = run(ctx, clouds, lib.preprocess_params(normals_radius=r))
    cnt = ball_counts(got[0]["xyz"], np.linspace(0, len(got[0]["xyz"]) - 1, 100).astype(int), r)
    if r == 0.005:
        assert np.isnan(got[0]["normals"][:, 0]).any() and cnt.min() < 3
    else:
        assert cnt.max() > TIER0_CAP


@pytest.mark.parametrize("supplied", [False, True])
@pytest.mark.parametrize("cell", [0.001, 0.005, 0.02])
def test_voxel_size(ctx, cell, supplied):
    rng = np.random.default_rng(1)
    clouds = [raw_scene(9, n=20000), raw_scene(10, n=15000, two_cameras=True)]
    if supplied:
        for c in clouds:
            c["normals"] = rng.standard_normal((len(c["xyz"]), 3))
    pp = lib.preprocess_params(voxel_size=cell, estimate_normals=0 if supplied else 1)
    got = run(ctx, clouds, pp)
    for g, c in zip(got, clouds):
        assert 0 < len(g["xyz"]) < filter_mask(c["xyz"], list(pp.workspace)).sum()


def test_lattice_on_voxel_boundaries(ctx):
    """An exact lattice whose step is the voxel size plus copies shifted inside the voxels, beside a raw scene and the
    lattice translated by whole voxels."""
    step = 4
    base = lattice((-100 * step, -80 * step, 512), (step, 0, 0), (0, step, 0), 120, 100)
    pts = np.vstack([base, base + np.float32([Q, Q, 0]), base + np.float32([3 * Q, 3 * Q, 0])])
    pts = pts[np.random.default_rng(2).permutation(len(pts))]
    moved = pts + np.float32([8 * step * Q, -4 * step * Q, 0])
    for est in (1, 0):
        pp = lib.preprocess_params(voxel_size=step * Q, estimate_normals=est)
        rng = np.random.default_rng(3)
        clouds = [raw(pts), raw_scene(4, n=10000), raw(moved)]
        if not est:
            for c in clouds:
                c["normals"] = rng.standard_normal((len(c["xyz"]), 3))
        got = run(ctx, clouds, pp)
        assert len(got[0]["xyz"]) == len(got[2]["xyz"]) == len(base)
        assert np.array_equal(np.sort(got[0]["xyz"], 0), np.sort(base, 0))


@pytest.mark.parametrize("vox", [1, 0])
def test_camera_counts(vox):
    """K_b = 1, 3, 4 and 8 in one batch, every seeing camera marked and 3 % of the rows zeroed. Detection at 12 channels:
    15-channel shadow bitmaps of more than 3 cameras do not fit shared memory."""
    clouds = [cams_raw(5, 1), cams_raw(6, 3), cams_raw(7, 4), cams_raw(8, 8)]
    ctx = context(12)
    got = run(ctx, clouds, lib.preprocess_params(voxelize=vox), o=3)
    ctx.close()
    for g, k in zip(got, (1, 3, 4, 8)):
        cs = g["cam_source"]
        assert cs.shape[1] == k and (cs.sum(1) == 0).any() and (g["normals"][cs.sum(1) == 0] == 0).all()
        assert k == 1 or (cs.sum(1) >= 2).mean() > 0.1


def test_camera_in_the_plane(ctx):
    """The exact plane of test_viewpoint_flip_and_reverse_use_the_right_cameras, once with its cameras and once with
    them in another order (so each cloud's own view points decide), beside a raw scene."""
    pts = lattice((-50 * 4, -50 * 4, 0), (4, 0, 0), (0, 4, 0), 100, 100)
    vp = np.array([[0.75, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 0.0, 1.0]])
    sets = [(0, 2), (1, 2), (0, 1), (1,), (2,)]
    want = [1.0, -1.0, -1.0, -1.0, 1.0]
    which = np.arange(len(pts)) % len(sets)
    cam = np.zeros((len(pts), 3), np.int32)
    for w, st in enumerate(sets):
        for c in st:
            cam[which == w, c] = 1
    perm = [2, 0, 1]  # camera j of the second cloud is camera perm[j] of the first
    clouds = [raw(pts, cam, vp), raw_scene(3, n=10000), raw(pts, cam[:, perm], vp[perm])]
    pp = lib.preprocess_params(voxelize=0)
    got = run(ctx, clouds, pp)
    for w, z in enumerate(want):
        assert (got[0]["normals"][which == w, 2] == z).all(), sets[w]
    c = clouds[2]
    assert_cloud_parity(oracle.preprocess(c["xyz"], c["cam_source"], c["view_points"], pp), got[2])
    assert (got[2]["normals"][:, :2] == 0).all() and (np.abs(got[2]["normals"][:, 2]) == 1).all()


def test_degenerate_clouds(ctx):
    """1- and 2-point clouds, coincident points and a collinear lattice (NaN normals) among ordinary clouds."""
    plane = lattice((-30 * 4, -30 * 4, 512), (4, 0, 0), (0, 4, 0), 60, 60)
    line = lattice((-100 * 4, 100, 500), (4, 0, 0), (0, 0, 0), 200, 1)
    coinc = np.vstack([np.tile(np.float32([0.2, 0.2, 0.6]), (5, 1)), lattice((-40, -40, 512), (4, 0, 0), (0, 4, 0), 20, 20)])
    clouds = [raw(plane[:1]), raw_scene(4, n=10000), raw(plane[:2]), raw(coinc), raw(line), raw(plane)]
    got = run(ctx, clouds, lib.preprocess_params(voxelize=0), o=3)
    assert np.isnan(got[0]["normals"]).all() and np.isnan(got[2]["normals"]).all()
    assert np.isnan(got[3]["normals"][:5]).all() and not np.isnan(got[3]["normals"][5:]).any()
    assert np.isnan(got[4]["normals"]).all() and not np.isnan(got[5]["normals"]).any()


@pytest.mark.parametrize("vox", [1, 0])
def test_workspace_bounds(ctx, vox):
    """Coordinates on each of the six bounds, one float32 step inside and outside, and NaN / +inf / -inf per axis."""
    ws = [-0.5, 0.5, -0.25, 0.1, 0.25, 1.0]
    base = lattice((-60 * 4, -40 * 4, 600), (4, 0, 0), (0, 4, 0), 120, 80)
    inside = np.float32([0.0, 0.0, 0.6])
    extra = []
    for a in range(3):
        for side in (0, 1):
            b = np.float32(ws[2 * a + side])
            for v in (b, np.nextafter(b, np.float32(0.6 if a == 2 else 0.0)), np.nextafter(b, np.float32(9 if side else -9))):
                p = inside.copy()
                p[a] = v
                extra.append(p)
        for bad in (np.nan, np.inf, -np.inf):
            p = inside.copy()
            p[a] = bad
            extra.append(p)
    pts = np.vstack([base, np.array(extra, np.float32)])
    other = np.vstack([np.array(extra, np.float32), base[::3]])
    clouds = [raw(pts), raw_scene(5, n=10000), raw(other)]
    got = run(ctx, clouds, lib.preprocess_params(workspace=ws, voxelize=vox))
    mask = filter_mask(pts, ws)
    assert not mask[len(base):].all() and mask[len(base):].any()
    assert set(got[0]["src"]) <= set(np.nonzero(mask)[0])


def test_grown_normals_grid(ctx):
    """voxelize = 0, workspace +-10 m, far points 8 m away on each axis: the normals grid of that cloud grows to 3 cm
    cells (the others keep 2 cm). That cloud against the oracle."""
    s = raw_scene(6, n=20000)
    fin = s["xyz"][np.isfinite(s["xyz"]).all(1)]
    far = (fin.astype(np.float64).mean(0) + 8.0 * np.eye(3)).astype(np.float32)
    grown = raw(np.vstack([s["xyz"], far]), np.vstack([s["cam_source"], np.ones((3, 1), np.int32)]), s["view_points"])
    pp = lib.preprocess_params(voxelize=0, workspace=[-10, 10, -10, 10, -10, 10])
    clouds = [raw_scene(4, n=10000), grown, raw_scene(8, n=10000, two_cameras=True)]
    got = run(ctx, clouds, pp, o=1)
    assert [grid_of(g["xyz"])[4] for g in got] == [0, 1, 0]
    assert np.isnan(got[1]["normals"][-3:]).all()  # the isolated far points
