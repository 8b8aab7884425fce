"""Inputs and independent references for the preprocessing tests off the default parameters (test_gpu_preprocess_params.py
on the device, test_preprocess_cases.py on the CPU).

The references here are plain numpy, written apart from the oracle: the NaN / workspace mask, the voxel set and its
order (numpy.unique of float32 floor((p - min) / cell)), and a float64 PCA of the r-ball of a point. The lattices use
coordinates that are multiples of 2^-10, so that every coordinate, every difference and every squared distance between
two of their points is exact in float32.
"""
import numpy as np

from gpd_b200 import scenes
from oracle import oracle

# cameras in front of the table (z = 0.9), looking along +z (test_gpu_geometry_params.py uses the same set)
CAMS = [[0.0, 0.0, 0.0], [0.6, 0.0, 0.0], [-0.5, 0.1, 0.05], [0.0, 0.5, 0.0], [0.1, -0.5, 0.1], [0.45, 0.45, 0.0],
        [-0.4, -0.4, 0.0], [0.3, -0.2, -0.2]]
GRID_CELL = 0.02      # first cell of the neighbour grid (geometry.cu k_batch_desc); grid_of grows it for large clouds
TIER0_CAP = 1024      # neighbours per point held by k_normals' first tier
TIER1_CAP = 8192      # ... by its second tier; beyond it gpdb_preprocess reports GPDB_ERR_CAPACITY
TABLE_WS = [-0.6, 0.6, -0.5, 0.5, 0.2, 1.0]
Q = 2.0 ** -10        # lattice quantum


def raw_table(seed=7, n_cams=1, mark_all=False, zero_rows=0.0, nan_fraction=0.0):
    """The ~60 k-point raw table scene (about 110 k raw points) with the first n_cams cameras of CAMS; a fraction
    `zero_rows` of the cam_source rows is zeroed (points no camera sees)."""
    s = scenes.synthetic_raw_scene(seed, n_points=60000, cameras=CAMS[:n_cams], mark_all_cameras=mark_all,
                                   nan_fraction=nan_fraction)
    if zero_rows > 0:
        rng = np.random.default_rng(seed + 77)
        s["cam_source"][rng.random(len(s["xyz"])) < zero_rows] = 0
    return s


def lattice(origin, u, v, nu, nv):
    """Points origin + i u + j v (i < nu, j < nv); origin, u, v in units of Q (integers): exact float32 coordinates."""
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    k = np.asarray(origin)[None] + i.reshape(-1, 1) * np.asarray(u)[None] + j.reshape(-1, 1) * np.asarray(v)[None]
    pts = (k * Q).astype(np.float32)
    assert is_exact(pts, k)
    return pts


def is_exact(pts, k):
    return np.array_equal(pts.astype(np.float64), np.asarray(k, np.float64) * Q)


def clusters(sizes, r, seed=3):
    """Isolated flat clusters (side 0.3 r in x, y and 0.03 r in z: diameter < 0.43 r), one per size, 4 r apart on x:
    every point of a cluster lies inside the r-ball of every other point of it and of no other cluster. Flat, so that
    the normal is well conditioned (eigen-gap ~ (0.3 r)^2 / 12)."""
    rng = np.random.default_rng(seed)
    out = []
    for c, n in enumerate(sizes):
        p = rng.uniform(-0.5, 0.5, (n, 3)) * [0.3 * r, 0.3 * r, 0.03 * r] + [-0.4 + 4 * r * c, 0.0, 0.5]
        out.append(p.astype(np.float32))
    return np.vstack(out)


def filter_mask(xyz, ws):
    """removeNans + filterWorkspace: finite, and strictly inside the float64 bounds."""
    x = np.asarray(xyz, np.float32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        m = np.isfinite(x).all(1)
        for a in range(3):
            m &= (x[:, a] > ws[2 * a]) & (x[:, a] < ws[2 * a + 1])
    return m


def voxel_reference(xyz, ws, cell):
    """The voxel set of the filtered cloud: (src, xyz) in the order of descending index of each voxel's first point,
    with float32 floor((p - min) / cell) and the corner min + cell * v."""
    keep = np.nonzero(filter_mask(xyz, ws))[0]
    p = np.asarray(xyz, np.float32)[keep]
    c = np.float32(cell)
    mn = p.min(0)
    vox = np.floor((p - mn) / c).astype(np.int64)
    uniq, first = np.unique(vox, axis=0, return_index=True)
    order = np.argsort(-first)
    return keep[first[order]], (mn + c * uniq[order].astype(np.float32)).astype(np.float32)


def grid_of(xyz):
    """(lo, dim, cell, cells, growth steps) of the neighbour grid of a cloud, in the float32 steps of k_batch_desc:
    2 cm cells from the cloud's minimum, grown by 1.5x while the grid would need more than 48e6 cells."""
    p = np.asarray(xyz, np.float32)
    lo, hi = p.min(0), p.max(0)
    cell, steps = np.float32(GRID_CELL), 0
    while True:
        dim = np.floor((hi - lo) / cell).astype(np.int64) + 2
        cells = float(np.prod(dim.astype(np.float64)))
        if cells <= 48e6:
            return lo, dim, cell, cells, steps
        cell, steps = np.float32(cell * np.float32(1.5)), steps + 1


def grid_rows(xyz, r):
    """Grid rows (y, z cell pairs) the ball scan of k_normals visits for each point: the cells of grid_of from the
    cloud's minimum, the ball widened as preprocess.cu's pre_normals does."""
    p = np.asarray(xyz, np.float32)
    lo, dim, cell, _, _ = grid_of(p)
    rf = np.float32(r) * np.float32(1.0001) + np.float32(1e-6)
    inv = np.float32(1.0) / cell
    rows = np.ones(len(p), np.int64)
    for a in (1, 2):
        c0 = np.clip(np.floor((p[:, a] - rf - lo[a]) * inv).astype(np.int64), 0, dim[a] - 1)
        c1 = np.clip(np.floor((p[:, a] + rf - lo[a]) * inv).astype(np.int64), 0, dim[a] - 1)
        rows *= c1 - c0 + 1
    return rows


def ball_counts(cloud_xyz, idx, r):
    """Neighbour counts (self included) of the points idx by the oracle's float32 radius search."""
    oc = oracle.OracleCloud(cloud_xyz, np.zeros((len(cloud_xyz), 3)))
    return np.array([len(oc.radius_search(cloud_xyz[i], r, cap=1 << 16)[0]) for i in idx])


def ball_float32(xyz, q, r):
    """Indices of the r-ball of q with FLANN's float32 predicate (L2_Simple: dx^2 + dy^2 + dz^2 summed in that order,
    against float32(r^2)), in numpy."""
    d = q - xyz
    dist = d[:, 0] * d[:, 0]
    dist = dist + d[:, 1] * d[:, 1]
    dist = dist + d[:, 2] * d[:, 2]
    return np.nonzero(dist < np.float32(r * r))[0]


def pca_check(cloud, r, idx):
    """Float64 PCA of the r-ball of each point idx (selected in numpy with the float32 predicate, ball_float32) against
    the estimated normal, sign-free. The bound on the angle is derived, not fitted: the float32 single-pass covariance
    carries an error of about sqrt(n) 2^-24 |p|^2 per entry (n neighbours, |p| the largest coordinate of the ball) and
    pcl::eigen33's float32 closed form about 2^-23 lambda_max; both tilt the eigenvector by (error) / (eigen-gap). With
    a factor 16 over that estimate: angle <= 16 (3 sqrt(n) 2^-24 |p|^2 + 2^-23 lambda_max) / gap + 1e-6.
    Returns (points checked, worst angle / bound); NaN normals (< 3 neighbours) and zero normals (no camera) are
    checked for exactly that."""
    xyz, nrm = cloud["xyz"], cloud["normals"]
    xyz = np.asarray(xyz, np.float32)
    seen = cloud["cam_source"].any(1)
    checked, worst = 0, 0.0
    for i in idx:
        nb = ball_float32(xyz, xyz[i], r)
        if not seen[i]:
            assert (nrm[i] == 0).all()
            continue
        if len(nb) < 3:
            assert np.isnan(nrm[i]).all()
            continue
        p = xyz[nb].astype(np.float64)
        w, v = np.linalg.eigh(np.cov(p.T, bias=True))
        gap = w[1] - w[0]
        bound = 16 * (3 * np.sqrt(len(nb)) * 2.0 ** -24 * np.abs(p).max() ** 2 + 2.0 ** -23 * w[2]) / max(gap, 1e-300) + 1e-6
        c = min(abs(float(v[:, 0] @ nrm[i])) / np.linalg.norm(nrm[i]), 1.0)
        ang = np.sqrt(max(0.0, 1 - c * c))
        worst = max(worst, ang / bound)
        checked += 1
    return checked, worst
