"""The restatements of include/gpd_b200_organized.h on constructed cases: the numpy restatement
(tests/organized_reference.py) and the C++ one over the header's helpers compiled for the host (tests/organized_oracle.cpp)
agree bit for bit (normals with their NaN positions, distance maps); the depth-change test at exactly its threshold and
one ulp either side; the wrap reads of the distance passes; the 40 x 40 / 41 x 41 edge of the border rule; and, away from
edges, the normals of a float64 PCA of the same window within a bound derived below."""
import numpy as np
import pytest

import depth_reference as dr
import organized_reference as orf

F = np.float32


def plane(H, W, tilt=(0.1, -0.05), z0=0.8, f=300.0):
    """A tilted plane seen by a pinhole camera: camera-frame points [H, W, 3]."""
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    x, y = (u - W / 2) / f, (v - H / 2) / f
    z = z0 / (1.0 - tilt[0] * x - tilt[1] * y)
    return np.stack([x * z, y * z, z], -1).astype(F)


def both(xyz, vp=(0.0, 0.0, 0.0)):
    n1, d1 = orf.normals(xyz, vp)
    n2, d2 = orf.cpp_normals(xyz, vp)
    assert np.array_equal(d1, d2)
    assert np.array_equal(n1, n2, equal_nan=True)
    return n1, d1


def test_nan_holes_and_a_depth_step():
    xyz = plane(70, 90)
    xyz[30:34, 40:47] = np.nan  # a hole
    xyz[:, 60:, 2] += F(0.2)  # a silhouette
    n, d = both(xyz)
    assert np.all(d[31, 40:47] == 0) and np.all(d[:-1, 59:61] == 0)
    assert np.all(np.isnan(n[30:34, 40:47]))
    fin = np.isfinite(n[..., 0])
    assert fin.sum() > 500 and not fin[:, 58:62].any()


def _step_at(a, t, k):
    """b with fabsf(a - b) = t moved by k ulps (b > a)."""
    b = F(a + t)
    while F(b - a) > t:
        b = np.nextafter(b, F(0))
    while F(b - a) < t:
        b = np.nextafter(b, F(np.inf))
    for _ in range(abs(k)):
        b = np.nextafter(b, F(np.inf) if k > 0 else F(0))
    return b


@pytest.mark.parametrize("a", [0.0, 1.0])
@pytest.mark.parametrize("k,breaks", [(-1, False), (0, False), (1, True)])
def test_depth_change_at_the_threshold(a, k, breaks):
    """a = 0: the step b = t is exact, so k = 0 tests fabsf(z - z') == t itself (no change); a = 1: the nearest steps."""
    H, W = 45, 45
    xyz = np.zeros((H, W, 3), F)
    a = F(a)
    t = (F(0.02) * (np.abs(a) + F(1.0))) * F(2.0)
    b = _step_at(a, t, k)
    if k == 0 and F(b - a) != t:
        assert a != 0  # a = 0 always has the exact step
        b = np.nextafter(b, F(0)) if F(b - a) > t else b  # the nearest step below t: no change either
    xyz[..., 2] = a
    xyz[:, 30:, 2] = b
    xyz[..., 0] = np.arange(W, dtype=F)[None, :] * F(1e-3)
    xyz[..., 1] = np.arange(H, dtype=F)[:, None] * F(1e-3)
    assert bool(orf.pair_breaks(a, b)) == breaks
    n, d = both(xyz)
    assert (orf.change_map(xyz[..., 2])[5, 29] == 0) == breaks


def test_the_wrap_reads_change_the_map():
    H, W = 50, 60
    xyz = plane(H, W)
    xyz[10, 0] = np.nan  # pass 1: (10, W-1) reads element 0 of its own row as its upper right
    xyz[30, W - 1] = np.nan  # pass 2: (30, 0) reads the last element of its own row as its lower left
    n, d = both(xyz)
    assert d[10, W - 1] == F(0.0) + F(1.4)
    assert d[30, 0] == F(0.0) + F(1.4)


@pytest.mark.parametrize("size,any_normal", [(40, False), (41, True)])
def test_border_rule_at_40_and_41(size, any_normal):
    n, _ = both(plane(size, size))
    assert np.isfinite(n[..., 0]).any() == any_normal
    if any_normal:
        assert np.isfinite(n[20, 20]).all() and np.isnan(n[19, 20]).all() and np.isnan(n[20, 21]).all()


def test_full_size_render_numpy_equals_cpp():
    view = dr.render_views([5], [1], 0, n_points=200000, width=640, height=480, f=520.0)[0][0]
    xyz = orf.camera_cloud(view[0], view[1], 0)
    # the numpy restatement's per-pixel loop is slow: compare the maps everywhere and the normals on a band of rows
    n2, d2 = orf.cpp_normals(xyz)
    assert np.array_equal(orf.distance_map(xyz[..., 2]), d2)
    band = xyz[200:260]
    n1, _ = orf.normals(band)
    nb, _ = orf.cpp_normals(band)
    assert np.array_equal(n1, nb, equal_nan=True)
    assert np.isfinite(n2[..., 0]).sum() > 1000


def test_normals_match_a_float64_pca_away_from_edges():
    """On a smooth plane with no depth change the window is the full 20 x 20 one. The float32 covariance sums of about 400
    points of size ~1 lose about 400 * 2^-24 * |z|^2 relative to each entry; after the centring (a cancellation of the
    sums against centre^2 / n) the absolute error of an entry is ~ 1e-4 * z^2 against an eigen-gap of the window's spread
    in x and y, ~ (10 px / f)^2 * z^2 * n. The tilt of the eigenvector is error / gap < 1e-2 rad here; we assert 2e-2."""
    xyz = plane(80, 80, tilt=(0.3, 0.2), f=200.0)
    n, d = both(xyz)
    for r in range(25, 55, 6):
        for c in range(25, 55, 6):
            win = xyz[r - 10:r + 10, c - 10:c + 10].reshape(-1, 3).astype(np.float64)
            w, V = np.linalg.eigh(np.cov(win.T))
            ref = V[:, 0] * np.sign(np.dot(V[:, 0], -xyz[r, c]))
            assert np.arccos(min(1.0, abs(float(np.dot(ref, n[r, c].astype(np.float64)))))) < 2e-2


def test_rotate_is_one_rounding_per_row():
    R = np.array([[0.6, -0.8, 0.0], [0.8, 0.6, 0.0], [0.0, 0.0, 1.0000001]])
    nc = np.array([[0.1, 0.2, 0.97], [np.nan, 0.0, 1.0]], F)
    out = np.zeros_like(nc)
    orf.cpp().org_oracle_rotate(2, orf._p(np.ascontiguousarray(R.ravel())), orf._p(nc), orf._p(out))
    assert np.array_equal(out, orf.rotate(R, nc), equal_nan=True)
