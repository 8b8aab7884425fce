"""The support-plane specification (include/gpd_b200_plane.h) on the CPU: the header's draw, sample and model functions
compiled for the host against the numpy restatement (tests/plane_reference.py), the restatement's refit against a float64
PCA, and the loop rules at their edges: empty and tiny clouds, collinear and coplanar clouds, points at the threshold,
and stopping points of rule 4 computed in advance."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import plane_reference as pr
from gpd_b200 import scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32

_SHIM = r"""
#include "gpd_b200_plane.h"
extern "C" {
void draw_sample(uint64_t key, uint32_t h, uint32_t a, uint32_t n, uint32_t *c4, uint32_t *idx3) {
  const gpdb_u32x4 c = gpdb_plane_draw(key, h, a);
  c4[0] = c.x, c4[1] = c.y, c4[2] = c.z, c4[3] = c.w;
  gpdb_plane_sample(c, n, idx3);
}
int model(const float *p9, float *coef) { return gpdb_plane_model(p9, p9 + 3, p9 + 6, coef) ? 1 : 0; }
float dist(const float *coef, float x, float y, float z) { return gpdb_plane_dist(coef, x, y, z); }
}
"""


@pytest.fixture(scope="module")
def header(tmp_path_factory):
    """The header's GPDB_HD functions built for the host (no FMA contraction, as the kernels are built)."""
    d = tmp_path_factory.mktemp("plane_header")
    src, so = d / "shim.cpp", d / "shim.so"
    src.write_text(_SHIM)
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                           "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.draw_sample.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.model.argtypes = [C.c_void_p, C.c_void_p]
    L.dist.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float]
    L.dist.restype = C.c_float
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_header_draws_and_samples_match_the_shuffle(header):
    """gpdb_plane_draw / gpdb_plane_sample against philox + a real partial Fisher-Yates shuffle, including the small n
    where the swaps collide (n = 3, 4, 5) and keys above 2^32."""
    rng = np.random.default_rng(1)
    c4, idx = np.zeros(4, np.uint32), np.zeros(3, np.uint32)
    for n in [3, 4, 5, 7, 1000, 2**31 - 1]:
        for key in [0, 7, 2**32 + 3, 2**64 - 1]:
            for h, a in [(0, 0), (1, 0), (0, 999), (1024, 5)] + [tuple(rng.integers(0, 1000, 2)) for _ in range(8)]:
                header.draw_sample(key, int(h), int(a), n, _p(c4), _p(idx))
                want = pr.draws(key, int(h), [int(a)])[0]
                assert c4.tolist() == want.tolist()
                fy = pr.fisher_yates3(want, n)
                assert idx.tolist() == fy and len(set(fy)) == 3 and max(fy) < n


def test_header_model_and_distance_match_numpy(header):
    """Rule 2 and 3, bit for bit: random triples, exact duplicates (zero normal), collinear triples (bad) and NaN
    ratios (good)."""
    rng = np.random.default_rng(2)
    coef = np.zeros(4, F)
    triples = [rng.normal(0, 1, (3, 3)).astype(F) for _ in range(200)]
    triples += [np.array([[0, 0, 0], [1, 2, 3], [2, 4, 6]], F),          # collinear: ratios equal -> bad
                np.array([[1, 1, 1], [1, 1, 1], [2, 3, 4]], F),          # p1 == p0: 0 / x ratios equal -> bad
                np.array([[1, 1, 1], [2, 3, 4], [1, 1, 1]], F),          # p2 == p0: x / 0 -> inf ratios equal -> bad
                np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], F),          # NaN ratios -> good, the z = 0 plane
                np.array([[0.1, 0.2, 0.9], [0.1, 0.2, 0.9], [0.1, 0.2, 0.9]], F)]  # all equal: NaN ratios -> good, n = 0
    for t in triples:
        good = header.model(_p(np.ascontiguousarray(t)), _p(coef))
        g2, c2 = pr.model(t[0], t[1], t[2])
        assert bool(good) == g2
        if g2:
            assert coef.tobytes() == c2.tobytes()
            for q in rng.normal(0, 1, (5, 3)).astype(F):
                assert np.float32(header.dist(_p(coef), *map(float, q))).tobytes() == pr.dist(c2, q[None])[0].tobytes()
    assert pr.model(*triples[-1])[1].tolist() == [0, 0, 0, 0]


def _angle_to_z(plane):
    n = plane[:3].astype(np.float64)
    return np.arccos(min(1.0, abs(n[2]) / np.linalg.norm(n)))


def _pca_bound(pts):
    """The bound of DESIGN.md 4b on the angle between the float32 single-pass refit and a float64 PCA of the same points:
    16 (3 sqrt(n) 2^-24 |p|^2 + 2^-23 lambda_max) / gap + 1e-6."""
    p = pts.astype(np.float64)
    w, v = np.linalg.eigh(np.cov(p.T, bias=True))
    bound = 16 * (3 * np.sqrt(len(p)) * 2.0 ** -24 * np.abs(p).max() ** 2 + 2.0 ** -23 * w[2]) / max(w[1] - w[0], 1e-300)
    return v[:, 0], bound + 1e-6


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_table_scene(seed):
    """The table of synthetic_table_scene: the refined normal within 1e-2 rad of +-z and within the float32 bound of a
    float64 PCA of the same inliers; every point within 5 mm of the table height is a final inlier; the mask is the
    complement of the final inliers."""
    xyz = scenes.synthetic_table_scene(seed, n_points=20000)["xyz"]
    r = pr.segment(xyz, key=seed)
    assert r["refit"] and r["best"] >= 0 and 1 <= r["n_hypotheses"] <= 51
    assert _angle_to_z(r["plane"]) < 1e-2
    v, bound = _pca_bound(r["best_inliers"])
    n = r["plane"][:3].astype(np.float64)
    ang = np.arccos(min(1.0, abs(float(v @ n)) / np.linalg.norm(n)))
    assert ang <= bound, (ang, bound)
    table_z = np.median(xyz[:, 2][xyz[:, 2] > 0.89])
    table = np.abs(xyz[:, 2].astype(np.float64) - table_z) < 0.005
    fin = r["eligible"] == 0
    assert table.sum() > 0.5 * len(xyz) and fin[table].all()
    assert r["n_inliers"] == fin.sum() and 0 < fin.sum() < len(xyz)


def test_tilted_plane_with_clutter():
    """A plane tilted by 30 degrees with 20 % clutter above it: found, and the clutter off it is eligible."""
    rng = np.random.default_rng(3)
    u, v = rng.uniform(-0.3, 0.3, (2, 4000))
    nrm = np.array([np.sin(np.pi / 6), 0.0, np.cos(np.pi / 6)])
    e1, e2 = np.array([np.cos(np.pi / 6), 0.0, -np.sin(np.pi / 6)]), np.array([0.0, 1.0, 0.0])
    plane_pts = 0.8 * nrm + u[:, None] * e1 + v[:, None] * e2 + rng.normal(0, 0.001, (4000, 1)) * nrm
    a, b = rng.uniform(-0.3, 0.3, (2, 1000))
    clutter = 0.8 * nrm + a[:, None] * e1 + b[:, None] * e2 - rng.uniform(0.03, 0.2, (1000, 1)) * nrm
    xyz = np.vstack([plane_pts, clutter]).astype(F)
    r = pr.segment(xyz, key=11)
    n = r["plane"][:3].astype(np.float64)
    assert abs(abs(n @ nrm) - 1) < 1e-4
    assert (r["eligible"][:4000] == 0).all() and (r["eligible"][4000:] == 1).all()
    v0, bound = _pca_bound(r["best_inliers"])
    assert np.arccos(min(1.0, abs(float(v0 @ n)) / np.linalg.norm(n))) <= bound


@pytest.mark.parametrize("n", [0, 1, 2])
def test_fewer_than_three_points_fail(n):
    r = pr.segment(np.zeros((n, 3), F) + np.arange(n)[:, None].astype(F))
    assert r["best"] == -1 and r["n_hypotheses"] == 0 and r["n_inliers"] == 0
    assert np.isnan(r["plane"]).all() and (r["eligible"] == 1).all() and len(r["eligible"]) == n


def test_three_points_keep_the_hypothesis():
    """N = 3: one plane through all three, 3 inliers (not more than 3): no refit, the hypothesis' coefficients stay;
    no point is off the plane, so every point stays eligible."""
    xyz = np.array([[0, 0, 1], [0.1, 0, 1], [0, 0.1, 1.01]], F)
    r = pr.segment(xyz)
    assert not r["refit"] and r["n_hypotheses"] == 1 and r["n_inliers"] == 3
    assert r["plane"].tobytes() == r["hyp_plane"].tobytes() and (r["eligible"] == 1).all()


def test_collinear_lattice_fails():
    """Every triple of a collinear lattice is bad: hypothesis 0 finds no sample in 1000 attempts, the fit fails."""
    xyz = (np.arange(50)[:, None] * np.array([[0.25, 0.5, 1.0]])).astype(F)
    r = pr.segment(xyz)
    assert r["hyps"] == [None] and r["n_hypotheses"] == 0 and np.isnan(r["plane"]).all() and (r["eligible"] == 1).all()


def test_coplanar_cloud_stops_after_one_hypothesis():
    """All points on z = 0.5: w = 1, q clamps to DBL_EPSILON <= 1 - p, so rule 4 stops after hypothesis 0; no point is
    off the plane and the fallback leaves every point eligible."""
    g = np.stack(np.meshgrid(np.arange(20) * 0.01, np.arange(20) * 0.01), -1).reshape(-1, 2)
    xyz = np.column_stack([g, np.full(len(g), 0.5)]).astype(F)
    r = pr.segment(xyz)
    assert r["n_hypotheses"] == 1 and r["n_inliers"] == len(xyz) and (r["eligible"] == 1).all()
    assert abs(abs(float(r["plane"][2])) - 1) < 1e-6


def test_threshold_is_strict():
    """Two probes at float32 distance exactly float32(threshold) from a flat grid (one above, one below, so that the
    refit stays z = 0 exactly): inliers iff (double)float32(threshold) < threshold, strictly. 0.25 is exact in float32
    (not inliers); float32(0.01) lies below 0.01 (inliers)."""
    base = np.stack(np.meshgrid(np.arange(10) * 0.05, np.arange(10) * 0.05), -1).reshape(-1, 2)
    flat = np.column_stack([base, np.zeros(len(base))]).astype(F)
    for thr, want in [(0.25, [1, 1]), (0.01, [0, 0])]:
        t32 = F(thr)
        xyz = np.vstack([flat, np.array([[0.2, 0.2, t32], [0.2, 0.2, -t32], [0.1, 0.1, 0.5]], F)])
        r = pr.segment(xyz, distance_threshold=thr)
        assert r["plane"][:2].tolist() == [0, 0] and abs(float(r["plane"][2])) == 1 and float(r["plane"][3]) == 0
        assert r["dist"][-3:-1].tolist() == [t32, t32]
        assert r["eligible"][-3:].tolist() == want + [1]


def _sparse_case():
    """200 points spread through a 1 m cube: with a 1 mm threshold each hypothesis holds a handful of points, w is
    about 0.02 and q^(h+1) stays above 0.01 for every h <= 1024, so only max_iterations stops the loop."""
    return np.random.default_rng(5).uniform(0, 1, (200, 3)).astype(F)


def _two_planes():
    """Two parallel 8 x 8 grids 1 m apart: hypotheses inside a grid count 64, triples across the grids a few."""
    g = np.stack(np.meshgrid(np.arange(8) * 0.1, np.arange(8) * 0.1), -1).reshape(-1, 2)
    return np.vstack([np.column_stack([g, np.zeros(64)]), np.column_stack([g, np.ones(64)])]).astype(F)


def _pcl_stop(counts, n, max_iterations, probability):
    """PCL's own loop (iterations < log(1 - p) / log(q), k = 1 before the first model) over the hypotheses' counts:
    the number of hypotheses it evaluates."""
    k, best, it = 1.0, -1, 0
    for c in counts:
        if not it < k:
            break
        if c > best:
            best = c
            q = min(max(1.0 - (c / n) ** 3, pr.DBL_EPS), 1.0 - pr.DBL_EPS)
            k = np.log(1.0 - probability) / np.log(q)
        it += 1
        if it > max_iterations:
            break
    return it


# (cloud, max_iterations, probability, threshold, hypotheses evaluated or None: PCL's log form over the counts)
STOPS = [("sparse", 1, 0.99, 0.001, 2),          # max_iterations stops at h + 1 = 2 > 1
         ("sparse", 1024, 0.99, 0.001, 1025),    # only max_iterations stops it
         ("planes", 50, 0.99, 0.01, None),
         ("planes", 50, 0.5, 0.01, None),
         ("planes", 200, 0.999, 0.01, None),
         ("planes", 50, 0.99, 0.001, None)]


@pytest.mark.parametrize("cloud,max_iterations,probability,thr,want", STOPS)
def test_rule4_stops_where_computed(cloud, max_iterations, probability, thr, want):
    xyz = _two_planes() if cloud == "planes" else _sparse_case()
    r = pr.segment(xyz, key=4, max_iterations=max_iterations, probability=probability, distance_threshold=thr)
    if want is None:
        # the counts of every hypothesis the loop could reach, then PCL's stop over them
        counts = [int(np.count_nonzero(pr.inliers(pr.hypothesis(xyz, 4, h)[2], xyz, thr)))
                  for h in range(max_iterations + 1)]
        assert counts[:r["n_hypotheses"]] == r["counts"]
        want = _pcl_stop(counts, len(xyz), max_iterations, probability)
        assert 1 < want <= max_iterations
    assert r["n_hypotheses"] == want == len(r["counts"])
    assert r["counts"][r["best"]] == max(r["counts"]) and r["counts"].index(max(r["counts"])) == r["best"]


def test_subsample_points_rule():
    """The per-point mask draw equals the depth rule on the eligible points; no mask is every point's draw."""
    from depth_reference import subsample
    off = np.array([0, 10, 10, 40])
    mask = (np.arange(40) % 3 != 0).astype(np.uint8)
    got = pr.subsample_points(off, mask, 5, 9)
    assert got[1].size == 0 and all(len(g) == 5 for g in (got[0], got[2]))
    assert all((mask[off[b] + g] == 1).all() for b, g in enumerate(got))
    nm = pr.subsample_points(off, None, 5, 9)
    assert nm[2].tolist() == subsample(30, 5, 9, 2).tolist()
