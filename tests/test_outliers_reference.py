"""The restatement of include/gpd_b200_outliers.h (tests/outliers_reference.py) on constructed cases: the header's helpers
compiled for the host equal it bit for bit; the mean distances do not depend on how neighbour ties are broken; a point
exactly at the threshold stays; clouds of at most mean_k points and of mean_k + 1; a cloud whose mean distances are all
equal; and the decisions of an independent float64 formulation everywhere except close to the threshold."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import outliers_reference as orf
import refine_reference as rr
from gpd_b200 import scenes
from test_refine_reference import lattice, with_duplicates

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_HELPERS = r"""
#include <stdint.h>
#include "gpd_b200_outliers.h"
// the header's helpers over given neighbour lists (n x (mean_k + 1), cloud-local), one cloud
extern "C" void outl_mean(int n, int mean_k, const float *xyz, const int32_t *nbr, float *d) {
  for (int i = 0; i < n; i++) {
    double s = 0.0;
    for (int r = 1; r <= mean_k; r++) s = gpdb_outlier_dist_add(s, gpdb_refine_l2(xyz + 3 * i, xyz + 3 * nbr[i * (mean_k + 1) + r]));
    d[i] = gpdb_outlier_mean(s, mean_k);
  }
}
extern "C" void outl_stats(int n, int mean_k, double mul, const float *d, double *out, uint8_t *keep) {
  double s = 0.0, sq = 0.0;
  for (int i = 0; i < n; i++) gpdb_outlier_stats_add(&s, &sq, d[i]);
  gpdb_outlier_stats(s, sq, n, mean_k, mul, out);
  for (int i = 0; i < n; i++) keep[i] = !gpdb_outlier_removed(d[i], out[2]);
}
"""


@functools.lru_cache(None)
def helpers():
    d = tempfile.mkdtemp(prefix="outliers_helpers_")
    src, so = os.path.join(d, "h.cpp"), os.path.join(d, "libh.so")
    with open(src, "w") as f:
        f.write(_HELPERS)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), "-o", so, src])
    L = C.CDLL(so)
    L.outl_mean.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.outl_stats.argtypes = [C.c_int, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_remove(xyz, mean_k, mul):
    """(kept bools, stats, d) from the header's helpers compiled for the host, over the restatement's lists."""
    xyz = np.ascontiguousarray(xyz, F)
    n = len(xyz)
    d = np.full(n, np.nan, F)
    if n > mean_k:  # rule 5: no lists of mean_k + 1 entries, no mean distances
        nbr = np.ascontiguousarray(rr.knn(xyz, mean_k + 1), np.int32)
        helpers().outl_mean(n, mean_k, _p(xyz), _p(nbr), _p(d))
    st, kp = np.zeros(3), np.zeros(n, np.uint8)
    helpers().outl_stats(n, mean_k, float(mul), _p(d), _p(st), _p(kp))
    return kp.astype(bool), st, d


@functools.lru_cache(None)
def noisy_table(seed=1, n=4000, n_fly=60):
    """A part of a synthetic table scene with flying pixels: points pulled off the surface along their view ray."""
    rng = np.random.default_rng(seed)
    xyz = scenes.synthetic_table_scene(seed, n_points=20000)["xyz"][:n].astype(np.float64)
    i = rng.choice(n, n_fly, replace=False)
    xyz[i] *= rng.uniform(0.8, 1.2, (n_fly, 1))
    return xyz.astype(F)


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("mean_k,mul", [(1, 1.0), (2, 0.0), (10, 1.0), (50, 1.0), (50, -0.5), (127, 2.0)])
def test_host_helpers_equal_the_restatement(mean_k, mul):
    for xyz in (noisy_table(), with_duplicates(4), lattice(7)):
        kept, st, d = orf.remove(xyz, mean_k, mul)
        hk, hst, hd = host_remove(xyz, mean_k, mul)
        assert np.array_equal(d.view(np.uint32), hd.view(np.uint32))
        assert np.array_equal(bits(st), bits(hst))
        assert np.array_equal(kept, hk)


def test_mean_distances_do_not_depend_on_the_tie_break():
    """Shuffling the entries of equal distance in every list, and renumbering the points, leaves every d_i as it was."""
    rng = np.random.default_rng(2)
    for xyz, k in ((lattice(6), 6), (lattice(6), 18), (with_duplicates(5), 10), (np.repeat(lattice(3), 3, axis=0), 8)):
        d = orf.mean_distances(xyz, k)
        nbr = rr.knn(xyz, k + 1)
        l2 = np.stack([rr.l2(xyz[i:i + 1], xyz[nbr[i]])[0] for i in range(len(xyz))])
        shuffled = nbr.copy()
        n_ties = 0
        for i in range(len(xyz)):
            for v in np.unique(l2[i]):
                at = np.nonzero(l2[i] == v)[0]
                if len(at) > 1:
                    shuffled[i, at] = nbr[i, rng.permutation(at)]
                    n_ties += 1
        assert n_ties > 0 and not np.array_equal(shuffled, nbr)
        assert np.array_equal(orf.mean_distances(xyz, k, shuffled).view(np.uint32), d.view(np.uint32))
        perm = rng.permutation(len(xyz))
        assert np.array_equal(orf.mean_distances(xyz[perm], k).view(np.uint32), d[perm].view(np.uint32))


def pairs(seps, gap=10.0):
    """Far-apart pairs of points, pair j from (0, y_j, z_j) to (seps[j], y_j, z_j): its distance is float32(seps[j])."""
    return np.array([[o, gap * (j % 32), gap * (j // 32)] for j, s in enumerate(seps) for o in (0.0, s)], F)


def test_a_point_at_the_threshold_stays():
    xyz = pairs([0.25, 0.5, 0.75])
    kept, st, d = orf.remove(xyz, 1, 0.0)
    assert list(d) == [0.25, 0.25, 0.5, 0.5, 0.75, 0.75] and st[0] == st[2] == 0.5
    assert list(kept) == [True, True, True, True, False, False]
    assert np.array_equal(host_remove(xyz, 1, 0.0)[0], kept)


def test_small_clouds():
    rng = np.random.default_rng(3)
    for n, k in ((0, 5), (1, 1), (5, 5), (4, 50), (50, 50)):
        kept, st, d = orf.remove(rng.uniform(0, 1, (n, 3)), k, 1.0)
        assert kept.all() and len(kept) == n and np.isnan(st).all() and d is None
        if n:
            hk, hst, _ = host_remove(rng.uniform(0, 1, (n, 3)), k, 1.0)
            assert hk.all() and np.isnan(hst).all()
    xyz = np.concatenate([rng.uniform(0, 0.01, (10, 3)), [[1, 1, 1]]]).astype(F)  # N = mean_k + 1: statistics exist
    kept, st, d = orf.remove(xyz, 10, 1.0)
    assert np.isfinite(st).all() and not kept[-1] and kept[:-1].all()
    hk, hst, _ = host_remove(xyz, 10, 1.0)
    assert np.array_equal(hk, kept) and np.array_equal(bits(hst), bits(st))


def test_equal_mean_distances():
    """Every d_i equal: mean == d_i, and the variance is a rounding residue of the float32 squares. It is positive for
    0.1 (with stddev_mul = -1 every point goes), negative for 0.3 (a NaN threshold: every point stays whatever
    stddev_mul) and exactly 0 for 0.25; the helpers reproduce each bit for bit."""
    for sep, n, residue in ((0.1, 1000, "positive"), (0.3, 777, "negative"), (0.25, 100, "zero")):
        xyz = pairs([sep] * n)
        for mul in (1.0, -1.0):
            kept, st, d = orf.remove(xyz, 1, mul)
            assert len(np.unique(d)) == 1 and st[0] == float(d[0])
            if residue == "positive":
                assert 0 < st[1] < 1e-3 * st[0] and kept.all() == (mul > 0) and kept.any() == (mul > 0)
            elif residue == "negative":
                assert np.isnan(st[1]) and np.isnan(st[2]) and kept.all()
            else:
                assert st[1] == 0 and st[2] == st[0] and kept.all()
            hk, hst, _ = host_remove(xyz, 1, mul)
            assert np.array_equal(hk, kept) and np.array_equal(bits(hst), bits(st))


@pytest.mark.parametrize("mean_k,mul", [(10, 1.0), (50, 1.0), (50, 0.0), (20, 2.0)])
def test_decisions_agree_with_float64_away_from_the_threshold(mean_k, mul):
    """cKDTree distances and np.std(ddof=1) in float64 decide every point the same way except within 1e-5 of the mean
    distance around the threshold, more than the float32 roundings of l2, sqrtf and d_i can move a mean distance."""
    from scipy.spatial import cKDTree
    xyz = noisy_table()
    kept, st, d = orf.remove(xyz, mean_k, mul)
    x64 = xyz.astype(np.float64)
    dist, _ = cKDTree(x64).query(x64, k=mean_k + 1)
    d64 = dist[:, 1:].mean(axis=1)
    thr = d64.mean() + mul * np.std(d64, ddof=1)
    near = np.abs(d64 - thr) <= 1e-5 * d64.mean()
    assert np.array_equal(kept[~near], (d64 <= thr)[~near])
    assert near.sum() <= 2 and abs(st[2] - thr) <= 1e-6 * d64.mean()
    assert 0 < (~kept).sum() < len(xyz)
