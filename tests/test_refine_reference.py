"""The restatement of include/gpd_b200_refine.h (tests/refine_reference.py) on constructed cases, and the C++ oracle
(tests/refine_oracle.cpp) against it bit for bit: neighbour lists against brute force (random clouds, exact distance ties
on lattices, duplicate points, k >= N), the FLT_EPSILON guard, skipped non-finite neighbours, the stop rule at 1 and at
15 iterations, and the float32 acos of the stop statistic against float64."""
import functools

import numpy as np
import pytest

import refine_oracle as ro
import refine_reference as rr
from gpd_b200 import scenes

F = np.float32


@functools.lru_cache(None)
def table(seed):
    """A part (4 000 points) of a synthetic table scene."""
    sc = scenes.synthetic_table_scene(seed, n_points=20000)
    return sc["xyz"][:4000], sc["normals"][:4000]


def naive_knn(xyz, k):
    """Rule 1 with Python sorting of (distance, index) pairs, distances from the float32 operations of L2_Simple."""
    xyz = np.asarray(xyz, F)
    out = []
    for i in range(len(xyz)):
        d = [rr.l2(xyz[i:i + 1], xyz[j:j + 1])[0, 0] for j in range(len(xyz))]
        out.append([j for _, j in sorted((float(d[j]), j) for j in range(len(xyz)))[:k]])
    return np.array(out, np.int32).reshape(len(xyz), min(k, len(xyz)))


def lattice(n=6, step=0.01):
    g = np.stack(np.meshgrid(*(np.arange(n) * step,) * 3, indexing="ij"), -1).reshape(-1, 3)
    return (g + 0.25).astype(F)


def with_duplicates(seed=0):
    rng = np.random.default_rng(seed)
    p = rng.uniform(0, 0.1, (300, 3)).astype(F)
    return np.concatenate([p, p[rng.integers(0, 300, 150)]])


def random_normals(n, seed=0):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def test_knn_brute_against_naive_sort():
    rng = np.random.default_rng(1)
    for xyz, k in [(rng.uniform(0, 1, (40, 3)).astype(F), 7), (lattice(3), 9), (with_duplicates()[:60], 12),
                   (lattice(2), 20)]:
        assert np.array_equal(rr.knn_brute(xyz, k), naive_knn(xyz, k))


@pytest.mark.parametrize("k", [1, 2, 10, 50, 128])
def test_knn_superset_path_equals_brute_force(k):
    rng = np.random.default_rng(k)
    clouds = [rng.uniform(0, 0.3, (3000, 3)).astype(F), lattice(12), with_duplicates(k),
              table(2)[0]]
    for xyz in clouds:
        assert np.array_equal(rr.knn(xyz, k, brute_below=0), rr.knn_brute(xyz, k))


def test_knn_ties_break_by_index_and_self_first():
    xyz = lattice(4)
    nbr = rr.knn_brute(xyz, 7)
    assert np.array_equal(nbr[:, 0], np.arange(len(xyz)))
    # an inner lattice point: its six face neighbours tie, in index order
    i = 1 * 16 + 1 * 4 + 1
    assert list(nbr[i, 1:]) == sorted([i - 16, i + 16, i - 4, i + 4, i - 1, i + 1])
    dup = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0]], F)
    assert list(rr.knn_brute(dup, 3)[2]) == [0, 2, 1]  # the earlier duplicate comes first, at distance 0


def test_k_at_least_n_lists_every_point():
    xyz = np.random.default_rng(2).uniform(0, 1, (9, 3)).astype(F)
    for k in (9, 10, 128):
        nbr = rr.knn(xyz, k)
        assert nbr.shape == (9, 9) and all(sorted(r) == list(range(9)) for r in nbr)


def test_flt_epsilon_guard_gives_nan():
    xyz = np.array([[0, 0, 0], [0.001, 0, 0]], F)
    out, it = rr.refine(xyz, np.array([[0, 0, 1.0], [0, 0, -1.0]]), 2)
    assert np.isnan(out).all() and it == 1  # the errors are 0 for non-finite normals: the mean is 0


def test_nonfinite_neighbours_are_skipped():
    xyz = np.array([[0, 0, 0], [0.001, 0, 0], [0.002, 0, 0]], F)
    nrm = np.array([[np.nan] * 3, [0, 0.6, 0.8], [0, 0, 1.0]])
    nbr = rr.knn(xyz, 3)
    m, err = rr.iterate(nbr, nrm.astype(F))
    s = np.array([0, 0.6, 0.8], F) + np.array([0, 0, 1], F)
    want = rr.refine_normal(s[None, 0], s[None, 1], s[None, 2])[0]
    assert np.array_equal(m[0], want) and np.all(np.isfinite(m))  # the NaN point gets a finite normal
    assert err[0] == 0


def test_stop_rule_after_one_iteration():
    xyz = np.random.default_rng(3).uniform(0, 0.1, (200, 3)).astype(F)
    out, it = rr.refine(xyz, np.tile([0, 0, 1.0], (200, 1)), 10)
    assert it == 1 and np.array_equal(out, np.tile([0, 0, 1.0], (200, 1)))


def test_stop_rule_runs_to_fifteen():
    xyz = (np.arange(400)[:, None] * np.array([[0.001, 0, 0]])).astype(F)
    trace = []
    _, it = rr.refine(xyz, random_normals(400, 4), 3, trace=trace)
    assert it == rr.MAX_ITERATIONS and all(t >= rr.CONVERGENCE for t in trace)


def two_clusters(seed=5):
    """1 000 lattice points with normal (0, 0, 1) and, 5 m away, a cluster of 10 with perturbed normals: with k = 10 the
    small cluster converges to within rounding in one iteration, so the mean drops under the threshold in the second."""
    rng = np.random.default_rng(seed)
    xyz = np.concatenate([lattice(10), 5 + rng.uniform(0, 0.001, (10, 3))]).astype(F)
    nrm = np.tile([0, 0, 1.0], (1010, 1))
    nrm[1000:] += 0.3 * random_normals(10, seed)
    return xyz, nrm / np.linalg.norm(nrm, axis=1, keepdims=True)


def test_stop_rule_in_between():
    xyz, nrm = two_clusters()
    trace = []
    _, it = rr.refine(xyz, nrm, 10, trace=trace)
    assert 1 < it < rr.MAX_ITERATIONS and trace[-1] < rr.CONVERGENCE <= trace[-2]


def test_acosf_against_float64():
    x = np.concatenate([np.linspace(-1, 1, 200001), [0.5, -0.5, 1 - 2 ** -24, -1 + 2 ** -24, 0.0]]).astype(F)
    got = rr.acosf(x).astype(np.float64)
    want = np.arccos(x.astype(np.float64))
    ulp = np.spacing(want.astype(F)).astype(np.float64)
    assert np.max(np.abs(got - want) / ulp) <= 4


def test_sequential_mean_is_not_pairwise():
    e = np.array([1.0] + [2 ** -24] * 4, F)
    assert rr.mean_error(e) == F(1) / F(5)  # each tiny term rounds away against the running sum


def cases():
    rng = np.random.default_rng(6)
    txyz, tnrm = table(3)
    nan_nrm = random_normals(500, 7)
    nan_nrm[rng.integers(0, 500, 40)] = np.nan
    return [("table", txyz, tnrm, 10),
            ("duplicates", with_duplicates(2), random_normals(450, 8), 20),
            ("lattice", lattice(7), random_normals(343, 9), 7),
            ("nan_normals", rng.uniform(0, 0.1, (500, 3)).astype(F), nan_nrm, 12),
            ("k_ge_n", rng.uniform(0, 1, (30, 3)).astype(F), random_normals(30, 10), 50),
            ("two_clusters",) + two_clusters() + (10,),
            ("line", (np.arange(400)[:, None] * np.array([[0.001, 0, 0]])).astype(F), random_normals(400, 11), 2)]


@pytest.mark.parametrize("name,xyz,nrm,k", cases(), ids=[c[0] for c in cases()])
def test_cpp_oracle_equals_numpy(name, xyz, nrm, k):
    nbr = rr.knn(xyz, k)
    assert np.array_equal(ro.knn(xyz, k), nbr)
    want, it = rr.refine(xyz, nrm, k, nbr=nbr)
    got, git = ro.refine(xyz, nrm, k)
    assert git == it
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))


def test_cpp_oracle_batch_equals_clouds_one_by_one():
    cs = cases()
    off = np.concatenate([[0], np.cumsum([len(c[1]) for c in cs[:4]] + [0])]).astype(np.int32)
    xyz = np.concatenate([c[1] for c in cs[:4]])
    nrm = np.concatenate([c[2] for c in cs[:4]])
    got, its = ro.refine_batch(off, xyz, nrm, 9, threads=3)
    want, wits = rr.refine_batch(off, xyz, nrm, 9)
    assert np.array_equal(its, wits) and wits[-1] == 0
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
