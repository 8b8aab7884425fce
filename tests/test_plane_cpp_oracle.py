"""The C++ oracle of the support plane (tests/plane_oracle.cpp) against the independent numpy restatement
(tests/plane_reference.py), bit for bit on every part: each hypothesis' attempt, sample indices, coefficients and inlier
count, the picked hypothesis, the hypotheses evaluated, the refined plane, the final inliers and the mask; on the table
scenes, a tilted plane with clutter, N = 0..3, a collinear lattice, a coplanar cloud, points at the threshold and the
stop points of the loop; and the threaded batch against the clouds one by one."""
import numpy as np
import pytest

import plane_oracle as po
import plane_reference as pr
from gpd_b200 import scenes

F = np.float32


def grid(z=0.5, n=20, step=0.01):
    g = np.stack(np.meshgrid(np.arange(n) * step, np.arange(n) * step), -1).reshape(-1, 2)
    return np.column_stack([g, np.full(len(g), z)]).astype(F)


def tilted():
    rng = np.random.default_rng(3)
    nrm = np.array([0.5, 0.0, np.sqrt(0.75)])
    e1, e2 = np.array([np.sqrt(0.75), 0.0, -0.5]), np.array([0.0, 1.0, 0.0])
    u, v = rng.uniform(-0.3, 0.3, (2, 3000))
    p = 0.8 * nrm + u[:, None] * e1 + v[:, None] * e2 + rng.normal(0, 0.001, (3000, 1)) * nrm
    p[2400:] -= rng.uniform(0.03, 0.2, (600, 1)) * nrm
    return p.astype(F)


def threshold_probes(thr):
    t = F(thr)
    return np.vstack([grid(0.0, 10, 0.05), np.array([[0.2, 0.2, t], [0.2, 0.2, -t], [0.1, 0.1, 0.5]], F)])


CASES = {
    "table0": lambda: scenes.synthetic_table_scene(0, n_points=20000)["xyz"],
    "table1": lambda: scenes.synthetic_table_scene(1, n_points=20000)["xyz"],
    "tilted": tilted,
    "n0": lambda: np.zeros((0, 3), F),
    "n1": lambda: np.array([[0, 0, 1]], F),
    "n2": lambda: np.array([[0, 0, 1], [0.1, 0, 1]], F),
    "n3": lambda: np.array([[0, 0, 1], [0.1, 0, 1], [0, 0.1, 1.01]], F),
    "collinear": lambda: (np.arange(50)[:, None] * np.array([[0.25, 0.5, 1.0]])).astype(F),
    "coplanar": grid,
    "sparse": lambda: np.random.default_rng(5).uniform(0, 1, (200, 3)).astype(F),
    "two_planes": lambda: np.vstack([grid(0.0, 8, 0.1), grid(1.0, 8, 0.1)]),
}
PARAMS = {"default": {}, "thr_1mm_1024": dict(distance_threshold=0.001, max_iterations=1024),
          "one_iteration": dict(max_iterations=1), "p_half": dict(probability=0.5), "p_0999_200": dict(probability=0.999, max_iterations=200)}


def check(xyz, key, **kw):
    o = po.segment(xyz, key=key, **kw)
    r = pr.segment(xyz, key=key, **kw)
    assert o["n_hypotheses"] == r["n_hypotheses"] and o["best"] == r["best"]
    drawn = [h for h in r["hyps"] if h is not None]
    for h, hy in enumerate(drawn):
        a, idx, coef = hy
        assert o["attempts"][h] == a and o["samples"][h].tolist() == list(idx)
        assert o["coefs"][h].tobytes() == coef.tobytes()
    assert o["counts"][:len(r["counts"])].tolist() == r["counts"]
    assert (o["counts"][len(r["counts"]):] == -1).all()
    if len(r["hyps"]) and r["hyps"][-1] is None:
        assert o["attempts"][len(r["hyps"]) - 1] == -1
    assert o["plane"].tobytes() == r["plane"].tobytes()
    assert o["n_inliers"] == r["n_inliers"] and np.array_equal(o["eligible"], r["eligible"])
    return o


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_equals_numpy(case):
    xyz = CASES[case]()
    for key in (0, 9, 2**40 + 1):
        check(xyz, key)


@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("case", ["table0", "sparse", "two_planes", "tilted"])
def test_oracle_equals_numpy_off_defaults(case, params):
    check(CASES[case](), 4, **PARAMS[params])


@pytest.mark.parametrize("thr,want", [(0.25, [1, 1, 1]), (0.01, [0, 0, 1])])
def test_oracle_threshold_is_strict(thr, want):
    o = check(threshold_probes(thr), 0, distance_threshold=thr)
    assert o["eligible"][-3:].tolist() == want


def test_oracle_edges():
    assert check(CASES["collinear"](), 0)["n_hypotheses"] == 0
    o = check(CASES["coplanar"](), 0)
    assert o["n_hypotheses"] == 1 and (o["eligible"] == 1).all() and o["n_inliers"] == 400
    assert check(CASES["sparse"](), 4, distance_threshold=0.001, max_iterations=1024)["n_hypotheses"] == 1025
    assert check(CASES["sparse"](), 4, distance_threshold=0.001, max_iterations=1)["n_hypotheses"] == 2
    for n in range(3):
        o = check(CASES[f"n{n}"](), 0)
        assert o["best"] == -1 and np.isnan(o["plane"]).all()


def test_threaded_batch_equals_the_clouds_one_by_one():
    clouds = [CASES[c]() for c in ("table0", "n0", "n2", "collinear", "coplanar", "tilted", "sparse", "table1")]
    off = np.concatenate([[0], np.cumsum([len(x) for x in clouds])])
    r = po.segment_batch(off, np.concatenate(clouds), seed=100, threads=3)
    for b, x in enumerate(clouds):
        o = po.segment(x, key=100 + b)
        assert r["planes"][b].tobytes() == o["plane"].tobytes()
        assert r["n_inliers"][b] == o["n_inliers"] and r["n_hypotheses"][b] == o["n_hypotheses"]
        assert np.array_equal(r["eligible"][off[b]:off[b + 1]], o["eligible"])
