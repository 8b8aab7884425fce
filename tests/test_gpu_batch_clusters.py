"""gpdb_find_clusters_batch: Clustering::findClusters on every group of hands in one call (-m gpu).

Each group's clusters must be bit-equal to gpdb_find_clusters on that group alone (one k_clusters warp per hand, the
inliers of its own group folded in index order), and equal the host Clustering::findClusters of the C++ shim.
"""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, lib, scenes

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "gpd_b200", "host")
SIZES = [0, 1, 31, 32, 33, 300]


@pytest.fixture(scope="module")
def hands():
    """400 real detections on krylon (scores, frames and positions that do form clusters) and a context without a cloud."""
    w, _ = load_weights(15)
    ctx = lib.Context(lib.default_params(channels=15))
    ctx.set_weights(w)
    k = scenes.krylon_cloud()
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    h = ctx.detect_select(np.arange(0, len(k["xyz"]), 2, dtype=np.int32), 400)["candidates"]
    ctx.close()
    assert len(h) == 400
    fresh = lib.Context(lib.default_params(channels=15))  # clustering needs no installed cloud
    yield fresh, h
    fresh.close()


def groups_of(h, sizes, seed):
    """Groups of the given sizes, drawn without replacement from h in a seeded order."""
    order = np.random.default_rng(seed).permutation(len(h))
    out, o = [], 0
    for s in sizes:
        out.append(h[np.sort(order[o:o + s])])
        o += s
    return out


@pytest.mark.parametrize("min_inliers", [0, 1, 3, 1000])
def test_batch_clusters_equal_single_group_calls(hands, min_inliers):
    ctx, h = hands
    for seed, sizes in ((0, SIZES), (1, SIZES[::-1]), (2, [33, 0, 0, 300, 1])):
        groups = groups_of(h, sizes, seed)
        got = ctx.find_clusters_batch(groups, min_inliers)
        assert len(got) == len(groups)
        total = 0
        for g, c in zip(groups, got):
            one = ctx.find_clusters(g, min_inliers)
            assert c.tobytes() == one.tobytes(), (sizes, len(g), min_inliers)
            if min_inliers > len(g):
                assert len(c) == 0
            total += len(c)
        if min_inliers in (0, 1):
            assert total > 0
        if min_inliers == 0:  # every hand has at least zero inliers: every hand is a cluster
            assert [len(c) for c in got] == sizes


def test_batch_clusters_equal_the_host_restatement(hands):
    """The per-group clusters against the shim's host Clustering::findClusters (remove_inliers = false)."""
    ctx, h = hands
    H = C.CDLL(os.path.join(HOST, "libgpd_host.so"))
    H.gpdFindClusters.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    groups = groups_of(h, SIZES, 3)
    for min_inliers in (1, 3):
        got = ctx.find_clusters_batch(groups, min_inliers)
        for g, c in zip(groups, got):
            g = np.ascontiguousarray(g)
            ref = np.zeros(max(len(g), 1), dtype=abi.POSE_DTYPE)
            n = H.gpdFindClusters(g.ctypes.data, len(g), min_inliers, 0, ref.ctypes.data)
            assert len(c) == n
            for f in ("position", "score", "frame", "sample_index", "pose_slot", "full_antipodal"):
                assert np.array_equal(c[f], ref[:n][f]), (len(g), min_inliers, f)


def test_batch_clusters_argument_errors(hands):
    ctx, h = hands
    assert ctx.find_clusters_batch([], 1) == []
    L = lib.lib()
    hh = np.ascontiguousarray(h[:10])
    out = np.zeros(10, dtype=abi.POSE_DTYPE)
    coff = np.zeros(3, np.int32)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for n_groups, hoff in ((2, [1, 5, 10]), (2, [0, 6, 5]), (-1, [0])):
        hoff = np.asarray(hoff, np.int32)
        assert L.gpdb_find_clusters_batch(ctx.h, n_groups, p(hoff), p(hh), 1, p(out), p(coff)) == -1
    ok = np.asarray([0, 4, 10], np.int32)
    assert L.gpdb_find_clusters_batch(ctx.h, 2, p(ok), p(hh), 1, p(out), None) == -1
    assert L.gpdb_find_clusters_batch(ctx.h, 2, p(ok), None, 1, p(out), p(coff)) == -1
    n = L.gpdb_find_clusters_batch(ctx.h, 2, p(ok), p(hh), 1, p(out), p(coff))
    assert n == coff[2] and coff[0] == 0 and coff[1] <= coff[2]
