"""GPU tests of the image stage's fast kernel (k_images2) on inputs built to reach its less common paths. Each case
compares the fast path's images bit for bit with the general tier (k_images, GPD_B200_IMAGES_KERNEL=1) and, within the
parity tolerance of tests/test_gpu_parity.py, with the CPU oracle, which shares no code with the kernels. The event
counters of gpdb_debug_phase_cycles show that each path ran: [0] shadow cell-sum entries whose low word carried, [1] the most
shadow voxels summed into one cell, [14] shadow casts that walked the grid because the in-ball list was full."""
import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import lib, scenes
from oracle import oracle

pytestmark = pytest.mark.gpu


def bench_cloud(copies=1, turn_copies=False):
    """The bench cloud (config 3) with every point `copies` times, at the same position. With turn_copies, each further
    copy has its normal turned by about 30 degrees (still of unit length)."""
    s = scenes.synthetic_table_scene(3)
    nrm = [s["normals"]]
    for _ in range(copies - 1):
        n = nrm[-1]
        if turn_copies:
            side = np.cross(n, np.array([0.3, 0.5, 0.8]))
            side /= np.linalg.norm(side, axis=1, keepdims=True)
            n = n + 0.6 * side
            n /= np.linalg.norm(n, axis=1, keepdims=True)
        nrm.append(n)
    cloud = {"xyz": np.ascontiguousarray(np.concatenate([s["xyz"]] * copies)),
             "normals": np.ascontiguousarray(np.concatenate(nrm)),
             "cam_source": np.ascontiguousarray(np.concatenate([s["cam_source"]] * copies)),
             "view_points": s["view_points"]}
    sidx = np.random.default_rng(11).choice(len(s["xyz"]), 1500, replace=False).astype(np.int32)
    return cloud, sidx


def run_tiers(cloud, sidx, monkeypatch, n_oracle):
    w, relu = load_weights(15)
    p = lib.default_params(channels=15, relu_after_conv=relu, keep_images=1)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    ctx.set_cloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    ctx.phase_cycles(1)
    fast = ctx.detect(sidx)
    counters = ctx.phase_cycles(0)
    monkeypatch.setenv("GPD_B200_IMAGES_KERNEL", "1")
    general = ctx.detect(sidx)
    monkeypatch.delenv("GPD_B200_IMAGES_KERNEL")
    assert fast["kernel_launches"] == general["kernel_launches"] + 1  # the fast path ran
    assert general["n_candidates"] > 100
    assert np.array_equal(general["images"], fast["images"])
    # a subset against the oracle
    sub = sidx[:n_oracle]
    rg = ctx.detect(sub)
    oc = oracle.OracleCloud(cloud["xyz"], cloud["normals"], cloud["cam_source"], cloud["view_points"])
    ro = oc.detect(p, oracle.WeightPack(w), sub)
    assert rg["n_candidates"] == ro["n_candidates"] > 0
    assert np.array_equal(ro["pose_flags"], rg["pose_flags"])
    d = np.abs(ro["images"].astype(np.int32) - rg["images"].astype(np.int32))
    assert d.max() <= 1 and np.count_nonzero(d) <= 1e-3 * d.size
    ctx.close()
    return counters


def test_carries_and_collapsed_shadow_voxels(monkeypatch):
    """The bench cloud as it is: cells with two or more points whose unit coordinate is at least 0.5 carry past 2^32, and
    shadow voxels stacked along a projection axis collapse into one cell."""
    counters = run_tiers(*bench_cloud(), monkeypatch, n_oracle=120)
    assert counters[0] > 0, "no cell sum carried out of its low word"
    assert counters[1] >= 10, f"at most {counters[1]} shadow voxels summed into one cell"


def test_distance_ties_broken_by_index(monkeypatch):
    """Every point twice, the copy (larger index) with its normal turned by about 30 degrees: every occupied cell holds an
    exact distance tie between two points with different normals, which only the index word of the arg-max key decides
    (the reference's last writer, the copy). A missing or reversed index max puts the other normal into the normal
    channels and fails the comparison with the oracle. The doubled neighbourhood (about 3 700 points in the r = 0.10
    ball) also overflows the 3 600-entry in-ball list in many images, whose shadow casting then walks the grid."""
    counters = run_tiers(*bench_cloud(2, turn_copies=True), monkeypatch, n_oracle=120)
    assert counters[14] > 0, "no image took the grid-walk fallback of the shadow casting"

