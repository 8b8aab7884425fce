"""CPU proofs for the shadow casting of the 15-channel images: the kernels' restatement (shadow_cast_reference.py) gives
the same in-box shadow as the header's restatement (image_reference.shadow_points); every filter the kernels put in
front of the float64 voxel arithmetic (slab cull, LCG window, bitmap AABB, float32 pre-test) keeps every voxel whose
jittered point lies in the box; and every case of shadow_cases.py reaches its count exactly."""
import math
from fractions import Fraction

import numpy as np
import pytest

import capacity_cases as cc
import image_cases as ic
import image_reference as ir
import shadow_cases as sc
import shadow_cast_reference as scr
from gpd_b200 import abi


def reference_in_box(cloud, pose, g):
    """image_reference.shadow_points of the pose, restricted to the image box."""
    idx, _ = ir.neighbourhood(cloud, pose["sample"], g.radius)
    sp = ir.shadow_points(cloud, idx, int(pose["sample_index"]), g.radius)
    return sp[scr.points_in_box(g, pose, sp)]


def same_points(a, b):
    sa = a[np.lexsort((a[:, 2], a[:, 1], a[:, 0]))] if len(a) else a
    sb = b[np.lexsort((b[:, 2], b[:, 1], b[:, 0]))] if len(b) else b
    return sa.shape == sb.shape and np.array_equal(sa, sb)


def filters_keep_the_box(res, g, pose, qtab):
    """Per cast camera: every voxel of an unfiltered draw whose jittered point lies in the box has its bit set."""
    st = res["setup"]
    d1 = int(st["bm_dims"][1])
    for k, c in enumerate(res["cams"]):
        if c is None:
            continue
        raw = np.unique(c["raw"], axis=0)
        inb = raw[scr.points_in_box(g, pose, scr.voxel_points(raw, qtab))]
        b = inb - st["bm_org"][None]
        assert ((b >= 0) & (b < st["bm_dims"][None])).all(), "an in-box voxel outside the bitmap AABB"
        codes = b[:, 0] + 64 * (b[:, 1] + d1 * b[:, 2])
        missing = np.setdiff1d(codes, c["codes"])
        assert len(missing) == 0, f"camera {k}: {len(missing)} in-box voxels dropped by the cull, window or pre-test"


def test_fmaf_rounds_the_exact_value():
    """Random operands against the exact value, and the two midpoint cases: a tie (to even), and an exact value just
    above a midpoint that the float64 sum rounds onto it (a double rounding would give the even neighbour)."""
    rng = np.random.default_rng(0)
    a, b = (rng.standard_normal((2, 500)) * np.array([[1.0], [0.1]])).astype(np.float32)
    c = (rng.standard_normal(500) * 1e-2).astype(np.float32)
    out = scr.fmaf(a, b, c)
    for i in range(500):
        ex = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        near = np.float32(float(ex))
        cands = [near, np.nextafter(near, np.float32(np.inf)), np.nextafter(near, np.float32(-np.inf))]
        assert out[i] == min(cands, key=lambda v: (abs(Fraction(float(v)) - ex), int(np.array(v).view(np.uint32)) & 1))
    one_up, one_down = np.float32(1.0 + 2.0 ** -23), np.float32(1.0 - 2.0 ** -24)  # product 1 + 2^-24 - 2^-47
    assert scr.fmaf(one_up, one_down, np.float32(2.0 ** -47)) == np.float32(1.0)
    assert scr.fmaf(one_up, one_down, np.float32(2.0 ** -47 + 2.0 ** -60)) == one_up


def test_centre_exactness_condition():
    assert scr.centre_is_exact(np.array([[0.5, 0.25, 0.125]], np.float32))
    assert scr.centre_is_exact(np.float32(np.random.default_rng(0).uniform(0.3, 0.7, (5000, 3))))
    # a coordinate near 0 has a fine resolution: 1e-30 next to 0.5 cannot be summed exactly
    assert not scr.centre_is_exact(np.array([[0.5, 0.5, 0.5], [1e-30, 0.5, 0.5]], np.float32))


def test_caps_and_geometries_of_the_cases():
    assert cc.bm_dim() == 48 and cc.bm_dim(volume_depth=0.05) == 46 and cc.bm_dim(volume_height=0.04) == 54
    assert cc.fast_path_15(46, 2) and not cc.fast_path_15(47, 2) and cc.fast_path_15(48, 1)
    assert not cc.fast_path_15(48, 2)  # two cameras at the default volume: k_images does the work
    # two cameras take the fast path up to bm_dim 46 (volume_depth 0.05); volume_depth 0.055 gives 47
    assert cc.bm_dim(volume_depth=0.055) == 47
    assert cc.bl_cap(54, 1) == 12600 and cc.bl_cap(48, 1) == 13824
    for name, geo in sc.GEOMETRIES.items():
        assert scr.Params(ir.Geometry(**geo)).bm_dim == cc.bm_dim(geo["w"], geo["d"], geo["h"]), name


@pytest.mark.parametrize("case", ic.shadow_cases(), ids=lambda c: c["name"])
def test_restatements_agree_on_the_covered_shadow_cases(case):
    g, cloud = case["geometry"], case["cloud"]
    qtab = ir.norm_quantile_table()
    for pose in case["poses"]:
        res = scr.cast(cloud, pose, g, qtab, raw=True)
        assert res["nset_all"] > 0 and same_points(res["in_box"], reference_in_box(cloud, pose, g))
        filters_keep_the_box(res, g, pose, qtab)


CAPACITY_SHADOW = [(40, 0, 1, 0.06), (1000, 900, 1, 0.06), (1000, 100, 1, 0.06), (1000, 100, 2, 0.05)]


@pytest.mark.parametrize("n_box,n_out,k,d", CAPACITY_SHADOW)
def test_restatements_agree_on_the_capacity_inputs(n_box, n_out, k, d):
    cloud, pose = cc.image_box(n_box, n_outside=n_out)
    if k == 2:
        cloud["view_points"] = np.array([[0.0, 0.0, 0.0], [0.3, 0.0, 0.0]])
        cloud["cam_source"] = np.ones((len(cloud["xyz"]), 2), np.int32)
    g = ir.Geometry(C=15, d=d)
    qtab = ir.norm_quantile_table()
    res = scr.cast(cloud, pose[0], g, qtab, raw=True)
    assert res["nset_all"] > 0 and same_points(res["in_box"], reference_in_box(cloud, pose[0], g))
    filters_keep_the_box(res, g, pose[0], qtab)


def _rotation(rng, kind):
    if kind == "45":
        a = rng.integers(3)
        c, s = math.cos(math.pi / 4), math.sin(math.pi / 4)
        R = np.eye(3)
        i, j = [(1, 2), (0, 2), (0, 1)][a]
        R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
        return R
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def random_pose_case(seed):
    """An object of 150-500 float32 points around a sample at (0.3, 0.2, 0.6) (no coordinate near 0): a slab in front of
    the box and a scatter through the ball; a rotated frame (45 degrees about one axis, or uniform), one to three
    cameras about 1 m away, random camera sets (camera 0 sometimes sees nothing), geometry default or varied."""
    rng = np.random.default_rng(seed)
    kind = "45" if seed % 2 == 0 else "uniform"
    R = _rotation(rng, kind)
    geo = dict(S=60, C=15, w=0.10, d=0.06, h=0.02)
    if seed % 5 == 4:
        geo.update(w=float(rng.uniform(0.06, 0.12)), d=float(rng.uniform(0.03, 0.07)), h=float(rng.uniform(0.01, 0.04)))
    g = ir.Geometry(**geo)
    s = np.array([0.3, 0.2, 0.6])
    pose = np.zeros(1, dtype=abi.POSE_DTYPE)
    pose["sample"][0] = s
    pose["frame"][0] = R.ravel()
    pose["bottom"] = rng.uniform(-0.02, 0.01)
    pose["center"] = rng.uniform(-0.02, 0.02)
    pose["top"] = pose["bottom"] + g.d
    pose["sample_index"] = int(rng.integers(0, 2 ** 31))
    K = int(rng.integers(1, 4))
    vp = s + rng.standard_normal((K, 3)) * 0.3 + np.array([0.0, 0.0, -1.0])
    n = int(rng.integers(150, 500))
    hand = np.stack([rng.uniform(-0.02, 0.08, n), rng.uniform(-0.06, 0.06, n), rng.uniform(-0.08, 0.04, n)], 1)
    hand[: n // 2, 2] = rng.uniform(-g.h - 0.03, -g.h, n // 2)   # a slab on the camera side of the box
    xyz = (s + hand @ R).astype(np.float32)
    cam = (rng.random((n, K)) < 0.9).astype(np.int32)
    if K > 1 and seed % 7 == 3:
        cam[:, 0] = 0
    nrm = cc._unit(rng.standard_normal((n, 3)))
    cloud = {"xyz": xyz, "normals": nrm, "cam_source": cam, "view_points": vp}
    return cloud, pose[0], g


@pytest.mark.parametrize("block", range(8))
def test_random_poses(block):
    """300 random poses: the restatements agree, the filters keep every in-box voxel, and the bitmap AABB fits bm_dim."""
    qtab = ir.norm_quantile_table()
    nonempty = 0
    for seed in range(block * 38, block * 38 + 38):
        cloud, pose, g = random_pose_case(seed)
        res = scr.cast(cloud, pose, g, qtab, raw=True)
        st = res["setup"]
        assert (st["aabb_hi"] - st["aabb_lo"] + 1 <= res["params"].bm_dim).all(), (seed, st["aabb_hi"] - st["aabb_lo"])
        assert same_points(res["in_box"], reference_in_box(cloud, pose, g)), seed
        filters_keep_the_box(res, g, pose, qtab)
        nonempty += len(res["in_box"]) > 0
    assert nonempty >= 19  # most poses cast some shadow into the box


@pytest.mark.parametrize("i", range(len(sc.EDGES)), ids=sc.IDS)
def test_every_case_reaches_its_count(i):
    case = sc.build(i)
    r = case["counts"]
    g, pose, cloud = case["geometry"], case["pose"][0], case["cloud"]
    name, edge, target = case["name"], case["edge"], case["target"]
    K = case["K"]
    again = scr.cast(cloud, pose, g)
    assert again["nset_all"] == r["nset_all"] and again["wl_n"] == r["wl_n"] and again["dl_n"] == r["dl_n"]
    assert same_points(r["in_box"], reference_in_box(cloud, pose, g))
    box = cc.box_count(cloud, case["pose"], g.w, g.d, g.h, g.radius)
    fast = cc.fast_path_15(scr.Params(g).bm_dim, K)
    if name.startswith("stash"):
        assert r["nset_all"] == target and fast and box <= cc.BOX_CAP2
        assert max(r["wl_n"]) <= cc.WL_CAP2 and max(r["dl_n"]) <= cc.DL_CAP and r["n_ball"] <= cc.BALL_CAP2
    elif name == "voxel_list":
        # k_images' voxel list is 12 600 entries at bm_dim 54; 12 600 voxels need more draws than the draw list holds,
        # so it overflows too (by an exact count: every listed point's 33 draws pass their window)
        assert r["nset_all"] == target and max(r["wl_n"]) <= cc.WL_CAP2 and r["n_ball"] <= cc.BALL_CAP2
        assert r["dl_n"][0] > cc.DL_CAP
    elif name.startswith("work_list"):
        # every point in the work list has a full window: the draw counts do not depend on which points are listed;
        # they exceed the draw list (nsp = 33 draws per point), which these cases leave overflowing
        assert r["wl_n"] == [target] * K
        for k in range(K):
            assert set(r["cams"][k]["draws"][r["cams"][k]["work"]]) == {scr.Params(g).nsp}
        assert box <= cc.BOX_CAP2 and fast
    elif name == "draw_list":
        assert r["dl_n"] == [target] and r["wl_n"][0] <= cc.WL_CAP2 and box <= cc.BOX_CAP2
    elif name == "ball":
        assert r["n_ball"] == target and max(r["wl_n"]) <= cc.WL_CAP2 and max(r["dl_n"]) <= cc.DL_CAP
        assert r["nset_all"] <= cc.st_cap2(48, 1)
    else:
        assert r["cam_or"] == 2 and r["nset_all"] == 0 and len(r["in_box"]) == 0
        assert r["wl_n"][0] == 0 and r["wl_n"][1] > 0 and fast
