"""The support plane on the device: gpdb_segment_plane, gpdb_segment_planes[_device] and
gpdb_subsample_clouds_points[_device] against the numpy restatement of include/gpd_b200_plane.h (tests/plane_reference.py).

Hypotheses evaluated are compared exactly. The refined plane is bit-equal, or (pcl::eigen33's atan2f / cosf / sinf, DESIGN.md
4b) within the float32 bound of the normals; then the masks may differ only at points whose distance lies within that
bound of the threshold, and the test counts them (0 on the table scenes)."""
import ctypes as C

import numpy as np
import pytest

import depth_reference as dr
import plane_reference as pr
from conftest import load_weights
from gpd_b200 import lib, scenes

pytestmark = pytest.mark.gpu
ERR_INVALID, ERR_STATE = -1, -3
F = np.float32


def torch_():
    return pytest.importorskip("torch")


def context(weights=False):
    w, relu = load_weights(12)
    ctx = lib.Context(lib.default_params(channels=12, relu_after_conv=relu))
    if weights:
        ctx.set_weights(w)
    return ctx


def cloud(xyz):
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    return {"xyz": xyz, "normals": np.tile([0.0, 0.0, 1.0], (len(xyz), 1)), "view_points": np.zeros((1, 3))}


def mixed_clouds():
    """Table scenes, 2 and 3 points, a collinear lattice (fails), a coplanar grid (w = 1), a tilted
    plane with clutter and a sparse cloud (many hypotheses)."""
    rng = np.random.default_rng(7)
    g = np.stack(np.meshgrid(np.arange(20) * 0.01, np.arange(20) * 0.01), -1).reshape(-1, 2)
    nrm = np.array([0.5, 0.0, np.sqrt(0.75)])
    e1, e2 = np.array([np.sqrt(0.75), 0.0, -0.5]), np.array([0.0, 1.0, 0.0])
    u, v = rng.uniform(-0.3, 0.3, (2, 3000))
    tilted = 0.8 * nrm + u[:, None] * e1 + v[:, None] * e2 + rng.normal(0, 0.001, (3000, 1)) * nrm
    tilted[2400:] -= rng.uniform(0.03, 0.2, (600, 1)) * nrm
    return [scenes.synthetic_table_scene(0, n_points=20000)["xyz"],
            np.array([[0, 0, 1], [0.1, 0, 1]], F),
            np.array([[0, 0, 1], [0.1, 0, 1], [0, 0.1, 1.01]], F),
            (np.arange(50)[:, None] * np.array([[0.25, 0.5, 1.0]])).astype(F),
            np.column_stack([g, np.full(len(g), 0.5)]).astype(F),
            tilted.astype(F),
            rng.uniform(0, 1, (300, 3)).astype(F),
            scenes.synthetic_table_scene(1, n_points=20000)["xyz"]]


def normal_bound(pts):
    p = pts.astype(np.float64)
    w = np.linalg.eigvalsh(np.cov(p.T, bias=True))
    return 16 * (3 * np.sqrt(len(p)) * 2.0 ** -24 * np.abs(p).max() ** 2 + 2.0 ** -23 * w[2]) / max(w[1] - w[0], 1e-300) + 1e-6


def check_cloud(xyz, ref, plane, n_inl, n_hyp, elig, thr=0.01):
    """One cloud's device result against the restatement; returns the mask differences near the threshold."""
    assert n_hyp == ref["n_hypotheses"]
    if ref["best"] < 0:
        assert np.isnan(plane).all() and n_inl == 0 and (elig == 1).all()
        return 0
    if plane.tobytes() == ref["plane"].tobytes():
        assert n_inl == ref["n_inliers"] and np.array_equal(elig, ref["eligible"])
        return 0
    assert ref["refit"], "without a refit the plane is the hypothesis' and must be bit-equal"
    n0, n1 = ref["plane"][:3].astype(np.float64), plane[:3].astype(np.float64)
    ang = np.arccos(min(1.0, abs(float(n0 @ n1)) / (np.linalg.norm(n0) * np.linalg.norm(n1))))
    bound = normal_bound(ref["best_inliers"])
    assert ang <= bound, (ang, bound)
    ext = float(np.abs(xyz).max())
    tol = bound * ext * 4 + abs(float(plane[3]) - float(ref["plane"][3])) + 1e-6
    diff = elig != ref["eligible"]
    near = np.abs(ref["dist"].astype(np.float64) - thr) <= tol
    assert not (diff & ~near).any()
    return int(diff.sum())


def test_batch_equals_the_restatement_and_batches_of_one():
    """B mixed clouds in one call (K_b = 1..8 camera counts), against the restatement with key seed + b; each cloud alone
    (a batch of one with seed + b) gives the same bytes; the table scenes differ in no mask byte."""
    clouds = mixed_clouds()
    cl = [dict(cloud(x), view_points=np.zeros((1 + b % 8, 3))) for b, x in enumerate(clouds)]
    ctx = context()
    ctx.set_clouds(cl)
    pl = lib.plane_params(seed=100)
    r = ctx.segment_planes(pl)
    off = np.concatenate([[0], np.cumsum([len(x) for x in clouds])])
    near = []
    for b, x in enumerate(clouds):
        ref = pr.segment(x, key=100 + b)
        e = r["eligible"][off[b]:off[b + 1]]
        near.append(check_cloud(x, ref, r["planes"][b], r["n_inliers"][b], r["n_hypotheses"][b], e))
    print("mask bytes differing near the threshold per cloud:", near)
    assert near[0] == 0 and near[-1] == 0
    for b, x in enumerate(clouds):
        ctx.set_clouds([cl[b]])
        one = ctx.segment_planes(lib.plane_params(seed=100 + b))
        assert one["planes"].tobytes() == r["planes"][b:b + 1].tobytes()
        assert one["n_inliers"][0] == r["n_inliers"][b] and one["n_hypotheses"][0] == r["n_hypotheses"][b]
        assert np.array_equal(one["eligible"], r["eligible"][off[b]:off[b + 1]])
    ctx.close()


@pytest.mark.parametrize("over", [dict(distance_threshold=0.002, max_iterations=1), dict(max_iterations=1024, probability=0.999999),
                                  dict(probability=0.5, seed=2**40 + 3)])
def test_off_default_parameters(over):
    clouds = [scenes.synthetic_table_scene(3, n_points=8000)["xyz"], np.random.default_rng(9).uniform(0, 1, (400, 3)).astype(F)]
    ctx = context()
    ctx.set_clouds([cloud(x) for x in clouds])
    pl = lib.plane_params(**over)
    r = ctx.segment_planes(pl)
    off = np.concatenate([[0], np.cumsum([len(x) for x in clouds])])
    for b, x in enumerate(clouds):
        ref = pr.segment(x, key=pl.seed + b, distance_threshold=pl.distance_threshold, max_iterations=pl.max_iterations,
                         probability=pl.probability)
        check_cloud(x, ref, r["planes"][b], r["n_inliers"][b], r["n_hypotheses"][b], r["eligible"][off[b]:off[b + 1]],
                    thr=pl.distance_threshold)
    ctx.close()


def test_twins_single_cloud_and_nothing_installed_changes():
    """Host and device twins are byte-equal (also on a side stream); gpdb_segment_plane on the single cloud equals a
    batch of one; the installed clouds and the sample draw are the same before and after."""
    torch = torch_()
    clouds = mixed_clouds()[:4]
    ctx = context()
    ctx.set_clouds([cloud(x) for x in clouds])
    before = ctx.get_clouds()
    draw0 = ctx.subsample_clouds(30, 5)
    h = ctx.segment_planes()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = ctx.segment_planes_tensors()
        de = d["eligible"].cpu().numpy()
    for k in ("planes", "n_inliers", "n_hypotheses"):
        assert h[k].tobytes() == d[k].tobytes()
    assert np.array_equal(h["eligible"], de)
    after = ctx.get_clouds()
    for x, y in zip(before, after):
        assert np.array_equal(x["xyz"], y["xyz"]) and np.array_equal(x["normals"], y["normals"])
    assert all(np.array_equal(a, b) for a, b in zip(draw0, ctx.subsample_clouds(30, 5)))
    c0 = cloud(clouds[0])
    ctx.set_cloud(c0["xyz"], c0["normals"])
    plane, n_inl, elig = ctx.segment_plane()
    assert plane.tobytes() == h["planes"][0].tobytes() and n_inl == h["n_inliers"][0]
    assert np.array_equal(elig, h["eligible"][:len(clouds[0])])
    ctx.close()


def test_subsample_clouds_points():
    """The per-point mask draw against the numpy rule, host and device twins; an all-zero mask draws nothing; no mask
    equals gpdb_subsample_clouds without one, bit for bit; it works after gpdb_set_clouds."""
    torch = torch_()
    clouds = [scenes.synthetic_table_scene(4, n_points=8000)["xyz"], np.random.default_rng(3).uniform(0, 1, (40, 3)).astype(F),
              np.random.default_rng(1).uniform(0, 1, (700, 3)).astype(F)]
    ctx = context()
    ctx.set_clouds([cloud(x) for x in clouds])
    off = np.concatenate([[0], np.cumsum([len(x) for x in clouds])]).astype(np.int32)
    mask = (np.random.default_rng(2).random(off[-1]) < 0.3).astype(np.uint8)
    for num in (0, 1, 50, 10000):
        want = pr.subsample_points(off, mask, num, 17)
        got = ctx.subsample_clouds_points(num, 17, mask)
        assert all(np.array_equal(a, b) for a, b in zip(got, want))
        soff, idx = ctx.subsample_clouds_points_tensors(num, 17, torch.from_numpy(mask).cuda())
        idx = idx.cpu().numpy()
        assert all(np.array_equal(idx[soff[b]:soff[b + 1]], want[b]) for b in range(len(clouds)))
        assert all(np.array_equal(a, b) for a, b in zip(ctx.subsample_clouds_points(num, 17), ctx.subsample_clouds(num, 17)))
    assert all(len(a) == 0 for a in ctx.subsample_clouds_points(20, 3, np.zeros(off[-1], np.uint8)))
    ctx.close()


def test_depth_to_grasps_above_the_table():
    """Rendered views -> preprocess_depth_tensors -> segment_planes_tensors -> subsample_clouds_points_tensors ->
    detect_batch_select_tensors: no sample index is a final inlier, and every table pixel's point is one. A blank view
    (an empty cloud) fails its fit and draws nothing."""
    torch = torch_()
    views = dr.render_views([51, 52, 53], [2, 1, 1], 0)
    blank = dr.default_cameras(1, width=32, height=24, f=40.0)[0]
    ks = [len(v) for v in views]
    cams = [c for v in views for _, c in v]
    ks.append(1)
    cams.append(blank)
    depth = np.concatenate([np.asarray(img).ravel() for v in views for img, _ in v] + [np.zeros(24 * 32, np.uint16)])
    depth = depth.view(np.int16)
    ctx = context(weights=True)
    poff = ctx.preprocess_depth_tensors(ks, cams, torch.from_numpy(depth).cuda(), lib.preprocess_params())
    seg = ctx.segment_planes_tensors()
    elig = seg["eligible"]
    soff, idx = ctx.subsample_clouds_points_tensors(60, 8, elig)
    rec, roff = ctx.detect_batch_select_tensors(soff, idx, 10)
    assert roff[-1] > 0
    e, ix = elig.cpu().numpy(), idx.cpu().numpy()
    clouds = ctx.get_clouds()
    assert poff[-1] == poff[-2] and np.isnan(seg["planes"][-1]).all() and seg["n_hypotheses"][-1] == 0
    assert soff[-1] == soff[-2]
    for b in range(len(views)):
        assert seg["n_inliers"][b] > 0 and 0 < (e[poff[b]:poff[b + 1]] == 0).sum() < poff[b + 1] - poff[b]
        assert (e[poff[b] + ix[soff[b]:soff[b + 1]]] == 1).all()
        z = clouds[b]["xyz"][:, 2]
        ref = pr.segment(clouds[b]["xyz"], key=b)
        assert seg["n_hypotheses"][b] == ref["n_hypotheses"]
        assert (e[poff[b]:poff[b + 1]][np.abs(z - np.median(z[z > 0.89])) < 0.004] == 0).all()
    ctx.close()


def test_errors_and_state():
    torch = torch_()
    ctx = context()
    with pytest.raises(lib.GpdbError) as ei:
        ctx.segment_plane()
    assert ei.value.code == ERR_STATE
    with pytest.raises(lib.GpdbError) as ei:
        ctx.segment_planes()
    assert ei.value.code == ERR_STATE
    with pytest.raises(lib.GpdbError) as ei:
        ctx.subsample_clouds_points(5, 0)
    assert ei.value.code == ERR_STATE
    x = scenes.synthetic_table_scene(5, n_points=8000)["xyz"]
    ctx.set_clouds([cloud(x)])
    c0 = cloud(x)
    ctx.set_cloud(c0["xyz"], c0["normals"])
    bad = [dict(distance_threshold=0.0), dict(distance_threshold=-0.01), dict(distance_threshold=float("nan")),
           dict(distance_threshold=float("inf")), dict(max_iterations=0), dict(max_iterations=1025),
           dict(probability=0.0), dict(probability=1.0), dict(probability=float("nan"))]
    for over in bad:
        for fn in (ctx.segment_plane, ctx.segment_planes, ctx.segment_planes_tensors):
            with pytest.raises(lib.GpdbError) as ei:
                fn(lib.plane_params(**over))
            assert ei.value.code == ERR_INVALID, over
    # a host pointer where device memory is required
    host = np.zeros(len(x), np.uint8)
    planes, cnt = np.zeros(4, F), np.zeros(1, np.int32)
    rc = lib.lib().gpdb_segment_planes_device(ctx.h, C.byref(lib.plane_params()), planes.ctypes.data_as(C.c_void_p),
                                              cnt.ctypes.data_as(C.c_void_p), None, host.ctypes.data_as(C.c_void_p))
    assert rc == ERR_INVALID and b"d_eligible_out" in lib.lib().gpdb_last_error(ctx.h)
    rc = lib.lib().gpdb_subsample_clouds_points_device(ctx.h, 5, 0, host.ctypes.data_as(C.c_void_p), None,
                                                       np.zeros(2, np.int32).ctypes.data_as(C.c_void_p))
    assert rc == ERR_INVALID
    # the calls still work afterwards
    r = ctx.segment_planes()
    assert r["n_inliers"][0] > 0
    ctx.close()
