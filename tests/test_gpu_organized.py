"""gpdb_normals_organized[_device] and gpdb_preprocess_depth_organized[_device] on the H100 against the restatements of
include/gpd_b200_organized.h. The standalone call: mixed-size batches (rendered depth images as organized clouds, the
wrap reads of the distance passes, the 40 x 40 / 41 x 41 border edge, an image smaller than the border, a full-size
640 x 480 render), the host and device twins, and the argument checks. The depth call: everything but the normals equal
to gpdb_preprocess_depth, the normals by rule 7 (organized ones as the restatement, fallbacks as the radius estimate),
the fallback counts, the twins, a failed call, a non-orthonormal R, and a hand search equal to one after set_clouds.

The restatements take pcl::eigen33 from the oracle, whose atan2f / cosf / sinf are glibc's; the device evaluates them in
float64 and rounds (DESIGN.md 4b). Where the two roundings differ the eigenvector moves by a few float32 ulps, so the
normals are compared bit for bit in their NaN positions and on all but a small share of pixels, and within 1e-5 (per
component) on the rest; the distance maps, which involve no libm call, bit for bit everywhere."""
import numpy as np
import pytest

import depth_reference as dr
import organized_reference as orf
from gpd_b200 import lib

pytestmark = pytest.mark.gpu
F = np.float32


def assert_normals(got, ref):
    """NaN positions equal, values bit-equal on >= 95 % of the finite entries and within 1e-5 on the others (about 1.5 % of
    the pixels of the rendered scenes differ, by at most 4e-7)."""
    got, ref = np.asarray(got), np.asarray(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    fin = ~np.isnan(ref)
    diff = got[fin] != ref[fin]
    assert diff.sum() <= 0.05 * max(fin.sum(), 1)
    assert np.all(np.abs(got[fin].astype(np.float64) - ref[fin]) <= 1e-5)


@pytest.fixture(scope="module")
def ctx():
    c = lib.Context(lib.default_params())
    yield c
    c.close()


def _clouds():
    """Mixed sizes: two renders, a 41 x 41 and a 40 x 40 plane with a hole, a tiny image and a full-size render."""
    out = []
    for seed, (w, h) in [(1, (160, 120)), (2, (97, 64))]:
        v = dr.render_views([seed], [1], 0, width=w, height=h, f=1.2 * w)[0][0]
        out.append(orf.camera_cloud(v[0], v[1], 0))
    from test_organized_reference import plane
    p = plane(41, 41)
    p[25, 22] = np.nan
    wrap = plane(50, 60)
    wrap[10, 0] = np.nan  # pass 1 reads element 0 of row 10 as the upper right of (10, 59)
    wrap[30, 59] = np.nan  # pass 2 reads element 59 of row 30 as the lower left of (30, 0)
    out += [p, plane(40, 40), plane(3, 7), wrap]
    v = dr.render_views([3], [1], 1, n_points=200000, width=640, height=480, f=520.0)[0][0]
    out.append(orf.camera_cloud(v[0], v[1], 1))
    return out  # the full-size render stays last


def test_normals_organized_bit_equal_to_the_restatement(ctx):
    clouds = _clouds()
    vps = np.array([[0, 0, 0], [0.1, -0.2, 0.05], [0, 0, -1], [0, 0, 0], [0, 0, 0], [0, 0, 0], [0.3, 0.0, 0.0]], F)
    ns, ds = ctx.normals_organized(clouds, vps)
    for xyz, vp, n, d in zip(clouds, vps, ns, ds):
        rn, rd = orf.cpp_normals(xyz, vp)
        assert np.array_equal(d, rd)
        assert_normals(n, rn)
    assert np.isfinite(ns[0][..., 0]).sum() > 100 and np.isfinite(ns[-1][..., 0]).sum() > 1000
    assert ds[5][10, 59] == F(1.4) and ds[5][30, 0] == F(1.4)  # the wrap reads took effect on the device


def test_normals_organized_device_twin(ctx):
    import torch
    clouds = _clouds()
    ns, ds = ctx.normals_organized(clouds)
    ts = [torch.from_numpy(c).cuda() for c in clouds]
    tn, td = ctx.normals_organized_tensors(ts)
    for a, b, c, d in zip(ns, tn, ds, td):
        assert np.array_equal(a, b.cpu().numpy(), equal_nan=True) and np.array_equal(c, d.cpu().numpy())
    tn2, td2 = ctx.normals_organized_tensors(ts[:1], distance=False)
    assert td2[0] is None and np.array_equal(ns[0], tn2[0].cpu().numpy(), equal_nan=True)


def test_normals_organized_argument_errors(ctx):
    L = lib.lib()
    assert L.gpdb_normals_organized(ctx.h, 0, None, None, None, None, None, None) == -1
    W, H = np.array([0], np.int32), np.array([5], np.int32)
    buf = np.zeros(16, F)
    assert L.gpdb_normals_organized(ctx.h, 1, lib._p(W), lib._p(H), lib._p(buf), lib._p(buf), lib._p(buf), None) == -1
    assert b"width and height" in L.gpdb_last_error(ctx.h)


def _views(K, fmt, n_views=2, pose_scale=None):
    views = dr.render_views(list(range(11, 11 + n_views)), [K] * n_views, fmt, width=160, height=120, f=190.0)
    if pose_scale is not None:  # a non-orthonormal R: the first column scaled
        for view in views:
            for _, cam in view:
                for i in range(3):
                    cam.pose[4 * i] *= pose_scale
    return views


def _expected(clouds, views, fmt, radius_normals):
    """Rule 7 from the C++ restatement: (normals per view, fallback counts [B])."""
    out, cnt = [], []
    for view, cl, rn in zip(views, clouds, radius_normals):
        cams = [c for _, c in view]
        per_cam = [orf.rotate(np.array(c.pose[:]).reshape(3, 4)[:, :3], orf.cpp_normals(orf.camera_cloud(img, c, fmt))[0])
                   for img, c in view]
        starts = np.cumsum([0] + [c.width * c.height for c in cams])
        vps = np.array([[c.pose[3], c.pose[7], c.pose[11]] for c in cams])
        nrm, n_fb = np.array(rn, copy=True), 0
        for j, (src, q, cm) in enumerate(zip(cl["src"], cl["xyz"], cl["cam_source"])):
            k = int(np.searchsorted(starts, src, side="right") - 1)
            n = per_cam[k].reshape(-1, 3)[src - starts[k]]
            if not np.all(np.isfinite(n)):
                n_fb += 1
                continue
            nd = n.astype(np.float64)
            rev = True
            for kk in range(len(cams)):
                if cm[kk]:
                    d = q.astype(np.float64) - vps[kk]
                    if (nd[0] * d[0] + nd[1] * d[1]) + nd[2] * d[2] < 0:
                        rev = False
                        break
            nrm[j] = -nd if rev else nd
        out.append(nrm)
        cnt.append(n_fb)
    return out, np.array(cnt)


@pytest.mark.parametrize("K,fmt,voxelize", [(1, 0, 1), (1, 1, 0), (2, 0, 0), (2, 1, 1), (8, 0, 1), (8, 1, 0)])
def test_preprocess_depth_organized_follows_rule_7(ctx, K, fmt, voxelize):
    views = _views(K, fmt, n_views=2 if K < 8 else 1)
    pp = lib.preprocess_params(voxelize=voxelize)
    ref = ctx.preprocess_depth(views, pp)
    got, fb = ctx.preprocess_depth_organized(views, pp)
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        for key in ("xyz", "cam_source", "src", "view_points"):
            assert np.array_equal(g[key], r[key]), key
    exp, cnt = _expected(got, views, fmt, [r["normals"] for r in ref])
    assert np.array_equal(fb, cnt)
    assert 0 < cnt.sum() < sum(len(g["xyz"]) for g in got)
    for g, e in zip(got, exp):
        assert_normals(g["normals"], e)


def test_preprocess_depth_organized_device_twin(ctx):
    import torch
    views = _views(2, 0)
    pp = lib.preprocess_params()
    host, fb = ctx.preprocess_depth_organized(views, pp)
    depth = torch.from_numpy(np.concatenate([img.ravel() for v in views for img, _ in v]).view(np.int16)).cuda()
    off, fb2 = ctx.preprocess_depth_organized_tensors([len(v) for v in views], [c for v in views for _, c in v], depth, pp)
    dev = ctx.get_clouds()
    assert np.array_equal(fb, fb2)
    for a, b in zip(host, dev):  # radius estimates of points with fewer than 3 neighbours are NaN in both
        for key in ("xyz", "normals", "cam_source", "src"):
            assert np.array_equal(a[key], b[key], equal_nan=True), key


def test_preprocess_depth_organized_failure_leaves_no_batch(ctx):
    views = _views(1, 0)
    ctx.preprocess_depth_organized(views)
    with pytest.raises(lib.GpdbError):
        ctx.preprocess_depth_organized(views, lib.preprocess_params(normals_radius=0.0))
    with pytest.raises(lib.GpdbError):
        ctx.subsample_clouds(10, 0)
    with pytest.raises(lib.GpdbError):
        ctx.preprocess_depth_organized(views, lib.preprocess_params(estimate_normals=0))
    with pytest.raises(lib.GpdbError):
        ctx.get_clouds()


def test_detect_path_equals_set_clouds_and_non_orthonormal_flag(ctx):
    """A batch from the organized call searches hands as the same points and normals installed by set_clouds do. With a
    scaled R the rotated normals are not of unit length; the install then sets the nonunit flag as set_clouds does, so
    the two still agree."""
    for scale in (None, 1.5):
        views = _views(1, 0, n_views=1, pose_scale=scale)
        got, _ = ctx.preprocess_depth_organized(views)
        sidx = [np.arange(0, len(got[0]["xyz"]), max(1, len(got[0]["xyz"]) // 24), dtype=np.int32)]
        a = ctx.hand_search_batch(sidx)
        cl = dict(got[0])
        del cl["src"]
        ctx.set_clouds([cl])
        b = ctx.hand_search_batch(sidx)
        assert np.array_equal(a[0]["pose_flags"], b[0]["pose_flags"])
        assert np.array_equal(a[0]["frames"], b[0]["frames"], equal_nan=True)
        ln = np.linalg.norm(cl["normals"], axis=1)
        assert np.any(np.abs(ln - 1.0) > 1e-3) == (scale is not None)
