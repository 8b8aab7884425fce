"""Depth images to grasps on the device: gpdb_preprocess_depth[_device] and gpdb_subsample_clouds[_device].

The oracle of the depth front is gpdb_preprocess_clouds on the raw cloud that include/gpd_b200_depth.h defines (built in
numpy by tests/depth_reference.py), bit for bit; the oracle of the sampling is the numpy restatement of its rule. Host and
device twins must agree exactly, also on a side stream, and the sampled indices must feed the batch calls as host lists do.
"""
import numpy as np
import pytest

import depth_reference as dr
from conftest import load_weights
from gpd_b200 import abi, lib

pytestmark = pytest.mark.gpu
ERR_INVALID, ERR_STATE = -1, -3


def torch_():
    return pytest.importorskip("torch")


def context(weights=False):
    w, relu = load_weights(12)
    ctx = lib.Context(lib.default_params(channels=12, relu_after_conv=relu))
    if weights:
        ctx.set_weights(w)
    return ctx


def dev(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        a = a.view(np.int16)  # the same bits; preprocess_depth_tensors reads int16 as uint16
    return torch_().from_numpy(a).cuda()


def flat(views):
    ks = [len(v) for v in views]
    cams = [c for v in views for _, c in v]
    depth = np.concatenate([np.asarray(img).ravel() for v in views for img, _ in v])
    return ks, cams, depth


def via_clouds(ctx, views, fmt, pp):
    """preprocess_clouds_tensors on the raw clouds of the specification; returns (offsets, clouds, raw offsets)."""
    raws = [dr.raw_cloud(v, fmt) for v in views]
    off = np.zeros(len(raws) + 1, np.int32)
    off[1:] = np.cumsum([len(r["xyz"]) for r in raws])
    xyz = np.concatenate([r["xyz"] for r in raws])
    cam = np.concatenate([r["cam_source"].ravel() for r in raws])
    ks = np.array([len(v) for v in views], np.int32)
    vps = np.concatenate([r["view_points"] for r in raws])
    poff = ctx.preprocess_clouds_tensors(off, dev(xyz), ks, vps, cam_source=dev(cam), pp=pp)
    return poff.copy(), ctx.get_clouds(), off


def via_depth(ctx, views, fmt, pp):
    ks, cams, depth = flat(views)
    poff = ctx.preprocess_depth_tensors(ks, cams, dev(depth), pp)
    return poff.copy(), ctx.get_clouds()


def assert_same_clouds(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(x["xyz"].view(np.uint32), y["xyz"].view(np.uint32))
        assert np.array_equal(x["normals"].view(np.uint64), y["normals"].view(np.uint64))
        assert np.array_equal(x["cam_source"], y["cam_source"])
        assert np.array_equal(x["src"], y["src"])
        assert np.array_equal(x["view_points"], y["view_points"])


def damage(views, fmt, seed):
    """Pixels with no return or out of range in every image: 0, and for float32 NaN, +-inf and negative values too; the
    cameras get min_depth 0.6 and max_depth 1.0 m, so the far table edge and anything nearer than 0.6 m drop out."""
    rng = np.random.default_rng(seed)
    out = []
    for v in views:
        nv = []
        for img, c in v:
            img = img.copy()
            f = img.reshape(-1)
            idx = rng.choice(f.size, f.size // 10, replace=False)
            bad = [0] if fmt == 0 else [0.0, np.nan, np.inf, -np.inf, -0.5]
            f[idx] = np.array(bad, dtype=img.dtype)[np.arange(len(idx)) % len(bad)]
            near = rng.choice(f.size, 40, replace=False)  # valid returns outside [min, max]
            f[near[:20]] = 0.3 / c.depth_scale
            f[near[20:]] = 1.5 / c.depth_scale
            c2 = lib.depth_camera(c.width, c.height, c.fx, c.fy, c.cx, c.cy, np.array(c.pose[:]).reshape(3, 4),
                                  c.depth_scale, 0.6, 1.0)
            nv.append((img, c2))
        out.append(nv)
    return out


def mixed_views(fmt, seed=0):
    scale = 0.001 if fmt == 0 else 1.0
    views = (dr.render_views([seed + 1], [1], fmt, scale=scale, width=120, height=90)
             + dr.render_views([seed + 2], [2], fmt, scale=scale, width=100, height=80, f=125.0)
             + dr.render_views([seed + 3], [3], fmt, scale=scale, width=64, height=48, f=80.0))
    views = damage(views, fmt, seed)
    # a view whose only camera sees nothing valid
    c = dr.default_cameras(1, width=32, height=24, f=40.0, scale=scale)[0]
    views.insert(2, [(np.zeros((24, 32), np.uint16 if fmt == 0 else np.float32), c)])
    return views


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("voxelize", [0, 1])
def test_depth_equals_preprocess_clouds_on_the_raw_cloud(fmt, voxelize):
    views = mixed_views(fmt, seed=10 * fmt + voxelize)
    for pp in (lib.preprocess_params(voxelize=voxelize),
               lib.preprocess_params(voxelize=voxelize, workspace=[-0.3, 0.35, -0.25, 0.3, 0.5, 1.05], voxel_size=0.004,
                                     normals_radius=0.02)):
        ctx = context()
        p_ref, ref, _ = via_clouds(ctx, views, fmt, pp)
        p_dep, got = via_depth(ctx, views, fmt, pp)
        assert np.array_equal(p_ref, p_dep)
        assert p_dep[3] == p_dep[2]  # the view without a valid pixel stays, with no points
        assert all(p_dep[b + 1] > p_dep[b] for b in (0, 1, 3))
        assert_same_clouds(ref, got)
        ctx.close()


@pytest.mark.parametrize("fmt", [0, 1])
def test_kernel_arithmetic_alone(fmt):
    views = mixed_views(fmt, seed=3)
    pp = lib.preprocess_params(voxelize=0, workspace=[-10, 10, -10, 10, -10, 10])
    ctx = context()
    _, got = via_depth(ctx, views, fmt, pp)
    for v, cl in zip(views, got):
        pts = np.concatenate([dr.back_project(img, c, fmt) for img, c in v])
        ok = np.flatnonzero(np.all(np.isfinite(pts), axis=1))
        assert np.array_equal(cl["src"], ok)
        assert np.array_equal(cl["xyz"].view(np.uint32), pts[ok].view(np.uint32))
    ctx.close()


def test_host_and_device_twins_are_identical_also_on_a_side_stream():
    torch = torch_()
    for fmt in (0, 1):
        views = mixed_views(fmt, seed=5)
        pp = lib.preprocess_params()
        ks, cams, depth = flat(views)
        ctx = context()
        h = ctx.preprocess_depth(views, pp)
        p_h = ctx._batch[0].copy()
        n_raw = len(depth)
        mask = (np.random.default_rng(1).random(n_raw) < 0.5).astype(np.uint8)
        s_h = [ctx.subsample_clouds(k, 77, m) for k in (0, 40) for m in (None, mask)]
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            d_depth = dev(depth)
            d_mask = dev(mask)
            p_d = ctx.preprocess_depth_tensors(ks, cams, d_depth, pp)
            s_d = [ctx.subsample_clouds_tensors(k, 77, m) for k in (0, 40) for m in (None, d_mask)]
        torch.cuda.synchronize()
        assert np.array_equal(p_h, p_d)
        assert_same_clouds(h, ctx.get_clouds())
        for lists, (soff, idx) in zip(s_h, s_d):
            idx = idx.cpu().numpy()
            assert all(np.array_equal(lists[b], idx[soff[b]:soff[b + 1]]) for b in range(len(lists)))
        ctx.close()


def test_sampling_equals_the_specification():
    torch_()
    views = mixed_views(0, seed=7)
    pp = lib.preprocess_params()
    ctx = context()
    _, cl, roff = via_clouds(ctx, views, 0, pp)  # preprocess_clouds keeps its raw offsets too
    poff, cl2 = via_depth(ctx, views, 0, pp)
    assert np.array_equal(roff, np.concatenate([[0], np.cumsum([sum(i.size for i, _ in v) for v in views])]))
    src = np.concatenate([c["src"] for c in cl2])
    mask = (np.random.default_rng(2).random(roff[-1]) < 0.3).astype(np.uint8)
    npts = np.diff(poff)
    assert npts[2] == 0
    for k in (0, 1, 25, int(npts.max()) + 1):
        for m in (None, mask):
            soff, idx = ctx.subsample_clouds_tensors(k, 123456789012, None if m is None else dev(m))
            want = dr.subsample_batch(poff, k, 123456789012, src, roff, m)
            idx = idx.cpu().numpy()
            assert soff[-1] == sum(len(w) for w in want)
            for b, w in enumerate(want):
                assert np.array_equal(idx[soff[b]:soff[b + 1]], w), (k, m is None, b)
    # after set_clouds_tensors there are no source indices: a mask is a state error, no mask is fine
    ctx.set_clouds_tensors(np.array([0, len(cl2[0]["xyz"])], np.int32), dev(cl2[0]["xyz"]), dev(cl2[0]["normals"]),
                           [len(views[0])], cl2[0]["view_points"])
    with pytest.raises(lib.GpdbError) as e:
        ctx.subsample_clouds_tensors(5, 1, dev(mask[:10]))
    assert e.value.code == ERR_STATE and "gpdb_set_clouds" in str(e.value)
    soff, idx = ctx.subsample_clouds_tensors(5, 1)
    assert np.array_equal(idx.cpu().numpy(), dr.subsample(len(cl2[0]["xyz"]), 5, 1, 0))
    with pytest.raises(lib.GpdbError) as e:
        ctx.subsample_clouds_tensors(-1, 1)
    assert e.value.code == ERR_INVALID
    ctx.close()


def test_sampled_indices_feed_select_and_sis_as_host_lists_do():
    views = dr.render_views([21, 22], [2, 1], 0)
    ctx = context(weights=True)
    ks, cams, depth = flat(views)
    ctx.preprocess_depth_tensors(ks, cams, dev(depth), lib.preprocess_params())
    soff, idx = ctx.subsample_clouds_tensors(30, 5)
    lists = [idx.cpu().numpy()[soff[b]:soff[b + 1]] for b in range(len(views))]
    rec, roff = ctx.detect_batch_select_tensors(soff, idx, 10)
    host = ctx.detect_batch_select(lists, 10)
    recs = lib.poses_from_tensor(rec)
    for b in range(len(views)):
        assert recs[roff[b]:roff[b + 1]].tobytes() == host[b].tobytes()
    sis = dict(num_iterations=2, num_samples_per_iteration=10, seed=3)
    srec, shoff, _ = ctx.sis_batch_tensors(soff, idx, **sis)
    shost = ctx.sis_batch(lists, **sis)["hands"]
    srecs = lib.poses_from_tensor(srec)
    for b in range(len(views)):
        assert srecs[shoff[b]:shoff[b + 1]].tobytes() == shost[b].tobytes()
    ctx.close()


def test_argument_errors_name_the_view_and_camera_and_leave_no_batch():
    views = dr.render_views([31, 32], [1, 2], 0, width=40, height=30, f=50.0)
    ks, cams, depth = flat(views)
    pp = lib.preprocess_params()
    ctx = context()

    def cam(k, **over):
        c = cams[k]
        kw = dict(width=c.width, height=c.height, fx=c.fx, fy=c.fy, cx=c.cx, cy=c.cy, pose=np.array(c.pose[:]).reshape(3, 4),
                  depth_scale=c.depth_scale, min_depth=c.min_depth, max_depth=c.max_depth)
        kw.update(over)
        return lib.depth_camera(**kw)

    bad_pose = np.array(cams[2].pose[:]).reshape(3, 4)
    bad_pose[1, 3] = np.nan
    cases = [(dict(fx=0.0), "fx and fy"), (dict(fy=-1.0), "fx and fy"), (dict(cx=np.inf), "non-finite"),
             (dict(pose=bad_pose), "non-finite"), (dict(depth_scale=0.0), "depth_scale"), (dict(min_depth=-0.1), "min_depth"),
             (dict(min_depth=1.0, max_depth=1.0), "max_depth"), (dict(width=0), "width and height"),
             (dict(height=0), "width and height")]
    for d_call in (False, True):
        for over, words in cases:
            ctx.preprocess_depth_tensors(ks, cams, dev(depth), pp)  # a batch to lose
            cs = cams[:2] + [cam(2, **over)]
            with pytest.raises(lib.GpdbError) as e:
                if d_call:
                    ctx._install_depth(lib.lib().gpdb_preprocess_depth_device, ks, cs, 0, dev(depth).data_ptr(), pp)
                else:
                    ctx._install_depth(lib.lib().gpdb_preprocess_depth, ks, cs, 0, depth.ctypes.data, pp)
            assert e.value.code == ERR_INVALID and "view 1 camera 1" in str(e.value) and words in str(e.value), str(e.value)
            with pytest.raises(lib.GpdbError) as e:
                ctx._check(lib.lib().gpdb_get_clouds(ctx.h, None, None, None, None))
            assert e.value.code == ERR_STATE
    for ks_bad in ([0, 3], [1, 9]):
        with pytest.raises(lib.GpdbError) as e:
            n = sum(ks_bad)
            ctx._install_depth(lib.lib().gpdb_preprocess_depth, ks_bad, (cams * 4)[:n], 0, depth.ctypes.data, pp)
        assert e.value.code == ERR_INVALID and "view" in str(e.value) and "cameras" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx._install_depth(lib.lib().gpdb_preprocess_depth, ks, cams, 2, depth.ctypes.data, pp)
    assert e.value.code == ERR_INVALID and "format" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx.preprocess_depth_tensors(ks, cams, dev(depth), lib.preprocess_params(estimate_normals=0))
    assert e.value.code == ERR_INVALID and "estimate_normals" in str(e.value)
    # 2^31 pixels: refused from the sizes alone, before anything is allocated or read (the buffers are tiny)
    huge = [lib.depth_camera(65536, 16384, 100, 100, 1, 1), lib.depth_camera(65536, 16384, 100, 100, 1, 1)]
    tiny = np.zeros(4, np.uint16)
    with pytest.raises(lib.GpdbError) as e:
        ctx._install_depth(lib.lib().gpdb_preprocess_depth, [2], huge, 0, tiny.ctypes.data, pp)
    assert e.value.code == ERR_INVALID and "2^31" in str(e.value) and "view 0 camera 1" in str(e.value)
    with pytest.raises(lib.GpdbError) as e:
        ctx._install_depth(lib.lib().gpdb_preprocess_depth_device, [2], huge, 0, dev(tiny).data_ptr(), pp)
    assert e.value.code == ERR_INVALID and "2^31" in str(e.value)
    # a host pointer as d_depth
    with pytest.raises(lib.GpdbError) as e:
        ctx._install_depth(lib.lib().gpdb_preprocess_depth_device, ks, cams, 0, depth.ctypes.data, pp)
    assert e.value.code == ERR_INVALID and "d_depth" in str(e.value)
    # no batch: the sampling is a state error
    with pytest.raises(lib.GpdbError) as e:
        ctx.subsample_clouds(5, 0)
    assert e.value.code == ERR_STATE
    ctx.close()


def test_depth_to_clustered_grasps_on_the_device():
    """Rendered views -> preprocess_depth -> subsample above the table -> select -> cluster; every selected grasp sits on
    a pixel of the mask."""
    views = dr.render_views([41, 42, 43], [2, 2, 1], 0)
    ks, cams, depth = flat(views)
    ctx = context(weights=True)
    poff = ctx.preprocess_depth_tensors(ks, cams, dev(depth), lib.preprocess_params())
    raw = np.concatenate([dr.raw_cloud(v, 0)["xyz"] for v in views])
    with np.errstate(invalid="ignore"):
        mask = (raw[:, 2] < 0.88).astype(np.uint8)  # the table lies at z ~ 0.9: the objects on it
    soff, idx = ctx.subsample_clouds_tensors(80, 11, dev(mask))
    rec, roff = ctx.detect_batch_select_tensors(soff, idx, 20)
    clusters, coff = ctx.find_clusters_batch_tensors(roff, rec, 1)
    assert roff[-1] > 0 and coff[-1] > 0
    recs = lib.poses_from_tensor(rec)
    idx = idx.cpu().numpy()
    clouds = ctx.get_clouds()
    roffs = np.concatenate([[0], np.cumsum([sum(i.size for i, _ in v) for v in views])])
    for b in range(len(views)):
        for r in recs[roff[b]:roff[b + 1]]:
            j = idx[soff[b] + r["sample_slot"]]
            assert mask[roffs[b] + clouds[b]["src"][j]] == 1
    assert poff[-1] == sum(len(c["xyz"]) for c in clouds)
    assert lib.poses_from_tensor(clusters).dtype == abi.POSE_DTYPE
    ctx.close()
