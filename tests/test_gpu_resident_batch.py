"""Device-resident batches (gpdb_preprocess_clouds_device, gpdb_set_clouds_device, gpdb_detect_batch_select_device,
gpdb_find_clusters_batch_device) through the tensor methods of lib.Context, on the GPU.

The oracle of every device route is its host route on the same seeded inputs, bit for bit: the processed clouds
(gpdb_get_clouds points, normals, camera sources, source indices), the selected records with their offsets, and the
clusters. The errors must be the host twin's (code and message, up to the entry point's name) and leave the single cloud
intact; a failed install leaves no batch.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import load_weights
from gpd_b200 import abi, lib, scenes

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

ERR_INVALID = -1
K3 = [(0.0, 0.0, 0.0), (0.3, 0.0, 0.0), (-0.3, 0.1, 0.0)]
K8 = [(-0.3, -0.2, 0.0), (0.0, -0.2, 0.0), (0.3, -0.2, 0.0), (-0.3, 0.2, 0.0), (0.0, 0.2, 0.0), (0.3, 0.2, 0.0),
      (0.0, 0.0, 0.0), (0.15, 0.0, 0.1)]


def context(**over):
    """12-channel images: the 15-channel shadow bitmaps of 8 cameras would not fit one CTA's shared memory."""
    w, relu = load_weights(12)
    ctx = lib.Context(lib.default_params(channels=12, relu_after_conv=relu, **over))
    ctx.set_weights(w)
    return ctx


def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def raw_view(seed, n=12000, cameras=None, shift=0.0, with_cam=True, with_normals=False):
    s = scenes.synthetic_raw_scene(seed, n_points=n, cameras=cameras, mark_all_cameras=cameras is not None)
    xyz = (s["xyz"] + np.float32([shift, 0.0, 0.0])).astype(np.float32)
    v = {"xyz": xyz, "cam_source": s["cam_source"] if with_cam else None, "view_points": s["view_points"], "normals": None}
    if with_normals:
        nrm = np.random.default_rng(seed).normal(size=(len(xyz), 3))
        v["normals"] = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    return v


def mixed_views(with_cam=True, with_normals=False):
    """K_b = 1, 3, 8 and 3 again, the third lying 5 m outside the workspace (the filter empties it)."""
    kw = dict(with_cam=with_cam, with_normals=with_normals)
    return [raw_view(21, **kw), raw_view(22, cameras=K3, **kw), raw_view(23, n=6000, shift=5.0, **kw),
            raw_view(24, cameras=K8, **kw), raw_view(25, cameras=K3, n=8000, **kw)]


def preprocess_device(ctx, views, pp):
    pk = lib.pack_clouds(views)
    return ctx.preprocess_clouds_tensors(pk["offsets"], dev(pk["xyz"]), pk["n_cameras"], pk["view_points"],
                                         cam_source=dev(pk["cam_source"]), normals=dev(pk["normals"]), pp=pp)


def assert_clouds_equal(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x["xyz"].tobytes() == y["xyz"].tobytes()
        assert x["normals"].tobytes() == y["normals"].tobytes()
        assert x["cam_source"].shape == y["cam_source"].shape and np.array_equal(x["cam_source"], y["cam_source"])
        assert ("src" in x) == ("src" in y)
        if "src" in x:
            assert np.array_equal(x["src"], y["src"])


def samples_for(n_points, seed, per_cloud=60, positions=None):
    out = []
    for b, n in enumerate(n_points):
        rng = np.random.default_rng(seed + b)
        s = rng.choice(n, min(per_cloud, n), replace=False) if n else np.zeros(0, np.int64)
        if positions is not None and len(positions[b]):
            s = rng.permutation(np.concatenate([s, n + np.arange(len(positions[b]))]))
        out.append(np.asarray(s, np.int32))
    return out


def select_both(ctx, samples, k):
    """(host records per cloud, device records per cloud, device offsets) of the installed batch."""
    host = ctx.detect_batch_select(samples, k)
    offsets, sidx = lib.pack_samples(samples)
    rec, soff = ctx.detect_batch_select_tensors(offsets, dev(sidx), k)
    assert rec.is_cuda and rec.dtype == torch.uint8 and rec.shape[1] == lib.POSE_BYTES
    got = lib.poses_from_tensor(rec)
    assert np.array_equal(np.diff(soff), [len(h) for h in host])
    assert got.tobytes() == b"".join(h.tobytes() for h in host)
    return host, rec, soff


def clusters_both(ctx, host_sel, rec, soff, min_inliers=1):
    host = ctx.find_clusters_batch(host_sel, min_inliers)
    cl, coff = ctx.find_clusters_batch_tensors(soff, rec, min_inliers)
    assert cl.is_cuda and np.array_equal(np.diff(coff), [len(h) for h in host])
    assert lib.poses_from_tensor(cl).tobytes() == b"".join(h.tobytes() for h in host)
    return host


def has_batch(ctx):
    return lib.lib().gpdb_get_clouds(ctx.h, None, None, None, None) >= 0


def detect_route(ctx, views, pp, k=10, seed=0):
    """preprocess -> select -> cluster, host route then device route; returns (processed clouds, selections, clusters)."""
    host_clouds = ctx.preprocess_clouds(views, pp)
    n = [len(c["xyz"]) for c in host_clouds]
    samples = samples_for(n, seed)
    host_sel = ctx.detect_batch_select(samples, k)
    host_cl = ctx.find_clusters_batch(host_sel, 1)
    poff = preprocess_device(ctx, views, pp)
    assert np.array_equal(np.diff(poff), n)
    assert_clouds_equal(ctx.get_clouds(), host_clouds)
    sel, rec, soff = select_both(ctx, samples, k)
    for a, b in zip(sel, host_sel):
        assert a.tobytes() == b.tobytes()
    cl = clusters_both(ctx, sel, rec, soff)
    for a, b in zip(cl, host_cl):
        assert a.tobytes() == b.tobytes()
    return host_clouds, sel, cl


@pytest.mark.parametrize("with_cam", [True, False], ids=["cam_source", "no_cam_source"])
@pytest.mark.parametrize("estimate_normals", [1, 0])
def test_raw_views_device_route_equals_host_route(with_cam, estimate_normals):
    ctx = context()
    views = mixed_views(with_cam=with_cam, with_normals=not estimate_normals)
    clouds, sel, cl = detect_route(ctx, views, lib.preprocess_params(estimate_normals=estimate_normals))
    assert len(clouds[2]["xyz"]) == 0 and len(sel[2]) == 0  # the emptied view stays, with no points
    assert [c["cam_source"].shape[1] for c in clouds] == [1, 3, 1, 8, 3]
    assert sum(len(s) for s in sel) > 0 and sum(len(c) for c in cl) > 0
    ctx.close()


def test_without_voxelisation_and_straddling_chunks():
    """voxelize = 0, and chunks of 37 samples, so that most chunks hold samples of two clouds."""
    ctx = context(chunk_samples=37)
    views = mixed_views()
    clouds, sel, _ = detect_route(ctx, views, lib.preprocess_params(voxelize=0), k=25, seed=7)
    assert len(clouds[0]["xyz"]) > 1000 and sum(len(s) for s in sel) > 0
    ctx.close()


def test_single_view_batch():
    ctx = context()
    _, sel, _ = detect_route(ctx, [raw_view(31, cameras=K3)], lib.preprocess_params(), k=50)
    assert len(sel) == 1 and len(sel[0]) == 50
    ctx.close()


def processed_tables():
    return [scenes.synthetic_table_scene(41, n_points=15000), scenes.synthetic_table_scene(42, n_points=9000, cameras=K3),
            scenes.synthetic_table_scene(43, n_points=12000, cameras=K8, mark_all_cameras=True),
            dict(scenes.synthetic_table_scene(44, n_points=8000), cam_source=None)]


def set_device(ctx, clouds):
    pk = lib.pack_clouds(clouds)
    ctx.set_clouds_tensors(pk["offsets"], dev(pk["xyz"]), dev(pk["normals"]), pk["n_cameras"], pk["view_points"],
                           cam_source=dev(pk["cam_source"]))


def test_installed_clouds_with_sample_positions():
    """set_clouds_tensors equals set_clouds, and sample indices addressing gpdb_set_clouds_samples positions select the
    same records on both routes."""
    ctx = context()
    clouds = processed_tables()
    ctx.set_clouds(clouds)
    host_clouds = ctx.get_clouds()
    set_device(ctx, clouds)
    assert_clouds_equal(ctx.get_clouds(), host_clouds)
    rng = np.random.default_rng(5)
    pos = [c["xyz"][rng.choice(len(c["xyz"]), m, replace=False)].astype(np.float64) + rng.normal(0, 0.002, (m, 3))
           for c, m in zip(clouds, (30, 0, 20, 12))]
    ctx.set_clouds_samples(pos)
    samples = samples_for([len(c["xyz"]) for c in clouds], 50, positions=pos)
    sel, rec, soff = select_both(ctx, samples, 30)
    assert any(np.any(s["sample_index"] >= len(c["xyz"])) for s, c in zip(sel, clouds))  # records at positions
    clusters_both(ctx, sel, rec, soff)
    ctx.close()


def single_cloud_check(ctx):
    k = scenes.krylon_cloud()
    ctx.set_cloud(k["xyz"], k["normals"], k["cam_source"], k["view_points"])
    sidx = scenes.sample_indices(1, len(k["xyz"]), 100)
    before = ctx.detect(sidx)
    return lambda: ctx.detect(sidx)["candidates"].tobytes() == before["candidates"].tobytes()


def refused(call):
    with pytest.raises(lib.GpdbError) as e:
        call()
    assert e.value.code == ERR_INVALID
    return str(e.value)


def test_errors_match_the_host_twins():
    ctx = context()
    intact = single_cloud_check(ctx)
    clouds = processed_tables()
    # a NaN coordinate in an install: the first bad point is named, no batch is left
    bad = [dict(c) for c in clouds]
    for b, i in ((1, 777), (3, 5)):
        bad[b]["xyz"] = bad[b]["xyz"].copy()
        bad[b]["xyz"][i, 1] = np.nan
    msg_h = refused(lambda: ctx.set_clouds(bad))
    set_device(ctx, clouds)
    msg_d = refused(lambda: set_device(ctx, bad))
    assert msg_d.replace("gpdb_set_clouds_device", "gpdb_set_clouds") == msg_h and f"point {15000 + 777} " in msg_h
    assert not has_batch(ctx) and intact()
    # cam_source value 2 without voxelisation
    views = mixed_views()
    views[3] = dict(views[3], cam_source=views[3]["cam_source"].copy())
    views[3]["cam_source"][100, 5] = 2
    pp = lib.preprocess_params(voxelize=0)
    msg_h = refused(lambda: ctx.preprocess_clouds(views, pp))
    preprocess_device(ctx, mixed_views(), pp)
    msg_d = refused(lambda: preprocess_device(ctx, views, pp))
    assert msg_d.replace("gpdb_preprocess_clouds_device", "gpdb_preprocess_clouds") == msg_h
    assert "cloud 3: cam_source[100][5] = 2" in msg_h
    assert not has_batch(ctx) and intact()
    # a host pointer as d_xyz: refused before any device work
    pk = lib.pack_clouds(clouds)
    nrm = dev(pk["normals"])
    rc = lib.lib().gpdb_set_clouds_device(ctx.h, len(clouds), lib._p(pk["offsets"]), lib._p(pk["xyz"]),
                                          C.c_void_p(nrm.data_ptr()), None, lib._p(pk["n_cameras"]), lib._p(pk["view_points"]))
    assert rc == ERR_INVALID and "d_xyz is not device memory" in lib.lib().gpdb_last_error(ctx.h).decode()
    assert not has_batch(ctx) and intact()
    # the tensor methods check device, dtype and size before the library sees the call
    with pytest.raises(ValueError):
        ctx.set_clouds_tensors(pk["offsets"], torch.from_numpy(pk["xyz"]), nrm, pk["n_cameras"], pk["view_points"])
    with pytest.raises(TypeError):
        ctx.set_clouds_tensors(pk["offsets"], dev(pk["xyz"]).double(), nrm, pk["n_cameras"], pk["view_points"])
    with pytest.raises(ValueError):
        ctx.set_clouds_tensors(pk["offsets"], dev(pk["xyz"])[:-1], nrm, pk["n_cameras"], pk["view_points"])
    # an index outside its cloud in a middle cloud: the message names the cloud and the position; the batch stays, as
    # after the host call
    ctx.set_clouds(clouds)
    n = [len(c["xyz"]) for c in clouds]
    samples = samples_for(n, 3)
    samples[2] = samples[2].copy()
    samples[2][17] = n[2]
    msg_h = refused(lambda: ctx.detect_batch_select(samples, 5))
    offsets, sidx = lib.pack_samples(samples)
    msg_d = refused(lambda: ctx.detect_batch_select_tensors(offsets, dev(sidx), 5))
    assert msg_d.replace("gpdb_detect_batch_select_device", "gpdb_detect_batch_select") == msg_h
    assert f"sample index {n[2]} at position {120 + 17} outside cloud 2" in msg_h
    assert has_batch(ctx) and intact()
    ctx.close()


def test_inputs_written_on_a_side_stream():
    """Inputs written by torch on a non-default stream, with no synchronisation before the calls, give the host route's
    records: the library reads them in order on the current stream."""
    ctx = context()
    views = mixed_views()
    pp = lib.preprocess_params()
    clouds = ctx.preprocess_clouds(views, pp)
    samples = samples_for([len(c["xyz"]) for c in clouds], 11)
    host_sel = ctx.detect_batch_select(samples, 20)
    host_cl = ctx.find_clusters_batch(host_sel, 1)
    pk = lib.pack_clouds(views)
    offsets, sidx = lib.pack_samples(samples)
    src = {k: torch.from_numpy(pk[k]).pin_memory() for k in ("xyz", "cam_source")}
    src["sidx"] = torch.from_numpy(sidx).pin_memory()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d = {k: torch.zeros(v.shape, dtype=v.dtype, device="cuda") for k, v in src.items()}
        torch.cuda._sleep(200_000_000)  # the copies below land long after the calls are queued behind them
        for k in d:
            d[k].copy_(src[k], non_blocking=True)
        ctx.preprocess_clouds_tensors(pk["offsets"], d["xyz"], pk["n_cameras"], pk["view_points"], cam_source=d["cam_source"],
                                      pp=pp)
        rec, soff = ctx.detect_batch_select_tensors(offsets, d["sidx"], 20)
        cl, coff = ctx.find_clusters_batch_tensors(soff, rec, 1)
    torch.cuda.synchronize()
    assert lib.poses_from_tensor(rec).tobytes() == b"".join(h.tobytes() for h in host_sel)
    assert np.array_equal(np.diff(soff), [len(h) for h in host_sel])
    assert lib.poses_from_tensor(cl).tobytes() == b"".join(h.tobytes() for h in host_cl)
    assert sum(len(h) for h in host_sel) > 0
    ctx.close()


def test_device_records_feed_host_calls():
    """The tensor records are gpdb_pose records: the host clustering of a device selection equals the device clustering."""
    ctx = context()
    clouds = processed_tables()
    set_device(ctx, clouds)
    samples = samples_for([len(c["xyz"]) for c in clouds], 60)
    offsets, sidx = lib.pack_samples(samples)
    rec, soff = ctx.detect_batch_select_tensors(offsets, dev(sidx), 40)
    recs = lib.poses_from_tensor(rec)
    assert recs.dtype == abi.POSE_DTYPE
    groups = [recs[soff[b]:soff[b + 1]] for b in range(len(clouds))]
    cl, coff = ctx.find_clusters_batch_tensors(soff, rec, 2)
    host = ctx.find_clusters_batch(groups, 2)
    assert lib.poses_from_tensor(cl).tobytes() == b"".join(h.tobytes() for h in host)
    ctx.close()
