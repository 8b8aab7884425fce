"""Sensor views on the device: gpdb_render_sensor_depth[_device] against tests/sensor_reference.py, the numpy restatement
of include/gpd_b200_sensor.h, bit for bit in depth and face images: table-scene batches with one and two cameras of mixed
sizes, each rule alone and all together, and the analytic shadow and grazing scenes. Zero parameters give the render,
the twins and repeated calls agree, a view's images do not depend on its batch, failures write nothing, and sensor views
feed the device's training-data chain."""
import ctypes as C

import numpy as np
import pytest

import depth_reference as dr
import sensor_reference as sr
from conftest import load_weights
from gpd_b200 import abi, lib, scenes
from test_sensor_reference import ERROR_CASES, camera, quad, wall_and_plate

pytestmark = pytest.mark.gpu
ERR_INVALID = -1

CASES = {"lateral": dict(lateral_sigma=1.3), "grazing": dict(min_cos_incidence=0.35),
         "shadow": dict(baseline=0.075, shadow_tolerance=0.01), "disparity": dict(baseline=0.075, disparity_sigma=0.4),
         "quantised": dict(baseline=0.075, disparity_step=0.125), "dropout": dict(dropout=0.2),
         "all": dict(baseline=0.075, lateral_sigma=0.7, disparity_sigma=0.25, disparity_step=0.125, min_cos_incidence=0.3,
                     shadow_tolerance=0.02, dropout=0.05)}


def torch_():
    return pytest.importorskip("torch")


def context():
    w, relu = load_weights(15)
    return lib.Context(lib.default_params(channels=15, relu_after_conv=relu))


def bits(a, fmt):
    return np.asarray(a).view(np.uint32 if fmt == 1 else np.uint16)


def check(ctx, meshes, cams, sp, seed, fmt, T):
    views, faces = ctx.render_sensor_depth(meshes, cams, sp, seed, np.float32 if fmt == 1 else np.uint16, face_ids=True)
    ref = sr.render(meshes, cams, sp, seed, fmt, T)
    for b in range(len(meshes)):
        for k in range(len(cams[b])):
            assert np.array_equal(bits(views[b][k][0], fmt), bits(ref[b][0][k], fmt)), (b, k)
            assert np.array_equal(faces[b][k], ref[b][1][k]), (b, k)
    return views, faces


def table_views(K):
    meshes = [scenes.mesh_table_scene(s, n_objects=5, segments=10)[:2] for s in (11, 12, 13)]
    sizes = [(96, 72), (80, 60), (64, 48)]
    cams = [dr.default_cameras(K, width=w, height=h, f=1.1 * w, scale=0.001) for w, h in sizes]
    return meshes, cams


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("fmt", [0, 1])
def test_table_scenes_equal_the_restatement(case, K, fmt):
    T = sr.table()
    meshes, cams = table_views(K)
    views, faces = check(context(), meshes, cams, lib.sensor_params(**CASES[case]), 2 ** 64 - 2, fmt, T)
    assert sum(int((f >= 0).sum()) for fs in faces for f in fs) > 3000


@pytest.mark.parametrize("fmt", [0, 1])
def test_analytic_scenes_equal_the_restatement(fmt):
    T = sr.table()
    ctx = context()
    scale = 0.001 if fmt == 0 else 1.0
    _, faces = check(ctx, [wall_and_plate()], [[camera(scale=scale)]], lib.sensor_params(baseline=0.075, shadow_tolerance=0.01),
                     5, fmt, T)
    assert (faces[0][0][240, 200:248] < 0).sum() >= 10
    tilted = quad(-3, -2, 3, 2, 1.0 - 3 * np.tan(1.2), 1.0 + 3 * np.tan(1.2))
    check(ctx, [tilted, tilted], [[camera(160, 120, 150.0, scale)], [camera(160, 120, 150.0, scale)]],
          lib.sensor_params(min_cos_incidence=np.cos(np.radians(75.0))), 1, fmt, T)


@pytest.mark.parametrize("fmt", [0, 1])
def test_zero_parameters_give_the_render(fmt):
    meshes, cams = table_views(2)
    ctx = context()
    dt = np.float32 if fmt == 1 else np.uint16
    v0, f0 = ctx.render_depth(meshes, cams, dt, face_ids=True)
    v1, f1 = ctx.render_sensor_depth(meshes, cams, lib.sensor_params(), 123, dt, face_ids=True)
    for b in range(3):
        for k in range(2):
            assert np.array_equal(bits(v0[b][k][0], fmt), bits(v1[b][k][0], fmt)) and np.array_equal(f0[b][k], f1[b][k])


def test_twins_repeats_and_batch_independence():
    torch = torch_()
    meshes, cams = table_views(2)
    sp = lib.sensor_params(**CASES["all"])
    ctx = context()
    seed = 77
    views, faces = ctx.render_sensor_depth(meshes, cams, sp, seed, np.float32, face_ids=True)
    again, faces2 = ctx.render_sensor_depth(meshes, cams, sp, seed, np.float32, face_ids=True)
    for b in range(3):
        for k in range(2):
            assert np.array_equal(bits(views[b][k][0], 1), bits(again[b][k][0], 1)) and np.array_equal(faces[b][k], faces2[b][k])
    # view b alone with the key seed + b
    for b in range(3):
        one, fone = ctx.render_sensor_depth(meshes[b:b + 1], cams[b:b + 1], sp, seed + b, np.float32, face_ids=True)
        for k in range(2):
            assert np.array_equal(bits(one[0][k][0], 1), bits(views[b][k][0], 1)) and np.array_equal(fone[0][k], faces[b][k])
    # the device twin, on a side stream
    m = lib.pack_meshes(meshes)
    dv, df = torch.from_numpy(m["vertices"]).cuda(), torch.from_numpy(m["faces"]).cuda()
    flat = [c for cs in cams for c in cs]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d, fc = ctx.render_sensor_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2, 2], flat, sp, seed,
                                                torch.float32, face_ids=True)
    s.synchronize()
    host = np.concatenate([img.ravel() for v in views for img, _ in v])
    assert np.array_equal(d.cpu().numpy().view(np.uint32), host.view(np.uint32))
    assert np.array_equal(fc.cpu().numpy(), np.concatenate([f.ravel() for fs in faces for f in fs]))
    with torch.cuda.stream(s):
        d16 = ctx.render_sensor_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2, 2], flat, sp, seed,
                                              torch.uint16)
    s.synchronize()
    h16 = np.concatenate([img.ravel() for v in ctx.render_sensor_depth(meshes, cams, sp, seed, np.uint16) for img, _ in v])
    assert np.array_equal(d16.cpu().view(torch.int16).numpy().view(np.uint16), h16)


def test_failures_write_nothing_and_name_the_view_or_camera():
    ctx = context()
    v, f = np.array([[-9, -9, 1.0], [9, -9, 1.0], [0, 9, 1.0]], np.float32), np.array([[0, 1, 2]], np.int32)
    cam = lib.depth_camera(4, 3, 4.0, 4.0, 2.0, 1.0, None, 0.001)
    L = lib.lib()

    def render(voff, vv, foff, ff, cams, sp, fmt=1):
        out = np.full(12 * len(cams), 7, np.float32)
        fo = np.full(12 * len(cams), 7, np.int32)
        arr = (abi.DepthCamera * len(cams))(*cams)
        ks = np.array([len(cams)], np.int32)
        rc = L.gpdb_render_sensor_depth(ctx.h, 1, lib._p(np.array(voff, np.int32)), lib._p(vv), lib._p(np.array(foff, np.int32)),
                                        lib._p(ff), lib._p(ks), C.cast(arr, C.c_void_p), fmt, lib._p(out), lib._p(fo),
                                        None if sp is None else C.c_void_p(C.addressof(sp)), C.c_uint64(3))
        assert rc == ERR_INVALID and (out == 7).all() and (fo == 7).all()
        return L.gpdb_last_error(ctx.h).decode()

    good = lib.sensor_params(**CASES["all"])
    for fields, msg in ERROR_CASES:
        assert "gpdb_render_sensor_depth: sensor: " + msg in render([0, 3], v, [0, 1], f, [cam], lib.sensor_params(**fields))
    assert "need sensor" in render([0, 3], v, [0, 1], f, [cam], None)
    assert "view 0: face 0 = (0, 1, 3) indexes outside its 3 vertices" in render([0, 3], v, [0, 1], np.array([[0, 1, 3]], np.int32),
                                                                                 [cam], good)
    nan_v = v.copy()
    nan_v[2, 1] = np.nan
    assert "view 0: vertex 2 has a non-finite coordinate" in render([0, 3], nan_v, [0, 1], f, [cam], good)
    bad_cam = lib.depth_camera(4, 3, -1.0, 4.0, 2.0, 1.0)
    assert "view 0 camera 1 (camera 1 of the call): fx and fy must be positive" in render([0, 3], v, [0, 1], f, [cam, bad_cam], good)
    assert "unknown depth format" in render([0, 3], v, [0, 1], f, [cam], good, fmt=4)
    assert "2^31 or more pixels" in render([0, 3], v, [0, 1], f, [lib.depth_camera(65536, 32768, 4.0, 4.0, 2.0, 1.0)], good)
    assert "vertex_offsets decrease at view 0" in render([0, -1], v, [0, 1], f, [cam], good)
    with pytest.raises(TypeError):
        ctx.render_sensor_depth([(v, f)], [[cam]], {"baseline": 0.1}, 0)


def test_sensor_views_feed_the_training_data_chain():
    torch = torch_()
    scenes_ = [scenes.mesh_table_scene(s, n_objects=10, segments=16) for s in (31, 32)]
    meshes = [s[:2] for s in scenes_]
    m = lib.pack_meshes(meshes)
    dv, df = torch.from_numpy(m["vertices"]).cuda(), torch.from_numpy(m["faces"]).cuda()
    cams = [c for _ in meshes for c in dr.default_cameras(2, width=320, height=240, f=400.0)]
    sp = lib.sensor_params(baseline=0.075, lateral_sigma=0.5, disparity_sigma=0.05, disparity_step=0.125,
                           min_cos_incidence=0.2, shadow_tolerance=0.01, dropout=0.01)
    w, relu = load_weights(15)
    a = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    a.set_weights(w)
    d, fc = a.render_sensor_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2], cams, sp, 5, torch.uint16,
                                          face_ids=True)
    clean = a.render_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2], cams, torch.uint16)
    lost = int(((clean.view(torch.int16) != 0) & (fc < 0)).sum())
    assert lost > 1000  # the sensor drops returns the clean render has
    a.preprocess_depth_tensors([2, 2], cams, d)
    mask = torch.zeros_like(fc, dtype=torch.uint8)
    px = 2 * 320 * 240
    for b, (_, _, ids) in enumerate(scenes_):
        fb = fc[b * px:(b + 1) * px]
        idt = torch.from_numpy(ids).cuda()
        mask[b * px:(b + 1) * px] = ((fb >= 0) & (idt[fb.clamp(min=0).long()] > 0)).to(torch.uint8)
    soff, sidx = a.subsample_clouds_tensors(300, 1, mask)
    rec, _, _, coff = a.detect_batch_tensors(soff, sidx)
    images = a.images_batch_tensors(coff, rec)
    assert images.shape[0] == int(coff[-1]) > 0
    g = context()
    poff, xyz, nrm = g.sample_meshes_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, 40000.0, 3)
    vp = np.array([[c.pose[3], c.pose[7], c.pose[11]] for c in cams[::2]])
    g.set_clouds_tensors(poff, xyz, nrm, [1, 1], vp)
    labels = g.reevaluate_batch_tensors(coff, rec)
    assert labels.shape[0] == images.shape[0]
    assert int((labels == 1).sum()) > 0 and int((labels != 1).sum()) > 0
