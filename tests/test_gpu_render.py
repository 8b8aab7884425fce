"""Training views from triangle meshes on the device: gpdb_render_depth[_device] and gpdb_sample_meshes[_device].

The oracle is tests/render_reference.py, the numpy restatement of include/gpd_b200_render.h, bit for bit: depth and face
images of constructed and random scenes, and the surface samples. Host and device twins agree, failures write nothing
and leave the installed batch alone, the renders feed preprocessing as the restatement's images do, and the whole
meshes -> views -> candidates -> labels -> training loop runs on the device.
"""
import numpy as np
import pytest

import depth_reference as dr
import render_reference as rr
from conftest import load_weights
from gpd_b200 import lib, scenes

pytestmark = pytest.mark.gpu
ERR_INVALID = -1


def torch_():
    return pytest.importorskip("torch")


def context(weights=False):
    w, relu = load_weights(15)
    ctx = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
    if weights:
        ctx.set_weights(w)
    return ctx


def random_pose(rng, t):
    q = rng.normal(0, 1, 4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    R = dr.rot_x(0.1 * rng.normal()) @ dr.rot_y(0.1 * rng.normal()) if rng.random() < 0.7 else R
    return dr.pose(R, t)


def soup(rng, n):
    """overlapping random faces in front of the origin, with degenerate, duplicate, straddling, behind-the-camera,
    edge-on and image-covering ones"""
    if n == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)
    c = rng.uniform([-0.4, -0.3, 0.6], [0.4, 0.3, 1.4], (n, 3))
    v = (c[:, None, :] + rng.normal(0, 0.15, (n, 3, 3))).reshape(-1, 3)
    v[3 * (n // 2):3 * (n // 2) + 3, 2] = [-0.5, 0.8, 1.0]  # straddles the camera plane
    v[3:6] = v[0:3]  # duplicate of face 0: the tie rule
    v[6:9, 1] = v[6, 1]  # a degenerate sliver if the x differ little; edge-on for cameras in its plane
    v[9:12] = [[0.0, 0.0, 0.0], [0.3, 0.1, 1.0], [-0.2, 0.3, 1.0]]  # a vertex at the camera centre: edge-on rays
    v[12:15] = [[-50, -50, 1.7], [50, -50, 1.75], [0, 80, 1.8]]  # covers the whole image
    v[15:18] = [[0.1, 0.1, -0.8], [0.3, 0.0, -0.9], [0.0, 0.3, -1.0]]  # behind the camera
    v[18:21] = [[0.1, 0.1, 0.9], [0.1, 0.1, 0.9], [0.1, 0.1, 0.9]]  # a point
    f = np.arange(3 * n, dtype=np.int32).reshape(n, 3)
    return v.astype(np.float32), f


def cams_for(rng, K, W, H):
    out = []
    for k in range(K):
        f = rng.uniform(0.8, 1.2) * max(W, H)
        t = rng.normal(0, 0.05, 3) if k else np.zeros(3)
        out.append(lib.depth_camera(W, H, f, f * 1.01, (W - 1) / 2 + 0.25, (H - 1) / 2 - 0.5,
                                    np.eye(4)[:3] if k == 0 and rng.random() < 0.3 else random_pose(rng, t),
                                    rng.choice([0.001, 0.0005]), 0.0, float("inf")))
    return out


def check_against_restatement(ctx, meshes, cams, fmt):
    dt = np.float32 if fmt == 1 else np.uint16
    views, faces = ctx.render_depth(meshes, cams, dt, face_ids=True)
    ref = rr.render(meshes, cams, fmt)
    for b in range(len(meshes)):
        for k in range(len(cams[b])):
            img, fc = ref[b][0][k], ref[b][1][k]
            got = views[b][k][0]
            assert np.array_equal(got.view(np.uint32 if fmt == 1 else np.uint16), img.view(np.uint32 if fmt == 1 else np.uint16)), (b, k)
            assert np.array_equal(faces[b][k], fc), (b, k)
    return views, faces


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("K,W,H,B", [(1, 1, 1, 3), (2, 17, 5, 17), (8, 17, 5, 2), (1, 64, 48, 4)])
def test_random_soups_equal_the_restatement(fmt, K, W, H, B):
    rng = np.random.default_rng(K * 1000 + W + B + 7 * fmt)
    ctx = context()
    meshes = [soup(rng, 0 if b == 1 else int(rng.integers(22, 60))) for b in range(B)]
    cams = [cams_for(rng, K, W, H) for _ in range(B)]
    views, faces = check_against_restatement(ctx, meshes, cams, fmt)
    if W > 1:
        assert sum(int((f >= 0).sum()) for fs in faces for f in fs) > 0


def tile_border_scene():
    """faces whose edges run exactly through pixel centres on the 16-pixel tile borders of a 640 x 480 image (fx = fy =
    512, principal point (320, 240), identity pose), sharing edges and vertices, plus a table covering every tile"""
    def vert(u, v, z):
        return [z * (u - 320) / 512.0, z * (v - 240) / 512.0, z]
    V, F = [], []
    for (u0, v0) in [(16, 16), (160, 96), (320, 240), (448, 432)]:
        base = len(V)
        V += [vert(u0, v0, 1.0), vert(u0 + 32, v0, 1.25), vert(u0 + 32, v0 + 32, 1.5), vert(u0, v0 + 32, 1.0),
              vert(u0 + 16, v0 + 16, 1.125)]
        F += [(base, base + 1, base + 4), (base + 1, base + 2, base + 4), (base + 2, base + 3, base + 4),
              (base + 3, base, base + 4), (base + 3, base + 4, base)]  # the last repeats a face: a tie
    base = len(V)
    V += [[-20, -20, 3.0], [20, -20, 3.0], [20, 20, 3.0], [-20, 20, 3.0]]
    F += [(base, base + 1, base + 2), (base, base + 2, base + 3)]
    return np.array(V, np.float32), np.array(F, np.int32)


@pytest.mark.parametrize("fmt", [0, 1])
def test_tile_borders_shared_edges_and_full_size(fmt):
    ctx = context()
    v, f = tile_border_scene()
    cam = lib.depth_camera(640, 480, 512.0, 512.0, 320.0, 240.0, None, 0.001 if fmt == 0 else 1.0)
    rng = np.random.default_rng(5)
    views, faces = check_against_restatement(ctx, [(v, f), soup(rng, 40)], [[cam], cams_for(rng, 2, 640, 480)], fmt)
    fc = faces[0][0]
    assert (fc >= 0).all()  # the table under everything: no pixel falls through
    # the fans' closed squares are covered by their own faces: no pixel between shared edges reaches the table
    for k, (u0, v0) in enumerate([(16, 16), (160, 96), (320, 240), (448, 432)]):
        assert (fc[v0:v0 + 33, u0:u0 + 33] // 5 == k).all()
    assert not (fc % 5 == 4).any()  # the repeated face ties with face 3 and loses


def test_u16_range_limits():
    ctx = context()
    # depth_scale 0.5 and exact plane distances: t / scale = 0.5 and 2.5 round half to even (0: no return, 2), 1.5 to 2,
    # 65535 is the largest value, 65535.5 and 65536 round out of range (no return)
    meshes, cams = [], []
    for d in (0.25, 0.75, 1.25, 32767.5, 32767.75, 32768.0):
        meshes.append(rr_plane(d))
        cams.append([lib.depth_camera(5, 3, 4.0, 4.0, 2.0, 1.0, None, 0.5)])
    views, faces = check_against_restatement(ctx, meshes, cams, 0)
    assert [int(v[0][0][1, 2]) for v in views] == [0, 2, 2, 65535, 0, 0]
    assert [int(f[0][1, 2]) for f in faces] == [-1, 0, 0, 0, -1, -1]


def rr_plane(d):
    return (np.array([[-100, -100, d], [100, -100, d], [0, 100, d]], np.float32), np.array([[0, 1, 2]], np.int32))


def test_twins_equal_also_on_a_side_stream():
    torch = torch_()
    rng = np.random.default_rng(3)
    meshes = [scenes.mesh_table_scene(s, n_objects=5, segments=10)[:2] for s in (1, 2, 3)]
    cams = [dr.default_cameras(2, width=160, height=120, f=200.0) for _ in meshes]
    ctx = context()
    for fmt, tdt in ((1, torch.float32), (0, torch.uint16)):
        views, faces = ctx.render_depth(meshes, cams, np.float32 if fmt else np.uint16, face_ids=True)
        m = lib.pack_meshes(meshes)
        dv, df = torch.from_numpy(m["vertices"]).cuda(), torch.from_numpy(m["faces"]).cuda()
        flat = [c for cs in cams for c in cs]
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            d, fc = ctx.render_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2, 2], flat, tdt, face_ids=True)
        s.synchronize()
        host = np.concatenate([img.ravel() for v in views for img, _ in v])
        got = d.cpu().view(torch.int16).numpy().view(np.uint16) if fmt == 0 else d.cpu().numpy()
        assert np.array_equal(got.view(np.uint8), host.view(np.uint8))
        assert np.array_equal(fc.cpu().numpy(), np.concatenate([f.ravel() for fs in faces for f in fs]))
    poff, xyz, nrm, face = ctx.sample_meshes(meshes, 3000.0, 9, face_ids=True)
    with torch.cuda.stream(torch.cuda.Stream()):
        p2, x2, n2, f2 = ctx.sample_meshes_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, 3000.0, 9, face_ids=True)
    torch.cuda.synchronize()
    assert np.array_equal(poff, p2) and np.array_equal(xyz, x2.cpu().numpy())
    assert np.array_equal(nrm, n2.cpu().numpy()) and np.array_equal(face, f2.cpu().numpy())


def installed(ctx):
    return [(c["xyz"].copy(), c["normals"].copy()) for c in ctx.get_clouds()]


def test_failures_write_nothing_and_leave_the_batch():
    ctx = context()
    gt = scenes.synthetic_table_scene(4, n_points=20000)
    ctx.set_clouds([gt, gt])
    before = installed(ctx)
    v, f = rr_plane(1.0)
    cam = lib.depth_camera(4, 3, 4.0, 4.0, 2.0, 1.0, None, 0.001)
    L = lib.lib()

    def render(voff, vv, foff, ff, cams, fmt=1, ks=None):
        out = np.full(12 * len(cams), 7, np.float32)
        fo = np.full(12 * len(cams), 7, np.int32)
        arr = (lib.abi.DepthCamera * len(cams))(*cams)
        ks = np.array([len(cams)] if ks is None else ks, np.int32)
        rc = L.gpdb_render_depth(ctx.h, len(ks), lib._p(np.array(voff, np.int32)), lib._p(vv), lib._p(np.array(foff, np.int32)),
                                 lib._p(ff), lib._p(ks), lib.C.cast(arr, lib.C.c_void_p), fmt, lib._p(out), lib._p(fo))
        assert rc == ERR_INVALID and (out == 7).all() and (fo == 7).all()
        return L.gpdb_last_error(ctx.h).decode()

    bad_f = np.array([[0, 1, 3]], np.int32)
    assert "view 0: face 0 = (0, 1, 3) indexes outside its 3 vertices" in render([0, 3], v, [0, 1], bad_f, [cam])
    nan_v = v.copy()
    nan_v[2, 1] = np.nan
    assert "view 0: vertex 2 has a non-finite coordinate" in render([0, 3], nan_v, [0, 1], f, [cam])
    assert "vertex_offsets decrease at view 0" in render([0, -1], v, [0, 1], f, [cam])
    assert "face_offsets" in render([0, 3], v, [1, 1], f, [cam])
    bad_cam = lib.depth_camera(4, 3, -1.0, 4.0, 2.0, 1.0)
    assert "view 0 camera 0 (camera 0 of the call): fx and fy must be positive" in render([0, 3], v, [0, 1], f, [bad_cam])
    big = lib.depth_camera(65536, 32768, 4.0, 4.0, 2.0, 1.0)
    assert "2^31 or more pixels" in render([0, 3], v, [0, 1], f, [big])
    assert "unknown depth format" in render([0, 3], v, [0, 1], f, [cam], fmt=5)
    assert "view 0 has 9 cameras" in render([0, 3], v, [0, 1], f, [cam] * 9)
    # samples
    for dens, msg in ((0.0, "density must be finite and > 0"), (float("inf"), "density must be finite"),
                      (1e18, "mesh 0: the call reaches 2^31 or more sampled points")):
        poff = np.full(2, 7, np.int32)
        xyz = np.full((4, 3), 7, np.float32)
        rc = L.gpdb_sample_meshes(ctx.h, 1, lib._p(np.array([0, 3], np.int32)), lib._p(v), lib._p(np.array([0, 1], np.int32)),
                                  lib._p(f), lib.C.c_double(dens), lib.C.c_uint64(0), lib._p(poff), lib._p(xyz), None, None)
        assert rc == ERR_INVALID and msg in L.gpdb_last_error(ctx.h).decode() and (poff == 7).all() and (xyz == 7).all()
    with pytest.raises(lib.GpdbError, match="mesh 0: face 0"):
        ctx.sample_meshes([(v, bad_f)], 100.0, 0)
    # successful calls do not touch the batch either
    ctx.render_depth([(v, f)], [[cam]], np.float32)
    ctx.sample_meshes([(v, f)], 100.0, 0)
    after = installed(ctx)
    assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(before, after))


def test_preprocessing_of_a_render_equals_the_restatement_and_lies_on_the_faces():
    torch = torch_()
    meshes = [scenes.mesh_table_scene(s, n_objects=6, segments=12)[:2] for s in (5, 6)]
    cams = [dr.default_cameras(2, width=160, height=120, f=200.0) for _ in meshes]
    ref = rr.render(meshes, cams, 0)
    a, b = context(), context()
    pp = lib.preprocess_params(voxelize=0)
    ra = a.preprocess_depth([[(ref[v][0][k], cams[v][k]) for k in range(2)] for v in range(2)], pp=pp)
    m = lib.pack_meshes(meshes)
    dv, df = torch.from_numpy(m["vertices"]).cuda(), torch.from_numpy(m["faces"]).cuda()
    flat = [c for cs in cams for c in cs]
    d, fc = b.render_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2], flat, torch.uint16, face_ids=True)
    b.preprocess_depth_tensors([2, 2], flat, d, pp=pp)
    rb = b.get_clouds()
    for x, y in zip(ra, rb):
        for key in ("xyz", "normals", "cam_source", "src"):
            assert np.array_equal(x[key], y[key]), key
    # every point back-projected from a pixel lies near the plane of the face that pixel hit: the stored depth is within
    # half a millimetre of the hit's t (U16), the point moves by that times |d| <= 1.12 along its ray, and the float32
    # back-projection adds well under a micrometre: 0.6 mm
    fcs = fc.cpu().numpy()
    roff = np.concatenate([[0], np.cumsum([sum(c.width * c.height for c in cs) for cs in cams])])
    for vb, cloud in enumerate(rb):
        verts, faces = meshes[vb]
        n, L = rr.face_normals(verts, faces)
        fid = fcs[roff[vb] + cloud["src"]]
        assert (fid >= 0).all()
        a0 = verts[faces[fid, 0]].astype(np.float64)
        p = cloud["xyz"].astype(np.float64)
        dist = np.abs(((p - a0) * n[fid]).sum(1)) / L[fid]
        assert (dist <= 6e-4).all(), dist.max()


def test_samples_equal_the_restatement():
    torch = torch_()
    ctx = context()
    meshes = [scenes.mesh_table_scene(s, n_objects=4, segments=8)[:2] for s in (1, 2)] + [rr_plane(1.0)]
    for density, seed in ((2000.0, 0), (15000.5, 2 ** 63 + 5), (1e-3, 3)):
        off, xyz, nrm, face = ctx.sample_meshes(meshes, density, seed, face_ids=True)
        r = rr.sample_meshes(meshes, density, seed)
        assert np.array_equal(off, r[0]) and np.array_equal(xyz, r[1]) and np.array_equal(face, r[3])
        assert np.array_equal(nrm.view(np.uint64), r[2].view(np.uint64))
        m = lib.pack_meshes(meshes)
        poff = np.zeros(4, np.int32)
        n = lib.lib().gpdb_sample_meshes(ctx.h, 3, lib._p(m["vertex_offsets"]), lib._p(m["vertices"]), lib._p(m["face_offsets"]),
                                         lib._p(m["faces"]), lib.C.c_double(density), lib.C.c_uint64(seed), lib._p(poff),
                                         None, None, None)
        assert n == off[-1] and np.array_equal(poff, off)
        one = ctx.sample_meshes(meshes[1:2], density, (seed + 1) % 2 ** 64)
        assert np.array_equal(one[1], xyz[off[1]:off[2]])


def test_meshes_to_trained_weights_end_to_end():
    torch = torch_()

    def run():
        scenes_ = [scenes.mesh_table_scene(s, n_objects=10, segments=16) for s in (21, 22)]
        meshes = [s[:2] for s in scenes_]
        m = lib.pack_meshes(meshes)
        dv, df = torch.from_numpy(m["vertices"]).cuda(), torch.from_numpy(m["faces"]).cuda()
        cams = [c for _ in meshes for c in dr.default_cameras(2, width=320, height=240, f=400.0)]
        a = context(weights=True)
        d, fc = a.render_depth_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, [2, 2], cams, torch.float32, face_ids=True)
        a.preprocess_depth_tensors([2, 2], cams, d)
        # the object mask: pixels whose face belongs to an object (id > 0) of their view's scene
        mask = torch.zeros_like(fc, dtype=torch.uint8)
        px = 2 * 320 * 240
        for b, (_, _, ids) in enumerate(scenes_):
            fb = fc[b * px:(b + 1) * px]
            idt = torch.from_numpy(ids).cuda()
            mask[b * px:(b + 1) * px] = ((fb >= 0) & (idt[fb.clamp(min=0).long()] > 0)).to(torch.uint8)
        soff, sidx = a.subsample_clouds_tensors(300, 1, mask)
        rec, _, _, coff = a.detect_batch_tensors(soff, sidx)
        images = a.images_batch_tensors(coff, rec)
        g = context()
        poff, xyz, nrm = g.sample_meshes_tensors(m["vertex_offsets"], dv, m["face_offsets"], df, 40000.0, 3)
        vp = np.array([[c.pose[3], c.pose[7], c.pose[11]] for c in cams[::2]])
        g.set_clouds_tensors(poff, xyz, nrm, [1, 1], vp)
        labels = (g.reevaluate_batch_tensors(coff, rec) == 1).to(torch.int32)
        pos, neg = (labels == 1).nonzero().flatten(), (labels == 0).nonzero().flatten()
        k = min(len(pos), len(neg), 32)
        assert k >= 4, (len(pos), len(neg))
        sel = torch.cat([pos[:k], neg[:k]])
        w, relu = load_weights(15)
        t = lib.Context(lib.default_params(channels=15, relu_after_conv=relu))
        t.train_begin(lib.train_params(optimizer="adam", lr=1e-4), init=w)
        losses = [float(t.train_step_tensors(images[sel].contiguous(), labels[sel].contiguous())) for _ in range(15)]
        return losses, labels.cpu().numpy(), t.train_weights()

    l1, lab1, w1 = run()
    assert l1[-1] < l1[0], l1
    l2, lab2, w2 = run()
    assert l1 == l2 and np.array_equal(lab1, lab2) and all(np.array_equal(x, y) for x, y in zip(w1, w2))
