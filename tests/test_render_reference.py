"""CPU tests of include/gpd_b200_render.h's restatement (tests/render_reference.py): analytic planes and spheres, the
watertightness of shared edges and vertices through pixel centres, the header's own helpers compiled for the host held
bit for bit against numpy, the surface-sample statistics, and the binding's bookkeeping (pack_meshes, the splitting of
the images and the count-then-fill of the samples) against a stand-in library."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import render_reference as rr
from gpd_b200 import abi, lib, scenes


def camera(W, H, f, cx, cy, pose=None, scale=1.0):
    return lib.depth_camera(W, H, f, f, cx, cy, pose, scale)


def quad(x0, y0, z0, x1, y1, z1):
    """two faces spanning x0..x1, y0..y1 (z0 at x0, z1 at x1): a plane of slope (z1 - z0) / (x1 - x0) along x"""
    v = np.array([[x0, y0, z0], [x1, y0, z1], [x1, y1, z1], [x0, y1, z0]], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int32)


def test_fronto_parallel_plane_renders_its_distance():
    for d in (0.75, 1.3125, 2.0):
        v, f = quad(-10, -10, d, 10, 10, d)
        pose = np.hstack([np.eye(3), [[0.0], [0.0], [0.0]]])
        img, face = rr.render_camera(v, f, camera(17, 5, 8.0, 8.0, 2.0, pose), 1)
        assert (img == np.float32(d)).all() and (face >= 0).all()
        img16, _ = rr.render_camera(v, f, camera(17, 5, 8.0, 8.0, 2.0, pose, scale=0.001), 0)
        assert (img16 == np.uint16(round(d * 1000))).all()


def test_tilted_plane_matches_the_closed_form_within_two_ulps():
    # z = 1 + x / 4: vertices exact in float32, identity pose, so the camera frame is exact
    v, f = quad(-2, -2, 0.5, 2, 2, 1.5)
    cam = camera(17, 5, 7.0, 8.3, 2.1)
    ok_all = []
    for fi in range(2):
        rec = rr.setup(*[rr.to_camera(v, rr.pose_of(cam))[f[fi, k]][None] for k in range(3)])[0]
        dx, dy = rr.rays(cam)
        ok, t = rr.hit(rec, dx, dy)
        ok_all.append(ok)
        for i in np.flatnonzero(ok):
            exact = Fraction(1) / (1 - Fraction(dx[i]) / 4)  # dx is the float64 ray the rule uses
            assert abs(Fraction(t[i]) - exact) <= 2 * Fraction(np.spacing(float(exact)))
    assert np.logical_or(*ok_all).all()


def test_sphere_silhouette_is_within_a_pixel_of_the_circle():
    r, D, fpx = 0.1, 0.5, 60.0
    v, f, _ = (None, None, None)
    v, f = scenes._mesh_sphere(np.array([0.0, 0.0, D]), r, 48)
    cam = camera(64, 64, fpx, 31.5, 31.5)
    _, face = rr.render_camera(v.astype(np.float32), f.astype(np.int32), cam, 1)
    rho = fpx * np.tan(np.arcsin(r / D))
    vv, uu = np.mgrid[0:64, 0:64]
    dist = np.hypot(uu - 31.5, vv - 31.5)
    covered = face >= 0
    assert covered[dist <= rho - 1].all() and not covered[dist >= rho + 1].any()


def fan_and_strip(z_of):
    """vertices on rays through pixel centres (fx = fy = 64, principal point (8, 8)): a closed fan of 8 faces around
    pixel (8, 8) and a strip of 12 faces between rows 13 and 16; z_of(du, dv) places each vertex on its ray"""
    def vert(du, dv):
        z = z_of(du, dv)
        return [z * du / 64.0, z * dv / 64.0, z]
    ring = [(4, 0), (3, 3), (0, 4), (-3, 3), (-4, 0), (-3, -3), (0, -4), (3, -3)]
    V = [vert(0, 0)] + [vert(*p) for p in ring]
    Fc = [(0, 1 + k, 1 + (k + 1) % 8) for k in range(8)]
    base = len(V)
    for k in range(7):
        V += [vert(-7 + 2 * k, 5), vert(-6 + 2 * k, 8)]
    Fs = []
    for k in range(12):
        Fs.append((base + k, base + k + 1, base + k + 2) if k % 2 == 0 else (base + k + 1, base + k, base + k + 2))
    return np.array(V, np.float32), np.array(Fc + Fs, np.int32), ring


def inside_hull(pts, poly):
    """pts [n, 2] integer pixel offsets inside or on the convex polygon poly (counter-clockwise, integer vertices)"""
    ok = np.ones(len(pts), bool)
    for k in range(len(poly)):
        (x0, y0), (x1, y1) = poly[k], poly[(k + 1) % len(poly)]
        ok &= (x1 - x0) * (pts[:, 1] - y0) - (y1 - y0) * (pts[:, 0] - x0) >= 0
    return ok


@pytest.mark.parametrize("z_of", [lambda du, dv: 1.0, lambda du, dv: 1.0 + du / 16.0 + dv / 32.0,
                                  lambda du, dv: 2.0 - (du * du + dv * dv) / 128.0])
def test_fans_and_strips_through_pixel_centres_leave_no_hole(z_of):
    v, f, ring = fan_and_strip(z_of)
    cam = camera(17, 17, 64.0, 8.0, 8.0)
    _, face = rr.render_camera(v, f, cam, 1)
    vv, uu = np.mgrid[0:17, 0:17]
    pts = np.stack([uu.ravel() - 8, vv.ravel() - 8], 1)
    fan = inside_hull(pts, ring).reshape(17, 17)
    assert (face[fan] >= 0).all() and np.isin(face[fan], np.arange(8)).all()
    # every pixel of each strip face's closed triangle is covered, by a strip face
    strip = np.zeros((17, 17), bool)
    for k in range(12):
        a, b, c = [((v[i, 0] / v[i, 2]) * 64, (v[i, 1] / v[i, 2]) * 64) for i in f[8 + k]]
        tri = [tuple(int(round(x)) for x in p) for p in (a, b, c)]
        if (tri[1][0] - tri[0][0]) * (tri[2][1] - tri[0][1]) - (tri[1][1] - tri[0][1]) * (tri[2][0] - tri[0][0]) < 0:
            tri = [tri[0], tri[2], tri[1]]
        strip |= inside_hull(pts, tri).reshape(17, 17)
    assert strip.sum() > 40 and (face[strip] >= 8).all()


def random_faces(rng, n):
    abc = rng.normal(0, 1, (n, 9))
    abc[:, 2::3] += 3.0
    abc[: n // 8, 3:6] = abc[: n // 8, 0:3]  # degenerate
    return abc


def test_header_helpers_equal_numpy_bit_for_bit():
    L = rr.cpp()
    rng = np.random.default_rng(1)
    n = 4000
    # rule 2
    p = rng.normal(0, 2, (n, 3)).astype(np.float32)
    pose = np.concatenate([rng.normal(0, 1, 9).reshape(3, 3), rng.normal(0, 1, (3, 1))], 1).ravel()
    q = np.zeros((n, 3))
    L.ro_to_camera(n, rr.p_(pose), rr.p_(p), rr.p_(q))
    assert np.array_equal(q.view(np.uint64), rr.to_camera(p, pose).view(np.uint64))
    # rule 4
    abc = random_faces(rng, n)
    d = rng.normal(0, 0.5, (n, 2))
    rec, t, cov = np.zeros((n, 13)), np.zeros(n), np.zeros(n, np.int32)
    L.ro_setup_hit(n, rr.p_(abc), rr.p_(d), rr.p_(rec), rr.p_(t), rr.p_(cov))
    rec2 = rr.setup(abc[:, 0:3], abc[:, 3:6], abc[:, 6:9])
    assert np.array_equal(rec.view(np.uint64), rec2.view(np.uint64))
    ok2 = np.zeros(n, bool)
    t2 = np.zeros(n)
    for i in range(n):
        o, tt = rr.hit(rec2[i], d[i, 0:1], d[i, 1:2])
        ok2[i], t2[i] = o[0], tt[0]
    assert np.array_equal(cov.astype(bool), ok2) and 0.02 < ok2.mean() < 0.8
    assert np.array_equal(t[ok2].view(np.uint64), t2[ok2].view(np.uint64))
    # rule 5, including the uint16 range ends and halves
    tt = np.concatenate([rng.uniform(0, 70, n), [0.0005, 0.0015, 0.0025, 65.5345, 65.5355, 65.5365, 1e300, 1e-300]])
    for fmt, scale in ((0, 0.001), (1, 1.0), (1, 1e-300)):
        raw, ret = np.zeros(len(tt), np.uint32), np.zeros(len(tt), np.int32)
        L.ro_raw(len(tt), rr.p_(tt), scale, fmt, rr.p_(raw), rr.p_(ret))
        raw2, ret2 = rr.raw_of(tt, scale, fmt)
        assert np.array_equal(ret.astype(bool), ret2)
        assert np.array_equal(raw, raw2.view(np.uint32) if fmt == 1 else raw2.astype(np.uint32))
    # rule 6
    abcf = abc.astype(np.float32)
    key = 0x1234567890ABCDEF
    cnt, pt, nrm, Ln = np.zeros(n), np.zeros((n, 3)), np.zeros((n, 3)), np.zeros(n)
    L.ro_mesh(n, rr.p_(abcf), C.c_uint64(key), 3.5, rr.p_(cnt), rr.p_(pt), rr.p_(nrm), rr.p_(Ln))
    v = abcf.reshape(-1, 3)
    f = np.arange(3 * n).reshape(n, 3)
    assert np.array_equal(cnt, rr.counts(v, f, 3.5, key))
    d1 = rr.draws(key, np.arange(n), 1)
    r1, r2 = rr.unit(d1[:, 0], d1[:, 1]), rr.unit(d1[:, 2], d1[:, 3])
    s = np.sqrt(r1)
    a, b, c = [abcf[:, 3 * k:3 * k + 3].astype(np.float64) for k in range(3)]
    p2 = ((1.0 - s)[:, None] * a + (s * (1.0 - r2))[:, None] * b) + (s * r2)[:, None] * c
    assert np.array_equal(pt.view(np.uint64), p2.view(np.uint64))
    n2, L2 = rr.face_normals(v, f)
    good = L2 > 0
    assert np.array_equal(Ln.view(np.uint64), L2.view(np.uint64))
    assert np.array_equal(nrm[good].view(np.uint64), (n2[good] / L2[good, None]).view(np.uint64))


def test_samples_follow_area_and_lie_on_their_faces():
    v, f, _ = scenes.mesh_table_scene(3, n_objects=6, segments=12)
    density = 20000.0
    off, xyz, nrm, face = rr.sample_meshes([(v, f)], density, 11)
    n, L = rr.face_normals(v, f)
    expect = (0.5 * L).sum() * density
    assert abs(len(xyz) - expect) <= 5 * 0.5 * np.sqrt(len(f)) and off[-1] == len(xyz)
    assert np.all(np.diff(face) >= 0)
    vd = v.astype(np.float64)
    a, b, c = vd[f[face, 0]], vd[f[face, 1]], vd[f[face, 2]]
    p = xyz.astype(np.float64)
    # on the plane: float32 rounding of each coordinate moves a point by at most 2^-24 |p| per axis
    dist = np.abs(((p - a) * nrm).sum(1))
    assert (dist <= 2.0 ** -24 * np.abs(p).max(1) * np.sqrt(3) * 1.01 + 1e-12).all()
    # inside: barycentric weights of the point (before its float32 rounding, recomputed from the draw) are >= 0
    e0, e1, e2 = b - a, c - a, p - a
    d00, d01, d11 = (e0 * e0).sum(1), (e0 * e1).sum(1), (e1 * e1).sum(1)
    d20, d21 = (e2 * e0).sum(1), (e2 * e1).sum(1)
    den = d00 * d11 - d01 * d01
    wb, wc = (d11 * d20 - d01 * d21) / den, (d00 * d21 - d01 * d20) / den
    tol = 1e-4
    assert (wb >= -tol).all() and (wc >= -tol).all() and (wb + wc <= 1 + tol).all()
    assert np.abs(np.linalg.norm(nrm, axis=1) - 1).max() < 4e-16
    assert ((nrm * n[face]).sum(1) > 0).all()
    # mesh b of a batch draws with seed + b
    off2, xyz2, _, _ = rr.sample_meshes([(v[:8], f[:12]), (v, f)], density, 10)
    assert np.array_equal(xyz2[off2[1]:], xyz)


def test_scene_is_closed_and_outward():
    v, f, ids = scenes.mesh_table_scene(0, n_objects=10, segments=10)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    s = set(map(tuple, e.tolist()))
    assert len(s) == len(e) and all((b, a) in s for a, b in s)
    assert ids.min() == 0 and ids.max() == 10 and len(ids) == len(f)
    n, _ = rr.face_normals(v, f)
    for k in range(11):
        sel = ids == k
        centre = v[np.unique(f[sel])].astype(np.float64).mean(0)
        cen = v[f[sel]].astype(np.float64).mean(1)
        assert (((cen - centre) * n[sel]).sum(1) > 0).all()


# ---- the binding against a stand-in library ----------------------------------------------------------------------------

class FakeLib:
    """Writes pixel i of the call as i (and face -i), and samples point i of mesh b as (b, i, 0)."""

    def __init__(self):
        self.calls = []

    def gpdb_render_depth(self, h, B, voff, vtx, foff, faces, ks, cams, fmt, depth, face):
        k = np.ctypeslib.as_array(C.cast(ks, C.POINTER(C.c_int32)), (B,))
        arr = C.cast(cams, C.POINTER(abi.DepthCamera))
        n = sum(arr[i].width * arr[i].height for i in range(int(k.sum())))
        dt = C.c_float if fmt == abi.DEPTH_F32 else C.c_uint16
        np.ctypeslib.as_array(C.cast(depth, C.POINTER(dt)), (n,))[:] = np.arange(n)
        if face:
            np.ctypeslib.as_array(C.cast(face, C.POINTER(C.c_int32)), (n,))[:] = -np.arange(n)
        self.calls.append(("render", B, np.ctypeslib.as_array(C.cast(voff, C.POINTER(C.c_int32)), (B + 1,)).copy()))
        return B

    def gpdb_sample_meshes(self, h, B, voff, vtx, foff, faces, density, seed, poff, xyz, nrm, face):
        counts = [3 * (b + 1) for b in range(B)]
        po = np.ctypeslib.as_array(C.cast(poff, C.POINTER(C.c_int32)), (B + 1,))
        po[:] = np.concatenate([[0], np.cumsum(counts)])
        n = int(po[-1])
        self.calls.append(("sample", xyz is not None, density.value, seed.value))
        if xyz:
            x = np.ctypeslib.as_array(C.cast(xyz, C.POINTER(C.c_float)), (n, 3))
            x[:, 0] = np.repeat(np.arange(B), counts)
            x[:, 1] = np.arange(n)
        return n

    def gpdb_last_error(self, h):
        return b"stand-in error"


def fake_context(monkeypatch):
    fake = FakeLib()
    monkeypatch.setattr(lib, "lib", lambda: fake)
    ctx = object.__new__(lib.Context)
    ctx.h = None
    ctx.params = abi.default_params(15)
    return ctx, fake


def test_pack_meshes_offsets_and_concatenation():
    m = lib.pack_meshes([(np.zeros((4, 3)), [[0, 1, 2], [0, 2, 3]]), (np.ones((3, 3)), np.zeros((0, 3))),
                         (np.full((3, 3), 2.0), [[2, 1, 0]])])
    assert m["vertex_offsets"].tolist() == [0, 4, 7, 10] and m["face_offsets"].tolist() == [0, 2, 2, 3]
    assert m["vertices"].dtype == np.float32 and m["vertices"].shape == (10, 3)
    assert m["faces"].dtype == np.int32 and m["faces"][2].tolist() == [2, 1, 0]
    with pytest.raises(ValueError):
        lib.pack_meshes([])


def test_render_depth_splits_views_and_cameras(monkeypatch):
    ctx, fake = fake_context(monkeypatch)
    meshes = [quad(-1, -1, 1, 1, 1, 1), quad(-1, -1, 2, 1, 1, 2)]
    cams = [[camera(3, 2, 1, 1, 1)], [camera(2, 2, 1, 1, 1), camera(4, 1, 1, 1, 1)]]
    views, faces = ctx.render_depth(meshes, cams, np.float32, face_ids=True)
    assert [len(v) for v in views] == [1, 2] and views[1][1][0].shape == (1, 4)
    assert views[1][0][0].ravel().tolist() == [6, 7, 8, 9] and faces[1][1].ravel().tolist() == [-10, -11, -12, -13]
    assert views[1][1][1] is cams[1][1] or views[1][1][1].width == 4
    assert fake.calls[-1][2].tolist() == [0, 4, 8]
    v16 = ctx.render_depth(meshes, cams, np.uint16)
    assert v16[0][0][0].dtype == np.uint16
    with pytest.raises(TypeError):
        ctx.render_depth(meshes, cams, np.int8)
    with pytest.raises(ValueError):
        ctx.render_depth(meshes, cams[:1], np.float32)


def test_sample_meshes_counts_then_fills(monkeypatch):
    ctx, fake = fake_context(monkeypatch)
    meshes = [quad(-1, -1, 1, 1, 1, 1)] * 3
    off, xyz, nrm, face = ctx.sample_meshes(meshes, 1000.0, 7, face_ids=True)
    assert off.tolist() == [0, 3, 9, 18] and xyz.shape == (18, 3) and nrm.dtype == np.float64 and face.shape == (18,)
    assert [c[1] for c in fake.calls] == [False, True] and fake.calls[0][2:] == (1000.0, 7)
    assert xyz[off[1]:off[2], 0].tolist() == [1.0] * 6
