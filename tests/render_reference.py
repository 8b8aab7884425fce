"""numpy restatement of include/gpd_b200_render.h: the depth rendering of triangle meshes and their surface samples.

numpy's float64 elementwise operations are single IEEE roundings and never fuse a multiply and an add, so every value
below is the header's value bit for bit. tests/render_oracle.cpp compiles the header's own helpers for the host.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from sis_reference import philox

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HERE = os.path.dirname(os.path.abspath(__file__))
MESH_STREAM = 4


def cross(a, b):
    """rule 1, rows of a x rows of b"""
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1],
                     a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def pose_of(cam):
    return np.array(cam.pose[:], np.float64)


def to_camera(vertices, pose):
    """rule 2: float32 world vertices [V, 3] -> float64 camera frame"""
    p = np.asarray(vertices, np.float32).astype(np.float64)
    d = [p[:, 0] - pose[3], p[:, 1] - pose[7], p[:, 2] - pose[11]]
    return np.stack([(pose[i] * d[0] + pose[4 + i] * d[1]) + pose[8 + i] * d[2] for i in range(3)], 1)


def rays(cam):
    """rule 3: (dx, dy) of every pixel, [H*W] each, row-major"""
    H, W = int(cam.height), int(cam.width)
    v, u = np.divmod(np.arange(H * W), W)
    return (u.astype(np.float64) - cam.cx) / cam.fx, (v.astype(np.float64) - cam.cy) / cam.fy


def setup(A, B, C_):
    """rule 4: [F, 13] = m0, m1, m2, n, h of the faces with camera-frame vertices A, B, C [F, 3]"""
    n = cross(B - A, C_ - A)
    h = (n[:, 0] * A[:, 0] + n[:, 1] * A[:, 1]) + n[:, 2] * A[:, 2]
    return np.concatenate([cross(A, B), cross(B, C_), cross(C_, A), n, h[:, None]], 1)


def hit(rec, dx, dy):
    """rule 4 for one face record and arrays of rays: (covers, t)"""
    e = [(rec[3 * k] * dx + rec[3 * k + 1] * dy) + rec[3 * k + 2] for k in range(3)]
    s = (rec[9] * dx + rec[10] * dy) + rec[11]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        t = rec[12] / s
        ok = (s != 0) & (((e[0] >= 0) & (e[1] >= 0) & (e[2] >= 0)) | ((e[0] <= 0) & (e[1] <= 0) & (e[2] <= 0)))
        ok &= np.isfinite(t) & (t > 0)
    return ok, t


def raw_of(t, scale, fmt):
    """rule 5: (raw values, is a return) of hit distances t (no hit: t = inf)"""
    with np.errstate(over="ignore", invalid="ignore"):
        q = t / scale
        if fmt == 1:
            raw = q.astype(np.float32)
            ret = np.isfinite(raw) & (raw > 0)
            return np.where(np.isfinite(t), raw, np.float32(0)), ret & np.isfinite(t)
        r = np.rint(q)
        ret = np.isfinite(t) & (r >= 1) & (r <= 65535)
        return np.where(ret, r, 0).astype(np.uint16), ret


def render_camera(vertices, faces, cam, fmt):
    """rules 2 - 5 for one camera: (image [H, W], face image [H, W] int32)"""
    H, W = int(cam.height), int(cam.width)
    q = to_camera(vertices, pose_of(cam))
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    recs = setup(q[faces[:, 0]], q[faces[:, 1]], q[faces[:, 2]]) if len(faces) else np.zeros((0, 13))
    dx, dy = rays(cam)
    bt = np.full(H * W, np.inf)
    bf = np.full(H * W, -1, np.int32)
    for f, rec in enumerate(recs):
        ok, t = hit(rec, dx, dy)
        better = ok & (t < bt)  # faces in increasing index: a tie keeps the smaller one
        bt[better] = t[better]
        bf[better] = f
    raw, ret = raw_of(bt, cam.depth_scale, fmt)
    return raw.reshape(H, W), np.where(ret, bf, -1).astype(np.int32).reshape(H, W)


def render(meshes, cameras_per_view, fmt):
    """every view's cameras: ([image per camera], [face image per camera]) per view"""
    return [tuple(map(list, zip(*[render_camera(v, f, c, fmt) for c in cams]))) for (v, f), cams in zip(meshes, cameras_per_view)]


# ---- rule 6 ----------------------------------------------------------------------------------------------------------

def unit(x, y):
    return ((x.astype(np.uint64) << np.uint64(32) | y.astype(np.uint64)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def draws(key, f, j):
    f = np.asarray(f, np.uint32)
    j = np.broadcast_to(np.asarray(j, np.uint32), f.shape)
    ctr = np.stack([f, j, np.full_like(f, MESH_STREAM), np.zeros_like(f)], 1)
    return philox(ctr, (int(key) & 0xFFFFFFFF, (int(key) >> 32) & 0xFFFFFFFF))


def face_normals(vertices, faces):
    """(n [F, 3], L [F]) in float64 from the float32 vertices"""
    v = np.asarray(vertices, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = cross(b - a, c - a)
    return n, np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])


def counts(vertices, faces, density, key):
    n, L = face_normals(vertices, faces)
    F = len(L)
    d = draws(key, np.arange(F), 0)
    with np.errstate(over="ignore", invalid="ignore"):
        c = np.floor((0.5 * L) * density + unit(d[:, 0], d[:, 1]))
    c[~(L > 0) | ~np.isfinite(L)] = 0
    return c


def sample_mesh(vertices, faces, density, key):
    """one mesh: (xyz [n, 3] float32, normals [n, 3] float64, face [n] int32)"""
    v = np.asarray(vertices, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    cnt = counts(vertices, faces, density, key).astype(np.int64)
    n, L = face_normals(vertices, faces)
    fi = np.repeat(np.arange(len(f)), cnt)
    k = np.arange(len(fi)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    d = draws(key, fi, k + 1)
    r1, r2 = unit(d[:, 0], d[:, 1]), unit(d[:, 2], d[:, 3])
    s = np.sqrt(r1)
    w0, w1, w2 = 1.0 - s, s * (1.0 - r2), s * r2
    a, b, c = v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]]
    p = (w0[:, None] * a + w1[:, None] * b) + w2[:, None] * c
    return p.astype(np.float32), n[fi] / L[fi, None], fi.astype(np.int32)


def sample_meshes(meshes, density, seed):
    """the batch: (point offsets [B+1], xyz, normals, face), mesh b with key seed + b"""
    out = [sample_mesh(v, f, density, (seed + b) & 0xFFFFFFFFFFFFFFFF) for b, (v, f) in enumerate(meshes)]
    off = np.zeros(len(out) + 1, np.int32)
    off[1:] = np.cumsum([len(o[0]) for o in out])
    return (off, np.concatenate([o[0] for o in out]).reshape(-1, 3), np.concatenate([o[1] for o in out]).reshape(-1, 3),
            np.concatenate([o[2] for o in out]))


# ---- the header's helpers compiled for the host ---------------------------------------------------------------------

def cpp():
    so = os.path.join(tempfile.mkdtemp(prefix="render_oracle_"), "librender_oracle.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), "-o", so, os.path.join(_HERE, "render_oracle.cpp")])
    L = C.CDLL(so)
    L.ro_to_camera.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.ro_setup_hit.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.ro_raw.argtypes = [C.c_int, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p]
    L.ro_mesh.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def p_(a):
    return a.ctypes.data_as(C.c_void_p)
