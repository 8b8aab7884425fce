"""numpy restatement of include/gpd_b200_sensor.h: the structured-light sensor model of gpdb_render_sensor_depth.

numpy's float64 elementwise operations are single IEEE roundings and never fuse a multiply and an add, so every value
below is the header's value bit for bit. The inverse-normal table is the library's own (gpdb_debug_sensor_table, which
needs no device); tests/sensor_oracle.cpp compiles the header's helpers for the host.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import render_reference as rr
from sis_reference import philox

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HERE = os.path.dirname(os.path.abspath(__file__))
SENSOR_STREAM = 5
FIELDS = ("baseline", "lateral_sigma", "disparity_sigma", "disparity_step", "min_cos_incidence", "shadow_tolerance",
          "dropout")


def table():
    """rule 2's table, as the library exports it"""
    from gpd_b200 import lib
    return lib.debug_sensor_table()


def params(sp):
    """a gpdb_sensor_params (or a dict) as a dict of floats"""
    return {f: float(sp[f] if isinstance(sp, dict) else getattr(sp, f)) for f in FIELDS}


def param_error(sp):
    """rule 9's parameter checks: the library's message for the first rule sp breaks, or None"""
    s = params(sp)
    for f in FIELDS:
        if not (s[f] >= 0) or not np.isfinite(s[f]):
            return f"{f} must be finite and >= 0"
    if s["dropout"] > 1:
        return "dropout must lie in [0, 1]"
    if s["shadow_tolerance"] >= 1:
        return "shadow_tolerance must be < 1"
    if s["min_cos_incidence"] > 1:
        return "min_cos_incidence must be <= 1"
    if (s["disparity_sigma"] > 0 or s["disparity_step"] > 0) and not s["baseline"] > 0:
        return "disparity_sigma and disparity_step need a baseline > 0"
    return None


def gauss(T, U):
    """rule 2: the draws of uniforms U in [0, 1)"""
    s = U * 4096.0
    i = s.astype(np.int64)
    f = s - i
    return T[i] + f * (T[i + 1] - T[i])


def draws(key, k, n):
    """rule 1 for pixel indices 0 .. n-1 of camera k: (g0, g1, g2, U)"""
    pix = np.arange(n, dtype=np.uint32)
    kk = (int(key) & 0xFFFFFFFF, (int(key) >> 32) & 0xFFFFFFFF)
    r = [philox(np.stack([pix, np.full_like(pix, k), np.full_like(pix, SENSOR_STREAM), np.full_like(pix, w)], 1), kk)
         for w in (0, 1)]
    return r[0], r[1]


def projector_pose(pose, baseline):
    """rule 5: the projector's camera-to-world pose"""
    p = np.array(pose, np.float64)
    for i in range(3):
        p[4 * i + 3] = pose[4 * i + 3] + baseline * pose[4 * i]
    return p


def clean(vertices, faces, cam, pose):
    """render rules 2 - 5 before the format conversion: (t [H*W], face [H*W]; inf and -1 where there is no hit)"""
    H, W = int(cam.height), int(cam.width)
    q = rr.to_camera(vertices, pose)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    recs = rr.setup(q[faces[:, 0]], q[faces[:, 1]], q[faces[:, 2]]) if len(faces) else np.zeros((0, 13))
    dx, dy = rr.rays(cam)
    bt = np.full(H * W, np.inf)
    bf = np.full(H * W, -1, np.int32)
    for f, rec in enumerate(recs):
        ok, t = rr.hit(rec, dx, dy)
        better = ok & (t < bt)
        bt[better] = t[better]
        bf[better] = f
    return bt, bf


def sensor_pixels(sp, T, key, k, cam, ct, cf, pt, pf, vertices, faces):
    """rules 1 and 3-7 for every pixel of one camera from its clean image (ct, cf) and its projector's (pt, pf): a dict of
    face [H*W] (-1: no return), z [H*W] (z'), and the intermediate du, dv (rule 3), D, Dp (rule 6, NaN unless reached)"""
    s = params(sp)
    H, W = int(cam.height), int(cam.width)
    n = H * W
    pose = rr.pose_of(cam)
    r0, r1 = draws(key, k, n)
    g0, g1 = gauss(T, rr.unit(r0[:, 0], r0[:, 1])), gauss(T, rr.unit(r0[:, 2], r0[:, 3]))
    g2, U = gauss(T, rr.unit(r1[:, 0], r1[:, 1])), rr.unit(r1[:, 2], r1[:, 3])
    v, u = np.divmod(np.arange(n), W)
    out = {"du": np.rint(s["lateral_sigma"] * g0), "dv": np.rint(s["lateral_sigma"] * g1)}
    with np.errstate(all="ignore"):
        su, sv = u + out["du"], v + out["dv"]
        ok = (su >= 0) & (su < W) & (sv >= 0) & (sv < H)
        ru, rv = np.where(ok, su, 0).astype(np.int64), np.where(ok, sv, 0).astype(np.int64)
        idx = rv * W + ru
        f = np.where(ok, cf[idx], -1)
        ok &= f >= 0
        t = np.where(ok, ct[idx], 1.0)
        dx, dy = (ru.astype(np.float64) - cam.cx) / cam.fx, (rv.astype(np.float64) - cam.cy) / cam.fy
        X = [t * dx, t * dy, t]
        if s["min_cos_incidence"] > 0:
            nw, _ = rr.face_normals(vertices, faces)
            nw = nw[np.maximum(f, 0)] if len(nw) else np.ones((n, 3))
            m = [(pose[i] * nw[:, 0] + pose[4 + i] * nw[:, 1]) + pose[8 + i] * nw[:, 2] for i in range(3)]
            mx = (m[0] * X[0] + m[1] * X[1]) + m[2] * X[2]
            mm, xx = (m[0] * m[0] + m[1] * m[1]) + m[2] * m[2], (X[0] * X[0] + X[1] * X[1]) + X[2] * X[2]
            c = np.abs(mx) / (np.sqrt(mm) * np.sqrt(xx))
            ok &= ~(c < s["min_cos_incidence"])
        z = X[2]
        out["D"] = out["Dp"] = np.full(n, np.nan)
        if s["baseline"] > 0:
            b = s["baseline"]
            pu = np.rint((cam.fx * (X[0] - b)) / X[2] + cam.cx)
            pv = np.rint((cam.fy * X[1]) / X[2] + cam.cy)
            inb = (pu >= 0) & (pu < W) & (pv >= 0) & (pv < H)
            pidx = np.where(inb, pv * W + pu, 0).astype(np.int64)
            ok &= inb & (pf[pidx] >= 0) & ~(pt[pidx] < X[2] * (1.0 - s["shadow_tolerance"]))
            fb = cam.fx * b
            D = fb / X[2]
            Dp = D + s["disparity_sigma"] * g2
            if s["disparity_step"] > 0:
                Dp = s["disparity_step"] * np.rint(Dp / s["disparity_step"])
            out["D"], out["Dp"] = np.where(ok, D, np.nan), np.where(ok, Dp, np.nan)
            ok &= (Dp > 0) & np.isfinite(Dp)
            z = fb / Dp
        ok &= ~(U < s["dropout"])
    out["face"] = np.where(ok, f, -1).astype(np.int32)
    out["z"] = np.where(ok, z, np.inf)
    return out


def sensor_camera(vertices, faces, cam, k, key, sp, T, fmt, detail=False):
    """rules 1-8 for camera k of a view with key `key`: (image [H, W], face image [H, W][, the sensor_pixels dict])"""
    H, W = int(cam.height), int(cam.width)
    pose = rr.pose_of(cam)
    ct, cf = clean(vertices, faces, cam, pose)
    b = params(sp)["baseline"]
    pt, pf = clean(vertices, faces, cam, projector_pose(pose, b)) if b > 0 else (ct, cf)
    px = sensor_pixels(sp, T, key, k, cam, ct, cf, pt, pf, vertices, faces)
    raw, ret = rr.raw_of(px["z"], cam.depth_scale, fmt)
    face = np.where(ret, px["face"], -1).astype(np.int32)
    res = (raw.reshape(H, W), face.reshape(H, W))
    return res + (px,) if detail else res


def render(meshes, cameras_per_view, sp, seed, fmt, T=None):
    """every view's cameras, view b with the key seed + b: ([image per camera], [face image per camera]) per view"""
    T = table() if T is None else T
    out = []
    for b, ((v, f), cams) in enumerate(zip(meshes, cameras_per_view)):
        key = (int(seed) + b) % 2 ** 64
        r = [sensor_camera(v, f, c, k, key, sp, T, fmt) for k, c in enumerate(cams)]
        out.append(([x[0] for x in r], [x[1] for x in r]))
    return out


def table_std(T):
    """the standard deviation of rule 2's draws: the piecewise-linear distribution of g = T[i] + f (T[i+1] - T[i])"""
    a, b = T[:-1], T[1:]
    return float(np.sqrt(((a * a + a * b + b * b) / 3.0).sum() / 4096.0))


def table_cdf(T, x):
    """P(g <= x) of rule 2's draws"""
    x = np.asarray(x, np.float64)
    i = np.clip(np.searchsorted(T, x, side="right") - 1, 0, 4095)
    with np.errstate(all="ignore"):
        f = np.where(T[i + 1] > T[i], (x - T[i]) / (T[i + 1] - T[i]), 1.0)
    return np.where(x < T[0], 0.0, np.where(x >= T[-1], 1.0, (i + np.clip(f, 0, 1)) / 4096.0))


# ---- the header's helpers compiled for the host ---------------------------------------------------------------------

def cpp():
    so = os.path.join(tempfile.mkdtemp(prefix="sensor_oracle_"), "libsensor_oracle.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), "-o", so, os.path.join(_HERE, "sensor_oracle.cpp")])
    L = C.CDLL(so)
    L.so_table.argtypes = [C.c_void_p]
    L.so_gauss.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.so_pixels.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p] + [C.c_void_p] * 6 + \
        [C.c_void_p, C.c_void_p]
    return L


def host_pixels(L, sp, T, key, k, cam, ct, cf, pt, pf, vertices, faces):
    """gpdb_sensor_pixel of every pixel through the host build: (face [H*W], z [H*W], inf where no return)"""
    from gpd_b200 import abi
    n = int(cam.width) * int(cam.height)
    p = abi.SensorParams(**params(sp))
    cam_ = (abi.DepthCamera * 1)(cam)
    face, z = np.zeros(n, np.int32), np.zeros(n, np.float64)
    arrs = [np.ascontiguousarray(a) for a in (np.asarray(T, np.float64), np.asarray(ct, np.float64), np.asarray(cf, np.int32),
                                             np.asarray(pt, np.float64), np.asarray(pf, np.int32),
                                             np.asarray(vertices, np.float32).reshape(-1, 3),
                                             np.asarray(faces, np.int32).reshape(-1, 3))]
    L.so_pixels(C.c_void_p(C.addressof(p)), rr.p_(arrs[0]), C.c_uint64(int(key)), C.c_uint32(k), C.cast(cam_, C.c_void_p),
                *[rr.p_(a) for a in arrs[1:]], rr.p_(face), rr.p_(z))
    return face, np.where(face >= 0, z, np.inf)
