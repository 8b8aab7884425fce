"""numpy restatement of include/gpd_b200_organized.h (test infrastructure only), and the loader of its C++ restatement
tests/organized_oracle.cpp, built on first use into a temporary directory against the oracle's libgpd_oracle.so (its
pcl::eigen33). The sequential passes of rules 3 and 4 run here as wavefronts over anti-diagonals: every value is
computed from the same operands with the same rounded operations, and numpy's float32 / float64 elementwise arithmetic
rounds each operation on its own."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np

F, D = np.float32, np.float64
_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
BORDER, SMOOTHING = 20, F(20.0)


def pair_breaks(a, b):
    """Rule 2 for pixel depths a (the loop's pixel) and b."""
    with np.errstate(invalid="ignore"):
        t = (F(0.02) * (np.abs(a) + F(1.0))) * F(2.0)
        return (np.abs(a - b) > t) | ~np.isfinite(a) | ~np.isfinite(b)


def change_map(z):
    """Rule 2: 1 = no depth change, 0 = a pair test touching the pixel failed."""
    z = np.asarray(z, F)
    H, W = z.shape
    ch = np.ones((H, W), np.uint8)
    h = pair_breaks(z[:H - 1, :W - 1], z[:H - 1, 1:W])
    v = pair_breaks(z[:H - 1, :W - 1], z[1:H, :W - 1])
    ch[:H - 1, :W - 1][h | v] = 0
    ch[:H - 1, 1:W][h] = 0
    ch[1:H, :W - 1][v] = 0
    return ch


def chamfer(d0, s0, s1, d1):
    a, b, c, d = d0 + F(1.4), s0 + F(1.0), s1 + F(1.0), d1 + F(1.4)
    m0 = np.where(b < a, b, a)
    m1 = np.where(d < c, d, c)
    return np.where(m1 < m0, m1, m0)


def distance_map(z):
    """Rule 3 over the flat array, pass 1 at t = (c-1) + 2(r-1), pass 2 at t = (W-2-c) + 2(H-2-r)."""
    H, W = z.shape
    flat = np.where(change_map(z) == 0, F(0.0), F(W + H)).astype(F).ravel()
    if W < 2 or H < 2:
        return flat.reshape(H, W)
    steps = (W - 2) + 2 * (H - 2) + 1
    rows = np.arange(1, H)
    for t in range(steps):
        c = t - 2 * (rows - 1) + 1
        ok = (c >= 1) & (c < W)
        r, c = rows[ok], c[ok]
        i = r * W + c
        m = chamfer(flat[i - W - 1], flat[i - W], flat[i - 1], flat[i - W + 1])
        flat[i] = np.where(m < flat[i], m, flat[i])
    js = np.arange(H - 1)
    for t in range(steps):
        r, c = H - 2 - js, W - 2 - t + 2 * js
        ok = (c >= 0) & (c <= W - 2)
        r, c = r[ok], c[ok]
        i = r * W + c
        m = chamfer(flat[i + W - 1], flat[i + W], flat[i + 1], flat[i + W + 1])
        flat[i] = np.where(m < flat[i], m, flat[i])
    return flat.reshape(H, W)


def integral_tables(xyz):
    """Rule 4: (sums [9, H+1, W+1] float64 (x y z xx xy xz yy yz zz), counts [H+1, W+1] int64), at t = r + c."""
    xyz = np.asarray(xyz, F)
    H, W, _ = xyz.shape
    x, y, z = xyz[..., 0], xyz[..., 1], xyz[..., 2]
    with np.errstate(invalid="ignore", over="ignore"):
        fin = np.isfinite((x + y) + z)
        add = np.stack([x.astype(D), y.astype(D), z.astype(D), (x * x).astype(D), (x * y).astype(D), (x * z).astype(D),
                        (y * y).astype(D), (y * z).astype(D), (z * z).astype(D)])
    S = np.zeros((9, H + 1, W + 1), D)
    N = np.zeros((H + 1, W + 1), np.int64)
    rows = np.arange(H)
    for t in range(W + H - 1):
        c = t - rows
        ok = (c >= 0) & (c < W)
        r, c = rows[ok], c[ok]
        v = (S[:, r, c + 1] + S[:, r + 1, c]) - S[:, r, c]
        f = fin[r, c]
        with np.errstate(invalid="ignore"):
            v = np.where(f, v + add[:, r, c], v)
        S[:, r + 1, c + 1] = v
        N[r + 1, c + 1] = N[r, c + 1] + N[r + 1, c] - N[r, c] + f
    return S, N


def normals(xyz, vp=(0.0, 0.0, 0.0)):
    """Rules 2 - 5 of one [H, W, 3] cloud: (normals [H, W, 3] float32, distance map [H, W] float32)."""
    from oracle import oracle
    xyz = np.asarray(xyz, F)
    H, W, _ = xyz.shape
    vp = np.asarray(vp, F)
    dist = distance_map(xyz[..., 2])
    S, N = integral_tables(xyz)
    out = np.full((H, W, 3), np.nan, F)
    for r in range(BORDER, H - BORDER):
        for c in range(BORDER, W - BORDER):
            q = xyz[r, c]
            if not np.isfinite(q[2]):
                continue
            s = SMOOTHING if SMOOTHING < dist[r, c] else dist[r, c]
            if not s > F(2.0):
                continue
            w = int(s)
            x0, y0 = c - w // 2, r - w // 2
            cnt = int(((N[y0 + w, x0 + w] + N[y0, x0]) - N[y0, x0 + w]) - N[y0 + w, x0])
            if cnt == 0:
                continue
            sm = ((S[:, y0 + w, x0 + w] + S[:, y0, x0]) - S[:, y0, x0 + w]) - S[:, y0 + w, x0]
            ctr = sm[:3].astype(F)
            so = sm[3:].astype(F)
            cov = np.zeros((3, 3), F)
            for e, (i, j) in enumerate([(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]):
                cov[i, j] = cov[j, i] = so[e] - (ctr[i] * ctr[j]) / F(cnt)
            _, n = oracle.pcl_eigen33(cov)
            n = n.astype(F)
            v = vp - q
            if (v[0] * n[0] + v[1] * n[1]) + v[2] * n[2] < F(0):
                n = -n
            out[r, c] = n
    return out, dist


def rotate(R, n):
    """Rule 6: float32 normals [..., 3] by the row-major 3 x 3 R, each row one double chain and one rounding."""
    R = np.asarray(R, D).reshape(3, 3)
    n = np.asarray(n, F).astype(D)
    with np.errstate(invalid="ignore"):
        return np.stack([((R[i, 0] * n[..., 0] + R[i, 1] * n[..., 1]) + R[i, 2] * n[..., 2]) for i in range(3)], -1).astype(F)


@functools.lru_cache(None)
def cpp():
    from oracle import oracle
    oracle.lib()  # builds oracle/libgpd_oracle.so if needed
    odir = os.path.join(ROOT, "oracle")
    so = os.path.join(tempfile.mkdtemp(prefix="organized_oracle_"), "liborganized_oracle.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                           "-o", so, os.path.join(_HERE, "organized_oracle.cpp"), "-L", odir, "-lgpd_oracle",
                           "-Wl,-rpath," + odir])
    L = C.CDLL(so)
    L.org_oracle_normals.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4
    L.org_oracle_rotate.argtypes = [C.c_int] + [C.c_void_p] * 3
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cpp_normals(xyz, vp=(0.0, 0.0, 0.0)):
    """normals() by the C++ restatement (fast enough for full-size images)."""
    xyz = np.ascontiguousarray(xyz, F)
    H, W, _ = xyz.shape
    vp = np.ascontiguousarray(vp, F)
    nrm, dist = np.zeros((H, W, 3), F), np.zeros((H, W), F)
    cpp().org_oracle_normals(W, H, _p(xyz), _p(vp), _p(nrm), _p(dist))
    return nrm, dist


def camera_cloud(raw, cam, fmt):
    """Rule 6: a depth image as its camera's organized cloud, the camera-frame points [H, W, 3] of gpd_b200_depth.h rule 2
    (no pose), NaN for an invalid pixel."""
    import depth_reference as dr
    H, W = raw.shape
    z, valid = dr.pixel_valid(raw, fmt, cam.depth_scale, cam.min_depth, cam.max_depth)
    u, v = np.meshgrid(np.arange(W, dtype=F), np.arange(H, dtype=F))
    with np.errstate(over="ignore", invalid="ignore"):
        xc = ((u - F(cam.cx)) * z) / F(cam.fx)
        yc = ((v - F(cam.cy)) * z) / F(cam.fy)
    out = np.stack([xc, yc, z], -1).astype(F)
    out[~valid] = np.nan
    return out
