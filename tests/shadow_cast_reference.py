"""A numpy restatement of the shadow casting of the 15-channel grasp images, per image and camera, as the image kernels
do it (gpd_b200/csrc/geometry.cu, by symbol; include/gpd_b200_shadow.h):

* ball_scan1: the float32 image ball, its count, the camera set (cam_or) and the float64 centre;
* shadow_setup: the bitmap AABB (bm_org / bm_dims, clamped at bm_dim) and the float32 invariants fs, fR, fbx_lo / hi,
  cull_lo / hi and cull_inv;
* cull: the float32 slab test of a point's shadow segment and its LCG window [r0, r1];
* cast_camera: the window test of every draw (the work list counts wl_n, the draw list counts dl_n);
* draw_bit: the float64 voxel, the AABB test and the float32 pre-test;
* intersect_bitmaps: the per-camera bitmaps intersected over the camera set, starting from camera 0's set even when
  camera 0 does not see the neighbourhood;
* the set bits (nset_all) and the subset whose jittered point passes the exact float64 box test.

Every float32 operation is a numpy float32 operation (correctly rounded); fmaf is fmaf() below. The centre is the float64
sum of float32 coordinates, which the kernel forms in warp-reduction order: cast() refuses a neighbourhood whose sum is
not exact in every order (centre_is_exact), so that the order does not matter. Draws follow the sequential LCG of
gpdb_fastrand; the kernels' skip-ahead tables must reproduce it."""
import math
from fractions import Fraction

import numpy as np

from image_reference import VOXEL, neighbourhood, norm_quantile_table, to_frame, in_box, _mix32

F32 = np.float32


def fmaf(a, b, c):
    """fmaf over float32 arrays (broadcast): a b is exact in float64, so the float64 sum a b + c is rounded once; its
    rounding to float32 is then correct unless it lies on a float32 midpoint, where the exact value decides."""
    a, b, c = np.broadcast_arrays(np.asarray(a, F32), np.asarray(b, F32), np.asarray(c, F32))
    shape = a.shape
    a, b, c = a.reshape(-1), b.reshape(-1), c.reshape(-1)
    with np.errstate(invalid="ignore", over="ignore"):
        r = a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)
        out = np.array(r.astype(F32))
        other = np.nextafter(out, np.where(r > out, F32(np.inf), F32(-np.inf)).astype(F32))
        mid = (r != out.astype(np.float64)) & (r == (out.astype(np.float64) + other.astype(np.float64)) / 2.0)
    for i in zip(*np.nonzero(mid)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        m = Fraction(float(r[i]))
        lo, hi = sorted([out[i], other[i]])
        if exact > m:
            out[i] = hi
        elif exact < m:
            out[i] = lo
        else:
            out[i] = lo if (int(np.array(lo, F32).view(np.uint32)) & 1) == 0 else hi
    return out.reshape(shape)


def centre_is_exact(pts):
    """True when every float64 partial sum of the float32 coordinates pts [n, 3], in any order, is exact: all of them
    are multiples of one power of two 2^-e and the sum of their magnitudes stays below 2^53 of those units."""
    v = np.abs(np.asarray(pts, np.float64))
    for e in range(0, 160):
        s = v * 2.0 ** e
        if np.array_equal(s, np.floor(s)):
            return bool(s.sum(0).max() < 2.0 ** 53)
    return False


class Params:
    """The DevParams a 15-channel geometry gives (api.cu fill_dev_params)."""

    def __init__(self, g):
        self.g = g
        self.r = g.radius
        self.shadow_length = g.radius
        self.vox_mult = 1.0 / VOXEL
        self.nsp = int(math.floor(self.shadow_length / VOXEL))
        diag = math.sqrt(g.d * g.d + g.w * g.w + 4.0 * g.h * g.h)
        self.bm_dim = int(math.ceil((diag + 2.0 * 3.2 * VOXEL * 0.3) / VOXEL)) + 4


def shadow_setup(P, pose, center, vp, gmax):
    """The bitmap AABB and the float32 invariants of the image (shadow_setup), and per camera the shadow vector and the
    slab reciprocals cull_inv."""
    g = P.g
    F = np.asarray(pose["frame"], np.float64).ravel()
    smp = np.asarray(pose["sample"], np.float64).ravel()
    bottom, cen = float(pose["bottom"]), float(pose["center"])
    half_od = g.w / 2.0
    st = {}
    wv = np.zeros((8, 3))
    for cr in range(8):
        cx = bottom + g.d if cr & 1 else bottom
        cy = cen + half_od if cr & 2 else cen - half_od
        cz = g.h if cr & 4 else -g.h
        for r in range(3):
            wv[cr, r] = F[r] * cx + F[3 + r] * cy + F[6 + r] * cz + smp[r]
    mn, mx = wv.min(0), wv.max(0)
    jmax = gmax * VOXEL * 0.3 + 1e-9
    lo = np.array([int(math.floor((mn[a] - jmax) * P.vox_mult)) - 1 for a in range(3)])
    hi = np.array([int(math.floor((mx[a] + jmax) * P.vox_mult)) + 1 for a in range(3)])
    st["aabb_lo"], st["aabb_hi"] = lo, hi
    st["bm_org"] = lo
    st["bm_dims"] = np.minimum(hi - lo + 1, P.bm_dim)
    st["fs"] = smp.astype(F32)
    jm = F32(gmax * VOXEL * 0.3 * 1.7320508075688772 + 2e-5)
    st["fbx_lo"] = np.array([F32(bottom), F32(cen - g.w / 2.0), F32(-g.h)], F32) - jm
    st["fbx_hi"] = np.array([F32(bottom + g.d), F32(cen + g.w / 2.0), F32(g.h)], F32) + jm
    wm = 0.0105
    bx_lo = [bottom - wm, cen - g.w / 2.0 - wm, -g.h - wm]
    bx_hi = [bottom + g.d + wm, cen + g.w / 2.0 + wm, g.h + wm]
    st["cull_lo"] = np.array(bx_lo, np.float64).astype(F32) - F32(1e-5)
    st["cull_hi"] = np.array(bx_hi, np.float64).astype(F32) + F32(1e-5)
    st["fR"] = F.astype(F32)
    sv, inv = [], []
    for k in range(len(vp)):
        s = center - vp[k]
        nn = math.sqrt((s[0] * s[0] + s[1] * s[1]) + s[2] * s[2])
        v = np.array([P.shadow_length * s[a] / nn for a in range(3)])
        sv.append(v)
        svh = to_frame(F, v[None])[0]
        dv = svh.astype(F32)
        with np.errstate(divide="ignore"):
            inv.append(np.where(np.abs(dv) < F32(1e-6), F32(0.0), F32(1.0) / dv).astype(F32))
    st["sv"], st["cull_inv"] = sv, inv
    return st


def _frame_f32(fR, w):
    """fmaf(fR[3r], wx, fmaf(fR[3r+1], wy, fR[3r+2] wz)) for r = 0, 1, 2 (w: float32 [n, 3])."""
    return np.stack([fmaf(fR[3 * r], w[:, 0], fmaf(fR[3 * r + 1], w[:, 1], fR[3 * r + 2] * w[:, 2])) for r in range(3)], 1)


def cull(st, k, p32):
    """The slab cull of camera k for float32 points p32 [n, 3]: (passes [n], r0 [n], r1 [n])."""
    w = (p32 - st["fs"][None]).astype(F32)
    o3 = _frame_f32(st["fR"], w)
    inv = st["cull_inv"][k]
    n = len(p32)
    tmin, tmax = np.zeros(n, F32), np.ones(n, F32)
    hit = np.ones(n, bool)
    for a in range(3):
        lo, hi = st["cull_lo"][a], st["cull_hi"][a]
        if inv[a] == 0.0:
            hit &= (o3[:, a] >= lo) & (o3[:, a] <= hi)
        else:
            t1 = ((lo - o3[:, a]).astype(F32) * inv[a]).astype(F32)
            t2 = ((hi - o3[:, a]).astype(F32) * inv[a]).astype(F32)
            tmin = np.maximum(tmin, np.minimum(t1, t2))
            tmax = np.minimum(tmax, np.maximum(t1, t2))
    ok = hit & ~(tmin > tmax)
    with np.errstate(invalid="ignore", over="ignore"):
        r0 = np.maximum(np.floor((tmin * F32(32767.0)).astype(F32)).astype(np.int64) - 1, 0)
        r1 = np.minimum(np.ceil((tmax * F32(32767.0)).astype(F32)).astype(np.int64) + 1, 32767)
    return ok, np.where(ok, r0, 0), np.where(ok, r1, -1)


def voxels(P, pts64, r, sv):
    """draw_bit's float64 voxel of draws with LCG values r [n] of points pts64 [n, 3]: trunc((p + u sv) vox_mult)."""
    u = r.astype(np.float64) * (1.0 / 32767.0)
    return np.trunc((pts64 + u[:, None] * sv[None, :]) * P.vox_mult).astype(np.int64)


def pretest(st, v):
    """draw_bit's float32 pre-test of voxel lattice points v [n, 3] against the box widened by the largest jitter."""
    w = fmaf(v.astype(F32), F32(0.003), -st["fs"][None])
    h = _frame_f32(st["fR"], w)
    return ((h >= st["fbx_lo"][None]) & (h <= st["fbx_hi"][None])).all(1)


def draw_codes(P, st, v):
    """Bit codes b0 + 64 (b1 + d1 b2) of voxels v [n, 3] in the bitmap, -1 where draw_bit rejects them."""
    b = v - st["bm_org"][None]
    d = st["bm_dims"]
    inside = ((b >= 0) & (b < d[None])).all(1)
    ok = inside.copy()
    if inside.any():
        ok[inside] = pretest(st, v[inside])
    return np.where(ok, b[:, 0] + 64 * (b[:, 1] + d[1] * b[:, 2]), -1)


def shadow_seed(sample_index, idx, k):
    return _mix32((np.uint64(np.uint32(sample_index)) * 0x9E3779B1 + np.asarray(idx).astype(np.uint64) * 0x85EBCA77
                   + np.uint64(k) * 0xC2B2AE3D) & 0xFFFFFFFF)


def cast_camera(P, st, p32, idx, k, sample_index, raw=False):
    """Camera k's casting of the ball points p32 [n, 3] (cloud indices idx): per point whether it enters the work list
    and how many of its draws pass the window; the set bit codes. raw: also every draw's voxel without any filter."""
    ok, r0, r1 = cull(st, k, p32)
    seed = shadow_seed(sample_index, idx, k)
    pts64 = p32.astype(np.float64)
    dl = np.zeros(len(p32), np.int64)
    codes, raw_v = [], []
    for _ in range(P.nsp):
        seed = (seed * 214013 + 2531011) & 0xFFFFFFFF
        r = ((seed >> 16) & 0x7FFF).astype(np.int64)
        win = ok & (r >= r0) & (r <= r1)
        dl += win
        if raw:
            raw_v.append(voxels(P, pts64, r, st["sv"][k]))
        if win.any():
            c = draw_codes(P, st, voxels(P, pts64[win], r[win], st["sv"][k]))
            codes.append(c[c >= 0])
    out = {"work": ok, "draws": dl, "codes": np.unique(np.concatenate(codes)) if codes else np.zeros(0, np.int64)}
    if raw:
        out["raw"] = np.concatenate(raw_v) if raw_v else np.zeros((0, 3), np.int64)
    return out


def voxel_points(v, qtab):
    """voxel -> jittered point (voxel_point_in_box, hand_set.cpp:196-199)."""
    hsh = _mix32(((v[:, 0].astype(np.uint64) & 0xFFFFFFFF) * 73856093 & 0xFFFFFFFF) ^
                 ((v[:, 1].astype(np.uint64) & 0xFFFFFFFF) * 19349663 & 0xFFFFFFFF) ^
                 ((v[:, 2].astype(np.uint64) & 0xFFFFFFFF) * 83492791 & 0xFFFFFFFF))
    g = np.asarray(qtab)[(hsh & 1023).astype(np.int64)]
    return v.astype(np.float64) * VOXEL + (1.0 * g * VOXEL * 0.3)[:, None]


def points_in_box(g, pose, pts):
    if len(pts) == 0:
        return np.zeros(0, bool)
    return in_box(g, pose, to_frame(pose["frame"], pts - np.asarray(pose["sample"], np.float64)))


def cast(cloud, pose, g, qtab=None, raw=False, index=None):
    """The shadow casting of one image (pose: one POSE_DTYPE record) at 15 channels. Returns a dict:
    n_ball, cam_or, center, per camera wl_n / dl_n (lists of K; 0 for a camera outside the camera set), the per-point
    work-list flags and draw counts of each cast camera (cams[k]: None when not cast), nset_all, voxels (the set bits
    as world voxels [nset_all, 3]), in_box (their jittered points inside the image box, sorted by voxel) and the
    shadow_setup invariants (setup). raw: cams[k]["raw"] holds every draw's voxel without any filter. index: the
    indices of cloud's points in the kernel's cloud (the LCG seeds), when cloud is a part of it."""
    qtab = norm_quantile_table() if qtab is None else np.asarray(qtab)
    P = Params(g)
    idx, _ = neighbourhood(cloud, pose["sample"], g.radius)
    p32 = np.asarray(cloud["xyz"], F32)[idx]
    vp = np.asarray(cloud["view_points"], np.float64).reshape(-1, 3)
    K = len(vp)
    cam = np.asarray(cloud["cam_source"]).reshape(len(cloud["xyz"]), -1)[idx] > 0
    n = len(idx)
    out = {"n_ball": n, "K": K, "wl_n": [0] * K, "dl_n": [0] * K, "cams": [None] * K, "nset_all": 0,
           "voxels": np.zeros((0, 3), np.int64), "in_box": np.zeros((0, 3)), "cam_or": 0}
    if n == 0:
        return out
    assert centre_is_exact(p32), "the float64 sum of the neighbourhood is not exact in every order"
    center = p32.astype(np.float64).sum(0) / float(n)
    cam_or = int(sum(1 << k for k in range(K) if cam[:, k].any()))
    st = shadow_setup(P, pose, center, vp, float(qtab[-1]))
    out.update(cam_or=cam_or, center=center, setup=st, params=P)
    for k in range(K):
        if not (cam_or >> k) & 1:
            continue
        c = cast_camera(P, st, p32, idx if index is None else np.asarray(index)[idx], k, int(pose["sample_index"]), raw)
        out["cams"][k] = c
        out["wl_n"][k] = int(c["work"].sum())
        out["dl_n"][k] = int(c["draws"].sum())
    acc = out["cams"][0]["codes"] if out["cams"][0] is not None else np.zeros(0, np.int64)
    for k in range(1, K):
        if out["cams"][k] is not None:
            acc = np.intersect1d(acc, out["cams"][k]["codes"])
    d1 = int(st["bm_dims"][1])
    b = np.stack([acc % 64, (acc // 64) % d1, acc // 64 // d1], 1)
    v = b + st["bm_org"][None]
    out["nset_all"] = len(acc)
    out["voxels"] = v
    pts = voxel_points(v, qtab)
    m = points_in_box(g, pose, pts)
    order = np.lexsort((v[m][:, 2], v[m][:, 1], v[m][:, 0]))
    out["in_box"] = pts[m][order]
    return out


def listed_draws_bounds(res, k, cap):
    """(least, most) dl_n of camera k when its work list holds only `cap` of its wl_n points: which ones it holds follows
    the kernel's scan order. Exact (least == most) when wl_n <= cap or every listed point has as many window draws."""
    c = res["cams"][k]
    d = np.sort(c["draws"][c["work"]])
    if len(d) <= cap:
        return int(d.sum()), int(d.sum())
    return int(d[:cap].sum()), int(d[-cap:].sum())
