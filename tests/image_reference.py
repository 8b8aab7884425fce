"""Two exact restatements of the grasp-image stage (A8, A10-A13) in numpy, for any image size, image volume and channel
count (1, 3, 12, 15):

* mode "reference": the oracle's semantics (ImageStrategy, image_strategy.cpp:32-233): cells by the reference formulas,
  a float32 running mean per cell, createNormalsImage's fold in the neighbourhood's (distance, index) order;
* mode "kernel": the arithmetic the image kernels specify (gpd_b200/csrc/geometry.cu: to_frame, unit_axis, unit_q32,
  cell_mean, the winner of a cell by key, the exact fold on a cloud with a normal of other than unit length).

Both share the output stage of the kernels (Quant, fully_covered, dilated_min, dilate_assemble), which equals the
reference's cv::dilate -> cv::normalize -> convertTo because the quantisation is monotone. `fault=` emulates one kernel
fault at a time (FAULTS). The shadow point set follows the deterministic variant of include/gpd_b200_shadow.h."""
import math
from fractions import Fraction

import numpy as np

DBL_EPSILON = np.finfo(np.float64).eps
RCP_N = 64            # geometry.cu: RCP_N = (NT_IMG / 32) * 4, the reciprocal table of cell_mean
VOXEL = 0.003         # GPDB_SHADOW_VOXEL
PROJ = [(0, 1, 2), (2, 1, 0), (2, 0, 1)]   # Proj(pj): (row axis, column axis, depth axis)

FAULTS = {
    "a": "general path skipped: the minimum is taken as 0 on covered groups",
    "b": "fully_covered evaluates border windows unclipped (cells outside the image count as occupied)",
    "c": "fully_covered ignores the third occupancy word a row can straddle (occf[w + 2])",
    "d": "no DBL_EPSILON branch in Quant",
    "e": "the cell from the reciprocal product alone, no 1e-9 fallback to the exact divisions",
    "f": "the fixed-point coordinate not saturated (u * 2^32 wraps modulo 2^32)",
    "g": "cell_mean reads the reciprocal table one entry low (rcp[c - 1])",
    "g2": "cell_mean takes the table for c <= RCP_N: rcp[RCP_N] lies past the table (here: memory holding 0)",
    "h": "box faces non-strict",
    "i": "a covered projection's cell accumulators left in the tiles for the next projection",
}


# ---------------------------------------------------------------------------------------------------- shadow points

def _mix32(h):
    h = np.asarray(h, np.uint64) & 0xFFFFFFFF
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    h ^= h >> 16
    return h


def norm_quantile_table():
    """QTAB[k] = standard-normal quantile at (k + 0.5) / 1024 (include/gpd_b200_shadow.h, Acklam's approximation)."""
    a = [-3.969683028665376e+01, 2.209460984245205e+02, -2.759285104469687e+02, 1.383577518672690e+02, -3.066479806614716e+01, 2.506628277459239e+00]
    b = [-5.447609879822406e+01, 1.615858368580409e+02, -1.556989798598866e+02, 6.680131188771972e+01, -1.328068155288572e+01]
    cc = [-7.784894002430293e-03, -3.223964580411365e-01, -2.400758277161838e+00, -2.549732539343734e+00, 4.374664141464968e+00, 2.938163982698783e+00]
    dd = [7.784695709041462e-03, 3.224671290700398e-01, 2.445134137142996e+00, 3.754408661907416e+00]
    tab = []
    for k in range(1024):
        p = (k + 0.5) / 1024
        if p < 0.02425 or p > 1.0 - 0.02425:
            q = math.sqrt(-2.0 * math.log(p if p < 0.5 else 1.0 - p))
            v = (((((cc[0] * q + cc[1]) * q + cc[2]) * q + cc[3]) * q + cc[4]) * q + cc[5]) / ((((dd[0] * q + dd[1]) * q + dd[2]) * q + dd[3]) * q + 1.0)
            tab.append(v if p < 0.5 else -v)
        else:
            q = p - 0.5
            r = q * q
            tab.append((((((a[0] * r + a[1]) * r + a[2]) * r + a[3]) * r + a[4]) * r + a[5]) * q /
                       (((((b[0] * r + b[1]) * r + b[2]) * r + b[3]) * r + b[4]) * r + 1.0))
    return np.array(tab)


def shadow_points(cloud, idx, sample_index, shadow_length=0.10, qtab=None):
    """HandSet::calculateShadow in the deterministic variant SPECIFIED by include/gpd_b200_shadow.h, restated from that
    header (steps 1-4): per (sample, point, camera) re-seeded LCG draws, float64 voxel arithmetic, set per camera,
    intersection starting from camera 0's set, voxel -> jittered point. idx: the neighbourhood in (distance, index)
    order (its sequential float64 sum is the centre). qtab: the jitter table (default: norm_quantile_table())."""
    pts = cloud["xyz"][idx].astype(np.float64)
    cam = np.asarray(cloud["cam_source"])[idx]
    vp = np.asarray(cloud["view_points"], np.float64)
    K = vp.shape[0]
    nsp = int(np.floor(shadow_length / VOXEL))
    if len(pts) == 0:
        return np.zeros((0, 3))
    center = np.zeros(3)
    for q in pts:                                            # sequential float64 sum, then / n (hand_set.cpp:131-136)
        center += q
    center /= float(len(pts))
    sets = []
    for k in range(K):
        if cam[:, k].sum() < 1:
            sets.append(None)
            continue
        sv = center - vp[k]
        sv = shadow_length * sv / np.sqrt((sv[0] * sv[0] + sv[1] * sv[1]) + sv[2] * sv[2])
        seed = _mix32((np.uint64(np.uint32(sample_index)) * 0x9E3779B1 + np.asarray(idx).astype(np.uint64) * 0x85EBCA77
                       + np.uint64(k) * 0xC2B2AE3D) & 0xFFFFFFFF)
        vox = []
        for _ in range(nsp):
            seed = (seed * 214013 + 2531011) & 0xFFFFFFFF
            u = ((seed >> 16) & 0x7FFF).astype(np.float64) * (1.0 / 32767.0)
            vox.append(np.trunc((pts + u[:, None] * sv[None, :]) * (1.0 / VOXEL)).astype(np.int64))
        sets.append(set(map(tuple, np.concatenate(vox))))
    allv = sets[0] or set()
    for k in range(1, K):
        if sets[k] is not None:
            allv = allv & sets[k]
    if not allv:
        return np.zeros((0, 3))
    v = np.array(sorted(allv), np.int64)
    hsh = _mix32(((v[:, 0].astype(np.uint64) & 0xFFFFFFFF) * 73856093 & 0xFFFFFFFF) ^ ((v[:, 1].astype(np.uint64) & 0xFFFFFFFF) * 19349663 & 0xFFFFFFFF)
                 ^ ((v[:, 2].astype(np.uint64) & 0xFFFFFFFF) * 83492791 & 0xFFFFFFFF))
    g = (norm_quantile_table() if qtab is None else np.asarray(qtab))[(hsh & 1023).astype(np.int64)]
    return v.astype(np.float64) * VOXEL + (1.0 * g * VOXEL * 0.3)[:, None]


# ---------------------------------------------------------------------------------------------------- geometry

class Geometry:
    def __init__(self, S=60, C=12, w=0.10, d=0.06, h=0.02):
        self.S, self.C, self.w, self.d, self.h = S, C, w, d, h

    @property
    def radius(self):   # image_generator.cpp:43-46
        return max(max(self.d, self.h / 2.0), self.w)

    @classmethod
    def of(cls, params):
        return cls(params.image_size, params.image_num_channels, params.volume_width, params.volume_depth,
                   params.volume_height)


def neighbourhood(cloud, sample, r):
    """The float32 image ball of the sample (FLANN's predicate) in (distance, index) order: indices, distance bits."""
    xyz = np.asarray(cloud["xyz"], np.float32)
    dd = np.asarray(sample, np.float64).astype(np.float32)[None] - xyz
    dist = dd[:, 0] * dd[:, 0]
    dist = dist + dd[:, 1] * dd[:, 1]
    dist = dist + dd[:, 2] * dd[:, 2]
    idx = np.flatnonzero(dist < np.float32(r * r))
    order = np.lexsort((idx, dist[idx]))
    return idx[order], dist[idx[order]].view(np.uint32)


def to_frame(frame, v):
    """geometry.cu to_frame: o_r = (F[3r] v0 + F[3r+1] v1) + F[3r+2] v2 in float64, element by element."""
    F = np.asarray(frame, np.float64)
    return np.stack([(F[3 * r] * v[:, 0] + F[3 * r + 1] * v[:, 1]) + F[3 * r + 2] * v[:, 2] for r in range(3)], 1)


def in_box(g, pose, P, strict=True):
    half = g.w / 2.0
    b, c = float(pose["bottom"]), float(pose["center"])
    x, y, z = P[:, 0], P[:, 1], P[:, 2]
    if strict:
        return (x > b) & (x < b + g.d) & (y > c - half) & (y < c + half) & (z > -1.0 * g.h) & (z < g.h)
    return (x >= b) & (x <= b + g.d) & (y >= c - half) & (y <= c + half) & (z >= -1.0 * g.h) & (z <= g.h)


def unit_cells(g, pose, P, mode, fault=None):
    """Unit coordinates [n, 3] and cells [n, 3]: the reference's divisions, or the kernels' unit_axis."""
    S = g.S
    lo = [float(pose["bottom"]), float(pose["center"]) - g.w / 2.0, -g.h]
    ext = [g.d, g.w, 2.0 * g.h]
    U = np.zeros_like(P)
    cell = np.zeros(P.shape, np.int64)
    cellsize = 1.0 / float(S)
    for a in range(3):
        v = P[:, a]
        if mode == "reference":
            u = (v - lo[a]) / ext[a] if a != 2 else (v + g.h) / ext[a]
            fq = np.floor(u / cellsize)
        else:
            u = (v - lo[a]) * (1.0 / ext[a])
            q = u * float(S)
            fq = np.floor(q)
            fr = q - fq
            if fault != "e":
                fb = (fr < 1e-9) | (fr > 1.0 - 1e-9)
                u = np.where(fb, (v - lo[a]) / ext[a], u)
                fq = np.where(fb, np.floor(u / cellsize), fq)
        U[:, a] = u
        cell[:, a] = np.minimum(fq.astype(np.int64), S - 1)
    return U, cell


def unit_q32(u, fault=None):
    t = np.trunc(u * 4294967296.0)
    if fault == "f":
        return (t.astype(np.uint64) & 0xFFFFFFFF).astype(np.int64)
    return np.clip(t, 0, 4294967295.0).astype(np.int64)


def cell_mean(s, c, fault=None):
    """cell_mean: sum / (count 2^32) as sum * rcp[c] for c < RCP_N, else a division; cast to float32."""
    s = np.asarray(s, np.float64)
    c = np.asarray(c, np.int64)
    with np.errstate(divide="ignore", invalid="ignore"):
        rc = 1.0 / (np.maximum(c - (1 if fault == "g" else 0), 0).astype(np.float64) * 4294967296.0)
        if fault == "g2":
            rc = np.where(c == RCP_N, 0.0, rc)
        n_tab = RCP_N + 1 if fault == "g2" else RCP_N
        return np.where(c < n_tab, s * rc, s / (c.astype(np.float64) * 4294967296.0)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------- per-cell values

def _fold(vals):
    """createNormalsImage's fold of a cell's |n| rows (float32 [m, 3]) in order; float32 / float64 steps as written."""
    v = np.zeros(3, np.float32)
    for a in vals:
        if v[0] == 0 and v[1] == 0 and v[2] == 0:
            v = a.copy()
        else:
            with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                f = np.float64(1.0) / np.float64(np.sqrt(np.float32(np.float32(v[0] * v[0]) + np.float32(v[1] * v[1]))
                                                         + np.float32(v[2] * v[2])))
                d = ((a - v).astype(np.float64) * f).astype(np.float32)
            v = (v + d).astype(np.float32)
    return v


def _running_mean(pix, z, SS):
    """float32 running mean per cell in the given order: avg += (z - avg) * (1.0 / count), count a float32."""
    avgs = np.zeros(SS, np.float32)
    counts = np.zeros(SS, np.float32)
    order_rank = np.zeros(len(pix), np.int64)   # rank within the cell: one vectorised step per rank
    seen = {}
    for i, p in enumerate(pix):
        order_rank[i] = seen.get(p, 0)
        seen[p] = order_rank[i] + 1
    for r in range(int(order_rank.max()) + 1 if len(pix) else 0):
        sel = order_rank == r
        p = pix[sel]
        counts[p] = (counts[p] + np.float32(1.0)).astype(np.float32)
        a = avgs[p].astype(np.float64)
        avgs[p] = (a + (z[sel] - a) * (1.0 / counts[p].astype(np.float64))).astype(np.float32)
    return avgs, counts > 0


# ---------------------------------------------------------------------------------------------------- output stage

def dilate(img):
    """3 x 3 max, border ignored; img [S, S] or [S, S, k]."""
    S = img.shape[0]
    lo = np.array(-np.inf, img.dtype) if img.dtype.kind == "f" else np.array(0, img.dtype)
    pad = np.full((S + 2, S + 2) + img.shape[2:], lo, img.dtype)
    pad[1:-1, 1:-1] = img
    out = pad[1:-1, 1:-1].copy()
    for dr in (-1, 0, 1):
        for dc in (-1, 0, 1):
            out = np.maximum(out, pad[1 + dr:S + 1 + dr, 1 + dc:S + 1 + dc])
    return out


def fully_covered(occ, fault=None):
    """geometry.cu fully_covered: no all-empty (clipped) 3 x 3 window of the occupancy [S, S]."""
    S = occ.shape[0]
    seen = occ.copy()
    if fault == "c":  # a row straddling three words loses the bits of the third
        for r in range(S):
            sh = (r * S) & 31
            if sh + S > 64:
                seen[r, 64 - sh:] = False
    pad = np.full((S + 2, S + 2), fault == "b", bool)
    pad[1:-1, 1:-1] = seen
    any_ = np.zeros((S, S), bool)
    for dr in (0, 1, 2):
        for dc in (0, 1, 2):
            any_ |= pad[dr:dr + S, dc:dc + S]
    return bool(any_.all())


def _fmaf(v, a, b):
    """fmaf(v, a, b) for float32 arrays v and float32 scalars a, b: v a is exact in float64; the float64 sum rounds to
    float32 correctly unless it lies on a float32 rounding midpoint, where the exact value decides."""
    with np.errstate(invalid="ignore", over="ignore"):
        r = v.astype(np.float64) * np.float64(a) + np.float64(b)
        out = r.astype(np.float32)
        if not (np.isfinite(a) and np.isfinite(b)):
            return out
        other = np.nextafter(out, np.where(r > out, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        mid = (r != out.astype(np.float64)) & (r == (out.astype(np.float64) + other.astype(np.float64)) / 2.0)
    for i in zip(*np.nonzero(mid)):
        exact = Fraction(float(v[i])) * Fraction(float(a)) + Fraction(float(b))
        m = Fraction(float(r[i]))
        lo, hi = sorted([out[i], other[i]])
        if exact > m:
            out[i] = hi
        elif exact < m:
            out[i] = lo
        else:
            out[i] = lo if (int(np.array(lo, np.float32).view(np.uint32)) & 1) == 0 else hi
    return out


def quantise(F, mn, mx, fault=None):
    """Quant: cv::normalize(NORM_MINMAX) + convertTo(CV_8U, 255) of float32 F with min mn and max mx, as the kernels
    evaluate it (NaN -> 0, +inf -> 255 as cvt.rni.s32.f32 and the clamp give)."""
    smin, smax = float(mn), float(mx)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if fault == "d":
            scale = 1.0 * (np.float64(1.0) / np.float64(smax - smin))
        else:
            scale = 1.0 * (1.0 / (smax - smin) if smax - smin > DBL_EPSILON else 0.0)
        shift = 0.0 - smin * scale
        a, b = np.float32(scale), np.float32(shift)
        t = _fmaf(np.asarray(F, np.float32), a, b)
        w = (t * np.float32(255.0)).astype(np.float32)
        q = np.rint(w)
        q = np.where(np.isnan(q), 0.0, np.clip(q, 0.0, 255.0))
    return q.astype(np.uint8)


def output_stage(F, occ, fault=None):
    """One channel group: float image F [S, S, k] (0 at empty cells), occupancy [S, S]. Returns (bytes [S, S, k] after
    the dilation, info)."""
    vals = F[occ]
    mx = np.float32(max(0.0, float(vals.max()))) if vals.size else np.float32(0.0)
    covered = fully_covered(occ, fault)
    mn = np.float32(0.0)
    if covered and fault != "a":
        mn = np.float32(dilate(F).min())
    q = quantise(F, mn, mx, fault)
    return dilate(q), {"covered": covered, "min": float(mn), "max": float(mx),
                       "constant": float(mx) - float(mn) <= DBL_EPSILON, "occupied": int(occ.sum())}


# ---------------------------------------------------------------------------------------------------- one image

def unit_normal(n):
    l2 = n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2]
    return np.abs(l2 - 1.0) <= 1e-5


def image(cloud, pose, g, mode="kernel", fault=None, qtab=None, shadow=None, info=None):
    """The grasp image [S, S, C] uint8 of one pose. mode "reference" | "kernel"; fault: a key of FAULTS (kernel mode).
    shadow: the shadow points (default: shadow_points with qtab). info: a dict that receives the intermediates
    ("box", "cells", "groups": {(pj, "n" | "d" | "s"): output_stage info}, "nonunit")."""
    assert mode in ("reference", "kernel") and (fault is None or mode == "kernel")
    S, C = g.S, g.C
    SS = S * S
    info = {} if info is None else info
    idx, dbits = neighbourhood(cloud, pose["sample"], g.radius)
    P = to_frame(pose["frame"], cloud["xyz"][idx].astype(np.float64) - np.asarray(pose["sample"], np.float64))
    m = in_box(g, pose, P, strict=fault != "h")
    bidx, P = idx[m], P[m]
    keys = (dbits[m].astype(np.uint64) << np.uint64(32)) | bidx.astype(np.uint64)   # ascending: (distance, index)
    N = np.abs(to_frame(pose["frame"], np.asarray(cloud["normals"], np.float64)[bidx])).astype(np.float32)
    nonunit = not unit_normal(np.asarray(cloud["normals"], np.float64)[bidx]).all()
    U, cell = unit_cells(g, pose, P, mode, fault)
    Q = unit_q32(U, fault) if mode == "kernel" else None
    info.update(box=len(bidx), cells=cell, units=U, box_index=bidx, nonunit=nonunit, groups={})

    sU = scell = sQ = None
    if C == 15:
        sp = shadow if shadow is not None else shadow_points(cloud, idx, int(pose["sample_index"]), g.radius, qtab)
        SP = to_frame(pose["frame"], sp - np.asarray(pose["sample"], np.float64)) if len(sp) else np.zeros((0, 3))
        SP = SP[in_box(g, pose, SP, strict=fault != "h")]
        sU, scell = unit_cells(g, pose, SP, mode, fault)
        sQ = unit_q32(sU, fault) if mode == "kernel" else None
        info["shadow_box"] = len(SP)

    out = np.zeros((S, S, C), np.uint8)
    nproj = 3 if C >= 12 else 1
    per = 5 if C == 15 else 4
    carry = None   # fault i: accumulators of a covered projection (key, sum, count per pixel)
    for pj in range(nproj):
        a0, a1, a2 = PROJ[pj]
        pix = (S - 1 - cell[:, a0]) * S + cell[:, a1]
        occ = np.zeros(SS, bool)
        occ[pix] = True
        Fn = np.zeros((SS, 3), np.float32)
        Fd = np.zeros(SS, np.float32)
        if mode == "kernel":
            sums = np.zeros(SS, np.int64)
            cnt = np.zeros(SS, np.int64)
            np.add.at(sums, pix, Q[:, a2])
            np.add.at(cnt, pix, 1)
            best = np.zeros(SS, np.uint64)
            np.maximum.at(best, pix, keys)
            if carry is not None:
                best = np.maximum(best, carry[0])
                sums += carry[1]
                cnt += carry[2]
                occ |= carry[2] > 0
            win = keys == best[pix]
            avg = cell_mean(sums, cnt, fault)
            for k in np.flatnonzero(win):
                p = pix[k]
                if nonunit:
                    same = np.flatnonzero(pix == p)
                    Fn[p] = _fold(N[same[np.argsort(keys[same])]])
                else:
                    Fn[p] = N[k]
                Fd[p] = np.float32(1.0 - float(avg[p]))
        else:
            order = np.argsort(keys)
            avgs, _ = _running_mean(pix[order], U[order, a2], SS)
            for p in np.unique(pix):
                same = order[pix[order] == p]
                Fn[p] = _fold(N[same])
                Fd[p] = np.float32(1.0 - float(avgs[p]))
        occ2 = occ.reshape(S, S)
        cb = 0 if C == 1 else pj * per
        covered_pts = False
        if C != 1:
            q, inf_ = output_stage(Fn.reshape(S, S, 3), occ2, fault)
            out[:, :, cb:cb + 3] = q
            info["groups"][(pj, "n")] = inf_
            covered_pts = inf_["covered"]
        if C == 1 or C >= 12:
            q, inf_ = output_stage(Fd.reshape(S, S, 1), occ2, fault)
            out[:, :, cb + (0 if C == 1 else 3):cb + (1 if C == 1 else 4)] = q
            info["groups"][(pj, "d")] = inf_
            covered_pts = inf_["covered"]
        carry = None
        if fault == "i" and covered_pts and mode == "kernel":
            carry = (best, sums, cnt)
        if C == 15:
            spix = (S - 1 - scell[:, a0]) * S + scell[:, a1]
            socc = np.zeros(SS, bool)
            socc[spix] = True
            if mode == "kernel":
                ssum = np.zeros(SS, np.int64)
                scnt = np.zeros(SS, np.int64)
                np.add.at(ssum, spix, sQ[:, a2])
                np.add.at(scnt, spix, 1)
                savg = cell_mean(ssum, scnt, fault)
            else:
                savg, _ = _running_mean(spix, sU[:, a2], SS)
            Fs = np.zeros(SS, np.float32)
            if socc.any():
                smax = np.float32(savg[socc].max())
                Fs[socc] = (smax - savg[socc]).astype(np.float32)
            q, inf_ = output_stage(Fs.reshape(S, S, 1), socc.reshape(S, S), fault)
            out[:, :, cb + 4:cb + 5] = q
            info["groups"][(pj, "s")] = inf_
    return out
