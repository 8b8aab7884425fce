"""numpy restatement of include/gpd_b200_plane.h: RANSAC plane fit with refit and the eligible mask of one cloud.

Written from the header's rules, not from the kernels: the partial Fisher-Yates shuffle runs on a real (sparse)
permutation, the float32 arithmetic is numpy float32 (every operation rounded on its own), the ordered sums are
np.add.accumulate (sequential), and pcl::eigen33 is the oracle's (oracle.pcl_eigen33). Every intermediate the GPU tests
compare is returned.
"""
import numpy as np

from sis_reference import philox

F = np.float32
STREAM = 3
SAMPLE_CHECKS = 1000
DBL_EPS = np.finfo(np.float64).eps


def draws(key, h, a):
    """gpdb_plane_draw for the attempts a (array) of hypothesis h -> [len(a), 4] uint32."""
    a = np.asarray(a, np.uint32)
    ctr = np.stack([np.full_like(a, h), a, np.full_like(a, STREAM), np.zeros_like(a)], axis=1)
    return philox(ctr, (int(key) & 0xFFFFFFFF, (int(key) >> 32) & 0xFFFFFFFF))


def fisher_yates3(c, n):
    """The first three entries of the identity permutation of 0..n-1 after swapping position i with i + (c[i] % (n-i))."""
    perm = {}
    out = []
    for i in range(3):
        j = i + int(c[i]) % (n - i)
        vi, vj = perm.get(i, i), perm.get(j, j)
        perm[i], perm[j] = vj, vi
        out.append(vj)
    return out


def model(p0, p1, p2):
    """Rule 2 in float32: (good, coefficients [4])."""
    a, b = (p1 - p0).astype(F), (p2 - p0).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = a / b
    if r[0] == r[1] and r[2] == r[1]:
        return False, None
    n = np.array([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]], F)
    s = np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
    if s > 0:
        n = n / s
    d = -((n[0] * p0[0] + n[1] * p0[1]) + n[2] * p0[2])
    return True, np.array([n[0], n[1], n[2], d], F)


def dist(coef, xyz):
    """Rule 3: float32 distances of the points xyz [N, 3]."""
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    c = coef.astype(F)
    return np.abs(((c[0] * x + c[1] * y) + c[2] * z) + c[3])


def inliers(coef, xyz, thr):
    return dist(coef, xyz).astype(np.float64) < thr


def hypothesis(xyz, key, h):
    """Rule 1 + 2: (attempt index, sample indices, coefficients) of hypothesis h, or None when all attempts are bad."""
    n = len(xyz)
    for a0 in (0, 16):
        a = np.arange(a0, 16 if a0 == 0 else SAMPLE_CHECKS)
        cs = draws(key, h, a)
        for k in range(len(a)):
            idx = fisher_yates3(cs[k], n)
            good, coef = model(xyz[idx[0]], xyz[idx[1]], xyz[idx[2]])
            if good:
                return int(a[k]), idx, coef
    return None


def refit(xyz_in):
    """Rule 5 on the inliers (index order), > 3 of them: the float32 single pass, eigen33 and d."""
    from oracle import oracle
    x, y, z = xyz_in[:, 0], xyz_in[:, 1], xyz_in[:, 2]
    terms = [x * x, x * y, x * z, y * y, y * z, z * z, x, y, z]
    acc = np.array([np.add.accumulate(t.astype(F), dtype=F)[-1] for t in terms], F) / F(len(xyz_in))
    cov = np.zeros((3, 3), F)
    cov[0, 0] = acc[0] - acc[6] * acc[6]
    cov[0, 1] = acc[1] - acc[6] * acc[7]
    cov[0, 2] = acc[2] - acc[6] * acc[8]
    cov[1, 1] = acc[3] - acc[7] * acc[7]
    cov[1, 2] = acc[4] - acc[7] * acc[8]
    cov[2, 2] = acc[5] - acc[8] * acc[8]
    cov[1, 0], cov[2, 0], cov[2, 1] = cov[0, 1], cov[0, 2], cov[1, 2]
    _, n = oracle.pcl_eigen33(cov)
    n = n.astype(F)
    d = -((n[0] * acc[6] + n[1] * acc[7]) + n[2] * acc[8])
    return np.array([n[0], n[1], n[2], d], F), cov, acc


def segment(xyz, key=0, distance_threshold=0.01, max_iterations=50, probability=0.99):
    """The whole header for one cloud. Returns a dict: hyps (list of (attempt, idx, coef) or None), counts, best,
    n_hypotheses, hyp_plane, plane (refined; NaN when failed), n_inliers, eligible [N] uint8, refit (bool)."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    n = len(xyz)
    thr = float(distance_threshold)
    hyps, counts = [], []
    best, best_h, ev, qp, q = None, -1, 0, 1.0, 1.0
    if n >= 3:
        for h in range(max_iterations + 1):
            hy = hypothesis(xyz, key, h)
            hyps.append(hy)
            if hy is None:
                break
            c = int(np.count_nonzero(inliers(hy[2], xyz, thr)))
            counts.append(c)
            ev = h + 1
            if best is None or c > best:
                best, best_h = c, h
                w = float(c) * (1.0 / float(n))
                q = min(max(1.0 - (w * w) * w, DBL_EPS), 1.0 - DBL_EPS)
                qp = 1.0
                for _ in range(h + 1):
                    qp = qp * q
            else:
                qp = qp * q
            if h + 1 > max_iterations or not (qp > 1.0 - float(probability)):
                break
    out = {"hyps": hyps, "counts": counts, "best": best_h, "n_hypotheses": ev, "refit": False}
    if best_h < 0:
        out.update(hyp_plane=None, plane=np.full(4, np.nan, F), n_inliers=0, eligible=np.ones(n, np.uint8))
        return out
    hp = hyps[best_h][2]
    m0 = inliers(hp, xyz, thr)
    plane = hp
    if np.count_nonzero(m0) > 3:
        plane, out["cov"], out["acc"] = refit(xyz[m0])
        out["refit"] = True
        out["best_inliers"] = xyz[m0]
    fin = inliers(plane, xyz, thr)
    elig = (~fin).astype(np.uint8)
    if not elig.any():
        elig[:] = 1
    out.update(hyp_plane=hp, plane=plane, n_inliers=int(np.count_nonzero(fin)), eligible=elig,
               dist=dist(plane, xyz))
    return out


def subsample_points(point_off, mask, num_samples, seed):
    """gpd_b200_depth.h 5 with one mask byte per installed point (concatenated by cloud): one array per cloud."""
    from depth_reference import subsample
    out = []
    for b in range(len(point_off) - 1):
        o0, o1 = int(point_off[b]), int(point_off[b + 1])
        out.append(subsample(o1 - o0, num_samples, seed, b, None if mask is None else np.asarray(mask[o0:o1]) != 0))
    return out
