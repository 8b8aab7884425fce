"""Numpy restatement of include/gpd_b200_refine.h (Cloud::refineNormals: k nearest neighbours, then
pcl::NormalRefinement with its defaults). Every float32 operation is a numpy float32 elementwise operation, so each is
rounded on its own. The sums the contract makes sequential stay sequential: the neighbour sums loop over list positions
(vectorised over points only), and the stop statistic is np.add.accumulate, a running sum in index order (np.sum is
pairwise)."""
import numpy as np

F = np.float32
MAX_K = 128
MAX_ITERATIONS = 15
CONVERGENCE = F(1e-5)
FLT_EPSILON = F(np.finfo(np.float32).eps)


def l2(q, p):
    """Rule 1: L2_Simple<float> of every query row q [m, 3] against every point p [n, 3] -> [m, n] float32."""
    q, p = np.asarray(q, F), np.asarray(p, F)
    dx = q[:, None, 0] - p[None, :, 0]
    dy = q[:, None, 1] - p[None, :, 1]
    dz = q[:, None, 2] - p[None, :, 2]
    d = dx * dx
    d = d + dy * dy
    return d + dz * dz


def keys(d, idx):
    """(float32 distance bits, index) as one uint64 per entry."""
    return (np.ascontiguousarray(d, F).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.asarray(idx, np.uint64)


def knn_brute(xyz, k, block=512):
    """Rule 1 by brute force: [N, min(k, N)] int32, each row ascending by key."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    n = len(xyz)
    L = min(k, n)
    out = np.zeros((n, L), np.int32)
    j = np.arange(n, dtype=np.uint64)
    for a in range(0, n, block):
        kk = keys(l2(xyz[a:a + block], xyz), j[None, :])
        part = np.partition(kk, L - 1, axis=1)[:, :L] if L < n else kk
        out[a:a + block] = (np.sort(part, axis=1) & np.uint64(0xffffffff)).astype(np.int32)
    return out


def knn(xyz, k, brute_below=4096):
    """Rule 1: brute force for small clouds; above, a cKDTree candidate superset (float64) re-ranked by the exact float32
    key, each row checked against the float32 rounding bound and redone by brute force where the check fails."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    n = len(xyz)
    if n <= brute_below:
        return knn_brute(xyz, k)
    from scipy.spatial import cKDTree
    L = min(k, n)
    kc = min(n, L + 16)
    x64 = xyz.astype(np.float64)
    dist, cand = cKDTree(x64).query(x64, k=kc)
    dx = xyz[:, None, :] - xyz[cand]
    d32 = dx[..., 0] * dx[..., 0]
    d32 = d32 + dx[..., 1] * dx[..., 1]
    d32 = d32 + dx[..., 2] * dx[..., 2]
    kk = np.sort(keys(d32, cand.astype(np.uint64)), axis=1)[:, :L]
    out = (kk & np.uint64(0xffffffff)).astype(np.int32)
    # every point outside the candidates lies at float64 distance >= the last candidate's; its float32 key exceeds the
    # L-th when that distance squared, less the rounding of five float32 operations, is above the L-th distance
    kth = (kk[:, -1] >> np.uint64(32)).astype(np.uint32).view(F).astype(np.float64)
    ok = (kc == n) | (dist[:, -1] ** 2 * (1.0 - 1e-6) > kth)
    for i in np.nonzero(~ok)[0]:
        out[i] = knn_brute_row(xyz, i, L)
    return out


def knn_brute_row(xyz, i, L):
    kk = np.sort(keys(l2(xyz[i:i + 1], xyz)[0], np.arange(len(xyz), dtype=np.uint64)))[:L]
    return (kk & np.uint64(0xffffffff)).astype(np.int32)


def finite3(m):
    return np.isfinite(m[:, 0]) & np.isfinite(m[:, 1]) & np.isfinite(m[:, 2])


def refine_normal(sx, sy, sz):
    """Rule 3 from the sums (arrays)."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        norm = np.sqrt((sx * sx + sy * sy) + sz * sz)
        ok = np.isfinite(norm) & (norm > FLT_EPSILON)
        safe = np.where(ok, norm, F(1))
        out = np.stack([sx / safe, sy / safe, sz / safe], 1).astype(F)
    out[~ok] = np.nan
    return out


def acosf(x):
    """Rule 4: gpdb_refine_acosf, elementwise."""
    x = np.asarray(x, F)
    a = np.abs(x)
    big = a > F(0.5)
    with np.errstate(invalid="ignore"):
        z = np.where(big, F(0.5) * (F(1) - a), a * a).astype(F)
        s = np.where(big, np.sqrt(F(0.5) * (F(1) - a)), a).astype(F)
    p = F(4.2163199048e-2) * z + F(2.4181311049e-2)
    p = p * z + F(4.5470025998e-2)
    p = p * z + F(7.4953002686e-2)
    p = p * z + F(1.6666752422e-1)
    r = s + (p * z) * s
    t = r + r
    neg = x < F(0)
    return np.where(big, np.where(neg, F(3.14159265358979) - t, t),
                    np.where(neg, F(1.57079632679490) + r, F(1.57079632679490) - r)).astype(F)


def error(o, m):
    """Rule 4: the error of every point between its previous normals o [n, 3] and new normals m [n, 3]."""
    with np.errstate(invalid="ignore"):
        d = (o[:, 0] * m[:, 0] + o[:, 1] * m[:, 1]) + o[:, 2] * m[:, 2]
    d = np.minimum(np.maximum(d, F(-1)), F(1))
    e = acosf(np.where(np.isfinite(d), d, F(0)))
    return np.where(finite3(o) & finite3(m), e, F(0)).astype(F)


def iterate(nbr, m):
    """Rule 3, one iteration over every point: (new normals, errors)."""
    n = len(m)
    s = np.zeros((n, 3), F)
    fin = finite3(m)
    for r in range(nbr.shape[1]):
        j = nbr[:, r]
        # adding +0 for a skipped neighbour equals skipping it: a sum from +0 is never -0
        s = s + np.where(fin[j][:, None], m[j], F(0))
    new = refine_normal(s[:, 0], s[:, 1], s[:, 2])
    return new, error(m, new)


def mean_error(err):
    """Rule 4: the sequential float32 sum in index order over (float)N."""
    if len(err) == 0:
        return F(0)
    return np.add.accumulate(err.astype(F), dtype=F)[-1] / F(len(err))


def refine(xyz, normals, k, nbr=None, trace=None):
    """Rules 1-5 for one cloud: (refined float64 normals [N, 3], iterations run). trace (a list) receives each
    iteration's mean error."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    normals = np.asarray(normals, np.float64).reshape(-1, 3)
    n = len(xyz)
    if n == 0:
        return normals.copy(), 0
    if nbr is None:
        nbr = knn(xyz, k)
    m = normals.astype(F)
    t = 0
    while t < MAX_ITERATIONS:
        m, err = iterate(nbr, m)
        t += 1
        mean = mean_error(err)
        if trace is not None:
            trace.append(mean)
        if mean < CONVERGENCE:
            break
    return m.astype(np.float64), t


def refine_batch(off, xyz, normals, k):
    """Every cloud of a CSR batch on its own: (normals [N, 3], iterations [B])."""
    out = np.asarray(normals, np.float64).reshape(-1, 3).copy()
    its = np.zeros(len(off) - 1, np.int32)
    for b in range(len(off) - 1):
        a, e = off[b], off[b + 1]
        out[a:e], its[b] = refine(xyz[a:e], out[a:e], k)
    return out, its
