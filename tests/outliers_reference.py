"""Numpy restatement of include/gpd_b200_outliers.h (Cloud::removeStatisticalOutliers: pcl::StatisticalOutlierRemoval over
the k nearest neighbours of tests/refine_reference.py). Every float32 operation is a numpy float32 elementwise operation,
so each is rounded on its own. The sums the contract makes sequential stay sequential: the distance sum loops over list
positions (vectorised over points only), and the cloud sums are np.cumsum, a running sum in index order (np.sum is
pairwise)."""
import numpy as np

import refine_reference as rr

F = np.float32
D = np.float64
MAX_K = rr.MAX_K - 1


def mean_distances(xyz, mean_k, nbr=None):
    """Rules 1 and 2: d [N] float32 of a cloud of N > mean_k points; nbr, when given, the lists of rule 1 [N, >= mean_k + 1]
    in any tie order."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    if nbr is None:
        nbr = rr.knn(xyz, mean_k + 1)
    s = np.zeros(len(xyz), D)
    for r in range(1, mean_k + 1):
        p = xyz[nbr[:, r]]
        dx, dy, dz = xyz[:, 0] - p[:, 0], xyz[:, 1] - p[:, 1], xyz[:, 2] - p[:, 2]
        l2 = dx * dx
        l2 = l2 + dy * dy
        l2 = l2 + dz * dz
        s = s + np.sqrt(l2).astype(D)  # np.sqrt of float32 is the correctly rounded sqrtf
    return (s / D(mean_k)).astype(F)


def stats(d, mean_k, stddev_mul):
    """Rules 3 and 5: (mean, stddev, threshold) of a cloud with mean distances d."""
    n = len(d)
    if n <= mean_k:
        return (np.nan,) * 3
    d = np.asarray(d, F)
    s = float(np.cumsum(d.astype(D))[-1])
    sq = float(np.cumsum((d * d).astype(D))[-1])
    mean = s / n
    variance = (sq - s * s / n) / (n - 1.0)
    with np.errstate(invalid="ignore"):
        stddev = float(np.sqrt(D(variance)))
    return mean, stddev, mean + float(stddev_mul) * stddev


def keep(d, threshold):
    """Rule 4: a point stays unless (double)d > threshold; a NaN threshold keeps every point."""
    return ~(np.asarray(d, F).astype(D) > threshold)


def remove(xyz, mean_k, stddev_mul, nbr=None):
    """Rules 1-6 for one cloud: (kept bools [N], (mean, stddev, threshold), mean distances or None)."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    n = len(xyz)
    if n <= mean_k:
        return np.ones(n, bool), (np.nan,) * 3, None
    d = mean_distances(xyz, mean_k, nbr)
    st = stats(d, mean_k, stddev_mul)
    return keep(d, st[2]), st, d


def remove_batch(off, xyz, mean_k, stddev_mul):
    """Every cloud of a CSR batch on its own: (kept bools [N], stats [B, 3], new offsets [B+1])."""
    xyz = np.ascontiguousarray(xyz, F).reshape(-1, 3)
    B = len(off) - 1
    kept = np.zeros(len(xyz), bool)
    st = np.zeros((B, 3))
    for b in range(B):
        kept[off[b]:off[b + 1]], st[b], _ = remove(xyz[off[b]:off[b + 1]], mean_k, stddev_mul)
    new = np.concatenate([[0], np.cumsum([kept[off[b]:off[b + 1]].sum() for b in range(B)])]).astype(np.int32)
    return kept, st, new
