"""ctypes loader of tests/plane_oracle.cpp, the C++ oracle of include/gpd_b200_plane.h (test infrastructure only). It is
built on first use into a temporary directory against the oracle's libgpd_oracle.so (its pcl::eigen33)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
_LIB = None


def lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    from oracle import oracle
    oracle.lib()  # builds oracle/libgpd_oracle.so if needed
    odir = os.path.join(ROOT, "oracle")
    so = os.path.join(tempfile.mkdtemp(prefix="plane_oracle_"), "libplane_oracle.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                           "-o", so, os.path.join(_HERE, "plane_oracle.cpp"), "-L", odir, "-lgpd_oracle", "-Wl,-rpath," + odir,
                           "-lpthread"])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.plane_oracle_segment.argtypes = [vp, C.c_int, C.c_uint64, C.c_double, C.c_int, C.c_double] + [vp] * 8
    L.plane_oracle_batch.argtypes = [C.c_int, vp, vp, C.c_uint64, C.c_double, C.c_int, C.c_double, vp, vp, vp, vp, C.c_int]
    L.plane_oracle_batch.restype = None
    _LIB = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def segment(xyz, key=0, distance_threshold=0.01, max_iterations=50, probability=0.99):
    """One cloud: a dict with attempts, samples, coefs, counts (per hypothesis, -1 / unset where not drawn), best,
    n_hypotheses, plane, n_inliers, eligible."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    H = max_iterations + 1
    att, smp, cnt = np.zeros(H, np.int32), np.zeros(3 * H, np.int32), np.zeros(H, np.int32)
    coef, plane = np.zeros(4 * H, np.float32), np.zeros(4, np.float32)
    best, n_inl = np.zeros(1, np.int32), np.zeros(1, np.int32)
    elig = np.zeros(max(len(xyz), 1), np.uint8)
    ev = lib().plane_oracle_segment(_p(xyz), len(xyz), int(key), float(distance_threshold), int(max_iterations),
                                    float(probability), _p(att), _p(smp), _p(coef), _p(cnt), _p(best), _p(plane), _p(n_inl),
                                    _p(elig))
    return {"attempts": att, "samples": smp.reshape(H, 3), "coefs": coef.reshape(H, 4), "counts": cnt, "best": int(best[0]),
            "n_hypotheses": int(ev), "plane": plane, "n_inliers": int(n_inl[0]), "eligible": elig[:len(xyz)]}


def segment_batch(off, xyz, seed=0, distance_threshold=0.01, max_iterations=50, probability=0.99, threads=None):
    off = np.ascontiguousarray(off, np.int32)
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    B = len(off) - 1
    planes, n_inl, n_hyp = np.zeros((B, 4), np.float32), np.zeros(B, np.int32), np.zeros(B, np.int32)
    elig = np.zeros(max(len(xyz), 1), np.uint8)
    lib().plane_oracle_batch(B, _p(off), _p(xyz), int(seed), float(distance_threshold), int(max_iterations), float(probability),
                             _p(planes), _p(n_inl), _p(n_hyp), _p(elig), int(threads or os.cpu_count() or 1))
    return {"planes": planes, "n_inliers": n_inl, "n_hypotheses": n_hyp, "eligible": elig[:len(xyz)]}
