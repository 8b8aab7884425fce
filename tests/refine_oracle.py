"""ctypes loader of tests/refine_oracle.cpp, the C++ oracle of include/gpd_b200_refine.h (test infrastructure only). It is
built on first use into a temporary directory."""
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
    so = os.path.join(tempfile.mkdtemp(prefix="refine_oracle_"), "librefine_oracle.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(ROOT, "include"),
                           "-o", so, os.path.join(_HERE, "refine_oracle.cpp"), "-lpthread"])
    L = C.CDLL(so)
    vp = C.c_void_p
    L.refine_oracle_knn.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int]
    L.refine_oracle_knn.restype = None
    L.refine_oracle_iterate.argtypes = [C.c_int, C.c_int, vp, vp]
    L.refine_oracle_batch.argtypes = [C.c_int, vp, vp, vp, C.c_int, vp, C.c_int]
    L.refine_oracle_batch.restype = None
    _LIB = L
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _threads(threads):
    return int(threads or os.cpu_count() or 1)


def knn(xyz, k, threads=None):
    """Rule 1: [N, min(k, N)] int32."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    n = len(xyz)
    nbr = np.zeros((max(n, 1), k), np.int32)
    lib().refine_oracle_knn(_p(xyz), n, int(k), _p(nbr), _threads(threads))
    return nbr[:n, :min(k, n)]


def refine(xyz, normals, k, nbr=None, threads=None):
    """Rules 1-5 for one cloud: (refined float64 normals [N, 3], iterations run)."""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    n = len(xyz)
    out = np.ascontiguousarray(normals, np.float64).reshape(-1, 3).copy()
    if nbr is None:
        nbr = knn(xyz, k, threads)
    full = np.zeros((max(n, 1), k), np.int32)
    full[:n, :nbr.shape[1]] = nbr
    it = lib().refine_oracle_iterate(n, int(k), _p(full), _p(out))
    return out, int(it)


def refine_batch(off, xyz, normals, k, threads=None):
    """Every cloud of a CSR batch on its own, the clouds spread over the host threads: (normals [N, 3], iterations [B])."""
    off = np.ascontiguousarray(off, np.int32)
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    out = np.ascontiguousarray(normals, np.float64).reshape(-1, 3).copy()
    its = np.zeros(max(len(off) - 1, 1), np.int32)
    lib().refine_oracle_batch(len(off) - 1, _p(off), _p(xyz), _p(out), int(k), _p(its), _threads(threads))
    return out, its[:len(off) - 1]
