"""ctypes loader of tests/train_chains.cpp, the sequential host restatement of include/gpd_b200_train.h rules 1, 2 and 5
(test infrastructure only), built on first use into a temporary directory.

Every function returns float32 (or uint8 choice) arrays computed by the header's own chains, so they compare with the
device's arrays bit for bit. Inputs are the .bin arrays, the images and per-image arrays named as the fields of
gpdb_train_debug (`Context.debug_train_step`): each stage restates one rule on the inputs it is given, so a stage can be
checked on the device's own input to it.
"""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
F = np.float32


def _compile(so, extra):
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", *extra, "-o", so,
           os.path.join(_HERE, "train_chains.cpp")]
    return subprocess.run(cmd, capture_output=True, text=True)


@functools.lru_cache(None)
def lib():
    so = os.path.join(tempfile.mkdtemp(prefix="train_chains_"), "libtrain_chains.so")
    # OpenMP spreads outputs over threads when the compiler has it; each output's chain stays in one thread either way
    r = _compile(so, ["-fopenmp"])
    if r.returncode != 0:
        r = _compile(so, [])
    if r.returncode != 0:
        raise RuntimeError("building train_chains.cpp failed:\n" + r.stderr)
    L = C.CDLL(so)
    vp, i = C.c_void_p, C.c_int
    L.tc_pool1.argtypes = [i, i, i, vp, vp, vp, i, vp, vp]
    L.tc_pool2.argtypes = [i, i, vp, vp, vp, i, vp, vp]
    L.tc_dip1.argtypes = [i, vp, vp, vp, vp]
    L.tc_dpool2.argtypes = [i, vp, vp, vp]
    L.tc_dconv2.argtypes = [i, i, vp, vp, vp, vp]
    L.tc_dpool1.argtypes = [i, vp, vp, i, vp]
    L.tc_conv2_grad.argtypes = [i, i, vp, vp, vp, vp, i, vp, vp]
    L.tc_conv1_grad.argtypes = [i, i, i, vp, vp, vp, vp, i, vp, vp]
    L.tc_ip_grads.argtypes = [i, vp, vp, vp, vp, i, vp, vp, vp, vp]
    for f in ("tc_pool1", "tc_pool2", "tc_dip1", "tc_dpool2", "tc_dconv2", "tc_dpool1", "tc_conv2_grad", "tc_conv1_grad",
              "tc_ip_grads"):
        getattr(L, f).restype = None
    return L


def _c(a, t=F):
    return np.ascontiguousarray(a, t)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _w(w, i):
    return _c(np.asarray(w[i]).ravel())


def pool1(images, w, relu, variant=0):
    """rules 1 and 2, conv1: (choice1 uint8 [n, 20, 28, 28], pool1 float32 [n, 20, 28, 28]); variant 1: last maximum"""
    images = _c(images, np.uint8)
    n, Cn = images.shape[0], images.shape[-1]
    ch, p = np.zeros((n, 20, 28, 28), np.uint8), np.zeros((n, 20, 28, 28), F)
    lib().tc_pool1(n, Cn, int(relu), _p(images), _p(_w(w, 0)), _p(_w(w, 1)), variant, _p(ch), _p(p))
    return ch, p


def pool2(p1, w, relu, variant=0):
    """rules 1 and 2, conv2 over pool1 [n, 20, 28, 28]: (choice2 uint8 [n, 7200], pool2 float32 [n, 7200]), k = c + 50 j"""
    p1 = _c(p1)
    n = p1.shape[0]
    ch, p = np.zeros((n, 7200), np.uint8), np.zeros((n, 7200), F)
    lib().tc_pool2(n, int(relu), _p(p1), _p(_w(w, 2)), _p(_w(w, 3)), variant, _p(ch), _p(p))
    return ch, p


def dip1(ip1, dz, w):
    ip1, dz = _c(ip1), _c(dz)
    out = np.zeros((len(ip1), 500), F)
    lib().tc_dip1(len(ip1), _p(ip1), _p(dz), _p(_w(w, 6)), _p(out))
    return out


def dpool2(dh, w):
    dh = _c(dh)
    out = np.zeros((len(dh), 7200), F)
    lib().tc_dpool2(len(dh), _p(dh), _p(_w(w, 4)), _p(out))
    return out


def dconv2(dx, p2, ch2, relu):
    """dense d conv2 [n, 50, 24, 24] from d pool2, pool2 and choice2 (k order)"""
    dx, p2, ch2 = _c(dx), _c(p2), _c(ch2, np.uint8)
    out = np.zeros((len(dx), 50, 24, 24), F)
    lib().tc_dconv2(len(dx), int(relu), _p(dx), _p(p2), _p(ch2), _p(out))
    return out


def dpool1(dc2, w, variant=0):
    """d pool1 [n, 20, 28, 28] from the dense d conv2; variant 1 chains over (kh, kw, o)"""
    dc2 = _c(dc2)
    out = np.zeros((len(dc2), 20, 28, 28), F)
    lib().tc_dpool1(len(dc2), _p(dc2), _p(_w(w, 2)), variant, _p(out))
    return out


def conv2_grads(p1, dx, p2, ch2, relu, restart=0):
    """(d conv2 weights [25000], d conv2 biases [50]); restart > 0 starts a second image chain there"""
    p1, dx, p2, ch2 = _c(p1), _c(dx), _c(p2), _c(ch2, np.uint8)
    gw, gb = np.zeros(25000, F), np.zeros(50, F)
    lib().tc_conv2_grad(len(dx), int(relu), _p(p1), _p(dx), _p(p2), _p(ch2), restart, _p(gw), _p(gb))
    return gw, gb


def conv1_grads(images, dp1, p1, ch1, relu, restart=0):
    """(d conv1 weights [20 C 25], d conv1 biases [20]); restart as conv2_grads"""
    images, dp1, p1, ch1 = _c(images, np.uint8), _c(dp1), _c(p1), _c(ch1, np.uint8)
    n, Cn = images.shape[0], images.shape[-1]
    gw, gb = np.zeros(20 * Cn * 25, F), np.zeros(20, F)
    lib().tc_conv1_grad(n, Cn, int(relu), _p(images), _p(dp1), _p(p1), _p(ch1), restart, _p(gw), _p(gb))
    return gw, gb


def ip_grads(p2, dh, ip1, dz, reverse=False):
    """(dW1 [3 600 000], db1 [500], dW2 [1000], db2 [2]); reverse chains dW1 over the images backwards"""
    p2, dh, ip1, dz = _c(p2), _c(dh), _c(ip1), _c(dz)
    dW1, db1, dW2, db2 = np.zeros(3600000, F), np.zeros(500, F), np.zeros(1000, F), np.zeros(2, F)
    lib().tc_ip_grads(len(dh), _p(p2), _p(dh), _p(ip1), _p(dz), int(reverse), _p(dW1), _p(db1), _p(dW2), _p(db2))
    return dW1, db1, dW2, db2


def grads(images, d, relu):
    """the eight gradients (.bin layouts) of a step, from per-image arrays d (keys of gpdb_train_debug)"""
    g1 = conv1_grads(images, d["dpool1"], d["pool1"], d["choice1"], relu)
    g2 = conv2_grads(d["pool1"], d["dpool2"], d["pool2"], d["choice2"], relu)
    return [*g1, *g2, *ip_grads(d["pool2"], d["dip1"], d["ip1"], d["dlogits"])]


def stages(images, d, w, relu):
    """the per-image stages of images (a subset of a step), each on the input d gives it: choice1 / pool1 from the images,
    choice2 / pool2 from d's pool1, dip1 from d's ip1 and d logits, dpool2 from d's dip1, dpool1 through the dense
    d conv2 of d's dpool2, pool2 and choice2"""
    out = {}
    out["choice1"], out["pool1"] = pool1(images, w, relu)
    out["choice2"], out["pool2"] = pool2(d["pool1"], w, relu)
    out["dip1"] = dip1(d["ip1"], d["dlogits"], w)
    out["dpool2"] = dpool2(d["dip1"], w)
    out["dpool1"] = dpool1(dconv2(d["dpool2"], d["pool2"], d["choice2"], relu), w)
    return out
