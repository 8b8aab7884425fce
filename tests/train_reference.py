"""Restatements of include/gpd_b200_train.h, shared by test_train_reference.py (CPU) and test_gpu_train.py (-m gpu).

- float32 numpy restatements of the loss, the d logits and the two optimisers (rules 3, 4, 6). expf and log1pf are the
  host's libm, called through ctypes, so the restatement and the header's helpers compiled for the host see the same
  exponentials and logarithms.
- the header's helpers compiled for the host with -ffp-contract=off (`helpers()`).
- a float64 restatement of the forward and every backward stage (rules 1, 2, 5) on the .bin arrays, `backward64`, which
  can take given pooling choices and stage inputs (the device's own, in the GPU test).
- the network in torch float64 with the .bin arrays mapped to torch's parameter layouts, `torch_grads64`: the reference's
  pytorch/network.py Net when relu = 1, the Caffe LeNet when relu = 0, trained with nn.CrossEntropyLoss.
- per-stage error bounds of the device's float32 arithmetic, `bounds`, derived as in lenet_layer_bounds.py: every stage
  on its own inputs, |err| <= gamma(m) * sum |terms| for a chain of m roundings.
"""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np

F = np.float32
U = 2.0 ** -24
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 256  # GPDB_TRAIN_CHUNK


def gamma(m):
    return m * U / (1.0 - m * U)


# ---- float32: rules 3, 4, 6 ----------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def _libm():
    L = C.CDLL("libm.so.6")
    for f in ("expf", "log1pf"):
        getattr(L, f).restype = C.c_float
        getattr(L, f).argtypes = [C.c_float]
    return L


def _vec(name, x):
    f = getattr(_libm(), name)
    return np.array([f(float(v)) for v in np.asarray(x, F).ravel()], F).reshape(np.shape(x))


def loss_f32(z, y):
    """rule 3 per image: z [n, 2] float32, y [n] in {0, 1}"""
    z0, z1 = z[:, 0].astype(F), z[:, 1].astype(F)
    d = np.abs(z1 - z0)
    l = _vec("log1pf", _vec("expf", -d))
    top = np.where(y == 1, z1 >= z0, z0 >= z1)
    return np.where(top, l, d + l).astype(F)


def mean_loss_f32(losses):
    s = F(0)
    for v in losses:
        s = F(s + v)
    return F(s / F(len(losses)))


def probs_f32(z):
    """rule 4: the probabilities (p0, p1) of logits z [m, 2]"""
    z0, z1 = z[:, 0].astype(F), z[:, 1].astype(F)
    e = _vec("expf", -np.abs(z1 - z0))
    s = F(1) + e
    pb, ps = F(1) / s, e / s
    return np.where(z1 >= z0, ps, pb), np.where(z1 >= z0, pb, ps)


def dlogits_f32(z, y, n):
    """rule 4: z [m, 2], y [m], n the step's image count"""
    p0, p1 = probs_f32(z)
    nf = F(n)
    return np.stack([(p0 - (y == 0).astype(F)) / nf, (p1 - (y == 1).astype(F)) / nf], 1).astype(F)


def sgd_f32(p, g, buf, lr, mu, wd, first):
    """rule 6, SGD: returns (p, buf), float32 arrays"""
    p, g, buf, lr, mu, wd = p.astype(F), g.astype(F), buf.astype(F), F(lr), F(mu), F(wd)
    if wd != 0:
        g = g + wd * p
    if mu != 0:
        buf = g.copy() if first else mu * buf + g
        g = buf
    return (p - lr * g).astype(F), buf


def adam_scalars(lr, b1, b2, t):
    bc1, bc2 = 1.0 - float(F(b1)) ** t, 1.0 - float(F(b2)) ** t
    return F(float(F(lr)) / bc1), F(np.sqrt(bc2))


def adam_f32(p, g, m, v, lr, b1, b2, eps, wd, t):
    """rule 6, Adam at step t >= 1: returns (p, m, v)"""
    p, g, m, v = p.astype(F), g.astype(F), m.astype(F), v.astype(F)
    b1, b2, eps, wd = F(b1), F(b2), F(eps), F(wd)
    step, r = adam_scalars(lr, b1, b2, t)
    if wd != 0:
        g = g + wd * p
    m = b1 * m + (F(1) - b1) * g
    v = b2 * v + (F(1) - b2) * (g * g)
    denom = np.sqrt(v) / r + eps
    return (p - step * (m / denom)).astype(F), m, v


# ---- the header's helpers, compiled for the host ------------------------------------------------------------------------
_HELPERS = r"""
#include <stdint.h>
#include "gpd_b200_train.h"
extern "C" void tr_loss(int n, int n_step, const float *z, const int32_t *y, float *loss, float *dz) {
  for (int i = 0; i < n; i++) {
    loss[i] = gpdb_train_loss(z[2 * i], z[2 * i + 1], y[i]);
    gpdb_train_dlogits(z[2 * i], z[2 * i + 1], y[i], (float)n_step, dz + 2 * i);
  }
}
extern "C" void tr_sgd(int n, float *p, const float *g, float *buf, float lr, float mu, float wd, int first) {
  for (int i = 0; i < n; i++) gpdb_train_sgd(p + i, g[i], buf + i, lr, mu, wd, first != 0);
}
extern "C" void tr_adam(int n, float *p, const float *g, float *m, float *v, float lr, float b1, float b2, float eps,
                        float wd, long long t) {
  float step, r;
  gpdb_train_adam_scalars(lr, b1, b2, t, &step, &r);
  for (int i = 0; i < n; i++) gpdb_train_adam(p + i, g[i], m + i, v + i, b1, 1.0f - b1, b2, 1.0f - b2, eps, wd, step, r);
}
"""


@functools.lru_cache(None)
def helpers():
    d = tempfile.mkdtemp(prefix="train_helpers_")
    src, so = os.path.join(d, "h.cpp"), os.path.join(d, "libh.so")
    with open(src, "w") as f:
        f.write(_HELPERS)
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "include"), "-o", so, src])
    L = C.CDLL(so)
    vp, fl = C.c_void_p, C.c_float
    L.tr_loss.argtypes = [C.c_int, C.c_int, vp, vp, vp, vp]
    L.tr_sgd.argtypes = [C.c_int, vp, vp, vp, fl, fl, fl, C.c_int]
    L.tr_adam.argtypes = [C.c_int, vp, vp, vp, vp, fl, fl, fl, fl, fl, C.c_longlong]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_loss(z, y, n_step):
    z, y = np.ascontiguousarray(z, F), np.ascontiguousarray(y, np.int32)
    loss, dz = np.zeros(len(y), F), np.zeros((len(y), 2), F)
    helpers().tr_loss(len(y), n_step, _p(z), _p(y), _p(loss), _p(dz))
    return loss, dz


def host_sgd(p, g, buf, lr, mu, wd, first):
    p, buf = p.astype(F).copy(), buf.astype(F).copy()
    g = np.ascontiguousarray(g, F)
    helpers().tr_sgd(p.size, _p(p), _p(g), _p(buf), lr, mu, wd, int(first))
    return p, buf


def host_adam(p, g, m, v, lr, b1, b2, eps, wd, t):
    p, m, v = p.astype(F).copy(), m.astype(F).copy(), v.astype(F).copy()
    g = np.ascontiguousarray(g, F)
    helpers().tr_adam(p.size, _p(p), _p(g), _p(m), _p(v), lr, b1, b2, eps, wd, t)
    return p, m, v


# ---- float64: rules 1, 2, 5 ----------------------------------------------------------------------------------------------
def chw(images):
    """HWC uint8 [n, 60, 60, C] -> float64 [n, C, 60, 60], the true transpose"""
    return np.asarray(images, np.float64).transpose(0, 3, 1, 2)


def _win(x):
    """[n, C, H, W] -> 5 x 5 windows [n, C, H-4, W-4, 5, 5]"""
    return np.lib.stride_tricks.sliding_window_view(x, (5, 5), axis=(2, 3))


def conv(x, w, b):
    return np.einsum("ncyxij,ocij->noyx", _win(x), w, optimize=True) + b[None, :, None, None]


def pool(v, choice=None):
    """2 x 2 max-pool: (pooled, choice), choice in row-major window order, the first maximum unless given"""
    n, o, H, W = v.shape
    q = v.reshape(n, o, H // 2, 2, W // 2, 2).transpose(0, 1, 2, 4, 3, 5).reshape(n, o, H // 2, W // 2, 4)
    if choice is None:
        choice = q.argmax(-1)
    return np.take_along_axis(q, choice[..., None].astype(np.int64), -1)[..., 0], choice


def unpool(g, choice):
    """scatter [n, o, P, P] to the chosen positions of [n, o, 2P, 2P]"""
    n, o, P, _ = g.shape
    q = np.zeros((n, o, P, P, 4))
    np.put_along_axis(q, choice[..., None].astype(np.int64), g[..., None], -1)
    return q.reshape(n, o, P, P, 2, 2).transpose(0, 1, 2, 4, 3, 5).reshape(n, o, 2 * P, 2 * P)


def flat(h):
    """[n, 50, 12, 12] -> [n, 7200], k = c + 50 j"""
    return h.reshape(h.shape[0], 50, -1).transpose(0, 2, 1).reshape(h.shape[0], -1)


def unflat(x):
    return x.reshape(x.shape[0], 144, 50).transpose(0, 2, 1).reshape(x.shape[0], 50, 12, 12)


def arrays64(w, C):
    w = [np.asarray(a, np.float64).ravel() for a in w]
    return (w[0].reshape(20, C, 5, 5), w[1], w[2].reshape(50, 20, 5, 5), w[3], w[4].reshape(7200, 500), w[5],
            w[6].reshape(500, 2), w[7])


def forward64(images, w, relu, choice1=None, choice2=None, p1_in=None):
    """rule 1 and 2 in float64; p1_in: pool1 to continue from (the device's) instead of this forward's"""
    C = images.shape[-1]
    w1, b1, w2, b2, W1, B1, W2, B2 = arrays64(w, C)
    x = chw(images)
    v1 = conv(x, w1, b1)
    p1, ch1 = pool(v1, choice1)
    if relu:
        p1 = np.maximum(p1, 0)
    if p1_in is not None:
        p1 = np.asarray(p1_in, np.float64)
    v2 = conv(p1, w2, b2)
    p2, ch2 = pool(v2, choice2)
    if relu:
        p2 = np.maximum(p2, 0)
    xf = flat(p2)
    h = np.maximum(xf @ W1 + B1, 0)
    z = h @ W2 + B2
    return {"x": x, "p1": p1, "ch1": ch1, "p2": p2, "ch2": ch2, "xf": xf, "h": h, "z": z}


def dlogits64(z, y, n):
    z = np.asarray(z, np.float64)
    e = np.exp(z - z.max(1, keepdims=True))
    p = e / e.sum(1, keepdims=True)
    return (p - np.eye(2)[np.asarray(y)]) / n


def backward64(images, labels, w, relu, dev=None, n_step=None):
    """every backward stage in float64. dev: a dict of the device's own stage inputs (keys of gpdb_train_debug: pool1,
    pool2 (k order), ip1, logits, choice1 ([n, 20, 28, 28]), choice2 (k order), dlogits, dip1, dpool2, dpool1); each
    stage then starts from the device's input to it. n_step: the image count of the whole step when images are a slice
    of it (the gradients of a step are the sums of its slices' gradients). Returns the stages and the eight gradients in
    the .bin layouts."""
    C = images.shape[-1]
    n = n_step or len(labels)
    w1, b1, w2, b2, W1, B1, W2, B2 = arrays64(w, C)
    dev = dev or {}
    ch1 = dev.get("choice1")
    ch2 = None if dev.get("choice2") is None else unflat(np.asarray(dev["choice2"]))
    if all(k in dev for k in ("pool1", "pool2", "ip1", "logits", "choice1", "choice2")):
        # every forward value is given: only the input and the choices are needed
        f = {"x": chw(images), "ch1": ch1, "ch2": ch2, "p1": None, "xf": None, "h": None, "z": None}
    else:
        f = forward64(images, w, relu, ch1, ch2, dev.get("pool1"))
    g = lambda k, v: np.asarray(dev[k], np.float64) if k in dev else v  # noqa: E731
    h, xf, p1, p2 = g("ip1", f["h"]), g("pool2", f["xf"]), g("pool1", f["p1"]), unflat(g("pool2", f["xf"]))
    dz = dlogits64(g("logits", f["z"]), labels, n)
    dzi = g("dlogits", dz)
    dh = (dzi @ W2.T) * (h > 0)
    dhi = g("dip1", dh)
    dx = dhi @ W1.T
    dxi = g("dpool2", dx)
    m2 = (p2 > 0) if relu else np.ones_like(p2, bool)
    g2 = unflat(dxi) * m2
    dc2 = unpool(g2, f["ch2"])
    pad = np.pad(dc2, ((0, 0), (0, 0), (4, 4), (4, 4)))
    dp1 = np.einsum("noyxij,ocij->ncyx", _win(pad), w2[:, :, ::-1, ::-1], optimize=True)
    dp1i = g("dpool1", dp1)
    m1 = (p1 > 0) if relu else np.ones_like(p1, bool)
    g1 = dp1i * m1
    dc1 = unpool(g1, f["ch1"])
    grads = [np.einsum("noyx,ncyxij->ocij", dc1, _win(f["x"]), optimize=True).ravel(), dc1.sum((0, 2, 3)),
             np.einsum("noyx,ncyxij->ocij", dc2, _win(p1), optimize=True).ravel(), dc2.sum((0, 2, 3)),
             (xf.T @ dhi).ravel(), dhi.sum(0), (h.T @ dzi).ravel(), dzi.sum(0)]
    return {"forward": f, "dlogits": dz, "dip1": dh, "dpool2": dx, "dpool1": dp1, "dconv2": dc2, "dconv1": dc1,
            "g2": g2, "g1": g1, "grad": grads, "h": h, "xf": xf, "p1": p1, "dz_in": dzi, "dh_in": dhi}


def bounds(images, labels, w, relu, st, n_step=None):
    """per-stage error bounds of the device's float32 arithmetic for the stages of backward64(..., dev) (each on the
    device's own input), and of the eight gradients; n_step as backward64 (the bound of a step's gradient is the sum of
    its slices' bounds)"""
    C = images.shape[-1]
    n = n_step or len(labels)
    w1, b1, w2, b2, W1, B1, W2, B2 = arrays64(w, C)
    tiny = 2.0 ** -140
    dz, dh, h, xf, p1 = np.abs(st["dz_in"]), np.abs(st["dh_in"]), np.abs(st["h"]), np.abs(st["xf"]), np.abs(st["p1"])
    x = np.abs(st["forward"]["x"])
    dc2, dc1 = np.abs(st["dconv2"]), np.abs(st["dconv1"])
    pad = np.pad(dc2, ((0, 0), (0, 0), (4, 4), (4, 4)))
    out = {
        # rule 4: the device's expf / log1pf (2 and 1 ulp), the subtraction and the division: a few ulp of 1 / n
        "dlogits": np.full((n, 2), 16 * U / n) + tiny,
        "dip1": gamma(2) * (dz @ np.abs(W2).T) + tiny,
        "dpool2": gamma(500) * (dh @ np.abs(W1).T) + tiny,
        "dpool1": gamma(1250) * np.einsum("noyxij,ocij->ncyx", _win(pad), np.abs(w2)[:, :, ::-1, ::-1], optimize=True) + tiny,
    }
    out["grad"] = [
        gamma(784 + n) * np.einsum("noyx,ncyxij->ocij", dc1, _win(x), optimize=True).ravel() + tiny,
        gamma(784 + n) * dc1.sum((0, 2, 3)) + tiny,
        gamma(144 + n) * np.einsum("noyx,ncyxij->ocij", dc2, _win(p1), optimize=True).ravel() + tiny,
        gamma(144 + n) * dc2.sum((0, 2, 3)) + tiny,
        gamma(n) * (xf.T @ dh).ravel() + tiny,
        gamma(n) * dh.sum(0) + tiny,
        gamma(n) * (h.T @ dz).ravel() + tiny,
        gamma(n) * dz.sum(0) + tiny,
    ]
    return out


def step_grad_bounds(images, labels, w, relu, dev, slice_size=64):
    """(the eight float64 gradients of backward64(..., dev), their bounds) for a whole step, summed over slices of
    slice_size images: the float64 windows of a few hundred images would take gigabytes"""
    n = len(labels)
    ref, bnd = [0.0] * 8, [0.0] * 8
    for s in range(0, n, slice_size):
        sl = slice(s, s + slice_size)
        d = {k: np.asarray(v)[sl] for k, v in dev.items() if k != "grad"}
        st = backward64(images[sl], labels[sl], w, relu, d, n_step=n)
        b = bounds(images[sl], labels[sl], w, relu, st, n_step=n)
        ref = [r + g for r, g in zip(ref, st["grad"])]
        bnd = [r + g for r, g in zip(bnd, b["grad"])]
    return ref, bnd


def torch_grads64(images, labels, w, relu):
    """(loss, logits, the eight gradients in the .bin layouts) of the network in torch float64 autograd"""
    import torch
    import torch.nn.functional as Fn
    C = images.shape[-1]
    w1, b1, w2, b2, W1, B1, W2, B2 = arrays64(w, C)
    t = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float64, requires_grad=True)  # noqa: E731
    # fc1.weight[o][144 c + j] = ip1_w[o + 500 (c + 50 j)];  fc2.weight[o][k] = ip2_w[o + 2 k]
    fc1 = W1.reshape(144, 50, 500).transpose(2, 1, 0).reshape(500, 7200)
    P = [t(w1), t(b1), t(w2), t(b2), t(fc1), t(B1), t(W2.T), t(B2)]
    x = torch.tensor(chw(images))
    a = Fn.conv2d(x, P[0], P[1])
    a = Fn.max_pool2d(Fn.relu(a) if relu else a, 2, 2)
    a = Fn.conv2d(a, P[2], P[3])
    a = Fn.max_pool2d(Fn.relu(a) if relu else a, 2, 2)
    a = Fn.relu(Fn.linear(a.reshape(a.shape[0], -1), P[4], P[5]))
    z = Fn.linear(a, P[6], P[7])
    loss = torch.nn.CrossEntropyLoss()(z, torch.tensor(np.asarray(labels), dtype=torch.long))
    loss.backward()
    g = [p.grad.numpy() for p in P]
    g[4] = g[4].reshape(500, 50, 144).transpose(2, 1, 0).reshape(-1)
    g[6] = g[6].T
    return float(loss.detach()), z.detach().numpy(), [a.ravel() for a in g]


def random_net(C, seed, scale=1.0):
    """eight .bin arrays of a random network whose activations stay O(1) on 0..255 images"""
    rng = np.random.default_rng(seed)
    sizes = [20 * C * 25, 20, 25000, 50, 3600000, 500, 1000, 2]
    fan = [C * 25 * 255, 1, 500, 1, 7200, 1, 500, 1]
    return [(rng.standard_normal(s) * scale / np.sqrt(f)).astype(F) for s, f in zip(sizes, fan)]


def random_images(n, C, seed, ties=False):
    rng = np.random.default_rng(seed)
    im = rng.integers(0, 256, (n, 60, 60, C), dtype=np.uint8)
    if ties:  # flat patches: every pooling window over them ties, and the first maximum must win
        im[:, 10:40, 10:40, :] = 77
        im[:, :, 50:, :] = 0
    return im
