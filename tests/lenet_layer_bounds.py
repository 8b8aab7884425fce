"""Float64 references and per-element error bounds of every LeNet layer, for both implementations (lenet_impl 0: conv1
on int8 tensor cores, conv2 / ip1 on fp16 hi/lo tensor cores, lenet_tc.cu; lenet_impl 1: float32 FMA chains,
lenet_simt.cu). Shared by test_lenet_layer_bounds.py (CPU: the bounds catch emulated kernel faults) and
test_gpu_lenet_layers.py (the device's layers against them).

Every layer is checked on the device's own input to it: pool1 from the uint8 images, pool2 from the device's pool1, ip1
from the device's pool2, the logits from the device's ip1. Errors then do not compound, and a bound speaks about one
kernel.

Notation, for one output element y = sum_i w_i x_i + b before ReLU and pooling:
  u = 2^-24 (float32 unit roundoff), gamma(m) = m u / (1 - m u);
  A = sum |w_i x_i|;  m = #{i : w_i x_i != 0}: adding an exact zero rounds nothing, so only the m nonzero products
  count (for a dense layer m is the reduction length K: 25 C, 500, 7 200);
  Sx = sum of |x_i| over w_i != 0,  Sw = sum of |w_i| over x_i != 0.
ReLU and max-pooling are 1-Lipschitz, so the bound of a pooled element is the max of its window's bounds.

lenet_impl 1 (float32): every product w_i x_i enters one FMA (one rounding), the bias one add:
  |err| <= gamma(m + 1) (A + |b|) + (m + 1) 2^-150                      [m + 1 roundings of partial sums <= A + |b|]
Every float32 rounding also errs by at most 2^-150 in absolute terms (a result in the subnormal range): the 2^-150
terms, which only matter for weights scaled down to ~1e-38.

pool1, lenet_impl 0: W_i = round(w_i / s_o) exactly, |s_o W_i - w_i| <= s_o / 2, and the int32 dot products are exact.
  The epilogue recombines the three digit sums with two float32 FMAs (two roundings, each of a value <= 1.01 A / s_o: the
  low two digits of W, |256 d1 + d2| <= 32 896, exceed |W| by < 1 %) and applies scale and bias with one more:
  |err| <= s_o / 2 * Sx + C1 u (A + |b|) + 3 * 2^-150,   C1 = 4 >= 1.01 + 1.01 + 1 (+ slack for the quantised A).

conv2 / ip1, lenet_impl 0: operands scaled by powers of two (exact) W = s_w w, X = s_x x, split W = Wh + Wl + eW with
  Wh = fp16(W), Wl = fp16(W - Wh): |eW| <= 2^-22 |W| + 2^-25 (the second term when Wl is an fp16 subnormal),
  |Wl| <= 2^-11 |W| + 2^-25; likewise X. The kernels sum Wh Xh + Wl Xh + Wh Xl (products of fp16 are exact in fp32),
  dropping Wl Xl:  WX - that = eW X + W eX - eW eX + Wl Xl, so per product, unscaled by 1 / (s_w s_x):
  |err_i| <= C2 2^-22 |w_i x_i| + 1.001 * 2^-25 (|x_i| / s_w + |w_i| / s_x) + 2^-49 / (s_w s_x),   C2 = 3.01
  (three terms of 2^-22 |WX| each, times (1 + 2^-11)^2, and the cross terms of the absolute parts).
  The 3 m nonzero products are accumulated in float32: gamma(3 m) * 1.001 A + 3 m 2^-150 / (s_w s_x).
  conv2's epilogue adds the bias in float32 (u (A + |b|)) and writes ip1's operand as an fp16 hi/lo pair of the scaled
  value (2^-22 |y| + 2^-25 / x3_scale); the device's pool2 IS that operand, so ip1's X split is exact (eX = 0, bounded
  anyway by the same formula). ip1's epilogue adds its two accumulators and the bias: 2 u (A + |b|). 3 * 2^-150 for the
  epilogue's roundings.

logits (both): k_ip2 sums 500 FMAs per logit over a lane split and a shuffle tree:  gamma(500) sum |w h| + u |b|.

Whether the wgmma float32 accumulation rounds like IEEE float32 is an assumption of the gamma terms, not a measurement.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
C1 = 4.0
C2 = 3.01
C1_W_MAX = 127.0 * 65536 + 127.0 * 257  # largest |W| of three balanced int8 digits with the top digit <= 127


def gamma(m):
    m = torch.as_tensor(m, dtype=torch.float64)
    return m * U / (1.0 - m * U)


# ---- the tensor-core scales (lenet_tc_upload), restated ----------------------------------------------------------------
def pow2_scale(maxabs, target=16.0):
    """2^floor(log2(target / maxabs)) in float32; 1 for an all-zero layer, 2^127 where target / maxabs overflows."""
    maxabs = float(np.float32(maxabs))
    if not maxabs > 0.0:
        return 1.0
    with np.errstate(over="ignore"):
        q = np.float32(target) / np.float32(maxabs)
    if np.isinf(q):
        return 2.0 ** 127
    return float(np.float32(2.0 ** math.floor(math.log2(float(q)))))


def safe_scale(bound, w_scale):
    """The largest 2^j with 2^j * bound <= 60000, held to |j + log2 w_scale| <= 120 and to a float32 exponent."""
    we = math.frexp(w_scale)[1] - 1
    lo, hi = max(-126, -120 - we), min(127, 120 - we)
    if not bound > 0.0:
        return 2.0 ** max(lo, min(hi, 0))
    j = math.floor(math.log2(60000.0 / bound))
    while j > lo and 2.0 ** j * bound > 60000.0:
        j -= 1
    while j < hi and 2.0 ** (j + 1) * bound <= 60000.0:
        j += 1
    return 2.0 ** max(lo, min(hi, j))


def conv1_scale(mxo):
    """s_o of one conv1 filter: fl32(max|w_o| / 8.3e6), stepped up until no weight needs more than the three digits."""
    mxo = float(np.float32(mxo))
    if not mxo > 0.0:
        return 1.0
    so = np.float32(mxo / 8300000.0)
    while so == 0 or mxo / float(so) > C1_W_MAX:
        so = np.nextafter(so, np.float32(np.inf))
    return float(so)


def tc_scales(w, C):
    """The scales lenet_tc_upload derives from the weights (the .bin layout): s_o [20], w2, a2, w3, x3."""
    w1 = np.abs(np.asarray(w[0], np.float64)).reshape(20, C * 25)
    s_o = np.array([conv1_scale(np.float32(np.abs(np.asarray(w[0], np.float32)).reshape(20, -1)[o].max())) for o in range(20)])
    a1 = float(np.max(w1.sum(1) * 255.0 + np.abs(np.asarray(w[1], np.float64))))
    a2 = float(np.max(np.abs(np.asarray(w[2], np.float64)).reshape(50, 500).sum(1) * a1 + np.abs(np.asarray(w[3], np.float64))))
    w2 = pow2_scale(np.abs(np.asarray(w[2], np.float32)).max())
    w3 = pow2_scale(np.abs(np.asarray(w[4], np.float32)).max())
    return {"s_o": s_o, "w2": w2, "a2": safe_scale(a1, w2), "w3": w3, "x3": safe_scale(a2, w3), "a1_bound": a1, "a2_bound": a2}


# ---- layers: float64 value and the statistics of the bounds -------------------------------------------------------------
def _t(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.float64)


def _conv_stats(x, wt, b):
    """x [n, Cin, H, W], wt [O, Cin, 5, 5] float64 tensors: y (with bias), A, m, Sx, Sw at every output pixel."""
    nzx, nzw = (x != 0).double(), (wt != 0).double()
    ax, aw = x.abs(), wt.abs()
    return {"y": F.conv2d(x, wt, b), "A": F.conv2d(ax, aw), "m": F.conv2d(nzx, nzw), "Sx": F.conv2d(ax, nzw),
            "Sw": F.conv2d(nzx, aw)}


def _pool(t):
    return F.max_pool2d(t, 2)


def _flat(h):
    """[n, 50, 12, 12] -> [n, 7200], k = c + 50 j."""
    return h.reshape(h.shape[0], 50, -1).transpose(1, 2).reshape(h.shape[0], -1)


def _tc_gemm_bound(s, s_w, s_x):
    return ((C2 * 2.0 ** -22 + 1.001 * gamma(3 * s["m"])) * s["A"] + 1.001 * 2.0 ** -25 * (s["Sx"] / s_w + s["Sw"] / s_x)
            + s["m"] * (2.0 ** -49 + 3 * 2.0 ** -150) / (s_w * s_x) + 3 * 2.0 ** -150)


def pool1(images, w, relu, scales):
    """images [n, 60, 60, C] uint8 -> (reference, {lenet_impl: bound}), each [n, 20, 28, 28] float64 (the input is the
    same for both implementations)."""
    C = images.shape[3]
    x = torch.from_numpy(np.ascontiguousarray(images)).permute(0, 3, 1, 2).to(torch.float64)
    b = _t(w[1])
    s = _conv_stats(x, _t(w[0]).reshape(20, C, 5, 5), b)
    ab = b.abs().view(1, 20, 1, 1)
    so = _t(scales["s_o"]).view(1, 20, 1, 1)
    e = {1: gamma(s["m"] + 1) * (s["A"] + ab) + (s["m"] + 1) * 2.0 ** -150,
         0: so / 2 * s["Sx"] + C1 * U * (s["A"] + ab) + 3 * 2.0 ** -150}
    y = F.relu(s["y"]) if relu else s["y"]
    return _pool(y), {k: _pool(v) for k, v in e.items()}


def pool2(p1, w, relu, impl, scales=None):
    """p1 [n, 20, 28, 28] (the device's pool1) -> (reference, bound), each [n, 7200] float64."""
    b = _t(w[3])
    s = _conv_stats(_t(p1), _t(w[2]).reshape(50, 20, 5, 5), b)
    ab = b.abs().view(1, 50, 1, 1)
    if impl == 1:
        e = gamma(s["m"] + 1) * (s["A"] + ab) + (s["m"] + 1) * 2.0 ** -150
    else:
        e = _tc_gemm_bound(s, scales["w2"], scales["a2"]) + (U + 1.001 * 2.0 ** -22) * (s["A"] + ab)
    y = F.relu(s["y"]) if relu else s["y"]
    e = _pool(e)
    if impl == 0:
        e = e + 2.0 ** -25 / scales["x3"]
    return _flat(_pool(y)), _flat(e)


def ip1(p2, w, impl, scales=None):
    """p2 [n, 7200] (the device's pool2) -> (reference, bound), each [n, 500] float64 (ReLU applied)."""
    x, W, b = _t(p2), _t(w[4]).reshape(7200, 500), _t(w[5])
    nzx, nzw = (x != 0).double(), (W != 0).double()
    s = {"y": x @ W + b, "A": x.abs() @ W.abs(), "m": nzx @ nzw, "Sx": x.abs() @ nzw, "Sw": nzx @ W.abs()}
    if impl == 1:
        e = gamma(s["m"] + 1) * (s["A"] + b.abs()) + (s["m"] + 1) * 2.0 ** -150
    else:
        e = _tc_gemm_bound(s, scales["w3"], scales["x3"]) + 2 * U * (s["A"] + b.abs())
    return F.relu(s["y"]), e


def logits(h, w):
    """h [n, 500] (the device's ip1) -> (reference, bound), each [n, 2] float64."""
    h, W, b = _t(h), _t(w[6]).reshape(500, 2), _t(w[7])
    return h @ W + b, gamma(500) * (h.abs() @ W.abs()) + U * b.abs() + 501 * 2.0 ** -150


# ---- Lipschitz propagation of an input difference (cross-implementation checks) -----------------------------------------
def conv_lipschitz(dx, wt):
    """max-pooled sum |w| |dx|: how far a conv + bias (+ReLU) + pool moves when its input moves by dx."""
    return _pool(F.conv2d(_t(dx).abs(), _t(wt).abs()))


def compare(name, got, ref, bound, index_names):
    """(max err / bound, message naming the worst element) of got against ref; bound > 0 everywhere it matters."""
    got, ref, bound = _t(got), _t(ref), _t(bound)
    if not torch.isfinite(got).all():
        bad = np.unravel_index(int(torch.argmax((~torch.isfinite(got)).int())), tuple(got.shape))
        return math.inf, f"{name}: non-finite value at {dict(zip(index_names, bad))}"
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    i = int(torch.argmax(ratio))
    idx = np.unravel_index(i, tuple(ratio.shape))
    where = ", ".join(f"{k} {v}" for k, v in zip(index_names, idx))
    r = float(ratio.flatten()[i])
    msg = (f"{name}: {where}: device {float(got.flatten()[i]):.9g}, reference {float(ref.flatten()[i]):.9g}, "
           f"err {float(err.flatten()[i]):.3g} / bound {float(bound.flatten()[i]):.3g} = {r:.3g}")
    return r, msg


P1_AXES = ("image", "channel", "y", "x")
P2_AXES = ("image", "k (= channel + 50 * pixel)")
IP_AXES = ("image", "unit")
LOGIT_AXES = ("image", "logit")


# ---- inputs -------------------------------------------------------------------------------------------------------------
# Impulse positions (one pixel of 255 in every channel, input row, column). An impulse at (Y, X) reaches conv1 outputs
# Y-4..Y x X-4..X. Columns 3, 4: conv1 output x 0..3 of a tile's second row sit in GEMM rows 60..63, the rest of that
# row in the other warpgroup (rows 64..); 55, 59: the last valid output column. Rows 15..17, 29..33, 45..47: conv2's tiles
# are its output rows 8T..8T+7 over pool1 rows 8T..8T+11 (input rows 16T..16T+27), so these impulses land in a tile's
# last rows, its 4 halo rows and the next tile's first rows; and they straddle conv1's two-row tiles either way.
IMPULSE_ROWS = (0, 4, 15, 16, 17, 29, 30, 31, 32, 33, 47, 59)
IMPULSE_COLS = (0, 3, 4, 30, 55, 59)


def impulse_images(C, rows=IMPULSE_ROWS, cols=IMPULSE_COLS):
    imgs = np.zeros((len(rows) * len(cols), 60, 60, C), np.uint8)
    for i, (y, x) in enumerate((y, x) for y in rows for x in cols):
        imgs[i, y, x, :] = 255
    return imgs


def layer_images(C, n_dense=12, n_sparse=12, seed=0, impulses=True):
    """Dense random images, sparse ones (20 % of the pixels nonzero), all-0, all-255 and the impulse images."""
    rng = np.random.default_rng(seed)
    dense = rng.integers(0, 256, (n_dense, 60, 60, C), dtype=np.uint8)
    sparse = (rng.integers(0, 256, (n_sparse, 60, 60, C)) * (rng.random((n_sparse, 60, 60, C)) < 0.2)).astype(np.uint8)
    flat = np.stack([np.zeros((60, 60, C), np.uint8), np.full((60, 60, C), 255, np.uint8)])
    parts = [dense, sparse, flat] + ([impulse_images(C)] if impulses else [])
    return np.concatenate(parts)


# a weight whose fp16 lo part is as large as it gets relative to the weight: 0.9 * 2^-11 (at any power-of-two scale)
PROBE_W = float(np.float32(0.125 * (1.0 + 0.9 * 2.0 ** -11)))
PROBE_K = 1 + 50 * 78  # ip1 input k = channel 1 of pool2 pixel (6, 6)


def probe_net(C, seed):
    """random_lenet_weights with two probes: conv2 filter 0 and ip1 unit 0 each keep a single weight, PROBE_W, so that
    their error is that of one product and a lost hi/lo product term stands out of the bound."""
    from gpd_b200 import scenes
    w = [np.array(a, np.float32, copy=True) for a in scenes.random_lenet_weights(C, seed=seed)]
    f0 = w[2].reshape(50, 20, 5, 5)[0]
    f0[:] = 0
    f0[0, 2, 2] = PROBE_W
    W = w[4].reshape(7200, 500)
    W[:, 0] = 0
    W[PROBE_K, 0] = PROBE_W
    w[5][0] = 0.01
    return w

