"""The per-layer LeNet error bounds (lenet_layer_bounds.py) have teeth: CPU tests, no device.

The arithmetic each implementation claims is emulated in float64 / numpy float16 on the inputs of the GPU layer tests:
conv1's 24-bit quantisation into three balanced int8 digits, conv2's and ip1's fp16 hi/lo splits at the library's
power-of-two scales with the lo * lo product dropped. The correct emulation stays within the bound at every element;
each emulated kernel fault exceeds it on at least one element. A bound that let one of these faults through would let
the same fault through on the device.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lenet_layer_bounds as B

C = 15
F16, F32 = np.float16, np.float32


# ---- emulation of the tensor-core arithmetic -----------------------------------------------------------------------------
def _digits(W):
    """Balanced base-256 digits of the integers W (least significant first), the top digit clamped to int8."""
    d2 = (W + 128) % 256 - 128
    W1 = (W - d2) // 256
    d1 = (W1 + 128) % 256 - 128
    return np.clip((W1 - d1) // 256, -128, 127), d1, d2


def quantised_conv1(w, s_o, drop_plane=False):
    """conv1 weights as the int8 tensor cores see them: s_o * (65536 d0 + 256 d1 + d2); drop_plane: without d2."""
    w = np.asarray(w, np.float64).reshape(20, -1)
    v = w / s_o[:, None]
    W = (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)  # lround
    d0, d1, d2 = _digits(W)
    if drop_plane:
        d2 = 0 * d2
    return ((65536 * d0 + 256 * d1 + d2) * s_o[:, None]).reshape(-1)


def _split(v):
    hi = np.asarray(v, F32).astype(F16)
    lo = (np.asarray(v, F32) - hi.astype(F32)).astype(F16)
    return torch.from_numpy(hi.astype(np.float64)), torch.from_numpy(lo.astype(np.float64))


def emu_pool1(images, w, relu, s_o, drop_plane=False, wrong_window=None):
    x = torch.from_numpy(np.ascontiguousarray(images)).permute(0, 3, 1, 2).to(torch.float64)
    wq = B._t(quantised_conv1(w[0], s_o, drop_plane)).reshape(20, images.shape[3], 5, 5)
    y = F.conv2d(x, wq, B._t(w[1]))
    if relu:
        y = F.relu(y)
    p = F.max_pool2d(y, 2)
    if wrong_window is not None:  # pooled element (c, py, px) reads the window's top-left element instead of the max
        c, py, px = wrong_window
        p[:, c, py, px] = y[:, c, 2 * py, 2 * px]
    return p.to(torch.float32).numpy()


def emu_pool2(p1, w, relu, sc, drop=None):
    """drop in {None, "wh_ah", "wl_ah", "wh_al"}: the conv2 product left out."""
    wh, wl = _split(np.asarray(w[2], F32).reshape(50, 20, 5, 5) * F32(sc["w2"]))
    ah, al = _split(np.asarray(p1, F32) * F32(sc["a2"]))
    terms = {"wh_ah": (ah, wh), "wl_ah": (ah, wl), "wh_al": (al, wh)}
    d = sum(F.conv2d(a, ww) for k, (a, ww) in terms.items() if k != drop)
    y = (d / (sc["a2"] * sc["w2"]) + B._t(w[3]).view(1, 50, 1, 1)).to(torch.float32).to(torch.float64)
    if relu:
        y = F.relu(y)
    xh, xl = _split(B._flat(F.max_pool2d(y, 2)).numpy() * sc["x3"])
    return ((xh + xl) / sc["x3"]).numpy()


def emu_ip1(p2, w, sc, drop=None, zero_unit=None):
    """drop in {None, "xl_wh", "xh_wl"}: the ip1 product left out (x_hi w_hi always stays)."""
    wh, wl = _split(np.asarray(w[4], F32).reshape(7200, 500) * F32(sc["w3"]))
    xh, xl = _split(np.asarray(p2, np.float64) * sc["x3"])
    terms = {"xh_wh": (xh, wh), "xl_wh": (xl, wh), "xh_wl": (xh, wl)}
    d = sum(x @ ww for k, (x, ww) in terms.items() if k != drop)
    h = F.relu(d / (sc["w3"] * sc["x3"]) + B._t(w[5])).to(torch.float32)
    if zero_unit is not None:
        h[:, zero_unit] = 0
    return h.numpy()


# ---- the inputs of the GPU layer tests, at a CPU-sized image count -------------------------------------------------------
@pytest.fixture(scope="module", params=[0, 1], ids=["relu0", "relu1"])
def case(request):
    relu = request.param
    w = B.probe_net(C, seed=100 + C)
    imgs = B.layer_images(C, n_dense=4, n_sparse=4, seed=C, impulses=False)
    imgs = np.concatenate([imgs, B.impulse_images(C, rows=(0, 16, 31, 59), cols=(0, 4, 55))])
    sc = B.tc_scales(w, C)
    ref1, bnd1 = B.pool1(imgs, w, relu, sc)
    return {"w": w, "imgs": imgs, "relu": relu, "sc": sc, "ref1": ref1, "bnd1": bnd1,
            "p1": emu_pool1(imgs, w, relu, sc["s_o"])}


def _ratio(got, ref, bnd):
    return B.compare("emulation", got, ref, bnd, ("i",) * np.ndim(got))[0]


def _with(w, i, fn):
    w = [np.array(a, F32, copy=True) for a in w]
    fn(w[i])
    return w


def test_correct_emulation_is_within_every_bound(case):
    w, relu, sc = case["w"], case["relu"], case["sc"]
    assert _ratio(case["p1"], case["ref1"], case["bnd1"][0]) <= 1.0
    p2 = emu_pool2(case["p1"], w, relu, sc)
    assert _ratio(p2, *B.pool2(case["p1"], w, relu, 0, sc)) <= 1.0
    h = emu_ip1(p2, w, sc)
    assert _ratio(h, *B.ip1(p2, w, 0, sc)) <= 1.0
    # the exact arithmetic is within the float32 bounds of lenet_impl 1 too
    assert _ratio(case["ref1"], case["ref1"], case["bnd1"][1]) == 0.0


def test_conv1_faults_exceed_the_bound(case):
    w, imgs, relu, sc = case["w"], case["imgs"], case["relu"], case["sc"]
    # 16-bit weights: the least significant digit plane dropped
    assert _ratio(emu_pool1(imgs, w, relu, sc["s_o"], drop_plane=True), case["ref1"], case["bnd1"][0]) > 1.0
    # filter 19 loses tap (4, 4) of every channel
    lost = _with(w, 0, lambda a: a.reshape(20, C, 5, 5).__setitem__((19, slice(None), 4, 4), 0))
    for impl in (0, 1):
        assert _ratio(emu_pool1(imgs, lost, relu, sc["s_o"]), case["ref1"], case["bnd1"][impl]) > 1.0, impl
    # pooled element (11, 11, 11) reads the top-left element of its window, not the max
    for impl in (0, 1):
        assert _ratio(emu_pool1(imgs, w, relu, sc["s_o"], wrong_window=(11, 11, 11)), case["ref1"], case["bnd1"][impl]) > 1.0


@pytest.mark.parametrize("drop", ["wh_ah", "wl_ah", "wh_al"])
def test_conv2_lost_product_exceeds_the_bound(case, drop):
    w, relu, sc, p1 = case["w"], case["relu"], case["sc"], case["p1"]
    assert _ratio(emu_pool2(p1, w, relu, sc, drop=drop), *B.pool2(p1, w, relu, 0, sc)) > 1.0


def test_conv2_lost_taps_exceed_the_bound(case):
    w, relu, sc, p1 = case["w"], case["relu"], case["sc"], case["p1"]
    tap = _with(w, 2, lambda a: a.reshape(50, 20, 5, 5).__setitem__((49, slice(None), 4, 4), 0))
    # the kw = 4 tap of channels 16..19, which plane 2 pairs with kw = 3 (c2_off)
    pair = _with(w, 2, lambda a: a.reshape(50, 20, 5, 5).__setitem__((slice(None), slice(16, 20), slice(None), 4), 0))
    for lost in (tap, pair):
        for impl in (0, 1):
            assert _ratio(emu_pool2(p1, lost, relu, sc), *B.pool2(p1, w, relu, impl, sc)) > 1.0, impl


@pytest.mark.parametrize("drop", ["xl_wh", "xh_wl"])
def test_ip1_lost_product_exceeds_the_bound(case, drop):
    w, relu, sc = case["w"], case["relu"], case["sc"]
    p2 = emu_pool2(case["p1"], w, relu, sc)
    assert _ratio(emu_ip1(p2, w, sc, drop=drop), *B.ip1(p2, w, 0, sc)) > 1.0


def test_ip1_zeroed_unit_exceeds_the_bound(case):
    w, relu, sc = case["w"], case["relu"], case["sc"]
    p2 = emu_pool2(case["p1"], w, relu, sc)
    for impl in (0, 1):
        assert _ratio(emu_ip1(p2, w, sc, zero_unit=499), *B.ip1(p2, w, impl, sc)) > 1.0, impl


def test_tiny_conv1_filters_need_the_stepped_scale():
    """max |w_o| = 5e-38: fl32(max / 8.3e6) is the subnormal 4 * 2^-149, max / s_o = 8.92e6 needs a top digit of 136,
    and the clamp to 127 leaves that weight ~7 % wrong, far out of the bound. The stepped scale stays within it."""
    rng = np.random.default_rng(3)
    w = B.probe_net(C, seed=3)
    f = w[0].reshape(20, -1)
    for o, mx in zip((5, 6, 7), (1e-36, 1e-37, 5e-38)):
        f[o] = (f[o] / np.abs(f[o]).max() * F32(mx)).astype(F32)
        w[1][o] = 0.0
    imgs = rng.integers(0, 256, (4, 60, 60, C), dtype=np.uint8)
    sc = B.tc_scales(w, C)
    ref, bnd = B.pool1(imgs, w, 0, sc)
    assert _ratio(emu_pool1(imgs, w, 0, sc["s_o"]), ref, bnd[0]) <= 1.0
    old = sc["s_o"].copy()
    old[5:8] = [float(F32(np.abs(f[o]).max() / 8300000.0)) for o in (5, 6, 7)]
    assert old[7] == 4 * 2.0 ** -149 and np.abs(f[7]).max() / old[7] > B.C1_W_MAX
    assert _ratio(emu_pool1(imgs, w, 0, old), ref, bnd[0]) > 1.0


# ---- the scale restatement against its documented rule --------------------------------------------------------------------
@pytest.mark.parametrize("bound", [1e-30, 3.7e-5, 1.0, 59999.0, 60000.0, 60001.0, 4.2e9, 1e30])
@pytest.mark.parametrize("w_scale", [2.0 ** -20, 1.0, 64.0, 2.0 ** 20])
def test_safe_scale_rule(bound, w_scale):
    s = B.safe_scale(bound, w_scale)
    j, we = math.log2(s), math.log2(w_scale)
    assert j == int(j) and -126 <= j <= 127 and abs(j + we) <= 120
    if -120 < j + we < 120 and -126 < j < 127:  # unclamped: the largest power of two that keeps scale * bound <= 60000
        assert s * bound <= 60000.0 < 2 * s * bound
    else:  # clamped: the clamp is the only reason to leave the rule
        free = 2.0 ** math.floor(math.log2(60000.0 / bound))
        assert (free > s and (j + we == 120 or j == 127)) or (free < s and (j + we == -120 or j == -126))


@pytest.mark.parametrize("mx", [0.17, 1e-3, 3e-30, 1.2e-36, 1e-36, 1e-37, 5e-38, 1e-39, 1e-44, 1.4e-45])
def test_conv1_scale_rule(mx):
    mx = float(F32(mx))
    s = B.conv1_scale(mx)
    assert s > 0 and float(F32(s)) == s
    assert mx / s <= B.C1_W_MAX  # no digit overflows
    below = float(np.nextafter(F32(s), F32(0)))
    assert below == 0 or mx / below > B.C1_W_MAX or s == float(F32(mx / 8300000.0))  # stepped no further than needed
    if mx >= 1e-30:
        assert s == float(F32(mx / 8300000.0))  # a normal scale is not moved
    p = B.pow2_scale(mx)  # conv2 / ip1 weight scale: clamped to the largest float32 power of two, never inf
    assert p * mx <= 16 and (16 < 2 * p * mx or p == 2.0 ** 127)
