"""Every LeNet layer of both implementations, element by element, against float64 (-m gpu).

gpdb_debug_lenet_layers returns what the device computed at each layer. Each layer is compared with a float64
reference of that layer applied to the device's own input to it, within a per-element bound derived from the
arithmetic the kernel claims to do (lenet_layer_bounds.py states the bounds and their derivations). The two
implementations are also compared with each other: their difference may not exceed the sum of their bounds plus how far
the layer moves under the difference of their inputs (sum |w| |dx|, ReLU and max-pooling being 1-Lipschitz).

Each case prints the largest err / bound per layer and implementation.
"""
import numpy as np
import pytest

import lenet_layer_bounds as B
from conftest import load_weights
from test_gpu_lenet_numerics import _scaled, activations_at_the_bound

pytestmark = pytest.mark.gpu

LAYERS = ("pool1", "pool2", "ip1", "logits")


def _device_layers(w, imgs, relu, impl):
    from gpd_b200 import lib
    ctx = lib.Context(lib.default_params(channels=imgs.shape[3], relu_after_conv=relu, lenet_impl=impl))
    try:
        ctx.set_weights(w)
        return ctx.lenet_layers(imgs)
    finally:
        ctx.close()


def check_layers(label, w, imgs, relu, coverage=False):
    """Runs both implementations on imgs and checks every layer against float64 and against each other. coverage: also
    assert that every pool1 channel, pool2 channel and ip1 unit is nonzero on some image (the case looked at every unit).
    Returns the device layers {impl: dict}."""
    C = imgs.shape[3]
    sc = B.tc_scales(w, C)
    dev = {impl: _device_layers(w, imgs, relu, impl) for impl in (0, 1)}
    ref1, bnd1 = B.pool1(imgs, w, relu, sc)
    fails, bounds, ratios = [], {}, {}
    for impl in (0, 1):
        d = dev[impl]
        checks = {"pool1": (ref1, bnd1[impl], B.P1_AXES)}
        checks["pool2"] = (*B.pool2(d["pool1"], w, relu, impl, sc), B.P2_AXES)
        checks["ip1"] = (*B.ip1(d["pool2"], w, impl, sc), B.IP_AXES)
        checks["logits"] = (*B.logits(d["ip1"], w), B.LOGIT_AXES)
        for layer in LAYERS:
            ref, bnd, axes = checks[layer]
            bounds[impl, layer] = bnd
            r, msg = B.compare(f"{label} lenet_impl {impl} {layer}", d[layer], ref, bnd, axes)
            ratios[impl, layer] = r
            if not r <= 1.0:
                fails.append(msg)
    # the two implementations against each other
    w_of = {"pool2": w[2].reshape(50, 20, 5, 5), "ip1": w[4].reshape(7200, 500), "logits": w[6].reshape(500, 2)}
    prev = {"pool2": "pool1", "ip1": "pool2", "logits": "ip1"}
    for layer, axes in zip(LAYERS, (B.P1_AXES, B.P2_AXES, B.IP_AXES, B.LOGIT_AXES)):
        tol = bounds[0, layer] + bounds[1, layer]
        if layer in prev:
            dx = B._t(dev[0][prev[layer]]) - B._t(dev[1][prev[layer]])
            tol = tol + (B._flat(B.conv_lipschitz(dx, w_of[layer])) if layer == "pool2" else dx.abs() @ B._t(w_of[layer]).abs())
        r, msg = B.compare(f"{label} lenet_impl 0 - 1 {layer}", dev[0][layer], B._t(dev[1][layer]), tol, axes)
        ratios["0-1", layer] = r
        if not r <= 1.0:
            fails.append(msg)
    print(f"{label}: max err / bound  " + "  ".join(
        f"[{impl}] " + " ".join(f"{layer} {ratios[impl, layer]:.3g}" for layer in LAYERS) for impl in (0, 1, "0-1")))
    assert not fails, "\n".join(fails)
    if coverage:
        for impl in (0, 1):
            d = dev[impl]
            dead1 = np.flatnonzero(~(d["pool1"] != 0).any(axis=(0, 2, 3)))
            dead2 = np.flatnonzero(~(d["pool2"].reshape(-1, 144, 50) != 0).any(axis=(0, 1)))
            dead3 = np.flatnonzero(~(d["ip1"] != 0).any(axis=0))
            assert dead1.size == dead2.size == dead3.size == 0, (
                f"{label} lenet_impl {impl}: never nonzero on these images: pool1 channels {dead1.tolist()}, pool2 "
                f"channels {dead2.tolist()}, ip1 units {dead3.tolist()}")
    return dev


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("C", [1, 3, 12, 15])
def test_layers_random_net(C, relu):
    """A random-init net with the two single-weight probes (conv2 filter 0, ip1 unit 0), on dense, sparse, flat and
    impulse images; every unit of the net is seen nonzero."""
    # seed 101 would leave two ip1 units of the 1-channel ReLU net below zero on every image; with 105 each unit of
    # both 1-channel nets reaches > 1e-3 of the largest ip1 output (float64 on the CPU), far above the rounding
    w = B.probe_net(C, seed=105 if C == 1 else 100 + C)
    check_layers(f"random C={C} relu={relu}", w, B.layer_images(C, seed=C), relu, coverage=True)


@pytest.mark.parametrize("C", [15, 3, 12])
def test_layers_shipped_net(C):
    w, relu = load_weights(C)
    check_layers(f"shipped C={C} relu={relu}", w, B.layer_images(C, seed=C), relu)


def edge_net(C=15, seed=5):
    """conv1 filters at the edges of the 24-bit quantisation, conv2 / ip1 weights spanning 2^-20 .. 1 (fp16 lo parts
    subnormal at the library's scales)."""
    rng = np.random.default_rng(seed)
    w = B.probe_net(C, seed)
    f = w[0].reshape(20, C * 25)
    f[0] *= 1e-4
    f[0, 37] = 0.04                                        # one weight 1e4 x larger than the rest
    f[1] = np.where(rng.random(C * 25) < 0.5, -0.05, 0.05)  # every weight +-max
    f[2] = 0.05                                            # every weight +max: top digit 127 everywhere
    f[3, 100] = -2 * np.abs(f[3]).max()                    # the largest weight negative
    f[4] = 0.0                                             # a zero filter
    for o, mx in zip((5, 6, 7), (1e-36, 1e-37, 5e-38)):    # subnormal conv1 scales s_o
        f[o] = (f[o] / np.abs(f[o]).max() * np.float32(mx)).astype(np.float32)
        w[1][o] = 0.0
    for i in (2, 4):
        sign = np.where(rng.random(w[i].size) < 0.5, -1.0, 1.0)
        span = np.ldexp(1.0, -rng.integers(0, 21, w[i].size)) * (1 + rng.random(w[i].size))
        keep = w[i] != 0  # the probes stay single weights
        w[i] = np.where(keep, sign * span / 2, 0.0).astype(np.float32)
    w[2].reshape(50, 500)[0, 0 * 25 + 12] = B.PROBE_W
    w[4].reshape(7200, 500)[B.PROBE_K, 0] = B.PROBE_W
    return w


@pytest.mark.parametrize("relu", [0, 1])
def test_layers_weight_edges(relu):
    """Large, +-max, negative-max, zero and tiny (max |w| 1e-36, 1e-37, 5e-38) conv1 filters; conv2 and ip1 weights from
    2^-20 to 1. The tiny filters have zero bias, so pool1 shows their weights alone."""
    w = edge_net()
    sc = B.tc_scales(w, 15)
    assert sc["s_o"][5:8].max() < 2.0 ** -126  # the conv1 scales of the tiny filters are subnormal
    check_layers(f"weight edges relu={relu}", w, B.layer_images(15, seed=21), relu)


@pytest.mark.parametrize("relu", [0, 1])
def test_layers_at_the_activation_bound(relu):
    """The all-positive net of test_activations_at_the_bound: pool1 at exactly the bound the fp16 scales come from."""
    w, imgs = activations_at_the_bound()
    check_layers(f"activation bound relu={relu}", w, imgs, relu)


@pytest.mark.parametrize("k", [-124, 112])
@pytest.mark.parametrize("C", [15, 12])
def test_layers_weight_scale_clamp(C, k):
    """conv1 weights and all biases times 2^k (as test_weight_scale_sweep_against_float64) at the exponents where
    safe_scale's clamp |j + log2 w_scale| <= 120 engages (k = -124: the activation scale 2^j would need j + log2 w2_scale
    above 120), and, at k = -124, conv1 scales s_o in the float32 subnormals."""
    w0, relu = load_weights(C)
    w = _scaled(w0, k)
    sc = B.tc_scales(w, C)
    clamped = [np.log2(sc["a2"] * sc["w2"]), np.log2(sc["x3"] * sc["w3"])]
    if k < 0:
        assert max(clamped) == 120, clamped
        assert sc["s_o"].min() < 2.0 ** -126
    check_layers(f"C={C} relu={relu} weights x 2^{k}", w, B.layer_images(C, seed=C, impulses=False), relu)


@pytest.mark.parametrize("layer", [2, 4])
def test_layers_tiny_conv2_or_ip1_weights(layer):
    """conv2 (layer 2) or ip1 (layer 4) weights times 2^-130 (max |w| ~ 1e-40, float32 subnormals), conv1 weights and
    the biases before them times 2^100 so that the activations stay normal: the fp16 weight scale 16 / max |w| overflows
    float32 and is held to 2^127."""
    w0, relu = load_weights(15)
    e = [100, 100, 0, 100, 0, -30, 0, -30] if layer == 4 else [100, 100, 0, -30, 0, -30, 0, -30]
    e[layer] = -130
    w = [np.ldexp(np.asarray(a, np.float32), k).astype(np.float32) for a, k in zip(w0, e)]
    assert np.abs(w[layer]).max() < 2.0 ** -126 and B.tc_scales(w, 15)["w2" if layer == 2 else "w3"] == 2.0 ** 127
    check_layers(f"weights of layer {layer} x 2^-130", w, B.layer_images(15, seed=layer, impulses=False), relu)


def test_layers_batch_shapes():
    """n = 2 x SMs + 3 against float64; the first 1, 127, 128, 129 of those images as their own batch give bit-equal
    layers (ip1's 128-image tiles with the padded outputs 500..511, the unequal grid-stride shares of conv1 / conv2)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    C, relu = 15, 0
    w = B.probe_net(C, seed=7)
    base = B.layer_images(C, seed=7)
    rng = np.random.default_rng(8)
    n = 2 * sms + 3
    extra = rng.integers(0, 256, (n - len(base), 60, 60, C), dtype=np.uint8)
    imgs = np.concatenate([base, extra])[:n]
    full = check_layers(f"batch of {n}", w, imgs, relu)
    for impl in (0, 1):
        for m in (1, 127, 128, 129):
            part = _device_layers(w, imgs[:m], relu, impl)
            for layer in LAYERS:
                assert np.array_equal(part[layer], full[impl][layer][:m]), (impl, m, layer)
