"""LeNet numerics off the shipped weights' scale: both implementations (lenet_impl 0 = wgmma with fp16 hi/lo split
operands, 1 = SIMT float32) against a plain float64 LeNet on the CPU.

The tensor-core path scales conv2's input and ip1's input into fp16 by powers of two derived from a bound on the
activations (lenet_tc.cu, safe_scale). Scaling conv1's weights and all four biases by 2^k scales every exact logit by
2^k (ReLU and max-pooling are positively homogeneous), so a correct choice of those scales makes the error relative to
max |logit| independent of k, and the tensor-core logits exactly 2^k times the unscaled ones.
"""
import os

import numpy as np
import pytest

from conftest import load_weights

# Largest error relative to max |logit| of the float64 reference, per implementation. Measured on one H100 80GB HBM3
# (400 W power limit) at k = 0, largest over the cases below: 2.5e-5 for lenet_impl 0 (the all-positive net at its
# activation bound; 1.7e-5 for the shipped 15-channel net) and 7.7e-7 for lenet_impl 1. Identical at every k.
REL_BOUND = {0: 4e-5, 1: 2e-6}


def lenet_reference(weights, images, relu_after_conv):
    """EigenClassifier's forward pass in float64 (torch on the CPU): conv1 -> [ReLU] -> max-pool 2x2 -> conv2 -> [ReLU] ->
    max-pool 2x2 -> ip1 + ReLU -> ip2. images [n, S, S, C] uint8 (the cv::Mat layout); weights in the .bin layout (conv
    OIHW row-major, ip matrices column-major (out, in), the flattened pool2 output indexed k = channel + 50 * pixel).
    Returns the logits [n, 2]."""
    import torch
    import torch.nn.functional as F

    w = [torch.from_numpy(np.asarray(a, dtype=np.float64)) for a in weights]
    C = images.shape[3]
    x = torch.from_numpy(np.ascontiguousarray(images)).permute(0, 3, 1, 2).to(torch.float64)
    h = F.conv2d(x, w[0].reshape(20, C, 5, 5), w[1])
    if relu_after_conv:
        h = F.relu(h)
    h = F.max_pool2d(h, 2)
    h = F.conv2d(h, w[2].reshape(50, 20, 5, 5), w[3])
    if relu_after_conv:
        h = F.relu(h)
    h = F.max_pool2d(h, 2)  # [n, 50, 12, 12]
    flat = h.reshape(h.shape[0], 50, -1).transpose(1, 2).reshape(h.shape[0], -1)  # k = c + 50 * j
    h3 = F.relu(flat @ w[4].reshape(-1, 500) + w[5])
    return (h3 @ w[6].reshape(500, 2) + w[7]).numpy()


@pytest.mark.parametrize("name,ch", [("lenet_caffe_15ch", 15), ("lenet_caffe_3ch", 3), ("lenet_ir_12ch", 12)])
def test_float64_reference_matches_reference_model_goldens(golden_dir, name, ch):
    """The float64 LeNet reproduces the logits the reference computed (float32) for its three shipped models."""
    g = np.load(os.path.join(golden_dir, name + ".npz"))
    w, relu = load_weights(ch)
    lo = lenet_reference(w, g["images"], relu)
    assert np.abs(lo - g["logits"]).max() <= 1e-5 * np.abs(g["logits"]).max()
    assert np.abs(lo).max() > 1.0


def _images(ch, n=256, seed=0):
    """Grasp-image-like inputs: sparse and dense random images plus all-0 and all-255 ones."""
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (n, 60, 60, ch), dtype=np.uint8)
    imgs[: n // 2] = ((rng.random((n // 2, 60, 60, ch)) < 0.2) * imgs[: n // 2]).astype(np.uint8)
    imgs[0] = 0
    imgs[1] = 255
    return imgs


def _scaled(w, k):
    """conv1 weights and the four biases times 2^k (exact in float32): every logit of the exact net times 2^k."""
    out = [np.array(a, dtype=np.float32, copy=True) for a in w]
    for i in (0, 1, 3, 5, 7):
        out[i] = np.ldexp(out[i], k).astype(np.float32)
    return out


def _classify(w, imgs, ch, relu, impl):
    from gpd_b200 import lib
    p = lib.default_params(channels=ch, relu_after_conv=relu, lenet_impl=impl)
    ctx = lib.Context(p)
    ctx.set_weights(w)
    logits = ctx.classify(imgs)[1]
    ctx.close()
    return logits


def _rel_err(lg, lo):
    assert np.isfinite(lg).all()
    err = float(np.abs(lg.astype(np.float64) - lo).max() / np.abs(lo).max())
    print(f"max |err| / max |logit| = {err:.3e}")
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("ch", [15, 12])  # 12: the ReLU net (relu_after_conv = 1)
def test_weight_scale_sweep_against_float64(ch):
    """Weight scales 2^k, k in {-20, -12, 0, 12, 20}: the error relative to max |logit| stays under REL_BOUND for both
    implementations, and the tensor-core logits are bit-exactly 2^k times the unscaled ones."""
    w, relu = load_weights(ch)
    assert relu == int(ch == 12)
    imgs = _images(ch, seed=ch)
    base = {}
    for k in (0, -20, -12, 12, 20):
        wk = _scaled(w, k)
        lo = lenet_reference(wk, imgs, relu)
        for impl in (0, 1):
            lg = _classify(wk, imgs, ch, relu, impl)
            err = _rel_err(lg, lo)
            assert err <= REL_BOUND[impl], (impl, k, err)
            if k == 0:
                base[impl] = lg
            elif impl == 0:
                assert np.array_equal(lg, np.ldexp(base[0], k).astype(np.float32)), k


def activations_at_the_bound():
    """The shipped 15-channel net with all-positive conv1 / conv2 weights and biases, and images of which 7 are all-255:
    (weights, images). test_gpu_lenet_layers.py checks the same case layer by layer."""
    w, _ = load_weights(15)
    w = [np.abs(a) if i < 4 else np.array(a) for i, a in enumerate(w)]
    imgs = _images(15, n=64, seed=3)
    imgs[2:8] = 255
    return w, imgs


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("relu", [0, 1])
def test_activations_at_the_bound(impl, relu):
    """All-positive conv1 / conv2 weights and biases with an all-255 image drive pool1 to exactly the bound the fp16
    activation scales are derived from (and pool2 close to its bound): the logits stay finite and match float64."""
    w, imgs = activations_at_the_bound()
    lo = lenet_reference(w, imgs, relu)
    lg = _classify(w, imgs, 15, relu, impl)
    assert _rel_err(lg, lo) <= REL_BOUND[impl]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [0, 1])
def test_zero_conv1_filter(impl):
    """A conv1 filter of zeros (its int8 digit planes use scale 1): that channel is its bias alone."""
    w, relu = load_weights(15)
    w = [np.array(a, dtype=np.float32, copy=True) for a in w]
    w[0].reshape(20, -1)[3] = 0.0
    w[0].reshape(20, -1)[17] = 0.0
    imgs = _images(15, n=128, seed=4)
    lo = lenet_reference(w, imgs, relu)
    assert _rel_err(_classify(w, imgs, 15, relu, impl), lo) <= REL_BOUND[impl]
