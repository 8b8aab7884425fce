"""The restatements of include/gpd_b200_train.h (tests/train_reference.py) on the CPU: the header's loss, d-logit and
optimiser helpers compiled for the host equal the numpy float32 restatement bit for bit; the float64 restatement of every
backward stage equals torch float64 autograd on the reference's network; the per-stage error bounds hold for exact
stages and catch emulated kernel faults; gpdb_write_weights_dir round-trips the .bin arrays
(through gpdb_load_weights_dir too in test_gpu_train.py)."""
import numpy as np
import pytest

import train_reference as tr
from conftest import load_weights
from gpd_b200 import lib, scenes

F = np.float32


def test_loss_and_dlogits_helpers_equal_the_restatement():
    rng = np.random.default_rng(0)
    z = np.concatenate([rng.standard_normal((300, 2)) * 5,
                        [[0, 0], [1, 1], [-3, -3], [0, 200], [200, 0], [-150, 150], [1e-30, -1e-30], [88, -88],
                         [0, 104], [0, 103.9]]]).astype(F)  # equal logits, and gaps where expf underflows
    for y in (np.zeros(len(z), np.int32), np.ones(len(z), np.int32), rng.integers(0, 2, len(z)).astype(np.int32)):
        for n in (1, len(z), 1000):
            loss, dz = tr.host_loss(z, y, n)
            assert np.array_equal(loss.view(np.uint32), tr.loss_f32(z, y).view(np.uint32))
            assert np.array_equal(dz.view(np.uint32), tr.dlogits_f32(z, y, n).view(np.uint32))
    # underflow: the larger logit's probability is exactly 1 and the other exactly 0
    loss, dz = tr.host_loss(np.array([[0, 200]], F), np.array([1], np.int32), 1)
    assert loss[0] == 0 and dz[0, 0] == 0 and dz[0, 1] == 0
    # against float64 where the arithmetic is benign
    zz, yy = z[:300], rng.integers(0, 2, 300).astype(np.int32)
    lse = np.logaddexp(zz[:, 0].astype(np.float64), zz[:, 1])
    assert np.allclose(tr.host_loss(zz, yy, 1)[0], lse - zz[np.arange(300), yy], rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("mu", [0.0, 0.9])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("lr", [0.0, 1e-3])
def test_sgd_helper_equals_the_restatement_over_steps(mu, wd, lr):
    rng = np.random.default_rng(1)
    p = rng.standard_normal(500).astype(F)
    ph, pn, bh, bn = p.copy(), p.copy(), np.zeros_like(p), np.zeros_like(p)
    for t in range(4):
        g = rng.standard_normal(500).astype(F)
        ph, bh = tr.host_sgd(ph, g, bh, lr, mu, wd, t == 0)
        pn, bn = tr.sgd_f32(pn, g, bn, lr, mu, wd, t == 0)
        assert np.array_equal(ph.view(np.uint32), pn.view(np.uint32)) and np.array_equal(bh.view(np.uint32), bn.view(np.uint32))
    if lr == 0:
        assert np.array_equal(ph, p)


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.5, 0.0)])
def test_adam_helper_equals_the_restatement_over_steps(wd, betas):
    rng = np.random.default_rng(2)
    p = rng.standard_normal(500).astype(F)
    h, nn_ = [p.copy(), np.zeros_like(p), np.zeros_like(p)], [p.copy(), np.zeros_like(p), np.zeros_like(p)]
    for t in range(1, 5):
        g = (rng.standard_normal(500) * 10.0 ** rng.integers(-6, 2, 500)).astype(F)
        h = list(tr.host_adam(*h[:1], g, *h[1:], 1e-3, betas[0], betas[1], 1e-8, wd, t))
        nn_ = list(tr.adam_f32(nn_[0], g, nn_[1], nn_[2], 1e-3, betas[0], betas[1], 1e-8, wd, t))
        for a, b in zip(h, nn_):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _check_vs_torch(images, labels, w, relu):
    st = tr.backward64(images, labels, w, relu)
    loss, z, g = tr.torch_grads64(images, labels, w, relu)
    assert np.allclose(st["forward"]["z"], z, rtol=1e-12, atol=1e-9)
    for i, (a, b) in enumerate(zip(st["grad"], g)):
        assert np.linalg.norm(a - b) <= 1e-10 * max(np.linalg.norm(b), 1e-300), i
    return st


@pytest.mark.parametrize("C", [1, 3, 12, 15])
@pytest.mark.parametrize("relu", [0, 1])
def test_backward_restatement_equals_torch_autograd(C, relu):
    w = tr.random_net(C, seed=C + 10 * relu)
    images = tr.random_images(3, C, seed=C, ties=True)
    st = _check_vs_torch(images, np.array([1, 0, 1]), w, relu)
    assert all(np.abs(a).max() > 0 for a in st["grad"])


def test_pooling_ties_take_the_first_maximum():
    """A flat image: every window of every pool ties, torch sends the gradient to position 0 of each window, and so
    does the restatement."""
    w = tr.random_net(3, seed=5)
    images = np.full((2, 60, 60, 3), 90, np.uint8)
    st = _check_vs_torch(images, np.array([0, 1]), w, 0)
    assert (st["forward"]["ch1"] == 0).all() and (st["forward"]["ch2"] == 0).all()


def test_shipped_net_layout_and_ip1_operand_order():
    """The shipped 3-channel net: the restatement's logits are those of the inference restatement
    (lenet_layer_bounds: k = c + 50 j), and torch with fc1 mapped from k = c + 50 j agrees; the transposed mapping does
    not."""
    import lenet_layer_bounds as lb
    w, relu = load_weights(3)
    images = tr.random_images(2, 3, seed=9)
    st = _check_vs_torch(images, np.array([0, 1]), w, relu)
    p1 = lb._t(st["forward"]["p1"])
    ref2, _ = lb.pool2(p1.numpy(), w, relu, 1)
    assert np.allclose(ref2.numpy(), st["forward"]["xf"], rtol=1e-12, atol=1e-12)
    wt = list(w)
    wt[4] = np.asarray(w[4]).reshape(50, 144, 500).transpose(1, 0, 2).reshape(-1)  # k = 144 c + j read as c + 50 j
    assert not np.allclose(tr.forward64(images, wt, relu)["z"], st["forward"]["z"], rtol=1e-6)


def _exceeds(dev, ref, bound):
    return bool((np.abs(np.asarray(dev, np.float64) - ref) > bound).any())


def test_bounds_hold_for_float32_stages_and_catch_faults():
    C, relu, n = 3, 1, 4
    w = tr.random_net(C, seed=3)
    images = tr.random_images(n, C, seed=4, ties=True)
    labels = np.array([0, 1, 1, 0])
    st = tr.backward64(images, labels, w, relu)
    b = tr.bounds(images, labels, w, relu, st)
    # stages rounded to float32 (one rounding each) stay inside their bounds
    for k in ("dlogits", "dip1", "dpool2", "dpool1"):
        assert not _exceeds(st[k].astype(F), st[k], b[k]), k
    for i in range(8):
        assert not _exceeds(st["grad"][i].astype(F), st["grad"][i], b["grad"][i]), i
    W1 = np.asarray(w[4], np.float64).reshape(7200, 500)
    # a dropped term: d pool2 without its largest product
    t = np.abs(st["dh_in"][0][None, :] * W1).argmax()
    k, o = np.unravel_index(t, W1.shape)
    bad = st["dpool2"].copy()
    bad[0, k] -= st["dh_in"][0, o] * W1[k, o]
    assert _exceeds(bad, st["dpool2"], b["dpool2"])
    # a missing 1 / n
    assert _exceeds(st["dlogits"] * n, st["dlogits"], b["dlogits"])
    # the ip1 operand order transposed: x read as k = 144 c + j
    xt = st["xf"].reshape(n, 144, 50).transpose(0, 2, 1).reshape(n, 7200)
    assert _exceeds((xt.T @ st["dh_in"]).ravel(), st["grad"][4], b["grad"][4])
    # a wrong pooling choice: one conv2 choice moved in every image
    dev = {"choice2": tr.flat(st["forward"]["ch2"]).copy()}
    j = np.abs(tr.flat(st["g2"])).argmax(1)
    dev["choice2"][np.arange(n), j] = (dev["choice2"][np.arange(n), j] + 1) % 4
    wrong = tr.backward64(images, labels, w, relu, dev)
    assert _exceeds(wrong["grad"][2], st["grad"][2], b["grad"][2])
    # a conv window shifted by one column: conv1 gradients against the image moved by one pixel
    x = st["forward"]["x"]
    xs = np.concatenate([x[..., 1:], x[..., :1]], -1)
    shifted = np.einsum("noyx,ncyxij->ocij", st["dconv1"], tr._win(xs), optimize=True).ravel()
    assert _exceeds(shifted, st["grad"][0], b["grad"][0])


@pytest.mark.parametrize("C", [1, 3, 12, 15])
def test_write_weights_dir_round_trips(tmp_path, C):
    w = load_weights(C)[0] if C != 1 else tr.random_net(1, seed=1)
    w = [np.asarray(a, F).ravel() for a in w]
    lib.write_weights_dir(tmp_path, C, w)
    back = scenes.load_weights_dir(str(tmp_path))
    for a, b in zip(w, back):
        assert a.tobytes() == b.tobytes()


def test_write_weights_dir_errors(tmp_path):
    w = tr.random_net(3, seed=0)
    with pytest.raises(lib.GpdbError, match=r"\[-1\]"):
        lib.write_weights_dir(tmp_path, 5, tr.random_net(5, seed=0))
    with pytest.raises(lib.GpdbError, match=r"\[-4\]"):
        lib.write_weights_dir(tmp_path / "missing", 3, w)
    with pytest.raises(ValueError):
        lib.write_weights_dir(tmp_path, 3, w[:7])
    import ctypes as C_
    assert lib.lib().gpdb_write_weights_dir(None, 3, None) == -1
    assert lib.lib().gpdb_write_weights_dir(str(tmp_path).encode(), 3, (C_.c_void_p * 8)()) == -1
